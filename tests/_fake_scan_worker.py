"""A stand-in worker process for the CPU tests of accumulate maps on fiber_b200.procpool (host logic only: each block's own
prefix folds placed by index, the wrap of blocks 1, 2, ... sent to one live worker with the block totals, re-sends after
deaths).  It speaks the worker protocol with the order-sensitive integer "combine" of _fake_fold_worker (acc * 31 + x mod
2^64) in place of a device body -- test infrastructure, never used by the product (the real worker is
``procpool.gpu_worker_main``)."""
import os
import pickle
import sys

import numpy as np

from ._fake_fold_worker import combine, tree


def prefix_folds(xs):
    """tree(xs[0..i]) for every i, by the pieces of [0, i) (levels of complete aligned subtrees), as the device computes it."""
    lv = [list(xs)]
    while len(lv[-1]) >= 2:
        prev = lv[-1]
        lv.append([combine(prev[2 * j], prev[2 * j + 1]) for j in range(len(prev) // 2)])
    out = []
    for i, acc in enumerate(xs):
        k = 0
        while i >> k:
            if (i >> k) & 1:
                acc = combine(lv[k][(i >> k) - 1], acc)
            k += 1
        out.append(acc)
    return out


def fake_scan_worker_main(device, conn, results, sys_path):
    for p in sys_path:
        if p not in sys.path:
            sys.path.insert(0, p)
    from fiber_b200.procpool import SharedSegment, _scan_pieces
    segs = {}
    conn.send(("ready", os.getpid()))
    while True:
        msg = conn.recv()
        if msg is None:
            break
        if msg[0] == "scan":
            _, job, ranges, todo, totals, body, shm_name, module = msg
            tot = np.frombuffer(totals, np.uint64).tolist()
            seg = segs.get(shm_name) or segs.setdefault(shm_name, SharedSegment(shm_name))
            mark = os.environ.get("FBR_TEST_SCAN_MARK")
            for b in todo:
                if body == "scan_dies_once" and mark and not os.path.exists(mark) and b == 2:
                    open(mark, "w").close()
                    os._exit(3)                          # dies half-way through the wraps, without a word
                if body == "scan_always_dies":
                    os._exit(3)
                lo, hi = ranges[b]
                pieces = _scan_pieces(lambda a, c: tree(tot[a:a + c]), tot, b)
                recs = np.array(seg.array[lo * 8:hi * 8]).view(np.uint64).tolist()
                for i, r in enumerate(recs):
                    for g in reversed(pieces):
                        r = combine(g, r)
                    recs[i] = r
                seg.array[lo * 8:hi * 8] = np.array(recs, np.uint64).view(np.uint8)
                conn.send(("scanned", job, b))
            conn.send(("folded", job))
            continue
        _, job, blk, body, kind, chunksize, payload, shm_name, off, attempt, module = msg
        items = range(*payload[1]) if payload[0] == "range" else pickle.loads(payload[1])
        xs = [int(x) for x in items]
        if attempt == 0 and 0xDEAD in xs:
            os._exit(3)                                  # the worker process dies mid-block
        seg = segs.get(shm_name) or segs.setdefault(shm_name, SharedSegment(shm_name))
        ys = np.array(prefix_folds(xs), np.uint64).view(np.uint8)
        seg.array[off:off + ys.nbytes] = ys
        conn.send(("done", job, blk, None))
    os._exit(0)
