"""A stand-in worker process for the CPU tests of fold maps on fiber_b200.procpool (host logic only: block totals placed in
block order, the fold of the totals sent to one live worker, re-queues after deaths).  It speaks the worker protocol with an
order-sensitive integer "combine" (acc * 31 + x mod 2^64) in place of a device body -- test infrastructure, never used by
the product (the real worker is ``procpool.gpu_worker_main``)."""
import os
import pickle
import sys

import numpy as np

M64 = (1 << 64) - 1


def combine(a, b):
    return (a * 31 + b) & M64


def tree(xs):
    xs = list(xs)
    while len(xs) > 1:
        nxt = [combine(xs[2 * i], xs[2 * i + 1]) for i in range(len(xs) // 2)]
        if len(xs) % 2:
            nxt.append(xs[-1])
        xs = nxt
    return xs[0]


def fake_fold_worker_main(device, conn, results, sys_path):
    for p in sys_path:
        if p not in sys.path:
            sys.path.insert(0, p)
    from fiber_b200.procpool import SharedSegment
    segs = {}
    conn.send(("ready", os.getpid()))
    while True:
        msg = conn.recv()
        if msg is None:
            break
        if msg[0] == "fold":
            _, job, n_blocks, body, shm_name, module = msg
            mark = os.environ.get("FBR_TEST_FOLD_MARK")
            if body == "fold_dies_once" and mark and not os.path.exists(mark):
                open(mark, "w").close()
                os._exit(3)                              # dies while folding the totals, without a word
            if body == "fold_always_dies":
                os._exit(3)
            seg = segs.get(shm_name) or segs.setdefault(shm_name, SharedSegment(shm_name))
            totals = np.array(seg.array[8:8 * (1 + n_blocks)]).view(np.uint64).tolist()
            seg.array[:8] = np.array([tree(totals)], np.uint64).view(np.uint8)
            conn.send(("folded", job))
            continue
        _, job, blk, body, kind, chunksize, payload, shm_name, off, attempt, module = msg
        items = range(*payload[1]) if payload[0] == "range" else pickle.loads(payload[1])
        xs = [int(x) for x in items]
        if attempt == 0 and 0xDEAD in xs:
            os._exit(3)                                  # the worker process dies mid-block
        seg = segs.get(shm_name) or segs.setdefault(shm_name, SharedSegment(shm_name))
        seg.array[off:off + 8] = np.array([tree(xs)], np.uint64).view(np.uint8)
        conn.send(("done", job, blk, None))
    os._exit(0)
