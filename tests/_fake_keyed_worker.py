"""A stand-in worker process for the CPU tests of keyed fold maps on fiber_b200.procpool (host logic only: each block's
n_keys totals and counts placed in its area, the per-key fold of the non-empty totals sent to one live worker, re-queues
after deaths).  It speaks the worker protocol with key(x) = x mod n_keys and the order-sensitive integer "combine" of
tests/_fake_fold_worker.py in place of a device body -- test infrastructure, never used by the product (the real worker is
``procpool.gpu_worker_main``)."""
import os
import pickle
import sys

import numpy as np

from ._fake_fold_worker import tree


def keyed(xs, n_keys):
    """Per key: tree() of the items whose key is k (0 for none), and the number of them."""
    groups = [[] for _ in range(n_keys)]
    for x in xs:
        groups[x % n_keys].append(x)
    return [tree(g) if g else 0 for g in groups], [len(g) for g in groups]


def fake_keyed_worker_main(device, conn, results, sys_path):
    for p in sys_path:
        if p not in sys.path:
            sys.path.insert(0, p)
    from fiber_b200.procpool import SharedSegment, keyed_sequence
    segs = {}
    conn.send(("ready", os.getpid()))
    while True:
        msg = conn.recv()
        if msg is None:
            break
        if msg[0] == "keyed":
            _, job, n_blocks, n_keys, body, shm_name, module = msg
            mark = os.environ.get("FBR_TEST_FOLD_MARK")
            if body == "keyed_dies_once" and mark and not os.path.exists(mark):
                open(mark, "w").close()
                os._exit(3)                              # dies while folding the totals, without a word
            seg = segs.get(shm_name) or segs.setdefault(shm_name, SharedSegment(shm_name))
            area = n_keys * 16
            values, offsets, counts = keyed_sequence([seg.array[(1 + b) * area:(2 + b) * area] for b in range(n_blocks)], n_keys, 8)
            totals = np.asarray(values).view(np.uint64).tolist()
            recs = [tree(totals[int(offsets[k]):int(offsets[k + 1])]) if offsets[k + 1] > offsets[k] else 0 for k in range(n_keys)]
            seg.array[:n_keys * 8] = np.array(recs, np.uint64).view(np.uint8)
            seg.array[n_keys * 8:area] = counts.view(np.uint8)
            conn.send(("folded", job))
            continue
        _, job, blk, body, kind, n_keys, payload, shm_name, off, attempt, module = msg
        items = range(*payload[1]) if payload[0] == "range" else pickle.loads(payload[1])
        xs = [int(x) for x in items]
        if attempt == 0 and 0xDEAD in xs:
            os._exit(3)                                  # the worker process dies mid-block
        recs, counts = keyed(xs, n_keys)
        seg = segs.get(shm_name) or segs.setdefault(shm_name, SharedSegment(shm_name))
        seg.array[off:off + n_keys * 16] = np.concatenate([np.array(recs, np.uint64), np.array(counts, np.uint64)]).view(np.uint8)
        conn.send(("done", job, blk, None))
    os._exit(0)
