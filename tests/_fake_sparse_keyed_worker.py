"""A stand-in worker process for the CPU tests of sparse keyed fold maps on fiber_b200.procpool (host logic only: each
block's records, counts and keys written to its own file, the merge and per-key fold sent to one live worker, re-queues
after deaths).  It speaks the worker protocol with key(x) = (x * 2654435761) mod 2^32 >> 20 and the order-sensitive integer
"combine" of tests/_fake_fold_worker.py in place of a device body -- test infrastructure, never used by the product (the
real worker is ``procpool.gpu_worker_main``)."""
import os
import pickle
import sys

import numpy as np

from ._fake_fold_worker import tree


def key_of(x):
    return (x * 2654435761 & 0xFFFFFFFF) >> 20


def sparse(xs):
    """Per distinct key in ascending order: tree() of the items whose key it is; the keys and the counts."""
    groups = {}
    for x in xs:
        groups.setdefault(key_of(x), []).append(x)
    keys = sorted(groups)
    return [tree(groups[k]) for k in keys], keys, [len(groups[k]) for k in keys]


def area(recs, keys, counts):
    """A block's (or the result's) file: records, uint64 counts, uint32 keys."""
    return np.concatenate([np.array(recs, np.uint64).view(np.uint8), np.array(counts, np.uint64).view(np.uint8),
                           np.array(keys, np.uint32).view(np.uint8)])


def fake_sparse_worker_main(device, conn, results, sys_path):
    for p in sys_path:
        if p not in sys.path:
            sys.path.insert(0, p)
    from fiber_b200.procpool import put_values, sparse_area, sparse_keyed_sequence, values_name
    conn.send(("ready", os.getpid()))
    while True:
        msg = conn.recv()
        if msg is None:
            break
        if msg[0] == "sparse":
            _, job, n_blocks, body, shm_name, module = msg
            mark = os.environ.get("FBR_TEST_FOLD_MARK")
            if body == "sparse_dies_once" and mark and not os.path.exists(mark):
                open(mark, "w").close()
                os._exit(3)                              # dies while merging the blocks, without a word
            areas = [sparse_area(np.fromfile(os.path.join("/dev/shm", values_name(shm_name, b)), np.uint8), 8) for b in range(n_blocks)]
            values, offsets, keys, counts = sparse_keyed_sequence(*zip(*areas))
            totals = np.asarray(values).view(np.uint64).tolist()
            recs = [tree(totals[int(offsets[k]):int(offsets[k + 1])]) for k in range(len(keys))]
            put_values(values_name(shm_name, n_blocks), area(recs, keys, counts))
            conn.send(("folded", job, len(keys)))
            continue
        _, job, blk, body, kind, _, payload, shm_name, off, attempt, module = msg
        items = range(*payload[1]) if payload[0] == "range" else pickle.loads(payload[1])
        xs = [int(x) for x in items]
        if attempt == 0 and 0xDEAD in xs:
            os._exit(3)                                  # the worker process dies mid-block
        put_values(values_name(shm_name, blk), area(*sparse(xs)))
        conn.send(("done", job, blk, None))
    os._exit(0)
