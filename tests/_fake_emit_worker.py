"""A stand-in worker process for the CPU test of process-isolated emit maps (tests/test_emit_procpool_cpu.py): it speaks
the worker protocol of fiber_b200.procpool and "computes" the emit body ``emit_range`` (task x returns ``range(x)``)
with NumPy, writing each block's block-local end offsets into the map's segment and its values beside it, as
``procpool.gpu_worker_main`` does.  Test infrastructure, never used by the product."""
import os
import pickle
import sys

import numpy as np


def fake_emit_worker_main(device, conn, results, sys_path):
    for p in sys_path:
        if p not in sys.path:
            sys.path.insert(0, p)
    from fiber_b200.procpool import SharedSegment, put_values, values_name
    segs = {}
    conn.send(("ready", os.getpid()))
    while True:
        msg = conn.recv()
        if msg is None:
            break
        _, job, blk, body, kind, chunksize, payload, shm_name, off, attempt, module = msg
        items = range(*payload[1]) if payload[0] == "range" else pickle.loads(payload[1])
        xs = np.asarray(list(items), dtype=np.int64)
        if attempt == 0 and (xs == 13).any():
            os._exit(3)                                  # the worker dies mid-block; its block is re-dispatched
        ends = np.cumsum(xs).astype(np.uint64)
        seg = segs.get(shm_name) or segs.setdefault(shm_name, SharedSegment(shm_name))
        raw = ends.view(np.uint8)
        seg.array[off:off + raw.nbytes] = raw
        put_values(values_name(shm_name, blk), np.concatenate([np.arange(x, dtype=np.int64) for x in xs]) if len(xs)
                   else np.empty(0, np.int64))
        conn.send(("done", job, blk, None))
    os._exit(0)
