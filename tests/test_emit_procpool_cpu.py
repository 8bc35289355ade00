"""CPU: process-isolated maps of an emit body (fiber_b200/procpool.py) with a stand-in worker (tests/_fake_emit_worker.py):
each block's end offsets land in the map's segment and its values in a file of their own; get() concatenates the
blocks in order and rebases their offsets, also when a worker died under a block and it was re-dispatched."""
import os

import numpy as np

from fiber_b200.pool import EmitResultArray
from fiber_b200.procpool import ProcessPool

from ._fake_emit_worker import fake_emit_worker_main


class _EmitSpec:
    """What the master needs of an emit body: its name, its 8-byte end-offset record and its values' dtype."""

    def __init__(self):
        self.name, self.result_bytes, self.flags = "emit_range", 8, 0
        self.out_dtype, self.out_as = np.dtype(np.int64), "list"

    def result_dtype(self):
        return np.dtype(np.uint64), ()


def test_blocks_are_stitched_and_rebased():
    pool = ProcessPool(3, devices=[0, 1, 2], results="bytes", worker_main=fake_emit_worker_main, block_tasks=7)
    try:
        xs = [(i * 7) % 11 for i in range(60)]          # some empty lists, blocks of 7 tasks, a short last block
        r = pool.submit(_EmitSpec(), None, "map", xs, 1).get(60)
        assert isinstance(r, EmitResultArray) and r == [list(range(x)) for x in xs]
        assert r.ragged.offsets[-1] == sum(xs)
        # a worker dies under the block holding 13; the re-dispatched block replaces its values whole
        ys = list(range(20))
        assert pool.submit(_EmitSpec(), None, "map", ys, 1).get(60) == [list(range(y)) for y in ys]
        assert pool.stats["blocks_redispatched"] >= 1
        assert len(pool.submit(_EmitSpec(), None, "map", [], 1).get(5)) == 0
        assert pool.submit(_EmitSpec(), None, "map", [0] * 9, 1).get(60) == [[]] * 9
        assert not [f for f in os.listdir("/dev/shm") if f.startswith("fbr_%d_" % os.getpid()) and "_v" in f]
    finally:
        pool.terminate()
        pool.join()
