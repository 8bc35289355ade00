"""CPU: which arrays count as one broadcast block (byte for byte, in either accepted form), and initargs checked in the
master process of a process-isolated pool before any worker starts."""
import numpy as np
import pytest

import fiber_b200
from fiber_b200 import registry

from . import broadcast_bodies as BB


def test_blocks_are_compared_as_bytes():
    s = registry.spec("kde_window_f64")
    pos = np.random.default_rng(4).standard_normal((50, 2))
    pos[3, 0] = 0.0
    neg = pos.copy()
    neg[3, 0] = -0.0                                     # equal values, different bytes: a different block
    b_pos = s.shared_block(pos)
    b_neg = s.shared_block(neg)
    assert b_neg is not b_pos and b_neg == neg.tobytes() and b_pos == pos.tobytes()
    with pytest.raises(ValueError, match="must share x_samples"):
        s.encode_starmap([(pos, 0.5), (neg, 0.7)])
    # a NaN never equals itself by value, but a copy of the array is the same block
    nan = pos.copy()
    nan[7, 1] = np.nan
    b_nan = s.shared_block(nan)
    assert s.shared_block(nan.copy()) is b_nan
    e = s.encode_starmap([(nan, 0.5), (nan.copy(), 0.7)])
    assert e.n == 2 and e.shared is b_nan


def test_plain_and_structured_forms_are_one_block():
    s = registry.spec("nearest_centroid_f32")
    C = BB.centroids(6, seed=3)
    P = BB.points(3, seed=4)
    e = s.encode_starmap([(C, P["p"][0]), (C["c"], P["p"][1]), (C["c"].copy(), P["p"][2])])
    assert e.n == 3 and e.shared == C.tobytes() and e.shared is s.shared_block(C["c"])
    C2 = C["c"].copy()
    C2[5, 15] = np.nextafter(C2[5, 15], np.float32(np.inf))
    with pytest.raises(ValueError, match="must share centroids"):
        s.encode_starmap([(C, P["p"][0]), (C2, P["p"][1])])


def test_process_pool_checks_initargs_before_starting_workers():
    bad = np.zeros((4, 8), np.float32)                  # centroids are 16 floats each
    p = fiber_b200.Pool(2, isolation="process", initializer=BB.set_centroids, initargs=(bad,))
    with pytest.raises(TypeError, match="centroids must be"):
        p.start_workers()
    assert p._proc is None                               # no worker process was started
    p = fiber_b200.Pool(1, isolation="process", initializer=BB.set_centroids, initargs=(BB.centroids(2), BB.centroids(2)))
    with pytest.raises(TypeError, match="exactly one argument"):
        p.start_workers()
    assert p._proc is None
