"""GPU: a caller's device-pointer broadcast block (FBR_ARGS_DEVICE) at a base that is not 16 B aligned, on the path that
reads it from global memory.  The bodies load their elements as 8 B (kde_window_f64: doubles) and 16 B vectors
(nearest_centroid: an alignas(16) struct); the engine reads such a block from an aligned copy, so every offset gives the
results the aligned block gives.  Staged blocks at the same offsets are covered too."""
import ctypes

import numpy as np
import pytest

import fiber_b200
from fiber_b200 import _abi, registry

from . import broadcast_bodies as BB

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pool():
    p = fiber_b200.Pool(1, devices=[0])
    p.start_workers()                                   # the raw ABI below needs the engine
    yield p
    p.terminate()
    p.join()


def _run(pool, name, n, flags, shared, shared_bytes, args, arg_stride):
    spec = registry.spec(name)
    eng = pool._engine
    d = _abi.MapDesc()
    d.func_id, d.flags, d.n_tasks, d.chunksize = spec.func_id, flags, n, 7
    d.shared, d.shared_bytes, d.args, d.arg_stride = shared, shared_bytes, args, arg_stride
    seq = ctypes.c_uint64()
    _abi.check(eng.lib.fbr_map_submit(eng.handle, ctypes.byref(d), ctypes.byref(seq)))
    res = _abi.Result()
    _abi.check(eng.lib.fbr_result_wait(eng.handle, seq.value, -1, ctypes.byref(res)))
    data = np.frombuffer((ctypes.c_char * (n * spec.result_bytes)).from_address(res.data), np.uint8).copy()
    _abi.check(eng.lib.fbr_result_release(eng.handle, seq.value))
    return data


def test_unaligned_device_block_on_the_global_path(pool):
    eng = pool._engine
    lib = eng.lib
    from oracle import bodies as B
    xs = np.ascontiguousarray(B.parzen_example_inputs()[0])          # 10 000 x 2 float64: 160 KB, beyond the budget
    widths = np.arange(1, 41, dtype=np.float64) * 0.25
    n = 30011
    P = BB.points(n, seed=41)
    cases = [  # body, block, argument records, NumPy restatement
        ("nearest_centroid_f32", BB.centroids(600, seed=42), P, lambda a, blk: BB.nearest_np(a, blk)),          # 38 KB > 32 KB
        ("nearest_centroid_global_f32", BB.centroids(64, seed=43), P, lambda a, blk: BB.nearest_np(a, blk)),    # never staged
        ("kde_window_f64", xs, widths, lambda a, blk: BB.kde_np(a, blk)),
        ("kde_window_f64", xs[:700], widths, lambda a, blk: BB.kde_np(a, blk)),                                  # staged
    ]
    d_args, d_blk = ctypes.c_void_p(), ctypes.c_void_p()
    _abi.check(lib.fbr_device_alloc(eng.handle, 0, n * 64, ctypes.byref(d_args)))
    _abi.check(lib.fbr_device_alloc(eng.handle, 0, xs.nbytes + 64, ctypes.byref(d_blk)))
    try:
        for name, blk, args, ref in cases:
            args = np.ascontiguousarray(args)
            blk = np.ascontiguousarray(blk)
            want = np.ascontiguousarray(ref(args, blk)).view(np.uint8)
            _abi.check(lib.fbr_memcpy_h2d(eng.handle, 0, d_args, args.ctypes.data, args.nbytes))
            stride = args.dtype.itemsize
            for off in (4, 8, 12, 0):
                base = ctypes.c_void_p(d_blk.value + off)
                _abi.check(lib.fbr_memcpy_h2d(eng.handle, 0, base, blk.ctypes.data, blk.nbytes))
                for flags in (0, _abi.FBR_VIA_RING):
                    got = _run(pool, name, len(args), flags | _abi.FBR_ARGS_DEVICE, base.value, blk.nbytes, d_args.value, stride)
                    assert np.array_equal(got, want), (name, len(blk), off, flags)
    finally:
        lib.fbr_device_free(eng.handle, 0, d_args)
        lib.fbr_device_free(eng.handle, 0, d_blk)
