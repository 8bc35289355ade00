"""GPU: the completion step of fold and accumulate maps reached through each call that can complete a map --
fbr_result_poll, fbr_result_fetch before any wait, and fbr_result_wait after a poll -- on one worker and on two (the
two-worker cases, several blocks, skip without a second GPU)."""
import ctypes

import numpy as np
import pytest

import fiber_b200
from fiber_b200 import _abi, registry

from . import fold_bodies as FB
from . import scan_bodies as SB
from .test_scan_bodies_gpu import _raw_scan, _two_gpus, inputs, raw_records

pytestmark = pytest.mark.gpu

N = 300_001          # two blocks on two workers


@pytest.fixture(scope="module", params=[1, 2], ids=["1worker", "2workers"])
def pool(request):
    if request.param == 2:
        _two_gpus()
    p = fiber_b200.Pool(request.param, devices=list(range(request.param)))
    p.accumulate(SB.affine_f64, inputs("affine_f64", 1, seed=0))      # starts the pool's workers
    yield p
    p.terminate()
    p.join()


def _submit(p, name, xs, flags):
    """Submits a map through the C ABI: its seq, and the encoded arguments, which must outlive the map."""
    spec = registry.spec(name)
    enc = spec.encode_map(xs)
    d = _abi.MapDesc()
    d.func_id, d.flags, d.n_tasks, d.arg_stride, d.args = spec.func_id, flags, enc.n, enc.arg_stride, enc.args.ctypes.data
    seq = ctypes.c_uint64()
    _abi.check(p._engine.lib.fbr_map_submit(p._engine.handle, ctypes.byref(d), ctypes.byref(seq)))
    return seq.value, enc


def _poll_until_done(p, seq, n):
    eng = p._engine
    done = ctypes.c_uint64()
    seen = set()
    while done.value != n:
        _abi.check(eng.lib.fbr_result_poll(eng.handle, seq, ctypes.byref(done)))
        seen.add(done.value)
    assert seen <= {0, n}, seen


@pytest.mark.parametrize("results", ["host", "device"])
def test_poll_of_an_accumulate_map(pool, results):
    xs = inputs("affine_f64", N, seed=51)
    R = registry.spec("affine_f64").result_bytes
    want = b"".join(raw_records(pool.accumulate(SB.affine_f64, xs), R))
    eng = pool._engine
    flags = _abi.FBR_SCAN | (_abi.FBR_RESULTS_ON_DEVICE if results == "device" else 0)
    seq, _enc = _submit(pool, "affine_f64", xs, flags)
    try:
        _poll_until_done(pool, seq, N)
        if results == "device":         # a poll that reports every task done leaves the wrapped windows to fetch
            got = np.zeros(N * R, np.uint8)
            _abi.check(eng.lib.fbr_result_fetch(eng.handle, seq, 0, N, got.ctypes.data))
            assert got.tobytes() == want
        res = _abi.Result()
        _abi.check(eng.lib.fbr_result_wait(eng.handle, seq, -1, ctypes.byref(res)))
        if results == "host":
            assert ctypes.string_at(res.data, N * R) == want
    finally:
        _abi.check(eng.lib.fbr_result_release(eng.handle, seq))
    got = [tuple(r) for r in pool.accumulate_async(SB.affine_f64, xs).iget_ordered()]
    assert got == [tuple(r) for r in pool.accumulate(SB.affine_f64, xs)]


def test_fetch_without_a_wait(pool):
    xs = inputs("affine_f64", N, seed=52)
    R = registry.spec("affine_f64").result_bytes
    want = _raw_scan(pool, "affine_f64", xs, flags=_abi.FBR_RESULTS_ON_DEVICE)
    eng = pool._engine
    seq, _enc = _submit(pool, "affine_f64", xs, _abi.FBR_SCAN | _abi.FBR_RESULTS_ON_DEVICE)
    try:
        got = np.zeros(N * R, np.uint8)
        half = N // 2
        _abi.check(eng.lib.fbr_result_fetch(eng.handle, seq, 0, half, got.ctypes.data))
        _abi.check(eng.lib.fbr_result_fetch(eng.handle, seq, half, N - half, got[half * R:].ctypes.data))
        assert got.tobytes() == want
        res = _abi.Result()
        _abi.check(eng.lib.fbr_result_wait(eng.handle, seq, -1, ctypes.byref(res)))
    finally:
        _abi.check(eng.lib.fbr_result_release(eng.handle, seq))


def test_fold_map_that_fails(pool):
    xs = range(0, N)
    with pytest.raises(RuntimeError) as folded:
        pool.fold(FB.fault_count_u64, xs)
    r = pool.fold_async(FB.fault_count_u64, xs)
    _poll_until_done(pool, r._seq, N)
    with pytest.raises(RuntimeError) as polled:
        r.get()
    assert str(polled.value) == str(folded.value)
