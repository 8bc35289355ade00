"""GPU: record bodies (FBR_EXPORT_RECORD_BODY) through dispatch_record_kernel -- fixed-size argument and result structs
of 8 to 1024 bytes, every map form, direct placement and the result ring, device-resident results, unaligned caller
buffers, resilient re-dispatch and process isolation.  Every result is compared bit for bit (``.view(np.uint8)``)
with the NumPy restatement in tests/record_bodies.py, and list for list with the Python definition at small n."""
import ctypes

import numpy as np
import pytest

import fiber_b200
from fiber_b200 import _abi, registry

from . import record_bodies as RB

pytestmark = pytest.mark.gpu

# body -> (seeded argument records, NumPy restatement)
CASES = {
    "polar_f64": (RB.polar_f64, RB.polar_args, RB.polar_np),
    "mix_i32x3": (RB.mix_i32x3, RB.mix_args, RB.mix_np),
    "row_stats_u32": (RB.row_stats_u32, RB.row_args, RB.row_stats_np),
    "scale5_f64": (RB.scale5_f64, RB.scale5_args, RB.scale5_np),
}


@pytest.fixture(scope="module")
def pool():
    p = fiber_b200.Pool(1, devices=[0])
    yield p
    p.terminate()
    p.join()


def _bytes(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _same(res, want):
    got = np.asarray(res)
    assert got.dtype == want.dtype and got.shape == want.shape
    assert np.array_equal(_bytes(got), _bytes(want))


def _unit(name, n, chunksize):
    p = _abi.Plan()
    _abi.check(_abi.load().fbr_plan_query(registry.spec(name).func_id, n, chunksize, 0, 1, 0, 132, ctypes.byref(p)))
    return p.unit_tasks


def _py_rows(func, args):
    """What the reference computes: f(*fields) per task (a sub-array field is passed as a list)."""
    return [func(*[v.tolist() for v in row.item()]) if isinstance(row.item()[0], np.ndarray) else func(*row.item())
            for row in args]


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("chunksize", [1, 7, 32])
def test_map_sizes(pool, name, chunksize):
    func, make, ref = CASES[name]
    big = (1 << 17) + 3 if name == "row_stats_u32" else 10 ** 6       # 1 KB argument records: 128 MB
    unit = _unit(name, big, chunksize)
    for n in (1, 7, unit - 1, unit + 1, big):
        args = make(n, seed=n)
        res = pool.map(func, args, chunksize)
        _same(res, ref(args))
        if n <= 1100:
            assert res.tolist() == _py_rows(func, args)


def test_map_forms(pool):
    args = RB.polar_args(3001, seed=3)
    want = RB.polar_np(args)
    pairs = [(float(x), float(y)) for x, y in args.tolist()]
    _same(pool.starmap(RB.polar_f64, pairs, 7), want)
    assert pool.starmap(RB.polar_f64, pairs[:50]) == [RB.polar_f64(*p) for p in pairs[:50]]
    assert pool.apply_async(RB.polar_f64, (3.0,), {"y": 4.0}).get() == (25.0, 5.0)
    assert pool.apply(RB.polar_f64, (), {"y": -1.5, "x": 2.0}) == RB.polar_f64(2.0, -1.5)
    assert list(pool.imap(RB.polar_f64, args, 1)) == want.tolist()
    assert sorted(pool.imap_unordered(RB.polar_f64, args[:500], 3)) == sorted(want[:500].tolist())
    # a one-parameter body over a list of rows, and over a plain (n, 256) uint32 array (zero-copy view)
    rows = RB.row_args(37, seed=5)
    assert pool.map(RB.row_stats_u32, [r.tolist() for r in rows["row"]]) == [RB.row_stats_u32(r) for r in rows["row"]]
    _same(pool.map(RB.row_stats_u32, rows["row"]), RB.row_stats_np(rows))
    mix = RB.mix_args(1000, seed=9)
    assert pool.starmap(RB.mix_i32x3, mix.tolist(), 32) == [RB.mix_i32x3(*t) for t in mix.tolist()]
    with pytest.raises(TypeError, match="missing 1 required positional argument: 'y'"):
        pool.apply_async(RB.polar_f64, (1.0,))
    with pytest.raises(TypeError):
        pool.map(RB.polar_f64, [1.0, 2.0])            # f(x, y) called with one argument


def test_index_body_over_range(pool):
    for n, start, step in ((1, 0, 1), (1023, 5, 3), (1025, -7, 1), (10 ** 6, 2 ** 40, 1)):
        r = range(start, start + n * step, step)
        res = pool.map(RB.splitmix_pair, r, 7)
        _same(res, RB.splitmix_pair_np(np.arange(start, start + n * step, step, dtype=np.int64)))
        if n < 2000:
            assert res.tolist() == [RB.splitmix_pair(i) for i in r]
    # explicit int64 arguments go through the staged argument path
    xs = np.random.default_rng(1).integers(-2 ** 63, 2 ** 63 - 1, 5001, dtype=np.int64)
    _same(pool.map(RB.splitmix_pair, xs), RB.splitmix_pair_np(xs))


def _raw(pool, name, n, flags, args=None, arg_stride=0, out=None, chunksize=0, seed=11):
    """One map through the C ABI; returns the result bytes (host results) or None (FBR_OUT_DEVICE)."""
    spec = registry.spec(name)
    eng = pool._engine
    d = _abi.MapDesc()
    d.func_id, d.flags, d.n_tasks, d.chunksize, d.shuffle_seed = spec.func_id, flags, n, chunksize, seed
    if args is None:
        d.index_start, d.index_step = 0, 1
    else:
        d.args, d.arg_stride = args, arg_stride
    if out is not None:
        d.out = out
    seq = ctypes.c_uint64()
    _abi.check(eng.lib.fbr_map_submit(eng.handle, ctypes.byref(d), ctypes.byref(seq)))
    res = _abi.Result()
    _abi.check(eng.lib.fbr_result_wait(eng.handle, seq.value, -1, ctypes.byref(res)))
    data = None
    if not flags & _abi.FBR_OUT_DEVICE:
        data = np.frombuffer((ctypes.c_char * (n * spec.result_bytes)).from_address(res.data), np.uint8).copy()
    _abi.check(eng.lib.fbr_result_release(eng.handle, seq.value))
    return data


@pytest.mark.parametrize("flags", [_abi.FBR_SHUFFLE, _abi.FBR_VIA_RING, 0])
def test_ring_and_direct_placement(pool, flags):
    """12 B and 24 B slots placed by index through the result ring (shuffled arrival, or FBR_VIA_RING) and directly."""
    before = pool.stats()
    for name, n in (("mix_i32x3", 300007), ("row_stats_u32", 20011), ("scale5_f64", 70001), ("polar_f64", 1 << 20)):
        _, make, ref = CASES[name]
        args = make(n, seed=2)
        got = _raw(pool, name, n, flags, args.ctypes.data, args.itemsize, chunksize=7)
        assert np.array_equal(got, _bytes(ref(args)))
    got = _raw(pool, "splitmix_pair", 100003, flags)
    assert np.array_equal(got, _bytes(RB.splitmix_pair_np(np.arange(100003))))
    st = pool.stats()
    if flags:
        assert st["gather_launches"] > before["gather_launches"]
    else:
        assert st["direct_waves"] > before["direct_waves"]


def test_shuffled_tail_unit_under_16_bytes(pool):
    """A last unit of one 12 B task has no bytes for a bulk store.  Under FBR_SHUFFLE it runs anywhere in a CTA's
    sequence of units, between units whose results are bulk-stored from the same two OUT stages; each must still
    land intact."""
    for chunksize in (1, 7):
        for k in (150, 977):
            n = k * _unit("mix_i32x3", 10 ** 6, chunksize) + 1
            assert n % _unit("mix_i32x3", n, chunksize) == 1
            args = RB.mix_args(n, seed=k)
            want = _bytes(RB.mix_np(args))
            for seed in (1, 2, 3):
                got = _raw(pool, "mix_i32x3", n, _abi.FBR_SHUFFLE, args.ctypes.data, 12, chunksize=chunksize, seed=seed)
                assert np.array_equal(got, want), (chunksize, k, seed)


def test_strided_and_unaligned_buffers(pool):
    """Argument records further apart than their size, and device-resident arguments / results at addresses that are
    not 16 B aligned: the kernel falls back to cooperative 16 B / 4 B copies."""
    n = 100003
    mix = RB.mix_args(n, seed=4)
    want = _bytes(RB.mix_np(mix))
    wide = np.zeros(n, [("rec", RB.MIX_ARG), ("pad", "<u4")])        # 16 B stride for 12 B records
    wide["rec"] = mix
    assert np.array_equal(_raw(pool, "mix_i32x3", n, 0, wide.ctypes.data, 16), want)
    assert np.array_equal(_raw(pool, "mix_i32x3", n, _abi.FBR_SHUFFLE, wide.ctypes.data, 16), want)
    eng = pool._engine
    lib = eng.lib
    base_in, base_out = ctypes.c_void_p(), ctypes.c_void_p()
    _abi.check(lib.fbr_device_alloc(eng.handle, 0, n * 12 + 64, ctypes.byref(base_in)))
    _abi.check(lib.fbr_device_alloc(eng.handle, 0, n * 12 + 64, ctypes.byref(base_out)))
    try:
        for ai, oi in ((4, 4), (0, 8), (8, 0), (0, 0)):
            a_ptr, o_ptr = base_in.value + ai, base_out.value + oi
            _abi.check(lib.fbr_memcpy_h2d(eng.handle, 0, ctypes.c_void_p(a_ptr), mix.ctypes.data, n * 12))
            for flags in (0, _abi.FBR_VIA_RING):
                _raw(pool, "mix_i32x3", n, flags | _abi.FBR_ARGS_DEVICE | _abi.FBR_OUT_DEVICE, a_ptr, 12, out=o_ptr, chunksize=5)
                got = np.empty(n * 12, np.uint8)
                _abi.check(lib.fbr_memcpy_d2h(eng.handle, 0, got.ctypes.data, ctypes.c_void_p(o_ptr), n * 12))
                assert np.array_equal(got, want), (ai, oi, flags)
    finally:
        lib.fbr_device_free(eng.handle, 0, base_in)
        lib.fbr_device_free(eng.handle, 0, base_out)


def test_results_on_device_fetch_unaligned_ranges():
    p = fiber_b200.Pool(1, devices=[0], results="device")
    try:
        for name in ("mix_i32x3", "row_stats_u32"):
            func, make, ref = CASES[name]
            args = make(50021, seed=8)
            want = ref(args)
            res = p.map(func, args)
            assert res.on_device and len(res) == len(args)
            assert res[3] == want[3:4].tolist()[0] and res[-1] == want[-1:].tolist()[0]
            assert res[1:4] == want[1:4].tolist() and res[4095:4113] == want[4095:4113].tolist()
            _same(res, want)
    finally:
        p.terminate()
        p.join()


def test_resilient_pool_redispatches_lost_units():
    args = RB.polar_args(200003, seed=6)
    args["y"][[0, 4097, 77777, 200002]] = -1.0            # these tasks lose their unit on its first attempt
    want = RB.polar_np(args)
    p = fiber_b200.Pool(1, devices=[0], error_handling=True)
    try:
        _same(p.map(RB.fault_polar_f64, args), want)
        assert p.stats()["units_redispatched"] > 0
        assert p.map(RB.fault_polar_f64, args[:100]).tolist() == _py_rows(RB.polar_f64, args[:100])
    finally:
        p.terminate()
        p.join()
    plain = fiber_b200.Pool(1, devices=[0])
    try:
        # without error_handling a lost unit is a task error, reported at the first task of the lowest lost unit
        with pytest.raises(RuntimeError, match="task 0 failed with device error code 3"):
            plain.map(RB.fault_polar_f64, args, 32)
    finally:
        plain.terminate()
        plain.join()


def test_two_gpus():
    n = ctypes.c_int(0)
    _abi.check(_abi.load().fbr_device_count(ctypes.byref(n)))
    if n.value < 2:
        pytest.skip("needs two GPUs")
    p = fiber_b200.Pool(2)
    try:
        args = RB.mix_args(10 ** 6, seed=12)
        _same(p.map(RB.mix_i32x3, args), RB.mix_np(args))
    finally:
        p.terminate()
        p.join()


def test_process_isolated_pool():
    """The worker processes register the body module with its two dtypes themselves."""
    p = fiber_b200.Pool(2, isolation="process")
    try:
        args = RB.polar_args(100003, seed=13)
        _same(p.map(RB.polar_f64, args), RB.polar_np(args))
        rows = RB.row_args(5000, seed=14)
        _same(p.map(RB.row_stats_u32, rows), RB.row_stats_np(rows))
        assert p.starmap(RB.mix_i32x3, [(1, 2, 3), (-4, 5, 6)]) == [RB.mix_i32x3(1, 2, 3), RB.mix_i32x3(-4, 5, 6)]
    finally:
        p.terminate()
        p.join()
