"""GPU: items record bodies through dispatch_record_kernel -- byte strings, float64 rows on a warp, a head record, a
broadcast table; every map form, skewed lengths, direct placement and the result ring,
device-resident items at unaligned bases, bad device offsets, resilient re-dispatch and process isolation.  Every result
is compared bit for bit with the restatements in tests/ragged_bodies.py."""
import ctypes

import numpy as np
import pytest

import fiber_b200
from fiber_b200 import _abi, registry

from . import ragged_bodies as RB

pytestmark = pytest.mark.gpu


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


def _sub(vals, offs, n):
    return vals[:int(offs[n])], offs[:n + 1]


STRINGS = RB.byte_strings(400_000, seed=1)                # about 100 MB of bytes, lengths 0 .. 512
ROWS = RB.lognormal_rows(200_000, seed=2)                 # about 100 MB of float64


@pytest.mark.parametrize("chunksize", [1, 7, 32])
@pytest.mark.parametrize("name", ["fnv1a_bytes", "ragged_stats_f64"])
def test_map_sizes(pool, name, chunksize):
    vals, offs = STRINGS if "fnv" in name else ROWS
    ref = RB.fnv1a_np if "fnv" in name else RB.ragged_stats_np
    func = getattr(RB, name)
    unit = _unit(name, len(offs) - 1, chunksize)
    sizes = sorted({n for n in (1, 7, unit - 1, unit + 1, 3 * unit + 5) if n > 0})
    if chunksize == 32:
        sizes.append(len(offs) - 1)
    for n in sizes:
        v, o = _sub(vals, offs, n)
        _same(pool.map(func, fiber_b200.Ragged(v, o), chunksize), ref(v, o))
    # lists of bytes / arrays; the Python definition at small n (np.sum's order differs from the device's lanes: the
    # statistics body is compared with its restatement only)
    v, o = _sub(vals, offs, 40)
    xs = [v[o[i]:o[i + 1]] for i in range(40)]
    if "fnv" in name:
        xs = [x.tobytes() for x in xs]
        assert pool.map(func, xs, chunksize).tolist() == [func(x) for x in xs]
    _same(pool.map(func, xs, chunksize), ref(v, o))


def test_skewed_lengths_long_and_empty(pool):
    """Mostly short strings with a few far longer than a claim unit's others (up to 1 MB), one 100 KB item alone, and
    maps of empty items only."""
    rng = np.random.default_rng(5)
    lens = rng.integers(0, 64, 50_000)
    lens[[3, 999, 20_000, 49_999]] = [70_000, 16_385, 1_000_000, 40_000]
    offs = np.zeros(len(lens) + 1, np.int64)
    np.cumsum(lens, out=offs[1:])
    vals = rng.integers(0, 256, int(offs[-1]), dtype=np.uint8)
    want = RB.fnv1a_np(vals, offs)
    _same(pool.map(RB.fnv1a_bytes, fiber_b200.Ragged(vals, offs), 7), want)
    long = rng.integers(0, 256, 100_000, dtype=np.uint8).tobytes()
    assert pool.map(RB.fnv1a_bytes, [long]).tolist() == [RB.fnv1a_bytes(long)]
    empty = pool.map(RB.fnv1a_bytes, [b""] * 1000)                          # only empty items: n_items = 0
    assert empty.tolist() == [RB.fnv1a_bytes(b"")] * 1000
    rows = pool.map(RB.ragged_stats_f64, [np.zeros(0)] * 100 + [np.arange(5000.0)])
    _same(rows, RB.ragged_stats_np(np.arange(5000.0), np.array([0] * 101 + [5000])))


def test_map_forms(pool):
    vals, offs = RB.lognormal_rows(5000, seed=3, max_len=2000)
    vals = vals.astype(np.float32)
    rng = np.random.default_rng(4)
    lo = rng.uniform(-1, 0, len(offs) - 1).astype(np.float32)
    hi = rng.uniform(0, 1, len(offs) - 1).astype(np.float32)
    want = RB.clip_sum_np(vals, offs, lo, hi)
    rows = [vals[offs[i]:offs[i + 1]] for i in range(len(offs) - 1)]
    spec = registry.spec("clip_sum_f32")
    _same(pool.starmap(RB.clip_sum_f32, list(zip(rows, lo, hi)), 7), want)
    assert pool.starmap(RB.clip_sum_f32, list(zip(rows[:20], lo[:20], hi[:20]))) == \
        [RB.clip_sum_f32(r, a, b) for r, a, b in zip(rows[:20], lo[:20], hi[:20])]
    assert pool.apply_async(RB.clip_sum_f32, (rows[3],), {"hi": hi[3], "lo": lo[3]}).get() == spec.rows_to_list(want[3:4])[0]
    assert pool.apply(RB.clip_sum_f32, (), {"row": rows[4], "lo": lo[4], "hi": hi[4]}) == spec.rows_to_list(want[4:5])[0]
    swant = RB.ragged_stats_np(*_sub(*ROWS, 3000))
    r = fiber_b200.Ragged(*_sub(*ROWS, 3000))
    assert list(pool.imap(RB.ragged_stats_f64, r, 32)) == swant.tolist()
    assert sorted(pool.imap_unordered(RB.ragged_stats_f64, r[:500], 3)) == sorted(swant[:500].tolist())
    # a broadcast table with the items; an out-of-range token is a bad argument
    w = np.random.default_rng(6).standard_normal(1000).astype(np.float32)
    tv, to = RB.byte_strings(20_000, seed=7, max_len=200)
    toks = (tv.astype(np.uint32) * 3)
    docs = [toks[to[i]:to[i + 1]] for i in range(len(to) - 1)]
    _same(pool.starmap(RB.token_weight_u32, [(w, d) for d in docs], 7), RB.token_weight_np(w, toks, to))
    with pytest.raises(ValueError, match="bad argument in task 2"):
        pool.starmap(RB.token_weight_u32, [(w, [1]), (w, [2]), (w, [5, 1000]), (w, [999])])


def _raw_items(pool, name, n, flags, items, offsets, n_items, out=None, chunksize=0, seed=11):
    spec = registry.spec(name)
    eng = pool._engine
    d = _abi.MapDesc()
    d.func_id, d.flags, d.n_tasks, d.chunksize, d.shuffle_seed = spec.func_id, flags, n, chunksize, seed
    if out is not None:
        d.out = out
    it = _abi.ItemsDesc()
    it.items, it.offsets, it.n_items, it.item_bytes = items, offsets, n_items, registry.spec(name).item_dtype.itemsize
    seq = ctypes.c_uint64()
    _abi.check(eng.lib.fbr_map_submit_items(eng.handle, ctypes.byref(d), ctypes.byref(it), ctypes.byref(seq)))
    res = _abi.Result()
    rc = eng.lib.fbr_result_wait(eng.handle, seq.value, -1, ctypes.byref(res))
    if rc != _abi.FBR_ETASK:
        _abi.check(rc)
    data = None
    if not flags & _abi.FBR_OUT_DEVICE and res.err_code == 0:
        data = np.frombuffer((ctypes.c_char * (n * spec.result_bytes)).from_address(res.data), np.uint8).copy()
    err = (res.err_code, res.err_task)
    _abi.check(eng.lib.fbr_result_release(eng.handle, seq.value))
    return data, err


@pytest.mark.parametrize("flags", [_abi.FBR_SHUFFLE, _abi.FBR_VIA_RING, 0])
def test_ring_and_direct_placement(pool, flags):
    before = pool.stats()
    for name, (vals, offs), ref in (("fnv1a_bytes", STRINGS, RB.fnv1a_np), ("ragged_stats_f64", ROWS, RB.ragged_stats_np)):
        v, o = _sub(vals, offs, 50_000)
        ou = o.astype(np.uint64)
        got, err = _raw_items(pool, name, 50_000, flags, v.ctypes.data, ou.ctypes.data, len(v), chunksize=7)
        assert err[0] == 0 and np.array_equal(got, _bytes(ref(v, o))), name
    st = pool.stats()
    if flags:
        assert st["gather_launches"] > before["gather_launches"]
    else:
        assert st["direct_waves"] > before["direct_waves"]
    # the other entry point is refused either way round
    d, it, seq = _abi.MapDesc(), _abi.ItemsDesc(), ctypes.c_uint64()
    d.func_id, d.n_tasks = registry.spec("fnv1a_bytes").func_id, 1
    with pytest.raises(_abi.EngineError, match="fbr_map_submit_items"):
        _abi.check(pool._engine.lib.fbr_map_submit(pool._engine.handle, ctypes.byref(d), ctypes.byref(seq)))
    d.func_id = registry.spec("polar_f64").func_id if "polar_f64" in fiber_b200.body_names() else 0
    with pytest.raises(_abi.EngineError, match="fbr_map_submit"):
        _abi.check(pool._engine.lib.fbr_map_submit_items(pool._engine.handle, ctypes.byref(d), ctypes.byref(it), ctypes.byref(seq)))


def test_device_resident_items(pool):
    """Device items at every base offset 1..15 (bytes) and 8 (float64), offsets that start past 0, and bad offsets."""
    eng = pool._engine
    lib = eng.lib
    vals, offs = _sub(*STRINGS, 20_000)
    n = 19_000
    o = offs[1000:1000 + n + 1].astype(np.uint64)             # offsets[0] != 0: a slice of the larger array
    want = RB.fnv1a_np(vals, offs[1000:1000 + n + 1])
    base, doffs, dout = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
    _abi.check(lib.fbr_device_alloc(eng.handle, 0, vals.nbytes + 64, ctypes.byref(base)))
    _abi.check(lib.fbr_device_alloc(eng.handle, 0, o.nbytes + 64, ctypes.byref(doffs)))
    _abi.check(lib.fbr_device_alloc(eng.handle, 0, n * 16 + 64, ctypes.byref(dout)))
    try:
        _abi.check(lib.fbr_memcpy_h2d(eng.handle, 0, doffs, o.ctypes.data, o.nbytes))
        for shift in range(16):
            ptr = ctypes.c_void_p(base.value + shift)
            _abi.check(lib.fbr_memcpy_h2d(eng.handle, 0, ptr, vals.ctypes.data, vals.nbytes))
            for flags in (0, _abi.FBR_VIA_RING):
                got, err = _raw_items(pool, "fnv1a_bytes", n, flags | _abi.FBR_ARGS_DEVICE, ptr.value, doffs.value, len(vals),
                                      chunksize=5)
                assert err[0] == 0 and np.array_equal(got, _bytes(want)), (shift, flags)
            got, err = _raw_items(pool, "fnv1a_bytes", n, _abi.FBR_ARGS_DEVICE | _abi.FBR_OUT_DEVICE, ptr.value,
                                  doffs.value, len(vals), out=dout.value)
            back = np.empty(n * 16, np.uint8)
            _abi.check(lib.fbr_memcpy_d2h(eng.handle, 0, back.ctypes.data, dout, back.nbytes))
            assert err[0] == 0 and np.array_equal(back, _bytes(want)), shift
        # bad device offsets: decreasing at task 5, past n_items at task 900 -- TASK_BADARG at the lowest, no fault
        for bad_task in (5, 900):
            b = o.copy()
            if bad_task == 5:
                b[6] = b[5] - 1
            else:
                b[901] = 10 ** 9
            _abi.check(lib.fbr_memcpy_h2d(eng.handle, 0, doffs, b.ctypes.data, b.nbytes))
            for flags in (0, _abi.FBR_VIA_RING):
                _, err = _raw_items(pool, "fnv1a_bytes", n, flags | _abi.FBR_ARGS_DEVICE, base.value, doffs.value, len(vals),
                                    chunksize=7)
                assert err == (_abi.FBR_TASK_BADARG, bad_task), (flags, err)
        # float64 rows at an 8 B (not 16 B) aligned base; a 4 B aligned one is refused
        rv, ro = _sub(*ROWS, 10_000)
        ro = ro.astype(np.uint64)
        rbase, roffs = ctypes.c_void_p(), ctypes.c_void_p()
        _abi.check(lib.fbr_device_alloc(eng.handle, 0, rv.nbytes + 64, ctypes.byref(rbase)))
        _abi.check(lib.fbr_device_alloc(eng.handle, 0, ro.nbytes + 64, ctypes.byref(roffs)))
        try:
            ptr = ctypes.c_void_p(rbase.value + 8)
            _abi.check(lib.fbr_memcpy_h2d(eng.handle, 0, ptr, rv.ctypes.data, rv.nbytes))
            _abi.check(lib.fbr_memcpy_h2d(eng.handle, 0, roffs, ro.ctypes.data, ro.nbytes))
            got, err = _raw_items(pool, "ragged_stats_f64", 10_000, _abi.FBR_ARGS_DEVICE, ptr.value, roffs.value, len(rv),
                                  chunksize=7)
            assert err[0] == 0 and np.array_equal(got, _bytes(RB.ragged_stats_np(rv, ro.astype(np.int64))))
            with pytest.raises(_abi.EngineError, match="8-byte aligned"):
                _raw_items(pool, "ragged_stats_f64", 10_000, _abi.FBR_ARGS_DEVICE, rbase.value + 4, roffs.value, len(rv))
        finally:
            lib.fbr_device_free(eng.handle, 0, rbase)
            lib.fbr_device_free(eng.handle, 0, roffs)
    finally:
        for p_ in (base, doffs, dout):
            lib.fbr_device_free(eng.handle, 0, p_)
    # host-resident bad offsets are refused before anything launches
    with pytest.raises(_abi.EngineError, match="decrease"):
        _raw_items(pool, "fnv1a_bytes", 2, 0, vals.ctypes.data, np.array([0, 5, 3], np.uint64).ctypes.data, 10)


def test_small_ring_cuts_waves_by_item_bytes():
    """Host items stream through two staging halves of ring_bytes: with 1 MiB halves a 5 MB map runs as many waves, each
    cut at a unit boundary by its item bytes, and a unit whose items alone exceed a half is refused before launch."""
    p = fiber_b200.Pool(1, devices=[0], ring_bytes=1 << 20)
    try:
        v, o = _sub(*STRINGS, 20_000)
        before = p.stats()
        _same(p.map(RB.fnv1a_bytes, fiber_b200.Ragged(v, o), 32), RB.fnv1a_np(v, o))
        st = p.stats()
        assert st["dispatch_launches"] - before["dispatch_launches"] >= v.nbytes // (1 << 20) + 1
        assert st["h2d_bytes"] - before["h2d_bytes"] >= v.nbytes + o.nbytes
        _same(p.map(RB.fnv1a_bytes, fiber_b200.Ragged(v, o), 7), RB.fnv1a_np(v, o))
        assert list(p.imap(RB.fnv1a_bytes, fiber_b200.Ragged(v, o)[:3000], 32)) == RB.fnv1a_np(*_sub(v, o, 3000)).tolist()
        ou = o.astype(np.uint64)
        for flags in (_abi.FBR_SHUFFLE, _abi.FBR_VIA_RING):
            got, err = _raw_items(p, "fnv1a_bytes", len(o) - 1, flags, v.ctypes.data, ou.ctypes.data, len(v), chunksize=7)
            assert err[0] == 0 and np.array_equal(got, _bytes(RB.fnv1a_np(v, o))), flags
        # a float64 head-less group body too
        rv, ro = _sub(*ROWS, 5000)
        _same(p.map(RB.ragged_stats_f64, fiber_b200.Ragged(rv, ro), 7), RB.ragged_stats_np(rv, ro))
        big = [b"a" * 10, np.random.default_rng(9).integers(0, 256, 2 << 20, dtype=np.uint8).tobytes(), b"b"]
        with pytest.raises(_abi.EngineError, match="ring_bytes"):
            p.map(RB.fnv1a_bytes, big)
        assert p.map(RB.fnv1a_bytes, [b"ok"]).tolist() == [RB.fnv1a_bytes(b"ok")]      # the pool still serves
    finally:
        p.terminate()
        p.join()


def test_results_on_device():
    p = fiber_b200.Pool(1, devices=[0], results="device")
    try:
        v, o = _sub(*ROWS, 20_000)
        want = RB.ragged_stats_np(v, o)
        res = p.map(RB.ragged_stats_f64, fiber_b200.Ragged(v, o))
        assert res.on_device and len(res) == len(want)
        _same(res, want)
    finally:
        p.terminate()
        p.join()


def test_resilient_pool_redispatches_lost_units():
    vals, offs = _sub(*STRINGS, 40_000)
    vals = vals.copy()
    for t in (0, 17, 30_001):
        if offs[t + 1] > offs[t]:
            vals[offs[t]] = 0xFF
    want = RB.fnv1a_np(vals, offs)
    p = fiber_b200.Pool(1, devices=[0], error_handling=True)
    try:
        _same(p.map(RB.fault_fnv1a_bytes, fiber_b200.Ragged(vals, offs)), want)
        assert p.stats()["units_redispatched"] > 0
        _same(p.map(RB.fault_fnv1a_bytes, fiber_b200.Ragged(vals, offs), 7), want)
    finally:
        p.terminate()
        p.join()


def test_process_isolated_pool():
    p = fiber_b200.Pool(2, isolation="process")
    try:
        v, o = _sub(*ROWS, 30_000)
        _same(p.map(RB.ragged_stats_f64, fiber_b200.Ragged(v, o)), RB.ragged_stats_np(v, o))
        docs = [b"abc", "déf", b""] * 1000
        assert p.map(RB.fnv1a_bytes, docs, 7).tolist() == [RB.fnv1a_bytes(d.encode() if isinstance(d, str) else d) for d in docs]
    finally:
        p.terminate()
        p.join()


def test_two_worker_pool():
    n = ctypes.c_int()
    _abi.check(_abi.load().fbr_device_count(ctypes.byref(n)))
    if n.value < 2:
        pytest.skip("needs two GPUs")
    p = fiber_b200.Pool(2)
    try:
        v, o = _sub(*STRINGS, 100_000)
        _same(p.map(RB.fnv1a_bytes, fiber_b200.Ragged(v, o), 7), RB.fnv1a_np(v, o))
    finally:
        p.terminate()
        p.join()
