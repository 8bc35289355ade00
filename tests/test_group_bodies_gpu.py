"""GPU: group record bodies (kGroup) through dispatch_record_kernel -- 8 KB and 32 KB rows on a warp per task, 8 KB
results per range() index, four-lane groups over 80 B records and a group body with a broadcast block; every map form,
direct placement and the result ring, device-resident results, strided and unaligned device buffers, resilient
re-dispatch and process isolation.  Every result is compared bit for bit with the NumPy restatement in
tests/group_bodies.py, which repeats each body's order of operations, and with the Python definitions at small n."""
import ctypes

import numpy as np
import pytest

import fiber_b200
from fiber_b200 import _abi, registry

from . import group_bodies as GB

pytestmark = pytest.mark.gpu

# body -> (Python definition, seeded argument records, NumPy restatement, the large n: about 100 MB of records)
CASES = {
    "row_moments_f64": (GB.row_moments_f64, GB.moments_args, GB.row_moments_np, 12007),
    "wide_row_max_f32": (GB.wide_row_max_f32, GB.wide_args, GB.wide_row_max_np, 3001),
    "mat4_apply_f32": (GB.mat4_apply_f32, GB.mat4_args, GB.mat4_np, 10 ** 6),
}
_ARGS = {}


def _args(name, n):
    """The first n records of one seeded array per body (made once: the large ones take a while)."""
    _, make, _, big = CASES[name]
    if name not in _ARGS:
        _ARGS[name] = make(big, seed=1)
    return _ARGS[name][:n]


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


def _sizes(name, big, chunksize):
    unit = _unit(name, big, chunksize)
    return sorted({n for n in (1, 7, unit - 1, unit + 1, big) if n > 0})


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("chunksize", [1, 7, 32])
def test_map_sizes(pool, name, chunksize):
    func, _, ref, big = CASES[name]
    spec = registry.spec(name)
    for n in _sizes(name, big, chunksize):
        args = _args(name, n)
        res = pool.map(func, args, chunksize)
        _same(res, ref(args))
        if n <= 40:
            fields = [args[f] for f in args.dtype.names]
            assert res.tolist() == [func(*[f[i] for f in fields]) for i in range(n)] == spec.rows_to_list(ref(args))


@pytest.mark.parametrize("chunksize", [1, 7, 32])
def test_index_body_over_range(pool, chunksize):
    big = 12007                                                      # 8 KB results per index: 98 MB
    for n in _sizes("splitmix_row_u32", big, chunksize):
        for start, step in ((0, 1), (-(2 ** 40), 3)):
            r = range(start, start + n * step, step)
            res = pool.map(GB.splitmix_row_u32, r, chunksize)
            _same(res, GB.splitmix_row_np(np.arange(start, start + n * step, step, dtype=np.int64)))
    assert pool.map(GB.splitmix_row_u32, range(-2, 3)).tolist() == [GB.splitmix_row_u32(i) for i in range(-2, 3)]
    # explicit int64 arguments go through the staged argument path (the kIndex = false instantiation)
    xs = np.random.default_rng(1).integers(-2 ** 63, 2 ** 63 - 1, 5001, dtype=np.int64)
    _same(pool.map(GB.splitmix_row_u32, xs, 7), GB.splitmix_row_np(xs))


def test_map_forms(pool):
    # map over a plain 2-D array: one task per row, passed without a copy
    rows = _args("row_moments_f64", 301)["x"]
    want = GB.row_moments_np(_args("row_moments_f64", 301))
    _same(pool.map(GB.row_moments_f64, rows), want)
    wide = np.ascontiguousarray(_args("wide_row_max_f32", 50)["x"])
    _same(pool.map(GB.wide_row_max_f32, wide, 7), GB.wide_row_max_np(_args("wide_row_max_f32", 50)))
    # starmap, apply_async, imap over the four-lane body
    m = _args("mat4_apply_f32", 3001)
    mwant = GB.mat4_np(m)
    spec = registry.spec("mat4_apply_f32")
    pairs = [(r["m"], r["v"]) for r in m]
    _same(pool.starmap(GB.mat4_apply_f32, pairs, 7), mwant)
    assert pool.starmap(GB.mat4_apply_f32, [(a.tolist(), b.tolist()) for a, b in pairs[:20]]) == \
        [GB.mat4_apply_f32(a, b) for a, b in pairs[:20]]
    assert pool.apply_async(GB.mat4_apply_f32, (m["m"][3],), {"v": m["v"][3]}).get() == spec.rows_to_list(mwant[3:4])[0]
    handles = [pool.apply_async(GB.row_moments_f64, (r,)) for r in rows[:40]]
    assert [h.get() for h in handles] == want[:40].tolist()
    assert list(pool.imap(GB.mat4_apply_f32, m, 1)) == spec.rows_to_list(mwant)
    assert list(pool.imap(GB.row_moments_f64, rows, 32)) == want.tolist()
    assert sorted(pool.imap_unordered(GB.row_moments_f64, rows[:100], 3)) == sorted(want[:100].tolist())


def _raw(pool, name, n, flags, args=None, arg_stride=0, out=None, chunksize=0, seed=11, shared=None, shared_bytes=0):
    """One map through the C ABI; returns the result bytes (host results) or None (FBR_OUT_DEVICE)."""
    spec = registry.spec(name)
    eng = pool._engine
    d = _abi.MapDesc()
    d.func_id, d.flags, d.n_tasks, d.chunksize, d.shuffle_seed = spec.func_id, flags, n, chunksize, seed
    d.shared, d.shared_bytes = shared, shared_bytes
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
    """32 B, 16 B, 20 B and 8 KB slots placed by index through the result ring (shuffled arrival, or FBR_VIA_RING) and
    directly."""
    before = pool.stats()
    for name in sorted(CASES):
        _, _, ref, big = CASES[name]
        args = _args(name, big)
        got = _raw(pool, name, big, flags, args.ctypes.data, args.itemsize, chunksize=7)
        assert np.array_equal(got, _bytes(ref(args))), name
    got = _raw(pool, "splitmix_row_u32", 10007, flags, chunksize=7)
    assert np.array_equal(got, _bytes(GB.splitmix_row_np(np.arange(10007))))
    st = pool.stats()
    if flags:
        assert st["gather_launches"] > before["gather_launches"]
    else:
        assert st["direct_waves"] > before["direct_waves"]


def test_strided_unaligned_device_buffers(pool):
    """Device-resident argument records 4 B further apart than their size, from a base that is 4 B but not 16 B
    aligned, into a result buffer at the same kind of address: the consumers gather the records by hand."""
    eng = pool._engine
    lib = eng.lib
    for name, n in (("row_moments_f64", 2001), ("wide_row_max_f32", 501), ("mat4_apply_f32", 100003)):
        _, _, ref, _ = CASES[name]
        args = _args(name, n)
        A, R = args.itemsize, registry.spec(name).result_bytes
        wide = np.zeros(n, [("rec", args.dtype), ("pad", "<u4")])         # stride A + 4
        wide["rec"] = args
        want = _bytes(ref(args))
        base_in, base_out = ctypes.c_void_p(), ctypes.c_void_p()
        _abi.check(lib.fbr_device_alloc(eng.handle, 0, wide.nbytes + 64, ctypes.byref(base_in)))
        _abi.check(lib.fbr_device_alloc(eng.handle, 0, n * R + 64, ctypes.byref(base_out)))
        try:
            a_ptr, o_ptr = base_in.value + 4, base_out.value + 4
            _abi.check(lib.fbr_memcpy_h2d(eng.handle, 0, ctypes.c_void_p(a_ptr), wide.ctypes.data, wide.nbytes))
            for flags in (0, _abi.FBR_VIA_RING):
                _raw(pool, name, n, flags | _abi.FBR_ARGS_DEVICE | _abi.FBR_OUT_DEVICE, a_ptr, A + 4, out=o_ptr, chunksize=5)
                got = np.empty(n * R, np.uint8)
                _abi.check(lib.fbr_memcpy_d2h(eng.handle, 0, got.ctypes.data, ctypes.c_void_p(o_ptr), n * R))
                assert np.array_equal(got, want), (name, flags)
        finally:
            lib.fbr_device_free(eng.handle, 0, base_in)
            lib.fbr_device_free(eng.handle, 0, base_out)
        # the same stride from host memory
        assert np.array_equal(_raw(pool, name, n, 0, wide.ctypes.data, A + 4, chunksize=7), want), name


def test_results_on_device():
    p = fiber_b200.Pool(1, devices=[0], results="device")
    try:
        for name in ("row_moments_f64", "wide_row_max_f32", "mat4_apply_f32"):
            func, _, ref, _ = CASES[name]
            args = _args(name, 2001)
            want = ref(args)
            res = p.map(func, args)
            assert res.on_device and len(res) == len(args)
            rows = registry.spec(name).rows_to_list(want)
            assert res[3] == rows[3] and res[-1] == rows[-1] and res[1:4] == rows[1:4]
            _same(res, want)
        res = p.map(GB.splitmix_row_u32, range(1000))
        _same(res, GB.splitmix_row_np(np.arange(1000)))
    finally:
        p.terminate()
        p.join()


def test_resilient_pool_redispatches_lost_units():
    args = GB.moments_args(4001, seed=6)
    args["x"][[0, 5, 2222, 4000], 1023] = -1.0            # these tasks lose their unit on its first attempt
    want = GB.row_moments_np(args)
    p = fiber_b200.Pool(1, devices=[0], error_handling=True)
    try:
        _same(p.map(GB.fault_row_moments_f64, args), want)
        assert p.stats()["units_redispatched"] > 0
        _same(p.map(GB.fault_row_moments_f64, args, 7), want)
        assert p.map(GB.fault_row_moments_f64, args[:10]).tolist() == [GB.row_moments_f64(r) for r in args["x"][:10]]
    finally:
        p.terminate()
        p.join()
    plain = fiber_b200.Pool(1, devices=[0])
    try:
        # without error_handling a lost unit is a task error, reported at the first task of the lowest lost unit
        with pytest.raises(RuntimeError, match="task 0 failed with device error code 3"):
            plain.map(GB.fault_row_moments_f64, args, 32)
    finally:
        plain.terminate()
        plain.join()


def test_process_isolated_pool():
    """The worker processes register the group body modules themselves."""
    p = fiber_b200.Pool(2, isolation="process")
    try:
        args = _args("row_moments_f64", 3001)
        _same(p.map(GB.row_moments_f64, args), GB.row_moments_np(args))
        m = _args("mat4_apply_f32", 20001)
        _same(p.map(GB.mat4_apply_f32, m, 7), GB.mat4_np(m))
    finally:
        p.terminate()
        p.join()


# 128 centroids of 256 B fill the 32 KB staging budget exactly; 129 and 300 are read from global memory
@pytest.mark.parametrize("k", [1, 37, 128, 129, 300])
def test_broadcast_group_body(k):
    C = GB.centroids64(k, seed=k)
    P = GB.points64(20011, seed=k + 1)
    want = GB.nearest64_np(P, C)
    p = fiber_b200.Pool(1, devices=[0], initializer=GB.set_centroids64, initargs=(C,))
    try:
        _same(p.map(GB.nearest_row_group_f32, P), want)                 # the initializer's block
        _same(p.map(GB.nearest_row_group_f32, P["p"], 7), want)          # plain (n, 64) rows
        _same(p.starmap(GB.nearest_row_group_f32, [(C, q) for q in P["p"][:300]], 1), want[:300])
        assert p.apply_async(GB.nearest_row_group_f32, (C, P["p"][5])).get() == tuple(want[5].tolist()) == \
            GB.nearest_row_group_f32(C, P["p"][5])
    finally:
        p.terminate()
        p.join()


@pytest.mark.parametrize("flags", [_abi.FBR_SHUFFLE, _abi.FBR_VIA_RING, 0])
def test_broadcast_group_body_placement(pool, flags):
    eng = pool._engine
    for k in (100, 200):                                                # staged, global
        C = GB.centroids64(k, seed=k)
        P = GB.points64(30011, seed=3)
        h = ctypes.c_uint64()
        _abi.check(eng.lib.fbr_shared_put(eng.handle, C.ctypes.data, C.nbytes, ctypes.byref(h)))
        got = _raw(pool, "nearest_row_group_f32", len(P), flags | _abi.FBR_SHARED_HANDLE, P.ctypes.data, P.itemsize,
                   chunksize=7, shared=h.value, shared_bytes=C.nbytes)
        eng.lib.fbr_shared_drop(eng.handle, h.value)
        assert np.array_equal(got, _bytes(GB.nearest64_np(P, C))), k
