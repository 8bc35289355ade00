"""GPU: multi-stream items record bodies -- two sorted uint32 lists, four streams of 1/2/4/8-byte integers with a head
record and a broadcast table, float64 pairs on a warp, and an emit body over two streams; every call form, skewed lengths,
direct placement and the result ring, device-resident streams, a staging cut decided by the second stream, resilient
re-dispatch, process isolation and a chain of maps.  Every result is compared bit for bit with the restatements in
tests/multi_items_bodies.py."""
import ctypes
from collections import Counter

import numpy as np
import pytest

import fiber_b200
from fiber_b200 import Columns, Ragged, _abi, registry

from . import emit_bodies as EB
from . import multi_items_bodies as M
from . import ragged_bodies  # noqa: F401  (fnv1a_bytes: a one-stream body for the stream-count checks)

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


A = M.sorted_lists(40_000, seed=1, empty_every=13)
B = M.sorted_lists(40_000, seed=2, max_len=16, empty_every=17)
WANT_AB = M.intersect_count_np(A, B)


@pytest.mark.parametrize("chunksize", [1, 7, 32])
def test_map_sizes(pool, chunksize):
    unit = _unit("intersect_count_u32", len(A), chunksize)
    sizes = sorted({n for n in (1, 7, unit - 1, unit + 1, 3 * unit + 5) if n > 0}) + ([len(A)] if chunksize == 32 else [])
    for n in sizes:
        _same(pool.starmap(M.intersect_count_u32, Columns(A[:n], B[:n]), chunksize), WANT_AB[:n])


def test_skewed_lengths(pool):
    """One stream empty while the other is long (longer than a claim unit's others together), and tasks empty in every
    stream."""
    rng = np.random.default_rng(3)
    long = np.sort(rng.integers(0, 1000, 200_000, dtype=np.uint32))
    empty = np.zeros(0, np.uint32)
    pairs = [(long, empty), (empty, long), (empty, empty), (long, long[::7].copy()), (empty, empty)] * 20
    want = M.intersect_count_np(Ragged(*_join([p[0] for p in pairs])), Ragged(*_join([p[1] for p in pairs])))
    for cs in (1, 7):
        _same(pool.starmap(M.intersect_count_u32, pairs, cs), want)
    only_empty = pool.starmap(M.intersect_count_u32, [(empty, empty)] * 1000)
    assert only_empty.tolist() == [(0, 0, 0)] * 1000
    # four streams, each empty on its own tasks
    w = rng.integers(0, 2 ** 32, 300, dtype=np.uint32)
    cols = [M.ragged_of(rng, 5000, d, 40, empty_every=e) for d, e in ((np.uint8, 2), (np.uint16, 3), (np.uint32, 5), (np.uint64, 7))]
    seeds = rng.integers(0, 2 ** 63, 5000, dtype=np.uint64)
    got = pool.starmap(M.mix4_u1_u2_u4_u8, [(w,) + tuple(c[i] for c in cols) + (seeds[i],) for i in range(5000)], 7)
    _same(got, M.mix4_np(w, cols, seeds))


def _join(arrays):
    offs = np.zeros(len(arrays) + 1, np.int64)
    np.cumsum([len(a) for a in arrays], out=offs[1:])
    return np.concatenate(arrays), offs


def test_call_forms(pool):
    n = 500
    a, b = [A[i] for i in range(n)], [B[i] for i in range(n)]
    want = WANT_AB[:n]
    f = M.intersect_count_u32
    _same(pool.starmap(f, list(zip(a, b)), 7), want)
    assert pool.starmap(f, list(zip(a[:20], b[:20]))).tolist() == [f(x.tolist(), y.tolist()) for x, y in zip(a[:20], b[:20])]
    assert pool.apply_async(f, (a[3],), {"b": b[3]}).get() == tuple(want[3].tolist())
    assert pool.apply(f, (), {"b": b[4], "a": a[4]}) == tuple(want[4].tolist())
    _same(pool.starmap(f, Columns(A[:n], B[:n])), want)
    with pytest.raises(TypeError, match=r"missing 1 required positional argument: 'b'"):
        pool.map(f, a[:3])
    with pytest.raises(TypeError, match=r"missing 1 required positional argument: 'b'"):
        list(pool.imap(f, a[:3]))
    # pair_dot on a warp, with its one-thread restatement of the lane order; rows of different lengths are bad arguments
    rng = np.random.default_rng(4)
    lens = rng.integers(0, 300, 2000)
    xs = [rng.standard_normal(k) for k in lens]
    ys = [rng.standard_normal(k) for k in lens]
    want = M.pair_dot_np(xs, ys)
    _same(pool.starmap(M.pair_dot_f64, list(zip(xs, ys)), 3), want)
    _same(pool.starmap(M.pair_dot_f64, Columns(Ragged(*_join(xs)), Ragged(*_join(ys)))), want)
    with pytest.raises(ValueError, match="bad argument in task 2"):
        pool.starmap(M.pair_dot_f64, [([1.0], [2.0]), ([], []), ([1.0, 2.0], [3.0]), ([1.0], [1.0, 2.0])])
    # the broadcast table from the pool initializer under Columns, from the tasks under starmap
    w = rng.integers(0, 2 ** 32, 1000, dtype=np.uint32)
    cols = [M.ragged_of(rng, 3000, d, 30) for d in (np.uint8, np.uint16, np.uint32, np.uint64)]
    seeds = rng.integers(0, 2 ** 63, 3000, dtype=np.uint64)
    want = M.mix4_np(w, cols, seeds)

    @fiber_b200.device_initializer("mix4_u1_u2_u4_u8")
    def init(w):
        pass

    p = fiber_b200.Pool(1, devices=[0], initializer=init, initargs=(w,))
    try:
        _same(p.starmap(M.mix4_u1_u2_u4_u8, Columns(*cols, seeds), 7), want)
        _same(p.starmap(M.mix4_u1_u2_u4_u8, Columns(*cols, list(seeds.tolist()))[:100]), want[:100])
    finally:
        p.terminate()
        p.join()
    kw = pool.apply(M.mix4_u1_u2_u4_u8, (w,), {"x0": cols[0][5], "x1": cols[1][5], "x2": cols[2][5], "x3": cols[3][5], "seed": seeds[5]})
    assert kw == (M.mix4_one(w, [c[5] for c in cols], int(seeds[5]), 0),) + tuple(len(c[5]) for c in cols)


def _raw(pool, name, n, flags, streams, chunksize=0, seed=11):
    """fbr_map_submit_items_n with `streams` = [(items pointer, offsets pointer, n_items)]: (result bytes, (err code, task))."""
    spec = registry.spec(name)
    eng = pool._engine
    d = _abi.MapDesc()
    d.func_id, d.flags, d.n_tasks, d.chunksize, d.shuffle_seed = spec.func_id, flags, n, chunksize, seed
    its = (_abi.ItemsDesc * len(streams))()
    for it, (items, offs, n_items), dt in zip(its, streams, spec.item_dtypes):
        it.items, it.offsets, it.n_items, it.item_bytes = items, offs, n_items, dt.itemsize
    seq = ctypes.c_uint64()
    _abi.check(eng.lib.fbr_map_submit_items_n(eng.handle, ctypes.byref(d), its, len(its), ctypes.byref(seq)))
    res = _abi.Result()
    rc = eng.lib.fbr_result_wait(eng.handle, seq.value, -1, ctypes.byref(res))
    if rc != _abi.FBR_ETASK:
        _abi.check(rc)
    data = None
    if res.err_code == 0:
        data = np.frombuffer((ctypes.c_char * (n * spec.result_bytes)).from_address(res.data), np.uint8).copy()
    err = (res.err_code, res.err_task)
    _abi.check(eng.lib.fbr_result_release(eng.handle, seq.value))
    return data, err


@pytest.mark.parametrize("flags", [_abi.FBR_SHUFFLE, _abi.FBR_VIA_RING, 0])
def test_ring_and_direct_placement(pool, flags):
    before = pool.stats()
    oa, ob = A.offsets.astype(np.uint64), B.offsets.astype(np.uint64)
    got, err = _raw(pool, "intersect_count_u32", len(A), flags,
                    [(A.values.ctypes.data, oa.ctypes.data, len(A.values)), (B.values.ctypes.data, ob.ctypes.data, len(B.values))], 7)
    assert err[0] == 0 and np.array_equal(got, _bytes(WANT_AB))
    st = pool.stats()
    if flags:
        assert st["gather_launches"] > before["gather_launches"]
    else:
        assert st["direct_waves"] > before["direct_waves"]
    # a stream-count mismatch either way round, and the one-stream entry point
    lib, h = pool._engine.lib, pool._engine.handle
    d, its, seq = _abi.MapDesc(), (_abi.ItemsDesc * 2)(), ctypes.c_uint64()
    d.func_id, d.n_tasks = registry.spec("intersect_count_u32").func_id, 1
    with pytest.raises(_abi.EngineError, match="takes 2 item streams, not 1"):
        _abi.check(lib.fbr_map_submit_items(h, ctypes.byref(d), its, ctypes.byref(seq)))
    d.func_id = registry.spec("fnv1a_bytes").func_id
    with pytest.raises(_abi.EngineError, match="takes 1 item stream, not 2"):
        _abi.check(lib.fbr_map_submit_items_n(h, ctypes.byref(d), its, 2, ctypes.byref(seq)))


def test_device_resident_streams(pool):
    """Both streams device-resident (offsets of stream 1 starting past 0), then bad offsets in stream 1 only."""
    eng = pool._engine
    lib = eng.lib
    n = 30_000
    bo = B.offsets[1000:1000 + n + 1].astype(np.uint64)              # offsets[0] != 0: a slice of the larger array
    want = M.intersect_count_np(A[:n], Ragged(B.values, B.offsets[1000:1000 + n + 1]))
    ptrs = []
    try:
        def put(arr):
            p = ctypes.c_void_p()
            _abi.check(lib.fbr_device_alloc(eng.handle, 0, max(16, arr.nbytes), ctypes.byref(p)))
            ptrs.append(p)
            _abi.check(lib.fbr_memcpy_h2d(eng.handle, 0, p, arr.ctypes.data, arr.nbytes))
            return p.value
        va, oa = put(A.values), put(A.offsets[:n + 1].astype(np.uint64))
        vb, ob = put(B.values), put(bo)
        for flags in (0, _abi.FBR_VIA_RING):
            got, err = _raw(pool, "intersect_count_u32", n, _abi.FBR_ARGS_DEVICE | flags,
                            [(va, oa, len(A.values)), (vb, ob, len(B.values))], 7)
            assert err[0] == 0 and np.array_equal(got, _bytes(want)), flags
        bad = bo.copy()
        bad[1235] = bad[1236] + 1                                   # stream 1 decreases at task 1235
        ob2 = put(bad)
        got, err = _raw(pool, "intersect_count_u32", n, _abi.FBR_ARGS_DEVICE, [(va, oa, len(A.values)), (vb, ob2, len(B.values))])
        assert err == (_abi.FBR_TASK_BADARG, 1235)
        bad = bo.copy()
        bad[n] = len(B.values) + 1                                   # the last task of stream 1 ends past n_items
        ob3 = put(bad)
        got, err = _raw(pool, "intersect_count_u32", n, _abi.FBR_ARGS_DEVICE, [(va, oa, len(A.values)), (vb, ob3, len(B.values))])
        assert err == (_abi.FBR_TASK_BADARG, n - 1)
    finally:
        for p in ptrs:
            lib.fbr_device_free(eng.handle, 0, p)


def test_small_ring_second_stream_cuts_waves():
    """With 1 MiB staging halves, a map whose stream 0 is tiny and whose stream 1 carries 2 KB per task runs as many waves
    as stream 1's bytes need, far more than stream 0 alone would; a unit whose two streams do not fit a half together is
    refused before launch."""
    rng = np.random.default_rng(6)
    n = 5000
    small = Ragged(np.arange(n, dtype=np.uint32), np.arange(n + 1))
    big_lists = [np.sort(rng.integers(0, 5000, 512, dtype=np.uint32)) for _ in range(n)]
    big = Ragged(*_join(big_lists))
    p = fiber_b200.Pool(1, devices=[0], ring_bytes=1 << 20)
    try:
        before = p.stats()
        _same(p.starmap(M.intersect_count_u32, Columns(small, small), 32), M.intersect_count_np(small, small))
        mid = p.stats()
        _same(p.starmap(M.intersect_count_u32, Columns(small, big), 32), M.intersect_count_np(small, big))
        st = p.stats()
        alone = mid["dispatch_launches"] - before["dispatch_launches"]
        both = st["dispatch_launches"] - mid["dispatch_launches"]
        assert both >= big.values.nbytes // (1 << 20) + 1 and both > alone, (alone, both)
        assert st["h2d_bytes"] - mid["h2d_bytes"] >= big.values.nbytes + small.values.nbytes
        huge = [np.zeros(1, np.uint32), np.zeros(300_000, np.uint32)]
        with pytest.raises(_abi.EngineError, match="ring_bytes"):
            p.starmap(M.intersect_count_u32, [(huge[0], huge[0]), (huge[0], huge[1]), (huge[0], huge[0])])
        assert p.starmap(M.intersect_count_u32, [([1, 2], [2])]).tolist() == [(1, 2, 1)]      # the pool still serves
    finally:
        p.terminate()
        p.join()


def test_results_on_device():
    p = fiber_b200.Pool(1, devices=[0], results="device")
    try:
        res = p.starmap(M.intersect_count_u32, Columns(A, B))
        assert res.on_device and len(res) == len(A)
        _same(res, WANT_AB)
        r = p.starmap(M.sorted_common_u32, Columns(A[:3000], B[:3000]))
        assert r == M.sorted_common_py(A[:3000], B[:3000])
    finally:
        p.terminate()
        p.join()


def test_resilient_pool_redispatches_lost_units():
    p = fiber_b200.Pool(1, devices=[0], error_handling=True)
    try:
        _same(p.starmap(M.fault_intersect_count_u32, Columns(A, B)), WANT_AB)
        assert p.stats()["units_redispatched"] > 0
        _same(p.starmap(M.fault_intersect_count_u32, Columns(A, B), 7), WANT_AB)
    finally:
        p.terminate()
        p.join()


def test_process_isolated_pool():
    p = fiber_b200.Pool(2, isolation="process")
    try:
        _same(p.starmap(M.intersect_count_u32, Columns(A, B)), WANT_AB)
        assert p.starmap(M.sorted_common_u32, Columns(A[:2000], B[:2000]), 7) == M.sorted_common_py(A[:2000], B[:2000])
    finally:
        p.terminate()
        p.join()


@pytest.mark.parametrize("n", [2047, 2048, 2049, 300_000])
def test_emit_sizes_around_the_scan_tile(pool, n):
    a = M.sorted_lists(n, seed=10 + n % 7, max_len=24, empty_every=11)
    b = M.sorted_lists(n, seed=20 + n % 5, max_len=24, empty_every=9)
    want = M.sorted_common_py(a, b)
    r = pool.starmap(M.sorted_common_u32, Columns(a, b), 7)
    lens = np.array([len(x) for x in want], np.int64)
    offs = np.zeros(n + 1, np.uint64)
    np.cumsum(lens, out=offs[1:])
    vals = np.array([v for x in want for v in x], np.uint32)
    assert np.array_equal(np.asarray(r.ragged.offsets, np.uint64), offs)
    assert np.array_equal(r.ragged.values, vals)
    if n < 3000:
        assert r == want


def _sorted_segments(rg):
    """Each task's values sorted, on the host: one lexsort by (value, task)."""
    o = np.asarray(rg.offsets, np.int64)
    task = np.repeat(np.arange(len(o) - 1), np.diff(o))
    order = np.lexsort((rg.values, task))
    return Ragged(rg.values[order], o)


def test_chain_tokenize_then_intersect(pool):
    docs_a = EB.documents(5000, seed=31, max_words=30)
    docs_b = EB.documents(5000, seed=32, max_words=30)
    r1, r2 = pool.map(EB.tokens_u32, docs_a), pool.map(EB.tokens_u32, docs_b)
    s1, s2 = _sorted_segments(r1.ragged), _sorted_segments(r2.ragged)
    got = pool.starmap(M.intersect_count_u32, Columns(s1, s2), 7)
    want = [(sum((Counter(x) & Counter(y)).values()), len(x), len(y)) for x, y in zip(r1, r2)]
    assert got.tolist() == want


def test_two_worker_pool():
    n = ctypes.c_int()
    _abi.check(_abi.load().fbr_device_count(ctypes.byref(n)))
    if n.value < 2:
        pytest.skip("needs two GPUs")
    p = fiber_b200.Pool(2)
    try:
        _same(p.starmap(M.intersect_count_u32, Columns(A, B), 7), WANT_AB)
    finally:
        p.terminate()
        p.join()
