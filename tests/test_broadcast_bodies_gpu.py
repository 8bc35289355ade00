"""GPU: record bodies that read a broadcast block -- blocks on both sides of the shared-memory staging budget, every map
form, the pool initializer (threads and worker processes), direct placement and the result ring, device-resident
blocks at unaligned addresses and the engine's size checks.  Results are compared bit for bit with the NumPy
restatements in tests/broadcast_bodies.py, and with the Python definitions at small n."""
import ctypes

import numpy as np
import pytest

import fiber_b200
from fiber_b200 import _abi, registry

from . import broadcast_bodies as BB

pytestmark = pytest.mark.gpu


@fiber_b200.device_initializer("table_mix_u32")
def set_table(table):
    raise RuntimeError("runs on the GPU workers")


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


# K = 512 fills the 32 KB budget exactly; 513 and 4096 centroids are read from global memory
@pytest.mark.parametrize("k", [1, 3, 64, 512, 513, 4096])
def test_nearest_centroid_block_sizes(k):
    C = BB.centroids(k, seed=k)
    n = 4099 if k == 4096 else 30011
    P = BB.points(n, seed=k + 1)
    want = BB.nearest_np(P, C)
    p = fiber_b200.Pool(1, devices=[0], initializer=BB.set_centroids, initargs=(C,))
    try:
        _same(p.map(BB.nearest_centroid_f32, P), want)                 # the initializer's block
        _same(p.map(BB.nearest_centroid_f32, P, 7), want)
        pts = [tuple(r) for r in P["p"][:300]]
        _same(p.starmap(BB.nearest_centroid_global_f32, [(C["c"], q) for q in pts]), want[:300])   # never staged
        assert p.starmap(BB.nearest_centroid_f32, [(C, q) for q in P["p"][:40]]) == \
            [BB.nearest_centroid_f32(C, q) for q in P["p"][:40]]
    finally:
        p.terminate()
        p.join()


def test_map_forms(pool):
    C = BB.centroids(100, seed=5)
    P = BB.points(3001, seed=6)
    want = BB.nearest_np(P, C)
    _same(pool.starmap(BB.nearest_centroid_f32, [(C, q) for q in P["p"]], 7), want)
    assert pool.apply_async(BB.nearest_centroid_f32, (C, P["p"][3])).get() == tuple(want[3].tolist())
    assert pool.apply(BB.nearest_centroid_f32, (P["p"][4],), {"centroids": C["c"]}) == tuple(want[4].tolist())
    handles = [pool.apply_async(BB.nearest_centroid_f32, (C, q)) for q in P["p"][:200]]
    assert [h.get() for h in handles] == want[:200].tolist()
    p = fiber_b200.Pool(1, devices=[0], initializer=BB.set_centroids, initargs=(C,))
    try:
        assert list(p.imap(BB.nearest_centroid_f32, P, 5)) == want.tolist()
        assert sorted(p.imap_unordered(BB.nearest_centroid_f32, P[:700], 3)) == sorted(want[:700].tolist())
        assert p.apply(BB.nearest_centroid_f32, (P["p"][9],)) == tuple(want[9].tolist())   # initializer block
    finally:
        p.terminate()
        p.join()
    with pytest.raises(TypeError, match="no initializer block"):
        pool.map(BB.nearest_centroid_f32, P)
    C2 = C.copy()
    C2["c"][0, 0] += 1.0
    with pytest.raises(ValueError, match="must share"):
        pool.starmap(BB.nearest_centroid_f32, [(C, P["p"][0]), (C2, P["p"][1])])


@pytest.mark.parametrize("size", [1, 3, 5, 1 << 20])
def test_table_mix(size):
    """Tables whose bytes are not a multiple of 16 (4, 12, 20 B: copied by hand into shared memory) and a 4 MiB one
    (global memory), over range() indices and explicit int64 arguments."""
    tab = BB.table(size, seed=size)
    p = fiber_b200.Pool(1, devices=[0], initializer=set_table, initargs=(tab,))
    try:
        for r in (range(0, 300007), range(-5, 2 ** 40, 2 ** 31 + 7), range(7, 8)):
            idx = np.arange(r.start, r.stop, r.step, dtype=np.int64)[:len(r)]
            _same(p.map(BB.table_mix_u32, r, 7), BB.table_mix_np(idx, tab))
        xs = np.random.default_rng(size).integers(-2 ** 63, 2 ** 63 - 1, 5003, dtype=np.int64)
        _same(p.map(BB.table_mix_u32, xs), BB.table_mix_np(xs, tab))
        assert p.starmap(BB.table_mix_u32, [(tab, int(i)) for i in xs[:50]]) == [BB.table_mix_u32(tab, int(i)) for i in xs[:50]]
    finally:
        p.terminate()
        p.join()


def _raw(pool, name, n, flags, shared, shared_bytes, args=None, arg_stride=0, out=None, chunksize=0, seed=11):
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


def _put(pool, arr):
    h = ctypes.c_uint64()
    buf = np.ascontiguousarray(arr)
    _abi.check(pool._engine.lib.fbr_shared_put(pool._engine.handle, buf.ctypes.data, buf.nbytes, ctypes.byref(h)))
    return h.value


@pytest.mark.parametrize("flags", [_abi.FBR_SHUFFLE, _abi.FBR_VIA_RING, 0])
def test_ring_and_direct_placement(pool, flags):
    before = pool.stats()
    H = _abi.FBR_SHARED_HANDLE
    for k in (64, 600):                                               # staged, global
        C = BB.centroids(k, seed=k)
        P = BB.points(100003, seed=3)
        h = _put(pool, C)
        got = _raw(pool, "nearest_centroid_f32", len(P), flags | H, h, C.nbytes, P.ctypes.data, 64, chunksize=7)
        assert np.array_equal(got, _bytes(BB.nearest_np(P, C))), k
        pool._engine.lib.fbr_shared_drop(pool._engine.handle, h)
    for size in (5, 1 << 20):
        tab = BB.table(size, seed=1)
        h = _put(pool, tab)
        got = _raw(pool, "table_mix_u32", 200003, flags | H, h, tab.nbytes)
        assert np.array_equal(got, _bytes(BB.table_mix_np(np.arange(200003), tab))), size
        pool._engine.lib.fbr_shared_drop(pool._engine.handle, h)
    st = pool.stats()
    if flags:
        assert st["gather_launches"] > before["gather_launches"]
    else:
        assert st["direct_waves"] > before["direct_waves"]


def test_results_on_device():
    C = BB.centroids(300, seed=8)
    P = BB.points(50021, seed=9)
    want = BB.nearest_np(P, C)
    p = fiber_b200.Pool(1, devices=[0], results="device", initializer=BB.set_centroids, initargs=(C,))
    try:
        res = p.map(BB.nearest_centroid_f32, P)
        assert res.on_device and len(res) == len(P)
        assert res[3] == tuple(want[3].tolist()) and res[4095:4113] == want[4095:4113].tolist()
        _same(res, want)
    finally:
        p.terminate()
        p.join()


def test_device_pointer_block_at_unaligned_base(pool):
    """A FBR_ARGS_DEVICE block is the caller's device pointer: at a base that is not 16 B aligned nothing is bulk-loaded,
    the consumers copy it word by word, and no byte past shared_bytes is read."""
    eng = pool._engine
    lib = eng.lib
    n = 70001
    P = BB.points(n, seed=12)
    xs = np.random.default_rng(13).integers(-2 ** 40, 2 ** 40, n, dtype=np.int64)
    d_args, d_blk = ctypes.c_void_p(), ctypes.c_void_p()
    _abi.check(lib.fbr_device_alloc(eng.handle, 0, n * 64, ctypes.byref(d_args)))
    _abi.check(lib.fbr_device_alloc(eng.handle, 0, (1 << 22) + 64, ctypes.byref(d_blk)))
    try:
        _abi.check(lib.fbr_memcpy_h2d(eng.handle, 0, d_args, P.ctypes.data, n * 64))
        for k in (1, 3, 64, 512):                                    # staged: the body's 16 B elements land aligned
            C = BB.centroids(k, seed=k)
            for off in (4, 16, 0):
                base = ctypes.c_void_p(d_blk.value + off)
                _abi.check(lib.fbr_memcpy_h2d(eng.handle, 0, base, C.ctypes.data, C.nbytes))
                got = _raw(pool, "nearest_centroid_f32", n, _abi.FBR_ARGS_DEVICE, base.value, C.nbytes, d_args.value, 64)
                assert np.array_equal(got, _bytes(BB.nearest_np(P, C))), (k, off)
        _abi.check(lib.fbr_memcpy_h2d(eng.handle, 0, d_args, xs.ctypes.data, n * 8))
        for size in (1, 3, 5, 4096, 4097, 1 << 20):                   # uint32 elements: any 4 B aligned base
            tab = BB.table(size, seed=size)
            for off in (4, 8, 12):
                base = ctypes.c_void_p(d_blk.value + off)
                _abi.check(lib.fbr_memcpy_h2d(eng.handle, 0, base, tab.ctypes.data, tab.nbytes))
                for flags in (0, _abi.FBR_VIA_RING):
                    got = _raw(pool, "table_mix_u32", n, flags | _abi.FBR_ARGS_DEVICE, base.value, tab.nbytes, d_args.value, 8)
                    assert np.array_equal(got, _bytes(BB.table_mix_np(xs, tab))), (size, off, flags)
    finally:
        lib.fbr_device_free(eng.handle, 0, d_args)
        lib.fbr_device_free(eng.handle, 0, d_blk)


def test_block_size_checks(pool):
    eng = pool._engine
    C = BB.centroids(8)
    P = BB.points(10)
    h = _put(pool, C)
    spec = registry.spec("nearest_centroid_f32")
    try:
        for shared, nbytes, flags, why in ((h, C.nbytes - 4, _abi.FBR_SHARED_HANDLE, "whole number"),
                                           (h, C.nbytes + 64, _abi.FBR_SHARED_HANDLE, "exceeds"),
                                           (h, 0, _abi.FBR_SHARED_HANDLE, "needs a broadcast block"),
                                           (None, 0, 0, "needs a broadcast block")):
            d = _abi.MapDesc()
            d.func_id, d.flags, d.n_tasks, d.args, d.arg_stride = spec.func_id, flags, len(P), P.ctypes.data, 64
            d.shared, d.shared_bytes = shared, nbytes
            seq = ctypes.c_uint64()
            assert eng.lib.fbr_map_submit(eng.handle, ctypes.byref(d), ctypes.byref(seq)) == _abi.FBR_EINVAL
            assert why in eng.lib.fbr_last_error().decode()
        # the same block at its recorded size runs
        assert np.array_equal(_raw(pool, "nearest_centroid_f32", len(P), _abi.FBR_SHARED_HANDLE, h, C.nbytes, P.ctypes.data, 64),
                              _bytes(BB.nearest_np(P, C)))
    finally:
        eng.lib.fbr_shared_drop(eng.handle, h)


def test_initializer_uploads_once_per_device():
    n_dev = ctypes.c_int(0)
    _abi.check(_abi.load().fbr_device_count(ctypes.byref(n_dev)))
    C = BB.centroids(4096, seed=21)                                   # 256 KB
    P = BB.points(200, seed=22)
    want = BB.nearest_np(P, C)
    p = fiber_b200.Pool(2, initializer=BB.set_centroids, initargs=(C,))
    try:
        for _ in range(3):
            _same(p.map(BB.nearest_centroid_f32, P, 1), want)
        _same(p.starmap(BB.nearest_centroid_f32, [(C, q) for q in P["p"]]), want)
        assert [h.get() for h in [p.apply_async(BB.nearest_centroid_f32, (C, q)) for q in P["p"][:20]]] == want[:20].tolist()
        workers = min(2, n_dev.value)
        # the 256 KB block went up once per device; the rest is 12.8 KB of points per map and 20 single records
        assert p.stats()["h2d_bytes"] < workers * C.nbytes + 4 * P.nbytes + 20 * 4096
    finally:
        p.terminate()
        p.join()


def test_process_isolation_runs_the_initializer_in_every_worker(golden):
    C = BB.centroids(200, seed=31)
    P = BB.points(70001, seed=32)
    p = fiber_b200.Pool(2, isolation="process", initializer=BB.set_centroids, initargs=(C,))
    try:
        _same(p.map(BB.nearest_centroid_f32, P), BB.nearest_np(P, C))
        assert p.starmap(BB.nearest_centroid_f32, [(C, q) for q in P["p"][:3]]) == BB.nearest_np(P[:3], C).tolist()
    finally:
        p.terminate()
        p.join()
    # the compiled-in parzen body's initializer too
    from examples import workloads as W
    from oracle import bodies as B
    xs, px, widths = B.parzen_example_inputs()
    want = [(float.fromhex(h), float.fromhex(d)) for h, d in golden("parzen_102")["results_hex"]]
    p = fiber_b200.Pool(2, isolation="process", initializer=W.set_parzen_samples, initargs=(xs, px))
    try:
        assert sorted(p.map(W.parzen_at, widths, 1)) == want
    finally:
        p.terminate()
        p.join()


def test_kde_window_matches_the_parzen_golden(pool, golden):
    """examples/parzen_estimation.py written as a user body: 10 000 x 2 float64 samples (160 KB, read from global
    memory), 102 widths; the results equal the reference's to the last bit."""
    from oracle import bodies as B
    xs, px, widths = B.parzen_example_inputs()
    assert not px.any()
    want = [(float.fromhex(h), float.fromhex(d)) for h, d in golden("parzen_102")["results_hex"]]
    handles = [pool.apply_async(BB.kde_window_f64, (xs, w)) for w in widths]
    assert sorted(h.get() for h in handles) == want
    assert sorted(pool.starmap(BB.kde_window_f64, [(xs, w) for w in widths], 1)) == want
    p = fiber_b200.Pool(1, devices=[0], initializer=BB.set_samples, initargs=(xs,))
    try:
        assert sorted(p.map(BB.kde_window_f64, widths)) == want
        # a sample set small enough to stage: against the NumPy restatement and the Python definition
        few = xs[:700]
        _same(pool.starmap(BB.kde_window_f64, [(few, w) for w in widths]), BB.kde_np(widths, few))
        assert pool.starmap(BB.kde_window_f64, [(few, w) for w in widths[:10]]) == [BB.kde_window_f64(few, w) for w in widths[:10]]
    finally:
        p.terminate()
        p.join()
