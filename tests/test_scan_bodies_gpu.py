"""GPU: accumulate maps (Pool.accumulate / staraccumulate, FBR_SCAN) of the fold bodies in tests/fold_bodies.py and the scan
bodies in tests/scan_bodies.py.  Every record is compared byte for byte (NaN-aware, as same_record) with the Python
restatement of run, combine and the prefix order, and sampled records with Pool.fold of the same prefix."""
import ctypes
import os

import numpy as np
import pytest

import fiber_b200
from fiber_b200 import _abi, registry

from . import fold_bodies as FB
from . import scan_bodies as SB
from .test_fold_bodies_gpu import QUERY, inputs as fold_inputs, run_all as fold_run_all, set_query  # noqa: F401

pytestmark = pytest.mark.gpu

SMALL_RING = 256 << 10


@pytest.fixture(scope="module")
def pool():
    p = fiber_b200.Pool(1, devices=[0], initializer=set_query, initargs=(QUERY,))
    yield p
    p.terminate()
    p.join()


@pytest.fixture(scope="module")
def small():
    p = fiber_b200.Pool(1, devices=[0], ring_bytes=SMALL_RING, initializer=set_query, initargs=(QUERY,))
    yield p
    p.terminate()
    p.join()


def fold_unit(name, n, ring_bytes=0):
    plan = _abi.Plan()
    _abi.check(_abi.load().fbr_plan_query(registry.spec(name).func_id, max(n, 1), _abi.FBR_PLAN_FOLD, ring_bytes, 1, 0, 132,
                                          ctypes.byref(plan)))
    return plan.unit_tasks


COMBINE = dict({k: v[0] for k, v in FB.RESTATED.items()}, affine_f64=SB.affine_combine, mix4k_u32=SB.mix4k_combine)
BODY = {"affine_f64": SB.affine_f64, "mix4k_u32": SB.mix4k_u32}


def inputs(name, n, seed):
    if name == "affine_f64":
        rng = np.random.default_rng(seed)
        xs = np.zeros(n, SB.AFFINE_ARG)
        xs["a"] = rng.uniform(0.5, 1.0, n)
        xs["b"] = rng.standard_normal(n)
        return xs
    if name == "mix4k_u32":
        return range(seed, seed + n)
    return fold_inputs(name, n, seed)


def run_all(name, xs):
    if name == "affine_f64":
        return [(float(a), float(b)) for a, b in xs.tolist()]
    if name == "mix4k_u32":
        return [SB.mix4k_run(i) for i in xs]
    return fold_run_all(name, xs)


def want_prefixes(name, xs):
    if name in ("sum_sq_idx_u64", "fault_count_u64"):     # mod 2^64 addition: any bracketing gives the same bits
        r = np.array(run_all(name, xs), np.uint64)
        return np.cumsum(r, dtype=np.uint64).tolist()
    return SB.prefix_folds(run_all(name, xs), COMBINE[name])


def body(name):
    return BODY.get(name) or getattr(FB, name)


def accumulate(p, name, xs):
    if name == "pair_overlap_u32":
        return p.staraccumulate(body(name), xs)
    return p.accumulate(body(name), xs)


def fold_raw(p, name, xs):
    r = p.starfold_async(body(name), xs) if name == "pair_overlap_u32" else p.fold_async(body(name), xs)
    r.get()
    return r.raw


def raw_records(res, R):
    a = np.ascontiguousarray(np.asarray(res)).view(np.uint8).reshape(-1)
    return [a[i * R:(i + 1) * R].tobytes() for i in range(len(a) // R)]


def norm(name, rec):
    if name in ("byte_hist_u8", "mix4k_u32"):
        return list(rec)
    return rec


def check_all(name, got, want):
    got = list(got)
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert FB.same_record(norm(name, g), norm(name, w)), (name, i, g, w)


def samples(n, units):
    s = {0, n - 1}
    k = 1
    while k < n:
        s |= {k - 1, k, k + 1}
        k *= 2
    for u in units:
        s |= {u - 1, u, u + 1, 2 * u, 2 * u + 1}
    return sorted(i for i in s if 0 <= i < n)


def sizes(name):
    u = fold_unit(name, 1 << 20)
    s = {1, 2, 3, u - 1, u, u + 1, 2 * u + 3}
    if name in ("moments_f64", "affine_f64", "nearest_query_f32", "pair_overlap_u32", "sum_sq_idx_u64"):
        s.add(70_000)
    if name == "sum_sq_idx_u64":
        s.add((1 << 20) + 5)
    return sorted(x for x in s if x >= 1)


BODIES = ["moments_f64", "row_sum_f64", "sum_sq_idx_u64", "byte_hist_u8", "pair_overlap_u32", "nearest_query_f32",
          "affine_f64", "mix4k_u32"]


@pytest.mark.parametrize("name", BODIES)
def test_prefixes_equal_the_restatement_and_the_fold(pool, name):
    R = registry.spec(name).result_bytes
    for n in sizes(name):
        xs = inputs(name, n, seed=n + 11)
        got = accumulate(pool, name, xs)
        check_all(name, got, want_prefixes(name, xs))
        recs = raw_records(got, R)
        for i in samples(n, {fold_unit(name, n), fold_unit(name, 1 << 20)}):
            assert recs[i] == fold_raw(pool, name, xs[:i + 1]), (name, n, i)
        assert recs[-1] == fold_raw(pool, name, xs)


def test_first_record_is_the_first_result(pool):
    xs = np.zeros(3, SB.AFFINE_ARG)
    xs["a"], xs["b"] = 2.0, -0.0
    got = np.asarray(pool.accumulate(SB.affine_f64, xs))
    assert np.signbit(got["b"][0])                           # -0.0, not identity (+) x0 = 2 * 0.0 + -0.0 = +0.0
    for name in ("moments_f64", "row_sum_f64", "nearest_query_f32"):
        xs = inputs(name, 5, seed=3)
        R = registry.spec(name).result_bytes
        assert raw_records(accumulate(pool, name, xs), R)[0] == raw_records(pool.map(body(name), xs), R)[0]
    assert len(pool.accumulate(FB.moments_f64, np.zeros(0))) == 0


def _raw_scan(p, name, xs, flags=0, chunksize=0, dev_args=False):
    """An accumulate through the C ABI: every record's bytes."""
    spec = registry.spec(name)
    enc = spec.encode_map(xs)
    eng = p._engine
    lib = eng.lib
    d = _abi.MapDesc()
    d.func_id, d.flags, d.n_tasks, d.chunksize, d.shuffle_seed = spec.func_id, flags | _abi.FBR_SCAN, enc.n, chunksize, 17
    d.arg_stride = enc.arg_stride
    dptr = ctypes.c_void_p()
    if enc.args is not None:
        if dev_args:
            _abi.check(lib.fbr_device_alloc(eng.handle, 0, enc.args.nbytes + 16, ctypes.byref(dptr)))
            _abi.check(lib.fbr_memcpy_h2d(eng.handle, 0, dptr, enc.args.ctypes.data, enc.args.nbytes))
            d.args = dptr.value
            d.flags |= _abi.FBR_ARGS_DEVICE
        else:
            d.args = enc.args.ctypes.data
    seq = ctypes.c_uint64()
    n, R = enc.n, spec.result_bytes
    try:
        _abi.check(lib.fbr_map_submit(eng.handle, ctypes.byref(d), ctypes.byref(seq)))
        res = _abi.Result()
        _abi.check(lib.fbr_result_wait(eng.handle, seq.value, -1, ctypes.byref(res)))
        if d.flags & _abi.FBR_RESULTS_ON_DEVICE:
            out = np.zeros(n * R, np.uint8)
            half = n // 2
            _abi.check(lib.fbr_result_fetch(eng.handle, seq.value, 0, half, out.ctypes.data))
            _abi.check(lib.fbr_result_fetch(eng.handle, seq.value, half, n - half, out[half * R:].ctypes.data))
            out = out.tobytes()
        else:
            out = ctypes.string_at(res.data, n * R)
        _abi.check(lib.fbr_result_release(eng.handle, seq.value))
    finally:
        if dptr.value:
            lib.fbr_device_free(eng.handle, 0, dptr)
    return out


@pytest.mark.parametrize("name", ["moments_f64", "affine_f64", "row_sum_f64"])
def test_result_does_not_depend_on_the_schedule(pool, small, name):
    n = 1_001 if name == "row_sum_f64" else 20_011
    xs = inputs(name, n, seed=5)
    for p in (pool, small):
        accumulate(p, name, xs[:1])                          # starts the pool's workers
    first = None
    runs = []
    for p in (pool, small):
        for flags in (_abi.FBR_SHUFFLE, _abi.FBR_VIA_RING, _abi.FBR_RESULTS_ON_DEVICE, _abi.FBR_RESILIENT):
            runs.append((p, dict(flags=flags)))
        runs.append((p, dict(dev_args=True)))
        runs.append((p, dict(dev_args=True, flags=_abi.FBR_VIA_RING)))
    for p, kw in runs:
        raw = _raw_scan(p, name, xs, **kw)
        if first is None:
            first = raw
        assert raw == first, kw
    for units in ("16", "100"):
        os.environ["FBR_UNIT_TASKS"] = units
        try:
            assert _raw_scan(pool, name, xs) == first
            assert _raw_scan(small, name, xs, flags=_abi.FBR_SHUFFLE, chunksize=3) == first
        finally:
            del os.environ["FBR_UNIT_TASKS"]
    spec = registry.spec(name)
    R = spec.result_bytes
    check_all(name, [spec.unpack_result(first[i * R:(i + 1) * R]) for i in range(n)], want_prefixes(name, xs))


@pytest.mark.parametrize("name", ["moments_f64", "affine_f64"])
def test_four_waves_of_a_small_ring(pool, small, name):
    xs = inputs(name, 150_000, seed=99)
    accumulate(small, name, xs[:1])
    before = small.stats()["dispatch_launches"]
    got = _raw_scan(small, name, xs)
    assert small.stats()["dispatch_launches"] - before >= 4
    assert got == _raw_scan(pool, name, xs)
    spec = registry.spec(name)
    R = spec.result_bytes
    check_all(name, [spec.unpack_result(got[i * R:(i + 1) * R]) for i in range(len(xs))], want_prefixes(name, xs))


def test_results_on_device():
    xs = inputs("moments_f64", 50_000, seed=7)
    want = want_prefixes("moments_f64", xs)
    p = fiber_b200.Pool(1, devices=[0], results="device")
    try:
        got = p.accumulate(FB.moments_f64, xs)
        check_all("moments_f64", got, want)
        check_all("moments_f64", list(got[1000:1010]), want[1000:1010])
    finally:
        p.terminate()
        p.join()


def test_error_handling():
    xs = range(0, 50_000)
    p = fiber_b200.Pool(1, devices=[0], error_handling=True)
    try:
        assert list(p.accumulate(FB.fault_count_u64, xs)) == want_prefixes("fault_count_u64", xs)
        assert p.stats()["units_redispatched"] > 0
    finally:
        p.terminate()
        p.join()
    p = fiber_b200.Pool(1, devices=[0])
    try:
        with pytest.raises(RuntimeError) as m:
            p.map(FB.fault_count_u64, xs)
        with pytest.raises(RuntimeError) as a:
            p.accumulate(FB.fault_count_u64, xs)
        assert str(a.value) == str(m.value)
    finally:
        p.terminate()
        p.join()


def test_forms(pool):
    cols = inputs("pair_overlap_u32", 3000, seed=9)
    check_all("pair_overlap_u32", pool.staraccumulate(FB.pair_overlap_u32, cols), want_prefixes("pair_overlap_u32", cols))
    xs = inputs("byte_hist_u8", 2000, seed=8)
    want = want_prefixes("byte_hist_u8", xs)
    check_all("byte_hist_u8", pool.accumulate(FB.byte_hist_u8, xs), want)
    check_all("byte_hist_u8", pool.accumulate(FB.byte_hist_u8, [bytes(np.asarray(xs[i])) for i in range(len(xs))]), want)
    pts = inputs("nearest_query_f32", 4000, seed=10)
    check_all("nearest_query_f32", pool.accumulate(FB.nearest_query_f32, pts), want_prefixes("nearest_query_f32", pts))
    q2 = np.array([1.0, 1.0, 1.0, 1.0], np.float32)
    got = pool.staraccumulate(FB.nearest_query_f32, [(q2, p) for p in pts[:500]])
    rs = [FB.nearest_run(q2, p, i) for i, p in enumerate(pts[:500].tolist())]
    check_all("nearest_query_f32", got, SB.prefix_folds(rs, FB.nearest_combine))


def test_device_ragged_items(pool):
    xs = inputs("byte_hist_u8", 3000, seed=12)
    want = want_prefixes("byte_hist_u8", xs)
    spec = registry.spec("byte_hist_u8")
    pool.accumulate(FB.byte_hist_u8, xs[:1])                 # starts the pool's workers
    eng = pool._engine
    lib = eng.lib
    vals, offs = np.asarray(xs.values), np.asarray(xs.offsets, np.uint64)
    dv, do = ctypes.c_void_p(), ctypes.c_void_p()
    _abi.check(lib.fbr_device_alloc(eng.handle, 0, vals.nbytes + 16, ctypes.byref(dv)))
    _abi.check(lib.fbr_device_alloc(eng.handle, 0, offs.nbytes + 16, ctypes.byref(do)))
    try:
        _abi.check(lib.fbr_memcpy_h2d(eng.handle, 0, dv, vals.ctypes.data, vals.nbytes))
        _abi.check(lib.fbr_memcpy_h2d(eng.handle, 0, do, offs.ctypes.data, offs.nbytes))
        d = _abi.MapDesc()
        d.func_id, d.n_tasks, d.flags = spec.func_id, len(xs), _abi.FBR_ARGS_DEVICE | _abi.FBR_SCAN
        it = _abi.ItemsDesc()
        it.items, it.offsets, it.n_items, it.item_bytes = dv.value, do.value, len(vals), 1
        seq = ctypes.c_uint64()
        _abi.check(lib.fbr_map_submit_items(eng.handle, ctypes.byref(d), ctypes.byref(it), ctypes.byref(seq)))
        res = _abi.Result()
        _abi.check(lib.fbr_result_wait(eng.handle, seq.value, -1, ctypes.byref(res)))
        R = spec.result_bytes
        raw = ctypes.string_at(res.data, len(xs) * R)
        check_all("byte_hist_u8", [spec.unpack_result(raw[i * R:(i + 1) * R]) for i in range(len(xs))], want)
        _abi.check(lib.fbr_result_release(eng.handle, seq.value))
    finally:
        lib.fbr_device_free(eng.handle, 0, dv)
        lib.fbr_device_free(eng.handle, 0, do)


def _submit_flags(p, name, flags, out=None):
    spec = registry.spec(name)
    d = _abi.MapDesc()
    d.func_id, d.flags, d.n_tasks, d.arg_stride = spec.func_id, flags, 4, 0
    if out is not None:
        d.out = out.ctypes.data
    d.index_start, d.index_step = 0, 1
    seq = ctypes.c_uint64()
    rc = p._engine.lib.fbr_map_submit(p._engine.handle, ctypes.byref(d), ctypes.byref(seq))
    return rc, _abi.load().fbr_last_error().decode()


def test_scan_refusals(pool):
    pool.accumulate(FB.sum_sq_idx_u64, range(3))
    S = _abi.FBR_SCAN
    for flags, why in ((S | _abi.FBR_FOLD, "FBR_FOLD"), (S | _abi.FBR_WANT_SUM, "FBR_WANT_SUM"),

                       (S | _abi.FBR_NO_ZERO_COPY, "FBR_NO_ZERO_COPY")):
        rc, msg = _submit_flags(pool, "sum_sq_idx_u64", flags)
        assert rc == _abi.FBR_EINVAL and why in msg, msg
    for flags in (S, S | _abi.FBR_OUT_DEVICE):
        rc, msg = _submit_flags(pool, "sum_sq_idx_u64", flags, out=np.zeros(4, np.uint64))
        assert rc == _abi.FBR_EINVAL and "owns its result window" in msg, msg
    rc, msg = _submit_flags(pool, "square_i64", S)
    assert rc == _abi.FBR_EINVAL and "FBR_BODY_SCAN" in msg, msg
    # a hand-written fold descriptor without the scan entry folds, but cannot accumulate
    fid = ctypes.c_int(-1)
    _abi.check(_abi.load().fbr_register_body(b"ok_fold", FB.BAD_MODULE.encode(), b"ok_fold", ctypes.byref(fid)))
    d = _abi.MapDesc()
    d.func_id, d.flags, d.n_tasks, d.arg_stride = fid.value, S, 4, 8
    args = np.arange(4, dtype=np.int64)
    d.args = args.ctypes.data
    seq = ctypes.c_uint64()
    assert pool._engine.lib.fbr_map_submit(pool._engine.handle, ctypes.byref(d), ctypes.byref(seq)) == _abi.FBR_EINVAL
    assert "FBR_BODY_SCAN" in _abi.load().fbr_last_error().decode()


@pytest.mark.parametrize("m", [0, 1, 3])
def test_scan_values(pool, m):
    rng = np.random.default_rng(m)
    recs = np.zeros(1000, SB.AFFINE_RES)
    recs["a"], recs["b"] = rng.uniform(0.5, 1.5, 1000), rng.standard_normal(1000)
    pieces = np.zeros(max(m, 1), SB.AFFINE_RES)
    pieces["a"], pieces["b"] = rng.uniform(0.5, 1.5, len(pieces)), rng.standard_normal(len(pieces))
    want = []
    for r in recs.tolist():
        acc = tuple(r)
        for g in reversed(pieces[:m].tolist()):
            acc = SB.affine_combine(tuple(g), acc)
        want.append(acc)
    pool.accumulate(SB.affine_f64, recs[:1])                 # starts the pool's workers
    eng = pool._engine
    _abi.check(eng.lib.fbr_scan_values(eng.handle, registry.spec("affine_f64").func_id, pieces.ctypes.data, m,
                                       recs.ctypes.data, len(recs)))
    check_all("affine_f64", [tuple(r) for r in recs.tolist()], want)


def _two_gpus():
    n = ctypes.c_int(0)
    _abi.check(_abi.load().fbr_device_count(ctypes.byref(n)))
    if n.value < 2:
        pytest.skip("needs two GPUs")


def _plan_bounds(n, n_workers):
    bounds = []
    for w in range(n_workers):
        plan = _abi.Plan()
        _abi.check(_abi.load().fbr_plan_query(registry.spec("moments_f64").func_id, n, _abi.FBR_PLAN_FOLD, 0, n_workers, w,
                                              132, ctypes.byref(plan)))
        if plan.block_count:
            bounds.append((plan.block_first, plan.block_first + plan.block_count))
    return bounds


def test_process_isolation_one_gpu():
    """One worker process, several blocks: each block accumulates in the worker, then the worker wraps blocks 1, 2, ..."""
    xs = inputs("moments_f64", 150_001, seed=42)
    p = fiber_b200.Pool(1, isolation="process", error_handling=True)
    try:
        check_all("moments_f64", p.accumulate(FB.moments_f64, xs[:10]), want_prefixes("moments_f64", xs[:10]))
        bounds = [(lo, hi) for lo, hi in p._proc.fold_blocks(len(xs)) if hi > lo]
        assert len(bounds) > 1
        got = p.accumulate(FB.moments_f64, xs)
        check_all("moments_f64", got, SB.block_prefix_folds(run_all("moments_f64", xs), bounds, FB.moments_combine))
        assert FB.same_record(tuple(np.asarray(got)[-1].tolist()), p.fold(FB.moments_f64, xs))
        cols = inputs("pair_overlap_u32", 70_000, seed=43)
        assert list(p.staraccumulate(FB.pair_overlap_u32, cols)) == want_prefixes("pair_overlap_u32", cols)
        assert len(p.accumulate(FB.moments_f64, xs[:0])) == 0
    finally:
        p.terminate()
        p.join()


def test_two_workers_thread():
    _two_gpus()
    xs = inputs("moments_f64", 300_001, seed=40)
    results = run_all("moments_f64", xs)
    bounds = _plan_bounds(len(xs), 2)
    want = SB.block_prefix_folds(results, bounds, FB.moments_combine)
    for results_mode in ("host", "device"):
        p = fiber_b200.Pool(2, results=results_mode)
        try:
            got = p.accumulate(FB.moments_f64, xs)
            check_all("moments_f64", got, want)
            assert raw_records(got, 24)[-1] == fold_raw(p, "moments_f64", xs)
        finally:
            p.terminate()
            p.join()
