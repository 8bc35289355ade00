"""GPU: fold maps (Pool.fold / starfold, FBR_FOLD) of the bodies in tests/fold_bodies.py -- every record form, sizes around
the claim unit and across several waves, the independence of the result from chunksize, unit size, ring size, shuffled
arrival, the result ring and argument placement, error handling, fbr_fold_values and two-worker pools.  Every result is
compared bit for bit, floats included, with the Python restatement of run, combine and tree."""
import ctypes
import functools
import os

import numpy as np
import pytest

import fiber_b200
from fiber_b200 import _abi, registry

from . import fold_bodies as FB

pytestmark = pytest.mark.gpu

SMALL_RING = 256 << 10


@fiber_b200.device_initializer("nearest_query_f32")
def set_query(q):
    raise RuntimeError("runs on the GPU workers")


QUERY = np.array([0.25, -1.5, 3.0, 0.125], np.float32)


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


# ---- inputs and restated results of each body -------------------------------------------------------------------------
def inputs(name, n, seed):
    rng = np.random.default_rng(seed)
    if name == "moments_f64":
        return rng.standard_normal(n) * 1e3 + 7.0
    if name == "row_sum_f64":
        return (rng.standard_normal((n, 256)) * 10.0 ** rng.integers(-3, 4, (n, 1))).astype(np.float64)
    if name in ("sum_sq_idx_u64", "fault_count_u64"):
        return range(5, 5 + 3 * n, 3)
    if name == "byte_hist_u8":
        lens = rng.integers(0, 40, n)
        offs = np.zeros(n + 1, np.int64)
        np.cumsum(lens, out=offs[1:])
        return fiber_b200.Ragged(rng.integers(0, 256, int(offs[-1]), dtype=np.uint8), offs)
    if name == "pair_overlap_u32":
        cols = []
        for _ in range(2):
            lens = rng.integers(0, 24, n)
            offs = np.zeros(n + 1, np.int64)
            np.cumsum(lens, out=offs[1:])
            vals = rng.integers(0, 30, int(offs[-1]), dtype=np.uint32)
            for i in range(n):
                vals[offs[i]:offs[i + 1]].sort()
            cols.append(fiber_b200.Ragged(vals, offs))
        return fiber_b200.Columns(*cols)
    if name == "nearest_query_f32":
        p = (rng.standard_normal((n, 4)) * 4).astype(np.float32)
        p[rng.random(n) < 0.05] = np.nan
        if n > 8:
            p[n // 2] = p[n // 3]              # a tie: the lower index wins
        return p
    raise KeyError(name)


def run_all(name, xs):
    """Each task's restated result, in task order."""
    if name == "moments_f64":
        return [FB.moments_run(x) for x in xs.tolist()]
    if name == "row_sum_f64":
        s = np.zeros((len(xs), 32))
        for k in range(8):
            s = s + xs[:, 32 * k:32 * (k + 1)]
        o = 16
        while o:
            s = s + s[:, np.arange(32) ^ o]
            o //= 2
        return [(float(v), 1.0) for v in s[:, 0]]
    if name == "sum_sq_idx_u64":
        return [(i * i) & FB.M64 for i in xs]
    if name == "fault_count_u64":
        return [(3 * i + 1) & FB.M64 for i in xs]
    if name == "byte_hist_u8":
        return [np.bincount(np.asarray(xs[i]), minlength=256).tolist() for i in range(len(xs))]
    if name == "pair_overlap_u32":
        a, b = xs.columns
        return [FB.pair_overlap_u32(a[i], b[i]) for i in range(len(a))]
    if name == "nearest_query_f32":
        return [FB.nearest_run(QUERY, p, i) for i, p in enumerate(xs.tolist())]
    raise KeyError(name)


def restated(name, xs):
    combine, identity = FB.RESTATED[name]
    return FB.fold_of(run_all(name, xs), combine, identity)


def as_tuple(name, got):
    if name == "byte_hist_u8":
        return list(got)
    return got


def do_fold(p, name, xs):
    f = getattr(FB, name)
    if name == "pair_overlap_u32":
        return p.starfold(f, xs)
    return p.fold(f, xs)


def check(name, got, want):
    got = as_tuple(name, got)
    assert FB.same_record(got, want), (name, got, want)


# fault_count_u64 faults without error handling: test_error_handling runs it
BODIES = ["moments_f64", "row_sum_f64", "sum_sq_idx_u64", "byte_hist_u8", "pair_overlap_u32", "nearest_query_f32"]


def unit_sizes(name):
    """0, 1, 2 and the sizes around the unit of a large map and of a small one (small maps take smaller units)."""
    sizes = {0, 1, 2}
    for u in {fold_unit(name, 1 << 20), fold_unit(name, 2000)}:
        sizes |= {u - 1, u, u + 1, 3 * u + 5}
    return sorted(sizes)


@pytest.mark.parametrize("name", BODIES)
def test_sizes_around_the_unit(pool, name):
    for n in unit_sizes(name):
        xs = inputs(name, n, seed=n + 3)
        check(name, do_fold(pool, name, xs), restated(name, xs))


@pytest.mark.parametrize("name", BODIES)
def test_four_waves_of_a_small_ring(small, name):
    u = fold_unit(name, 1 << 20, SMALL_RING)
    n = {"row_sum_f64": 40 * u + 3, "nearest_query_f32": 70_000, "moments_f64": 150_000}.get(name, 40_000)
    xs = inputs(name, n, seed=99)
    before = small.stats()["dispatch_launches"]
    check(name, do_fold(small, name, xs), restated(name, xs))
    if name not in ("sum_sq_idx_u64",):          # range() maps stream no arguments: one wave
        assert small.stats()["dispatch_launches"] - before >= 4


def _raw_fold(p, name, xs, flags=0, chunksize=0, dev_args=False):
    """A fold map through the C ABI (chunksize and map flags the Pool API does not take): the result record's bytes."""
    spec = registry.spec(name)
    enc = spec.encode_map(xs)
    eng = p._engine
    lib = eng.lib
    d = _abi.MapDesc()
    d.func_id, d.flags, d.n_tasks, d.chunksize, d.shuffle_seed = spec.func_id, flags | _abi.FBR_FOLD, enc.n, chunksize, 17
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
    try:
        _abi.check(lib.fbr_map_submit(eng.handle, ctypes.byref(d), ctypes.byref(seq)))
        res = _abi.Result()
        _abi.check(lib.fbr_result_wait(eng.handle, seq.value, -1, ctypes.byref(res)))
        assert res.result_bytes == spec.result_bytes and res.n_tasks == enc.n
        out = ctypes.string_at(res.data, res.result_bytes)
        _abi.check(lib.fbr_result_release(eng.handle, seq.value))
    finally:
        if dptr.value:
            lib.fbr_device_free(eng.handle, 0, dptr)
    return out


@pytest.mark.parametrize("name", ["moments_f64", "row_sum_f64"])
def test_result_does_not_depend_on_the_schedule(pool, small, name):
    n = 20_011 if name == "moments_f64" else 1_001
    xs = inputs(name, n, seed=5)
    want = restated(name, xs)
    spec = registry.spec(name)
    first = None
    runs = []
    for p in (pool, small):
        for cs in (1, 7, 32, 4096):
            runs.append((p, dict(chunksize=cs)))
        for flags in (_abi.FBR_SHUFFLE, _abi.FBR_VIA_RING, _abi.FBR_RESULTS_ON_DEVICE):
            runs.append((p, dict(flags=flags)))
        runs.append((p, dict(dev_args=True)))
        runs.append((p, dict(dev_args=True, flags=_abi.FBR_VIA_RING)))
    for p, kw in runs:
        raw = _raw_fold(p, name, xs, **kw)
        if first is None:
            first = raw
        assert raw == first, kw
    for units in ("16", "100"):
        os.environ["FBR_UNIT_TASKS"] = units
        try:
            assert _raw_fold(pool, name, xs) == first
            assert _raw_fold(small, name, xs, flags=_abi.FBR_SHUFFLE, chunksize=3) == first
        finally:
            del os.environ["FBR_UNIT_TASKS"]
    check(name, spec.unpack_result(first), want)


def test_ragged_columns_and_broadcast_forms(pool):
    xs = inputs("byte_hist_u8", 5000, seed=8)
    want = restated("byte_hist_u8", xs)
    check("byte_hist_u8", pool.fold(FB.byte_hist_u8, xs), want)
    check("byte_hist_u8", pool.fold(FB.byte_hist_u8, [bytes(np.asarray(xs[i])) for i in range(len(xs))]), want)
    cols = inputs("pair_overlap_u32", 3000, seed=9)
    check("pair_overlap_u32", pool.starfold(FB.pair_overlap_u32, cols), restated("pair_overlap_u32", cols))
    pts = inputs("nearest_query_f32", 4000, seed=10)
    want = restated("nearest_query_f32", pts)
    check("nearest_query_f32", pool.fold(FB.nearest_query_f32, pts), want)                     # the initializer's block
    q2 = np.array([1.0, 1.0, 1.0, 1.0], np.float32)
    got = pool.starfold(FB.nearest_query_f32, [(q2, p) for p in pts[:500]])                    # the block in every tuple
    rs = [FB.nearest_run(q2, p, i) for i, p in enumerate(pts[:500].tolist())]
    check("nearest_query_f32", got, FB.fold_of(rs, FB.nearest_combine, FB.NEAR_ID))


def test_device_ragged_items(pool):
    xs = inputs("byte_hist_u8", 3000, seed=12)
    want = restated("byte_hist_u8", xs)
    spec = registry.spec("byte_hist_u8")
    eng = pool._engine
    lib = eng.lib
    vals, offs = np.asarray(xs.values), np.asarray(xs.offsets, np.uint64)
    dv, do = ctypes.c_void_p(), ctypes.c_void_p()
    _abi.check(lib.fbr_device_alloc(eng.handle, 0, vals.nbytes + 16, ctypes.byref(dv)))
    _abi.check(lib.fbr_device_alloc(eng.handle, 0, offs.nbytes + 16, ctypes.byref(do)))
    try:
        _abi.check(lib.fbr_memcpy_h2d(eng.handle, 0, dv, vals.ctypes.data, vals.nbytes))
        bad = offs.copy()
        for o, code in ((offs, 0), (bad, _abi.FBR_TASK_BADARG)):
            if code:
                bad[1001] = bad[1002] + 1                  # task 1001's offsets decrease
            _abi.check(lib.fbr_memcpy_h2d(eng.handle, 0, do, o.ctypes.data, o.nbytes))
            errs = []
            for fold in (True, False):
                d = _abi.MapDesc()
                d.func_id, d.n_tasks = spec.func_id, len(xs)
                d.flags = _abi.FBR_ARGS_DEVICE | (_abi.FBR_FOLD if fold else 0)
                it = _abi.ItemsDesc()
                it.items, it.offsets, it.n_items, it.item_bytes = dv.value, do.value, len(vals), 1
                seq = ctypes.c_uint64()
                _abi.check(lib.fbr_map_submit_items(eng.handle, ctypes.byref(d), ctypes.byref(it), ctypes.byref(seq)))
                res = _abi.Result()
                rc = lib.fbr_result_wait(eng.handle, seq.value, -1, ctypes.byref(res))
                errs.append((rc, res.err_code, res.err_task))
                if fold and not code:
                    _abi.check(rc)
                    check("byte_hist_u8", spec.unpack_result(ctypes.string_at(res.data, res.result_bytes)), want)
                _abi.check(lib.fbr_result_release(eng.handle, seq.value))
            assert errs[0] == errs[1]
            assert errs[0][1] == code and (not code or errs[0][2] == 1001)
    finally:
        lib.fbr_device_free(eng.handle, 0, dv)
        lib.fbr_device_free(eng.handle, 0, do)


def test_error_handling():
    xs = range(0, 50_000)
    want = FB.fold_of(run_all("fault_count_u64", xs), FB.add_u64, 0)
    p = fiber_b200.Pool(1, devices=[0], error_handling=True)
    try:
        assert p.fold(FB.fault_count_u64, xs) == want
        assert p.fold(FB.fault_count_u64, range(3)) == 1 + 4 + 7
        for n in unit_sizes("fault_count_u64"):
            ys = inputs("fault_count_u64", n, seed=n)
            assert p.fold(FB.fault_count_u64, ys) == restated("fault_count_u64", ys)
        assert p.stats()["units_redispatched"] > 0
    finally:
        p.terminate()
        p.join()
    p = fiber_b200.Pool(1, devices=[0])
    try:
        with pytest.raises(RuntimeError) as m:
            p.map(FB.fault_count_u64, xs)
        with pytest.raises(RuntimeError) as f:
            p.fold(FB.fault_count_u64, xs)
        assert str(f.value) == str(m.value)
        r = p.fold_async(FB.fault_count_u64, xs)
        with pytest.raises(RuntimeError):
            r.get()
        with pytest.raises(RuntimeError):
            r.get()                                    # the error is remembered
    finally:
        p.terminate()
        p.join()


@pytest.mark.parametrize("name", ["sum_sq_idx_u64", "byte_hist_u8", "pair_overlap_u32"])
def test_fold_equals_reduce_of_the_map(pool, name):
    xs = inputs(name, 7777, seed=21)
    combine, _ = FB.RESTATED[name]
    f = getattr(FB, name)
    mapped = list(pool.starmap(f, xs) if name == "pair_overlap_u32" else pool.map(f, xs))
    check(name, do_fold(pool, name, xs), functools.reduce(combine, mapped))
    assert mapped == run_all(name, xs)                  # plain maps of a fold body keep their results


def test_plain_maps_of_fold_bodies(pool):
    xs = inputs("moments_f64", 3000, seed=4)
    got = np.asarray(pool.map(FB.moments_f64, xs))
    assert np.array_equal(got["mean"], xs) and np.all(got["n"] == 1.0) and np.all(got["m2"] == 0.0)
    rows = inputs("row_sum_f64", 100, seed=4)
    got = pool.map(FB.row_sum_f64, rows)
    assert [tuple(r) for r in got] == run_all("row_sum_f64", rows)


def test_async_poll_and_fetch(pool):
    xs = inputs("moments_f64", 100_000, seed=30)
    spec = registry.spec("moments_f64")
    eng = pool._engine
    d = _abi.MapDesc()
    d.func_id, d.flags, d.n_tasks, d.arg_stride = spec.func_id, _abi.FBR_FOLD, len(xs), 8
    d.args = xs.ctypes.data
    seq = ctypes.c_uint64()
    _abi.check(eng.lib.fbr_map_submit(eng.handle, ctypes.byref(d), ctypes.byref(seq)))
    done = ctypes.c_uint64()
    while True:
        _abi.check(eng.lib.fbr_result_poll(eng.handle, seq.value, ctypes.byref(done)))
        assert done.value in (0, len(xs))
        if done.value:
            break
    buf = np.zeros(24, np.uint8)
    assert eng.lib.fbr_result_fetch(eng.handle, seq.value, 0, 1, buf.ctypes.data) == _abi.FBR_EINVAL
    res = _abi.Result()
    _abi.check(eng.lib.fbr_result_wait(eng.handle, seq.value, -1, ctypes.byref(res)))
    check("moments_f64", spec.unpack_result(ctypes.string_at(res.data, 24)), restated("moments_f64", xs))
    _abi.check(eng.lib.fbr_result_release(eng.handle, seq.value))
    r = pool.fold_async(FB.moments_f64, xs)
    with pytest.raises(TypeError, match="a fold has one result"):
        r.iget_ordered()
    check("moments_f64", r.get(), restated("moments_f64", xs))


@pytest.mark.parametrize("n", [0, 1, 2, 3, 1000, 70_000])
def test_fold_values(pool, n):
    rng = np.random.default_rng(n)
    recs = np.zeros(n, FB.MOMENTS_RES)
    recs["n"] = rng.integers(0, 5, n)
    recs["mean"] = rng.standard_normal(n)
    recs["m2"] = rng.random(n) * recs["n"]
    spec = registry.spec("moments_f64")
    out = np.zeros(1, FB.MOMENTS_RES)
    eng = pool._engine
    _abi.check(eng.lib.fbr_fold_values(eng.handle, spec.func_id, recs.ctypes.data if n else None, n, out.ctypes.data))
    want = FB.fold_of([tuple(float(v) for v in r) for r in recs.tolist()], FB.moments_combine, FB.MOMENTS_ID)
    check("moments_f64", tuple(float(v) for v in out[0].tolist()), want)


def _process_fold_want(p, name, xs):
    """tree over the totals of the blocks a process-isolated pool cuts the map into, in block order."""
    combine, identity = FB.RESTATED[name]
    results = run_all(name, xs)
    return FB.fold_of([FB.tree(results[lo:hi], combine) for lo, hi in p._proc.fold_blocks(len(results)) if hi > lo],
                      combine, identity)


def test_process_isolation_one_gpu():
    """One worker process, several blocks: each block folds in the worker, then the worker folds the block totals."""
    xs = inputs("moments_f64", 150_001, seed=41)
    p = fiber_b200.Pool(1, isolation="process", error_handling=True)
    try:
        check("moments_f64", p.fold(FB.moments_f64, xs[:10]), restated("moments_f64", xs[:10]))   # one block
        assert len(p._proc.fold_blocks(len(xs))) > 1
        check("moments_f64", p.fold(FB.moments_f64, xs), _process_fold_want(p, "moments_f64", xs))
        cols = inputs("pair_overlap_u32", 70_000, seed=42)
        check("pair_overlap_u32", p.starfold(FB.pair_overlap_u32, cols), restated("pair_overlap_u32", cols))
        assert p.fold(FB.sum_sq_idx_u64, range(200_000)) == restated("sum_sq_idx_u64", range(200_000))
        check("moments_f64", p.fold(FB.moments_f64, xs[:0]), FB.MOMENTS_ID)
    finally:
        p.terminate()
        p.join()


def _two_gpus():
    n = ctypes.c_int(0)
    _abi.check(_abi.load().fbr_device_count(ctypes.byref(n)))
    if n.value < 2:
        pytest.skip("needs two GPUs")


def _block_tree(name, xs, n_workers):
    """tree over the totals of the blocks fbr_plan_query gives a fold map on n_workers workers."""
    combine, identity = FB.RESTATED[name]
    results = run_all(name, xs)
    totals = []
    for w in range(n_workers):
        plan = _abi.Plan()
        _abi.check(_abi.load().fbr_plan_query(registry.spec(name).func_id, len(results), _abi.FBR_PLAN_FOLD, 0, n_workers, w,
                                              132, ctypes.byref(plan)))
        if plan.block_count:
            totals.append(FB.tree(results[plan.block_first:plan.block_first + plan.block_count], combine))
    return FB.fold_of(totals, combine, identity)


@pytest.mark.parametrize("isolation", ["thread", "process"])
def test_two_workers(isolation):
    _two_gpus()
    xs = inputs("moments_f64", 300_001, seed=40)
    p = fiber_b200.Pool(2, isolation=isolation)
    try:
        got = p.fold(FB.moments_f64, xs)
        if isolation == "thread":
            check("moments_f64", got, _block_tree("moments_f64", xs, 2))
        else:
            check("moments_f64", got, _process_fold_want(p, "moments_f64", xs))
        assert p.fold(FB.sum_sq_idx_u64, range(10 ** 6)) == sum(i * i for i in range(10 ** 6)) & FB.M64
    finally:
        p.terminate()
        p.join()
