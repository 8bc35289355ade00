"""CPU: fold bodies -- registration rules (hand-written descriptors), fbr_body_fold_info, header constants, the TypeError of
bodies that cannot fold, the fold order tree() and the property the engine relies on (aligned power-of-two tiles are
subtrees), the fold plan, and the process-pool side of fold maps with a stand-in worker (tests/_fake_fold_worker.py)."""
import ctypes
import math
import os
import re
import struct

import numpy as np
import pytest

import fiber_b200
from fiber_b200 import _abi, registry
from fiber_b200.procpool import BLOCK_ALIGN, ProcessPool

from . import fold_bodies as FB
from ._fake_fold_worker import fake_fold_worker_main
from ._fake_fold_worker import tree as fake_tree

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FOLD_BODIES = ["moments_f64", "row_sum_f64", "sum_sq_idx_u64", "byte_hist_u8", "pair_overlap_u32", "fault_count_u64",
               "nearest_query_f32"]


def _register(entry):
    fid = ctypes.c_int(-1)
    rc = _abi.load().fbr_register_body(entry.encode(), FB.BAD_MODULE.encode(), entry.encode(), ctypes.byref(fid))
    return rc, fid.value, _abi.load().fbr_last_error().decode()


@pytest.mark.parametrize("entry,why", [
    ("bad_fold_flag_only", "lacks the fold entry or the identity record"),
    ("bad_fold_no_id", "lacks the fold entry or the identity record"),
    ("bad_fold_fields_only", "lacks FBR_BODY_FOLD"),
    ("bad_fold_thread", "only record bodies fold"),
    ("bad_fold_emit", "an emit body cannot fold"),
    ("bad_fold_summable", "cannot also be FBR_BODY_SUMMABLE"),
    ("bad_fold_id_size", "the identity record must be result_bytes long"),
    ("bad_fold_id_size_only", "describes an identity size but lacks FBR_BODY_FOLD"),
])
def test_registration_rejects_bad_fold_descriptors(entry, why):
    rc, _, msg = _register(entry)
    assert rc == _abi.FBR_EINVAL and why in msg, msg


def test_registration_accepts_a_fold_descriptor():
    rc, fid, msg = _register("ok_fold")
    assert rc == _abi.FBR_OK, msg
    info = _abi.BodyInfo()
    _abi.check(_abi.load().fbr_body_info(fid, ctypes.byref(info)))
    assert info.flags & _abi.FBR_BODY_FOLD


def _identity(name):
    lib = _abi.load()
    nb = ctypes.c_uint32(0)
    _abi.check(lib.fbr_body_fold_info(registry.spec(name).func_id, None, ctypes.byref(nb)))
    buf = ctypes.create_string_buffer(max(1, nb.value))
    _abi.check(lib.fbr_body_fold_info(registry.spec(name).func_id, buf, ctypes.byref(nb)))
    return buf.raw[:nb.value]


def test_fold_info_and_flags():
    for name in FOLD_BODIES:
        spec = registry.spec(name)
        assert spec.flags & (_abi.FBR_BODY_RECORD | _abi.FBR_BODY_FOLD) == _abi.FBR_BODY_RECORD | _abi.FBR_BODY_FOLD
        assert not spec.flags & (_abi.FBR_BODY_SUMMABLE | _abi.FBR_BODY_EMIT)
        assert len(_identity(name)) == spec.result_bytes
    zero = {"moments_f64": 24, "row_sum_f64": 16, "sum_sq_idx_u64": 8, "byte_hist_u8": 1024, "pair_overlap_u32": 8,
            "fault_count_u64": 8}
    for name, nb in zero.items():
        assert _identity(name) == bytes(nb)
    assert _identity("nearest_query_f32") == struct.pack("<IIQ", 0x7FC00000, 0, FB.M64)
    assert registry.spec("nearest_query_f32").unpack_result(_identity("nearest_query_f32"))[2] == FB.M64
    for name in ("square_i64", "polar_f64", "tokens_u32"):          # a thread body, a record body, an emit body
        if name != "square_i64":
            __import__("tests.record_bodies") if name == "polar_f64" else __import__("tests.emit_bodies")
        assert not registry.spec(name).flags & _abi.FBR_BODY_FOLD
        assert _identity(name) == b""


def test_header_constants_match_abi():
    h = open(os.path.join(ROOT, "include", "fiber_b200.h")).read()
    assert int(re.search(r"#define FBR_BODY_FOLD (0x[0-9a-f]+)u", h).group(1), 16) == _abi.FBR_BODY_FOLD == 0x100
    assert int(re.search(r"#define FBR_FOLD (0x[0-9a-f]+)u", h).group(1), 16) == _abi.FBR_FOLD == 0x4000
    assert int(re.search(r"#define FBR_PLAN_FOLD (0x[0-9a-f]+)u", h).group(1), 16) == _abi.FBR_PLAN_FOLD
    assert re.search(r"#define FBR_BODY_MODULE_ABI (\d+)", h).group(1) == str(_abi.FBR_BODY_MODULE_ABI) == "4"


def test_bodies_that_cannot_fold_raise_type_error():
    from examples import workloads as W
    from . import record_bodies as RB
    p = fiber_b200.Pool(1)                            # nothing starts: the check comes before any submission
    with pytest.raises(TypeError, match=r"square_i64 cannot fold.*sum\(pool.map"):
        p.fold(W.f, [1, 2, 3])
    with pytest.raises(TypeError, match=r"polar_f64 cannot fold.*identity\(\) and combine\(\)"):
        p.starfold(RB.polar_f64, [(1.0, 2.0)])
    with pytest.raises(TypeError, match="cannot fold"):
        p.fold_async(RB.polar_f64, [])
    assert p._engine is None and p._proc is None


def test_fold_result_is_not_iterable():
    from fiber_b200.pool import FoldResult
    r = FoldResult(None, None, registry.spec("moments_f64"), 0, 0, None)
    for it in (r.iget_ordered, r.iget_unordered):
        with pytest.raises(TypeError, match="moments_f64: a fold has one result"):
            it()


def _nested(c):
    return FB.tree(range(c), lambda a, b: (a, b))


def _recursive(lo, hi):
    """tree over [lo, hi) by its recursive form: the largest power of two below the length splits it."""
    if hi - lo == 1:
        return lo
    h = 1 << ((hi - lo - 1).bit_length() - 1)
    return (_recursive(lo, lo + h), _recursive(lo + h, hi))


def test_tree_equals_its_recursive_definition():
    assert _nested(0) is None
    for c in range(1, 5001):
        assert _nested(c) == _recursive(0, c), c


def _kernel_tree(xs, combine):
    """The in-place pairing of the fold pass and fold_tree_kernel: level s combines x[j] and x[j + s] for every multiple j
    of 2s with j + s < c."""
    xs = list(xs)
    s = 1
    while s < len(xs):
        for j in range(0, len(xs) - s, 2 * s):
            xs[j] = combine(xs[j], xs[j + s])
        s *= 2
    return xs[0] if xs else None


def test_aligned_tiles_are_subtrees():
    pair = lambda a, b: (a, b)  # noqa: E731
    for c in list(range(1, 300)) + [1023, 1024, 1025, 3 * 1024 + 5, 5000]:
        whole = FB.tree(range(c), pair)
        assert _kernel_tree(range(c), pair) == whole
        for t in (1, 2, 4, 16, 512, 1024):
            tiles = [FB.tree(range(lo, min(c, lo + t)), pair) for lo in range(0, c, t)]
            assert FB.tree(tiles, pair) == whole, (c, t)
            # units inside tiles (the engine: unit partials, then fold_tree_kernel tiles over them)
            if t >= 4:
                units = [FB.tree(range(lo, min(c, lo + 4)), pair) for lo in range(0, c, 4)]
                tiles_of_units = [FB.tree(units[k:k + t], pair) for k in range(0, len(units), t)]
                assert FB.tree(tiles_of_units, pair) == whole


def test_restated_combines():
    # Chan's merge agrees with the two-pass moments of the whole column (to rounding), and the identity is neutral
    xs = np.random.default_rng(1).standard_normal(1001) * 3 + 1
    n, mean, m2 = FB.fold_of([FB.moments_run(x) for x in xs], FB.moments_combine, FB.MOMENTS_ID)
    assert n == 1001 and math.isclose(mean, xs.mean(), rel_tol=1e-12) and math.isclose(m2, ((xs - xs.mean()) ** 2).sum(), rel_tol=1e-9)
    assert FB.moments_combine(FB.MOMENTS_ID, (2.0, 1.5, 0.25)) == (2.0, 1.5, 0.25)
    near = [(1.0, 0, 5), (float("nan"), 0, 0), (1.0, 0, 2), (0.5, 0, 9)]
    assert FB.fold_of(near, FB.nearest_combine, FB.NEAR_ID) == (0.5, 0, 9)
    assert FB.fold_of(near[:3], FB.nearest_combine, FB.NEAR_ID) == (1.0, 0, 2)
    assert FB.same_record(FB.fold_of(near[1:2], FB.nearest_combine, FB.NEAR_ID), (float("nan"), 0, 0))


def _plan(name, n, chunksize, ring=0, n_workers=1, worker=0):
    plan = _abi.Plan()
    _abi.check(_abi.load().fbr_plan_query(registry.spec(name).func_id, n, chunksize, ring, n_workers, worker, 132,
                                          ctypes.byref(plan)))
    return plan


def test_fold_plan_units_are_powers_of_two():
    for name in FOLD_BODIES:
        for n in (1, 1000, 10 ** 6):
            for ring in (0, 256 << 10):
                u = _plan(name, n, _abi.FBR_PLAN_FOLD, ring).unit_tasks
                assert u & (u - 1) == 0, (name, n, ring, u)
    os.environ["FBR_UNIT_TASKS"] = "100"
    try:
        assert _plan("moments_f64", 10 ** 6, _abi.FBR_PLAN_FOLD).unit_tasks == 64
        assert _plan("moments_f64", 10 ** 6, 32).unit_tasks == 96          # plain maps keep their chunk-aligned unit
    finally:
        del os.environ["FBR_UNIT_TASKS"]
    # the blocks of a two-worker fold map are whole units
    u = _plan("moments_f64", 10 ** 6, _abi.FBR_PLAN_FOLD, n_workers=2).unit_tasks
    b = _plan("moments_f64", 10 ** 6, _abi.FBR_PLAN_FOLD, n_workers=2, worker=1)
    assert b.block_first % u == 0 and b.block_first + b.block_count == 10 ** 6


class _FoldSpec:
    """What the process-pool master needs of a fold body (name, record size, flags, result decoding)."""

    def __init__(self, name):
        self.name, self.result_bytes, self.flags = name, 8, _abi.FBR_BODY_RECORD | _abi.FBR_BODY_FOLD

    def result_dtype(self):
        return np.dtype(np.uint64), ()

    def unpack_result(self, raw):
        return int.from_bytes(raw, "little")


def _pool(n, **kw):
    return ProcessPool(n, devices=list(range(n)), results="bytes", worker_main=fake_fold_worker_main, **kw)


def _want(pool, xs):
    return fake_tree([fake_tree(xs[lo:hi]) for lo, hi in pool.fold_blocks(len(xs)) if hi > lo])


def test_process_pool_folds_block_totals_in_block_order():
    pool = _pool(3, block_tasks=BLOCK_ALIGN)
    try:
        for n in (1, BLOCK_ALIGN, 7 * BLOCK_ALIGN + 123):
            xs = list(range(60000, 60000 + n))          # 0xDEAD (a worker-killing item) is not among them
            r = pool.submit_fold(_FoldSpec("fold_u64"), "map", range(60000, 60000 + n))
            assert r.get(60) == _want(pool, xs)
            assert r.get(1) == _want(pool, xs)
        assert len(pool.fold_blocks(7 * BLOCK_ALIGN + 123)) == 8
        xs = list(range(60000, 60000 + 5 * BLOCK_ALIGN))
        assert pool.submit_fold(_FoldSpec("fold_u64"), "starmap", xs).get(60) == _want(pool, xs)
    finally:
        pool.terminate()
        pool.join()


def test_process_pool_requeues_a_dead_workers_block_and_fold(tmp_path, monkeypatch):
    monkeypatch.setenv("FBR_TEST_FOLD_MARK", str(tmp_path / "died"))
    pool = _pool(2, block_tasks=BLOCK_ALIGN)
    try:
        n = 6 * BLOCK_ALIGN                      # the block holding 0xDEAD kills its worker on the first attempt
        xs = list(range(n))
        assert pool.submit_fold(_FoldSpec("fold_u64"), "map", range(n)).get(120) == _want(pool, xs)
        assert pool.stats["workers_lost"] == 1 and pool.stats["blocks_redispatched"] == 1
        # a worker that dies while folding the totals: the fold goes to another worker
        assert pool.submit_fold(_FoldSpec("fold_dies_once"), "map", range(60000, 60000 + n)).get(120) == \
            _want(pool, list(range(60000, 60000 + n)))
        assert pool.stats["workers_lost"] == 2 and os.path.exists(tmp_path / "died")
    finally:
        pool.terminate()
        pool.join()


def test_process_pool_folds_after_close():
    """close() lets queued folds finish, their block totals included; get() gives the fold, never the untouched record."""
    pool = _pool(2, block_tasks=BLOCK_ALIGN)
    try:
        xs = list(range(60000, 60000 + 5 * BLOCK_ALIGN + 17))
        r1 = pool.submit_fold(_FoldSpec("fold_u64"), "map", range(60000, 60000 + len(xs)))
        r2 = pool.submit_fold(_FoldSpec("fold_u64"), "map", xs[:3 * BLOCK_ALIGN])
        pool.close()
        pool.join(120)
        assert r1.get(1) == _want(pool, xs)
        assert r2.get(1) == _want(pool, xs[:3 * BLOCK_ALIGN])
    finally:
        pool.terminate()
        pool.join()


def test_process_pool_fold_deaths_are_bounded():
    from fiber_b200.procpool import MAX_ATTEMPTS, WorkerDied
    xs = range(60000, 60000 + 2 * BLOCK_ALIGN)
    pool = _pool(2, block_tasks=BLOCK_ALIGN)
    try:
        with pytest.raises(WorkerDied, match="killed its worker %d times" % MAX_ATTEMPTS):
            pool.submit_fold(_FoldSpec("fold_always_dies"), "map", xs).get(120)
        assert pool.stats["workers_lost"] == MAX_ATTEMPTS
        assert pool.submit_fold(_FoldSpec("fold_u64"), "map", xs).get(120) == _want(pool, list(xs))   # the pool keeps serving
    finally:
        pool.terminate()
        pool.join()
    pool = _pool(2, block_tasks=BLOCK_ALIGN, redispatch=False)
    try:
        with pytest.raises(WorkerDied, match="without error_handling"):
            pool.submit_fold(_FoldSpec("fold_always_dies"), "map", xs).get(120)
        assert pool.stats["workers_lost"] == 1
    finally:
        pool.terminate()
        pool.join()
