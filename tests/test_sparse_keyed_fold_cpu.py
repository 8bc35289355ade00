"""CPU: sparse keyed folds -- header constants, the checks Pool.fold_by_sparse_key makes before anything starts, the result
handle and layout, the host merge of the process pool's last step (sparse_keyed_sequence) against a Python restatement,
and the process-pool side of sparse keyed fold maps with a stand-in worker (tests/_fake_sparse_keyed_worker.py)."""
import collections
import os
import re

import numpy as np
import pytest

import fiber_b200
from fiber_b200 import _abi, registry
from fiber_b200.pool import SparseKeyedFoldResult, SparseKeyedResultArray, host_result

from . import fold_bodies as FB
from . import keyed_bodies as KB

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_constants_match_abi():
    h = open(os.path.join(ROOT, "include", "fiber_b200.h")).read()
    assert int(re.search(r"#define FBR_FOLD_SPARSE_KEYS (0x[0-9a-f]+)u", h).group(1), 16) == _abi.FBR_FOLD_SPARSE_KEYS == 0x20000
    assert not _abi.FBR_FOLD_SPARSE_KEYS & (_abi.FBR_FOLD | _abi.FBR_SCAN | _abi.FBR_FOLD_KEYS | _abi.FBR_NO_ZERO_COPY)
    assert re.search(r"int fbr_result_groups\(fbr_pool_t\* pool, uint64_t seq, uint64_t\* n_groups", h)
    assert "fbr_result_groups" in _abi.SYMBOLS and hasattr(_abi.load(), "fbr_result_groups")


def test_argument_checks_before_anything_starts():
    from . import record_bodies as RB
    p = fiber_b200.Pool(1)
    with pytest.raises(TypeError, match=r"moments_f64 cannot fold by key: it has no key\(\)"):
        p.fold_by_sparse_key(FB.moments_f64, [1.0])
    with pytest.raises(TypeError, match=r"moments_f64 cannot fold by key: it has no key\(\)"):
        p.fold_by_sparse_key_async(FB.moments_f64, [1.0])
    with pytest.raises(TypeError, match="polar_f64 cannot fold"):
        p.starfold_by_sparse_key(RB.polar_f64, [(1.0, 2.0)])
    with pytest.raises(TypeError):
        p.fold_by_sparse_key(KB.class_moments_f64, [], 4)            # no n_keys, no chunksize
    assert p._engine is None and p._proc is None


def test_sparse_result_is_not_iterable():
    h = SparseKeyedFoldResult(None, None, registry.spec("label_sum_u64"), 0, 0, None, _abi.FBR_FOLD_SPARSE_KEYS)
    for it in (h.iget_ordered, h.iget_unordered):
        with pytest.raises(TypeError, match="label_sum_u64: a sparse keyed fold has one result per distinct key"):
            it()
    r = h.get()                                  # a map over no tasks: no record, key or count
    assert isinstance(r, SparseKeyedResultArray) and len(r) == 0 and r.keys.dtype == np.uint32 and r.counts.dtype == np.uint64


def test_host_result_reads_records_counts_and_keys():
    spec = registry.spec("label_sum_u64")
    recs = np.array([(5, 3, 2), (9, 70_000, 3), (1, 0xFFFFFFFE, 1)], KB.LABEL_RES)
    data = np.concatenate([recs.view(np.uint8), np.array([2, 3, 1], np.uint64).view(np.uint8),
                           np.array([3, 70_000, 0xFFFFFFFE], np.uint32).view(np.uint8)])
    r = host_result(spec, "sparse", data, 3)
    assert r.tolist() == [(5, 3, 2), (9, 70_000, 3), (1, 0xFFFFFFFE, 1)]
    assert r.keys.dtype == np.uint32 and r.keys.tolist() == [3, 70_000, 0xFFFFFFFE]
    assert r.counts.dtype == np.uint64 and r.counts.tolist() == [2, 3, 1]
    assert r.get(70_000) == (9, 70_000, 3) and r.get(4) is None and r.get(0xFFFFFFFF, "none") == "none"
    assert r.get(np.uint32(3)) == (5, 3, 2) and r[-1] == (1, 0xFFFFFFFE, 1)
    assert len(host_result(spec, "sparse", None, 0)) == 0


def _restated(blocks):
    """sparse_keyed_sequence restated: per key in ascending order, the block totals of the blocks holding it in block
    order, and the summed counts."""
    per_key = collections.defaultdict(list)
    counts = collections.Counter()
    for keys, recs, cnt in blocks:
        for k, r, c in zip(keys.tolist(), recs, cnt.tolist()):
            per_key[k].append(bytes(r))
            counts[k] += c
    keys = sorted(per_key)
    values = b"".join(b"".join(per_key[k]) for k in keys)
    offsets = np.cumsum([0] + [len(per_key[k]) for k in keys]).tolist()
    return values, offsets, keys, [counts[k] for k in keys]


@pytest.mark.parametrize("seed", range(12))
def test_sparse_keyed_sequence_against_its_restatement(seed):
    from fiber_b200.procpool import sparse_keyed_sequence
    rng = np.random.default_rng(seed)
    R = int(rng.choice([4, 8, 24]))
    pool_keys = rng.integers(0, 0xFFFFFFFF, int(rng.integers(1, 50)), dtype=np.uint64).astype(np.uint32)
    blocks = []
    for _ in range(int(rng.integers(1, 6))):
        D = int(rng.integers(0, len(pool_keys) + 1))       # empty blocks too; keys shared by some blocks only
        keys = np.sort(rng.choice(pool_keys, D, replace=False)).astype(np.uint32)
        blocks.append((keys, rng.integers(0, 256, (D, R), dtype=np.uint8), rng.integers(1, 1000, D, dtype=np.uint64)))
    values, offsets, keys, counts = sparse_keyed_sequence(*zip(*blocks))
    want = _restated(blocks)
    assert values.tobytes() == want[0] and offsets.tolist() == want[1]
    assert keys.dtype == np.uint32 and keys.tolist() == want[2]
    assert counts.dtype == np.uint64 and counts.tolist() == want[3]


def test_sparse_area_reads_a_block_file():
    from fiber_b200.procpool import sparse_area
    from ._fake_sparse_keyed_worker import area
    keys, recs, counts = sparse_area(area([10, 20], [4, 1 << 31], [7, 1]), 8)
    assert keys.tolist() == [4, 1 << 31] and recs.view(np.uint64).ravel().tolist() == [10, 20] and counts.tolist() == [7, 1]


# ---- process isolation, with a stand-in worker (tests/_fake_sparse_keyed_worker.py) -------------------------------------
class _SparseSpec:
    """What the process-pool master needs of a keyed body (name, record size, flags, result decoding)."""

    def __init__(self, name):
        self.name, self.result_bytes = name, 8
        self.flags = _abi.FBR_BODY_RECORD | _abi.FBR_BODY_FOLD | _abi.FBR_BODY_KEYED

    def result_dtype(self):
        return np.dtype(np.uint64), ()

    def to_python(self, row):
        return int(row)

    def rows_to_list(self, arr):
        return [int(x) for x in arr]


def _proc_pool(n, **kw):
    from fiber_b200.procpool import ProcessPool
    from ._fake_sparse_keyed_worker import fake_sparse_worker_main
    return ProcessPool(n, devices=list(range(n)), results="bytes", worker_main=fake_sparse_worker_main, **kw)


def _proc_want(pool, xs):
    """The sparse keyed result of the process pool's block cut: per key, tree() over the block totals in block order."""
    from ._fake_fold_worker import tree
    from ._fake_sparse_keyed_worker import sparse
    totals, counts = collections.defaultdict(list), collections.Counter()
    for lo, hi in pool.fold_blocks(len(xs)):
        for r, k, c in zip(*sparse(xs[lo:hi])):
            totals[k].append(r)
            counts[k] += c
    keys = sorted(totals)
    return [tree(totals[k]) for k in keys], keys, [counts[k] for k in keys]


def _check_proc(r, want):
    assert r.tolist() == want[0] and r.keys.tolist() == want[1] and r.counts.tolist() == want[2]


def test_process_pool_folds_each_key_over_block_totals_in_block_order():
    from fiber_b200.procpool import BLOCK_ALIGN
    pool = _proc_pool(3, block_tasks=BLOCK_ALIGN)
    try:
        for n in (1, BLOCK_ALIGN, 7 * BLOCK_ALIGN + 123):
            xs = list(range(60000, 60000 + n))          # 0xDEAD (a worker-killing item) is not among them
            _check_proc(pool.submit_fold_by_sparse_key(_SparseSpec("sparse_u64"), "map", range(60000, 60000 + n)).get(60),
                        _proc_want(pool, xs))
        xs = list(range(60000, 60000 + 5 * BLOCK_ALIGN))
        _check_proc(pool.submit_fold_by_sparse_key(_SparseSpec("sparse_u64"), "starmap", xs).get(60), _proc_want(pool, xs))
        r = pool.submit_fold_by_sparse_key(_SparseSpec("sparse_u64"), "map", range(0)).get(10)
        assert len(r) == 0
    finally:
        pool.terminate()
        pool.join()


def test_process_pool_requeues_a_dead_workers_block_and_sparse_step(tmp_path, monkeypatch):
    from fiber_b200.procpool import BLOCK_ALIGN
    monkeypatch.setenv("FBR_TEST_FOLD_MARK", str(tmp_path / "died"))
    pool = _proc_pool(2, block_tasks=BLOCK_ALIGN)
    try:
        n = 6 * BLOCK_ALIGN                      # the block holding 0xDEAD kills its worker on the first attempt
        _check_proc(pool.submit_fold_by_sparse_key(_SparseSpec("sparse_u64"), "map", range(n)).get(120), _proc_want(pool, list(range(n))))
        assert pool.stats["workers_lost"] == 1 and pool.stats["blocks_redispatched"] == 1
        # a worker that dies during the last step: the step goes to another worker
        xs = list(range(60000, 60000 + n))
        _check_proc(pool.submit_fold_by_sparse_key(_SparseSpec("sparse_dies_once"), "map", range(60000, 60000 + n)).get(120),
                    _proc_want(pool, xs))
        assert pool.stats["workers_lost"] == 2 and os.path.exists(tmp_path / "died")
    finally:
        pool.terminate()
        pool.join()


def test_process_pool_sparse_step_runs_after_close_and_not_after_terminate():
    from fiber_b200.procpool import BLOCK_ALIGN
    pool = _proc_pool(2, block_tasks=BLOCK_ALIGN)
    try:
        xs = list(range(60000, 60000 + 5 * BLOCK_ALIGN + 17))
        r = pool.submit_fold_by_sparse_key(_SparseSpec("sparse_u64"), "map", range(60000, 60000 + len(xs)))
        pool.close()
        pool.join(120)
        _check_proc(r.get(1), _proc_want(pool, xs))
    finally:
        pool.terminate()
        pool.join()
    pool = _proc_pool(1, block_tasks=BLOCK_ALIGN)
    try:
        pool.wait_until_workers_up()
        pool.terminate()
        with pytest.raises(ValueError, match="Pool is not running"):
            pool.submit_fold_by_sparse_key(_SparseSpec("sparse_u64"), "map", range(10))
    finally:
        pool.join()
