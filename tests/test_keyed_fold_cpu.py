"""CPU: keyed folds -- registration of hand-written keyed descriptors, header constants, the argument checks Pool.fold_by_key
makes before anything starts, the result handle and layout, the keyed tree() restated in Python (one key is the fold, and
the several-block rule with one block is the one-worker rule), and the process-pool side of keyed fold maps with a
stand-in worker (tests/_fake_keyed_worker.py)."""
import ctypes
import os
import re

import numpy as np
import pytest

import fiber_b200
from fiber_b200 import _abi, registry
from fiber_b200.pool import KeyedFoldResult, KeyedResultArray, host_result

from . import fold_bodies as FB
from . import keyed_bodies as KB

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYED = ["label_sum_u64", "class_moments_f64", "kmeans_step_f32", "label_hist_1k", "wide_sum_16k", "fault_label_u64"]


def _register(entry):
    fid = ctypes.c_int(-1)
    rc = _abi.load().fbr_register_body(entry.encode(), KB.BAD_MODULE.encode(), entry.encode(), ctypes.byref(fid))
    return rc, fid.value, _abi.load().fbr_last_error().decode()


@pytest.mark.parametrize("entry,why", [
    ("bad_keyed_no_fold", "FBR_BODY_KEYED needs FBR_BODY_FOLD"),
    ("bad_keyed_no_keys", "lacks the keys or the fold_segments entry"),
    ("bad_keyed_no_segments", "lacks the keys or the fold_segments entry"),
])
def test_registration_rejects_bad_keyed_descriptors(entry, why):
    rc, _, msg = _register(entry)
    assert rc == _abi.FBR_EINVAL and why in msg, msg


def test_registration_accepts_keyed_descriptors():
    for entry, keyed in (("ok_keyed", True), ("ok_keyed_unflagged", False)):
        rc, fid, msg = _register(entry)
        assert rc == _abi.FBR_OK, msg
        info = _abi.BodyInfo()
        _abi.check(_abi.load().fbr_body_info(fid, ctypes.byref(info)))
        assert info.flags & _abi.FBR_BODY_FOLD
        assert bool(info.flags & _abi.FBR_BODY_KEYED) == keyed


def test_keyed_flags():
    for name in KEYED:
        flags = registry.spec(name).flags
        assert flags & (_abi.FBR_BODY_FOLD | _abi.FBR_BODY_SCAN | _abi.FBR_BODY_KEYED) == 0x700, name
    for name in ("moments_f64", "sum_sq_idx_u64", "nearest_query_f32"):
        assert not registry.spec(name).flags & _abi.FBR_BODY_KEYED


def test_header_constants_match_abi():
    h = open(os.path.join(ROOT, "include", "fiber_b200.h")).read()
    assert int(re.search(r"#define FBR_BODY_KEYED (0x[0-9a-f]+)u", h).group(1), 16) == _abi.FBR_BODY_KEYED == 0x400
    assert int(re.search(r"#define FBR_FOLD_KEYS (0x[0-9a-f]+)u", h).group(1), 16) == _abi.FBR_FOLD_KEYS == 0x10000
    assert int(re.search(r"#define FBR_MAX_KEYS (\d+)u", h).group(1)) == _abi.FBR_MAX_KEYS == 65536
    assert re.search(r"FBR_TASK_KEY = (\d+)", h).group(1) == str(_abi.FBR_TASK_KEY) == "5"
    assert re.search(r"#define FBR_BODY_MODULE_ABI (\d+)", h).group(1) == "4"
    assert ctypes.sizeof(_abi.MapDesc) == 104 and _abi.MapDesc.n_keys.offset == 100
    assert "fbr_fold_segments" in _abi.SYMBOLS
    assert hasattr(_abi.load(), "fbr_fold_segments")


def test_argument_checks_before_anything_starts():
    from . import record_bodies as RB
    p = fiber_b200.Pool(1)
    with pytest.raises(TypeError, match=r"moments_f64 cannot fold by key: it has no key\(\)"):
        p.fold_by_key(FB.moments_f64, [1.0], 2)
    with pytest.raises(TypeError, match="polar_f64 cannot fold"):
        p.starfold_by_key(RB.polar_f64, [(1.0, 2.0)], 2)
    for bad in (0, 65537, -1, 2.0, None, True, np.bool_(True), np.int64(0)):
        with pytest.raises(ValueError, match="n_keys must be an int in 1 .. 65536"):
            p.starfold_by_key(KB.label_sum_u64, [(0, 1)], bad)
    assert p._engine is None and p._proc is None
    from fiber_b200.pool import _n_keys
    assert [_n_keys(k) for k in (1, np.int64(7), np.uint32(65536), np.arange(300).max() + 1)] == [1, 7, 65536, 300]


def test_keyed_result_is_not_iterable():
    h = KeyedFoldResult(None, None, registry.spec("label_sum_u64"), 0, 0, None, _abi.FBR_FOLD_KEYS, n_keys=2)
    for it in (h.iget_ordered, h.iget_unordered):
        with pytest.raises(TypeError, match="label_sum_u64: a keyed fold has one result per key"):
            it()


def test_host_result_reads_records_then_counts():
    import numpy as np
    spec = registry.spec("label_sum_u64")
    recs = np.array([(5, 0, 2), (0, 0, 0), (9, 2, 3)], KB.LABEL_RES)
    data = np.concatenate([recs.view(np.uint8), np.array([2, 0, 3], np.uint64).view(np.uint8)])
    r = host_result(spec, "keyed", data, 3)
    assert r.tolist() == [(5, 0, 2), (0, 0, 0), (9, 2, 3)] and r.counts.dtype == np.uint64 and r.counts.tolist() == [2, 0, 3]


def _label_results(labels, vals):
    return [KB.label_sum_u64(int(k), int(v)) for k, v in zip(labels, vals)]


def test_one_key_is_the_fold():
    import random
    rnd = random.Random(1)
    xs = [(rnd.random() * 100 - 50, 0) for _ in range(777)]
    rs = [KB.class_moments_f64(x, k) for x, k in xs]
    recs, counts = KB.keyed_tree(rs, KB.KEY_OF["class_moments_f64"], KB.moments_combine, KB.MOMENTS_ID, 1)
    assert recs[0] == FB.tree(rs, KB.moments_combine) and counts == [777]


def test_key_k_is_the_fold_of_its_subsequence():
    import random
    rnd = random.Random(2)
    labels = [rnd.randrange(5) for _ in range(1000)]
    rs = [KB.class_moments_f64(rnd.random(), k) for k in labels]
    recs, counts = KB.keyed_tree(rs, KB.KEY_OF["class_moments_f64"], KB.moments_combine, KB.MOMENTS_ID, 6)
    for k in range(6):
        sub = [r for r in rs if r[3] == k]
        assert recs[k] == (FB.tree(sub, KB.moments_combine) if sub else KB.MOMENTS_ID)
        assert counts[k] == len(sub)
    assert counts[5] == 0 and recs[5] == KB.MOMENTS_ID


def test_block_rule():
    import random
    rnd = random.Random(3)
    labels = [rnd.randrange(4) for _ in range(300)]
    rs = _label_results(labels, [rnd.randrange(1 << 32) for _ in labels])
    key, comb = KB.KEY_OF["label_sum_u64"], KB.label_combine
    assert KB.keyed_blocks(rs, key, comb, KB.LABEL_ID, 4, [(0, 300)]) == KB.keyed_tree(rs, key, comb, KB.LABEL_ID, 4)
    # an integer sum does not depend on the cut; the counts never do
    two = KB.keyed_blocks(rs, key, comb, KB.LABEL_ID, 4, [(0, 128), (128, 300)])
    assert two == KB.keyed_tree(rs, key, comb, KB.LABEL_ID, 4)


# ---- process isolation, with a stand-in worker (tests/_fake_keyed_worker.py) ----------------------------------------------
class _KeyedSpec:
    """What the process-pool master needs of a keyed body (name, record size, flags, result decoding)."""

    def __init__(self, name):
        self.name, self.result_bytes = name, 8
        self.flags = _abi.FBR_BODY_RECORD | _abi.FBR_BODY_FOLD | _abi.FBR_BODY_KEYED

    def result_dtype(self):
        import numpy as np
        return np.dtype(np.uint64), ()

    def to_python(self, row):
        return int(row)

    def rows_to_list(self, arr):
        return [int(x) for x in arr]


def _proc_pool(n, **kw):
    from fiber_b200.procpool import ProcessPool
    from ._fake_keyed_worker import fake_keyed_worker_main
    return ProcessPool(n, devices=list(range(n)), results="bytes", worker_main=fake_keyed_worker_main, **kw)


def _proc_want(pool, xs, n_keys):
    """The keyed result of the process pool's block cut: per key, tree() over the non-empty block totals in block order."""
    from ._fake_fold_worker import tree
    from ._fake_keyed_worker import keyed
    totals, counts = [[] for _ in range(n_keys)], [0] * n_keys
    for lo, hi in pool.fold_blocks(len(xs)):
        recs, cnt = keyed(xs[lo:hi], n_keys)
        for k in range(n_keys):
            if cnt[k]:
                totals[k].append(recs[k])
                counts[k] += cnt[k]
    return [tree(t) if t else 0 for t in totals], counts


def _check_proc(r, want):
    assert r.tolist() == want[0] and r.counts.tolist() == want[1]


def test_process_pool_folds_each_key_over_block_totals_in_block_order():
    from fiber_b200.procpool import BLOCK_ALIGN
    pool = _proc_pool(3, block_tasks=BLOCK_ALIGN)
    try:
        for n, n_keys in ((1, 3), (BLOCK_ALIGN, 1), (7 * BLOCK_ALIGN + 123, 5), (3 * BLOCK_ALIGN, 300)):
            xs = list(range(60000, 60000 + n))          # 0xDEAD (a worker-killing item) is not among them
            _check_proc(pool.submit_fold_by_key(_KeyedSpec("keyed_u64"), "map", range(60000, 60000 + n), n_keys).get(60),
                        _proc_want(pool, xs, n_keys))
        xs = list(range(60000, 60000 + 5 * BLOCK_ALIGN))
        _check_proc(pool.submit_fold_by_key(_KeyedSpec("keyed_u64"), "starmap", xs, 4).get(60), _proc_want(pool, xs, 4))
    finally:
        pool.terminate()
        pool.join()


def test_process_pool_requeues_a_dead_workers_block_and_keyed_step(tmp_path, monkeypatch):
    from fiber_b200.procpool import BLOCK_ALIGN
    monkeypatch.setenv("FBR_TEST_FOLD_MARK", str(tmp_path / "died"))
    pool = _proc_pool(2, block_tasks=BLOCK_ALIGN)
    try:
        n = 6 * BLOCK_ALIGN                      # the block holding 0xDEAD kills its worker on the first attempt
        _check_proc(pool.submit_fold_by_key(_KeyedSpec("keyed_u64"), "map", range(n), 6).get(120), _proc_want(pool, list(range(n)), 6))
        assert pool.stats["workers_lost"] == 1 and pool.stats["blocks_redispatched"] == 1
        # a worker that dies while folding the totals: the step goes to another worker
        xs = list(range(60000, 60000 + n))
        _check_proc(pool.submit_fold_by_key(_KeyedSpec("keyed_dies_once"), "map", range(60000, 60000 + n), 6).get(120),
                    _proc_want(pool, xs, 6))
        assert pool.stats["workers_lost"] == 2 and os.path.exists(tmp_path / "died")
    finally:
        pool.terminate()
        pool.join()


def test_process_pool_keyed_step_runs_after_close_and_not_after_terminate():
    from fiber_b200.procpool import BLOCK_ALIGN
    pool = _proc_pool(2, block_tasks=BLOCK_ALIGN)
    try:
        xs = list(range(60000, 60000 + 5 * BLOCK_ALIGN + 17))
        r = pool.submit_fold_by_key(_KeyedSpec("keyed_u64"), "map", range(60000, 60000 + len(xs)), 9)
        pool.close()
        pool.join(120)
        _check_proc(r.get(1), _proc_want(pool, xs, 9))
    finally:
        pool.terminate()
        pool.join()
    pool = _proc_pool(1, block_tasks=BLOCK_ALIGN)
    try:
        pool.wait_until_workers_up()
        pool.terminate()
        with pytest.raises(ValueError, match="Pool is not running"):
            pool.submit_fold_by_key(_KeyedSpec("keyed_u64"), "map", range(10), 2)
    finally:
        pool.join()


def test_keyed_sequence_is_key_major_in_block_order():
    import numpy as np
    from fiber_b200.procpool import keyed_sequence

    def area(recs, counts):
        return np.concatenate([np.array(recs, np.uint64), np.array(counts, np.uint64)]).view(np.uint8)
    values, offsets, counts = keyed_sequence([area([10, 11, 12], [1, 0, 2]), area([20, 21, 22], [3, 0, 0])], 3, 8)
    assert values.view(np.uint64).tolist() == [10, 20, 12] and offsets.tolist() == [0, 2, 2, 3] and counts.tolist() == [4, 0, 2]
