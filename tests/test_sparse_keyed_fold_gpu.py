"""GPU: sparse keyed folds (Pool.fold_by_sparse_key / starfold_by_sparse_key, FBR_FOLD_SPARSE_KEYS) of the bodies in
tests/keyed_bodies.py -- sizes around the scan tile and the sort tile, key distributions that exercise each radix pass
alone, float combines bit for bit against the Python restatement, the identity with fold_by_key on dense keys, independence
from ring size, chunksize, arrival and placement, error handling, the items and group record paths, a word count, the
reserved key, the refusals, the bytes that cross PCIe, process isolation and two GPUs.  Every record is compared byte for
byte, and every key and count exactly."""
import collections
import ctypes

import numpy as np
import pytest

import fiber_b200
from fiber_b200 import _abi, registry

from . import emit_bodies as EB
from . import keyed_bodies as KB

pytestmark = pytest.mark.gpu

SMALL_RING = 256 << 10
RESERVED = 0xFFFFFFFF


def sparse_keyed_tree(results, key, combine):
    """FBR_FOLD_SPARSE_KEYS on one worker: for each distinct key in ascending order, tree() of the results whose key it is,
    in task order; the keys and the counts."""
    groups = collections.defaultdict(list)
    for r in results:
        groups[key(r)].append(r)
    keys = sorted(groups)
    return [KB.tree(groups[k], combine) for k in keys], keys, [len(groups[k]) for k in keys]


def sparse_keyed_blocks(results, key, combine, cuts):
    """FBR_FOLD_SPARSE_KEYS on several blocks: each block [lo, hi) of ``cuts`` folds its own keys, and record k is tree()
    over the totals of the blocks where k has a task, in block order; counts are summed."""
    totals, counts = collections.defaultdict(list), collections.Counter()
    for lo, hi in cuts:
        recs, keys, cnt = sparse_keyed_tree(results[lo:hi], key, combine)
        for r, k, c in zip(recs, keys, cnt):
            totals[k].append(r)
            counts[k] += c
    keys = sorted(totals)
    return [KB.tree(totals[k], combine) for k in keys], keys, [counts[k] for k in keys]


@pytest.fixture(scope="module")
def pool():
    p = fiber_b200.Pool(1, devices=[0])
    yield p
    p.terminate()
    p.join()


@pytest.fixture(scope="module")
def small():
    p = fiber_b200.Pool(1, devices=[0], ring_bytes=SMALL_RING)
    yield p
    p.terminate()
    p.join()


def sparse_labels(n, dist, seed=0):
    """n uint32 keys of distribution ``dist`` (never the reserved key)."""
    rng = np.random.default_rng(seed)
    if dist == "single":
        k = np.full(n, 0x9E3779B9, np.uint64)
    elif dist == "distinct":                            # D = n
        k = rng.permutation(n).astype(np.uint64) * 2654435761 % RESERVED
    elif dist == "uniform32":
        k = rng.integers(0, RESERVED, n, dtype=np.uint64)
    elif dist.startswith("byte"):                       # keys that differ in byte j only: radix pass j alone sorts them
        j = int(dist[4:])
        k = (np.uint64(0x5A5A5A5A) & ~np.uint64(0xFF << (8 * j))) | (rng.integers(0, 256, n, dtype=np.uint64) << np.uint64(8 * j))
    elif dist == "clustered":                           # at both ends of the key range
        off = rng.integers(0, 16, n, dtype=np.uint64)
        k = np.where(rng.integers(0, 2, n) == 1, off, np.uint64(RESERVED - 1) - off)
    else:                                               # "zipf"
        k = np.minimum(rng.zipf(1.3, n), RESERVED - 1).astype(np.uint64)
    return k.astype(np.uint32), rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)


def label_expected(labels, vals):
    """The records, keys and counts of label_sum_u64: an integer sum per key, so any order gives the same bits."""
    keys, inv = np.unique(labels, return_inverse=True)
    sums = np.zeros(len(keys), np.uint64)
    np.add.at(sums, inv, vals.astype(np.uint64))
    counts = np.bincount(inv, minlength=len(keys)).astype(np.uint64)
    want = np.zeros(len(keys), KB.LABEL_RES)
    want["sum"], want["key"], want["n"] = sums, keys, counts.astype(np.uint32)
    return want, keys.astype(np.uint32), counts


def check_label(r, labels, vals):
    want, keys, counts = label_expected(labels, vals)
    assert len(r) == len(keys)
    np.testing.assert_array_equal(r.keys, keys)
    np.testing.assert_array_equal(r.counts, counts)
    assert r.keys.dtype == np.uint32 and r.counts.dtype == np.uint64
    assert np.asarray(r.array).tobytes() == want.tobytes()


def same_bits(a, b):
    return (np.asarray(a.array).tobytes() == np.asarray(b.array).tobytes() and np.array_equal(a.keys, b.keys)
            and np.array_equal(a.counts, b.counts))


SIZES = (0, 1, 2, 2047, 2048, 2049, 4095, 4096, 4097, 1_000_003)


@pytest.mark.parametrize("dist", ["single", "distinct", "uniform32", "byte0", "byte1", "byte2", "byte3", "clustered", "zipf"])
def test_sizes_and_key_distributions(pool, dist):
    for n in SIZES:
        labels, vals = sparse_labels(n, dist, seed=n + len(dist))
        r = pool.starfold_by_sparse_key(KB.label_sum_u64, fiber_b200.Columns(labels, vals))
        check_label(r, labels, vals)
        if dist == "distinct":
            assert len(r) == n
        if n and dist == "single":
            assert len(r) == 1


def moments_inputs(n, keys, seed):
    rng = np.random.default_rng(seed)
    a = np.zeros(n, KB.MOMENTS_ARG)
    a["x"] = rng.standard_normal(n) * 1e3
    a["label"] = rng.choice(np.asarray(keys, np.uint32), n)
    return a


def moments_results(a):
    return [KB.class_moments_f64(float(x), int(k)) for x, k in zip(a["x"], a["label"])]


def test_class_moments_bits(pool):
    for n, n_keys in ((1, 3), (513, 3), (4097, 40), (20_000, 7), (20_000, 3000)):
        keys = np.random.default_rng(n).integers(0, RESERVED, n_keys, dtype=np.uint64)
        a = moments_inputs(n, keys, seed=n + n_keys)
        r = pool.fold_by_sparse_key(KB.class_moments_f64, a)
        want, wkeys, counts = sparse_keyed_tree(moments_results(a), KB.KEY_OF["class_moments_f64"], KB.moments_combine)
        assert r.tolist() == want and r.keys.tolist() == wkeys and r.counts.tolist() == counts
        assert r.get(wkeys[-1]) == want[-1] and r.get(RESERVED) is None and r.get(RESERVED, 5) == 5


def test_each_key_is_the_fold_of_its_subsequence(pool):
    a = moments_inputs(30_000, [7, 1 << 20, 0xABCDEF01, RESERVED - 1], seed=8)
    r = pool.fold_by_sparse_key(KB.class_moments_f64, a)
    for i, k in enumerate(r.keys):
        assert r[i] == pool.fold(KB.class_moments_f64, a[a["label"] == k]), k


def test_dense_keys_equal_fold_by_key_without_its_empty_keys(pool):
    for n, dist, seed in ((100_000, "uniform", 1), (5_000, "sparse", 2), (70_001, "skewed", 3)):
        rng = np.random.default_rng(seed)
        labels = {"uniform": rng.integers(0, 65536, n), "sparse": rng.choice(np.arange(0, 65536, 977), n),
                  "skewed": np.minimum(rng.geometric(0.01, n), 65535)}[dist]
        a = moments_inputs(n, [0], seed)
        a["label"] = labels
        dense = pool.fold_by_key(KB.class_moments_f64, a, 65536)
        r = pool.fold_by_sparse_key(KB.class_moments_f64, a)
        nz = np.flatnonzero(dense.counts)
        np.testing.assert_array_equal(r.keys, nz)
        np.testing.assert_array_equal(r.counts, dense.counts[nz])
        assert np.asarray(r.array).tobytes() == np.asarray(dense.array)[nz].tobytes()


def _raw_sparse(p, name, xs, flags=0, dev_args=False, chunksize=0, n_keys=0):
    """A sparse keyed fold through the C ABI (map flags the Pool API does not take): (record bytes, keys, counts)."""
    spec = registry.spec(name)
    star = isinstance(xs, fiber_b200.Columns)
    enc = spec.encode_starmap(xs) if star else spec.encode_map(xs)
    eng, lib = p._engine, p._engine.lib
    d = _abi.MapDesc()
    d.func_id, d.flags, d.n_tasks, d.n_keys, d.shuffle_seed = spec.func_id, flags | _abi.FBR_FOLD_SPARSE_KEYS, enc.n, n_keys, 17
    d.flags |= _abi.FBR_STARMAP if star else _abi.FBR_MAP
    d.arg_stride, d.chunksize = enc.arg_stride, chunksize
    dptr = ctypes.c_void_p()
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
        done = ctypes.c_uint64(1)
        _abi.check(lib.fbr_result_poll(eng.handle, seq.value, ctypes.byref(done)))
        assert done.value in (0, enc.n)
        g, kp, cp = ctypes.c_uint64(), ctypes.c_void_p(), ctypes.c_void_p()
        assert lib.fbr_result_groups(eng.handle, seq.value, ctypes.byref(g), ctypes.byref(kp), ctypes.byref(cp)) == _abi.FBR_EINVAL \
            or done.value == enc.n
        res = _abi.Result()
        _abi.check(lib.fbr_result_wait(eng.handle, seq.value, -1, ctypes.byref(res)))
        _abi.check(lib.fbr_result_groups(eng.handle, seq.value, ctypes.byref(g), ctypes.byref(kp), ctypes.byref(cp)))
        D = g.value
        out = ctypes.string_at(res.data, D * spec.result_bytes)
        keys = np.frombuffer(ctypes.string_at(kp, 4 * D), np.uint32)
        counts = np.frombuffer(ctypes.string_at(cp, 8 * D), np.uint64)
        assert lib.fbr_result_fetch(eng.handle, seq.value, 0, 0, None) == _abi.FBR_EINVAL
        _abi.check(lib.fbr_result_release(eng.handle, seq.value))
    finally:
        if dptr.value:
            lib.fbr_device_free(eng.handle, 0, dptr)
    return out, keys, counts


def test_independent_of_ring_chunksize_arrival_and_placement(pool, small):
    a = moments_inputs(60_000, np.random.default_rng(12).integers(0, RESERVED, 3000, dtype=np.uint64), seed=12)
    want = pool.fold_by_sparse_key(KB.class_moments_f64, a)
    ref = (np.asarray(want.array).tobytes(), np.asarray(want.keys), np.asarray(want.counts))
    before = small.stats()["dispatch_launches"]
    assert same_bits(small.fold_by_sparse_key(KB.class_moments_f64, a), want)
    assert small.stats()["dispatch_launches"] - before >= 4          # many waves
    cases = [(pool, _abi.FBR_SHUFFLE, False, 0), (pool, _abi.FBR_VIA_RING, False, 0), (small, _abi.FBR_SHUFFLE, False, 0),
             (pool, 0, True, 0), (pool, _abi.FBR_RESULTS_ON_DEVICE, False, 0)]
    cases += [(p, 0, False, c) for p in (pool, small) for c in (1, 7, 32, 1000)]
    for p, flags, dev, chunk in cases:
        recs, keys, counts = _raw_sparse(p, "class_moments_f64", a, flags, dev, chunk)
        assert recs == ref[0] and np.array_equal(keys, ref[1]) and np.array_equal(counts, ref[2]), (flags, dev, chunk)


def test_results_on_device():
    a = moments_inputs(10_000, [3, 99, 1 << 31], seed=13)
    p = fiber_b200.Pool(1, devices=[0], results="device")
    q = fiber_b200.Pool(1, devices=[0])
    try:
        assert same_bits(p.fold_by_sparse_key(KB.class_moments_f64, a), q.fold_by_sparse_key(KB.class_moments_f64, a))
    finally:
        for x in (p, q):
            x.terminate()
            x.join()


def test_error_handling_gives_the_same_bits():
    xs = range(50_000)
    rs = [KB.fault_label_u64(i) for i in xs]
    want, keys, counts = sparse_keyed_tree(rs, KB.KEY_OF["fault_label_u64"], KB.label_combine)
    p = fiber_b200.Pool(1, devices=[0], error_handling=True)
    try:
        r = p.fold_by_sparse_key(KB.fault_label_u64, xs)
        assert r.tolist() == want and r.keys.tolist() == keys and r.counts.tolist() == counts
        assert p.stats()["units_redispatched"] > 0
    finally:
        p.terminate()
        p.join()


def test_items_and_group_bodies(pool):
    rng = np.random.default_rng(11)
    labels = rng.choice(np.array([5, 1 << 17, 0xFFFF0000, 77], np.uint32), 1500)
    strs = [bytes(rng.integers(0, 256, rng.integers(0, 300), dtype=np.uint8)) for _ in labels]
    r = pool.starfold_by_sparse_key(KB.label_hist_1k, list(zip(strs, labels.tolist())))
    rs = [KB.label_hist_1k(s, int(k)) for k, s in zip(labels, strs)]
    want, keys, counts = sparse_keyed_tree(rs, KB.KEY_OF["label_hist_1k"], KB.hist_combine)
    assert r.keys.tolist() == keys and r.counts.tolist() == counts
    assert [(list(x[0]), x[1]) for x in r.tolist()] == [(list(w[0]), w[1]) for w in want]

    w = np.zeros(700, KB.WIDE_ARG)
    w["label"] = rng.choice(np.array([0, 9, 1 << 30, RESERVED - 1], np.uint32), 700)
    w["seed"] = rng.integers(0, 1 << 32, 700, dtype=np.uint64)
    r = pool.fold_by_sparse_key(KB.wide_sum_16k, w)
    ukeys = np.unique(w["label"])
    np.testing.assert_array_equal(r.keys, ukeys)
    for i, k in enumerate(ukeys):
        sel = w[w["label"] == k]
        v = np.zeros(4092, np.uint64)
        for s in sel["seed"]:
            v += KB.wide_words(int(s))
        assert r.counts[i] == len(sel)
        assert np.array_equal(np.asarray(r.array[i]["v"]), (v & np.uint64(KB.M32)).astype(np.uint32)), k
        assert r.array[i]["key"] == k


def test_word_count(pool):
    rng = np.random.default_rng(21)
    vocab = [bytes(rng.integers(97, 123, rng.integers(1, 12), dtype=np.uint8)) for _ in range(5000)]
    zipf = np.minimum(rng.zipf(1.2, 200_000), len(vocab)) - 1
    docs, at = [], 0
    while at < len(zipf):
        k = int(rng.integers(0, 400))
        docs.append(b" ".join(vocab[i] for i in zipf[at:at + k]) + b"\n" * int(rng.integers(0, 2)))
        at += k
    h = np.asarray(pool.map(EB.tokens_u32, docs).ragged.values, np.uint32)
    ones = np.ones(len(h), np.uint32)
    r = pool.starfold_by_sparse_key(KB.label_sum_u64, fiber_b200.Columns(h, ones))
    want = collections.Counter(EB.fnv1a32(t) for d in docs for t in d.split())
    assert r.keys.tolist() == sorted(want)
    assert r.counts.tolist() == [want[k] for k in sorted(want)]
    assert [x[0] for x in r.tolist()] == [want[k] for k in sorted(want)]


def test_reserved_key_raises_for_the_lowest_task(pool):
    labels, vals = sparse_labels(100_000, "uniform32", seed=14)
    labels[[70_000, 31_337, 99_999]] = RESERVED
    with pytest.raises(ValueError, match=r"label_sum_u64: key\(\) of task 31337 is 0xffffffff, which fold_by_sparse_key reserves"):
        pool.starfold_by_sparse_key(KB.label_sum_u64, fiber_b200.Columns(labels, vals))
    labels[[70_000, 31_337, 99_999]] = RESERVED - 1
    check_label(pool.starfold_by_sparse_key(KB.label_sum_u64, fiber_b200.Columns(labels, vals)), labels, vals)


def test_empty_map(pool):
    r = pool.starfold_by_sparse_key(KB.class_moments_f64, [])
    assert len(r) == 0 and r.keys.tolist() == [] and r.counts.tolist() == [] and r.get(3) is None


def test_refusals(pool):
    spec = registry.spec("label_sum_u64")
    labels, vals = sparse_labels(100, "uniform32")
    cols = fiber_b200.Columns(labels, vals)
    for flags in (_abi.FBR_FOLD, _abi.FBR_SCAN, _abi.FBR_FOLD_KEYS):
        with pytest.raises(_abi.EngineError, match="FBR_FOLD_SPARSE_KEYS cannot be combined"):
            _raw_sparse(pool, "label_sum_u64", cols, flags, n_keys=4 if flags == _abi.FBR_FOLD_KEYS else 0)
    for flags in (_abi.FBR_WANT_SUM, _abi.FBR_NO_ZERO_COPY):
        with pytest.raises(_abi.EngineError, match="sparse keyed fold map .* owns its result records"):
            _raw_sparse(pool, "label_sum_u64", cols, flags)
    out = np.zeros(100 * spec.result_bytes, np.uint8)
    for flags in (0, _abi.FBR_OUT_DEVICE):
        enc = spec.encode_starmap(cols)
        d = _abi.MapDesc()
        d.func_id, d.flags, d.n_tasks = spec.func_id, flags | _abi.FBR_FOLD_SPARSE_KEYS | _abi.FBR_STARMAP, enc.n
        d.arg_stride, d.args, d.out = enc.arg_stride, enc.args.ctypes.data, out.ctypes.data
        rc = pool._engine.lib.fbr_map_submit(pool._engine.handle, ctypes.byref(d), ctypes.byref(ctypes.c_uint64()))
        assert rc == _abi.FBR_EINVAL and "owns its result records" in _abi.load().fbr_last_error().decode()
    with pytest.raises(_abi.EngineError, match="takes no n_keys"):
        _raw_sparse(pool, "label_sum_u64", cols, n_keys=5)
    with pytest.raises(_abi.EngineError, match="has no key"):
        d = _abi.MapDesc()
        d.func_id, d.flags, d.n_tasks = registry.spec("sum_sq_idx_u64").func_id, _abi.FBR_FOLD_SPARSE_KEYS, 10
        _abi.check(pool._engine.lib.fbr_map_submit(pool._engine.handle, ctypes.byref(d), ctypes.byref(ctypes.c_uint64())))
    # fbr_result_groups refuses other maps
    r = pool.starfold_by_key_async(KB.label_sum_u64, fiber_b200.Columns(labels % 4, vals), 4)
    r.get()
    g, kp, cp = ctypes.c_uint64(), ctypes.c_void_p(), ctypes.c_void_p()
    assert pool._engine.lib.fbr_result_groups(pool._engine.handle, r._seq, ctypes.byref(g), ctypes.byref(kp),
                                              ctypes.byref(cp)) == _abi.FBR_EINVAL


def test_d2h_bytes_follow_the_distinct_keys_not_the_tasks(pool):
    R = registry.spec("label_sum_u64").result_bytes
    for n, n_keys in ((1_000_000, 10), (1_000_000, 1000)):
        rng = np.random.default_rng(n_keys)
        labels = rng.choice(rng.integers(0, RESERVED, n_keys, dtype=np.uint64), n).astype(np.uint32)
        vals = np.ones(n, np.uint32)
        before = pool.stats()["d2h_bytes"]
        r = pool.starfold_by_sparse_key(KB.label_sum_u64, fiber_b200.Columns(labels, vals))
        D = len(r)
        assert D == len(np.unique(labels))
        assert pool.stats()["d2h_bytes"] - before == D * R + 4 * D + 8 * (D + 1)


def test_process_isolation_equals_thread_isolation_on_the_same_block_cut():
    """A process-isolated pool cuts the map into blocks of its own: each block's sparse keyed fold is what a thread pool
    gives for that block, and record k folds the totals of the blocks where k has a task, in block order."""
    keys = np.random.default_rng(18).integers(0, RESERVED, 40, dtype=np.uint64)
    a = moments_inputs(150_001, keys, seed=18)
    a["label"][:5000] = 3                                   # a key of the first block only
    p = fiber_b200.Pool(1, isolation="process", error_handling=True)
    q = fiber_b200.Pool(1, devices=[0])
    try:
        r = p.fold_by_sparse_key(KB.class_moments_f64, a)
        cuts = p._proc.fold_blocks(len(a))
        assert len(cuts) > 1
        want, wkeys, counts = sparse_keyed_blocks(moments_results(a), KB.KEY_OF["class_moments_f64"], KB.moments_combine, cuts)
        assert r.tolist() == want and r.keys.tolist() == wkeys and r.counts.tolist() == counts
        blocks = [q.fold_by_sparse_key(KB.class_moments_f64, a[lo:hi]) for lo, hi in cuts]
        for i, k in enumerate(r.keys):
            totals = [b.get(k) for b in blocks if b.get(k) is not None]
            assert r[i] == KB.tree(totals, KB.moments_combine), k
        one = p.fold_by_sparse_key(KB.class_moments_f64, a[:100])                 # one block
        assert same_bits(one, q.fold_by_sparse_key(KB.class_moments_f64, a[:100]))
        labels, vals = sparse_labels(300_000, "zipf", seed=19)
        check_label(p.starfold_by_sparse_key(KB.label_sum_u64, fiber_b200.Columns(labels, vals)), labels, vals)
        empty = p.fold_by_sparse_key(KB.class_moments_f64, a[:0])
        assert len(empty) == 0 and empty.keys.tolist() == []
    finally:
        for x in (p, q):
            x.terminate()
            x.join()


def test_two_workers_follow_the_block_rule():
    n_dev = ctypes.c_int(0)
    _abi.check(_abi.load().fbr_device_count(ctypes.byref(n_dev)))
    if n_dev.value < 2:
        pytest.skip("needs two GPUs")
    keys = np.random.default_rng(17).integers(0, RESERVED, 300, dtype=np.uint64)
    a = moments_inputs(100_000, keys, seed=17)
    a["label"][:3000] = 11                                  # a key of the first block only
    p = fiber_b200.Pool(2, devices=[0, 1])
    try:
        r = p.fold_by_sparse_key(KB.class_moments_f64, a)
        plan = _abi.Plan()
        cuts = []
        for w in range(2):
            _abi.check(_abi.load().fbr_plan_query(registry.spec("class_moments_f64").func_id, len(a), _abi.FBR_PLAN_FOLD, 0, 2, w,
                                                  132, ctypes.byref(plan)))
            cuts.append((plan.block_first, plan.block_first + plan.block_count))
        want, wkeys, counts = sparse_keyed_blocks(moments_results(a), KB.KEY_OF["class_moments_f64"], KB.moments_combine, cuts)
        assert r.tolist() == want and r.keys.tolist() == wkeys and r.counts.tolist() == counts
    finally:
        p.terminate()
        p.join()
