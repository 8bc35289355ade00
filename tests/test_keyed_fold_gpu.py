"""GPU: keyed folds (Pool.fold_by_key / starfold_by_key, FBR_FOLD_KEYS) of the bodies in tests/keyed_bodies.py -- 0, 1 and 2
radix passes, sizes around the claim unit and the sort tile and across several waves, key distributions, the identities
with Pool.fold, independence from ring size, shuffled arrival, the result ring and argument placement, error handling, bad
keys, device-resident results, fbr_fold_segments and the argument refusals.  Every record is compared bit for bit, floats
included, with the Python restatement, and every count with np.bincount."""
import ctypes

import numpy as np
import pytest

import fiber_b200
from fiber_b200 import _abi, registry

from . import keyed_bodies as KB

pytestmark = pytest.mark.gpu

SMALL_RING = 256 << 10
CENTROIDS = np.random.default_rng(5).standard_normal((64, 16)).astype(np.float32)


@pytest.fixture(scope="module")
def pool():
    p = fiber_b200.Pool(1, devices=[0], initializer=KB.set_centroids, initargs=(CENTROIDS,))
    yield p
    p.terminate()
    p.join()


@pytest.fixture(scope="module")
def small():
    p = fiber_b200.Pool(1, devices=[0], ring_bytes=SMALL_RING)
    yield p
    p.terminate()
    p.join()


def label_inputs(n, n_keys, dist, seed=0):
    rng = np.random.default_rng(seed)
    if dist == "uniform":
        labels = rng.integers(0, n_keys, n)
    elif dist == "equal":
        labels = np.full(n, n_keys - 1)
    elif dist == "distinct":
        labels = rng.permutation(n) % n_keys
    elif dist == "skewed":
        labels = np.minimum(rng.geometric(0.3, n) - 1, n_keys - 1)
    else:                                               # "sparse": most keys empty
        labels = rng.choice(np.arange(0, n_keys, max(1, n_keys // 5)), n)
    return labels.astype(np.uint32), rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)


def label_expected(labels, vals, n_keys):
    """The records and counts of label_sum_u64: an integer sum per key, so any order gives the same bits."""
    sums = np.zeros(n_keys, np.uint64)
    np.add.at(sums, labels, vals.astype(np.uint64))
    counts = np.bincount(labels, minlength=n_keys).astype(np.uint64)
    want = np.zeros(n_keys, KB.LABEL_RES)
    want["sum"], want["n"] = sums, counts.astype(np.uint32)
    want["key"] = np.where(counts > 0, np.arange(n_keys), 0)
    return want, counts


def same_bits(a, b):
    """Two keyed results hold the same record bytes and the same counts."""
    return np.asarray(a.array).tobytes() == np.asarray(b.array).tobytes() and np.array_equal(a.counts, b.counts)


def check_label(r, labels, vals, n_keys):
    want, counts = label_expected(labels, vals, n_keys)
    assert len(r) == n_keys
    np.testing.assert_array_equal(r.counts, counts)
    assert np.array_equal(np.asarray(r.array).view(np.uint8), want.view(np.uint8))


@pytest.mark.parametrize("n_keys", [1, 2, 255, 256, 257, 4096, 65536])
def test_label_sum_every_pass_count(pool, n_keys):
    for n in (1, 2, 4095, 4096, 4097, 70_001):
        labels, vals = label_inputs(n, n_keys, "uniform", seed=n + n_keys)
        check_label(pool.starfold_by_key(KB.label_sum_u64, fiber_b200.Columns(labels, vals), n_keys), labels, vals, n_keys)


@pytest.mark.parametrize("dist", ["equal", "distinct", "skewed", "sparse"])
def test_key_distributions(pool, dist):
    for n_keys, n in ((300, 50_000), (65536, 65536), (7, 3_000_000)):
        labels, vals = label_inputs(n, n_keys, dist, seed=3)
        check_label(pool.starfold_by_key(KB.label_sum_u64, fiber_b200.Columns(labels, vals), n_keys), labels, vals, n_keys)


def test_several_waves(small):
    labels, vals = label_inputs(400_000, 1000, "uniform", seed=4)
    before = small.stats()["dispatch_launches"]
    check_label(small.starfold_by_key(KB.label_sum_u64, fiber_b200.Columns(labels, vals), 1000), labels, vals, 1000)
    assert small.stats()["dispatch_launches"] - before >= 4


def moments_inputs(n, n_keys, seed):
    rng = np.random.default_rng(seed)
    a = np.zeros(n, KB.MOMENTS_ARG)
    a["x"] = rng.standard_normal(n) * 1e3
    a["label"] = rng.integers(0, n_keys, n)
    return a


def moments_results(a):
    return [KB.class_moments_f64(float(x), int(k)) for x, k in zip(a["x"], a["label"])]


def test_class_moments_bits(pool):
    for n, n_keys in ((1, 3), (513, 3), (20_000, 7), (20_000, 300)):
        a = moments_inputs(n, n_keys, seed=n + n_keys)
        r = pool.fold_by_key(KB.class_moments_f64, a, n_keys)
        want, counts = KB.keyed_tree(moments_results(a), KB.KEY_OF["class_moments_f64"], KB.moments_combine, KB.MOMENTS_ID, n_keys)
        assert r.tolist() == want and r.counts.tolist() == counts


def test_one_key_is_fold_and_each_key_is_fold_of_its_subsequence(pool):
    a = moments_inputs(30_000, 5, seed=8)
    one = a.copy()
    one["label"] = 0
    assert pool.fold_by_key(KB.class_moments_f64, one, 1).tolist() == [pool.fold(KB.class_moments_f64, one)]
    r = pool.fold_by_key(KB.class_moments_f64, a, 6)
    for k in range(6):
        sub = a[a["label"] == k]
        assert r[k] == pool.fold(KB.class_moments_f64, sub), k
    assert r[5] == KB.MOMENTS_ID and r.counts[5] == 0


def test_kmeans_step(pool):
    rng = np.random.default_rng(9)
    pts = rng.standard_normal((200_000, 16)).astype(np.float32)
    args = np.zeros(len(pts), KB.POINT)
    args["p"] = pts
    r = pool.fold_by_key(KB.kmeans_step_f32, args, 64)
    keys = KB.kmeans_keys(CENTROIDS, pts)
    np.testing.assert_array_equal(r.counts, np.bincount(keys, minlength=64))
    small = args[:3000]
    rs = [KB.kmeans_run(CENTROIDS, p) for p in small["p"]]
    want, counts = KB.keyed_tree(rs, KB.KEY_OF["kmeans_step_f32"], KB.kmeans_combine, KB.KMEANS_ID, 64)
    got = pool.fold_by_key(KB.kmeans_step_f32, small, 64)
    assert got.counts.tolist() == counts
    for k in range(64):
        g = got[k]
        assert np.array_equal(np.asarray(g[0], np.float32), np.asarray(want[k][0], np.float32)) and g[1:] == tuple(want[k][1:]), k


def test_items_and_group_bodies(pool):
    rng = np.random.default_rng(11)
    labels = rng.integers(0, 9, 1500).astype(np.uint32)
    strs = [bytes(rng.integers(0, 256, rng.integers(0, 300), dtype=np.uint8)) for _ in labels]
    r = pool.starfold_by_key(KB.label_hist_1k, list(zip(strs, labels.tolist())), 9)
    rs = [KB.label_hist_1k(s, int(k)) for k, s in zip(labels, strs)]
    want, counts = KB.keyed_tree(rs, KB.KEY_OF["label_hist_1k"], KB.hist_combine, KB.HIST_ID, 9)
    assert r.counts.tolist() == counts and [(list(x[0]), x[1]) for x in r.tolist()] == [(list(w[0]), w[1]) for w in want]

    w = np.zeros(700, KB.WIDE_ARG)
    w["label"] = rng.integers(0, 5, 700)
    w["seed"] = rng.integers(0, 1 << 32, 700, dtype=np.uint64)
    r = pool.fold_by_key(KB.wide_sum_16k, w, 6)
    np.testing.assert_array_equal(r.counts, np.bincount(w["label"], minlength=6))
    for k in range(6):
        sel = w[w["label"] == k]
        v = np.zeros(4092, np.uint64)
        for s in sel["seed"]:
            v += KB.wide_words(int(s))
        assert np.array_equal(np.asarray(r.array[k]["v"]), (v & np.uint64(KB.M32)).astype(np.uint32)), k
        assert r.array[k]["key"] == (k if len(sel) else 0)


def _raw_keyed(p, name, xs, n_keys, flags=0, dev_args=False):
    """A keyed fold through the C ABI (map flags the Pool API does not take): (record bytes, counts)."""
    spec = registry.spec(name)
    star = isinstance(xs, fiber_b200.Columns)
    enc = spec.encode_starmap(xs) if star else spec.encode_map(xs)
    eng, lib = p._engine, p._engine.lib
    d = _abi.MapDesc()
    d.func_id, d.flags, d.n_tasks, d.n_keys, d.shuffle_seed = spec.func_id, flags | _abi.FBR_FOLD_KEYS, enc.n, n_keys, 17
    d.flags |= _abi.FBR_STARMAP if star else _abi.FBR_MAP
    d.arg_stride = enc.arg_stride
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
        res = _abi.Result()
        _abi.check(lib.fbr_result_wait(eng.handle, seq.value, -1, ctypes.byref(res)))
        R = spec.result_bytes
        out = ctypes.string_at(res.data, n_keys * (R + 8))
        assert lib.fbr_result_fetch(eng.handle, seq.value, 0, 0, None) == _abi.FBR_EINVAL
        _abi.check(lib.fbr_result_release(eng.handle, seq.value))
    finally:
        if dptr.value:
            lib.fbr_device_free(eng.handle, 0, dptr)
    return out[:n_keys * R], np.frombuffer(out[n_keys * R:], np.uint64)


def test_independent_of_ring_arrival_and_placement(pool, small):
    a = moments_inputs(60_000, 300, seed=12)
    want = pool.fold_by_key(KB.class_moments_f64, a, 300)
    ref = (np.asarray(want.array).tobytes(), np.asarray(want.counts))
    assert same_bits(small.fold_by_key(KB.class_moments_f64, a, 300), want)
    for p, flags, dev in ((pool, _abi.FBR_SHUFFLE, False), (pool, _abi.FBR_VIA_RING, False), (small, _abi.FBR_SHUFFLE, False),
                          (pool, 0, True), (pool, _abi.FBR_RESULTS_ON_DEVICE, False)):
        recs, counts = _raw_keyed(p, "class_moments_f64", a, 300, flags, dev)
        assert recs == ref[0] and np.array_equal(counts, ref[1]), (flags, dev)


def test_results_on_device():
    a = moments_inputs(10_000, 40, seed=13)
    p = fiber_b200.Pool(1, devices=[0], results="device")
    q = fiber_b200.Pool(1, devices=[0])
    try:
        assert same_bits(p.fold_by_key(KB.class_moments_f64, a, 40), q.fold_by_key(KB.class_moments_f64, a, 40))
    finally:
        for x in (p, q):
            x.terminate()
            x.join()


def test_error_handling_gives_the_same_bits():
    xs = range(50_000)
    rs = [KB.fault_label_u64(i) for i in xs]
    want, counts = KB.keyed_tree(rs, KB.KEY_OF["fault_label_u64"], KB.label_combine, KB.LABEL_ID, 7)
    p = fiber_b200.Pool(1, devices=[0], error_handling=True)
    try:
        r = p.fold_by_key(KB.fault_label_u64, xs, 7)
        assert r.tolist() == want and r.counts.tolist() == counts
        assert p.stats()["units_redispatched"] > 0
    finally:
        p.terminate()
        p.join()


def test_bad_key_raises_for_the_lowest_task(pool):
    labels, vals = label_inputs(100_000, 10, "uniform", seed=14)
    labels[[70_000, 31_337, 99_999]] = [12, 10, 4000]
    with pytest.raises(ValueError, match=r"label_sum_u64: key\(\) of task 31337 is not below n_keys=10"):
        pool.starfold_by_key(KB.label_sum_u64, fiber_b200.Columns(labels, vals), 10)
    check_label(pool.starfold_by_key(KB.label_sum_u64, fiber_b200.Columns(labels, vals), 4001), labels, vals, 4001)


def test_empty_map(pool):
    r = pool.starfold_by_key(KB.class_moments_f64, [], 3)
    assert r.tolist() == [KB.MOMENTS_ID] * 3 and r.counts.tolist() == [0, 0, 0]


def test_refusals(pool, small):
    spec = registry.spec("label_sum_u64")
    labels, vals = label_inputs(100, 4, "uniform")
    with pytest.raises(_abi.EngineError, match="exceed ring_bytes"):
        small.starfold_by_key(KB.label_sum_u64, fiber_b200.Columns(labels, vals), 65536)
    for flags in (_abi.FBR_FOLD, _abi.FBR_SCAN, _abi.FBR_WANT_SUM, _abi.FBR_NO_ZERO_COPY):
        with pytest.raises(_abi.EngineError, match="FBR_FOLD_KEYS|keyed fold map"):
            _raw_keyed(pool, "label_sum_u64", fiber_b200.Columns(labels, vals), 4, flags)
    out = np.zeros(4 * spec.result_bytes, np.uint8)
    for flags, where in ((0, out.ctypes.data), (_abi.FBR_OUT_DEVICE, out.ctypes.data)):
        enc = spec.encode_starmap(fiber_b200.Columns(labels, vals))
        d = _abi.MapDesc()
        d.func_id, d.flags, d.n_tasks, d.n_keys = spec.func_id, flags | _abi.FBR_FOLD_KEYS | _abi.FBR_STARMAP, enc.n, 4
        d.arg_stride, d.args, d.out = enc.arg_stride, enc.args.ctypes.data, where
        rc = pool._engine.lib.fbr_map_submit(pool._engine.handle, ctypes.byref(d), ctypes.byref(ctypes.c_uint64()))
        assert rc == _abi.FBR_EINVAL and "owns its result records" in _abi.load().fbr_last_error().decode()
    for bad in (0, 65537):
        with pytest.raises(_abi.EngineError, match="n_keys"):
            _raw_keyed(pool, "label_sum_u64", fiber_b200.Columns(labels, vals), bad)
    with pytest.raises(_abi.EngineError, match="has no key"):
        d = _abi.MapDesc()
        d.func_id, d.flags, d.n_tasks, d.n_keys = registry.spec("sum_sq_idx_u64").func_id, _abi.FBR_FOLD_KEYS, 10, 2
        _abi.check(pool._engine.lib.fbr_map_submit(pool._engine.handle, ctypes.byref(d), ctypes.byref(ctypes.c_uint64())))
    assert spec.flags & _abi.FBR_BODY_KEYED


def test_fold_segments(pool):
    sizes = [0, 1, 0, 513, 2, 0, 70_000, 3, 0]
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint64)
    a = moments_inputs(int(offs[-1]), 1, seed=16)
    rs = moments_results(a)
    vals = np.zeros(len(rs), KB.MOMENTS_RES)
    vals[:] = rs
    out = np.zeros(len(sizes), KB.MOMENTS_RES)
    lib = pool._engine.lib
    _abi.check(lib.fbr_fold_segments(pool._engine.handle, registry.spec("class_moments_f64").func_id, vals.ctypes.data,
                                     offs.ctypes.data, len(sizes), out.ctypes.data))
    for k in range(len(sizes)):
        seg = rs[int(offs[k]):int(offs[k + 1])]
        want = KB.tree(seg, KB.moments_combine) if seg else KB.MOMENTS_ID
        assert tuple(out[k].tolist()) == tuple(want), k
    bad = offs.copy()
    bad[3] = 0
    assert lib.fbr_fold_segments(pool._engine.handle, registry.spec("class_moments_f64").func_id, vals.ctypes.data,
                                 bad.ctypes.data, len(sizes), out.ctypes.data) == _abi.FBR_EINVAL


def test_two_workers_follow_the_block_rule():
    n_dev = ctypes.c_int(0)
    _abi.check(_abi.load().fbr_device_count(ctypes.byref(n_dev)))
    if n_dev.value < 2:
        pytest.skip("needs two GPUs")
    a = moments_inputs(100_000, 9, seed=17)
    p = fiber_b200.Pool(2, devices=[0, 1])
    try:
        r = p.fold_by_key(KB.class_moments_f64, a, 10)
        plan = _abi.Plan()
        cuts = []
        for w in range(2):
            _abi.check(_abi.load().fbr_plan_query(registry.spec("class_moments_f64").func_id, len(a), _abi.FBR_PLAN_FOLD, 0, 2, w,
                                                  132, ctypes.byref(plan)))
            cuts.append((plan.block_first, plan.block_first + plan.block_count))
        want, counts = KB.keyed_blocks(moments_results(a), KB.KEY_OF["class_moments_f64"], KB.moments_combine, KB.MOMENTS_ID, 10, cuts)
        assert r.tolist() == want and r.counts.tolist() == counts
    finally:
        p.terminate()
        p.join()


def test_process_isolation_equals_thread_isolation_on_the_same_block_cut():
    """A process-isolated pool cuts the map into blocks of its own: each block's keyed fold (one worker, its own x_k) is what
    a thread pool gives for that block, and record k folds the non-empty block totals in block order."""
    a = moments_inputs(150_001, 9, seed=18)
    p = fiber_b200.Pool(1, isolation="process", error_handling=True)
    q = fiber_b200.Pool(1, devices=[0])
    try:
        r = p.fold_by_key(KB.class_moments_f64, a, 10)
        cuts = p._proc.fold_blocks(len(a))
        assert len(cuts) > 1
        want, counts = KB.keyed_blocks(moments_results(a), KB.KEY_OF["class_moments_f64"], KB.moments_combine, KB.MOMENTS_ID, 10,
                                       cuts)
        assert r.tolist() == want and r.counts.tolist() == counts
        # the blocks themselves: the thread pool's keyed fold of each block is the process pool's block total
        blocks = [q.fold_by_key(KB.class_moments_f64, a[lo:hi], 10) for lo, hi in cuts]
        for k in range(10):
            totals = [b[k] for b in blocks if b.counts[k]]
            assert r[k] == (KB.tree(totals, KB.moments_combine) if totals else KB.MOMENTS_ID), k
        one = p.fold_by_key(KB.class_moments_f64, a[:100], 10)                 # one block
        assert same_bits(one, q.fold_by_key(KB.class_moments_f64, a[:100], 10))
        labels, vals = label_inputs(300_000, 4096, "uniform", seed=19)
        check_label(p.starfold_by_key(KB.label_sum_u64, fiber_b200.Columns(labels, vals), 4096), labels, vals, 4096)
        empty = p.fold_by_key(KB.class_moments_f64, a[:0], 3)
        assert empty.tolist() == [KB.MOMENTS_ID] * 3 and empty.counts.tolist() == [0, 0, 0]
    finally:
        for x in (p, q):
            x.terminate()
            x.join()
