"""GPU: emit record bodies -- every task returns a variable-length array.  The count pass, scan_counts_kernel and the emit
pass run for tokens of byte strings (one thread, items), prime factors over range() (kIndexArg), positions above a
threshold on a warp (push_if), radius neighbours in a broadcast block and ASCII uppercase through a count() hook.  Every
map form, empty results, skewed lengths, scan sizes across its tiles, the result ring, many waves, results="device",
resilient re-dispatch (also of an attempt that faults before pushing anything), the FBR_TASK_EMIT error, a count pass
that fails, device-resident inputs, values streamed through small staging halves and the unit too large for one,
process isolation and the tokenize -> items-body chain.  Every value is compared with the
restatements in tests/emit_bodies.py."""
import ctypes

import numpy as np
import pytest

import fiber_b200
from fiber_b200 import _abi, registry

from . import emit_bodies as EB
from . import ragged_bodies as RB

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pool():
    p = fiber_b200.Pool(1, devices=[0])
    yield p
    p.terminate()
    p.join()


def _unit(name, n, chunksize):
    p = _abi.Plan()
    _abi.check(_abi.load().fbr_plan_query(registry.spec(name).func_id, n, chunksize, 0, 1, 0, 132, ctypes.byref(p)))
    return p.unit_tasks


DOCS = EB.documents(20_000, seed=3, empty_every=7)
DOCS_REF = [EB.tokens_u32(d) for d in DOCS]


@pytest.mark.parametrize("chunksize", [1, 7, 32])
def test_tokens_sizes(pool, chunksize):
    unit = _unit("tokens_u32", len(DOCS), chunksize)
    sizes = sorted({n for n in (1, 7, unit - 1, unit, unit + 1, 3 * unit + 5, len(DOCS)) if 0 < n <= len(DOCS)})
    for n in sizes:
        r = pool.map(EB.tokens_u32, DOCS[:n], chunksize=chunksize)
        assert len(r) == n and r == DOCS_REF[:n], n


def test_empty_results(pool):
    blank = [b"", b" ", b"\t\n", b"   \r\n"] * 1000
    r = pool.map(EB.tokens_u32, blank)
    assert r == [[]] * len(blank)
    assert len(r.ragged.values) == 0
    assert pool.map(EB.tokens_u32, []) == []


def test_skewed_lengths(pool):
    # a few documents carry most of the tokens: the units holding them emit more than a 32 KB value stage and store their
    # values to global memory directly, every other unit stages its values in shared memory
    docs = [b"w " * 20_000 if i % 997 == 0 else b"a b" for i in range(5000)]
    r = pool.map(EB.tokens_u32, docs)
    assert r == [EB.tokens_u32(d) for d in docs]


@pytest.mark.parametrize("n", [1, 2047, 2048, 2049, 3 * 2048 + 1, 300_000])
def test_prime_factors_scan_sizes(pool, n):
    # range() maps: the scan's tiles hold 2048 counts
    r = pool.map(EB.prime_factors_i64, range(2, 2 + n))
    assert len(r) == n
    want = [EB.prime_factors(k) for k in range(2, 2 + n)]
    assert r == want
    assert np.array_equal(r.ragged.values, np.array([v for f in want for v in f], np.int64))


def test_map_forms(pool):
    docs = DOCS[:500]
    assert pool.starmap(EB.tokens_u32, [(d,) for d in docs]) == DOCS_REF[:500]
    assert pool.apply_async(EB.tokens_u32, (docs[3],)).get() == DOCS_REF[3]
    assert pool.apply(EB.prime_factors_i64, (360,)) == [2, 2, 2, 3, 3, 5]
    assert list(pool.imap(EB.tokens_u32, DOCS)) == DOCS_REF
    assert list(pool.imap_unordered(EB.prime_factors_i64, range(2, 5000))) == [EB.prime_factors(k) for k in range(2, 5000)]


def test_above_mask_push_if(pool):
    vals, offs = RB.lognormal_rows(20_000, seed=4, mean_len=48.0)
    rows = [vals[offs[i]:offs[i + 1]] for i in range(len(offs) - 1)]
    ts = np.random.default_rng(5).standard_normal(len(rows))
    for chunksize in (1, 32):
        r = pool.starmap(EB.above_mask_f64, list(zip(rows, ts.tolist())), chunksize=chunksize)
        assert r == [np.flatnonzero(row > t).tolist() for row, t in zip(rows, ts)]


def test_radius_neighbors_broadcast(pool):
    rng = np.random.default_rng(6)
    pts = np.zeros(3000, EB.POINT)
    pts["x"], pts["y"] = rng.random(3000, dtype=np.float32), rng.random(3000, dtype=np.float32)
    q = np.zeros(2000, EB.QUERY)
    q["x"], q["y"] = rng.random(2000, dtype=np.float32), rng.random(2000, dtype=np.float32)
    q["r"] = rng.random(2000, dtype=np.float32) * np.float32(0.1)
    want = EB.radius_neighbors_np(pts, q)
    # 3000 points (24 KB) are read from global memory, 1000 (8 KB) from shared memory
    for m in (3000, 1000):
        r = pool.starmap(EB.radius_neighbors_f32, [(pts[:m], float(a["x"]), float(a["y"]), float(a["r"])) for a in q])
        assert r == (want if m == 3000 else EB.radius_neighbors_np(pts[:m], q))


def test_upper_ascii_count_hook(pool):
    rng = np.random.default_rng(7)
    words = ["".join(chr(c) for c in rng.integers(32, 127, int(rng.integers(0, 60)))) for _ in range(5000)]
    r = pool.map(EB.upper_ascii_u8, words)
    assert r == [w.upper() for w in words]
    assert r[1] == words[1].upper()


def test_via_ring_and_shuffle(pool):
    spec = registry.spec("tokens_u32")
    for flags in (_abi.FBR_VIA_RING, _abi.FBR_SHUFFLE):
        r = pool._submit(EB.tokens_u32, spec.encode_map(DOCS), _abi.FBR_MAP, 7, extra_flags=flags).get()
        assert r == DOCS_REF


def test_many_waves():
    p = fiber_b200.Pool(1, devices=[0], ring_bytes=1 << 20)
    try:
        assert p.map(EB.tokens_u32, DOCS) == DOCS_REF
        assert p.map(EB.prime_factors_i64, range(2, 200_000)) == [EB.prime_factors(k) for k in range(2, 200_000)]
    finally:
        p.terminate()
        p.join()


def test_results_on_device():
    p = fiber_b200.Pool(1, devices=[0], results="device")
    try:
        r = p.map(EB.tokens_u32, DOCS)
        assert r.on_device
        assert r[0] == DOCS_REF[0] and r[-1] == DOCS_REF[-1] and r[100:250] == DOCS_REF[100:250]
        assert r == DOCS_REF
        assert p.map(EB.tokens_u32, [b" "] * 10) == [[]] * 10
    finally:
        p.terminate()
        p.join()


def test_resilient_redispatch():
    p = fiber_b200.Pool(1, devices=[0], error_handling=True)
    try:
        docs = [(b"!" + d) if i % 11 == 0 else d for i, d in enumerate(DOCS)]
        want = [EB.tokens_u32(d) for d in docs]
        r = p.map(EB.fault_tokens_u32, docs, chunksize=7)
        assert r == want
        assert p.stats()["units_redispatched"] > 0
        # a faulting attempt that pushes nothing: its count mismatch goes with the discarded attempt
        assert p.map(EB.early_fault_tokens_u32, docs, chunksize=7) == want
    finally:
        p.terminate()
        p.join()


def test_emit_count_mismatch(pool):
    docs = [b"x" * (i % 9) for i in range(1, 4000)]
    lowest = next(i for i, d in enumerate(docs) if len(d) % 5 == 3)
    with pytest.raises(RuntimeError, match=r"bad_count_u32: task %d emitted another number of values than the 4 its count "
                                           r"pass gave" % lowest):
        pool.map(EB.bad_count_u32, docs)
    ok = [d for d in docs if len(d) % 5 != 3]
    assert pool.map(EB.bad_count_u32, ok) == [list(d) for d in ok]


def test_chain_tokenize_then_items_body(pool):
    r = pool.map(EB.tokens_u32, DOCS)
    s = pool.map(EB.token_sum_u32, r.ragged)
    assert s == [sum(t) for t in DOCS_REF]


def test_two_workers():
    n = ctypes.c_int(0)
    _abi.check(_abi.load().fbr_device_count(ctypes.byref(n)))
    if n.value < 2:
        pytest.skip("needs two GPUs")
    p = fiber_b200.Pool(2)
    try:
        assert p.map(EB.tokens_u32, DOCS) == DOCS_REF
        assert p.map(EB.prime_factors_i64, range(2, 100_000)) == [EB.prime_factors(k) for k in range(2, 100_000)]
    finally:
        p.terminate()
        p.join()


def _device_items(pool, values, offsets):
    """values and offsets copied to device memory of worker 0 (engine allocations, freed by the caller)."""
    eng = pool._engine
    ptrs = []
    for a in (values, offsets):
        p = ctypes.c_void_p()
        _abi.check(eng.lib.fbr_device_alloc(eng.handle, 0, max(16, a.nbytes), ctypes.byref(p)))
        if a.nbytes:
            _abi.check(eng.lib.fbr_memcpy_h2d(eng.handle, 0, p, a.ctypes.data, a.nbytes))
        ptrs.append(p)
    return ptrs


def _submit_device(pool, values, offsets, flags, n):
    eng = pool._engine
    dv, do = _device_items(pool, values, offsets)
    d = _abi.MapDesc()
    d.func_id, d.flags, d.n_tasks = registry.spec("tokens_u32").func_id, _abi.FBR_ARGS_DEVICE | flags, n
    it = _abi.ItemsDesc()
    it.items, it.offsets, it.n_items, it.item_bytes = dv.value, do.value, len(values), 1
    seq = ctypes.c_uint64()
    _abi.check(eng.lib.fbr_map_submit_items(eng.handle, ctypes.byref(d), ctypes.byref(it), ctypes.byref(seq)))
    return seq.value, (dv, do)


def test_device_resident_inputs(pool):
    eng = pool._engine
    vals = np.frombuffer(b"".join(DOCS), np.uint8)
    offs = np.zeros(len(DOCS) + 1, np.uint64)
    np.cumsum([len(d) for d in DOCS], out=offs[1:])
    want_vals = np.array([v for t in DOCS_REF for v in t], np.uint32)
    want_ends = np.cumsum([len(t) for t in DOCS_REF]).astype(np.uint64)
    for flags in (0, _abi.FBR_RESULTS_ON_DEVICE):
        seq, bufs = _submit_device(pool, vals, offs, flags, len(DOCS))
        try:
            res = _abi.Result()
            _abi.check(eng.lib.fbr_result_wait(eng.handle, seq, -1, ctypes.byref(res)))
            assert res.result_kind == _abi.FBR_RES_OFFSETS
            ends, got = np.zeros(len(DOCS), np.uint64), np.zeros(len(want_vals), np.uint32)
            if flags:
                _abi.check(eng.lib.fbr_result_fetch(eng.handle, seq, 0, len(DOCS), ends.ctypes.data))
                _abi.check(eng.lib.fbr_result_fetch_values(eng.handle, seq, 0, len(got), got.ctypes.data))
            else:
                ctypes.memmove(ends.ctypes.data, res.data, ends.nbytes)
                vp, nv = ctypes.c_void_p(), ctypes.c_uint64()
                _abi.check(eng.lib.fbr_result_values(eng.handle, seq, ctypes.byref(vp), ctypes.byref(nv)))
                assert nv.value == len(want_vals)
                ctypes.memmove(got.ctypes.data, vp.value, got.nbytes)
            assert np.array_equal(ends, want_ends) and np.array_equal(got, want_vals)
        finally:
            eng.lib.fbr_result_release(eng.handle, seq)
            for b in bufs:
                eng.lib.fbr_device_free(eng.handle, 0, b)


def test_failed_count_pass(pool):
    # device-resident offsets that decrease: the count pass reports TASK_BADARG, and the map is born finished with it
    eng = pool._engine
    vals = np.frombuffer(b"a b c d e f", np.uint8)
    offs = np.array([0, 3, 7, 5, 11], np.uint64)
    seq, bufs = _submit_device(pool, vals, offs, 0, 4)
    try:
        done = ctypes.c_uint64()
        _abi.check(eng.lib.fbr_result_poll(eng.handle, seq, ctypes.byref(done)))
        assert done.value == 4
        res = _abi.Result()
        assert eng.lib.fbr_result_wait(eng.handle, seq, -1, ctypes.byref(res)) == _abi.FBR_ETASK
        assert (res.err_code, res.err_task) == (_abi.FBR_TASK_BADARG, 2)
    finally:
        eng.lib.fbr_result_release(eng.handle, seq)
        for b in bufs:
            eng.lib.fbr_device_free(eng.handle, 0, b)


def test_emit_waves_and_the_over_large_unit():
    p = fiber_b200.Pool(1, devices=[0], ring_bytes=1 << 20)
    try:
        # 12 MB of 1-byte values: every wave's values fit a 1 MiB staging half, so the map runs in many waves
        rng = np.random.default_rng(8)
        words = ["".join(chr(c) for c in rng.integers(32, 127, 1200)) for _ in range(10_000)]
        res = p.map_async(EB.upper_ascii_u8, words)
        assert res.get() == [w.upper() for w in words]
        assert res.n_waves >= 12
        assert list(p.imap(EB.upper_ascii_u8, words)) == [w.upper() for w in words]
        # one task whose values alone (1.2 MB of token hashes from 600 KB of text) exceed a staging half
        with pytest.raises(_abi.EngineError, match="ring_bytes"):
            p.map(EB.tokens_u32, [b"a " * 300_000])
        assert p.map(EB.tokens_u32, DOCS[:100]) == DOCS_REF[:100]      # the pool keeps serving
    finally:
        p.terminate()
        p.join()


def test_process_isolation():
    p = fiber_b200.Pool(2, isolation="process")
    try:
        assert p.map(EB.tokens_u32, DOCS, chunksize=7) == DOCS_REF
        assert p.starmap(EB.above_mask_f64, [(np.array([0.5, -1.0, 2.0]), 0.0), (np.array([]), 0.0)]) == [[0, 2], []]
        assert p.map(EB.prime_factors_i64, range(2, 3000)) == [EB.prime_factors(k) for k in range(2, 3000)]
        assert p.apply(EB.upper_ascii_u8, ("abc",)) == "ABC"
        assert p.map(EB.upper_ascii_u8, []) == []
    finally:
        p.terminate()
        p.join()
