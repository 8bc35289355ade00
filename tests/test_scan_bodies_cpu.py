"""CPU: the prefix order of FBR_SCAN (Pool.accumulate) -- the pieces form against tree() of every prefix, its multi-block
form, the scan kernels' level sweep restated -- the registration rules of FBR_BODY_SCAN, the header constants, and the
TypeError of bodies that cannot accumulate."""
import os
import re

import pytest

import fiber_b200
from fiber_b200 import _abi, registry

from . import fold_bodies as FB
from . import scan_bodies as SB

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def pair(a, b):
    """The symbolic combine: the result records its own bracketing."""
    return (a, b)


def test_pieces_form_equals_tree_of_every_prefix():
    xs = list(range(5000))
    got = SB.prefix_folds(xs, pair)
    for i in range(len(xs)):
        assert got[i] == FB.tree(xs[:i + 1], pair), i
    assert got[0] == 0                                   # the first record itself, no identity


def _kernel_sweep(xs, combine):
    """scan_level_kernel and scan_wrap_kernel restated: levels 1 .. from level 0, an odd i starts at level 1's node i >> 1."""
    n = len(xs)
    lv = [list(xs)]
    for k in range(1, max(1, n.bit_length())):
        prev = lv[-1]
        lv.append([combine(prev[2 * j], prev[2 * j + 1]) for j in range(n >> k)])
    out = []
    for i in range(n):
        bits = i
        acc = xs[i]
        if bits & 1:
            acc, bits = lv[1][i >> 1], bits & ~1
        k = 1
        while bits:
            if (bits >> k) & 1:
                acc = combine(lv[k][(i >> k) - 1], acc)
                bits &= ~(1 << k)
            k += 1
        out.append(acc)
    return out


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 7, 8, 31, 64, 100, 255, 256, 257, 1023, 1024, 1025, 3000])
def test_kernel_sweep_equals_the_definition(n):
    xs = list(range(n))
    want = SB.tree_prefixes(xs, pair) if n <= 1100 else SB.prefix_folds(xs, pair)
    assert _kernel_sweep(xs, pair) == want


@pytest.mark.parametrize("sizes", [[5], [4, 4], [3, 5, 1], [8, 8, 8, 3], [1, 1, 1, 1, 1, 1, 1], [16, 7, 9, 2, 11]])
def test_block_form(sizes):
    xs = list(range(sum(sizes)))
    bounds, lo = [], 0
    for s in sizes:
        bounds.append((lo, lo + s))
        lo += s
    got = SB.block_prefix_folds(xs, bounds, pair)
    for b, (lo, hi) in enumerate(bounds):
        totals = [FB.tree(xs[a:z], pair) for a, z in bounds[:b]]
        for i in range(lo, hi):
            assert got[i] == FB.tree(totals + [FB.tree(xs[lo:i + 1], pair)], pair), (sizes, i)
    assert got[-1] == FB.tree([FB.tree(xs[a:z], pair) for a, z in bounds], pair)


def test_header_constants_match_abi():
    h = open(os.path.join(ROOT, "include", "fiber_b200.h")).read()
    for name in ("FBR_BODY_SCAN", "FBR_SCAN"):
        m = re.search(r"#define %s (0x[0-9a-fA-F]+)u" % name, h)
        assert m and int(m.group(1), 16) == getattr(_abi, name), name
    assert _abi.FBR_BODY_MODULE_ABI == 4
    assert "fbr_scan_values" in _abi.SYMBOLS


def test_scan_flags_of_fold_bodies():
    for name in list(FB.RESTATED) + ["affine_f64", "mix4k_u32"]:
        spec = registry.spec(name)
        assert spec.flags & _abi.FBR_BODY_SCAN and spec.flags & _abi.FBR_BODY_FOLD, name
    for name in ("square_i64",):
        assert not registry.spec(name).flags & _abi.FBR_BODY_SCAN


def test_non_fold_bodies_raise_type_error():
    __import__("tests.record_bodies")
    from tests import record_bodies
    p = fiber_b200.Pool.__new__(fiber_b200.Pool)
    for f in (record_bodies.polar_f64,):
        with pytest.raises(TypeError, match="cannot fold"):
            p._fold_spec(f)


# ---- registration of hand-written descriptors ---------------------------------------------------------------------------
def _register(entry):
    import ctypes
    fid = ctypes.c_int(-1)
    rc = _abi.load().fbr_register_body(entry.encode(), SB.BAD_MODULE.encode(), entry.encode(), ctypes.byref(fid))
    return rc, fid.value, _abi.load().fbr_last_error().decode()


def _flags(fid):
    import ctypes
    info = _abi.BodyInfo()
    _abi.check(_abi.load().fbr_body_info(fid, ctypes.byref(info)))
    return info.flags


@pytest.mark.parametrize("entry,why", [
    ("bad_scan_no_fold", "FBR_BODY_SCAN needs FBR_BODY_FOLD"),
    ("bad_scan_no_entry", "sets FBR_BODY_SCAN but its descriptor lacks the scan entry"),
])
def test_registration_rejects_bad_scan_descriptors(entry, why):
    rc, _, msg = _register(entry)
    assert rc == _abi.FBR_EINVAL and why in msg, msg


def test_registration_accepts_scan_and_fold_only_descriptors():
    rc, fid, msg = _register("ok_scan")
    assert rc == _abi.FBR_OK, msg
    assert _flags(fid) & (_abi.FBR_BODY_FOLD | _abi.FBR_BODY_SCAN) == _abi.FBR_BODY_FOLD | _abi.FBR_BODY_SCAN
    rc, fid, msg = _register("ok_fold_without_scan")
    assert rc == _abi.FBR_OK, msg
    assert _flags(fid) & _abi.FBR_BODY_FOLD and not _flags(fid) & _abi.FBR_BODY_SCAN


# ---- the process-pool side of accumulate maps, with a stand-in worker (tests/_fake_scan_worker.py) -------------------------
class _ScanSpec:
    """What the process-pool master needs of a scan body (name, record size, flags, result decoding)."""

    def __init__(self, name):
        self.name, self.result_bytes = name, 8
        self.flags = _abi.FBR_BODY_RECORD | _abi.FBR_BODY_FOLD | _abi.FBR_BODY_SCAN

    def result_dtype(self):
        import numpy as np
        return np.dtype(np.uint64), ()

    def unpack_result(self, raw):
        return int.from_bytes(raw, "little")


def _pool(n, **kw):
    from fiber_b200.procpool import ProcessPool
    from ._fake_scan_worker import fake_scan_worker_main
    return ProcessPool(n, devices=list(range(n)), results="bytes", worker_main=fake_scan_worker_main, **kw)


def _ints(res):
    import numpy as np
    return [int(v) for v in np.asarray(res).tolist()]


def _want(pool, xs):
    from ._fake_fold_worker import combine
    return SB.block_prefix_folds(xs, [(lo, hi) for lo, hi in pool.fold_blocks(len(xs)) if hi > lo], combine)


def test_process_pool_accumulates_in_block_order():
    from fiber_b200.procpool import BLOCK_ALIGN
    pool = _pool(3, block_tasks=BLOCK_ALIGN)
    try:
        for n in (1, BLOCK_ALIGN, 7 * BLOCK_ALIGN + 123):
            xs = list(range(60000, 60000 + n))
            got = pool.submit_accumulate(_ScanSpec("scan_u64"), "map", range(60000, 60000 + n)).get(120)
            assert _ints(got) == _want(pool, xs)
        xs = list(range(60000, 60000 + 5 * BLOCK_ALIGN))
        got = pool.submit_accumulate(_ScanSpec("scan_u64"), "starmap", xs).get(120)
        assert _ints(got) == _want(pool, xs)
        assert len(pool.submit_accumulate(_ScanSpec("scan_u64"), "map", range(0)).get(10)) == 0
    finally:
        pool.terminate()
        pool.join()


def test_process_pool_resends_a_dead_workers_block_and_wrap(tmp_path, monkeypatch):
    from fiber_b200.procpool import BLOCK_ALIGN
    monkeypatch.setenv("FBR_TEST_SCAN_MARK", str(tmp_path / "died"))
    pool = _pool(2, block_tasks=BLOCK_ALIGN)
    try:
        n = 6 * BLOCK_ALIGN                      # the block holding 0xDEAD kills its worker on the first attempt
        got = pool.submit_accumulate(_ScanSpec("scan_u64"), "map", range(n)).get(120)
        assert _ints(got) == _want(pool, list(range(n)))
        assert pool.stats["workers_lost"] == 1 and pool.stats["blocks_redispatched"] == 1
        # a worker that dies after wrapping block 1: the rest of the wrap goes to another worker, block 1 is not wrapped twice
        xs = list(range(60000, 60000 + n))
        got = pool.submit_accumulate(_ScanSpec("scan_dies_once"), "map", range(60000, 60000 + n)).get(120)
        assert _ints(got) == _want(pool, xs)
        assert pool.stats["workers_lost"] == 2 and os.path.exists(tmp_path / "died")
    finally:
        pool.terminate()
        pool.join()


def test_process_pool_accumulates_after_close():
    from fiber_b200.procpool import BLOCK_ALIGN
    pool = _pool(2, block_tasks=BLOCK_ALIGN)
    try:
        xs = list(range(60000, 60000 + 5 * BLOCK_ALIGN + 17))
        r1 = pool.submit_accumulate(_ScanSpec("scan_u64"), "map", range(60000, 60000 + len(xs)))
        r2 = pool.submit_accumulate(_ScanSpec("scan_u64"), "map", xs[:3 * BLOCK_ALIGN])
        pool.close()
        pool.join(120)
        assert _ints(r1.get(1)) == _want(pool, xs)
        assert _ints(r2.get(1)) == _want(pool, xs[:3 * BLOCK_ALIGN])
    finally:
        pool.terminate()
        pool.join()


def test_process_pool_wrap_deaths_are_bounded():
    from fiber_b200.procpool import BLOCK_ALIGN, MAX_ATTEMPTS, WorkerDied
    xs = range(60000, 60000 + 2 * BLOCK_ALIGN)
    pool = _pool(2, block_tasks=BLOCK_ALIGN)
    try:
        with pytest.raises(WorkerDied, match="killed its worker %d times" % MAX_ATTEMPTS):
            pool.submit_accumulate(_ScanSpec("scan_always_dies"), "map", xs).get(120)
        got = pool.submit_accumulate(_ScanSpec("scan_u64"), "map", xs).get(120)    # the pool keeps serving
        assert _ints(got) == _want(pool, list(xs))
    finally:
        pool.terminate()
        pool.join()
    pool = _pool(2, block_tasks=BLOCK_ALIGN, redispatch=False)
    try:
        with pytest.raises(WorkerDied, match="without error_handling"):
            pool.submit_accumulate(_ScanSpec("scan_always_dies"), "map", xs).get(120)
    finally:
        pool.terminate()
        pool.join()
