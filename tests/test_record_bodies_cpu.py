"""CPU: record bodies (FBR_EXPORT_RECORD_BODY) -- registration rules, the dtype-driven encoders and decoders, and the
claim-unit plan that keeps both sides of every unit 16 B aligned.  No device is needed for any of it."""
import ctypes

import numpy as np
import pytest

import fiber_b200
from fiber_b200 import _abi, registry
from fiber_b200.pool import ResultArray

from . import layout_bodies as LB
from . import record_bodies as RB


def _register(name, entry=None):
    fid = ctypes.c_int(-1)
    rc = _abi.load().fbr_register_body(name.encode(), RB.BAD_MODULE.encode(), (entry or name).encode(), ctypes.byref(fid))
    return rc, _abi.load().fbr_last_error().decode()


def test_registration_accepts_the_test_bodies():
    want = {"polar_f64": (16, 16), "fault_polar_f64": (16, 16), "mix_i32x3": (12, 12), "row_stats_u32": (1024, 24),
            "splitmix_pair": (8, 16), "scale5_f64": (40, 40)}
    for name, (a, r) in want.items():
        s = registry.spec(name)
        assert isinstance(s, registry._Record) and (s.arg_bytes, s.result_bytes) == (a, r)
        assert s.flags & _abi.FBR_BODY_RECORD and s.result_kind == _abi.FBR_RES_BYTES
        assert not s.flags & _abi.FBR_BODY_SUMMABLE
    assert registry.spec("splitmix_pair").flags & _abi.FBR_BODY_INDEX_ARG
    mod = registry.module_of("polar_f64")
    assert mod[2] == RB.POLAR_ARG and mod[4] == RB.POLAR_RES and mod[3] is None


def test_registration_rejects_bad_layouts():
    for name, why in (("bad_arg6", "multiples of 4"), ("bad_res6", "multiples of 4"), ("bad_summable", "SUMMABLE"), ("bad_shared", "NEEDS_SHARED"),
                      ("bad_oversize", "at most 4096"), ("bad_twin", "no bit-packed twin")):
        rc, msg = _register(name)
        assert rc == _abi.FBR_EINVAL and why in msg, (name, msg)
    assert _register("ok_f32")[0] == _abi.FBR_OK
    # the dtypes must describe the module's records
    with pytest.raises(ValueError, match="argument dtype"):
        registry.register_module("ok_f32", RB.BAD_MODULE, "ok_f32", args="<f8", result="<f4")
    with pytest.raises(ValueError, match="result dtype"):
        registry.register_module("ok_f32", RB.BAD_MODULE, "ok_f32", args="<f4", result=[("a", "<f4"), ("b", "<f4")])
    with pytest.raises(TypeError, match="big-endian"):
        registry.register_module("ok_f32", RB.BAD_MODULE, "ok_f32", args=">f4", result="<f4")
    with pytest.raises(TypeError, match="Python objects"):
        registry.register_module("ok_f32", RB.BAD_MODULE, "ok_f32", args="<f4", result=[("o", "O")])
    with pytest.raises(ValueError, match="result="):
        registry.register_module("ok_f32", RB.BAD_MODULE, "ok_f32", args="<f4")
    s = registry.register_module("ok_f32", RB.BAD_MODULE, "ok_f32", args=[("x", "<f4")], result="<f4")
    assert s.params == ("x",) and s.result_dtype() == (np.dtype("<f4"), ())
    # registered again: the same layouts return the same spec; other layouts of the same size are refused, and the
    # module record worker processes read keeps the first registration
    assert registry.register_module("ok_f32", RB.BAD_MODULE, "ok_f32", args=[("x", "<f4")], result="<f4") is s
    with pytest.raises(ValueError, match="registered already"):
        registry.register_module("ok_f32", RB.BAD_MODULE, "ok_f32", args=[("y", "<f4")], result="<i4")
    assert registry.module_of("ok_f32")[2] == np.dtype([("x", "<f4")]) and registry.module_of("ok_f32")[4] == np.dtype("<f4")
    with pytest.raises(ValueError, match="registered already"):
        fiber_b200.device_body("polar_f64", source=RB.POLAR_SRC, entry="polar_entry", args=RB.POLAR_ARG,
                               result=[("a", "<f8"), ("b", "<f8")])
    assert registry.module_of("polar_f64")[4] == RB.POLAR_RES
    # a thread body keeps its string layouts and takes no result dtype
    from . import device_bodies as D
    with pytest.raises(ValueError, match="not a record body"):
        registry.register_module("collatz_steps", *registry.module_of("collatz_steps")[:2], result="<i8")
    assert registry.spec("collatz_steps").encode_map([3, 4]).args.tolist() == [3, 4] and D.collatz_steps(3) == 7


def test_plan_keeps_every_unit_16_byte_aligned():
    lib = _abi.load()
    for name in ("polar_f64", "mix_i32x3", "row_stats_u32", "splitmix_pair", "scale5_f64") + tuple(LB.BY_NAME):
        s = registry.spec(name)
        for n in (1, 7, 1000, 10 ** 6, 10 ** 8):
            for cs in (1, 3, 7, 32, 100, 5000):
                p = _abi.Plan()
                assert lib.fbr_plan_query(s.func_id, n, cs, 0, 1, 0, 132, ctypes.byref(p)) == 0
                assert p.unit_tasks * s.result_bytes % 16 == 0 and p.unit_tasks * s.arg_bytes % 16 == 0, (name, n, cs)
                assert p.slot_stride == p.unit_tasks * s.result_bytes and p.unit_tasks % LB.align_tasks(s.arg_bytes, s.result_bytes) == 0
                info = _abi.BodyInfo()
                assert lib.fbr_body_info(s.func_id, ctypes.byref(info)) == 0 and p.unit_tasks <= info.unit_tasks


def _gather_route(slot_stride, unit, R, resilient):
    """The gather kernel the wave planner picks for a map's full units (engine.cu, pick_gather):
    gather_bulk_kernel for 16 KB multiples (not on resilient maps), gather_rows_kernel for 4 KB multiples, else
    gather_ordered_kernel (flat)."""
    rows = unit * R == slot_stride and slot_stride % 4096 == 0
    if rows and not resilient and slot_stride % 16384 == 0:
        return "bulk"
    return "rows" if rows else "flat"


# (A, R, G, kAlign, kUnit, gather route of a full unit at the default chunksize) of the fixed-record layouts
LAYOUT_TABLE = {
    "lay_a4_r4": (4, 4, 1, 4, 1024, "rows"), "lay_a4_r4096": (4, 4096, 1, 4, 8, "bulk"),
    "lay_a4092_r4": (4092, 4, 1, 4, 8, "flat"), "lay_a8_r24": (8, 24, 1, 2, 1024, "rows"),
    "lay_a24_r8": (24, 8, 1, 2, 1024, "rows"), "lay_a12_r4096": (12, 4096, 1, 4, 8, "bulk"),
    "lay_a4096_r12": (4096, 12, 1, 4, 8, "flat"), "lay_a2052_r2052": (2052, 2052, 1, 4, 8, "flat"),
    "lay_a20_r20": (20, 20, 1, 4, 1024, "rows"), "lay_i8_r4096": (8, 4096, 1, 2, 8, "bulk"),
    "lay_i8_r12": (8, 12, 1, 4, 1024, "rows"), "lay_a8_r16384_g2": (8, 16384, 2, 2, 2, "bulk"),
    "lay_a16384_r8_g2": (16384, 8, 2, 2, 2, "flat"), "lay_a4_r8188_g4": (4, 8188, 4, 4, 4, "flat"),
    "lay_a8188_r4_g4": (8188, 4, 4, 4, 4, "flat"), "lay_a32768_r32768_g32": (32768, 32768, 32, 1, 1, "bulk"),
    "lay_a16_r32768_g32": (16, 32768, 32, 1, 1, "bulk"), "lay_a32768_r16_g8": (32768, 16, 8, 1, 1, "flat"),
    "lay_a20_r36_g16": (20, 36, 16, 4, 512, "flat"), "lay_i8_r16384_g32": (8, 16384, 32, 2, 2, "bulk"),
    "lay_i8_r8184_g8": (8, 8184, 8, 2, 4, "flat"),
}


def test_layout_sweep_reaches_every_layout_rule():
    """The generated sweep bodies (tests/layout_bodies.py) land where they claim: the restated Layout<B>::kUnit and
    align_tasks match what the module reports, the planner's slot stride gives the gather route of the table, and the
    sweep as a whole reaches every kAlign class, group size, gather route (resilient maps too), staged and global broadcast
    blocks, and every item and Out size class.  A change to any of these rules fails here instead of thinning the sweep."""
    lib = _abi.load()
    routes = {False: set(), True: set()}
    for b in LB.LAYOUTS:
        s = registry.spec(b.name)
        info = _abi.BodyInfo()
        assert lib.fbr_body_info(s.func_id, ctypes.byref(info)) == 0
        assert (info.arg_bytes, info.result_bytes, info.unit_tasks) == (b.A, b.R, b.k_unit), b.name
        assert info.flags & _abi.FBR_BODY_RECORD and bool(info.flags & _abi.FBR_BODY_INDEX_ARG) == b.index
        assert b.smem <= LB.SMEM_BUDGET, b.name
        p = _abi.Plan()
        assert lib.fbr_plan_query(s.func_id, 10 ** 6, 0, 0, 1, 0, 132, ctypes.byref(p)) == 0
        assert p.unit_tasks == b.k_unit and p.slot_stride == b.k_unit * b.R, b.name
        for resilient in (False, True):
            if resilient or not b.fault:
                routes[resilient].add(_gather_route(p.slot_stride, p.unit_tasks, b.R, resilient))
        if b.name in LAYOUT_TABLE:
            A, R, G, al, unit, route = LAYOUT_TABLE[b.name]
            assert (b.A, b.R, b.group, b.k_align, b.k_unit) == (A, R, G, al, unit), b.name
            assert _gather_route(p.slot_stride, p.unit_tasks, R, False) == route, b.name
    fixed = [LB.BY_NAME[n] for n in LAYOUT_TABLE]
    assert {b.k_align for b in fixed} == {1, 2, 4}
    assert {b.group for b in fixed} == {1, 2, 4, 8, 16, 32}
    # the largest record of each kAlign class: 4096 B one-thread, 16 KB with kAlign 2, 8 KB with kAlign 4, 32 KB
    for al, G, size in ((4, 1, 4096), (2, 2, 16384), (4, 4, 8188), (1, 32, 32768), (2, 32, 16384)):
        assert any(b.k_align == al and b.group == G and max(b.A, b.R) == size for b in fixed), (al, G, size)
    assert any(b.A == b.R == 32768 for b in fixed) and any(b.R >= 32 * b.A for b in fixed) and any(b.A >= 32 * b.R for b in fixed)
    # a large slot that is not a multiple of 4 KB goes to the flat gather
    assert any(b.k_unit * b.R > 16384 and b.k_unit * b.R % 4096 for b in fixed)
    assert routes[False] == {"flat", "rows", "bulk"} and routes[True] == {"flat", "rows"}
    faults = {_gather_route(b.k_unit * b.R, b.k_unit, b.R, False) for b in LB.LAYOUTS if b.fault}
    assert faults == {"flat", "rows", "bulk"}                        # the bulk-sized slot goes to the rows kernel resilient
    # broadcast blocks: never staged, staged, and a stage as large as the budget allows next to the layout's stages
    stages = {b.shared[1] for b in LB.LAYOUTS if b.shared}
    assert 0 in stages and 4096 in stages
    assert any(b.smem == LB.SMEM_BUDGET for b in LB.LAYOUTS if b.shared)
    assert {b.shared[0] for b in LB.LAYOUTS if b.shared} >= {4, 12, 4096}
    for b in LB.LAYOUTS:
        if b.shared:
            elem, stage = ctypes.c_uint32(), ctypes.c_uint32()
            assert lib.fbr_body_shared_info(registry.spec(b.name).func_id, ctypes.byref(elem), ctypes.byref(stage)) == 0
            assert (elem.value, stage.value) == b.shared
    items = [b for b in LB.LAYOUTS if b.items]
    assert {b.items for b in items if len(b.items) == 1} >= {(1,), (2,), (8,), (12,), (4096,)}
    assert (1, 2, 12, 4096) in {b.items for b in items}
    assert {b.A for b in items} == {0, 12} and {8, 32} <= {b.group for b in items}
    emits = [b for b in LB.LAYOUTS if b.out is not None]
    assert {b.out[0] for b in emits} >= {1, 2, 8, 12, 4096}
    assert {b.out[2] for b in emits if b.group == 1} == {True, False} and 32 in {b.group for b in emits}
    assert any(b.items and b.shared and b.group > 1 for b in emits)
    for b in emits:
        ob = ctypes.c_uint32()
        assert lib.fbr_body_emit_info(registry.spec(b.name).func_id, ctypes.byref(ob)) == 0 and ob.value == b.out[0]


def test_encoders():
    s = registry.spec("polar_f64")
    a = RB.polar_args(10)
    e = s.encode_map(a)
    assert e.args is a and (e.n, e.arg_stride) == (10, 16)                 # exactly the argument dtype: no copy
    e = s.encode_map(a[::2])
    assert e.n == 5 and np.array_equal(e.args, a[::2]) and e.args.flags.c_contiguous
    e = s.encode_starmap([(1.0, 2.0), (3, 4)])
    assert e.args.tolist() == [(1.0, 2.0), (3.0, 4.0)] and e.args.tobytes() == np.array([1, 2, 3, 4], "<f8").tobytes()
    assert s.encode_apply((1.5,), {"y": 2.5}).args.tolist() == [(1.5, 2.5)]
    assert s.encode_apply((), {"y": 2.5, "x": 0.5}).args.tolist() == [(0.5, 2.5)]
    for args, kwds, msg in (((1.0,), {}, r"missing 1 required positional argument: 'y'"),
                            ((), {}, r"missing 2 required positional arguments: 'x' and 'y'"),
                            ((1.0, 2.0, 3.0), {}, r"takes 2 positional arguments but 3 were given"),
                            ((1.0,), {"x": 2.0}, r"got multiple values for argument 'x'"),
                            ((1.0, 2.0), {"z": 2.0}, r"got an unexpected keyword argument 'z'")):
        with pytest.raises(TypeError, match=msg):
            s.encode_apply(args, kwds)
    with pytest.raises(TypeError, match="missing 1 required"):
        s.encode_map([1.0, 2.0])                                           # map passes one argument to f(x, y)
    with pytest.raises(TypeError, match="starmap items must be argument tuples"):
        s.encode_starmap([1.0])
    # one sub-array parameter: lists of rows, or a plain (n, 256) uint32 array viewed in place
    r = registry.spec("row_stats_u32")
    rows = RB.row_args(4)
    e = r.encode_map(rows["row"])
    assert e.args.dtype == RB.ROW_ARG and np.shares_memory(e.args, rows) and e.arg_stride == 1024
    assert np.array_equal(r.encode_map([x.tolist() for x in rows["row"]]).args, rows)
    assert r.encode_apply((), {"row": rows["row"][1]}).args.tobytes() == rows[1:2].tobytes()
    # a plain scalar dtype: lists of scalars, range() for an index body
    p = registry.spec("splitmix_pair")
    e = p.encode_map(range(5, 50, 3))
    assert (e.n, e.arg_stride, e.index_start, e.index_step) == (15, 0, 5, 3)
    e = p.encode_map([1, -2, 3])
    assert e.arg_stride == 8 and e.args.tobytes() == np.array([1, -2, 3], "<i8").tobytes()
    with pytest.raises(TypeError, match="unexpected keyword"):
        p.encode_apply((), {"i": 3})
    with pytest.raises(OverflowError):
        p.encode_map(range(2 ** 63, 2 ** 63 + 2))
    # a body that is not an index body takes range() as a list of values
    m = registry.spec("mix_i32x3")
    with pytest.raises(TypeError):
        m.encode_map(range(3))
    m3 = m.encode_starmap([(1, 2, 3)])
    assert m3.arg_stride == 12 and m3.args.tobytes() == np.array([1, 2, 3], "<i4").tobytes()


def test_decoding_and_sum():
    polar = registry.spec("polar_f64")
    out = RB.polar_np(RB.polar_args(1000, seed=1))
    ra = ResultArray(polar, out)
    assert ra.array is out and ra[0] == tuple(out[0].tolist()) and isinstance(ra[0][0], float)
    assert ra.tolist() == out.tolist() and ra[10:13] == out[10:13].tolist()
    with pytest.raises(TypeError, match="tuple"):
        ra.sum()                                                        # sum() of tuples fails in Python too
    # one value per task: floats and ints, summed as Python sums the list
    ok = registry.register_module("ok_f32", RB.BAD_MODULE, "ok_f32", args=[("x", "<f4")], result="<f4")
    vals = np.random.default_rng(2).standard_normal(1001).astype("<f4") * 1e6
    ra = ResultArray(ok, vals)
    assert ra.tolist() == vals.tolist() and isinstance(ra[3], float)
    assert ra.sum() == sum(vals.tolist()) and isinstance(ra.sum(), float)
    mix = registry.spec("mix_i32x3")
    m = RB.mix_np(RB.mix_args(50))
    assert ResultArray(mix, m)[7] == tuple(m[7].tolist()) and all(isinstance(v, int) for v in ResultArray(mix, m)[7])
    rows = ResultArray(registry.spec("row_stats_u32"), RB.row_stats_np(RB.row_args(5)))
    assert rows[2] == RB.row_stats_u32(RB.row_args(5)["row"][2])
    scale = registry.spec("scale5_f64")
    s5 = RB.scale5_np(RB.scale5_args(3))
    assert ResultArray(scale, s5)[1] == s5["w"][1].tolist()
    with pytest.raises(TypeError):
        ResultArray(scale, s5).sum()
    pair = registry.spec("splitmix_pair")
    pr = RB.splitmix_pair_np(np.arange(20))
    assert ResultArray(pair, pr).tolist() == [RB.splitmix_pair(i) for i in range(20)]
    assert pair.unpack_result(pr[4].tobytes()) == RB.splitmix_pair(4)
    # existing layouts keep their sums
    assert ResultArray(registry.spec("square_i64"), np.array([2 ** 62, 2 ** 62, 2 ** 62], np.int64)).sum() == 3 * 2 ** 62


def test_device_body_decorator_checks_result_dtype():
    with pytest.raises(ValueError, match="result dtype"):
        fiber_b200.device_body("polar_f64", source=RB.POLAR_SRC, entry="polar_entry", args=RB.POLAR_ARG, result="<f8")
    assert registry.spec("polar_f64").res_dtype == RB.POLAR_RES
