"""CPU: group record bodies (kGroup) -- registration rules for group_threads and the 32 KB records they allow, the
claim-unit plans of the new sizes, and the zero-copy encoders for 2-D arrays of 8 KB and 32 KB rows.  No device is
needed for any of it."""
import ctypes

import numpy as np

from fiber_b200 import _abi, registry

from . import group_bodies as GB


def _register(name):
    fid = ctypes.c_int(-1)
    rc = _abi.load().fbr_register_body(name.encode(), GB.BAD_MODULE.encode(), name.encode(), ctypes.byref(fid))
    return rc, _abi.load().fbr_last_error().decode()


def _plan(name, n, chunksize):
    p = _abi.Plan()
    assert _abi.load().fbr_plan_query(registry.spec(name).func_id, n, chunksize, 0, 1, 0, 132, ctypes.byref(p)) == 0
    return p


def test_registration_accepts_the_group_bodies():
    want = {"row_moments_f64": (8192, 32), "fault_row_moments_f64": (8192, 32), "wide_row_max_f32": (32768, 16),
            "splitmix_row_u32": (8, 8192), "mat4_apply_f32": (80, 20), "nearest_row_group_f32": (256, 8)}
    for name, (a, r) in want.items():
        s = registry.spec(name)
        assert isinstance(s, registry._Record) and (s.arg_bytes, s.result_bytes) == (a, r), name
        assert s.flags & _abi.FBR_BODY_RECORD and s.result_kind == _abi.FBR_RES_BYTES
    assert registry.spec("splitmix_row_u32").flags & _abi.FBR_BODY_INDEX_ARG
    assert registry.spec("nearest_row_group_f32").flags & _abi.FBR_BODY_BROADCAST
    assert isinstance(registry.spec("nearest_row_group_f32"), registry._Broadcast)


def test_registration_rejects_bad_groups():
    for name, why in (("bad_group3", "group_threads 3 is not"), ("bad_group64", "group_threads 64 is not"),
                      ("bad_group_thread", "only record bodies run a task on a group"),
                      ("bad_group_64k", "at most 32768 bytes"),
                      ("bad_group_align", "kAlign * max(arg_bytes, result_bytes) <= 32768"),
                      ("bad_thread_8k", "at most 4096 bytes")):
        rc, msg = _register(name)
        assert rc == _abi.FBR_EINVAL and why in msg, (name, msg)
    assert _register("ok_group")[0] == _abi.FBR_OK


def test_plan_units_of_the_new_sizes():
    # 32 KB argument records: one task per unit whatever the chunksize, and a 16 B slot
    for n in (1, 7, 3000, 10 ** 6):
        for cs in (1, 7, 32, 1000):
            p = _plan("wide_row_max_f32", n, cs)
            assert (p.unit_tasks, p.slot_stride) == (1, 16), (n, cs)
            assert p.n_units == n
    # 8 KB records: four tasks fill the 32 KB stage
    for name in ("row_moments_f64", "splitmix_row_u32"):
        assert _plan(name, 10 ** 6, 32).unit_tasks == 4
        assert _plan(name, 10 ** 6, 1).unit_tasks == 4
    assert _plan("splitmix_row_u32", 10 ** 6, 7).slot_stride == 4 * 8192
    # 80 B -> 20 B: units are multiples of 4 tasks, so every slot and argument offset stays 16 B aligned; at most the
    # 256 tasks (20 KB of arguments) of one stage
    info = _abi.BodyInfo()
    assert _abi.load().fbr_body_info(registry.spec("mat4_apply_f32").func_id, ctypes.byref(info)) == 0
    assert info.unit_tasks == 256
    for n in (1, 7, 1000, 10 ** 6):
        for cs in (1, 3, 7, 32, 100, 5000):
            p = _plan("mat4_apply_f32", n, cs)
            assert p.unit_tasks % 4 == 0 and p.slot_stride == p.unit_tasks * 20 and p.unit_tasks <= 256, (n, cs)


def test_encoders_take_2d_rows_without_a_copy():
    m = registry.spec("row_moments_f64")
    rows = np.random.default_rng(0).standard_normal((5, 1024))            # 8 KB rows
    e = m.encode_map(rows)
    assert e.n == 5 and e.arg_stride == 8192 and e.args.dtype == GB.MOMENTS_ARG and np.shares_memory(e.args, rows)
    assert np.array_equal(e.args["x"], rows)
    w = registry.spec("wide_row_max_f32")
    wide = np.random.default_rng(1).standard_normal((3, 8192), dtype=np.float32)   # 32 KB rows
    e = w.encode_map(wide)
    assert e.n == 3 and e.arg_stride == 32768 and e.args.dtype == GB.WIDE_ARG and np.shares_memory(e.args, wide)
    a = GB.wide_args(4)
    assert w.encode_map(a).args is a
    # rows of a Fortran-ordered array are copied into one contiguous block
    f = np.asfortranarray(rows)
    e = m.encode_map(f)
    assert not np.shares_memory(e.args, f) and np.array_equal(e.args["x"], rows)


def test_python_definitions_match_the_restatements():
    """The Python definitions repeat each body's order of operations, so they agree with the NumPy restatements bit for
    bit (what the GPU tests compare the device against)."""
    a = GB.moments_args(3, seed=4)
    want = GB.row_moments_np(a)
    assert [GB.row_moments_f64(r) for r in a["x"]] == want.tolist()
    w = GB.wide_args(3, seed=5)
    assert [GB.wide_row_max_f32(r) for r in w["x"]] == [(t[0], t[1], list(t[2])) for t in GB.wide_row_max_np(w).tolist()]
    assert GB.wide_row_max_np(w)["argmax"][1] == 100
    assert GB.splitmix_row_u32(-3) == GB.splitmix_row_np([-3])["w"][0].tolist()
    m = GB.mat4_args(20, seed=6)
    got = [GB.mat4_apply_f32(r["m"], r["v"]) for r in m]
    assert got == [(list(y), n) for y, n in GB.mat4_np(m).tolist()]
    c = GB.centroids64(9, seed=7)
    p = GB.points64(6, seed=8)
    assert [GB.nearest_row_group_f32(c, q) for q in p["p"]] == GB.nearest64_np(p, c).tolist()
