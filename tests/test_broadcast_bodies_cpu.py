"""CPU: record bodies that read a broadcast block -- descriptor flags and fields, registration rules, the element dtype,
the encoders that split the shared array from the per-task records, initializer binding and claim-unit plans.  No
device is needed for any of it."""
import ctypes

import numpy as np
import pytest

import fiber_b200
from fiber_b200 import _abi, registry

from . import broadcast_bodies as BB
from . import record_bodies as RB


def _shared_info(name):
    e, s = ctypes.c_uint32(), ctypes.c_uint32()
    assert _abi.load().fbr_body_shared_info(registry.spec(name).func_id, ctypes.byref(e), ctypes.byref(s)) == 0
    return e.value, s.value


def _register(name):
    fid = ctypes.c_int(-1)
    rc = _abi.load().fbr_register_body(name.encode(), BB.BAD_MODULE.encode(), name.encode(), ctypes.byref(fid))
    return rc, _abi.load().fbr_last_error().decode()


def test_flags_and_shared_info():
    want = {"nearest_centroid_f32": (64, 8, 64, 32768), "nearest_centroid_global_f32": (64, 8, 64, 0),
            "kde_window_f64": (8, 16, 16, 16384), "table_mix_u32": (8, 4, 4, 16384)}
    for name, (a, r, elem, stage) in want.items():
        s = registry.spec(name)
        assert isinstance(s, registry._Broadcast) and (s.arg_bytes, s.result_bytes) == (a, r)
        need = _abi.FBR_BODY_RECORD | _abi.FBR_BODY_NEEDS_SHARED | _abi.FBR_BODY_BROADCAST
        assert s.flags & need == need and not s.flags & _abi.FBR_BODY_SUMMABLE
        assert _shared_info(name) == (elem, stage) == (s.elem_bytes, s.stage_bytes)
    assert registry.spec("table_mix_u32").flags & _abi.FBR_BODY_INDEX_ARG
    # every other body: no broadcast element
    for name in ("polar_f64", "parzen_f64", "square_i64"):
        assert _shared_info(name) == (0, 0) and not registry.spec(name).flags & _abi.FBR_BODY_BROADCAST
    assert registry.spec("parzen_f64").flags & _abi.FBR_BODY_NEEDS_SHARED
    assert _abi.load().fbr_body_shared_info(10 ** 6, ctypes.byref(ctypes.c_uint32()), ctypes.byref(ctypes.c_uint32())) == _abi.FBR_EINVAL
    mod = registry.module_of("nearest_centroid_f32")
    assert mod[2] == BB.POINT and mod[4] == BB.NEAREST_RES and mod[5] == ("centroids", BB.CENTROID)


def test_registration_refusals():
    for name, why in (("bad_no_needs", "needs FBR_BODY_NEEDS_SHARED"), ("bad_thread", "only record bodies"),
                      ("bad_fields", "lacks FBR_BODY_BROADCAST"), ("bad_stage_only", "lacks FBR_BODY_BROADCAST"),
                      ("bad_elem0", "multiple of 4 bytes up to 4096"), ("bad_elem6", "multiple of 4 bytes up to 4096"),
                      ("bad_elem_big", "multiple of 4 bytes up to 4096"), ("bad_stage24", "multiple of 16"),
                      ("bad_stage_big", "exceed 200 KB")):
        rc, msg = _register(name)
        assert rc == _abi.FBR_EINVAL and why in msg, (name, msg)
    assert _register("ok_bcast")[0] == _abi.FBR_OK
    # the record-body rule still holds: NEEDS_SHARED without a Shared type is refused
    fid = ctypes.c_int(-1)
    assert _abi.load().fbr_register_body(b"bad_shared", RB.BAD_MODULE.encode(), b"bad_shared", ctypes.byref(fid)) == _abi.FBR_EINVAL
    assert "NEEDS_SHARED" in _abi.load().fbr_last_error().decode()


def test_shared_dtype_validation():
    reg = lambda **kw: registry.register_module("ok_bcast", BB.BAD_MODULE, "ok_bcast", args="<f4", result="<f4", **kw)
    with pytest.raises(ValueError, match="shared="):
        reg()                                                              # a broadcast body needs shared=
    with pytest.raises(ValueError, match="broadcast element dtype"):
        reg(shared=("w", "<f8"))
    with pytest.raises(TypeError, match="big-endian"):
        reg(shared=("w", ">f4"))
    with pytest.raises(TypeError, match="Python objects"):
        reg(shared=("w", [("o", "O")]))
    with pytest.raises(ValueError, match="parameter name"):
        reg(shared=("not a name", "<f4"))
    with pytest.raises(ValueError, match="also an argument field"):
        registry.register_module("ok_bcast", BB.BAD_MODULE, "ok_bcast", args=[("w", "<f4")], result="<f4", shared=("w", "<f4"))
    s = reg(shared=("w", "<f4"))
    assert s.shared_name == "w" and s.shared_dtype == np.dtype("<f4")
    assert reg(shared=("w", "<f4")) is s
    with pytest.raises(ValueError, match="registered already"):
        reg(shared=("v", "<f4"))
    assert registry.module_of("ok_bcast")[5] == ("w", np.dtype("<f4"))
    # shared= is refused for bodies that read no block
    with pytest.raises(ValueError, match="broadcast bodies only"):
        registry.register_module("polar_f64", *registry.module_of("polar_f64")[:2], args=RB.POLAR_ARG, result=RB.POLAR_RES,
                                 shared=("c", "<f4"))
    from . import device_bodies  # noqa: F401  (registers collatz_steps, a thread body)
    with pytest.raises(ValueError, match="broadcast bodies only"):
        registry.register_module("collatz_steps", *registry.module_of("collatz_steps")[:2], shared=("c", "<f4"))


def test_encoders_bind_the_block():
    s = registry.spec("nearest_centroid_f32")
    C = BB.centroids(5)
    P = BB.points(4)
    plain = C["c"]                                                         # (5, 16) float32: a view of the elements
    e = s.encode_starmap([(C, p) for p in P["p"]])
    assert e.n == 4 and e.args.tobytes() == P.tobytes() and e.shared == C.tobytes()
    assert s.encode_starmap([(plain, p) for p in P["p"]]).shared is s.shared_block(C)   # equal content: the same block
    e = s.encode_apply((C, P["p"][1]), {})
    assert e.n == 1 and e.args.tobytes() == P[1:2].tobytes() and e.shared is s.shared_block(C)
    e = s.encode_apply((P["p"][2],), {"centroids": plain})
    assert e.args.tobytes() == P[2:3].tobytes() and e.shared is s.shared_block(C)
    e = s.encode_apply((), {"p": P["p"][3], "centroids": C})
    assert e.args.tobytes() == P[3:4].tobytes() and e.shared is s.shared_block(C)
    # without the block: the pool's initializer block (enc.shared None)
    e = s.encode_map(P)
    assert e.args is P and e.shared is None
    e = s.encode_starmap([(p,) for p in P["p"]])
    assert e.shared is None and e.args.tobytes() == P.tobytes()
    with pytest.raises(TypeError, match="mixed items"):
        s.encode_starmap([(C, P["p"][0]), (P["p"][1],)])
    with pytest.raises(TypeError, match="mixed items"):
        s.encode_starmap([(P["p"][1],), (C, P["p"][0])])
    C2 = C.copy()
    C2["c"][3, 7] += 1.0
    with pytest.raises(ValueError, match="must share centroids"):
        s.encode_starmap([(C, P["p"][0]), (C2, P["p"][1])])
    assert s.encode_starmap([(C, P["p"][0]), (C.copy(), P["p"][1])]).shared == C.tobytes()   # equal arrays are accepted
    # the element must match: dtype and trailing shape
    for bad in (plain.astype(np.float64), plain[:, :8], plain.reshape(-1), np.zeros((0, 16), np.float32)):
        with pytest.raises((TypeError, ValueError)):
            s.encode_apply((bad, P["p"][0]), {})
    with pytest.raises(TypeError, match="missing 1 required positional argument: 'p'"):
        s.encode_apply((), {"centroids": C})
    # a scalar element: a 1-D uint32 table
    t = registry.spec("table_mix_u32")
    tab = BB.table(3)
    e = t.encode_starmap([(tab, 5), (tab, 9)])
    assert e.shared == tab.tobytes() and e.args.tobytes() == np.array([5, 9], "<i8").tobytes()
    e = t.encode_map(range(2, 12, 3))
    assert (e.n, e.arg_stride, e.index_start, e.index_step, e.shared) == (4, 0, 2, 3, None)
    with pytest.raises(TypeError):
        t.encode_apply((tab.astype(np.int32), 5), {})


def test_last_block_is_kept_and_rebuilt():
    s = registry.spec("kde_window_f64")
    xs = np.random.default_rng(3).standard_normal((300, 2))
    b1 = s.shared_block(xs)
    assert s.shared_block(xs) is b1 and s.shared_block(xs.copy()) is b1 and len(b1) == xs.nbytes
    xs[4, 1] += 1.0                                                        # changed in place: rebuilt
    b2 = s.shared_block(xs)
    assert b2 is not b1 and b2 == xs.tobytes()
    with pytest.raises(TypeError, match="exactly one argument"):
        s.shared_block(xs, xs)
    # parzen keeps its own last block the same way
    p = registry.spec("parzen_f64")
    px = np.zeros((2, 1))
    pb = p.shared_block(xs, px)
    assert p.shared_block(xs.copy(), px.copy()) is pb


def test_device_initializer_binding():
    assert BB.set_centroids.__fbr_init_body__ == "nearest_centroid_f32"
    pool = fiber_b200.Pool(1, initializer=BB.set_centroids, initargs=(BB.centroids(3),))
    assert pool._initializer is BB.set_centroids
    assert registry.spec("nearest_centroid_f32").shared_block(*pool._initargs) == BB.centroids(3).tobytes()
    # the worker processes of an isolated pool rebuild the same initializer from (body, initargs, module)
    from fiber_b200.procpool import _initializer_for
    f = _initializer_for("kde_window_f64")
    assert f.__fbr_init_body__ == "kde_window_f64"
    with pytest.raises(RuntimeError):
        f()


def test_plans_match_plain_record_bodies():
    """A broadcast body plans its claim units like any record body of the same argument and result sizes."""
    lib = _abi.load()
    # the record-body rules: both sides of every unit 16 B aligned, a unit never exceeds the kernel's stage
    for bname in ("nearest_centroid_f32", "nearest_centroid_global_f32", "kde_window_f64", "table_mix_u32"):
        s = registry.spec(bname)
        info = _abi.BodyInfo()
        assert lib.fbr_body_info(s.func_id, ctypes.byref(info)) == 0
        for n in (1, 7, 1000, 10 ** 6, 10 ** 8):
            for cs in (1, 7, 32, 5000):
                p = _abi.Plan()
                assert lib.fbr_plan_query(s.func_id, n, cs, 0, 1, 0, 132, ctypes.byref(p)) == 0
                assert p.unit_tasks * s.result_bytes % 16 == 0 and p.unit_tasks * s.arg_bytes % 16 == 0
                assert p.unit_tasks <= info.unit_tasks and p.slot_stride == p.unit_tasks * s.result_bytes
    # kde (8 B -> 16 B) against the plain record body splitmix_pair (8 B -> 16 B): identical plans
    a, b = registry.spec("kde_window_f64"), registry.spec("splitmix_pair")
    for n in (1, 7, 1000, 10 ** 6, 10 ** 8):
        for cs in (1, 3, 7, 32, 100, 5000):
            pa, pb = _abi.Plan(), _abi.Plan()
            assert lib.fbr_plan_query(a.func_id, n, cs, 0, 2, 1, 132, ctypes.byref(pa)) == 0
            assert lib.fbr_plan_query(b.func_id, n, cs, 0, 2, 1, 132, ctypes.byref(pb)) == 0
            assert bytes(pa) == bytes(pb), (n, cs)
