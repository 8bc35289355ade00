"""CPU: emit record bodies -- registration rules, flags and fbr_body_emit_info, out= / out_as= validation, header constants,
and EmitResultArray / Ragged assembly from fabricated end offsets and values.  No GPU needed."""
import ctypes
import os
import re

import numpy as np
import pytest

import fiber_b200
from fiber_b200 import _abi, registry
from fiber_b200.pool import EmitResultArray

from . import emit_bodies as EB

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _register(name):
    fid = ctypes.c_int(-1)
    rc = _abi.load().fbr_register_body(name.encode(), EB.BAD_MODULE.encode(), name.encode(), ctypes.byref(fid))
    return rc, _abi.load().fbr_last_error().decode()


@pytest.mark.parametrize("name,why", [
    ("bad_emit_fields", "describes an out element but lacks FBR_BODY_EMIT"),
    ("bad_emit_thread", "only record bodies"),
    ("bad_emit_res", "no fixed result record"),
    ("bad_emit_kind", "no fixed result record"),
    ("bad_out0", "the out size must be 1, 2 or a multiple of 4"),
    ("bad_out3", "the out size must be 1, 2 or a multiple of 4"),
    ("bad_out_big", "the out size must be 1, 2 or a multiple of 4"),
    ("bad_emit_sum", "cannot be folded on the device"),
])
def test_registration_rules(name, why):
    rc, msg = _register(name)
    assert rc == _abi.FBR_EINVAL and why in msg, msg


def test_flags_and_emit_info():
    rc, msg = _register("ok_emit")
    assert rc == _abi.FBR_OK, msg
    L = _abi.load()
    for name, out_bytes, extra in [("tokens_u32", 4, _abi.FBR_BODY_ITEMS), ("prime_factors_i64", 8, _abi.FBR_BODY_INDEX_ARG),
                                   ("above_mask_f64", 4, _abi.FBR_BODY_ITEMS), ("upper_ascii_u8", 1, _abi.FBR_BODY_ITEMS),
                                   ("radius_neighbors_f32", 4, _abi.FBR_BODY_BROADCAST), ("ok_emit", 4, _abi.FBR_BODY_ITEMS)]:
        spec = registry.spec(name) if name != "ok_emit" else None
        fid = spec.func_id if spec else ctypes.c_int(-1)
        if spec is None:
            _abi.check(L.fbr_body_lookup(b"ok_emit", ctypes.byref(fid)))
            fid = fid.value
        info = _abi.BodyInfo()
        _abi.check(L.fbr_body_info(fid, ctypes.byref(info)))
        assert info.flags & (_abi.FBR_BODY_RECORD | _abi.FBR_BODY_EMIT | extra) == _abi.FBR_BODY_RECORD | _abi.FBR_BODY_EMIT | extra
        assert not info.flags & _abi.FBR_BODY_SUMMABLE
        assert (info.result_bytes, info.result_kind) == (8, _abi.FBR_RES_OFFSETS)
        ob = ctypes.c_uint32(99)
        _abi.check(L.fbr_body_emit_info(fid, ctypes.byref(ob)))
        assert ob.value == out_bytes
    ob = ctypes.c_uint32(99)
    _abi.check(L.fbr_body_emit_info(registry.spec("token_sum_u32").func_id, ctypes.byref(ob)))
    assert ob.value == 0


def test_out_parameter_validation():
    path = fiber_b200.bodies.compile_module("tokens_u32", EB.TOKENS_SRC)
    reg = lambda **kw: registry.register_module("tokens_u32", path, "tokens_entry", args=None, items=("doc", "u1"), **kw)
    with pytest.raises(ValueError, match="pass out="):
        reg()
    with pytest.raises(ValueError, match="result= is for fixed-size results"):
        reg(out="<u4", result="<u8")
    with pytest.raises(ValueError, match="out dtype .* is 8 bytes, the body's Out is 4"):
        reg(out="<u8")
    with pytest.raises(ValueError, match="out_as is 'list', 'bytes' or 'str'"):
        reg(out="<u4", out_as="tuple")
    with pytest.raises(ValueError, match="needs a 1-byte out element"):
        reg(out="<u4", out_as="str")
    reg(out="<u4")
    with pytest.raises(ValueError, match="out= is for emit bodies only"):
        registry.register_module("token_sum_u32", fiber_b200.bodies.compile_module("token_sum_u32", EB.TOKEN_SUM_SRC),
                                 "token_sum_entry", args=None, items=("xs", "<u4"), result=EB.TOKEN_SUM_RES, out="<u4")


def test_header_constants_match_abi():
    with open(os.path.join(ROOT, "include", "fiber_b200.h")) as fh:
        h = fh.read()
    assert int(re.search(r"#define FBR_BODY_EMIT (0x[0-9a-f]+)u", h).group(1), 16) == _abi.FBR_BODY_EMIT
    assert int(re.search(r"FBR_RES_OFFSETS = (\d+)", h).group(1)) == _abi.FBR_RES_OFFSETS
    assert int(re.search(r"FBR_TASK_EMIT = (\d+)", h).group(1)) == _abi.FBR_TASK_EMIT
    with open(os.path.join(ROOT, "fiber_b200", "csrc", "bodies.cuh")) as fh:
        assert "TASK_EMIT = %d" % _abi.FBR_TASK_EMIT in fh.read()
    L = _abi.load()
    for sym in ("fbr_body_emit_info", "fbr_result_values", "fbr_result_fetch_values"):
        assert hasattr(L, sym) and sym in _abi.SYMBOLS


def _fabricated(spec, lists):
    ends = np.cumsum([len(x) for x in lists]).astype(np.uint64)
    values = np.array([v for x in lists for v in x], spec.out_dtype)
    return ends, values


def test_result_array_assembly():
    spec = registry.spec("tokens_u32")
    lists = [[1, 2, 3], [], [4], [], [], [5, 6], []]
    ends, values = _fabricated(spec, lists)
    r = EmitResultArray(spec, ends, values)
    assert len(r) == len(lists) and r == lists and r.tolist() == lists and list(r) == lists
    assert r[0] == [1, 2, 3] and r[1] == [] and r[-2] == [5, 6] and r[2:6] == lists[2:6] and r[::2] == lists[::2]
    with pytest.raises(IndexError):
        r[len(lists)]
    with pytest.raises(TypeError):
        r.sum()
    rg = r.ragged
    assert isinstance(rg, registry.Ragged) and len(rg) == len(lists)
    assert [rg[i].tolist() for i in range(len(rg))] == lists
    assert np.shares_memory(rg.values, values)
    # the device-resident form fetches ranges of end offsets and values
    fetched = []
    r2 = EmitResultArray(spec, None, None, n=len(lists), fetch=lambda lo, hi: (fetched.append((lo, hi)), ends[lo:hi])[1],
                         fetch_values=lambda lo, hi: values[lo:hi])
    assert r2[5] == [5, 6] and fetched == [(4, 6)]
    assert r2 == lists


def test_result_array_strings():
    spec = registry.spec("upper_ascii_u8")
    words = ["ALPHA", "", "B C", "\t"]
    ends, values = _fabricated(spec, [list(w.encode()) for w in words])
    r = EmitResultArray(spec, ends, values)
    assert r.tolist() == words and r[2] == "B C"

