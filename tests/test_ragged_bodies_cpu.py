"""CPU: items record bodies -- registration rules, the items encoders, Ragged and the header constants.  No GPU needed: registration, planning and encoding are host code."""
import ctypes
import os

import numpy as np
import pytest

import fiber_b200
from fiber_b200 import _abi, registry

from . import ragged_bodies as RB

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _register(name):
    fid = ctypes.c_int(-1)
    rc = _abi.load().fbr_register_body(name.encode(), RB.BAD_MODULE.encode(), name.encode(), ctypes.byref(fid))
    return rc, _abi.load().fbr_last_error().decode()


@pytest.mark.parametrize("name,why", [
    ("bad_items_fields", "lacks FBR_BODY_ITEMS"),
    ("bad_items_thread", "only record bodies take items"),
    ("bad_item0", "1, 2 or a multiple of 4 up to 4096"),
    ("bad_item3", "1, 2 or a multiple of 4 up to 4096"),
    ("bad_item_big", "1, 2 or a multiple of 4 up to 4096"),
    ("bad_items_index", "FBR_BODY_INDEX_ARG"),
    ("bad_noarg", "only for an items body"),
])
def test_registration_rules(name, why):
    rc, msg = _register(name)
    assert rc == _abi.FBR_EINVAL and why in msg, msg


def _items_info(name):
    ib = ctypes.c_uint32()
    _abi.check(_abi.load().fbr_body_items_info(registry.spec(name).func_id, ctypes.byref(ib)))
    return ib.value


def test_flags_and_items_info():
    assert _register("ok_items")[0] == _abi.FBR_OK
    want = {"fnv1a_bytes": (0, 16, 1), "fault_fnv1a_bytes": (0, 16, 1), "ragged_stats_f64": (0, 32, 8),
            "clip_sum_f32": (8, 8, 4), "token_weight_u32": (0, 8, 4)}
    for name, (a, r, ib) in want.items():
        s = registry.spec(name)
        assert isinstance(s, registry._Items) and (s.arg_bytes, s.result_bytes) == (a, r)
        assert s.flags & (_abi.FBR_BODY_RECORD | _abi.FBR_BODY_ITEMS) == _abi.FBR_BODY_RECORD | _abi.FBR_BODY_ITEMS
        assert _items_info(name) == ib
    assert registry.spec("token_weight_u32").flags & _abi.FBR_BODY_BROADCAST
    assert _items_info("square_i64") == 0


def test_encoders():
    s = registry.spec("fnv1a_bytes")
    enc = s.encode_map([b"ab", "cé", bytearray(b"xyz"), memoryview(b""), b"q"])
    v, o = enc.items
    assert enc.n == 5 and bytes(v) == b"abc\xc3\xa9xyzq" and o.tolist() == [0, 2, 5, 8, 8, 9] and o.dtype == np.uint64
    arrs = [np.arange(3, dtype=np.uint8), [4, 5], np.zeros(0, np.uint8)]
    v, o = s.encode_map(arrs).items
    assert v.tolist() == [0, 1, 2, 4, 5] and o.tolist() == [0, 3, 5, 5]
    enc = s.encode_map([])
    assert enc.n == 0 and enc.items[1].tolist() == [0]
    with pytest.raises(TypeError, match="mixed"):
        s.encode_map([b"ab", np.arange(2, dtype=np.uint8)])
    with pytest.raises(TypeError, match="1-D"):
        s.encode_map([np.zeros((2, 2), np.uint8)])
    f8 = registry.spec("ragged_stats_f64")
    with pytest.raises(TypeError, match="1-byte"):
        f8.encode_map(["abc"])
    with pytest.raises(TypeError, match="not convertible"):
        f8.encode_map([["a", "b"]])
    for bad in ([-1], [300], [1.7], np.array([256]), np.array([0.5]), ["1"]):
        with pytest.raises(TypeError):
            s.encode_map([bad])                              # never wrapped or truncated into uint8
    v, o = f8.encode_map([[1.0, 2.0], np.array([3], np.int32)]).items
    assert v.dtype == np.float64 and v.tolist() == [1.0, 2.0, 3.0] and o.tolist() == [0, 2, 3]
    # starmap / apply bind the items and the head record like a Python call
    c = registry.spec("clip_sum_f32")
    enc = c.encode_starmap([([1, 2], 0.5, 1.5), (np.ones(3, np.float32), 0, 1)])
    assert enc.args.tolist() == [(0.5, 1.5), (0.0, 1.0)] and enc.items[1].tolist() == [0, 2, 5]
    enc = c.encode_apply(([1.0],), {"hi": 2, "lo": -1})
    assert enc.args.tolist() == [(-1.0, 2.0)]
    enc = c.encode_apply((), {"row": [1.0, 2.0], "lo": 0, "hi": 1})
    assert enc.items[0].tolist() == [1.0, 2.0]
    with pytest.raises(TypeError, match="missing 1 required"):
        c.encode_apply(([1.0], 0), {})
    with pytest.raises(TypeError):
        s.encode_starmap([(b"ab", 3)])
    t = registry.spec("token_weight_u32")
    w = np.ones(4, np.float32)
    enc = t.encode_starmap([(w, [1, 2]), (w, [3])])
    assert enc.shared == w.tobytes() and enc.items[0].tolist() == [1, 2, 3]
    with pytest.raises(ValueError, match="share"):
        t.encode_starmap([(w, [1]), (w * 2, [1])])
    # the Python definitions agree with the restatements
    vals, offs = RB.byte_strings(50, seed=3, max_len=40)
    want = RB.fnv1a_np(vals, offs)
    assert [RB.fnv1a_bytes(vals[offs[i]:offs[i + 1]].tobytes()) for i in range(50)] == want.tolist()


def test_ragged_zero_copy_and_validation():
    vals = np.arange(20, dtype=np.float64)
    offs = np.array([2, 5, 5, 20], np.int64)                       # offsets[0] need not be 0
    r = fiber_b200.Ragged(vals, offs)
    assert len(r) == 3 and r[0].tolist() == [2.0, 3.0, 4.0] and len(r[1]) == 0 and r[-1].tolist() == list(range(5, 20))
    v, o = registry.spec("ragged_stats_f64").encode_map(r).items
    assert np.shares_memory(v, vals) and np.shares_memory(o, offs) and o.dtype == np.uint64
    sub = r[1:3]
    assert sub.offsets.tolist() == [0, 0, 15] and sub[1].tolist() == list(range(5, 20))
    import pickle
    assert pickle.loads(pickle.dumps(sub))[1].tolist() == sub[1].tolist()
    with pytest.raises(ValueError, match="decrease"):
        fiber_b200.Ragged(vals, [0, 5, 3])
    with pytest.raises(ValueError, match=r"\[0, len\(values\)\]"):
        fiber_b200.Ragged(vals, [0, 21])
    with pytest.raises(ValueError, match=r"\[0, len\(values\)\]"):
        fiber_b200.Ragged(vals, [-1, 2])
    with pytest.raises(ValueError, match="1-D"):
        fiber_b200.Ragged(vals.reshape(4, 5), [0, 1])
    with pytest.raises(IndexError):
        r[3]
    with pytest.raises(TypeError, match="Ragged values"):
        registry.spec("fnv1a_bytes").encode_map(r)


def test_items_parameter_validation():
    reg = lambda **kw: registry.register_module("ok_items", RB.BAD_MODULE, "ok_items", result=RB.FNV_RES, **kw)
    with pytest.raises(ValueError, match="items="):
        reg()
    with pytest.raises(ValueError, match="item dtype"):
        reg(items=("s", "<u2"))
    with pytest.raises(ValueError, match="parameter name"):
        reg(items=("not a name", "u1"))
    s = reg(items=("s", "u1"))
    assert reg(items=("s", "u1")) is s and registry.module_of("ok_items")[6] == ("s", np.dtype("u1"))
    with pytest.raises(ValueError, match="registered already"):
        reg(items=("t", "u1"))
    with pytest.raises(ValueError, match="items bodies only"):
        path, entry = registry.module_of("padded_stats_f64")[:2]
        registry.register_module("padded_stats_f64", path, entry, args=RB.PADDED_ARG, result=RB.STATS_RES, items=("s", "u1"))


def test_header_constants_match_abi():
    with open(os.path.join(ROOT, "include", "fiber_b200.h")) as fh:
        h = fh.read()
    assert "#define FBR_BODY_ITEMS 0x40u" in h and _abi.FBR_BODY_ITEMS == 0x40
    assert "#define FBR_BODY_MODULE_ABI %d" % _abi.FBR_BODY_MODULE_ABI in h and _abi.FBR_BODY_MODULE_ABI == 4
    assert "#define FBR_ABI_VERSION 2" in h and _abi.FBR_ABI_VERSION == 2
    for sym in ("fbr_map_submit_items", "fbr_body_items_info"):
        assert sym in h and sym in _abi.SYMBOLS
    assert ctypes.sizeof(_abi.ItemsDesc) == 32 and ctypes.sizeof(_abi.MapDesc) == 104


def test_submit_refuses_the_wrong_entry_point():
    """Without a pool the calls fail on the NULL pool first; the body check needs a pool, so it is covered on the GPU."""
    d = _abi.MapDesc()
    seq = ctypes.c_uint64()
    assert _abi.load().fbr_map_submit(None, ctypes.byref(d), ctypes.byref(seq)) == _abi.FBR_EINVAL
    it = _abi.ItemsDesc()
    assert _abi.load().fbr_map_submit_items(None, ctypes.byref(d), ctypes.byref(it), ctypes.byref(seq)) == _abi.FBR_EINVAL
