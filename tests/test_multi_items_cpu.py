"""CPU: multi-stream items bodies without a GPU -- registration rules and messages (hand-written descriptors and wrong
``items=`` lists), fbr_body_items_streams, the header constants, the submit entry points' stream checks, the encoders
(starmap and keyword binding, map refusal), ``Columns`` (lengths, zero copy, slicing, pickling) and process-pool blocks
of a ``Columns`` map."""
import ctypes
import os
import pickle
import re

import numpy as np
import pytest

import fiber_b200
from fiber_b200 import Columns, Ragged, _abi, registry
from fiber_b200.procpool import BLOCK_ALIGN, ProcessPool

from . import multi_items_bodies as M
from . import ragged_bodies, record_bodies  # noqa: F401  (one-stream and non-items bodies to compare with)
from ._fake_worker import fake_worker_main

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _register(name, entry=None):
    L = _abi.load()
    fid = ctypes.c_int(-1)
    rc = L.fbr_register_body(name.encode(), M.BAD_MODULE.encode(), (entry or name).encode(), ctypes.byref(fid))
    return rc, L.fbr_last_error().decode(), fid.value


@pytest.mark.parametrize("name, why", [
    ("bad_streams5", "takes at most 4 item streams"),
    ("bad_streams_flag", "lacks FBR_BODY_ITEMS"),
    ("bad_stream_size", "the item size of every stream must be 1, 2 or a multiple of 4 up to 4096 bytes"),
    ("bad_stream_size0", "the item size of every stream must be 1, 2 or a multiple of 4 up to 4096 bytes"),
    ("bad_stream_extra", "describes the item size of a stream past its item_streams"),
])
def test_bad_descriptors_are_refused(name, why):
    rc, msg, _ = _register(name)
    assert rc == _abi.FBR_EINVAL and why in msg and name in msg


def test_streams_info_and_flags():
    rc, msg, fid = _register("ok_streams")
    assert rc == _abi.FBR_OK, msg
    L = _abi.load()
    n, sizes, ib = ctypes.c_uint32(), (ctypes.c_uint32 * 4)(), ctypes.c_uint32()
    _abi.check(L.fbr_body_items_streams(fid, ctypes.byref(n), sizes))
    assert n.value == 2 and list(sizes) == [4, 4, 0, 0]
    _abi.check(L.fbr_body_items_info(fid, ctypes.byref(ib)))
    assert ib.value == 4
    for name, want in (("mix4_u1_u2_u4_u8", (4, [1, 2, 4, 8])), ("pair_dot_f64", (2, [8, 8, 0, 0])),
                       ("fnv1a_bytes", (1, [1, 0, 0, 0])), ("polar_f64", (0, [0, 0, 0, 0]))):
        _abi.check(L.fbr_body_items_streams(registry.spec(name).func_id, ctypes.byref(n), sizes))
        assert (n.value, list(sizes)) == want, name
    spec = registry.spec("mix4_u1_u2_u4_u8")
    assert spec.flags & _abi.FBR_BODY_ITEMS and spec.flags & _abi.FBR_BODY_BROADCAST
    assert registry.spec("sorted_common_u32").flags & _abi.FBR_BODY_EMIT
    assert L.fbr_body_items_streams(10 ** 6, ctypes.byref(n), sizes) == _abi.FBR_EINVAL


def test_header_constants_match_abi():
    with open(os.path.join(ROOT, "include", "fiber_b200.h")) as fh:
        h = fh.read()
    assert int(re.search(r"#define FBR_BODY_MODULE_ABI (\d+)", h).group(1)) == _abi.FBR_BODY_MODULE_ABI
    assert "uint32_t more_item_bytes[%d];" % (_abi.MAX_ITEM_STREAMS - 1) in h
    for sym in ("fbr_map_submit_items_n", "fbr_body_items_streams"):
        assert sym in h and sym in _abi.SYMBOLS


def test_submit_stream_checks():
    L = _abi.load()
    d, its, seq = _abi.MapDesc(), (_abi.ItemsDesc * 4)(), ctypes.c_uint64()
    d.func_id, d.n_tasks = registry.spec("intersect_count_u32").func_id, 1
    # checked before the pool is looked at: a NULL pool still gets the stream errors
    assert L.fbr_map_submit_items(None, ctypes.byref(d), its, ctypes.byref(seq)) == _abi.FBR_EINVAL
    assert L.fbr_map_submit_items_n(ctypes.c_void_p(1), ctypes.byref(d), its, 1, ctypes.byref(seq)) == _abi.FBR_EINVAL
    assert "takes 2 item streams, not 1" in L.fbr_last_error().decode()
    assert L.fbr_map_submit_items_n(ctypes.c_void_p(1), ctypes.byref(d), its, 3, ctypes.byref(seq)) == _abi.FBR_EINVAL
    assert "takes 2 item streams, not 3" in L.fbr_last_error().decode()
    offs = np.array([0, 1], np.uint64)
    vals = np.array([5], np.uint32)
    for it in its[:2]:
        it.items, it.offsets, it.n_items, it.item_bytes = vals.ctypes.data, offs.ctypes.data, 1, 4
    its[1].item_bytes = 8
    assert L.fbr_map_submit_items_n(ctypes.c_void_p(1), ctypes.byref(d), its, 2, ctypes.byref(seq)) == _abi.FBR_EINVAL
    assert "stream 1: item_bytes 8 does not match body intersect_count_u32 (4)" in L.fbr_last_error().decode()
    its[1].item_bytes = 4
    bad = np.array([1, 0], np.uint64)
    its[1].offsets = bad.ctypes.data
    assert L.fbr_map_submit_items_n(ctypes.c_void_p(1), ctypes.byref(d), its, 2, ctypes.byref(seq)) == _abi.FBR_EINVAL
    assert "stream 1: offsets decrease at task 0" in L.fbr_last_error().decode()
    past = np.array([0, 2], np.uint64)
    its[1].offsets = past.ctypes.data
    assert L.fbr_map_submit_items_n(ctypes.c_void_p(1), ctypes.byref(d), its, 2, ctypes.byref(seq)) == _abi.FBR_EINVAL
    assert "stream 1: offsets[1] = 2 is past n_items 1" in L.fbr_last_error().decode()
    its[1].offsets, its[1].items = offs.ctypes.data, None
    assert L.fbr_map_submit_items_n(ctypes.c_void_p(1), ctypes.byref(d), its, 2, ctypes.byref(seq)) == _abi.FBR_EINVAL
    assert "stream 1: items is NULL" in L.fbr_last_error().decode()


def test_register_items_lists():
    path, entry = registry.module_of("intersect_count_u32")[:2]

    def reg(name, items, **kw):
        return registry.register_module(name, path, entry, args=None, result=M.COUNT_RES, items=items, **kw)

    assert registry.module_of("intersect_count_u32")[6] == (("a", np.dtype("<u4")), ("b", np.dtype("<u4")))
    assert reg("intersect_count_u32", [("a", "<u4"), ("b", "<u4")]) is registry.spec("intersect_count_u32")
    with pytest.raises(ValueError, match="items= describes 1 item stream, the body takes 2"):
        reg("intersect_count_u32", [("a", "<u4")])
    with pytest.raises(ValueError, match="items= describes 1 item stream, the body takes 2"):
        reg("intersect_count_u32", ("a", "<u4"))
    with pytest.raises(ValueError, match="items= describes 3 item streams, the body takes 2"):
        reg("intersect_count_u32", [("a", "<u4"), ("b", "<u4"), ("c", "<u4")])
    with pytest.raises(ValueError, match="item dtype uint16 is 2 bytes, the body's stream 1 item is 4"):
        reg("intersect_count_u32", [("a", "<u4"), ("b", "<u2")])
    with pytest.raises(ValueError, match="the items parameter 'a' is also another parameter"):
        reg("intersect_count_u32", [("a", "<u4"), ("a", "<u4")])
    with pytest.raises(ValueError, match="list of \\(<parameter name>, <element dtype>\\) pairs"):
        reg("intersect_count_u32", [("a", "<u4"), "b"])
    mpath, mentry = registry.module_of("mix4_u1_u2_u4_u8")[:2]
    with pytest.raises(ValueError, match="the items parameter 'w' is also another parameter"):
        registry.register_module("mix4_u1_u2_u4_u8", mpath, mentry, args=M.MIX_ARG, result=M.MIX_RES, shared=("w", "<u4"),
                                 items=[("x0", "u1"), ("w", "<u2"), ("x2", "<u4"), ("x3", "<u8")])
    with pytest.raises(ValueError, match="the items parameter 'seed' is also another parameter"):
        registry.register_module("mix4_u1_u2_u4_u8", mpath, mentry, args=M.MIX_ARG, result=M.MIX_RES, shared=("w", "<u4"),
                                 items=[("x0", "u1"), ("x1", "<u2"), ("seed", "<u4"), ("x3", "<u8")])
    # the one-stream form is unchanged and takes a one-pair list too
    fnv = registry.spec("fnv1a_bytes")
    fpath, fentry = registry.module_of("fnv1a_bytes")[:2]
    one = registry.register_module("fnv1a_bytes", fpath, fentry, args=None, result=fnv.res_dtype, items=[(fnv.item_name, "u1")])
    assert one is fnv and fnv.item_names == (fnv.item_name,) and registry.module_of("fnv1a_bytes")[6] == (fnv.item_name, np.dtype("u1"))


def test_encoders_bind_every_stream():
    spec = registry.spec("intersect_count_u32")
    a, b = [np.array([1, 2], np.uint32), np.array([], np.uint32)], [[2, 3, 4], [7]]
    enc = spec.encode_starmap(list(zip(a, b)))
    assert enc.n == 2 and len(enc.streams) == 2
    assert enc.streams[0][0].tolist() == [1, 2] and enc.streams[0][1].tolist() == [0, 2, 2]
    assert enc.streams[1][0].tolist() == [2, 3, 4, 7] and enc.streams[1][1].tolist() == [0, 3, 4]
    assert enc.items is enc.streams[0]
    ka = spec.encode_apply((), {"a": [5], "b": [5, 6]})
    assert [s[0].tolist() for s in ka.streams] == [[5], [5, 6]] and ka.n == 1
    with pytest.raises(TypeError, match="intersect_count_u32\\(\\) missing 1 required positional argument: 'b'"):
        spec.encode_map([[1, 2]])
    with pytest.raises(TypeError, match="missing 2 required positional arguments: 'a' and 'b'"):
        spec.encode_apply((), {})
    with pytest.raises(TypeError, match="takes 2 positional arguments but more were given"):
        spec.encode_starmap([([1], [2], [3])])
    with pytest.raises(TypeError, match="not convertible"):
        spec.encode_starmap([([1.5], [2])])
    # four streams, a head record and a broadcast array in the tasks
    mix = registry.spec("mix4_u1_u2_u4_u8")
    w = np.arange(4, dtype=np.uint32)
    none = np.zeros(0, np.uint16)
    e = mix.encode_starmap([(w, b"ab", [1, 2], [3], np.zeros(0, np.uint64), 9), (w, "c", none, [4, 5], [6], 10)])
    assert [s[0].dtype.itemsize for s in e.streams] == [1, 2, 4, 8]
    assert e.streams[0][0].tobytes() == b"abc" and e.args["seed"].tolist() == [9, 10] and e.shared == w.tobytes()
    ek = mix.encode_apply((w,), {"x3": [1], "x2": [2], "x1": [3], "x0": b"", "seed": 4})
    assert [s[0].tolist() for s in ek.streams] == [[], [3], [2], [1]] and ek.args["seed"].tolist() == [4]


def test_columns():
    ra = Ragged(np.arange(10, dtype=np.uint32), np.array([0, 3, 3, 7, 10]))
    rb = Ragged(np.arange(6, dtype=np.uint32), np.array([0, 1, 2, 4, 6], np.uint64))
    with pytest.raises(ValueError, match="column 1 has 3 entries, column 0 has 4"):
        Columns(ra, rb[:3])
    with pytest.raises(ValueError, match="at least one column"):
        Columns()
    c = Columns(ra, rb)
    assert len(c) == 4 and [x.tolist() for x in c[2]] == [[3, 4, 5, 6], [2, 3]]
    assert [[x.tolist() for x in t] for t in c][1] == [[], [1]]
    # zero copy: the Ragged arrays themselves reach the encoder, so their data pointers reach the descriptor
    enc = registry.spec("intersect_count_u32").encode_starmap(c)
    assert enc.n == 4
    assert enc.streams[0][0].ctypes.data == ra.values.ctypes.data and enc.streams[1][0].ctypes.data == rb.values.ctypes.data
    assert enc.streams[0][1].ctypes.data == ra.offsets.ctypes.data and enc.streams[1][1].ctypes.data == rb.offsets.ctypes.data
    s = c[1:3]
    assert isinstance(s, Columns) and len(s) == 2
    assert s.columns[0].offsets.tolist() == [0, 0, 4] and s.columns[0].values.tolist() == [3, 4, 5, 6]
    back = pickle.loads(pickle.dumps(s))
    assert isinstance(back, Columns) and [[x.tolist() for x in t] for t in back] == [[x.tolist() for x in t] for t in s]
    # a head-record column and a Columns of the wrong width
    mix = registry.spec("mix4_u1_u2_u4_u8")
    cols = [Ragged(np.zeros(2, d), np.array([0, 1, 2])) for d in (np.uint8, np.uint16, np.uint32, np.uint64)]
    e = mix.encode_starmap(Columns(*cols, [7, 8]))
    assert e.n == 2 and e.args["seed"].tolist() == [7, 8] and e.shared is None
    with pytest.raises(TypeError, match="takes 5 arguments after the broadcast parameter, got 4 columns"):
        mix.encode_starmap(Columns(*cols))


class _Spec:
    def __init__(self, name):
        self.name, self.result_bytes, self.flags = name, 8, 0x4

    def result_dtype(self):
        return np.dtype(np.int64), ()

    def to_python(self, row):
        return row.item()

    def rows_to_list(self, arr):
        return arr.tolist()


def test_process_pool_ships_columns_blocks():
    """Each block's payload is the pickled slice of the Columns (a Ragged column rebased); the stand-in worker answers
    column 0's value per task, so the results show every block arrived whole and in place."""
    pool = ProcessPool(2, devices=[0, 1], results="bytes", worker_main=fake_worker_main, block_tasks=BLOCK_ALIGN)
    try:
        n = 3 * BLOCK_ALIGN + 77
        rg = Ragged(np.arange(2 * n, dtype=np.uint32), np.arange(0, 2 * n + 1, 2))
        r = pool.submit(_Spec("identity_i64"), None, "starmap", Columns(np.arange(n, dtype=np.int64), rg), 32).get(60)
        assert np.array_equal(np.asarray(r), np.arange(n)) and pool.stats["blocks_dispatched"] >= 4
    finally:
        pool.terminate()
        pool.join()
