"""The placement matrix: maps whose exact side effects -- copies, launches, waves and result bytes -- pin where the engine
puts each block's arguments and results.

Every map runs alone on a one-worker pool, through the C ABI, so any map flag can be set.  ``run_map`` returns what the
map did to the pool's counters (``STATS``), the result's wave count and a fingerprint of every result byte the map
produced (results, values of an emit map, records and counts of a keyed fold).  tests/golden/make_placement_stats.py
writes these for every case into tests/golden/placement_stats.json, and tests/test_placement_stats_gpu.py checks that
every case still does exactly that.
"""
import ctypes
from collections import namedtuple

import numpy as np

import fiber_b200
from fiber_b200 import _abi, registry

from . import broadcast_bodies as BB
from . import emit_bodies as EB
from . import fold_bodies  # noqa: F401 -- registers sum_sq_idx_u64
from . import keyed_bodies  # noqa: F401 -- registers label_sum_u64
from . import multi_items_bodies as MI
from . import scan_bodies as SB

STATS = ("units_dispatched", "dispatch_launches", "gather_launches", "fill_launches", "h2d_bytes", "d2h_bytes", "gather_bytes",
         "dispatch_bytes", "records_copied", "direct_waves", "peer_push_bytes", "units_redispatched")

SMALL_RING = 1 << 20
GOLDEN = "placement_stats.json"

F = {"direct": 0, "ring": _abi.FBR_VIA_RING, "shuffle": _abi.FBR_SHUFFLE, "resilient": _abi.FBR_RESILIENT,
     "full_window": _abi.FBR_FULL_WINDOW, "on_device": _abi.FBR_RESULTS_ON_DEVICE, "out0": _abi.FBR_OUT_DEVICE,
     "out4": _abi.FBR_OUT_DEVICE, "args_dev": _abi.FBR_ARGS_DEVICE, "no_zero_copy": _abi.FBR_NO_ZERO_COPY,
     "sum": _abi.FBR_WANT_SUM}


class Case(namedtuple("Case", "body inputs place ring pool_flags kind n_keys")):
    """body: the body name; inputs: a key of INPUTS; place: "+"-joined keys of F; ring: the pool's ring_bytes (0: the
    default); pool_flags: fbr_pool_create flags; kind: "map", "fold", "scan" or "keyed"."""

    @property
    def id(self):
        return "%s:%s:%s:ring=%dK%s" % (self.body, self.inputs, self.place, (self.ring or 256 << 20) >> 10,
                                       ":overlap" if self.pool_flags & _abi.FBR_POOL_OVERLAP else "")

    @property
    def flags(self):
        f = {"map": 0, "fold": _abi.FBR_FOLD, "scan": _abi.FBR_SCAN, "keyed": _abi.FBR_FOLD_KEYS}[self.kind]
        for k in self.place.split("+"):
            f |= F[k]
        return f

    @property
    def out_offset(self):
        return 4 if "out4" in self.place.split("+") else 0


def _case(body, inputs, place="direct", ring=0, pool_flags=0, kind="map", n_keys=0):
    return Case(body, inputs, place, ring, pool_flags, kind, n_keys)


# ---- inputs: name -> (encoded map, whether its shared block is passed by handle) -------------------------------------------
def _pi(n):
    return registry.Encoded(n, index_start=0, index_step=1)


def _pi_bits(n):
    return registry.spec("pi_inside_bits8").from_encoded(_pi(n))


def _payload(n):
    from oracle import cref
    return registry.Encoded(n, args=np.ascontiguousarray(cref.payload_records(7, n)), arg_stride=4096)


def _table(n, handle):
    enc = registry.Encoded(n, args=np.arange(n, dtype=np.int64), arg_stride=8)
    enc.shared = BB.table(5000, seed=1).tobytes()
    return enc, handle


def _columns(spec, *cols):
    return registry.spec(spec).encode_starmap(fiber_b200.Columns(*cols))


def _labels(n, keys):
    rng = np.random.default_rng(5)
    return rng.integers(0, keys, n, dtype=np.uint32), rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)


def _affine(n):
    rng = np.random.default_rng(6)
    xs = np.zeros(n, SB.AFFINE_ARG)
    xs["a"] = rng.uniform(0.5, 1.0, n)
    xs["b"] = rng.standard_normal(n)
    return registry.spec("affine_f64").encode_map(xs)


INPUTS = {
    "pi_3m": lambda: (_pi(3_000_001), False),
    "pi_bits_9m": lambda: (_pi_bits(9_000_003), False),
    "payload_1000": lambda: (_payload(1000), False),
    "table_host_200k": lambda: _table(200_003, False),
    "table_handle_200k": lambda: _table(200_003, True),
    "pairs_30k": lambda: (_columns("intersect_count_u32", MI.sorted_lists(30_011, 1), MI.sorted_lists(30_011, 2)), False),
    "docs_20k": lambda: (registry.spec("tokens_u32").encode_map(EB.documents(20_000, seed=3, empty_every=7)), False),
    "factors_50k": lambda: (registry.spec("prime_factors_i64").encode_map(range(2, 50_002)), False),
    "sum_sq_300k": lambda: (registry.spec("sum_sq_idx_u64").encode_map(np.arange(300_007, dtype=np.int64)), False),
    "affine_100k": lambda: (_affine(100_003), False),
    "labels_200k": lambda: (_columns("label_sum_u64", *_labels(200_009, 37)), False),
}


def _build():
    C = []
    for place in ("direct", "ring", "shuffle", "resilient", "full_window", "on_device", "out0", "out4", "no_zero_copy", "sum",
                  "ring+sum"):
        C.append(_case("pi_inside_det", "pi_3m", place))
        C.append(_case("pi_inside_det", "pi_3m", place, ring=SMALL_RING))
    for place in ("direct", "ring", "shuffle", "resilient", "full_window", "on_device", "out0", "no_zero_copy", "sum"):
        C.append(_case("pi_inside_bits8", "pi_bits_9m", place))
    for place in ("direct", "ring", "shuffle", "resilient", "full_window", "on_device", "out0", "out4", "args_dev",
                  "args_dev+ring", "args_dev+resilient", "no_zero_copy"):
        C.append(_case("payload_map_4k", "payload_1000", place, ring=8 << 20))
    C.append(_case("payload_map_4k", "payload_1000", "direct"))
    for place in ("ring", "full_window", "direct"):
        C.append(_case("pi_inside_det", "pi_3m", place, ring=SMALL_RING, pool_flags=_abi.FBR_POOL_OVERLAP))
        C.append(_case("payload_map_4k", "payload_1000", place, ring=8 << 20, pool_flags=_abi.FBR_POOL_OVERLAP))
    C.append(_case("intersect_count_u32", "pairs_30k", "ring", ring=SMALL_RING, pool_flags=_abi.FBR_POOL_OVERLAP))
    for inp in ("table_host_200k", "table_handle_200k"):
        for place in ("direct", "ring", "resilient", "on_device"):
            C.append(_case("table_mix_u32", inp, place, ring=SMALL_RING))
    C.append(_case("table_mix_u32", "table_handle_200k", "args_dev", ring=SMALL_RING))
    for place in ("direct", "ring", "shuffle", "resilient", "full_window", "on_device", "args_dev"):
        C.append(_case("intersect_count_u32", "pairs_30k", place, ring=SMALL_RING))
    for place in ("direct", "ring", "resilient", "full_window", "on_device", "args_dev"):
        C.append(_case("tokens_u32", "docs_20k", place, ring=SMALL_RING))
    for place in ("direct", "on_device", "full_window"):
        C.append(_case("prime_factors_i64", "factors_50k", place, ring=SMALL_RING))
    for place in ("direct", "ring", "shuffle", "resilient", "args_dev"):
        C.append(_case("sum_sq_idx_u64", "sum_sq_300k", place, ring=SMALL_RING, kind="fold"))
    for place in ("direct", "ring", "resilient", "on_device", "args_dev"):
        C.append(_case("affine_f64", "affine_100k", place, ring=SMALL_RING, kind="scan"))
    for place in ("direct", "ring", "shuffle", "resilient", "args_dev"):
        C.append(_case("label_sum_u64", "labels_200k", place, ring=8 << 20, kind="keyed", n_keys=37))
    return C


CASES = _build()
BY_ID = {c.id: c for c in CASES}
assert len(BY_ID) == len(CASES)


# ---- running a case --------------------------------------------------------------------------------------------------------
class RawPool:
    """A one-worker engine pool on device 0 with the given ring_bytes and fbr_pool_create flags."""

    def __init__(self, ring, flags):
        self.lib = _abi.load()
        ids = (ctypes.c_int * 1)(0)
        self.handle = ctypes.c_void_p()
        _abi.check(self.lib.fbr_pool_create(1, ids, ring, flags, ctypes.byref(self.handle)))

    def stats(self):
        s = _abi.Stats()
        _abi.check(self.lib.fbr_pool_stats(self.handle, ctypes.byref(s)))
        return s.as_dict()

    def alloc(self, nbytes):
        p = ctypes.c_void_p()
        _abi.check(self.lib.fbr_device_alloc(self.handle, 0, max(16, nbytes) + 64, ctypes.byref(p)))
        return p

    def h2d(self, arr):
        a = np.ascontiguousarray(arr)
        p = self.alloc(a.nbytes)
        if a.nbytes:
            _abi.check(self.lib.fbr_memcpy_h2d(self.handle, 0, p, a.ctypes.data, a.nbytes))
        return p

    def close(self):
        self.lib.fbr_pool_destroy(self.handle)


def run_map(pool, c):
    """Run case c on pool (a RawPool of c.ring and c.pool_flags).  Returns (stats delta over STATS, n_waves, hex
    fingerprint of the result bytes)."""
    lib, h = pool.lib, pool.handle
    enc, by_handle = INPUTS[c.inputs]()
    spec = registry.spec(c.body)
    R = spec.result_bytes
    flags = c.flags
    args_dev = bool(flags & _abi.FBR_ARGS_DEVICE)
    dev, keep = [], [enc]
    before = pool.stats()
    d = _abi.MapDesc()
    d.func_id, d.flags, d.n_tasks, d.chunksize, d.shuffle_seed = spec.func_id, flags, enc.n, 0 if c.kind != "map" else 32, 0x5EED
    d.arg_stride, d.index_start, d.index_step, d.n_items, d.task_index_base = (enc.arg_stride, enc.index_start, enc.index_step,
                                                                               enc.n_items, enc.task_index_base)
    d.n_keys = c.n_keys
    if enc.args is not None and enc.n:
        if args_dev:
            dev.append(pool.h2d(enc.args))
            d.args = dev[-1].value
        else:
            d.args = enc.args.ctypes.data
    shared_handle = None
    if enc.shared is not None:
        blob = np.frombuffer(enc.shared, np.uint8)
        keep.append(blob)
        if by_handle:
            hv = ctypes.c_uint64()
            _abi.check(lib.fbr_shared_put(h, blob.ctypes.data, blob.nbytes, ctypes.byref(hv)))
            shared_handle = hv.value
            d.shared = shared_handle
            d.flags |= _abi.FBR_SHARED_HANDLE
        else:
            d.shared = blob.ctypes.data
        d.shared_bytes = blob.nbytes
    out = None
    if flags & _abi.FBR_OUT_DEVICE:
        dev.append(pool.alloc(enc.n * R))
        out = dev[-1].value + c.out_offset
        d.out = out
    seq = ctypes.c_uint64()
    try:
        if enc.streams is not None:
            streams = (_abi.ItemsDesc * len(enc.streams))()
            for it, (values, offsets) in zip(streams, enc.streams):
                if args_dev:
                    dev += [pool.h2d(values), pool.h2d(offsets)]
                    it.items, it.offsets = dev[-2].value, dev[-1].value
                else:
                    it.items, it.offsets = values.ctypes.data, offsets.ctypes.data
                it.n_items, it.item_bytes = len(values), values.dtype.itemsize
            _abi.check(lib.fbr_map_submit_items_n(h, ctypes.byref(d), streams, len(streams), ctypes.byref(seq)))
        else:
            _abi.check(lib.fbr_map_submit(h, ctypes.byref(d), ctypes.byref(seq)))
        res = _abi.Result()
        try:
            _abi.check(lib.fbr_result_wait(h, seq.value, -1, ctypes.byref(res)))
            parts = [int(res.sum).to_bytes(8, "little", signed=True)] if flags & _abi.FBR_WANT_SUM else []
            if c.kind == "fold":
                parts.append(ctypes.string_at(res.data, R))
            elif c.kind == "keyed":
                parts.append(ctypes.string_at(res.data, c.n_keys * (R + 8)))
            else:
                data = np.zeros(enc.n * R, np.uint8)
                if out is not None:
                    _abi.check(lib.fbr_memcpy_d2h(h, 0, data.ctypes.data, ctypes.c_void_p(out), data.nbytes))
                elif flags & _abi.FBR_RESULTS_ON_DEVICE:
                    _abi.check(lib.fbr_result_fetch(h, seq.value, 0, enc.n, data.ctypes.data))
                else:
                    ctypes.memmove(data.ctypes.data, res.data, data.nbytes)
                parts.append(data.tobytes())
                if spec.flags & _abi.FBR_BODY_EMIT:
                    vp, nv = ctypes.c_void_p(), ctypes.c_uint64()
                    _abi.check(lib.fbr_result_values(h, seq.value, ctypes.byref(vp), ctypes.byref(nv)))
                    vals = np.zeros(nv.value * spec.out_dtype.itemsize, np.uint8)
                    if flags & _abi.FBR_RESULTS_ON_DEVICE:
                        _abi.check(lib.fbr_result_fetch_values(h, seq.value, 0, nv.value, vals.ctypes.data))
                    elif vals.nbytes:
                        ctypes.memmove(vals.ctypes.data, vp.value, vals.nbytes)
                    parts.append(vals.tobytes())
            n_waves = int(res.n_waves)
        finally:
            _abi.check(lib.fbr_result_release(h, seq.value))
    finally:
        if shared_handle is not None:
            lib.fbr_shared_drop(h, shared_handle)
        for p in dev:
            lib.fbr_device_free(h, 0, p)
    after = pool.stats()
    return {k: after[k] - before[k] for k in STATS}, n_waves, registry.fingerprint(b"".join(parts)).hex()


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def run_all(cases=CASES):
    """{case id: {"stats": ..., "n_waves": ..., "fingerprint": ...}} of every case, one pool per (ring, pool flags)."""
    pools, out = {}, {}
    try:
        for c in cases:
            key = (c.ring, c.pool_flags)
            if key not in pools:
                pools[key] = RawPool(c.ring, c.pool_flags)
            st, waves, fp = run_map(pools[key], c)
            out[c.id] = {"stats": st, "n_waves": waves, "fingerprint": fp}
    finally:
        for p in pools.values():
            p.close()
    return out
