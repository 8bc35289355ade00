"""Items record bodies: every task also takes one variable-length array (``using Item = ...`` in the body's struct).

Each CUDA source below is compiled by ``fiber_b200.device_body(name, source=..., items=..., result=...)`` and registered at
import time.  Next to each body: its Python definition (what the reference would run) and a NumPy / Python restatement
the GPU results are compared against bit for bit.  Where a body reduces across its lanes, the restatement repeats the
device's order exactly: lane ``rank`` takes items ``rank, rank + G, ...`` in sequence with explicitly rounded adds, then
the lanes combine in an xor butterfly with offsets G/2, ..., 1 (as in ``group_bodies.py``).
"""
import numpy as np

import fiber_b200
import fiber_b200.bodies

FNV_RES = np.dtype([("h", "<u8"), ("n", "<u4"), ("pad", "<u4")])

FNV_SRC = r'''
#include "fiber_b200_body.cuh"

// FNV-1a 64 of a byte string, and its length
struct Fnv1a {
    using Item = uint8_t;
    using Arg = fbr::NoArg;
    struct Res { uint64_t h; uint32_t n, pad; };
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static __forceinline__ void run(const fbr::Items<Item>& x, Res& r, uint64_t, const fbr::ErrSink&, uint32_t) {
        uint64_t h = 0xcbf29ce484222325ull;
        for (uint64_t k = 0; k < x.n; ++k) h = (h ^ x.data[k]) * 0x100000001b3ull;
        r.h = h; r.n = (uint32_t)x.n; r.pad = 0;
    }
};
FBR_EXPORT_RECORD_BODY(Fnv1a, "fnv1a_bytes", fnv1a_entry, 0)

// the same, but a string whose first byte is 0xFF "kills its worker" on the first attempt: the unit is re-dispatched
struct FaultFnv1a {
    using Item = uint8_t;
    using Arg = fbr::NoArg;
    using Res = Fnv1a::Res;
    static constexpr bool kIndexArg = false, kCanFault = true;
    __device__ static __forceinline__ void run(const fbr::Items<Item>& x, Res& r, uint64_t gidx, const fbr::ErrSink& es,
                                               uint32_t attempt) {
        if (attempt == 0 && x.n > 0 && x.data[0] == 0xFF) es.report(fbr::TASK_FAULT, gidx);
        Fnv1a::run(x, r, gidx, es, attempt);
    }
};
FBR_EXPORT_RECORD_BODY(FaultFnv1a, "fault_fnv1a_bytes", fault_fnv1a_entry, 0)
'''

STATS_RES = np.dtype([("sum", "<f8"), ("min", "<f8"), ("max", "<f8"), ("n", "<u8")])

STATS_SRC = r'''
#include "fiber_b200_body.cuh"

// a row of float64 -> (sum, min, max, n) on a warp: lane k sums x[k], x[k + 32], ... in order, then the lanes add in an
// xor butterfly (offsets 16 .. 1).  An empty row gives (0, inf, -inf, 0)
struct RaggedStats {
    using Item = double;
    using Arg = fbr::NoArg;
    struct Res { double sum, mn, mx; uint64_t n; };
    static constexpr uint32_t kGroup = 32;
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static __forceinline__ void run(const fbr::Items<Item>& x, Res& r, const fbr::Group<32>& g, uint64_t,
                                               const fbr::ErrSink&, uint32_t) {
        double s = 0.0, mn = INFINITY, mx = -INFINITY;
        for (uint64_t k = g.rank; k < x.n; k += g.size) {
            const double v = x.data[k];
            s = __dadd_rn(s, v);
            mn = fmin(mn, v);
            mx = fmax(mx, v);
        }
#pragma unroll
        for (uint32_t o = g.size / 2; o > 0; o >>= 1) {
            s = __dadd_rn(s, __shfl_xor_sync(g.mask, s, o));
            mn = fmin(mn, __shfl_xor_sync(g.mask, mn, o));
            mx = fmax(mx, __shfl_xor_sync(g.mask, mx, o));
        }
        if (g.rank == 0) { r.sum = s; r.mn = mn; r.mx = mx; r.n = x.n; }
    }
};
FBR_EXPORT_RECORD_BODY(RaggedStats, "ragged_stats_f64", ragged_stats_entry, 0)
'''

CLIP_ARG = np.dtype([("lo", "<f4"), ("hi", "<f4")])
CLIP_RES = np.dtype([("s", "<f4"), ("n", "<u4")])

CLIP_SRC = r'''
#include "fiber_b200_body.cuh"

// (row, lo, hi) -> sum of the row clipped to [lo, hi], left to right in float32, and its length
struct ClipSum {
    using Item = float;
    struct Arg { float lo, hi; };
    struct Res { float s; uint32_t n; };
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static __forceinline__ void run(const Arg& a, const fbr::Items<Item>& x, Res& r, uint64_t, const fbr::ErrSink&,
                                               uint32_t) {
        float s = 0.0f;
        for (uint64_t k = 0; k < x.n; ++k) s = __fadd_rn(s, fminf(fmaxf(x.data[k], a.lo), a.hi));
        r.s = s; r.n = (uint32_t)x.n;
    }
};
FBR_EXPORT_RECORD_BODY(ClipSum, "clip_sum_f32", clip_sum_entry, 0)
'''

TOKEN_RES = np.dtype([("w", "<f4"), ("n", "<u4")])

TOKEN_SRC = r'''
#include "fiber_b200_body.cuh"

// (weights, tokens) -> sum of weights[token] left to right in float32, and the number of tokens.  A token id past the
// weight table is a bad argument
struct TokenWeight {
    using Item = uint32_t;
    using Shared = float;
    static constexpr uint32_t kSharedStage = 16384;
    using Arg = fbr::NoArg;
    struct Res { float w; uint32_t n; };
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static __forceinline__ void run(const fbr::Items<Item>& x, Res& r, const fbr::Broadcast<Shared>& table,
                                               uint64_t gidx, const fbr::ErrSink& es, uint32_t) {
        float s = 0.0f;
        for (uint64_t k = 0; k < x.n; ++k) {
            const uint32_t t = x.data[k];
            if (t >= table.n) { es.report(fbr::TASK_BADARG, gidx); return; }
            s = __fadd_rn(s, table.data[t]);
        }
        r.w = s; r.n = (uint32_t)x.n;
    }
};
FBR_EXPORT_RECORD_BODY(TokenWeight, "token_weight_u32", token_weight_entry, 0)
'''

# The workaround an items body replaces: rows padded to a fixed length, one group record body over the padded records
PADDED_LEN = 1023
PADDED_ARG = np.dtype([("x", "<f8", (PADDED_LEN,)), ("n", "<u8")])

PADDED_SRC = r'''
#include "fiber_b200_body.cuh"

// ragged_stats_f64 over a row padded to 1023 float64 with its length in the last word
struct PaddedStats {
    struct Arg { double x[1023]; uint64_t n; };
    struct Res { double sum, mn, mx; uint64_t n; };
    static constexpr uint32_t kGroup = 32;
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static __forceinline__ void run(const Arg& a, Res& r, const fbr::Group<32>& g, uint64_t, const fbr::ErrSink&,
                                               uint32_t) {
        double s = 0.0, mn = INFINITY, mx = -INFINITY;
        const uint64_t n = a.n;
        for (uint64_t k = g.rank; k < n; k += g.size) {
            const double v = a.x[k];
            s = __dadd_rn(s, v);
            mn = fmin(mn, v);
            mx = fmax(mx, v);
        }
#pragma unroll
        for (uint32_t o = g.size / 2; o > 0; o >>= 1) {
            s = __dadd_rn(s, __shfl_xor_sync(g.mask, s, o));
            mn = fmin(mn, __shfl_xor_sync(g.mask, mn, o));
            mx = fmax(mx, __shfl_xor_sync(g.mask, mx, o));
        }
        if (g.rank == 0) { r.sum = s; r.mn = mn; r.mx = mx; r.n = n; }
    }
};
FBR_EXPORT_RECORD_BODY(PaddedStats, "padded_stats_f64", padded_stats_entry, 0)
'''


@fiber_b200.device_body("fnv1a_bytes", source=FNV_SRC, entry="fnv1a_entry", items=("s", "u1"), result=FNV_RES)
def fnv1a_bytes(s):
    h = 0xcbf29ce484222325
    for b in s:
        h = ((h ^ b) * 0x100000001b3) & 0xFFFFFFFFFFFFFFFF
    return h, len(s), 0


@fiber_b200.device_body("fault_fnv1a_bytes", source=FNV_SRC, entry="fault_fnv1a_entry", items=("s", "u1"), result=FNV_RES)
def fault_fnv1a_bytes(s):
    return fnv1a_bytes(s)


@fiber_b200.device_body("ragged_stats_f64", source=STATS_SRC, entry="ragged_stats_entry", items=("row", "<f8"), result=STATS_RES)
def ragged_stats_f64(row):
    return float(np.sum(row)), float(np.min(row, initial=np.inf)), float(np.max(row, initial=-np.inf)), len(row)


@fiber_b200.device_body("clip_sum_f32", source=CLIP_SRC, entry="clip_sum_entry", items=("row", "<f4"), args=CLIP_ARG,
                        result=CLIP_RES)
def clip_sum_f32(row, lo, hi):
    s = np.float32(0)
    for v in np.asarray(row, np.float32):
        s = np.float32(s + min(max(v, np.float32(lo)), np.float32(hi)))
    return float(s), len(row)


@fiber_b200.device_body("token_weight_u32", source=TOKEN_SRC, entry="token_weight_entry", items=("tokens", "<u4"),
                        result=TOKEN_RES, shared=("weights", "<f4"))
def token_weight_u32(weights, tokens):
    s = np.float32(0)
    for t in tokens:
        s = np.float32(s + np.float32(weights[t]))
    return float(s), len(tokens)


@fiber_b200.device_body("padded_stats_f64", source=PADDED_SRC, entry="padded_stats_entry", args=PADDED_ARG, result=STATS_RES)
def padded_stats_f64(x, n):
    return ragged_stats_f64(x[:n])


# ---- NumPy restatements (bit for bit) ----------------------------------------------------------------------------------
FNV_OFFSET = np.uint64(0xcbf29ce484222325)
FNV_PRIME = np.uint64(0x100000001b3)


def fnv1a_np(values, offsets):
    """FNV-1a 64 and length of every byte string: one vectorised step per byte position (rows end at their lengths)."""
    values = np.asarray(values, np.uint8)
    offsets = np.asarray(offsets, np.int64)
    lens = np.diff(offsets)
    out = np.zeros(len(lens), FNV_RES)
    h = np.full(len(lens), FNV_OFFSET, np.uint64)
    if len(lens):
        for k in range(int(lens.max(initial=0))):
            live = np.nonzero(lens > k)[0]
            h[live] = (h[live] ^ values[offsets[live] + k].astype(np.uint64)) * FNV_PRIME
    out["h"], out["n"] = h, lens
    return out


def _lane_fold(vals, lens, op, init, G=32):
    """The device order of a lane-strided reduction: lane j folds items j, j + G, ... in sequence, then an xor butterfly."""
    n_rows = len(lens)
    acc = np.full((n_rows, G), init, np.float64)
    width = int(lens.max(initial=0))
    for k in range(width):
        live = np.nonzero(lens > k)[0]
        acc[live, k % G] = op(acc[live, k % G], vals[live, k])
    o = G // 2
    while o:
        acc = op(acc, acc[:, np.arange(G) ^ o])
        o //= 2
    return acc[:, 0]


def ragged_stats_np(values, offsets):
    values = np.asarray(values, np.float64)
    offsets = np.asarray(offsets, np.int64)
    lens = np.diff(offsets)
    width = max(int(lens.max(initial=0)), 1)
    idx = offsets[:-1, None] + np.arange(width)[None, :]
    mask = np.arange(width)[None, :] < lens[:, None]
    vals = np.where(mask, values[np.minimum(idx, max(len(values) - 1, 0))] if len(values) else 0.0, 0.0)
    out = np.zeros(len(lens), STATS_RES)
    out["sum"] = _lane_fold(vals, lens, np.add, 0.0)
    out["min"] = _lane_fold(vals, lens, np.fmin, np.inf)
    out["max"] = _lane_fold(vals, lens, np.fmax, -np.inf)
    out["n"] = lens
    return out


def clip_sum_np(values, offsets, lo, hi):
    values = np.asarray(values, np.float32)
    offsets = np.asarray(offsets, np.int64)
    lens = np.diff(offsets)
    lo, hi = np.asarray(lo, np.float32), np.asarray(hi, np.float32)
    s = np.zeros(len(lens), np.float32)
    for k in range(int(lens.max(initial=0))):
        live = np.nonzero(lens > k)[0]
        s[live] = s[live] + np.fmin(np.fmax(values[offsets[live] + k], lo[live]), hi[live])
    out = np.zeros(len(lens), CLIP_RES)
    out["s"], out["n"] = s, lens
    return out


def token_weight_np(weights, values, offsets):
    weights = np.asarray(weights, np.float32)
    values = np.asarray(values, np.int64)
    offsets = np.asarray(offsets, np.int64)
    lens = np.diff(offsets)
    s = np.zeros(len(lens), np.float32)
    for k in range(int(lens.max(initial=0))):
        live = np.nonzero(lens > k)[0]
        s[live] = s[live] + weights[values[offsets[live] + k]]
    out = np.zeros(len(lens), TOKEN_RES)
    out["w"], out["n"] = s, lens
    return out


# Hand-written descriptors that break the items rules; registration must refuse every one of them except ok_items.
# (FBR_EXPORT_RECORD_BODY derives the flags and fields from the struct, so a real body cannot get there.)
BAD_SRC = r'''
#include "fiber_b200_body.cuh"

#define BAD_ITEMS(entry, name, flags, arg_bytes, unit, item)                                                \
    extern "C" const fbr_body_module_t* entry(void) {                                                            \
        static const fbr_body_module_t m = {FBR_BODY_MODULE_ABI, (uint32_t)sizeof(fbr::WaveParams), name, (arg_bytes), \
                                            16u, FBR_RES_BYTES, (flags), (unit),                                 \
                                            fbr_body_export::launch_record<Fnv1aLike>,                           \
                                            fbr_body_export::occupancy_record<Fnv1aLike>, 0u, 0u, 0u, (item)};     \
        return &m;                                                                                               \
    }
struct Fnv1aLike {
    using Item = uint8_t;
    using Arg = fbr::NoArg;
    struct Res { uint64_t h; uint32_t n, pad; };
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static void run(const fbr::Items<Item>& x, Res& r, uint64_t, const fbr::ErrSink&, uint32_t) { r.n = (uint32_t)x.n; }
};
#define REC FBR_BODY_RECORD
#define IT (FBR_BODY_RECORD | FBR_BODY_ITEMS)
BAD_ITEMS(bad_items_fields, "bad_items_fields", REC, 4u, 16u, 1u)              // an item size without the flag
BAD_ITEMS(bad_items_thread, "bad_items_thread", FBR_BODY_ITEMS, 8u, 16u, 1u)   // not a record body
BAD_ITEMS(bad_item0, "bad_item0", IT, 0u, 16u, 0u)
BAD_ITEMS(bad_item3, "bad_item3", IT, 0u, 16u, 3u)
BAD_ITEMS(bad_item_big, "bad_item_big", IT, 0u, 16u, 8192u)
BAD_ITEMS(bad_items_index, "bad_items_index", IT | FBR_BODY_INDEX_ARG, 8u, 16u, 1u)
BAD_ITEMS(bad_noarg, "bad_noarg", REC, 0u, 16u, 0u)                            // arg_bytes 0 without items
BAD_ITEMS(ok_items, "ok_items", IT, 0u, 1024u, 1u)
'''
BAD_MODULE = fiber_b200.bodies.compile_module("ragged_bad_descriptors", BAD_SRC)


# ---- seeded inputs ------------------------------------------------------------------------------------------------------
def byte_strings(n, seed, max_len=512):
    """n byte strings of seeded lengths 0 .. max_len, as (values, offsets)."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, max_len + 1, n, dtype=np.int64)
    offsets = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=offsets[1:])
    values = rng.integers(0, 256, int(offsets[-1]), dtype=np.uint8)
    return values, offsets


def lognormal_rows(n, seed, mean_len=64.0, max_len=None):
    """n float64 rows of seeded lognormal lengths, as (values, offsets)."""
    rng = np.random.default_rng(seed)
    lens = np.floor(rng.lognormal(np.log(mean_len), 1.0, n)).astype(np.int64)
    if max_len is not None:
        lens = np.minimum(lens, max_len)
    offsets = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=offsets[1:])
    values = rng.standard_normal(int(offsets[-1]))
    return values, offsets
