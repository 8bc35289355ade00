"""Fold record bodies: record bodies that also define ``identity()`` and ``combine()``, so ``Pool.fold`` reduces a whole map
to one result on the device.

Each CUDA source below is compiled by ``fiber_b200.device_body(name, source=..., ...)`` and registered at import time.  Next
to each body: a Python restatement of its ``run`` (``*_run``), its ``combine`` (``*_combine``) and the fold order ``tree``,
which the GPU results are compared against bit for bit, floats included.  Float bodies round every operation explicitly
(``__dadd_rn`` and friends), so Python floats (binary64) and NumPy float32 scalars restate them exactly.
"""
import math

import numpy as np

import fiber_b200
import fiber_b200.bodies

M64 = (1 << 64) - 1


def tree(xs, combine):
    """The fold order of FBR_FOLD: while c > 1, x[i] <- combine(x[2i], x[2i+1]) for every i with 2i+1 < c, an odd last
    element carried to x[c/2]; c <- ceil(c/2).  None for no element (the caller uses the identity)."""
    xs = list(xs)
    while len(xs) > 1:
        nxt = [combine(xs[2 * i], xs[2 * i + 1]) for i in range(len(xs) // 2)]
        if len(xs) % 2:
            nxt.append(xs[-1])
        xs = nxt
    return xs[0] if xs else None


def fold_of(results, combine, identity):
    r = tree(results, combine)
    return identity if r is None else r


# ---- moments_f64: count, mean and M2 of a float64 column (Chan et al.'s merge) ------------------------------------------
MOMENTS_RES = np.dtype([("n", "<f8"), ("mean", "<f8"), ("m2", "<f8")])

MOMENTS_SRC = r'''
#include "fiber_b200_body.cuh"

struct Moments {
    struct Arg { double x; };
    struct Res { double n, mean, m2; };
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static void run(const Arg& a, Res& r, uint64_t, const fbr::ErrSink&, uint32_t) { r = Res{1.0, a.x, 0.0}; }
    __host__ __device__ static Res identity() { return Res{0.0, 0.0, 0.0}; }
    __device__ static __forceinline__ void combine(Res& acc, const Res& x) {
        if (x.n == 0.0) return;
        if (acc.n == 0.0) { acc = x; return; }
        const double n = __dadd_rn(acc.n, x.n), d = __dsub_rn(x.mean, acc.mean);
        const double mean = __dadd_rn(acc.mean, __ddiv_rn(__dmul_rn(d, x.n), n));
        const double m2 = __dadd_rn(__dadd_rn(acc.m2, x.m2), __ddiv_rn(__dmul_rn(__dmul_rn(d, d), __dmul_rn(acc.n, x.n)), n));
        acc.n = n; acc.mean = mean; acc.m2 = m2;
    }
};
FBR_EXPORT_RECORD_BODY(Moments, "moments_f64", moments_entry, 0)

// a 2 KB row of float64 summed by a warp: lane k adds x[k], x[k + 32], ... in order, then the lanes add in an xor
// butterfly (offsets 16 .. 1); the fold adds the row sums and counts the rows
struct RowSum {
    struct Arg { double x[256]; };
    struct Res { double s, rows; };
    static constexpr uint32_t kGroup = 32;
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static void run(const Arg& a, Res& r, const fbr::Group<32>& g, uint64_t, const fbr::ErrSink&, uint32_t) {
        double s = 0.0;
        for (uint32_t k = g.rank; k < 256; k += g.size) s = __dadd_rn(s, a.x[k]);
#pragma unroll
        for (uint32_t o = g.size / 2; o > 0; o >>= 1) s = __dadd_rn(s, __shfl_xor_sync(g.mask, s, o));
        if (g.rank == 0) { r.s = s; r.rows = 1.0; }
    }
    __host__ __device__ static Res identity() { return Res{0.0, 0.0}; }
    __device__ static __forceinline__ void combine(Res& acc, const Res& x) { acc.s = __dadd_rn(acc.s, x.s); acc.rows = __dadd_rn(acc.rows, x.rows); }
};
FBR_EXPORT_RECORD_BODY(RowSum, "row_sum_f64", row_sum_entry, 0)
'''

ROW_ARG = np.dtype([("x", "<f8", (256,))])
ROW_RES = np.dtype([("s", "<f8"), ("rows", "<f8")])


@fiber_b200.device_body("moments_f64", source=MOMENTS_SRC, entry="moments_entry", args=np.dtype([("x", "<f8")]),
                        result=MOMENTS_RES)
def moments_f64(x):
    return (1.0, x, 0.0)


def moments_run(x):
    return (1.0, float(x), 0.0)


def moments_combine(a, b):
    if b[0] == 0.0:
        return a
    if a[0] == 0.0:
        return b
    n, d = a[0] + b[0], b[1] - a[1]
    return (n, a[1] + (d * b[0]) / n, (a[2] + b[2]) + ((d * d) * (a[0] * b[0])) / n)


MOMENTS_ID = (0.0, 0.0, 0.0)


@fiber_b200.device_body("row_sum_f64", source=MOMENTS_SRC, entry="row_sum_entry", args=ROW_ARG, result=ROW_RES)
def row_sum_f64(x):
    return row_sum_run(x)


def row_sum_run(x):
    lanes = [0.0] * 32
    for r in range(32):
        s = 0.0
        for k in range(r, 256, 32):
            s += float(x[k])
        lanes[r] = s
    o = 16
    while o:
        lanes = [lanes[i] + lanes[i ^ o] for i in range(32)]
        o //= 2
    return (lanes[0], 1.0)


def row_sum_combine(a, b):
    return (a[0] + b[0], a[1] + b[1])


ROW_ID = (0.0, 0.0)

# ---- integer bodies: a range() index, items with a group, two item streams, and a body that faults ---------------------
INT_SRC = r'''
#include "fiber_b200_body.cuh"

struct SumSqIdx {
    using Arg = int64_t;
    struct Res { uint64_t s; };
    static constexpr bool kIndexArg = true, kCanFault = false;
    __device__ static void run(const Arg& a, Res& r, uint64_t, const fbr::ErrSink&, uint32_t) { r.s = (uint64_t)a * (uint64_t)a; }
    __host__ __device__ static Res identity() { return Res{0}; }
    __device__ static __forceinline__ void combine(Res& acc, const Res& x) { acc.s += x.s; }
};
FBR_EXPORT_RECORD_BODY(SumSqIdx, "sum_sq_idx_u64", sum_sq_idx_entry, FBR_BODY_INDEX_ARG)

// a histogram of a byte string on a warp
struct ByteHist {
    using Item = uint8_t;
    using Arg = fbr::NoArg;
    struct Res { uint32_t c[256]; };
    static constexpr uint32_t kGroup = 32;
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static void run(const fbr::Items<uint8_t>& x, Res& r, const fbr::Group<32>& g, uint64_t, const fbr::ErrSink&, uint32_t) {
        for (uint32_t k = g.rank; k < 256; k += g.size) r.c[k] = 0;
        g.sync();
        for (uint64_t k = g.rank; k < x.n; k += g.size) atomicAdd(&r.c[x.data[k]], 1u);
        g.sync();
    }
    __host__ __device__ static Res identity() { return Res{}; }
    __device__ static __forceinline__ void combine(Res& acc, const Res& x) {
        for (uint32_t k = 0; k < 256; ++k) acc.c[k] += x.c[k];
    }
};
FBR_EXPORT_RECORD_BODY(ByteHist, "byte_hist_u8", byte_hist_entry, 0)

// the number of values two sorted uint32 lists have in common (multiset intersection), summed over the map
struct PairOverlap {
    using Items = fbr::ItemTypes<uint32_t, uint32_t>;
    using Arg = fbr::NoArg;
    struct Res { uint64_t common; };
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static void run(const fbr::Items<uint32_t>& a, const fbr::Items<uint32_t>& b, Res& r, uint64_t, const fbr::ErrSink&,
                               uint32_t) {
        uint64_t i = 0, j = 0, c = 0;
        while (i < a.n && j < b.n) {
            const uint32_t x = a.data[i], y = b.data[j];
            c += x == y;
            i += x <= y;
            j += y <= x;
        }
        r.common = c;
    }
    __host__ __device__ static Res identity() { return Res{0}; }
    __device__ static __forceinline__ void combine(Res& acc, const Res& x) { acc.common += x.common; }
};
FBR_EXPORT_RECORD_BODY(PairOverlap, "pair_overlap_u32", pair_overlap_entry, 0)

// 3 i + 1, but every task whose index is 5 mod 997 "kills its worker" on the first attempt, leaving a wrong result behind:
// only the unit's re-dispatch gives the right total
struct FaultCount {
    using Arg = int64_t;
    struct Res { uint64_t v; };
    static constexpr bool kIndexArg = true, kCanFault = true;
    __device__ static void run(const Arg& a, Res& r, uint64_t gidx, const fbr::ErrSink& es, uint32_t attempt) {
        r.v = 3u * (uint64_t)a + 1u;
        if (attempt == 0 && gidx % 997 == 5) {
            es.report(fbr::TASK_FAULT, gidx);
            r.v = 0x5eed;
        }
    }
    __host__ __device__ static Res identity() { return Res{0}; }
    __device__ static __forceinline__ void combine(Res& acc, const Res& x) { acc.v += x.v; }
};
FBR_EXPORT_RECORD_BODY(FaultCount, "fault_count_u64", fault_count_entry, FBR_BODY_INDEX_ARG)
'''


@fiber_b200.device_body("sum_sq_idx_u64", source=INT_SRC, entry="sum_sq_idx_entry", args="<i8", result="<u8")
def sum_sq_idx_u64(i):
    return (i * i) & M64


def add_u64(a, b):
    return (a + b) & M64


@fiber_b200.device_body("byte_hist_u8", source=INT_SRC, entry="byte_hist_entry", args=None, items=("x", "u1"),
                        result=np.dtype([("c", "<u4", (256,))]))
def byte_hist_u8(x):
    return np.bincount(np.frombuffer(bytes(x), np.uint8), minlength=256).astype(np.uint32).tolist()


def hist_combine(a, b):
    return [(x + y) & 0xFFFFFFFF for x, y in zip(a, b)]


HIST_ID = [0] * 256


@fiber_b200.device_body("pair_overlap_u32", source=INT_SRC, entry="pair_overlap_entry", args=None,
                        items=[("a", "<u4"), ("b", "<u4")], result="<u8")
def pair_overlap_u32(a, b):
    from collections import Counter
    return sum((Counter(np.asarray(a).tolist()) & Counter(np.asarray(b).tolist())).values())


@fiber_b200.device_body("fault_count_u64", source=INT_SRC, entry="fault_count_entry", args="<i8", result="<u8")
def fault_count_u64(i):
    return (3 * i + 1) & M64


# ---- nearest_query_f32: the point nearest a broadcast query ---------------------------------------------------------------
NEAREST_SRC = r'''
#include "fiber_b200_body.cuh"
#include <string.h>

// squared float32 distance of a 4-d point to the broadcast query (its first 4 floats), and the task's index.  The fold keeps
// the smaller d2; ties go to the lower index, and a NaN distance loses to every number
struct NearestQuery {
    struct Arg { float p[4]; };
    struct Res { float d2; uint32_t pad; uint64_t idx; };
    using Shared = float;
    static constexpr uint32_t kSharedStage = 64;
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static void run(const Arg& a, Res& r, const fbr::Broadcast<float>& q, uint64_t gidx, const fbr::ErrSink&, uint32_t) {
        float d2 = 0.0f;
        for (int k = 0; k < 4; ++k) {
            const float d = __fsub_rn(a.p[k], q.data[k]);
            d2 = __fadd_rn(d2, __fmul_rn(d, d));
        }
        r.d2 = d2; r.pad = 0; r.idx = gidx;
    }
    __host__ __device__ static Res identity() {
        Res r{0.0f, 0u, ~0ull};
        const uint32_t nan = 0x7fc00000u;
        memcpy(&r.d2, &nan, sizeof nan);
        return r;
    }
    __device__ static __forceinline__ bool before(const Res& x, const Res& y) {   // x is nearer than y
        const bool xn = x.d2 != x.d2, yn = y.d2 != y.d2;
        if (xn != yn) return yn;
        if (!xn && x.d2 != y.d2) return x.d2 < y.d2;
        return x.idx < y.idx;
    }
    __device__ static __forceinline__ void combine(Res& acc, const Res& x) { if (before(x, acc)) acc = x; }
};
FBR_EXPORT_RECORD_BODY(NearestQuery, "nearest_query_f32", nearest_query_entry, 0)
'''

NEAR_ARG = np.dtype([("p", "<f4", (4,))])
NEAR_RES = np.dtype([("d2", "<f4"), ("pad", "<u4"), ("idx", "<u8")])


@fiber_b200.device_body("nearest_query_f32", source=NEAREST_SRC, entry="nearest_query_entry", args=NEAR_ARG,
                        result=NEAR_RES, shared=("q", "<f4"))
def nearest_query_f32(q, p):
    return nearest_run(q, p, None)


def nearest_run(q, p, idx):
    d2 = np.float32(0.0)
    for k in range(4):
        d = np.float32(np.float32(p[k]) - np.float32(q[k]))
        d2 = np.float32(d2 + np.float32(d * d))
    return (float(d2), 0, idx)


def _near_key(r):
    return (math.isnan(r[0]), 0.0 if math.isnan(r[0]) else r[0], r[2])


def nearest_combine(a, b):
    return b if _near_key(b) < _near_key(a) else a


NEAR_ID = (float("nan"), 0, M64)


def same_record(a, b):
    """Bit-for-bit equality of two restated records (tuples of floats and ints).  A NaN equals any NaN: the GPU returns
    the canonical NaN from arithmetic on a NaN operand, where the CPU propagates the operand's payload."""
    import struct
    if isinstance(a, (tuple, list)):
        return isinstance(b, (tuple, list)) and len(a) == len(b) and all(same_record(x, y) for x, y in zip(a, b))
    if isinstance(a, float) or isinstance(b, float):
        if math.isnan(a) and math.isnan(b):
            return True
        return struct.pack("<d", float(a)) == struct.pack("<d", float(b))
    return a == b


# ---- hand-written descriptors that break the fold rules: registration must refuse all but ok_fold ------------------------
BAD_SRC = r'''
#include "fiber_b200_body.cuh"

struct Sum {
    using Arg = int64_t;
    struct Res { uint64_t s; };
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static void run(const Arg& a, Res& r, uint64_t, const fbr::ErrSink&, uint32_t) { r.s = (uint64_t)a; }
    __host__ __device__ static Res identity() { return Res{0}; }
    __device__ static __forceinline__ void combine(Res& acc, const Res& x) { acc.s += x.s; }
};
static const Sum::Res kZero{0};

#define BAD_FOLD(entry, name, flags, kind, fold, id) BAD_FOLD_N(entry, name, flags, kind, fold, id, (id) ? 8u : 0u)
#define BAD_FOLD_N(entry, name, flags, kind, fold, id, id_bytes)                                                   \
    extern "C" const fbr_body_module_t* entry(void) {                                                            \
        static const fbr_body_module_t m = {FBR_BODY_MODULE_ABI, (uint32_t)sizeof(fbr::WaveParams), name, 8u,     \
                                            ((flags) & FBR_BODY_EMIT) ? 8u : 8u, (kind), (flags), 1024u,          \
                                            fbr_body_export::launch_record<Sum>,                                 \
                                            fbr_body_export::occupancy_record<Sum>, 0u, 0u, 0u, 0u,              \
                                            ((flags) & FBR_BODY_EMIT) ? 4u : 0u, 0u, {0u, 0u, 0u}, (fold), (id), (id_bytes)}; \
        return &m;                                                                                               \
    }
#define RB (FBR_BODY_RECORD)
BAD_FOLD(bad_fold_flag_only, "bad_fold_flag_only", RB | FBR_BODY_FOLD, FBR_RES_BYTES, nullptr, nullptr)     // flag, no fields
BAD_FOLD(bad_fold_no_id, "bad_fold_no_id", RB | FBR_BODY_FOLD, FBR_RES_BYTES, fbr_body_export::launch_fold<Sum>, nullptr)
BAD_FOLD(bad_fold_fields_only, "bad_fold_fields_only", RB, FBR_RES_BYTES, fbr_body_export::launch_fold<Sum>, &kZero)
BAD_FOLD(bad_fold_thread, "bad_fold_thread", FBR_BODY_FOLD, FBR_RES_I64, fbr_body_export::launch_fold<Sum>, &kZero)
BAD_FOLD(bad_fold_emit, "bad_fold_emit", RB | FBR_BODY_EMIT | FBR_BODY_FOLD, FBR_RES_OFFSETS, fbr_body_export::launch_fold<Sum>, &kZero)
BAD_FOLD(bad_fold_summable, "bad_fold_summable", RB | FBR_BODY_SUMMABLE | FBR_BODY_FOLD, FBR_RES_BYTES,
         fbr_body_export::launch_fold<Sum>, &kZero)
BAD_FOLD_N(bad_fold_id_size, "bad_fold_id_size", RB | FBR_BODY_FOLD, FBR_RES_BYTES, fbr_body_export::launch_fold<Sum>, &kZero, 4u)
BAD_FOLD_N(bad_fold_id_size_only, "bad_fold_id_size_only", RB, FBR_RES_BYTES, nullptr, nullptr, 8u)
BAD_FOLD(ok_fold, "ok_fold", RB | FBR_BODY_FOLD, FBR_RES_BYTES, fbr_body_export::launch_fold<Sum>, &kZero)
'''
BAD_MODULE = fiber_b200.bodies.compile_module("fold_bad_descriptors", BAD_SRC)
BAD_ENTRIES = ["bad_fold_flag_only", "bad_fold_no_id", "bad_fold_fields_only", "bad_fold_thread", "bad_fold_emit",
               "bad_fold_summable", "bad_fold_id_size", "bad_fold_id_size_only"]

# restatements by body name: (run over one task's arguments, combine, identity)
RESTATED = {
    "moments_f64": (moments_combine, MOMENTS_ID),
    "row_sum_f64": (row_sum_combine, ROW_ID),
    "sum_sq_idx_u64": (add_u64, 0),
    "byte_hist_u8": (hist_combine, HIST_ID),
    "pair_overlap_u32": (add_u64, 0),
    "fault_count_u64": (add_u64, 0),
    "nearest_query_f32": (nearest_combine, NEAR_ID),
}
