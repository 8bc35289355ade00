"""Multi-stream items record bodies: every task takes 2 to 4 variable-length arrays, each with its own element type and
offsets (``using Items = fbr::ItemTypes<...>;`` in the body's struct).

Each CUDA source below is compiled by ``fiber_b200.device_body(name, source=..., items=[...], ...)`` and registered at
import time.  Next to each body: its Python definition (what the reference would run) and a NumPy / Python restatement
the GPU results are compared against bit for bit.  The group body's restatement repeats the device's order exactly: lane
``rank`` takes pairs ``rank, rank + 32, ...`` with explicitly rounded multiplies and adds, then the lanes combine in an xor
butterfly with offsets 16, ..., 1 (as in ``group_bodies.py``).
"""
import numpy as np

import fiber_b200
import fiber_b200.bodies

COUNT_RES = np.dtype([("common", "<u4"), ("na", "<u4"), ("nb", "<u4")])

U32_SRC = r'''
#include "fiber_b200_body.cuh"

// the size of the multiset intersection of two sorted uint32 lists (a merge), and both lengths
__device__ __forceinline__ uint32_t common_count(const fbr::Items<uint32_t>& a, const fbr::Items<uint32_t>& b) {
    uint64_t i = 0, j = 0;
    uint32_t c = 0;
    while (i < a.n && j < b.n) {
        const uint32_t x = a.data[i], y = b.data[j];
        c += x == y;
        i += x <= y;
        j += y <= x;
    }
    return c;
}

struct IntersectCount {
    using Items = fbr::ItemTypes<uint32_t, uint32_t>;
    using Arg = fbr::NoArg;
    struct Res { uint32_t common, na, nb; };
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static __forceinline__ void run(const fbr::Items<uint32_t>& a, const fbr::Items<uint32_t>& b, Res& r, uint64_t,
                                               const fbr::ErrSink&, uint32_t) {
        r.common = common_count(a, b);
        r.na = (uint32_t)a.n;
        r.nb = (uint32_t)b.n;
    }
};
FBR_EXPORT_RECORD_BODY(IntersectCount, "intersect_count_u32", intersect_count_entry, 0)

// the same, but every task whose index is 7 mod 1000 "kills its worker" on the first attempt: the unit is re-dispatched
struct FaultIntersectCount {
    using Items = IntersectCount::Items;
    using Arg = fbr::NoArg;
    using Res = IntersectCount::Res;
    static constexpr bool kIndexArg = false, kCanFault = true;
    __device__ static __forceinline__ void run(const fbr::Items<uint32_t>& a, const fbr::Items<uint32_t>& b, Res& r,
                                               uint64_t gidx, const fbr::ErrSink& es, uint32_t attempt) {
        if (attempt == 0 && gidx % 1000 == 7) es.report(fbr::TASK_FAULT, gidx);
        IntersectCount::run(a, b, r, gidx, es, attempt);
    }
};
FBR_EXPORT_RECORD_BODY(FaultIntersectCount, "fault_intersect_count_u32", fault_intersect_count_entry, 0)

// the values two sorted uint32 lists have in common (multiset intersection, ascending); count() is the merge's count
struct SortedCommon {
    using Items = fbr::ItemTypes<uint32_t, uint32_t>;
    using Arg = fbr::NoArg;
    using Out = uint32_t;
    using Res = fbr::NoRes;
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static __forceinline__ uint64_t count(const fbr::Items<uint32_t>& a, const fbr::Items<uint32_t>& b, uint64_t) {
        return common_count(a, b);
    }
    __device__ static __forceinline__ void run(const fbr::Items<uint32_t>& a, const fbr::Items<uint32_t>& b, fbr::Emit<Out>& y,
                                               uint64_t, const fbr::ErrSink&, uint32_t) {
        uint64_t i = 0, j = 0;
        while (i < a.n && j < b.n) {
            const uint32_t x = a.data[i], v = b.data[j];
            if (x == v) y.push(x);
            i += x <= v;
            j += v <= x;
        }
    }
};
FBR_EXPORT_RECORD_BODY(SortedCommon, "sorted_common_u32", sorted_common_entry, 0)
'''

MIX_ARG = np.dtype([("seed", "<u8")])
MIX_RES = np.dtype([("h", "<u8"), ("n0", "<u4"), ("n1", "<u4"), ("n2", "<u4"), ("n3", "<u4")])
DOT_RES = np.dtype([("dot", "<f8"), ("n", "<u8")])

MIX_SRC = r'''
#include "fiber_b200_body.cuh"

// four streams of 1-, 2-, 4- and 8-byte integers, a head record and a broadcast table of uint32: an integer hash of
// everything the task sees
struct Mix4 {
    using Items = fbr::ItemTypes<uint8_t, uint16_t, uint32_t, uint64_t>;
    struct Arg { uint64_t seed; };
    struct Res { uint64_t h; uint32_t n0, n1, n2, n3; };
    using Shared = uint32_t;
    static constexpr uint32_t kSharedStage = 4096;
    static constexpr bool kIndexArg = false, kCanFault = false;
    template <class T>
    __device__ static __forceinline__ uint64_t fold(uint64_t h, const fbr::Items<T>& x) {
        for (uint64_t k = 0; k < x.n; ++k) h = (h ^ (uint64_t)x.data[k]) * 0x100000001b3ull;
        return h * 0x9e3779b97f4a7c15ull + x.n;
    }
    __device__ static __forceinline__ void run(const Arg& a, const fbr::Items<uint8_t>& x0, const fbr::Items<uint16_t>& x1,
                                               const fbr::Items<uint32_t>& x2, const fbr::Items<uint64_t>& x3, Res& r,
                                               const fbr::Broadcast<uint32_t>& w, uint64_t gidx, const fbr::ErrSink&, uint32_t) {
        uint64_t h = fold(fold(fold(fold(a.seed, x0), x1), x2), x3);
        r.h = h ^ w.data[gidx % w.n];
        r.n0 = (uint32_t)x0.n; r.n1 = (uint32_t)x1.n; r.n2 = (uint32_t)x2.n; r.n3 = (uint32_t)x3.n;
    }
};
FBR_EXPORT_RECORD_BODY(Mix4, "mix4_u1_u2_u4_u8", mix4_entry, 0)

// the dot product of two float64 rows on a warp: lane k adds x[k] * y[k], x[k + 32] * y[k + 32], ... in order, then the
// lanes add in an xor butterfly (offsets 16 .. 1).  Rows of different lengths are a bad argument
struct PairDot {
    using Items = fbr::ItemTypes<double, double>;
    using Arg = fbr::NoArg;
    struct Res { double dot; uint64_t n; };
    static constexpr uint32_t kGroup = 32;
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static __forceinline__ void run(const fbr::Items<double>& x, const fbr::Items<double>& y, Res& r,
                                               const fbr::Group<32>& g, uint64_t gidx, const fbr::ErrSink& es, uint32_t) {
        if (x.n != y.n) {
            if (g.rank == 0) es.report(fbr::TASK_BADARG, gidx);
            return;
        }
        double s = 0.0;
        const double* const end = x.data + x.n;
        for (const double *p = x.data + g.rank, *q = y.data + g.rank; p < end; p += g.size, q += g.size) s = __dadd_rn(s, __dmul_rn(*p, *q));
#pragma unroll
        for (uint32_t o = g.size / 2; o > 0; o >>= 1) s = __dadd_rn(s, __shfl_xor_sync(g.mask, s, o));
        if (g.rank == 0) { r.dot = s; r.n = x.n; }
    }
};
FBR_EXPORT_RECORD_BODY(PairDot, "pair_dot_f64", pair_dot_entry, 0)
'''


@fiber_b200.device_body("intersect_count_u32", source=U32_SRC, entry="intersect_count_entry", args=None,
                        items=[("a", "<u4"), ("b", "<u4")], result=COUNT_RES)
def intersect_count_u32(a, b):
    from collections import Counter
    return (sum((Counter(a) & Counter(b)).values()), len(a), len(b))


@fiber_b200.device_body("fault_intersect_count_u32", source=U32_SRC, entry="fault_intersect_count_entry", args=None,
                        items=[("a", "<u4"), ("b", "<u4")], result=COUNT_RES)
def fault_intersect_count_u32(a, b):
    return intersect_count_u32(a, b)


@fiber_b200.device_body("sorted_common_u32", source=U32_SRC, entry="sorted_common_entry", args=None,
                        items=[("a", "<u4"), ("b", "<u4")], out="<u4")
def sorted_common_u32(a, b):
    from collections import Counter
    return sorted((Counter(a) & Counter(b)).elements())


@fiber_b200.device_body("mix4_u1_u2_u4_u8", source=MIX_SRC, entry="mix4_entry", args=MIX_ARG, shared=("w", "<u4"),
                        items=[("x0", "u1"), ("x1", "<u2"), ("x2", "<u4"), ("x3", "<u8")], result=MIX_RES)
def mix4_u1_u2_u4_u8(w, x0, x1, x2, x3, seed):
    return mix4_one(w, [x0, x1, x2, x3], seed, None)


@fiber_b200.device_body("pair_dot_f64", source=MIX_SRC, entry="pair_dot_entry", args=None,
                        items=[("x", "<f8"), ("y", "<f8")], result=DOT_RES)
def pair_dot_f64(x, y):
    return pair_dot_one(np.asarray(x, np.float64), np.asarray(y, np.float64))


# ---- restatements ------------------------------------------------------------------------------------------------------
M64 = (1 << 64) - 1


def _spans(offs):
    o = np.asarray(offs, np.int64)
    return o[:-1], o[1:]


def intersect_count_np(a, b):
    """(common, |a|, |b|) for Ragged columns a, b of sorted uint32 lists: a multiset intersection per task."""
    out = np.zeros(len(a), COUNT_RES)
    for i in range(len(a)):
        x, y = a[i], b[i]
        vx, cx = np.unique(x, return_counts=True)
        vy, cy = np.unique(y, return_counts=True)
        _, ix, iy = np.intersect1d(vx, vy, assume_unique=True, return_indices=True)
        out[i] = (int(np.minimum(cx[ix], cy[iy]).sum()), len(x), len(y))
    return out


def sorted_common_py(a, b):
    out = []
    for i in range(len(a)):
        x, y = a[i].tolist(), b[i].tolist()
        p = q = 0
        row = []
        while p < len(x) and q < len(y):
            if x[p] == y[q]:
                row.append(x[p])
            p, q = p + (x[p] <= y[q]), q + (y[q] <= x[p])
        out.append(row)
    return out


def mix4_one(w, xs, seed, gidx):
    h = int(seed)
    for x in xs:
        for v in np.asarray(x).tolist():
            h = ((h ^ int(v)) * 0x100000001b3) & M64
        h = (h * 0x9e3779b97f4a7c15 + len(x)) & M64
    w = np.asarray(w, np.uint32)
    if gidx is not None:
        h ^= int(w[gidx % len(w)])
    return h


def mix4_np(w, cols, seeds, base=0):
    """Results of mix4_u1_u2_u4_u8 over Ragged columns cols[0..3] and the seeds, for tasks base, base + 1, ..."""
    out = np.zeros(len(seeds), MIX_RES)
    for i in range(len(seeds)):
        xs = [c[i] for c in cols]
        out[i] = (mix4_one(w, xs, int(seeds[i]), base + i),) + tuple(len(x) for x in xs)
    return out


def pair_dot_one(x, y):
    lanes = np.zeros(32, np.float64)
    for r in range(32):
        s = np.float64(0.0)
        for k in range(r, len(x), 32):
            s = np.float64(s + np.float64(x[k] * y[k]))
        lanes[r] = s
    o = 16
    while o:
        lanes = lanes + lanes[np.arange(32) ^ o]
        o //= 2
    return (float(lanes[0]), len(x))


def pair_dot_np(x, y):
    out = np.zeros(len(x), DOT_RES)
    for i in range(len(x)):
        out[i] = pair_dot_one(x[i], y[i])
    return out


# ---- seeded inputs ------------------------------------------------------------------------------------------------------
def sorted_lists(n, seed, max_len=64, vocab=200, empty_every=0):
    """A Ragged of n sorted uint32 lists with skewed lengths (most short, a few up to 16 * max_len) drawn from a small
    vocabulary, so two lists share values; every `empty_every`-th list (if non-zero) is empty."""
    rng = np.random.default_rng(seed)
    lens = np.minimum(rng.geometric(1.0 / max(1, max_len // 4), n) - 1, 16 * max_len)
    if empty_every:
        lens[::empty_every] = 0
    offs = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=offs[1:])
    vals = rng.integers(0, vocab, int(offs[-1]), dtype=np.uint32)
    for i in range(n):
        vals[offs[i]:offs[i + 1]].sort()
    return fiber_b200.Ragged(vals, offs)


def ragged_of(rng, n, dtype, max_len, empty_every=0):
    lens = rng.integers(0, max_len + 1, n)
    if empty_every:
        lens[::empty_every] = 0
    offs = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=offs[1:])
    info = np.iinfo(dtype)
    vals = rng.integers(0, int(info.max), int(offs[-1]), dtype=dtype, endpoint=True)
    return fiber_b200.Ragged(vals, offs)


# Hand-written descriptors that break the multi-stream rules; registration must refuse every one of them except
# ok_streams.  (FBR_EXPORT_RECORD_BODY derives the fields from the struct, so a real body cannot get there.)
BAD_SRC = r'''
#include "fiber_b200_body.cuh"

#define BAD_STREAMS(entry, name, flags, n, b1, b2, b3)                                                             \
    extern "C" const fbr_body_module_t* entry(void) {                                                            \
        static const fbr_body_module_t m = {FBR_BODY_MODULE_ABI, (uint32_t)sizeof(fbr::WaveParams), name, 0u,     \
                                            12u, FBR_RES_BYTES, (flags), 1024u,                                  \
                                            fbr_body_export::launch_record<Pair>,                                \
                                            fbr_body_export::occupancy_record<Pair>, 0u, 0u, 0u,                 \
                                            ((flags) & FBR_BODY_ITEMS) ? 4u : 0u, 0u, (n),                      \
                                            {(b1), (b2), (b3)}};                                                 \
        return &m;                                                                                               \
    }
struct Pair {
    using Items = fbr::ItemTypes<uint32_t, uint32_t>;
    using Arg = fbr::NoArg;
    struct Res { uint32_t a, b, c; };
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static void run(const fbr::Items<uint32_t>& a, const fbr::Items<uint32_t>& b, Res& r, uint64_t, const fbr::ErrSink&,
                               uint32_t) { r.a = (uint32_t)a.n; r.b = (uint32_t)b.n; r.c = 0; }
};
#define IT (FBR_BODY_RECORD | FBR_BODY_ITEMS)
BAD_STREAMS(bad_streams5, "bad_streams5", IT, 5u, 4u, 4u, 4u)              // more than 4 streams
BAD_STREAMS(bad_streams_flag, "bad_streams_flag", FBR_BODY_RECORD, 2u, 4u, 0u, 0u)   // several streams without FBR_BODY_ITEMS
BAD_STREAMS(bad_stream_size, "bad_stream_size", IT, 2u, 3u, 0u, 0u)         // stream 1's element size
BAD_STREAMS(bad_stream_size0, "bad_stream_size0", IT, 3u, 4u, 0u, 0u)       // stream 2 without a size
BAD_STREAMS(bad_stream_extra, "bad_stream_extra", IT, 2u, 4u, 8u, 0u)       // a size past item_streams
BAD_STREAMS(ok_streams, "ok_streams", IT, 2u, 4u, 0u, 0u)
'''
BAD_MODULE = fiber_b200.bodies.compile_module("multi_items_bad_descriptors", BAD_SRC)
