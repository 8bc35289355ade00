"""Group record bodies: G threads of one warp run each task together (``static constexpr uint32_t kGroup = G``).

Each CUDA source below is compiled by ``fiber_b200.device_body(name, source=..., args=..., result=...)`` and registered
at import time.  Next to each body: its Python definition (what the reference would run) and a NumPy restatement the
GPU results are compared against bit for bit.  Where a body reduces across its lanes, the restatement repeats the
device's order exactly: lane ``rank`` takes elements ``rank, rank + G, ...`` in sequence with explicitly rounded
operations (``__dadd_rn`` / ``__dmul_rn``, ``__fadd_rn`` / ``__fmul_rn``: no contraction into FMAs), then the lanes
combine in an xor butterfly with offsets G/2, ..., 1.
"""
import numpy as np

import fiber_b200
from fiber_b200 import bodies

from .record_bodies import splitmix64, splitmix_np

# ---- row moments: 1024 float64 (8 KB) -> sum, sum of squares, min, max -----------------------------------------------
MOMENTS_ARG = np.dtype([("x", "<f8", (1024,))])
MOMENTS_RES = np.dtype([("sum", "<f8"), ("sumsq", "<f8"), ("min", "<f8"), ("max", "<f8")])

MOMENTS_SRC = r'''
#include "fiber_b200_body.cuh"

// a row of 1024 float64 -> (sum, sum of squares, min, max) on a warp: lane k sums x[k], x[k + 32], ... in order, then
// the lanes add in an xor butterfly (offsets 16 .. 1), so every lane ends with the same value
struct RowMoments {
    struct Arg { double x[1024]; };
    struct Res { double sum, sumsq, mn, mx; };
    static constexpr uint32_t kGroup = 32;
    static constexpr bool kIndexArg = false;
    static constexpr bool kCanFault = false;
    __device__ static __forceinline__ void run(const Arg& a, Res& r, const fbr::Group<32>& g, uint64_t,
                                               const fbr::ErrSink&, uint32_t) {
        double s = 0.0, q = 0.0, mn = INFINITY, mx = -INFINITY;
#pragma unroll 8
        for (uint32_t k = g.rank; k < 1024; k += g.size) {
            const double x = a.x[k];
            s = __dadd_rn(s, x);
            q = __dadd_rn(q, __dmul_rn(x, x));
            mn = fmin(mn, x);
            mx = fmax(mx, x);
        }
#pragma unroll
        for (uint32_t o = g.size / 2; o > 0; o >>= 1) {
            s = __dadd_rn(s, __shfl_xor_sync(g.mask, s, o));
            q = __dadd_rn(q, __shfl_xor_sync(g.mask, q, o));
            mn = fmin(mn, __shfl_xor_sync(g.mask, mn, o));
            mx = fmax(mx, __shfl_xor_sync(g.mask, mx, o));
        }
        if (g.rank == 0) { r.sum = s; r.sumsq = q; r.mn = mn; r.mx = mx; }
    }
};
FBR_EXPORT_RECORD_BODY(RowMoments, "row_moments_f64", row_moments_entry, 0)

// the same, but a task whose last element is -1.0 "kills its worker" on its first attempt (the lane that owns
// x[1023], rank 31, reports it: the unit is lost and re-dispatched)
struct FaultRowMoments {
    using Arg = RowMoments::Arg;
    using Res = RowMoments::Res;
    static constexpr uint32_t kGroup = 32;
    static constexpr bool kIndexArg = false;
    static constexpr bool kCanFault = true;
    __device__ static __forceinline__ void run(const Arg& a, Res& r, const fbr::Group<32>& g, uint64_t gidx,
                                               const fbr::ErrSink& es, uint32_t attempt) {
        if (attempt == 0 && g.rank == 31 && a.x[1023] == -1.0) es.report(fbr::TASK_FAULT, gidx);
        RowMoments::run(a, r, g, gidx, es, attempt);
    }
};
FBR_EXPORT_RECORD_BODY(FaultRowMoments, "fault_row_moments_f64", fault_row_moments_entry, 0)
'''

# ---- the largest record: 8192 float32 (32 KB) -> max and its lowest index ---------------------------------------------
WIDE_ARG = np.dtype([("x", "<f4", (8192,))])
WIDE_RES = np.dtype([("max", "<f4"), ("argmax", "<u4"), ("pad", "<u4", (2,))])

WIDE_SRC = r'''
#include "fiber_b200_body.cuh"

// a row of 8192 float32 -> (max, lowest index of the max, 0, 0): a claim unit is one task, so one of the eight warps
// of consumers runs it.  (v, i) pairs combine by the larger v, then the lower i, which is associative and commutative
struct WideRowMax {
    struct Arg { float x[8192]; };
    struct Res { float mx; uint32_t argmax; uint32_t pad[2]; };
    static constexpr uint32_t kGroup = 32;
    static constexpr bool kIndexArg = false;
    static constexpr bool kCanFault = false;
    __device__ static __forceinline__ void run(const Arg& a, Res& r, const fbr::Group<32>& g, uint64_t,
                                               const fbr::ErrSink&, uint32_t) {
        float v = a.x[g.rank];
        uint32_t i = g.rank;
#pragma unroll 8
        for (uint32_t k = g.rank + g.size; k < 8192; k += g.size) {
            const float x = a.x[k];
            if (x > v) { v = x; i = k; }
        }
#pragma unroll
        for (uint32_t o = g.size / 2; o > 0; o >>= 1) {
            const float v2 = __shfl_xor_sync(g.mask, v, o);
            const uint32_t i2 = __shfl_xor_sync(g.mask, i, o);
            if (v2 > v || (v2 == v && i2 < i)) { v = v2; i = i2; }
        }
        if (g.rank == 0) { r.mx = v; r.argmax = i; r.pad[0] = 0; r.pad[1] = 0; }
    }
};
FBR_EXPORT_RECORD_BODY(WideRowMax, "wide_row_max_f32", wide_row_max_entry, 0)
'''

# ---- a large result per range() index: 2048 uint32 (8 KB) ------------------------------------------------------------
SPLITROW_RES = np.dtype([("w", "<u4", (2048,))])

SPLITROW_SRC = r'''
#include "fiber_b200_body.cuh"

// index i -> w[k] = low32(splitmix64(i * 2048 + k)), k < 2048, written by 16 lanes (lane k % 16 writes w[k])
struct SplitmixRow {
    using Arg = int64_t;
    struct Res { uint32_t w[2048]; };
    static constexpr uint32_t kGroup = 16;
    static constexpr bool kIndexArg = true;
    static constexpr bool kCanFault = false;
    __device__ static __forceinline__ void run(const Arg& i, Res& r, const fbr::Group<16>& g, uint64_t,
                                               const fbr::ErrSink&, uint32_t) {
        const uint64_t base = (uint64_t)i * 2048u;
#pragma unroll 4
        for (uint32_t k = g.rank; k < 2048; k += g.size) r.w[k] = (uint32_t)fbr::splitmix64(base + k);
    }
};
FBR_EXPORT_RECORD_BODY(SplitmixRow, "splitmix_row_u32", splitmix_row_entry, FBR_BODY_INDEX_ARG)
'''

# ---- sub-warp groups: a 4x4 matrix times a vector, on four lanes --------------------------------------------------------
MAT4_ARG = np.dtype([("m", "<f4", (16,)), ("v", "<f4", (4,))])
MAT4_RES = np.dtype([("y", "<f4", (4,)), ("norm2", "<f4")])

MAT4_SRC = r'''
#include "fiber_b200_body.cuh"

// (m, v) -> (y = m v, |y|^2): lane k computes y[k] = ((m[k][0] v[0] + m[k][1] v[1]) + m[k][2] v[2]) + m[k][3] v[3];
// the squares add in an xor butterfly (offsets 2, 1).  80 B -> 20 B records: eight groups per warp
struct Mat4Apply {
    struct Arg { float m[16]; float v[4]; };
    struct Res { float y[4]; float norm2; };
    static constexpr uint32_t kGroup = 4;
    static constexpr bool kIndexArg = false;
    static constexpr bool kCanFault = false;
    __device__ static __forceinline__ void run(const Arg& a, Res& r, const fbr::Group<4>& g, uint64_t,
                                               const fbr::ErrSink&, uint32_t) {
        const float* row = a.m + 4 * g.rank;
        float y = __fmul_rn(row[0], a.v[0]);
#pragma unroll
        for (int j = 1; j < 4; ++j) y = __fadd_rn(y, __fmul_rn(row[j], a.v[j]));
        r.y[g.rank] = y;
        float t = __fmul_rn(y, y);
#pragma unroll
        for (uint32_t o = g.size / 2; o > 0; o >>= 1) t = __fadd_rn(t, __shfl_xor_sync(g.mask, t, o));
        if (g.rank == 0) r.norm2 = t;
    }
};
FBR_EXPORT_RECORD_BODY(Mat4Apply, "mat4_apply_f32", mat4_apply_entry, 0)
'''

# ---- a group body with a broadcast block: 64-dimensional nearest centroid on eight lanes -----------------------------
POINT64 = np.dtype([("p", "<f4", (64,))])
CENTROID64 = np.dtype([("c", "<f4", (64,))])
NEAREST64_RES = np.dtype([("k", "<u4"), ("d2", "<f4")])

NEAREST64_SRC = r'''
#include "fiber_b200_body.cuh"

// p -> (k, d2): the nearest of K 64-dimensional centroids on eight lanes.  For every centroid, lane j sums
// (p[d] - c[d])^2 over d = j, j + 8, ... in order, then the lanes add in an xor butterfly (offsets 4, 2, 1); a strictly
// smaller d2 replaces the best, so the lowest k wins ties.  Blocks of up to 128 centroids (32 KB) are staged
struct NearestRowGroup {
    struct Arg { float p[64]; };
    struct Res { uint32_t k; float d2; };
    struct Centroid { float c[64]; };
    using Shared = Centroid;
    static constexpr uint32_t kSharedStage = 32768;
    static constexpr uint32_t kGroup = 8;
    static constexpr bool kIndexArg = false;
    static constexpr bool kCanFault = false;
    __device__ static __forceinline__ void run(const Arg& a, Res& r, const fbr::Broadcast<Shared>& sh,
                                               const fbr::Group<8>& g, uint64_t, const fbr::ErrSink&, uint32_t) {
        float p[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) p[j] = a.p[g.rank + 8 * j];
        const uint32_t n = (uint32_t)sh.n;
        uint32_t best_k = 0;
        float best = 0.0f;
        for (uint32_t k = 0; k < n; ++k) {
            const float* c = sh.data[k].c + g.rank;
            float d2 = 0.0f;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float t = __fsub_rn(p[j], c[8 * j]);
                d2 = __fadd_rn(d2, __fmul_rn(t, t));
            }
#pragma unroll
            for (uint32_t o = g.size / 2; o > 0; o >>= 1) d2 = __fadd_rn(d2, __shfl_xor_sync(g.mask, d2, o));
            if (k == 0 || d2 < best) { best = d2; best_k = k; }
        }
        if (g.rank == 0) { r.k = best_k; r.d2 = best; }
    }
};
FBR_EXPORT_RECORD_BODY(NearestRowGroup, "nearest_row_group_f32", nearest_row_group_entry, 0)
'''

# Hand-written descriptors that break the group rules; registration must refuse every one of them except ok_group.
# (FBR_EXPORT_RECORD_BODY derives group_threads from kGroup and checks the sizes at compile time, so a real body cannot
# get there.)
BAD_SRC = r'''
#include "fiber_b200_body.cuh"

struct OkG {
    struct Arg { float x[4]; };
    struct Res { float y[4]; };
    static constexpr uint32_t kGroup = 4;
    static constexpr bool kIndexArg = false;
    static constexpr bool kCanFault = false;
    __device__ static void run(const Arg& a, Res& r, const fbr::Group<4>& g, uint64_t, const fbr::ErrSink&, uint32_t) {
        r.y[g.rank] = a.x[g.rank];
    }
};
#define BAD_GROUP(entry, name, ab, rb, flags, group)                                                               \
    extern "C" const fbr_body_module_t* entry(void) {                                                            \
        static const fbr_body_module_t m = {FBR_BODY_MODULE_ABI, (uint32_t)sizeof(fbr::WaveParams), name, ab, rb, \
                                            FBR_RES_BYTES, (flags), 1u,                                          \
                                            fbr_body_export::launch_record<OkG>, fbr_body_export::occupancy_record<OkG>, \
                                            0u, 0u, (group)};                                                    \
        return &m;                                                                                               \
    }
#define REC FBR_BODY_RECORD
BAD_GROUP(bad_group3, "bad_group3", 16u, 16u, REC, 3u)
BAD_GROUP(bad_group64, "bad_group64", 16u, 16u, REC, 64u)
BAD_GROUP(bad_group_thread, "bad_group_thread", 8u, 8u, 0u, 4u)                    // not a record body
BAD_GROUP(bad_group_64k, "bad_group_64k", 65536u, 16u, REC, 32u)
BAD_GROUP(bad_group_align, "bad_group_align", 32768u, 12u, REC, 32u)              // kAlign 4: 4 * 32 KB per group
BAD_GROUP(bad_thread_8k, "bad_thread_8k", 8192u, 16u, REC, 1u)                     // one thread: 4096 at most
BAD_GROUP(ok_group, "ok_group", 16u, 16u, REC, 4u)
'''


@fiber_b200.device_body("row_moments_f64", source=MOMENTS_SRC, entry="row_moments_entry", args=MOMENTS_ARG,
                        result=MOMENTS_RES)
def row_moments_f64(x):
    """Sums in the body's order: 32 running sums over x[k::32], then the xor butterfly (Python floats round like
    __dadd_rn / __dmul_rn)."""
    x = [float(v) for v in x]

    def tree(lanes):
        o = len(lanes) // 2
        while o:
            lanes = [lanes[k] + lanes[k ^ o] for k in range(len(lanes))]
            o //= 2
        return lanes[0]
    s = [0.0] * 32
    q = [0.0] * 32
    for j, v in enumerate(x):
        s[j % 32] += v
        q[j % 32] += v * v
    return (tree(s), tree(q), min(x), max(x))


@fiber_b200.device_body("fault_row_moments_f64", source=MOMENTS_SRC, entry="fault_row_moments_entry",
                        args=MOMENTS_ARG, result=MOMENTS_RES)
def fault_row_moments_f64(x):
    return row_moments_f64(x)


@fiber_b200.device_body("wide_row_max_f32", source=WIDE_SRC, entry="wide_row_max_entry", args=WIDE_ARG, result=WIDE_RES)
def wide_row_max_f32(x):
    x = [float(v) for v in x]
    mx = max(x)
    return (mx, x.index(mx), [0, 0])


_M64 = (1 << 64) - 1


@fiber_b200.device_body("splitmix_row_u32", source=SPLITROW_SRC, entry="splitmix_row_entry", args="<i8",
                        result=SPLITROW_RES)
def splitmix_row_u32(i):
    base = (i * 2048) & _M64
    return [splitmix64((base + k) & _M64) & 0xFFFFFFFF for k in range(2048)]


@fiber_b200.device_body("mat4_apply_f32", source=MAT4_SRC, entry="mat4_apply_entry", args=MAT4_ARG, result=MAT4_RES)
def mat4_apply_f32(m, v):
    m = np.asarray(m, np.float32).reshape(4, 4)
    v = np.asarray(v, np.float32)
    y = [m[k, 0] * v[0] + m[k, 1] * v[1] + m[k, 2] * v[2] + m[k, 3] * v[3] for k in range(4)]   # float32 scalars
    t = [yk * yk for yk in y]
    return ([float(yk) for yk in y], float((t[0] + t[2]) + (t[1] + t[3])))


@fiber_b200.device_body("nearest_row_group_f32", source=NEAREST64_SRC, entry="nearest_row_group_entry", args=POINT64,
                        result=NEAREST64_RES, shared=("centroids", CENTROID64))
def nearest_row_group_f32(centroids, p):
    r = nearest64_np(np.asarray(p, np.float32).reshape(1, 64), centroids)[0]
    return (int(r["k"]), float(r["d2"]))


@fiber_b200.device_initializer("nearest_row_group_f32")
def set_centroids64(centroids):
    """Pool initializer: the centroids every task compares against, uploaded once per worker."""
    raise RuntimeError("runs on the GPU workers")


BAD_MODULE = bodies.compile_module("bad_group_bodies", BAD_SRC)


# ---- NumPy restatements ---------------------------------------------------------------------------------------------
def _butterfly(lanes, op):
    """The xor butterfly over the last axis (G lanes): offsets G/2 .. 1, lane l combines with lane l ^ o."""
    g = lanes.shape[-1]
    idx = np.arange(g)
    o = g // 2
    while o:
        lanes = op(lanes, lanes[..., idx ^ o])
        o //= 2
    return lanes[..., 0]


def _lanes(rows, g):
    """rows (n, m) -> (n, m / g, g): [:, j, k] is element k + g * j, the j-th element lane k takes."""
    return rows.reshape(len(rows), -1, g)


def row_moments_np(args):
    x = _lanes(np.ascontiguousarray(args["x"]), 32)
    s = np.zeros((len(x), 32))
    q = np.zeros((len(x), 32))
    for j in range(x.shape[1]):
        s = s + x[:, j]
        q = q + x[:, j] * x[:, j]
    out = np.empty(len(x), MOMENTS_RES)
    out["sum"] = _butterfly(s, np.add)
    out["sumsq"] = _butterfly(q, np.add)
    out["min"] = args["x"].min(axis=1)
    out["max"] = args["x"].max(axis=1)
    return out


def wide_row_max_np(args):
    x = args["x"]
    out = np.zeros(len(x), WIDE_RES)
    i = x.argmax(axis=1)
    out["argmax"] = i
    out["max"] = x[np.arange(len(x)), i]
    return out


def splitmix_row_np(idx):
    u = np.asarray(idx, dtype=np.int64).view(np.uint64)
    out = np.empty(len(u), SPLITROW_RES)
    with np.errstate(over="ignore"):
        z = u[:, None] * np.uint64(2048) + np.arange(2048, dtype=np.uint64)[None, :]
        out["w"] = (splitmix_np(z) & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    return out


def mat4_np(args):
    m = args["m"].reshape(-1, 4, 4)
    v = args["v"]
    y = m[:, :, 0] * v[:, 0:1]
    for j in range(1, 4):
        y = y + m[:, :, j] * v[:, j:j + 1]
    out = np.empty(len(args), MAT4_RES)
    out["y"] = y
    out["norm2"] = _butterfly(y * y, np.add)
    return out


def nearest64_np(points, centroids):
    p = _lanes(np.ascontiguousarray(points).view(np.float32).reshape(-1, 64), 8)
    c = _lanes(np.ascontiguousarray(centroids).view(np.float32).reshape(-1, 64), 8)
    best = np.zeros(len(p), np.float32)
    best_k = np.zeros(len(p), np.uint32)
    for k in range(len(c)):
        d2 = np.zeros((len(p), 8), np.float32)
        for j in range(8):
            t = p[:, j] - c[k, j]
            d2 = d2 + t * t
        d2 = _butterfly(d2, np.add)
        upd = d2 < best if k else np.ones(len(p), bool)
        best = np.where(upd, d2, best)
        best_k = np.where(upd, np.uint32(k), best_k)
    out = np.empty(len(p), NEAREST64_RES)
    out["k"], out["d2"] = best_k, best
    return out


# ---- seeded inputs --------------------------------------------------------------------------------------------------
def moments_args(n, seed=0):
    rng = np.random.default_rng(seed)
    a = np.empty(n, MOMENTS_ARG)
    a["x"] = rng.standard_normal((n, 1024)) * np.exp2(rng.integers(-20, 20, (n, 1)))
    return a


def wide_args(n, seed=0):
    rng = np.random.default_rng(seed)
    a = np.empty(n, WIDE_ARG)
    a["x"] = rng.standard_normal((n, 8192), dtype=np.float32)
    if n > 1:
        a["x"][1, [100, 5000]] = 1e30                  # a tie: the lower index wins
    return a


def mat4_args(n, seed=0):
    rng = np.random.default_rng(seed)
    a = np.empty(n, MAT4_ARG)
    a["m"] = rng.standard_normal((n, 16), dtype=np.float32)
    a["v"] = rng.standard_normal((n, 4), dtype=np.float32)
    return a


def points64(n, seed=0):
    rng = np.random.default_rng(seed)
    a = np.empty(n, POINT64)
    a["p"] = rng.standard_normal((n, 64), dtype=np.float32)
    return a


def centroids64(k, seed=1):
    rng = np.random.default_rng(seed)
    c = np.empty(k, CENTROID64)
    c["c"] = rng.standard_normal((k, 64), dtype=np.float32)
    return c
