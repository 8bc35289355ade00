"""Record bodies that read a broadcast block: one array every task of a map shares (``using Shared = ...``).

Each CUDA source below is compiled by ``fiber_b200.device_body(name, source=..., args=..., result=..., shared=...)``
and registered at import time.  Next to each body: its Python definition (what the reference would run, with the
shared array as the first parameter) and a NumPy restatement the GPU results are compared against bit for bit.
Floating-point bodies use explicitly rounded operations (``__fsub_rn`` / ``__fmul_rn`` / ``__fadd_rn``, ``__ddiv_rn``):
no contraction into FMAs, so every result is the IEEE value NumPy computes in the same order.
"""
import numpy as np

import fiber_b200
from fiber_b200 import bodies

from .record_bodies import splitmix64, splitmix_np

# ---- nearest centroid: 16-dimensional float32 points against K centroids ---------------------------------------------
POINT = np.dtype([("p", "<f4", (16,))])
CENTROID = np.dtype([("c", "<f4", (16,))])
NEAREST_RES = np.dtype([("k", "<u4"), ("d2", "<f4")])

NEAREST_SRC = r'''
#include "fiber_b200_body.cuh"

// p -> (k, d2): the index of the centroid nearest to p and its squared distance, summed in dimension order; on equal
// distances the lowest k wins.  Blocks of up to 512 centroids (32 KB) are staged in shared memory.
struct NearestCentroid {
    struct Arg { float p[16]; };
    struct Res { uint32_t k; float d2; };
    struct alignas(16) Centroid { float c[16]; };
    using Shared = Centroid;
    static constexpr uint32_t kSharedStage = 32768;
    static constexpr bool kIndexArg = false;
    static constexpr bool kCanFault = false;
    __device__ static __forceinline__ void run(const Arg& a, Res& r, const fbr::Broadcast<Shared>& sh, uint64_t,
                                               const fbr::ErrSink&, uint32_t) {
        float p[16];
#pragma unroll
        for (int d = 0; d < 16; ++d) p[d] = a.p[d];
        const uint32_t n = (uint32_t)sh.n;
        uint32_t best_k = 0;
        float best = 0.0f;
        for (uint32_t k = 0; k < n; ++k) {
            const Centroid& c = sh.data[k];
            float d2 = 0.0f;
#pragma unroll
            for (int d = 0; d < 16; ++d) {
                const float t = __fsub_rn(p[d], c.c[d]);
                d2 = __fadd_rn(d2, __fmul_rn(t, t));
            }
            if (k == 0 || d2 < best) { best = d2; best_k = k; }
        }
        r.k = best_k;
        r.d2 = best;
    }
};
FBR_EXPORT_RECORD_BODY(NearestCentroid, "nearest_centroid_f32", nearest_entry, 0)

// the same body with no shared-memory budget: every block is read from global memory
struct NearestCentroidGlobal : NearestCentroid {
    static constexpr uint32_t kSharedStage = 0;
};
FBR_EXPORT_RECORD_BODY(NearestCentroidGlobal, "nearest_centroid_global_f32", nearest_global_entry, 0)
'''

# ---- kernel density estimate: examples/parzen_estimation.py as a user body --------------------------------------------
SAMPLE = np.dtype([("x", "<f8", (2,))])
KDE_RES = np.dtype([("h", "<f8"), ("density", "<f8")])

KDE_SRC = r'''
#include "fiber_b200_body.cuh"

// h -> (h, (k_n / n) / h): the share of the n 2-D samples inside the hypercube of edge h around the origin, with the
// window test of the compiled-in parzen_f64 (|(0 - x_d) / h| > 1/2 is outside; a NaN counts as inside)
struct KdeWindow {
    using Arg = double;
    struct Res { double h, density; };
    struct Sample { double x[2]; };
    using Shared = Sample;
    static constexpr uint32_t kSharedStage = 16384;
    static constexpr bool kIndexArg = false;
    static constexpr bool kCanFault = false;
    __device__ static __forceinline__ void run(const Arg& h, Res& r, const fbr::Broadcast<Shared>& sh, uint64_t,
                                               const fbr::ErrSink&, uint32_t) {
        const uint32_t n = (uint32_t)sh.n;
        uint32_t k = 0;
        for (uint32_t j = 0; j < n; ++j) {
            const Sample s = sh.data[j];
            bool inside = true;
#pragma unroll
            for (int d = 0; d < 2; ++d) {
                const double q = __ddiv_rn(__dsub_rn(0.0, s.x[d]), h);
                inside = inside && !(fabs(q) > 0.5);
            }
            k += inside ? 1u : 0u;
        }
        r.h = h;
        r.density = __ddiv_rn(__ddiv_rn((double)k, (double)n), __dmul_rn(1.0, h));
    }
};
FBR_EXPORT_RECORD_BODY(KdeWindow, "kde_window_f64", kde_entry, 0)
'''

# ---- table lookup over range() indices ------------------------------------------------------------------------------
TABLE_SRC = r'''
#include "fiber_b200_body.cuh"

// i -> table[splitmix64(i) % n] ^ (uint32)i: random access into a table of n uint32
struct TableMix {
    using Arg = int64_t;
    using Res = uint32_t;
    using Shared = uint32_t;
    static constexpr uint32_t kSharedStage = 16384;
    static constexpr bool kIndexArg = true;
    static constexpr bool kCanFault = false;
    __device__ static __forceinline__ void run(const Arg& i, Res& r, const fbr::Broadcast<Shared>& sh, uint64_t,
                                               const fbr::ErrSink&, uint32_t) {
        r = sh.data[fbr::splitmix64((uint64_t)i) % sh.n] ^ (uint32_t)i;
    }
};
FBR_EXPORT_RECORD_BODY(TableMix, "table_mix_u32", table_mix_entry, FBR_BODY_INDEX_ARG)
'''

# Hand-written descriptors that break the broadcast rules; registration must refuse every one of them except ok_bcast.
# (FBR_EXPORT_RECORD_BODY derives the flags and fields from the struct, so a real body cannot get there.)
BAD_SRC = r'''
#include "fiber_b200_body.cuh"

struct OkB {
    struct Arg { float x; };
    struct Res { float y; };
    using Shared = float;
    static constexpr uint32_t kSharedStage = 0;
    static constexpr bool kIndexArg = false;
    static constexpr bool kCanFault = false;
    __device__ static void run(const Arg& a, Res& r, const fbr::Broadcast<Shared>& sh, uint64_t, const fbr::ErrSink&, uint32_t) {
        r.y = a.x + sh.data[0];
    }
};
#define BAD_BCAST(entry, name, flags, elem, stage)                                                                 \
    extern "C" const fbr_body_module_t* entry(void) {                                                            \
        static const fbr_body_module_t m = {FBR_BODY_MODULE_ABI, (uint32_t)sizeof(fbr::WaveParams), name, 4u, 4u, \
                                            FBR_RES_BYTES, (flags), 16u,                                         \
                                            fbr_body_export::launch_record<OkB>, fbr_body_export::occupancy_record<OkB>, \
                                            (elem), (stage)};                                                    \
        return &m;                                                                                               \
    }
#define REC FBR_BODY_RECORD
#define BC (FBR_BODY_NEEDS_SHARED | FBR_BODY_BROADCAST)
BAD_BCAST(bad_no_needs, "bad_no_needs", REC | FBR_BODY_BROADCAST, 4u, 0u)          // a block it may not get
BAD_BCAST(bad_thread, "bad_thread", BC, 4u, 0u)                                    // not a record body
BAD_BCAST(bad_fields, "bad_fields", REC, 4u, 0u)                                   // element without the flag
BAD_BCAST(bad_stage_only, "bad_stage_only", REC, 0u, 16u)                          // budget without the flag
BAD_BCAST(bad_elem0, "bad_elem0", REC | BC, 0u, 0u)
BAD_BCAST(bad_elem6, "bad_elem6", REC | BC, 6u, 0u)
BAD_BCAST(bad_elem_big, "bad_elem_big", REC | BC, 8192u, 0u)
BAD_BCAST(bad_stage24, "bad_stage24", REC | BC, 4u, 24u)
BAD_BCAST(bad_stage_big, "bad_stage_big", REC | BC, 4u, 200u << 10)
BAD_BCAST(ok_bcast, "ok_bcast", REC | BC, 4u, 0u)
'''


@fiber_b200.device_body("nearest_centroid_f32", source=NEAREST_SRC, entry="nearest_entry", args=POINT,
                        result=NEAREST_RES, shared=("centroids", CENTROID))
def nearest_centroid_f32(centroids, p):
    c = np.ascontiguousarray(centroids).view(np.float32).reshape(-1, 16)
    p = np.asarray(p, np.float32).reshape(16)
    best = None
    for k, row in enumerate(c):
        d2 = np.float32(0.0)
        for d in range(16):
            t = p[d] - row[d]                     # float32 scalars: every operation rounds to float32
            d2 = d2 + t * t
        if best is None or d2 < best[1]:
            best = (k, d2)
    return (best[0], float(best[1]))


@fiber_b200.device_body("nearest_centroid_global_f32", source=NEAREST_SRC, entry="nearest_global_entry", args=POINT,
                        result=NEAREST_RES, shared=("centroids", CENTROID))
def nearest_centroid_global_f32(centroids, p):
    return nearest_centroid_f32(centroids, p)


@fiber_b200.device_initializer("nearest_centroid_f32")
def set_centroids(centroids):
    """Pool initializer: the centroids every task compares against, uploaded once per worker."""
    raise RuntimeError("runs on the GPU workers")


@fiber_b200.device_body("kde_window_f64", source=KDE_SRC, entry="kde_entry", args="<f8", result=KDE_RES,
                        shared=("x_samples", SAMPLE))
def kde_window_f64(x_samples, h):
    """parzen_estimation(x_samples, point_x=0, h) (examples/parzen_estimation.py:6-15)."""
    xs = np.ascontiguousarray(x_samples)
    xs = xs.view(np.float64).reshape(-1, 2) if xs.dtype.names else xs.astype(np.float64).reshape(-1, 2)
    k = int(np.sum(~np.any(np.abs((0.0 - xs) / h) > 0.5, axis=1)))
    return (h, (k / len(xs)) / h)


@fiber_b200.device_initializer("kde_window_f64")
def set_samples(x_samples):
    raise RuntimeError("runs on the GPU workers")


@fiber_b200.device_body("table_mix_u32", source=TABLE_SRC, entry="table_mix_entry", args="<i8", result="<u4",
                        shared=("table", "<u4"))
def table_mix_u32(table, i):
    return int(table[splitmix64(i & ((1 << 64) - 1)) % len(table)]) ^ (i & 0xFFFFFFFF)


BAD_MODULE = bodies.compile_module("bad_broadcast_bodies", BAD_SRC)


# ---- NumPy restatements ---------------------------------------------------------------------------------------------
def nearest_np(points, centroids):
    """float32 in the device's order: for every k, d2 = (((0 + t0^2) + t1^2) + ...) with each operation rounded to
    float32; a strictly smaller d2 replaces the best, so the lowest k wins ties."""
    p = np.ascontiguousarray(points).view(np.float32).reshape(-1, 16)
    c = np.ascontiguousarray(centroids).view(np.float32).reshape(-1, 16)
    best = np.zeros(len(p), np.float32)
    best_k = np.zeros(len(p), np.uint32)
    for k in range(len(c)):
        d2 = np.zeros(len(p), np.float32)
        for d in range(16):
            t = p[:, d] - c[k, d]
            d2 = d2 + t * t
        upd = d2 < best if k else np.ones(len(p), bool)
        best = np.where(upd, d2, best)
        best_k = np.where(upd, np.uint32(k), best_k)
    out = np.empty(len(p), NEAREST_RES)
    out["k"], out["d2"] = best_k, best
    return out


def kde_np(widths, samples):
    xs = np.ascontiguousarray(samples).view(np.float64).reshape(-1, 2)
    out = np.empty(len(widths), KDE_RES)
    for i, h in enumerate(np.asarray(widths, np.float64)):
        q = (0.0 - xs) / h
        k = int(np.sum(~np.any(np.abs(q) > 0.5, axis=1)))
        out[i] = (h, (k / len(xs)) / h)
    return out


def table_mix_np(idx, table):
    u = np.asarray(idx, dtype=np.int64).view(np.uint64)
    with np.errstate(over="ignore"):
        j = splitmix_np(u) % np.uint64(len(table))
    return (np.asarray(table, np.uint32)[j] ^ (u & np.uint64(0xFFFFFFFF)).astype(np.uint32)).astype(np.uint32)


# ---- seeded inputs --------------------------------------------------------------------------------------------------
def points(n, seed=0):
    rng = np.random.default_rng(seed)
    a = np.empty(n, POINT)
    a["p"] = rng.standard_normal((n, 16)).astype(np.float32)
    return a


def centroids(k, seed=1):
    rng = np.random.default_rng(seed)
    c = np.empty(k, CENTROID)
    c["c"] = rng.standard_normal((k, 16)).astype(np.float32)
    return c


def table(n, seed=2):
    return np.random.default_rng(seed).integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)
