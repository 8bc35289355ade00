"""Record bodies defined OUTSIDE libfiber_b200: fixed-size argument and result structs (FBR_EXPORT_RECORD_BODY).

Each CUDA source below is compiled by ``fiber_b200.device_body(name, source=..., args=<dtype>, result=<dtype>)`` into
a body module under ``fiber_b200/_lib/bodies/`` and registered at import time.  Next to each body: its Python
definition (what the reference would run) and a NumPy restatement the GPU results are compared against bit for bit.
Floating-point bodies use explicitly rounded operations (``__dmul_rn`` / ``__dadd_rn`` / ``__dsqrt_rn``): no
contraction into FMAs, so every result is the correctly rounded IEEE value NumPy computes too.
"""
import math

import numpy as np

import fiber_b200
from fiber_b200 import bodies

POLAR_ARG = np.dtype([("x", "<f8"), ("y", "<f8")])
POLAR_RES = np.dtype([("r2", "<f8"), ("r", "<f8")])

POLAR_SRC = r'''
#include "fiber_b200_body.cuh"

// (x, y) -> (x*x + y*y, sqrt(x*x + y*y)), every operation correctly rounded
struct Polar {
    struct Arg { double x, y; };
    struct Res { double r2, r; };
    static constexpr bool kIndexArg = false;
    static constexpr bool kCanFault = false;
    __device__ static __forceinline__ void run(const Arg& a, Res& r, uint64_t, const fbr::ErrSink&, uint32_t) {
        const double r2 = __dadd_rn(__dmul_rn(a.x, a.x), __dmul_rn(a.y, a.y));
        r.r2 = r2;
        r.r = __dsqrt_rn(r2);
    }
};
FBR_EXPORT_RECORD_BODY(Polar, "polar_f64", polar_entry, 0)

// the same, but a task whose y is -1.0 "kills its worker" on its first attempt (the unit is lost and re-dispatched)
struct FaultPolar {
    using Arg = Polar::Arg;
    using Res = Polar::Res;
    static constexpr bool kIndexArg = false;
    static constexpr bool kCanFault = true;
    __device__ static __forceinline__ void run(const Arg& a, Res& r, uint64_t gidx, const fbr::ErrSink& es, uint32_t attempt) {
        if (attempt == 0 && a.y == -1.0) es.report(fbr::TASK_FAULT, gidx);
        Polar::run(a, r, gidx, es, attempt);
    }
};
FBR_EXPORT_RECORD_BODY(FaultPolar, "fault_polar_f64", fault_polar_entry, 0)
'''

MIX_ARG = np.dtype([("a", "<i4"), ("b", "<i4"), ("c", "<i4")])
MIX_RES = np.dtype([("p", "<i4"), ("q", "<i4"), ("r", "<i4")])

MIX_SRC = r'''
#include "fiber_b200_body.cuh"

// three int32 -> (a + b, b ^ c, 3a - c), wrapping modulo 2^32: 12 B -> 12 B records
struct MixI32x3 {
    struct Arg { int32_t a, b, c; };
    struct Res { int32_t p, q, r; };
    static constexpr bool kIndexArg = false;
    static constexpr bool kCanFault = false;
    __device__ static __forceinline__ void run(const Arg& x, Res& y, uint64_t, const fbr::ErrSink&, uint32_t) {
        const uint32_t a = (uint32_t)x.a, b = (uint32_t)x.b, c = (uint32_t)x.c;
        y.p = (int32_t)(a + b);
        y.q = (int32_t)(b ^ c);
        y.r = (int32_t)(3u * a - c);
    }
};
FBR_EXPORT_RECORD_BODY(MixI32x3, "mix_i32x3", mix_entry, 0)
'''

ROW_ARG = np.dtype([("row", "<u4", (256,))])
ROW_RES = np.dtype([("sum", "<u8"), ("min", "<u4"), ("max", "<u4"), ("argmax", "<u4"), ("pad", "<u4")])

ROW_SRC = r'''
#include "fiber_b200_body.cuh"

// a row of 256 uint32 -> (sum, min, max, first index of the max, 0): 1024 B -> 24 B records.  The row is read from
// shared memory in 16 B vectors (a lane's record starts 1024 B after its neighbour's: word loads would all hit one bank).
struct RowStatsU32 {
    struct Arg { uint32_t row[256]; };
    struct Res { uint64_t sum; uint32_t mn, mx, argmax, pad; };
    static constexpr bool kIndexArg = false;
    static constexpr bool kCanFault = false;
    __device__ static __forceinline__ void run(const Arg& a, Res& r, uint64_t, const fbr::ErrSink&, uint32_t) {
        const uint4* v = reinterpret_cast<const uint4*>(a.row);
        uint64_t s = 0;
        uint32_t mn = 0xffffffffu, mx = 0u, am = 0u;
#pragma unroll 4
        for (uint32_t k = 0; k < 64; ++k) {
            const uint4 q = v[k];
            const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                s += w[j];
                mn = min(mn, w[j]);
                if (w[j] > mx || (k == 0 && j == 0)) { mx = w[j]; am = 4 * k + j; }
            }
        }
        r.sum = s; r.mn = mn; r.mx = mx; r.argmax = am; r.pad = 0;
    }
};
FBR_EXPORT_RECORD_BODY(RowStatsU32, "row_stats_u32", row_stats_entry, 0)
'''

PAIR_RES = np.dtype([("a", "<u8"), ("b", "<u8")])

PAIR_SRC = r'''
#include "fiber_b200_body.cuh"

// index -> (splitmix64(i), splitmix64(i ^ 0x5851F42D4C957F2D)): maps over range() need no argument bytes
struct SplitmixPair {
    using Arg = int64_t;
    struct Res { uint64_t a, b; };
    static constexpr bool kIndexArg = true;
    static constexpr bool kCanFault = false;
    __device__ static __forceinline__ void run(const Arg& i, Res& r, uint64_t, const fbr::ErrSink&, uint32_t) {
        r.a = fbr::splitmix64((uint64_t)i);
        r.b = fbr::splitmix64((uint64_t)i ^ 0x5851F42D4C957F2Dull);
    }
};
FBR_EXPORT_RECORD_BODY(SplitmixPair, "splitmix_pair", splitmix_pair_entry, FBR_BODY_INDEX_ARG)
'''

SCALE5_ARG = np.dtype([("v", "<f8", (5,))])
SCALE5_RES = np.dtype([("w", "<f8", (5,))])

SCALE5_SRC = r'''
#include "fiber_b200_body.cuh"

// five float64 -> 2 v[k] + k: 40 B -> 40 B records (slots of odd multiples of 8 bytes)
struct Scale5 {
    struct Arg { double v[5]; };
    struct Res { double w[5]; };
    static constexpr bool kIndexArg = false;
    static constexpr bool kCanFault = false;
    __device__ static __forceinline__ void run(const Arg& a, Res& r, uint64_t, const fbr::ErrSink&, uint32_t) {
#pragma unroll
        for (int k = 0; k < 5; ++k) r.w[k] = __dadd_rn(__dmul_rn(a.v[k], 2.0), (double)k);
    }
};
FBR_EXPORT_RECORD_BODY(Scale5, "scale5_f64", scale5_entry, 0)
'''

# Hand-written descriptors that break the record-body rules; registration must refuse every one of them.  (The macro
# checks the same rules at compile time, so a real body cannot get there.)
BAD_SRC = r'''
#include "fiber_b200_body.cuh"

struct Ok {
    struct Arg { float x; };
    struct Res { float y; };
    static constexpr bool kIndexArg = false;
    static constexpr bool kCanFault = false;
    __device__ static void run(const Arg& a, Res& r, uint64_t, const fbr::ErrSink&, uint32_t) { r.y = a.x; }
};
#define BAD_BODY(entry, name, ab, rb, kind, flags)                                                                 \
    extern "C" const fbr_body_module_t* entry(void) {                                                            \
        static const fbr_body_module_t m = {FBR_BODY_MODULE_ABI, (uint32_t)sizeof(fbr::WaveParams), name, ab, rb, \
                                            kind, (flags) | FBR_BODY_RECORD, 16u,                                \
                                            fbr_body_export::launch_record<Ok>, fbr_body_export::occupancy_record<Ok>}; \
        return &m;                                                                                               \
    }
BAD_BODY(bad_arg6, "bad_arg6", 6u, 4u, FBR_RES_BYTES, 0)
BAD_BODY(bad_res6, "bad_res6", 4u, 6u, FBR_RES_BYTES, 0)
BAD_BODY(bad_summable, "bad_summable", 4u, 4u, FBR_RES_BYTES, FBR_BODY_SUMMABLE)
BAD_BODY(bad_shared, "bad_shared", 4u, 4u, FBR_RES_BYTES, FBR_BODY_NEEDS_SHARED)
BAD_BODY(bad_oversize, "bad_oversize", 8192u, 4u, FBR_RES_BYTES, 0)
BAD_BODY(bad_twin, "bad_twin", 64u, 4u, FBR_RES_BITS8, 0)
BAD_BODY(ok_f32, "ok_f32", 4u, 4u, FBR_RES_BYTES, 0)
'''


@fiber_b200.device_body("polar_f64", source=POLAR_SRC, entry="polar_entry", args=POLAR_ARG, result=POLAR_RES)
def polar_f64(x, y):
    r2 = x * x + y * y
    return (r2, math.sqrt(r2))


@fiber_b200.device_body("fault_polar_f64", source=POLAR_SRC, entry="fault_polar_entry", args=POLAR_ARG, result=POLAR_RES)
def fault_polar_f64(x, y):
    return polar_f64(x, y)


def _i32(v):
    v &= 0xFFFFFFFF
    return v - (1 << 32) if v >= (1 << 31) else v


@fiber_b200.device_body("mix_i32x3", source=MIX_SRC, entry="mix_entry", args=MIX_ARG, result=MIX_RES)
def mix_i32x3(a, b, c):
    return (_i32(a + b), _i32(b ^ c), _i32(3 * a - c))


@fiber_b200.device_body("row_stats_u32", source=ROW_SRC, entry="row_stats_entry", args=ROW_ARG, result=ROW_RES)
def row_stats_u32(row):
    row = [int(v) for v in row]
    mx = max(row)
    return (sum(row), min(row), mx, row.index(mx), 0)


_M64 = (1 << 64) - 1


def splitmix64(x):
    z = (x + 0x9E3779B97F4A7C15) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


@fiber_b200.device_body("splitmix_pair", source=PAIR_SRC, entry="splitmix_pair_entry", args="<i8", result=PAIR_RES)
def splitmix_pair(i):
    u = i & _M64
    return (splitmix64(u), splitmix64(u ^ 0x5851F42D4C957F2D))


@fiber_b200.device_body("scale5_f64", source=SCALE5_SRC, entry="scale5_entry", args=SCALE5_ARG, result=SCALE5_RES)
def scale5_f64(v):
    return [x * 2.0 + k for k, x in enumerate(v)]


BAD_MODULE = bodies.compile_module("bad_record_bodies", BAD_SRC)


# ---- NumPy restatements ---------------------------------------------------------------------------------------------
def polar_np(args):
    x, y = args["x"], args["y"]
    out = np.empty(len(args), POLAR_RES)
    out["r2"] = x * x + y * y
    out["r"] = np.sqrt(out["r2"])
    return out


def mix_np(args):
    a, b, c = (args[k].astype(np.int64).view(np.uint64) for k in "abc")
    out = np.empty(len(args), MIX_RES)
    m = np.uint64(0xFFFFFFFF)
    out["p"] = ((a + b) & m).astype(np.uint32).view(np.int32)
    out["q"] = ((b ^ c) & m).astype(np.uint32).view(np.int32)
    out["r"] = ((np.uint64(3) * a - c) & m).astype(np.uint32).view(np.int32)
    return out


def row_stats_np(args):
    rows = args["row"]
    out = np.zeros(len(args), ROW_RES)
    out["sum"] = rows.sum(axis=1, dtype=np.uint64)
    out["min"] = rows.min(axis=1)
    out["max"] = rows.max(axis=1)
    out["argmax"] = rows.argmax(axis=1)
    return out


def splitmix_np(x):
    z = np.asarray(x, dtype=np.uint64) + np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def splitmix_pair_np(idx):
    u = np.asarray(idx, dtype=np.int64).view(np.uint64)
    out = np.empty(len(u), PAIR_RES)
    with np.errstate(over="ignore"):
        out["a"] = splitmix_np(u)
        out["b"] = splitmix_np(u ^ np.uint64(0x5851F42D4C957F2D))
    return out


def scale5_np(args):
    out = np.empty(len(args), SCALE5_RES)
    out["w"] = args["v"] * 2.0 + np.arange(5, dtype=np.float64)
    return out


# ---- seeded inputs --------------------------------------------------------------------------------------------------
def polar_args(n, seed=0):
    rng = np.random.default_rng(seed)
    a = np.empty(n, POLAR_ARG)
    a["x"] = rng.standard_normal(n) * 1e3
    a["y"] = rng.standard_normal(n) * 1e-3
    return a


def mix_args(n, seed=0):
    rng = np.random.default_rng(seed)
    a = np.empty(n, MIX_ARG)
    for k in "abc":
        a[k] = rng.integers(-2 ** 31, 2 ** 31, n, dtype=np.int64).astype(np.int32)
    return a


def row_args(n, seed=0):
    rng = np.random.default_rng(seed)
    a = np.empty(n, ROW_ARG)
    a["row"] = rng.integers(0, 2 ** 32, (n, 256), dtype=np.uint64).astype(np.uint32)
    return a


def scale5_args(n, seed=0):
    rng = np.random.default_rng(seed)
    a = np.empty(n, SCALE5_ARG)
    a["v"] = rng.standard_normal((n, 5))
    return a
