"""Scan (accumulate) test bodies and the Python restatement of FBR_SCAN's prefix folds.

Every fold body of ``tests/fold_bodies.py`` accumulates as it is.  Two more bodies cover what those do not:
``affine_f64`` composes affine maps (a non-commutative combine, so any reordering shows) and ``mix4k_u32`` is a group body
(G = 32) with a 4 KB ``Res``, which the scan kernels combine in global memory rather than in registers.

``prefix_folds`` restates the order of FBR_SCAN (include/fiber_b200.h) with the levels of complete aligned subtrees, and
``block_prefix_folds`` restates it over a block cut.
"""
import numpy as np

import fiber_b200
import fiber_b200.bodies
from tests.fold_bodies import tree

M32 = (1 << 32) - 1

SCAN_SRC = r'''
#include "fiber_b200_body.cuh"

// h_t = a_t h_{t-1} + b_t as a map (a, b); acc (+) x applies acc first, then x.  Every operation is rounded explicitly
struct Affine {
    struct Arg { double a, b; };
    struct Res { double a, b; };
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static void run(const Arg& x, Res& r, uint64_t, const fbr::ErrSink&, uint32_t) { r = Res{x.a, x.b}; }
    __host__ __device__ static Res identity() { return Res{1.0, 0.0}; }
    __device__ static __forceinline__ void combine(Res& acc, const Res& x) {
        const double a = __dmul_rn(x.a, acc.a), b = __dadd_rn(__dmul_rn(x.a, acc.b), x.b);
        acc.a = a; acc.b = b;
    }
};
FBR_EXPORT_RECORD_BODY(Affine, "affine_f64", affine_entry, 0)

// 1024 uint32 lanes of a range() index on a warp; the combine is order-sensitive (acc * 31 + x per lane)
struct Mix4k {
    using Arg = int64_t;
    struct Res { uint32_t c[1024]; };
    static constexpr uint32_t kGroup = 32;
    static constexpr bool kIndexArg = true, kCanFault = false;
    __device__ static void run(const Arg& i, Res& r, const fbr::Group<32>& g, uint64_t, const fbr::ErrSink&, uint32_t) {
        for (uint32_t k = g.rank; k < 1024; k += g.size) r.c[k] = (uint32_t)i * 2654435761u + k;
    }
    __host__ __device__ static Res identity() { return Res{}; }
    __device__ static __forceinline__ void combine(Res& acc, const Res& x) {
        for (uint32_t k = 0; k < 1024; ++k) acc.c[k] = acc.c[k] * 31u + x.c[k];
    }
};
FBR_EXPORT_RECORD_BODY(Mix4k, "mix4k_u32", mix4k_entry, FBR_BODY_INDEX_ARG)
'''

AFFINE_ARG = np.dtype([("a", "<f8"), ("b", "<f8")])
AFFINE_RES = np.dtype([("a", "<f8"), ("b", "<f8")])


@fiber_b200.device_body("affine_f64", source=SCAN_SRC, entry="affine_entry", args=AFFINE_ARG, result=AFFINE_RES)
def affine_f64(x):
    return (float(x[0]), float(x[1]))


def affine_combine(acc, x):
    return (x[0] * acc[0], x[0] * acc[1] + x[1])


AFFINE_ID = (1.0, 0.0)


@fiber_b200.device_body("mix4k_u32", source=SCAN_SRC, entry="mix4k_entry", args="<i8",
                        result=np.dtype([("c", "<u4", (1024,))]))
def mix4k_u32(i):
    return mix4k_run(i)


def mix4k_run(i):
    return tuple(((i * 2654435761) + np.arange(1024, dtype=np.uint64)).astype(np.uint32).tolist())


def mix4k_combine(acc, x):
    return tuple(((np.array(acc, np.uint64) * 31 + np.array(x, np.uint64)) & M32).astype(np.uint32).tolist())


# ---- the order of FBR_SCAN ----------------------------------------------------------------------------------------------
def levels_of(xs, combine):
    """Level k holds the len(xs) >> k complete aligned subtrees of 2^k records (level 0 is xs)."""
    lv = [list(xs)]
    while len(lv[-1]) >= 2:
        prev = lv[-1]
        lv.append([combine(prev[2 * j], prev[2 * j + 1]) for j in range(len(prev) // 2)])
    return lv


def wrap(lv, i, x, combine):
    """F_1 (+) (F_2 (+) ( ... (+) (F_k (+) x))), F_1 .. F_k the pieces of [0, i) given by the set bits of i."""
    acc, k = x, 0
    while i >> k:
        if (i >> k) & 1:
            acc = combine(lv[k][(i >> k) - 1], acc)
        k += 1
    return acc


def prefix_folds(xs, combine):
    """y[i] = tree(xs[0..i]) by the pieces form, popcount(i) combines per element."""
    lv = levels_of(xs, combine)
    return [wrap(lv, i, x, combine) for i, x in enumerate(lv[0])]


def block_prefix_folds(xs, bounds, combine):
    """FBR_SCAN over a block cut [(lo, hi), ...] in block order: task i of block b gets tree(t_0, ..., t_{b-1}, p_i)."""
    local = [prefix_folds(xs[lo:hi], combine) for lo, hi in bounds]
    totals = [p[-1] for p in local]
    out = []
    for b, p in enumerate(local):
        lv = levels_of(totals[:b], combine)
        out += [wrap(lv, b, y, combine) for y in p]
    return out


def tree_prefixes(xs, combine):
    """The definition, quadratic: tree(xs[0..i]) for every i."""
    return [tree(xs[:i + 1], combine) for i in range(len(xs))]


# ---- hand-written descriptors for the FBR_BODY_SCAN registration rules: all but the ok_* entries are refused -------------
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

#define SCAN_DESC(entry, name, flags, fold, id, scan)                                                                \
    extern "C" const fbr_body_module_t* entry(void) {                                                            \
        static const fbr_body_module_t m = {FBR_BODY_MODULE_ABI, (uint32_t)sizeof(fbr::WaveParams), name, 8u, 8u,  \
                                            FBR_RES_BYTES, (flags), 1024u, fbr_body_export::launch_record<Sum>,  \
                                            fbr_body_export::occupancy_record<Sum>, 0u, 0u, 0u, 0u, 0u, 0u,      \
                                            {0u, 0u, 0u}, (fold), (id), (id) ? 8u : 0u, (scan)};                 \
        return &m;                                                                                               \
    }
#define RB (FBR_BODY_RECORD)
#define FOLD fbr_body_export::launch_fold<Sum>
#define SCAN fbr_body_export::launch_scan<Sum>
SCAN_DESC(bad_scan_no_fold, "bad_scan_no_fold", RB | FBR_BODY_SCAN, nullptr, nullptr, SCAN)         // scan without a fold
SCAN_DESC(bad_scan_no_entry, "bad_scan_no_entry", RB | FBR_BODY_FOLD | FBR_BODY_SCAN, FOLD, &kZero, nullptr)
SCAN_DESC(ok_scan, "ok_scan", RB | FBR_BODY_FOLD | FBR_BODY_SCAN, FOLD, &kZero, SCAN)
// a fold descriptor written against the header before `scan`: it ends at identity_bytes and stays a fold body
extern "C" const fbr_body_module_t* ok_fold_without_scan(void) {
    static const fbr_body_module_t m = {FBR_BODY_MODULE_ABI, (uint32_t)sizeof(fbr::WaveParams), "ok_fold_without_scan", 8u,
                                        8u, FBR_RES_BYTES, RB | FBR_BODY_FOLD, 1024u, fbr_body_export::launch_record<Sum>,
                                        fbr_body_export::occupancy_record<Sum>, 0u, 0u, 0u, 0u, 0u, 0u, {0u, 0u, 0u}, FOLD,
                                        &kZero, 8u};
    return &m;
}
'''
BAD_MODULE = fiber_b200.bodies.compile_module("scan_bad_descriptors", BAD_SRC)
