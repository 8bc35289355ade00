"""Keyed fold bodies: fold bodies that also define ``key()``, so ``Pool.fold_by_key`` folds the results of each key on the
device.

Each CUDA source below is compiled by ``fiber_b200.device_body(name, source=..., ...)`` and registered at import time.  Next
to each body: a Python restatement of its ``run`` (``*_run``, records as tuples or lists), its ``combine`` and its ``key``,
and ``keyed_tree``, the order of FBR_FOLD_KEYS on one worker, which the GPU results are compared against bit for bit.  Float
bodies round every operation explicitly (``__dadd_rn``, ``__fadd_rn`` and friends), so Python floats and NumPy float32
scalars restate them exactly.
"""
import numpy as np

import fiber_b200
import fiber_b200.bodies

from .fold_bodies import tree

M64 = (1 << 64) - 1
M32 = (1 << 32) - 1


def keyed_tree(results, key, combine, identity, n_keys):
    """FBR_FOLD_KEYS on one worker: record k = tree() of the results whose key is k, in task order; identity() for none."""
    groups = [[] for _ in range(n_keys)]
    for r in results:
        groups[key(r)].append(r)
    out = [tree(g, combine) for g in groups]
    return [identity if r is None else r for r in out], [len(g) for g in groups]


def keyed_blocks(results, key, combine, identity, n_keys, cuts):
    """FBR_FOLD_KEYS on several workers: each block [lo, hi) of ``cuts`` folds its own keys, and record k is tree() over the
    totals of the blocks where k has a task, in block order."""
    totals = [[] for _ in range(n_keys)]
    counts = [0] * n_keys
    for lo, hi in cuts:
        recs, cnt = keyed_tree(results[lo:hi], key, combine, identity, n_keys)
        for k in range(n_keys):
            if cnt[k]:
                totals[k].append(recs[k])
                counts[k] += cnt[k]
    out = [tree(t, combine) for t in totals]
    return [identity if r is None else r for r in out], counts


SRC = r'''
#include "fiber_b200_body.cuh"

// the sum and number of the values of each label: the key is the argument's own label, so a test picks the keys
struct LabelSum {
    struct Arg { uint32_t label, v; };
    struct Res { uint64_t sum; uint32_t key, n; };
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static void run(const Arg& a, Res& r, uint64_t, const fbr::ErrSink&, uint32_t) { r = Res{a.v, a.label, 1u}; }
    __host__ __device__ static Res identity() { return Res{0, 0, 0}; }
    __device__ static __forceinline__ void combine(Res& acc, const Res& x) { acc.sum += x.sum; acc.n += x.n; }
    __device__ static uint32_t key(const Res& r) { return r.key; }
};
FBR_EXPORT_RECORD_BODY(LabelSum, "label_sum_u64", label_sum_entry, 0)

// count, mean and M2 of a float64 column per label (Chan et al.'s merge): a float combine whose bits depend on the order
struct ClassMoments {
    struct Arg { double x; uint32_t label, pad; };
    struct Res { double n, mean, m2; uint32_t key, pad; };
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static void run(const Arg& a, Res& r, uint64_t, const fbr::ErrSink&, uint32_t) { r = Res{1.0, a.x, 0.0, a.label, 0u}; }
    __host__ __device__ static Res identity() { return Res{0.0, 0.0, 0.0, 0u, 0u}; }
    __device__ static __forceinline__ void combine(Res& acc, const Res& x) {
        if (x.n == 0.0) return;
        if (acc.n == 0.0) { acc = x; return; }
        const double n = __dadd_rn(acc.n, x.n), d = __dsub_rn(x.mean, acc.mean);
        const double mean = __dadd_rn(acc.mean, __ddiv_rn(__dmul_rn(d, x.n), n));
        const double m2 = __dadd_rn(__dadd_rn(acc.m2, x.m2), __ddiv_rn(__dmul_rn(__dmul_rn(d, d), __dmul_rn(acc.n, x.n)), n));
        acc.n = n; acc.mean = mean; acc.m2 = m2;
    }
    __device__ static uint32_t key(const Res& r) { return r.key; }
};
FBR_EXPORT_RECORD_BODY(ClassMoments, "class_moments_f64", class_moments_entry, 0)

// the update step of k-means: the key is the centroid nearest to p (the lowest index on a tie), the record the point
// itself and a count of one; the fold per key sums each centroid's points in float32
struct KmeansStep {
    struct Arg { float p[16]; };
    struct Res { float s[16]; uint32_t n, key; };
    struct alignas(16) Centroid { float c[16]; };
    using Shared = Centroid;
    static constexpr uint32_t kSharedStage = 16384;
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static void run(const Arg& a, Res& r, const fbr::Broadcast<Shared>& sh, uint64_t, const fbr::ErrSink&, uint32_t) {
        uint32_t best_k = 0;
        float best = 0.0f;
        for (uint32_t k = 0; k < (uint32_t)sh.n; ++k) {
            float d2 = 0.0f;
#pragma unroll
            for (int d = 0; d < 16; ++d) {
                const float t = __fsub_rn(a.p[d], sh.data[k].c[d]);
                d2 = __fadd_rn(d2, __fmul_rn(t, t));
            }
            if (k == 0 || d2 < best) { best = d2; best_k = k; }
        }
        for (int d = 0; d < 16; ++d) r.s[d] = a.p[d];
        r.n = 1u;
        r.key = best_k;
    }
    __host__ __device__ static Res identity() { return Res{}; }
    __device__ static __forceinline__ void combine(Res& acc, const Res& x) {
        for (int d = 0; d < 16; ++d) acc.s[d] = __fadd_rn(acc.s[d], x.s[d]);
        acc.n += x.n;
    }
    __device__ static uint32_t key(const Res& r) { return r.key; }
};
FBR_EXPORT_RECORD_BODY(KmeansStep, "kmeans_step_f32", kmeans_step_entry, 0)

// a 1 KB record: a byte string's histogram of byte % 255 per label, the label taken from the head record
struct LabelHist {
    using Item = uint8_t;
    struct Arg { uint32_t label; };
    struct Res { uint32_t c[255]; uint32_t key; };
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static void run(const Arg& a, const fbr::Items<uint8_t>& x, Res& r, uint64_t, const fbr::ErrSink&, uint32_t) {
        for (uint32_t k = 0; k < 255; ++k) r.c[k] = 0;
        for (uint64_t k = 0; k < x.n; ++k) r.c[x.data[k] % 255u] += 1u;
        r.key = a.label;
    }
    __host__ __device__ static Res identity() { return Res{}; }
    __device__ static __forceinline__ void combine(Res& acc, const Res& x) {
        for (uint32_t k = 0; k < 255; ++k) acc.c[k] += x.c[k];
    }
    __device__ static uint32_t key(const Res& r) { return r.key; }
};
FBR_EXPORT_RECORD_BODY(LabelHist, "label_hist_1k", label_hist_entry, 0)

// a 16 KB record on a warp: word j of task (label, seed) is seed * (j + 1) mod 2^32, summed per label
struct WideSum {
    struct Arg { uint32_t label, seed, pad[2]; };
    struct Res { uint32_t key, pad[3]; uint32_t v[4092]; };
    static constexpr uint32_t kGroup = 32;
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static void run(const Arg& a, Res& r, const fbr::Group<32>& g, uint64_t, const fbr::ErrSink&, uint32_t) {
        for (uint32_t j = g.rank; j < 4092; j += g.size) r.v[j] = a.seed * (j + 1u);
        if (g.rank == 0) { r.key = a.label; r.pad[0] = r.pad[1] = r.pad[2] = 0; }
    }
    __host__ __device__ static Res identity() { return Res{}; }
    __device__ static __forceinline__ void combine(Res& acc, const Res& x) {
        for (uint32_t j = 0; j < 4092; ++j) acc.v[j] += x.v[j];
    }
    __device__ static uint32_t key(const Res& r) { return r.key; }
};
FBR_EXPORT_RECORD_BODY(WideSum, "wide_sum_16k", wide_sum_entry, 0)

// the label sum of range() indices, key i % 7, but every task whose index is 5 mod 997 "kills its worker" on its first
// attempt and leaves a wrong record with key 0 behind: only the unit's re-dispatch gives the right records
struct FaultLabel {
    using Arg = int64_t;
    struct Res { uint64_t sum; uint32_t key, n; };
    static constexpr bool kIndexArg = true, kCanFault = true;
    __device__ static void run(const Arg& a, Res& r, uint64_t gidx, const fbr::ErrSink& es, uint32_t attempt) {
        r = Res{(uint64_t)a * 3u + 1u, (uint32_t)(a % 7), 1u};
        if (attempt == 0 && gidx % 997 == 5) {
            es.report(fbr::TASK_FAULT, gidx);
            r = Res{0x5eed, 0u, 1u};
        }
    }
    __host__ __device__ static Res identity() { return Res{0, 0, 0}; }
    __device__ static __forceinline__ void combine(Res& acc, const Res& x) { acc.sum += x.sum; acc.n += x.n; }
    __device__ static uint32_t key(const Res& r) { return r.key; }
};
FBR_EXPORT_RECORD_BODY(FaultLabel, "fault_label_u64", fault_label_entry, FBR_BODY_INDEX_ARG)
'''

# ---- label_sum_u64 ----------------------------------------------------------------------------------------------------
LABEL_ARG = np.dtype([("label", "<u4"), ("v", "<u4")])
LABEL_RES = np.dtype([("sum", "<u8"), ("key", "<u4"), ("n", "<u4")])


@fiber_b200.device_body("label_sum_u64", source=SRC, entry="label_sum_entry", args=LABEL_ARG, result=LABEL_RES)
def label_sum_u64(label, v):
    return (v, label, 1)


def label_combine(a, b):
    return ((a[0] + b[0]) & M64, a[1], (a[2] + b[2]) & M32)


LABEL_ID = (0, 0, 0)

# ---- class_moments_f64 ------------------------------------------------------------------------------------------------
MOMENTS_ARG = np.dtype([("x", "<f8"), ("label", "<u4"), ("pad", "<u4")])
MOMENTS_RES = np.dtype([("n", "<f8"), ("mean", "<f8"), ("m2", "<f8"), ("key", "<u4"), ("pad", "<u4")])


@fiber_b200.device_body("class_moments_f64", source=SRC, entry="class_moments_entry", args=MOMENTS_ARG, result=MOMENTS_RES)
def class_moments_f64(x, label, pad=0):
    return (1.0, float(x), 0.0, label, 0)


def moments_combine(a, b):
    if b[0] == 0.0:
        return a
    if a[0] == 0.0:
        return b
    n = a[0] + b[0]
    d = b[1] - a[1]
    mean = a[1] + (d * b[0]) / n
    m2 = (a[2] + b[2]) + ((d * d) * (a[0] * b[0])) / n
    return (n, mean, m2, a[3], a[4])


MOMENTS_ID = (0.0, 0.0, 0.0, 0, 0)

# ---- kmeans_step_f32 --------------------------------------------------------------------------------------------------
POINT = np.dtype([("p", "<f4", (16,))])
CENTROID = np.dtype([("c", "<f4", (16,))])
KMEANS_RES = np.dtype([("s", "<f4", (16,)), ("n", "<u4"), ("key", "<u4")])


@fiber_b200.device_body("kmeans_step_f32", source=SRC, entry="kmeans_step_entry", args=POINT, result=KMEANS_RES,
                        shared=("centroids", CENTROID))
def kmeans_step_f32(centroids, p):
    return kmeans_run(np.ascontiguousarray(centroids).view(np.float32).reshape(-1, 16), p)


def kmeans_run(c, p):
    p = np.asarray(p, np.float32).reshape(16)
    best_k, best = 0, None
    for k, row in enumerate(c):
        d2 = np.float32(0.0)
        for d in range(16):
            t = p[d] - row[d]                     # float32 scalars: every operation rounds to float32
            d2 = d2 + t * t
        if best is None or d2 < best:
            best_k, best = k, d2
    return (p.tolist(), 1, best_k)


def kmeans_keys(c, pts):
    """The nearest centroid of every point, vectorised in the body's order of operations (float32, dimension order)."""
    d2 = np.zeros((len(pts), len(c)), np.float32)
    for d in range(16):
        t = pts[:, d:d + 1] - c[None, :, d]
        d2 = d2 + t * t
    return np.argmin(d2, axis=1)                # the first minimum: the lowest index on a tie


def kmeans_combine(a, b):
    s = (np.asarray(a[0], np.float32) + np.asarray(b[0], np.float32)).tolist()
    return (s, (a[1] + b[1]) & M32, a[2])


KMEANS_ID = ([0.0] * 16, 0, 0)


@fiber_b200.device_initializer("kmeans_step_f32")
def set_centroids(centroids):
    raise RuntimeError("runs on the GPU workers")


# ---- label_hist_1k ----------------------------------------------------------------------------------------------------
HIST_RES = np.dtype([("c", "<u4", (255,)), ("key", "<u4")])


@fiber_b200.device_body("label_hist_1k", source=SRC, entry="label_hist_entry", args=np.dtype([("label", "<u4")]),
                        items=("x", "u1"), result=HIST_RES)
def label_hist_1k(x, label):
    c = np.bincount(np.frombuffer(bytes(x), np.uint8) % 255, minlength=255).astype(np.uint32).tolist()
    return (c, label)


def hist_combine(a, b):
    return ([(x + y) & M32 for x, y in zip(a[0], b[0])], a[1])


HIST_ID = ([0] * 255, 0)

# ---- wide_sum_16k -----------------------------------------------------------------------------------------------------
WIDE_ARG = np.dtype([("label", "<u4"), ("seed", "<u4"), ("pad", "<u4", (2,))])
WIDE_RES = np.dtype([("key", "<u4"), ("pad", "<u4", (3,)), ("v", "<u4", (4092,))])


@fiber_b200.device_body("wide_sum_16k", source=SRC, entry="wide_sum_entry", args=WIDE_ARG, result=WIDE_RES)
def wide_sum_16k(label, seed, pad=(0, 0)):
    return (label, [0, 0, 0], wide_words(seed).tolist())


def wide_words(seed):
    return (np.uint64(seed) * np.arange(1, 4093, dtype=np.uint64) & np.uint64(M32)).astype(np.uint32)


def wide_combine(a, b):
    return (a[0], a[1], ((np.asarray(a[2], np.uint64) + np.asarray(b[2], np.uint64)) & np.uint64(M32)).tolist())


WIDE_ID = (0, [0, 0, 0], [0] * 4092)

# ---- fault_label_u64 --------------------------------------------------------------------------------------------------


@fiber_b200.device_body("fault_label_u64", source=SRC, entry="fault_label_entry", args="<i8", result=LABEL_RES)
def fault_label_u64(i):
    return ((3 * i + 1) & M64, i % 7, 1)

# ---- hand-written descriptors: registration must refuse the bad ones ----------------------------------------------------
BAD_SRC = r'''
#include "fiber_b200_body.cuh"

struct Sum {
    using Arg = int64_t;
    struct Res { uint64_t s; };
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static void run(const Arg& a, Res& r, uint64_t, const fbr::ErrSink&, uint32_t) { r.s = (uint64_t)a; }
    __host__ __device__ static Res identity() { return Res{0}; }
    __device__ static __forceinline__ void combine(Res& acc, const Res& x) { acc.s += x.s; }
    __device__ static uint32_t key(const Res& r) { return (uint32_t)(r.s & 3u); }
};
static const Sum::Res kZero{0};

#define KEYED_DESC(entry, flags, fold, id, keys, segs)                                                              \
    extern "C" const fbr_body_module_t* entry(void) {                                                            \
        static const fbr_body_module_t m = {FBR_BODY_MODULE_ABI, (uint32_t)sizeof(fbr::WaveParams), #entry, 8u, 8u,  \
                                            FBR_RES_BYTES, (flags), 1024u, fbr_body_export::launch_record<Sum>,   \
                                            fbr_body_export::occupancy_record<Sum>, 0u, 0u, 0u, 0u, 0u, 0u, {0u, 0u, 0u}, \
                                            (fold), (id), (id) ? 8u : 0u, fbr_body_export::launch_scan<Sum>, (keys), (segs)}; \
        return &m;                                                                                               \
    }
#define RB (FBR_BODY_RECORD)
#define FOLD fbr_body_export::launch_fold<Sum>
#define KEYS fbr_body_export::launch_keys<Sum>
#define SEGS fbr_body_export::launch_fold_segments<Sum>
KEYED_DESC(bad_keyed_no_fold, RB | FBR_BODY_KEYED, nullptr, nullptr, KEYS, SEGS)
KEYED_DESC(bad_keyed_no_keys, RB | FBR_BODY_FOLD | FBR_BODY_SCAN | FBR_BODY_KEYED, FOLD, &kZero, nullptr, SEGS)
KEYED_DESC(bad_keyed_no_segments, RB | FBR_BODY_FOLD | FBR_BODY_SCAN | FBR_BODY_KEYED, FOLD, &kZero, KEYS, nullptr)
KEYED_DESC(ok_keyed, RB | FBR_BODY_FOLD | FBR_BODY_SCAN | FBR_BODY_KEYED, FOLD, &kZero, KEYS, SEGS)
KEYED_DESC(ok_keyed_unflagged, RB | FBR_BODY_FOLD | FBR_BODY_SCAN, FOLD, &kZero, KEYS, SEGS)   // entries ignored: a fold body
'''
BAD_MODULE = fiber_b200.bodies.compile_module("keyed_bad_descriptors", BAD_SRC)

# restatements by body name: (combine, identity, key of a result record)
RESTATED = {
    "label_sum_u64": (label_combine, LABEL_ID),
    "class_moments_f64": (moments_combine, MOMENTS_ID),
    "kmeans_step_f32": (kmeans_combine, KMEANS_ID),
    "label_hist_1k": (hist_combine, HIST_ID),
    "wide_sum_16k": (wide_combine, WIDE_ID),
    "fault_label_u64": (label_combine, LABEL_ID),
}
KEY_OF = {"label_sum_u64": lambda r: r[1], "class_moments_f64": lambda r: r[3], "kmeans_step_f32": lambda r: r[2],
          "label_hist_1k": lambda r: r[1], "wide_sum_16k": lambda r: r[0], "fault_label_u64": lambda r: r[1]}
