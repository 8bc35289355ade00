"""Emit record bodies: every task returns a variable-length array (``using Out = ...`` in the body's struct).

Each CUDA source below is compiled by ``fiber_b200.device_body(name, source=..., out=...)`` and registered at import time.
Next to each body: its Python definition (what the reference would run) and a NumPy / Python restatement the GPU results
are compared against bit for bit.
"""
import numpy as np

import fiber_b200
import fiber_b200.bodies

TOKENS_SRC = r'''
#include "fiber_b200_body.cuh"

__device__ __forceinline__ bool ascii_space(uint8_t c) { return c == ' ' || (c >= '\t' && c <= '\r'); }

// the 32-bit FNV-1a of every token of a byte string, tokens split on ASCII whitespace
struct Tokens {
    using Item = uint8_t;
    using Arg = fbr::NoArg;
    using Out = uint32_t;
    using Res = fbr::NoRes;
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static __forceinline__ void run(const fbr::Items<Item>& x, fbr::Emit<Out>& y, uint64_t, const fbr::ErrSink&,
                                               uint32_t) {
        uint32_t h = 0x811c9dc5u;
        bool in = false;
        for (uint64_t k = 0; k < x.n; ++k) {
            const uint8_t c = x.data[k];
            if (ascii_space(c)) {
                if (in) y.push(h);
                in = false;
                h = 0x811c9dc5u;
            } else {
                h = (h ^ c) * 0x01000193u;
                in = true;
            }
        }
        if (in) y.push(h);
    }
};
FBR_EXPORT_RECORD_BODY(Tokens, "tokens_u32", tokens_entry, 0)

// the same, but a string that starts with '!' "kills its worker" on the first attempt: the unit is re-dispatched
struct FaultTokens : Tokens {
    static constexpr bool kCanFault = true;
    __device__ static __forceinline__ void run(const fbr::Items<Item>& x, fbr::Emit<Out>& y, uint64_t gidx, const fbr::ErrSink& es,
                                               uint32_t attempt) {
        if (attempt == 0 && x.n > 0 && x.data[0] == '!') es.report(fbr::TASK_FAULT, gidx);
        Tokens::run(x, y, gidx, es, attempt);
    }
};
FBR_EXPORT_RECORD_BODY(FaultTokens, "fault_tokens_u32", fault_tokens_entry, 0)

// the same fault, but the faulting attempt returns at once, having pushed nothing: its count mismatch must be discarded
// with the rest of the attempt
struct EarlyFaultTokens : Tokens {
    static constexpr bool kCanFault = true;
    __device__ static __forceinline__ void run(const fbr::Items<Item>& x, fbr::Emit<Out>& y, uint64_t gidx, const fbr::ErrSink& es,
                                               uint32_t attempt) {
        if (attempt == 0 && x.n > 0 && x.data[0] == '!') { es.report(fbr::TASK_FAULT, gidx); return; }
        Tokens::run(x, y, gidx, es, attempt);
    }
};
FBR_EXPORT_RECORD_BODY(EarlyFaultTokens, "early_fault_tokens_u32", early_fault_tokens_entry, 0)

// each byte once, but count() says one value more for strings whose length is 3 mod 5: such a task emits fewer values
// than its count pass gave
struct BadCount {
    using Item = uint8_t;
    using Arg = fbr::NoArg;
    using Out = uint32_t;
    using Res = fbr::NoRes;
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static uint64_t count(const fbr::Items<Item>& x, uint64_t) { return x.n + (x.n % 5 == 3 ? 1 : 0); }
    __device__ static __forceinline__ void run(const fbr::Items<Item>& x, fbr::Emit<Out>& y, uint64_t, const fbr::ErrSink&,
                                               uint32_t) {
        for (uint64_t k = 0; k < x.n; ++k) y.push(x.data[k]);
    }
};
FBR_EXPORT_RECORD_BODY(BadCount, "bad_count_u32", bad_count_entry, 0)
'''

PRIMES_SRC = r'''
#include "fiber_b200_body.cuh"

// prime factors of n with multiplicity, ascending (none for n < 2)
struct PrimeFactors {
    using Arg = int64_t;
    using Out = int64_t;
    using Res = fbr::NoRes;
    static constexpr bool kIndexArg = true, kCanFault = false;
    __device__ static __forceinline__ void run(const Arg& a, fbr::Emit<Out>& y, uint64_t, const fbr::ErrSink&, uint32_t) {
        int64_t n = a;
        if (n < 2) return;
        while ((n & 1) == 0) { y.push(2); n >>= 1; }
        for (int64_t p = 3; p <= n / p; p += 2)
            while (n % p == 0) { y.push(p); n /= p; }
        if (n > 1) y.push(n);
    }
};
FBR_EXPORT_RECORD_BODY(PrimeFactors, "prime_factors_i64", prime_factors_entry, FBR_BODY_INDEX_ARG)
'''

ABOVE_ARG = np.dtype([("t", "<f8")])

ABOVE_SRC = r'''
#include "fiber_b200_body.cuh"

// positions k of a float64 row where x[k] > t, on a warp: lanes take k = rank, rank + 32, ... and append in rank order
struct AboveMask {
    struct Arg { double t; };
    using Item = double;
    using Out = uint32_t;
    using Res = fbr::NoRes;
    static constexpr uint32_t kGroup = 32;
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static __forceinline__ void run(const Arg& a, const fbr::Items<Item>& x, fbr::Emit<Out, 32>& y,
                                               const fbr::Group<32>& g, uint64_t, const fbr::ErrSink&, uint32_t) {
        for (uint64_t base = 0; base < x.n; base += g.size) {
            const uint64_t k = base + g.rank;
            y.push_if(g, k < x.n && x.data[k] > a.t, (uint32_t)k);
        }
    }
};
FBR_EXPORT_RECORD_BODY(AboveMask, "above_mask_f64", above_mask_entry, 0)
'''

QUERY = np.dtype([("x", "<f4"), ("y", "<f4"), ("r", "<f4")])
POINT = np.dtype([("x", "<f4"), ("y", "<f4")])

RADIUS_SRC = r'''
#include "fiber_b200_body.cuh"

// indices of the broadcast points within r of (x, y): (px - x)^2 + (py - y)^2 <= r^2, every operation rounded in float32
struct RadiusNeighbors {
    struct Arg { float x, y, r; };
    struct Point { float x, y; };
    using Shared = Point;
    static constexpr uint32_t kSharedStage = 16384;
    using Out = uint32_t;
    using Res = fbr::NoRes;
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static __forceinline__ void run(const Arg& a, fbr::Emit<Out>& y, const fbr::Broadcast<Shared>& pts, uint64_t,
                                               const fbr::ErrSink&, uint32_t) {
        const float r2 = __fmul_rn(a.r, a.r);
        for (uint64_t j = 0; j < pts.n; ++j) {
            const float dx = __fsub_rn(pts.data[j].x, a.x), dy = __fsub_rn(pts.data[j].y, a.y);
            if (__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)) <= r2) y.push((uint32_t)j);
        }
    }
};
FBR_EXPORT_RECORD_BODY(RadiusNeighbors, "radius_neighbors_f32", radius_neighbors_entry, 0)
'''

UPPER_SRC = r'''
#include "fiber_b200_body.cuh"

// ASCII uppercase of a byte string; its count is its length, so the count pass never runs the body
struct UpperAscii {
    using Item = uint8_t;
    using Arg = fbr::NoArg;
    using Out = uint8_t;
    using Res = fbr::NoRes;
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static uint64_t count(const fbr::Items<Item>& x, uint64_t) { return x.n; }
    __device__ static __forceinline__ void run(const fbr::Items<Item>& x, fbr::Emit<Out>& y, uint64_t, const fbr::ErrSink&,
                                               uint32_t) {
        for (uint64_t k = 0; k < x.n; ++k) {
            const uint8_t c = x.data[k];
            y.push(c >= 'a' && c <= 'z' ? (uint8_t)(c - 32) : c);
        }
    }
};
FBR_EXPORT_RECORD_BODY(UpperAscii, "upper_ascii_u8", upper_ascii_entry, 0)
'''

TOKEN_SUM_RES = np.dtype([("s", "<u8")])

TOKEN_SUM_SRC = r'''
#include "fiber_b200_body.cuh"

// the sum of a list of uint32 (an items body: the end of the tokenize -> sum chain)
struct TokenSum {
    using Item = uint32_t;
    using Arg = fbr::NoArg;
    struct Res { uint64_t s; };
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static __forceinline__ void run(const fbr::Items<Item>& x, Res& r, uint64_t, const fbr::ErrSink&, uint32_t) {
        uint64_t s = 0;
        for (uint64_t k = 0; k < x.n; ++k) s += x.data[k];
        r.s = s;
    }
};
FBR_EXPORT_RECORD_BODY(TokenSum, "token_sum_u32", token_sum_entry, 0)
'''


@fiber_b200.device_body("tokens_u32", source=TOKENS_SRC, entry="tokens_entry", args=None, items=("doc", "u1"), out="<u4")
def tokens_u32(doc):
    return [fnv1a32(t) for t in bytes(doc).split()]


@fiber_b200.device_body("fault_tokens_u32", source=TOKENS_SRC, entry="fault_tokens_entry", args=None, items=("doc", "u1"),
                        out="<u4")
def fault_tokens_u32(doc):
    return tokens_u32(doc)


@fiber_b200.device_body("early_fault_tokens_u32", source=TOKENS_SRC, entry="early_fault_tokens_entry", args=None,
                        items=("doc", "u1"), out="<u4")
def early_fault_tokens_u32(doc):
    return tokens_u32(doc)


@fiber_b200.device_body("bad_count_u32", source=TOKENS_SRC, entry="bad_count_entry", args=None, items=("doc", "u1"),
                        out="<u4")
def bad_count_u32(doc):
    return list(bytes(doc))


@fiber_b200.device_body("prime_factors_i64", source=PRIMES_SRC, entry="prime_factors_entry", args="<i8", out="<i8")
def prime_factors_i64(n):
    return prime_factors(n)


@fiber_b200.device_body("above_mask_f64", source=ABOVE_SRC, entry="above_mask_entry", args=ABOVE_ARG, items=("row", "<f8"),
                        out="<u4")
def above_mask_f64(row, t):
    return np.flatnonzero(np.asarray(row) > t).tolist()


@fiber_b200.device_body("radius_neighbors_f32", source=RADIUS_SRC, entry="radius_neighbors_entry", args=QUERY,
                        shared=("points", POINT), out="<u4")
def radius_neighbors_f32(points, x, y, r):
    return radius_neighbors_np(points, np.array([(x, y, r)], QUERY))[0]


@fiber_b200.device_body("upper_ascii_u8", source=UPPER_SRC, entry="upper_ascii_entry", args=None, items=("s", "u1"), out="u1",
                        out_as="str")
def upper_ascii_u8(s):
    return s.encode().upper().decode()


@fiber_b200.device_body("token_sum_u32", source=TOKEN_SUM_SRC, entry="token_sum_entry", args=None, items=("xs", "<u4"),
                        result=TOKEN_SUM_RES)
def token_sum_u32(xs):
    return sum(int(v) for v in xs)


# ---- restatements ------------------------------------------------------------------------------------------------------
def fnv1a32(token):
    h = 0x811C9DC5
    for c in token:
        h = ((h ^ c) * 0x01000193) & 0xFFFFFFFF
    return h


def prime_factors(n):
    out, p = [], 2
    if n < 2:
        return out
    while n % 2 == 0:
        out.append(2)
        n //= 2
    p = 3
    while p <= n // p:
        while n % p == 0:
            out.append(p)
            n //= p
        p += 2
    if n > 1:
        out.append(n)
    return out


def radius_neighbors_np(points, queries):
    px, py = points["x"].astype(np.float32), points["y"].astype(np.float32)
    out = []
    for q in queries:
        dx, dy = px - np.float32(q["x"]), py - np.float32(q["y"])
        d2 = dx * dx + dy * dy
        out.append(np.flatnonzero(d2 <= np.float32(q["r"]) * np.float32(q["r"])).tolist())
    return out


# ---- seeded inputs ------------------------------------------------------------------------------------------------------
def documents(n, seed, max_words=40, empty_every=0):
    """n byte strings of seeded words (lowercase letters) separated by runs of ASCII whitespace; every `empty_every`-th
    document (if non-zero) is all whitespace, so it has no token."""
    rng = np.random.default_rng(seed)
    spaces = [b" ", b"  ", b"\t", b"\n", b" \r\n", b"\x0b", b"\x0c"]
    docs = []
    for i in range(n):
        if empty_every and i % empty_every == 0:
            docs.append(b" \t" * int(rng.integers(0, 3)))
            continue
        words = int(rng.integers(0, max_words + 1))
        parts = []
        for _ in range(words):
            parts.append(bytes(rng.integers(97, 123, int(rng.integers(1, 12)), dtype=np.uint8)))
            parts.append(spaces[int(rng.integers(0, len(spaces)))])
        doc = b"".join(parts)
        docs.append(doc[:-1] if words and rng.integers(0, 2) else doc)
    return docs


# Hand-written descriptors that break the emit rules; registration must refuse every one of them except ok_emit.
# (FBR_EXPORT_RECORD_BODY derives the flags and fields from the struct, so a real body cannot get there.)
BAD_SRC = r'''
#include "fiber_b200_body.cuh"

#define BAD_EMIT(entry, name, flags, rbytes, kind, out)                                                            \
    extern "C" const fbr_body_module_t* entry(void) {                                                            \
        static const fbr_body_module_t m = {FBR_BODY_MODULE_ABI, (uint32_t)sizeof(fbr::WaveParams), name, 0u,     \
                                            (rbytes), (kind), (flags), 1024u,                                    \
                                            fbr_body_export::launch_emit<TokensLike>,                            \
                                            fbr_body_export::occupancy_emit<TokensLike>, 0u, 0u, 0u, 1u, (out)};  \
        return &m;                                                                                               \
    }
struct TokensLike {
    using Item = uint8_t;
    using Arg = fbr::NoArg;
    using Out = uint32_t;
    using Res = fbr::NoRes;
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static void run(const fbr::Items<Item>& x, fbr::Emit<Out>& y, uint64_t, const fbr::ErrSink&, uint32_t) { y.push((uint32_t)x.n); }
};
#define IT (FBR_BODY_RECORD | FBR_BODY_ITEMS)
#define EM (FBR_BODY_RECORD | FBR_BODY_ITEMS | FBR_BODY_EMIT)
BAD_EMIT(bad_emit_fields, "bad_emit_fields", IT, 8u, FBR_RES_OFFSETS, 4u)                  // an out size without the flag
BAD_EMIT(bad_emit_thread, "bad_emit_thread", FBR_BODY_ITEMS | FBR_BODY_EMIT, 8u, FBR_RES_OFFSETS, 4u)   // not a record body
BAD_EMIT(bad_emit_res, "bad_emit_res", EM, 16u, FBR_RES_OFFSETS, 4u)                        // a fixed result record
BAD_EMIT(bad_emit_kind, "bad_emit_kind", EM, 8u, FBR_RES_BYTES, 4u)
BAD_EMIT(bad_out0, "bad_out0", EM, 8u, FBR_RES_OFFSETS, 0u)
BAD_EMIT(bad_out3, "bad_out3", EM, 8u, FBR_RES_OFFSETS, 3u)
BAD_EMIT(bad_out_big, "bad_out_big", EM, 8u, FBR_RES_OFFSETS, 8192u)
BAD_EMIT(bad_emit_sum, "bad_emit_sum", EM | FBR_BODY_SUMMABLE, 8u, FBR_RES_OFFSETS, 4u)
BAD_EMIT(ok_emit, "ok_emit", EM, 8u, FBR_RES_OFFSETS, 4u)
'''
BAD_MODULE = fiber_b200.bodies.compile_module("emit_bad_descriptors", BAD_SRC)
