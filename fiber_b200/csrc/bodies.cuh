// bodies.cuh -- the mapped function bodies, as device code.
//
// In the reference the mapped function is a pickled Python callable executed by the worker at
// fiber/pool.py:806,809,820.  Here each supported callable has a compiled-in device body selected
// by func_id in the task record.  Three execution shapes:
//   * ThreadBody  : one thread per task, results packed 16 B per store       (square, pi, ...)
//   * RecordBody  : one CTA streams 4 KB records through registers            (payload_map)
//   * ReduceBody  : a warp / CTA cooperates on one task and emits a scalar    (checksum, parzen)
// Integer/byte bodies are bit-exact against oracle/bodies.py; parzen_f32 carries the north-star's
// stated fp32 tolerance, parzen_f64 is bit-exact.
#pragma once
#include <stdint.h>

namespace fbr {

enum FuncId : int32_t {
    F_SQUARE_I64 = 0,        // tests/test_pool.py:18-19   f(x) = x*x
    F_MUL2_I64 = 1,          // tests/test_pool.py:21-22   f2(x, y) = x*y
    F_SQUARE_SCALE_I64 = 2,  // tests/test_pool.py:24-25   fy(x, y=1) = x*x*y
    F_IDENTITY_I64 = 3,      // tests/test_pool.py:60-68   random_error_worker's return value
    F_PI_INSIDE_DET = 4,     // examples/pi_estimation.py:9-11 (deterministic restatement)
    F_PARZEN_F32 = 5,        // examples/parzen_estimation.py:6-15, fp32 window test
    F_PARZEN_F64 = 6,        // same, fp64 window test (bit-exact k_n)
    F_PAYLOAD_MAP_4K = 7,    // BASELINE.json config 4: 4 KB record -> 4 KB record
    F_PAYLOAD_CHECKSUM_4K = 8,  // 4 KB record -> u32
    F_SLEEP_F64 = 9,         // tests/test_pool.py:56-57   sleep_worker(duration) -> None
    F_FAULT_IDENTITY_I64 = 10,  // identity with injected faults (resilient pool tests)
    F_PI_INSIDE_BITS8 = 11,  // pi_inside_det over 8 consecutive items (range() indices or int64 arguments) -> one byte, bit k = item 8g+k
    F_TRAP_IDENTITY_I64 = 12,  // identity that executes `trap` on chosen arguments: kills the worker's CUDA context for real
    F_COUNT = 13             // compiled-in bodies; bodies registered at run time (fbr_register_body) get ids from here up
};

enum TaskError : uint32_t { TASK_OK = 0, TASK_OVERFLOW = 1, TASK_BADARG = 2, TASK_FAULT = 3, TASK_EMIT = 4, TASK_KEY = 5 };

// Lowest failing task wins, like the first exception a reference worker would have raised on the
// lowest index.  Packed as (task_index << 8 | code) so a single atomicMin orders by index.
// A TASK_FAULT is different: it models a worker *dying* inside a chunk (tests/test_pool.py:60-68):
// the whole claim unit is marked lost in its ring-slot header and the resilient host layer
// re-dispatches it (fiber/pool.py:1635-1654), so it only raises the CTA-local unit_fault flag.
struct ErrSink {
    unsigned long long* word;  // device, initialised to ~0ull
    int* unit_fault;           // shared memory, one per CTA
    __device__ __forceinline__ void report(uint32_t code, uint64_t task_index) const {
        if (code == TASK_FAULT) { *unit_fault = 1; return; }
        atomicMin(word, (unsigned long long)((task_index << 8) | (uint64_t)code));
    }
};

// ------------------------------------------------------------------------------------------------
// checked int64 arithmetic: Python ints are unbounded, so overflow must fail loudly, not wrap.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int64_t mul_i64_checked(int64_t a, int64_t b, bool& ovf) {
    // low half in unsigned arithmetic: signed overflow is UB and nvcc exploits it (it folded
    // `a*a >> 63` to 0 for the square body, hiding every overflow)
    int64_t lo = (int64_t)((uint64_t)a * (uint64_t)b);
    int64_t hi = __mul64hi(a, b);
    ovf |= (hi != (lo >> 63));
    return lo;
}

// ------------------------------------------------------------------------------------------------
// Philox4x32-10 (Random123).  Matches oracle/bodies.py:philox4x32_10 bit for bit.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void philox4x32_10(uint32_t& c0, uint32_t& c1, uint32_t& c2, uint32_t& c3,
                                              uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
}

// examples/pi_estimation.py:9-11 with random.random() replaced by one Philox block keyed by p
// (oracle/bodies.py:pi_inside_det).  x*x + y*y < 1 is evaluated as three separately rounded
// float64 operations (__dmul_rn/__dadd_rn forbid FMA contraction) exactly as CPython does.
__device__ __forceinline__ uint8_t pi_inside_from_block(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3) {
    // (a>>5)*2^26 + (b>>6) is an exact 53-bit integer; the division by 2^53 is exact.  The 64-bit
    // value is assembled with a funnel shift ({a>>5 : b} >> 6); written as a shift of a widened
    // product it compiled to an IMAD.WIDE, i.e. two more trips through the multiply pipe per task.
    const uint32_t a5 = c0 >> 5, b5 = c2 >> 5;
    const uint64_t xi = ((uint64_t)(a5 >> 6) << 32) | (uint64_t)__funnelshift_r(c1, a5, 6);
    const uint64_t yi = ((uint64_t)(b5 >> 6) << 32) | (uint64_t)__funnelshift_r(c3, b5, 6);
    const double x = __dmul_rn((double)xi, 0x1.0p-53);
    const double y = __dmul_rn((double)yi, 0x1.0p-53);
    return __dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)) < 1.0 ? 1 : 0;
}
__device__ __forceinline__ uint8_t pi_inside_det(int64_t p) {
    uint32_t c0 = (uint32_t)((uint64_t)p), c1 = (uint32_t)((uint64_t)p >> 32), c2 = 0u, c3 = 0u;
    philox4x32_10(c0, c1, c2, c3, 0xF1BE5EEDu, 0u);
    return pi_inside_from_block(c0, c1, c2, c3);
}

// 32 x 32 -> 64 as ONE multiply-pipe instruction (IMAD.WIDE.U32).  Spelled with __umulhi + `*`, or
// as a 64-bit C++ product, ptxas split most of the unrolled multiplies into IMAD + IMAD.HI pairs
// (twice the pipe time) or padded them with adds of zero.
__device__ __forceinline__ void mulhilo(uint32_t a, uint32_t b, uint32_t& hi, uint32_t& lo) {
    asm("{\n\t.reg .b64 t;\n\tmul.wide.u32 t, %2, %3;\n\tmov.b64 {%0, %1}, t;\n\t}" : "=r"(lo), "=r"(hi) : "r"(a), "r"(b));
}

// The same block for a counter (lo, hi, 0, 0) with the work that does not depend on `lo` taken out:
// round 1 multiplies a zero word (free) and round 2's M0 * (hi ^ key) is the same for every task
// whose index shares the high word -- `hk` is that product, computed once per 16 tasks.  18 wide
// multiplies per task instead of 20; bit-identical to philox4x32_10 by construction (and by test).
__device__ __forceinline__ void philox_block_lo(uint32_t lo, uint2 hk /* (hi, lo) of M0 * (p_hi ^ K) */,
                                                uint32_t& c0, uint32_t& c1, uint32_t& c2, uint32_t& c3) {
    constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u, K = 0xF1BE5EEDu;
    // round 1: c = (lo, hi, 0, 0), k = (K, 0)      -> c = (hi ^ K, 0, hi(M0*lo), lo(M0*lo))
    uint32_t p1h, p1l, p2h, p2l;
    mulhilo(M0, lo, p1h, p1l);
    // round 2: k = (K + W0, W1)                    -> c = (hi(M1*c2) ^ k0, lo(M1*c2), hk.hi ^ c3 ^ k1, hk.lo)
    mulhilo(M1, p1h, p2h, p2l);
    c0 = p2h ^ (K + W0); c1 = p2l; c2 = hk.x ^ p1l ^ W1; c3 = hk.y;
    uint32_t k0 = K + 2u * W0, k1 = 2u * W1;
#pragma unroll
    for (int r = 2; r < 10; ++r) {
        uint32_t hi0, lo0, hi1, lo1;
        mulhilo(M0, c0, hi0, lo0);
        mulhilo(M1, c2, hi1, lo1);
        const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
        k0 += W0; k1 += W1;
    }
}
__device__ __forceinline__ uint8_t pi_inside_det_lo(uint32_t lo, uint2 hk) {
    uint32_t c0, c1, c2, c3;
    philox_block_lo(lo, hk, c0, c1, c2, c3);
    return pi_inside_from_block(c0, c1, c2, c3);
}

// fp32 screen of x*x + y*y < 1 on the top 23 bits of each coordinate (no int->double conversion, no
// FP64: those instructions hold the SM sub-partition's dispatch port for several cycles each and take
// issue slots from the multiply pipe -- profiles/microbench/imad_peak.cu compares the two bodies).
//   xf = (c0 >> 9) * 2^-23 exactly ((1 + xf) - 1 with the fraction funnel-shifted under the exponent
//   of 1.0f), so x is in [xf, xf + 2^-23), likewise y, and with S = x^2 + y^2, Sf = xf^2 + yf^2:
//       Sf <= S < Sf + 2^-22 (xf + yf) + 2^-45 < Sf + 2^-21 + 2^-45
//   d = fma(xf, xf, fma(yf, yf, -1)) differs from Sf - 1 by at most two roundings of values <= 1,
//   i.e. by less than 2^-23, hence |(S - 1) - d| < 2^-20.
//   The float64 value the reference compares, fl(fl(x*x) + fl(y*y)), is within 2^-51 of S.
// So whenever |d| >= 2^-19 the sign of d IS the reference's answer (d < 0: inside); the caller
// re-evaluates the (about 3 in 10^6) closer points in float64.  `dmin` tracks min |d|.
__device__ __forceinline__ float pi_screen(uint32_t c0, uint32_t c2, float& dmin) {
    const float xf = __fadd_rn(__uint_as_float(__funnelshift_r(c0, 0x7Fu, 9)), -1.0f);
    const float yf = __fadd_rn(__uint_as_float(__funnelshift_r(c2, 0x7Fu, 9)), -1.0f);
    const float d = __fmaf_rn(xf, xf, __fmaf_rn(yf, yf, -1.0f));
    dmin = fminf(dmin, fabsf(d));
    return d;
}
// The screens of two tasks a and b.  sm_90 has no packed FP32 instructions, so each lane is its own
// scalar FADD/FFMA chain (4 FMA-pipe instructions per task); the pair keeps the callers' loop shape.
__device__ __forceinline__ void pi_screen2(uint32_t c0a, uint32_t c2a, uint32_t c0b, uint32_t c2b, float& da, float& db, float& dmin) {
    da = pi_screen(c0a, c2a, dmin);
    db = pi_screen(c0b, c2b, dmin);
}
// four screen values -> four result bytes (0/1): the answer is the sign bit of d, so gather the top
// bytes with three PRMTs and keep bit 7 of each -- 5 instructions instead of 4 x (FSETP, SEL, LOP3)
__device__ __forceinline__ uint32_t pi_pack4(float d0, float d1, float d2, float d3) {
    const uint32_t w01 = __byte_perm(__float_as_uint(d0), __float_as_uint(d1), 0x0073);
    const uint32_t w23 = __byte_perm(__float_as_uint(d2), __float_as_uint(d3), 0x0073);
    return (__byte_perm(w01, w23, 0x5410) >> 7) & 0x01010101u;
}
constexpr float kPiScreenMargin = 0x1.0p-19f;

// SplitMix64 finaliser; oracle/bodies.py:splitmix64.
__device__ __host__ __forceinline__ uint64_t splitmix64(uint64_t x) {
    uint64_t z = x + 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
constexpr uint32_t kPayloadWords = 1024;
constexpr uint32_t kPayloadBytes = 4096;
constexpr uint64_t kPayloadSeed = 0xF1BE5ull;
constexpr uint32_t kPayloadMul = 2654435761u;

// ================================================================================================
// ThreadBody concept:  struct { using Arg; using Res; static Res run(const Arg&, uint64_t gidx, const ErrSink&, uint32_t attempt) }
//   Arg is loaded from the argument ring, or (kIndexArg && arg_stride==0) synthesised from the
//   task index: arg = index_start + i*index_step (a Python range()).
// ================================================================================================
struct I64x2 { int64_t x, y; };

struct SquareI64 {
    using Arg = int64_t; using Res = int64_t;
    static constexpr bool kIndexArg = true;
    static constexpr bool kVecIndex = false;
    static constexpr bool kCanFault = false;
    __device__ static __forceinline__ Res run(const Arg& a, uint64_t gidx, const ErrSink& es, uint32_t) {
        bool ovf = false;
        const int64_t r = mul_i64_checked(a, a, ovf);
        if (ovf) es.report(TASK_OVERFLOW, gidx);
        return r;
    }
};
struct Mul2I64 {
    using Arg = I64x2; using Res = int64_t;
    static constexpr bool kIndexArg = false;
    static constexpr bool kVecIndex = false;
    static constexpr bool kCanFault = false;
    __device__ static __forceinline__ Res run(const Arg& a, uint64_t gidx, const ErrSink& es, uint32_t) {
        bool ovf = false;
        const int64_t r = mul_i64_checked(a.x, a.y, ovf);
        if (ovf) es.report(TASK_OVERFLOW, gidx);
        return r;
    }
};
struct SquareScaleI64 {
    using Arg = I64x2; using Res = int64_t;
    static constexpr bool kIndexArg = false;
    static constexpr bool kVecIndex = false;
    static constexpr bool kCanFault = false;
    __device__ static __forceinline__ Res run(const Arg& a, uint64_t gidx, const ErrSink& es, uint32_t) {
        bool ovf = false;
        const int64_t r = mul_i64_checked(mul_i64_checked(a.x, a.x, ovf), a.y, ovf);
        if (ovf) es.report(TASK_OVERFLOW, gidx);
        return r;
    }
};
struct IdentityI64 {
    using Arg = int64_t; using Res = int64_t;
    static constexpr bool kIndexArg = true;
    static constexpr bool kVecIndex = false;
    static constexpr bool kCanFault = false;
    __device__ static __forceinline__ Res run(const Arg& a, uint64_t, const ErrSink&, uint32_t) { return a; }
};
// Identity whose tasks "kill their worker" with probability ~5 % per attempt, as
// random_error_worker does (tests/test_pool.py:60-68).  The attempt number is carried in the
// task record flags so a re-dispatched unit draws fresh faults.
struct FaultIdentityI64 {
    using Arg = int64_t; using Res = int64_t;
    static constexpr bool kIndexArg = true;
    static constexpr bool kVecIndex = false;
    static constexpr bool kCanFault = true;   // reports TASK_FAULT: the unit is marked lost
    __device__ static __forceinline__ Res run(const Arg& a, uint64_t gidx, const ErrSink& es, uint32_t attempt) {
        const uint64_t h = splitmix64((gidx << 8) ^ (uint64_t)attempt ^ 0xFA17ull);
        if ((h % 100ull) < 5ull) es.report(TASK_FAULT, gidx);
        return a;
    }
};
// Identity whose first attempt at an argument with low 20 bits 0xDEAD executes `trap`: the kernel dies, the
// device's context takes a sticky error and every later call on it fails -- a worker process killed for real
// (the reference's dead worker: fiber/pool.py:1623-1656 notices it and re-queues its chunks elsewhere).
struct TrapIdentityI64 {
    using Arg = int64_t; using Res = int64_t;
    static constexpr bool kIndexArg = true;
    static constexpr bool kVecIndex = false;
    static constexpr bool kCanFault = false;
    __device__ static __forceinline__ Res run(const Arg& a, uint64_t, const ErrSink&, uint32_t attempt) {
        if (attempt == 0u && ((uint64_t)a & 0xFFFFFull) == 0xDEADull) asm volatile("trap;");
        return a;
    }
};
struct PiInsideDet {
    using Arg = int64_t; using Res = uint8_t;
    static constexpr bool kIndexArg = true;
    static constexpr bool kVecIndex = true;
    static constexpr bool kCanFault = false;
    __device__ static __forceinline__ Res run(const Arg& a, uint64_t, const ErrSink&, uint32_t) { return pi_inside_det(a); }
    // V consecutive range() arguments a0, a0 + step, ...: results packed one byte each into pk
    template <int V>
    __device__ static __forceinline__ void run_index_vec(int64_t a0, int64_t step, uint32_t (&pk)[4]) {
        const uint64_t u0 = (uint64_t)a0, u_last = u0 + (uint64_t)(V - 1) * (uint64_t)step;
        const uint32_t hi = (uint32_t)(u0 >> 32);
        if (hi == (uint32_t)(u_last >> 32)) {
            // the progression is monotone, so every index in between shares the high word
            const uint32_t hx = hi ^ 0xF1BE5EEDu;
            const uint2 hk = make_uint2(__umulhi(0xD2511F53u, hx), 0xD2511F53u * hx);
            const uint32_t lo0 = (uint32_t)u0, lstep = (uint32_t)(uint64_t)step;
            static_assert(V % 4 == 0, "results are packed four to a word");
            float dmin = 1.0f;
#pragma unroll
            for (int g = 0; g < V / 4; ++g) {
                float d[4];
#pragma unroll
                for (int k = 0; k < 4; k += 2) {
                    uint32_t a0, a1, a2, a3, b0, b1, b2, b3;
                    philox_block_lo(lo0 + (uint32_t)(4 * g + k) * lstep, hk, a0, a1, a2, a3);
                    philox_block_lo(lo0 + (uint32_t)(4 * g + k + 1) * lstep, hk, b0, b1, b2, b3);
                    pi_screen2(a0, a2, b0, b2, d[k], d[k + 1], dmin);
                }
                pk[g] = pi_pack4(d[0], d[1], d[2], d[3]);
            }
            if (dmin < kPiScreenMargin) {
                // some point of this vector is within 2^-19 of the circle: redo the vector in float64
                pk[0] = pk[1] = pk[2] = pk[3] = 0u;
#pragma unroll 1
                for (int v = 0; v < V; ++v) {
                    const uint32_t r = pi_inside_det_lo(lo0 + (uint32_t)v * lstep, hk);
                    pk[v >> 2] |= r << ((v & 3) * 8);
                }
            }
        } else {
#pragma unroll 1
            for (int v = 0; v < V; ++v) {
                const uint32_t r = pi_inside_det((int64_t)(u0 + (uint64_t)v * (uint64_t)step));
                pk[v >> 2] |= r << ((v & 3) * 8);   // v is a run-time index here: rare path (2^32 crossing)
            }
        }
    }
    // The same 16 consecutive arguments, one BIT per result: bit v of the return value is
    // is_inside(a0 + v*step).  (Body pi_inside_bits8: a bool needs one bit, not one byte, on its way
    // through the ring, the gather and PCIe.)
    __device__ static __forceinline__ uint32_t run_index_bits16(int64_t a0, int64_t step) {
        const uint64_t u0 = (uint64_t)a0, u_last = u0 + 15ull * (uint64_t)step;
        const uint32_t hi = (uint32_t)(u0 >> 32);
        uint32_t bits = 0;
        if (hi == (uint32_t)(u_last >> 32)) {
            const uint32_t hx = hi ^ 0xF1BE5EEDu;
            const uint2 hk = make_uint2(__umulhi(0xD2511F53u, hx), 0xD2511F53u * hx);
            const uint32_t lo0 = (uint32_t)u0, lstep = (uint32_t)(uint64_t)step;
            float dmin = 1.0f;
#pragma unroll
            for (int g = 0; g < 4; ++g) {
                float d[4];
#pragma unroll
                for (int k = 0; k < 4; k += 2) {
                    uint32_t a0, a1, a2, a3, b0, b1, b2, b3;
                    philox_block_lo(lo0 + (uint32_t)(4 * g + k) * lstep, hk, a0, a1, a2, a3);
                    philox_block_lo(lo0 + (uint32_t)(4 * g + k + 1) * lstep, hk, b0, b1, b2, b3);
                    pi_screen2(a0, a2, b0, b2, d[k], d[k + 1], dmin);
                }
                // bytes (b0, b1, b2, b3) of 0/1 -> nibble b0 | b1<<1 | b2<<2 | b3<<3: one multiply moves
                // byte i's bit to position 28+i (the partial products land on distinct bits: no carries)
                bits |= ((pi_pack4(d[0], d[1], d[2], d[3]) * 0x10204080u) >> 28) << (4 * g);
            }
            if (dmin < kPiScreenMargin) {
                bits = 0;
#pragma unroll 1
                for (int v = 0; v < 16; ++v) bits |= (uint32_t)pi_inside_det_lo(lo0 + (uint32_t)v * lstep, hk) << v;
            }
        } else {
#pragma unroll 1
            for (int v = 0; v < 16; ++v) bits |= (uint32_t)pi_inside_det((int64_t)(u0 + (uint64_t)v * (uint64_t)step)) << v;
        }
        return bits;
    }
};
// sleep_worker(duration): busy-wait on the global nanosecond timer; returns None (one pad byte).
struct SleepF64 {
    using Arg = double; using Res = uint8_t;
    static constexpr bool kIndexArg = false;
    static constexpr bool kVecIndex = false;
    static constexpr bool kCanFault = false;
    __device__ static __forceinline__ Res run(const Arg& a, uint64_t gidx, const ErrSink& es, uint32_t) {
        if (!(a >= 0.0) || a > 10.0) { es.report(TASK_BADARG, gidx); return 0; }
        unsigned long long t0, t1;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
        const unsigned long long dur = (unsigned long long)(a * 1e9);
        do {
            __nanosleep(1000);
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        } while (t1 - t0 < dur);
        return 0;
    }
};

// ================================================================================================
// Parzen window (examples/parzen_estimation.py:6-15).  Shared block layout (host writes it once,
// it is broadcast to every task instead of being pickled 102 times, SURVEY.md 3.2):
//   struct ParzenShared { u32 n_samples; u32 dims; u32 power; u32 elem_bytes; f64 point_x[8]; }
//   followed (at byte 80) by samples[n_samples][dims] in f32 or f64.
// Per-task argument: h (f64).  Result: (h, (k_n / n) / h**power) as two f64.
// ================================================================================================
struct ParzenShared {
    uint32_t n_samples, dims, power, elem_bytes;
    double point_x[8];
};
static_assert(sizeof(ParzenShared) == 80, "layout is part of the ABI");

template <typename T>
__device__ __forceinline__ bool parzen_inside(const T* __restrict__ row, const ParzenShared& sh, T h) {
    bool inside = true;
    for (uint32_t d = 0; d < sh.dims; ++d) {
        // (point_x - x) / h with IEEE division, then `abs(q) > 1/2` breaks (reference lines 9-12);
        // written as !(|q| > 0.5) so a NaN counts as inside exactly like the reference.
        const T q = ((T)sh.point_x[d] - row[d]) / h;
        inside = inside && !(fabs(q) > (T)0.5);
    }
    return inside;
}

}  // namespace fbr
