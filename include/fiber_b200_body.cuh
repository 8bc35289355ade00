// fiber_b200_body.cuh -- what an OUT-OF-TREE device body is compiled against.
//
// The reference ships any Python callable to its workers (fiber/pool.py:961) and the worker calls it
// (fiber/pool.py:806,809,820).  A GPU worker runs device code, so a user function needs a device body;
// this header lets that body live outside libfiber_b200: write a ThreadBody struct, export it, build a
// shared object, register it.
//
//     #include "fiber_b200_body.cuh"
//     struct Collatz {                                   // steps of the Collatz iteration from x
//         using Arg = int64_t; using Res = int64_t;
//         static constexpr bool kIndexArg = true;        // may be mapped over a range() with no argument bytes
//         static constexpr bool kVecIndex = false;
//         static constexpr bool kCanFault = false;
//         __device__ static Res run(const Arg& a, uint64_t task_index, const fbr::ErrSink& es, uint32_t attempt) { ... }
//     };
//     FBR_EXPORT_THREAD_BODY(Collatz, "collatz_steps", collatz_entry, FBR_RES_I64, FBR_BODY_INDEX_ARG | FBR_BODY_SUMMABLE)
//
//     nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -shared -Xcompiler -fPIC -I<repo>/include -I<repo>/fiber_b200/csrc body.cu -o libbody.so
//     fbr_register_body("collatz_steps", "libbody.so", "collatz_entry", &func_id);
//
// (fiber_b200.device_body(name, source=...) does the last two steps from Python.)  The body is instantiated
// into the same persistent-CTA dispatch kernel template the compiled-in bodies use, so it gets the ticket
// claim, record synthesis, direct placement / result ring, sum fold and resilient re-dispatch for free.
//
// A ThreadBody returns a 1- or 8-byte value.  A function over other fixed-size records -- f(x: float) -> float,
// f(x, y) -> (r, theta), a row of 256 uint32 -> a few statistics -- is a RECORD body: Arg and Res are any
// trivially copyable structs (sizeof a multiple of 4, at most 4096 bytes; a group body below may reach 32 KB), and
// run() writes the result in place:
//
//     struct Polar {
//         struct Arg { double x, y; }; struct Res { double r2, r; };
//         static constexpr bool kIndexArg = false;       // true: Arg = int64_t, range() maps need no argument bytes
//         static constexpr bool kCanFault = false;
//         __device__ static void run(const Arg& a, Res& r, uint64_t task_index, const fbr::ErrSink& es, uint32_t attempt) {
//             r.r2 = __dadd_rn(__dmul_rn(a.x, a.x), __dmul_rn(a.y, a.y)); r.r = __dsqrt_rn(r.r2);
//         }
//     };
//     FBR_EXPORT_RECORD_BODY(Polar, "polar_f64", polar_entry, 0)
//
// `a` and `r` refer to shared memory: dispatch_record_kernel bulk-loads each claim unit's argument records into a
// shared-memory stage and bulk-stores the unit's results from another, so a large record is never copied into
// registers.  From Python: fiber_b200.device_body("polar_f64", source=..., entry="polar_entry",
// args=[("x", "<f8"), ("y", "<f8")], result=[("r2", "<f8"), ("r", "<f8")]) -- the NumPy dtypes describe the
// two structs byte for byte (INTEGRATION.md).  Record bodies cannot fold sums on the device and have no
// bit-packed twin.
//
// A record body may also read one array every task of a map shares (the pool initializer's initargs, or the same array
// in every task tuple): it declares the array's element type and a shared-memory budget, and run() gets the block
// after the result:
//
//     struct NearestCentroid {
//         struct Arg { float p[16]; }; struct Res { uint32_t k; float d2; };
//         struct Centroid { float c[16]; };
//         using Shared = Centroid;                        // trivially copyable, sizeof a multiple of 4, at most 4096
//         static constexpr uint32_t kSharedStage = 32768; // blocks up to this many bytes are staged in shared memory;
//                                                         // with the IN / OUT stages at most 200 KB in all
//         static constexpr bool kIndexArg = false, kCanFault = false;
//         __device__ static void run(const Arg& a, Res& r, const fbr::Broadcast<Shared>& sh, uint64_t task_index,
//                                    const fbr::ErrSink& es, uint32_t attempt) { ... sh.data[0 .. sh.n) ... }
//     };
//
// FBR_EXPORT_RECORD_BODY then sets FBR_BODY_NEEDS_SHARED | FBR_BODY_BROADCAST itself.  sh.n is shared_bytes /
// sizeof(Shared).  A block of at most kSharedStage bytes is bulk-loaded into shared memory once per CTA (sh.data points
// there); a larger one, or any block when kSharedStage is 0, is read from global memory.
//
// A GROUP record body runs each task on G threads of one warp (G = 2, 4, 8, 16 or 32): the lanes of a group read
// consecutive words of one record (no shared-memory bank conflicts) and reduce with shuffles, and its records may reach
// 32 KB.  It declares kGroup, and run() gets a const fbr::Group<G>& after the result (after the broadcast block, if any):
//
//     struct RowSum {
//         struct Arg { double x[1024]; }; struct Res { double s; uint32_t pad[2]; };
//         static constexpr uint32_t kGroup = 32;
//         static constexpr bool kIndexArg = false, kCanFault = false;
//         __device__ static void run(const Arg& a, Res& r, const fbr::Group<32>& g, uint64_t task_index,
//                                    const fbr::ErrSink& es, uint32_t attempt) {
//             double s = 0.0;
//             for (uint32_t k = g.rank; k < 1024; k += g.size) s = __dadd_rn(s, a.x[k]);
//             for (uint32_t o = g.size / 2; o > 0; o >>= 1) s = __dadd_rn(s, __shfl_xor_sync(g.mask, s, o));
//             if (g.rank == 0) r.s = s;
//         }
//     };
//
// g.rank is 0 .. G-1, g.size is G, g.mask is the group's lanes within its warp (for __shfl_*_sync), g.sync() is
// __syncwarp(g.mask).  The contract:
//   - all G threads call run() for the same task, with the same a, r, task_index and attempt;
//   - a and r are in shared memory, and any thread may write any part of r;
//   - every thread of the group reaches the same collective calls (shuffles, g.sync());
//   - a fault reported through es by any thread marks the task's unit, as for a one-thread body.
// Sizes: sizeof(Arg) and sizeof(Res) are multiples of 4 up to 32768, and kAlign * max(sizeof(Arg), sizeof(Res)) <= 32768,
// where kAlign (fbr::record::Layout<B>::kAlign) is 1 when both sizes are multiples of 16, 2 when both are multiples of
// 8, else 4: records that are multiples of 16 may reach 32 KB, multiples of 8 16 KB, any other pair 8 KB.  A body
// without kGroup is a one-thread body with records up to 4096 bytes.  FBR_EXPORT_RECORD_BODY checks all of this.
//
// An ITEMS record body's task also takes one variable-length array (a string, a document's tokens, a user's session):
// it declares the element type, and run() gets the task's items after its head record.  Arg = fbr::NoArg means no head record (run() then starts with the items):
//
//     struct Fnv1a {
//         using Item = uint8_t;                           // sizeof 1, 2, or a multiple of 4 up to 4096
//         using Arg = fbr::NoArg;
//         struct Res { uint64_t h; uint32_t n, pad; };
//         static constexpr bool kIndexArg = false, kCanFault = false;
//         __device__ static void run(const fbr::Items<Item>& x, Res& r, uint64_t task_index, const fbr::ErrSink& es,
//                                    uint32_t attempt) { ... x.data[0 .. x.n) ... }
//     };
//     FBR_EXPORT_RECORD_BODY(Fnv1a, "fnv1a_bytes", fnv1a_entry, 0)
//
// The full signature is run([const Arg& a,] const fbr::Items<Item>& x, Res& r, [Broadcast], [Group], task_index, es,
// attempt).  x.data is read-only and points into the map's item array in global memory, so vector loads legal on the
// array are legal on x.data.  All G lanes of a group body get the same x.  Items bodies cannot have kIndexArg.
// FBR_EXPORT_RECORD_BODY sets FBR_BODY_ITEMS and writes item_bytes.
//
// A task may take 2 to 4 variable-length arrays (two strings to compare, two token lists to intersect, a series and its
// weights): the body lists their element types, which may differ, and run() gets one view per stream, in order, where the
// single x goes above.  Each stream has its own offsets, so each task's arrays have their own lengths:
//
//     struct CommonPrefix {                               // length of the common prefix of two byte strings
//         using Items = fbr::ItemTypes<uint8_t, uint8_t>; // not together with `using Item`
//         using Arg = fbr::NoArg;
//         struct Res { uint32_t n; };
//         static constexpr bool kIndexArg = false, kCanFault = false;
//         __device__ static void run(const fbr::Items<uint8_t>& a, const fbr::Items<uint8_t>& b, Res& r, uint64_t task_index,
//                                    const fbr::ErrSink& es, uint32_t attempt) {
//             uint32_t k = 0;
//             while (k < a.n && k < b.n && a.data[k] == b.data[k]) ++k;
//             r.n = k;
//         }
//     };
//     FBR_EXPORT_RECORD_BODY(CommonPrefix, "common_prefix_u1", common_prefix_entry, 0)
//
// The full signature is run([const Arg& a,] const fbr::Items<T0>& x0, ..., const fbr::Items<Tk-1>& xk-1, Res& r |
// Emit<Out[,G]>& y, [Broadcast], [Group], task_index, es, attempt), and an emit body's count() takes the same leading
// parameters.  All G lanes of a group get the same views.  A task whose offsets decrease or leave their stream's items in
// any stream reports FBR_TASK_BADARG without its body being called.  FBR_EXPORT_RECORD_BODY writes item_streams and the
// element sizes of streams 1 to 3.
//
// An EMIT record body's task returns a variable-length array (a document's tokens, an integer's prime factors): it declares
// the element type and Res = fbr::NoRes, and run() appends to an emitter where other record bodies write Res& r:
//
//     struct Tokens {
//         using Item = uint8_t;  using Arg = fbr::NoArg;
//         using Out = uint32_t;                           // sizeof 1, 2, or a multiple of 4 up to 4096
//         using Res = fbr::NoRes;
//         static constexpr bool kIndexArg = false, kCanFault = false;
//         __device__ static void run(const fbr::Items<Item>& x, fbr::Emit<Out>& y, uint64_t task_index,
//                                    const fbr::ErrSink& es, uint32_t attempt) { ... y.push(h); ... }
//     };
//     FBR_EXPORT_RECORD_BODY(Tokens, "tokens_u32", tokens_entry, 0)
//
// The emitter goes where Res& r goes in every form above (head record or range() index, items, broadcast block, group).
// A group body takes fbr::Emit<Out, G>& and calls the collective y.push_if(g, pred, v) on every lane: lanes whose pred holds
// append v in rank order.  y.n is the number of values pushed so far.  Each map runs the body twice per task -- a count
// pass (y.data is nullptr), then, once the counts are scanned into offsets, an emit pass that writes each task's values
// at their final place -- so a task's values depend only on its inputs and task_index, never on attempt.  A one-thread body
// may define `static uint64_t count(...)` (run()'s parameters without y, es and attempt), which the count pass calls
// instead of run().  A task that pushes another number of values in the emit pass reports FBR_TASK_EMIT, and values past
// its count are never written.  FBR_EXPORT_RECORD_BODY sets FBR_BODY_EMIT, writes out_bytes, and reports result_bytes 8
// (each task's uint64 end offset) with result kind FBR_RES_OFFSETS.
#pragma once
#include "fiber_b200.h"
#include "kernels.cuh"      // fiber_b200/csrc: dispatch_thread_kernel, WaveParams, ErrSink, TaskError

#include <algorithm>
#include <type_traits>

namespace fbr_body_export {
using fbr_body_launch_fn = void (*)(const void* wave_params, int grid, void* cuda_stream);
using fbr_body_occupancy_fn = int (*)(int index_mode);
// CTAs of `kernel` per SM, at least 1 (a failed query leaves no sticky error behind)
inline int occupancy_of(const void* kernel, int threads, size_t smem) {
    int occ = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, threads, smem) != cudaSuccess) { cudaGetLastError(); return 1; }
    return occ > 0 ? occ : 1;
}

template <class B>
void launch(const void* wpv, int grid, void* sv) {
    const fbr::WaveParams& wp = *(const fbr::WaveParams*)wpv;
    cudaStream_t s = (cudaStream_t)sv;
    if constexpr (B::kIndexArg) {
        if (wp.arg_stride == 0) {
            fbr::dispatch_thread_kernel<B, true><<<grid, fbr::kThreads, 0, s>>>(wp);
            return;
        }
    }
    fbr::dispatch_thread_kernel<B, false><<<grid, fbr::kThreads, 0, s>>>(wp);
}
template <class B>
int occupancy(int index_mode) {
    if constexpr (B::kIndexArg) {
        if (index_mode) return occupancy_of((const void*)fbr::dispatch_thread_kernel<B, true>, fbr::kThreads, 0);
    }
    return occupancy_of((const void*)fbr::dispatch_thread_kernel<B, false>, fbr::kThreads, 0);
}

// the bit-packed twin of a bool body: 8 items (explicit records or range() indices) per result byte
template <class B>
void launch_bits(const void* wpv, int grid, void* sv) {
    const fbr::WaveParams& wp = *(const fbr::WaveParams*)wpv;
    cudaStream_t s = (cudaStream_t)sv;
    if constexpr (B::kIndexArg) {
        if (wp.arg_stride == 0) {
            fbr::dispatch_bits_items_kernel<B, true><<<grid, fbr::kThreads, 0, s>>>(wp);
            return;
        }
    }
    fbr::dispatch_bits_items_kernel<B, false><<<grid, fbr::kThreads, 0, s>>>(wp);
}
template <class B>
int occupancy_bits(int index_mode) {
    const void* k = (const void*)fbr::dispatch_bits_items_kernel<B, false>;
    if constexpr (B::kIndexArg) {
        if (index_mode) k = (const void*)fbr::dispatch_bits_items_kernel<B, true>;
    }
    return occupancy_of(k, fbr::kThreads, 0);
}
}  // namespace fbr_body_export

// A bool body (Res = uint8_t, 0/1) additionally exports its bit-packed twin "<name>_bits8" (result kind
// FBR_RES_BITS8, 8 items per task): register both and bool results travel one bit each.
#define FBR_EXPORT_BOOL_BODY_BITS(Body, twin_name, entry, body_flags)                                              \
    extern "C" const fbr_body_module_t* entry(void) {                                                            \
        static const fbr_body_module_t m = {FBR_BODY_MODULE_ABI, (uint32_t)sizeof(fbr::WaveParams), twin_name,   \
                                            8u * (uint32_t)sizeof(typename Body::Arg), 1u, (uint32_t)FBR_RES_BITS8, \
                                            (uint32_t)(body_flags), 512u,                                        \
                                            fbr_body_export::launch_bits<Body>, fbr_body_export::occupancy_bits<Body>}; \
        return &m;                                                                                               \
    }

namespace fbr_body_export {
// record bodies: dispatch_record_kernel, dynamic shared memory of Layout<B>::smem(index) bytes
template <class B>
void launch_record(const void* wpv, int grid, void* sv) {
    const fbr::WaveParams& wp = *(const fbr::WaveParams*)wpv;
    cudaStream_t s = (cudaStream_t)sv;
    using L = fbr::record::Layout<B>;
    if constexpr (B::kIndexArg) {
        if (wp.arg_stride == 0) {
            fbr::dispatch_record_kernel<B, true><<<grid, fbr::record::kThreads, L::smem(true), s>>>(wp);
            return;
        }
    }
    fbr::dispatch_record_kernel<B, false><<<grid, fbr::record::kThreads, L::smem(false), s>>>(wp);
}
// Also raises the kernels' dynamic shared-memory limit on the current device; the engine asks for the occupancy on
// every device before the body's first launch there.
template <class B>
int occupancy_record(int index_mode) {
    using L = fbr::record::Layout<B>;
    const void* k = (const void*)fbr::dispatch_record_kernel<B, false>;
    size_t smem = L::smem(false);
    cudaFuncSetAttribute(fbr::dispatch_record_kernel<B, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L::smem(false));
    if constexpr (B::kIndexArg) {
        cudaFuncSetAttribute(fbr::dispatch_record_kernel<B, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L::smem(true));
        if (index_mode) {
            k = (const void*)fbr::dispatch_record_kernel<B, true>;
            smem = L::smem(true);
        }
    }
    return occupancy_of(k, fbr::record::kThreads, smem);
}
// emit bodies: the count pass when wp.emit_values is nullptr, else the emit pass; the occupancy is the smaller of the two
template <class B>
void launch_emit(const void* wpv, int grid, void* sv) {
    if (((const fbr::WaveParams*)wpv)->emit_values == nullptr) launch_record<fbr::record::EmitPass<B, false>>(wpv, grid, sv);
    else launch_record<fbr::record::EmitPass<B, true>>(wpv, grid, sv);
}
template <class B>
int occupancy_emit(int index_mode) {
    return std::min(occupancy_record<fbr::record::EmitPass<B, false>>(index_mode), occupancy_record<fbr::record::EmitPass<B, true>>(index_mode));
}
template <class B>
constexpr fbr_body_launch_fn record_launch() {
    if constexpr (fbr::record::EmitOf<B>::kOn) return launch_emit<B>;
    else return launch_record<B>;
}
template <class B>
constexpr fbr_body_occupancy_fn record_occupancy() {
    if constexpr (fbr::record::EmitOf<B>::kOn) return occupancy_emit<B>;
    else return occupancy_record<B>;
}
template <class B>
constexpr bool record_body_ok() {
    static_assert(std::is_trivially_copyable<typename B::Arg>::value && std::is_trivially_copyable<typename B::Res>::value,
                  "record bodies: Arg and Res are trivially copyable");
    static_assert(!B::kIndexArg || std::is_same<typename B::Arg, int64_t>::value, "record bodies with kIndexArg take Arg = int64_t");
    static_assert(fbr::record::EmitOf<B>::kOn || !std::is_same<typename B::Res, fbr::NoRes>::value,
                  "record bodies: Res = fbr::NoRes needs an Out element type (an emit body)");
    return true;
}
// the flags a record body's descriptor carries on top of the exported ones: broadcast bodies need a block and take it
template <class B>
constexpr uint32_t record_flags() {
    return FBR_BODY_RECORD | (fbr::record::BroadcastOf<B>::kOn ? (FBR_BODY_NEEDS_SHARED | FBR_BODY_BROADCAST) : 0u) |
           (fbr::record::ItemsOf<B>::kOn ? FBR_BODY_ITEMS : 0u) | (fbr::record::EmitOf<B>::kOn ? FBR_BODY_EMIT : 0u);
}
// the descriptor's group_threads: kGroup of a group body, 0 for a one-thread body
template <class B>
constexpr uint32_t record_group() {
    return fbr::record::GroupOf<B>::kG > 1 ? fbr::record::GroupOf<B>::kG : 0u;
}
}  // namespace fbr_body_export

// Body: a RecordBody -- Arg and Res are trivially copyable, sizeof a multiple of 4 and at most 4096, or 32768 for a group
// body within one stage (see the header comment).  The result kind is FBR_RES_BYTES; FBR_BODY_RECORD is added to
// body_flags, which carry FBR_BODY_INDEX_ARG exactly when Body::kIndexArg is true (a range() map of a body without the
// index instantiation would read no arguments).  unit_tasks is the number of tasks whose records fill one shared-memory
// stage of dispatch_record_kernel.  A body with a Shared type also gets FBR_BODY_NEEDS_SHARED | FBR_BODY_BROADCAST and
// its element size and staging budget; a body with kGroup gets group_threads = kGroup; a body with an Item type (or an
// Items = fbr::ItemTypes<...> list) gets FBR_BODY_ITEMS, its item streams and their item sizes.
#define FBR_EXPORT_RECORD_BODY(Body, body_name, entry, body_flags)                                                \
    static_assert(fbr_body_export::record_body_ok<Body>(), "record body");                                       \
    static_assert((((body_flags) & FBR_BODY_INDEX_ARG) != 0) == Body::kIndexArg,                                 \
                  "record bodies: FBR_BODY_INDEX_ARG in the flags if and only if kIndexArg");                     \
    extern "C" const fbr_body_module_t* entry(void) {                                                            \
        static const fbr_body_module_t m = {FBR_BODY_MODULE_ABI, (uint32_t)sizeof(fbr::WaveParams), body_name,   \
                                            fbr::record::Layout<Body>::A, fbr::record::Layout<Body>::R,          \
                                            (uint32_t)(fbr::record::EmitOf<Body>::kOn ? FBR_RES_OFFSETS : FBR_RES_BYTES), \
                                            (uint32_t)(body_flags) | fbr_body_export::record_flags<Body>(),      \
                                            fbr::record::Layout<Body>::kUnit,                                    \
                                            fbr_body_export::record_launch<Body>(), fbr_body_export::record_occupancy<Body>(), \
                                            fbr::record::BroadcastOf<Body>::kElem, fbr::record::BroadcastOf<Body>::kStage, \
                                            fbr_body_export::record_group<Body>(),                               \
                                            fbr::record::ItemsOf<Body>::kElem, fbr::record::EmitOf<Body>::kElem, \
                                            fbr::record::ItemsOf<Body>::kStreams,                                \
                                            {fbr::record::ItemsOf<Body>::elem(1), fbr::record::ItemsOf<Body>::elem(2), \
                                             fbr::record::ItemsOf<Body>::elem(3)}};                              \
        return &m;                                                                                               \
    }

// Body: a ThreadBody (see bodies.cuh) whose Res is 1 or 8 bytes.  result_kind: FBR_RES_BOOL / FBR_RES_I64 / ...
#define FBR_EXPORT_THREAD_BODY(Body, body_name, entry, kind, body_flags)                                         \
    extern "C" const fbr_body_module_t* entry(void) {                                                            \
        static const fbr_body_module_t m = {FBR_BODY_MODULE_ABI, (uint32_t)sizeof(fbr::WaveParams), body_name,   \
                                            (uint32_t)sizeof(typename Body::Arg), (uint32_t)sizeof(typename Body::Res), \
                                            (uint32_t)(kind), (uint32_t)(body_flags), 4096u,                     \
                                            fbr_body_export::launch<Body>, fbr_body_export::occupancy<Body>};    \
        return &m;                                                                                               \
    }
