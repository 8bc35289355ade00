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
// two structs byte for byte (INTEGRATION.md).  Record bodies have no bit-packed twin and no FBR_WANT_SUM; a record body
// that defines identity() and combine() reduces a whole map to one Res on the device instead (a FOLD body, below).
//
// A FOLD record body defines, next to run():
//
//     __host__ __device__ static Res identity();                  // the result of a map of no tasks
//     __device__ static void combine(Res& acc, const Res& x);     // acc <- acc (+) x; one thread; either operand may be
//                                                                 // in shared or in global memory
//
// Res must also be default-constructible (the fold pass holds results in registers).  FBR_EXPORT_RECORD_BODY then sets
// FBR_BODY_FOLD and exports fold_tree_kernel and identity() (evaluated on the host) with its size.
// Any record form may fold (head record or range() index, items, broadcast block, group).  Pool.fold(f, xs) returns
//     tree(x[0..c)): while c > 1: x[i] <- combine(x[2i], x[2i+1]) for every i with 2i+1 < c, an odd last element is
//                    carried to x[c/2]; c <- ceil(c/2)
// over each worker block's results in task order, then over the blocks' totals in block order (identity() for no tasks).
// The order does not depend on chunksize, waves or scheduling, so a float combine gives the same bits on every run of a
// pool of the same size.  Plain maps of a fold body run exactly as before.
//
// A fold body also gets its running fold with no more code (FBR_BODY_SCAN): Pool.accumulate(f, xs) returns n records,
// record i the fold of results 0 .. i under the same block cut.  On one worker y[i] = tree(x[0..i]), which is
// Pool.fold(f, xs[:i+1]) bit for bit; on several, task i of block b gets tree(t_0, ..., t_{b-1}, p_i), t_k block k's
// total and p_i tree() over block b's results up to i, so y[n-1] is Pool.fold(f, xs).  y[0] is the first result itself.
// It is computed without a running carry: with F_1 .. F_k the aligned power-of-two pieces of [0, i) given by the set bits
// of i, largest first (each a complete aligned subtree of tree()), y[i] = F_1 (+) (F_2 (+) ( ... (+) (F_k (+) x[i]))).
//
// A fold body may also define a key for each result (FBR_BODY_KEYED):
//
//     __device__ static uint32_t key(const Res& r);               // which group the result belongs to
//
// Pool.fold_by_key(f, xs, n_keys) then returns n_keys records and a count per key: record k folds the results whose key()
// is k, taken in task order (the subsequence x_k).  On one worker record k is tree(x_k), so it equals
// Pool.fold(f, [x for x in xs if key(f(x)) == k]) bit for bit; on several it is tree() over the per-block trees of x_k in
// block order, counting only blocks where key k has a task.  A key with no task gets identity().  The key is part of the
// result: run() computes it (the nearest centroid, a label taken from the argument), and combine() normally leaves acc's
// key field alone, so a non-empty group's record carries its key and an empty group's record is identity().  A task whose
// key() is not below n_keys fails the map with FBR_TASK_KEY.  FBR_EXPORT_RECORD_BODY exports the keys entry (keys_kernel)
// and the fold_segments entry (a segmented tree()) after scan.
//
// The same body also folds by any 32-bit key: Pool.fold_by_sparse_key(f, xs) returns one record per distinct key that some
// task produced, in ascending key order, with its key and its count (FBR_FOLD_SPARSE_KEYS).  Record k is fold_by_key's
// record k with the keys without tasks left out, so one worker again gives Pool.fold(f, [x for x in xs if key(f(x)) == k]).
// The key 0xFFFFFFFF is reserved: the engine calls the keys entry with n_keys = 0xFFFFFFFF, and a task whose key() is
// 0xFFFFFFFF fails the map with FBR_TASK_KEY.  No other body code is needed.
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
// fold bodies: FoldPass<B> for a fold map (wp.fold_partials set), else the plain kernels.  index_mode bit 1 asks for the
// fold pass's occupancy, so plain maps keep their own
template <class B>
void launch_foldable(const void* wpv, int grid, void* sv) {
    if (((const fbr::WaveParams*)wpv)->fold_partials != nullptr) launch_record<fbr::record::FoldPass<B>>(wpv, grid, sv);
    else launch_record<B>(wpv, grid, sv);
}
template <class B>
int occupancy_foldable(int index_mode) {
    if (index_mode & 2) return occupancy_record<fbr::record::FoldPass<B>>(index_mode & 1);
    return occupancy_record<B>(index_mode);
}
// tree() over n >= 1 device records (overwritten) into dst: fold_tree_kernel over tiles, then over the tile totals
template <class B>
void launch_fold(void* values, uint64_t n, void* dst, void* sv) {
    constexpr uint64_t T = fbr::record::kFoldTile;
    uint64_t stride = sizeof(typename B::Res);
    for (;;) {
        const uint64_t tiles = (n + T - 1) / T;
        fbr::fold_tree_kernel<B><<<(unsigned)std::min<uint64_t>(tiles, 1u << 16), fbr::kThreads, 0, (cudaStream_t)sv>>>(
            (uint8_t*)values, n, stride, tiles == 1 ? (uint8_t*)dst : nullptr);
        if (tiles <= 1) return;
        n = tiles;
        stride *= T;
    }
}
template <class B>
const void* fold_identity() {
    if constexpr (fbr::record::FoldOf<B>::kOn) {
        static const typename B::Res id = B::identity();
        return &id;
    } else {
        return nullptr;
    }
}
// prefix folds of n device records (in place) of a fold body, then wrapped with n_pieces device records, right-nested
// (scan_level_kernel per level of complete subtrees, then scan_wrap_kernel); returns a cudaError_t.  The levels (fewer
// than n records) and, for records over kScanRegBytes, one scratch record per thread are allocated on the stream.
template <class B>
int launch_scan(void* values, uint64_t n, int prefix, const void* pieces, uint32_t n_pieces, void* sv) {
    constexpr uint64_t R = sizeof(typename B::Res);
    const cudaStream_t s = (cudaStream_t)sv;
    if (n == 0) return (int)cudaSuccess;
    // this module's own last error: a launch of its other entries has already been reported through the engine's checks
    (void)cudaGetLastError();
    uint64_t off[fbr::kScanMaxLevels] = {}, level_records = 0;
    int levels = 0;   // levels 1 .. levels hold n >> k complete subtrees each
    if (prefix)
        for (uint64_t c = n >> 1; c; c >>= 1) {
            off[++levels] = level_records;
            level_records += c;
        }
    uint64_t grid = std::min<uint64_t>((n + fbr::kThreads - 1) / fbr::kThreads, 4096);
    if (R > fbr::kScanRegBytes)   // scratch records: at most 64 MiB of them
        grid = std::min<uint64_t>(grid, std::max<uint64_t>(1, (64ull << 20) / (R * fbr::kThreads)));
    const uint64_t tmp_bytes = R > fbr::kScanRegBytes ? grid * fbr::kThreads * R : 0;
    uint8_t* buf = nullptr;
    cudaError_t e = cudaSuccess;
    if (level_records * R + tmp_bytes) e = cudaMallocAsync((void**)&buf, level_records * R + tmp_bytes, s);
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        return (int)e;
    }
    fbr::ScanLevels lv{};
    const uint8_t* src = (const uint8_t*)values;
    for (int k = 1; k <= levels; ++k) {
        uint8_t* dst = buf + off[k] * R;
        const uint64_t c = n >> k;
        fbr::scan_level_kernel<B><<<(unsigned)std::min<uint64_t>((c + fbr::kThreads - 1) / fbr::kThreads, 4096), fbr::kThreads, 0, s>>>(
            src, dst, c);
        lv.at[k] = src = dst;
        if ((e = cudaGetLastError()) != cudaSuccess) break;
    }
    if (e == cudaSuccess) {
        fbr::scan_wrap_kernel<B><<<(unsigned)grid, fbr::kThreads, 0, s>>>((uint8_t*)values, n, prefix, lv, (const uint8_t*)pieces,
                                                                          n_pieces, buf ? buf + level_records * R : nullptr);
        e = cudaGetLastError();
    }
    if (buf) cudaFreeAsync(buf, s);
    return (int)e;
}
// keyed fold bodies: key[i] = B::key(values[i]) for n device records; a key >= n_keys is stored as 0 and the lowest such
// task, first_task + i, goes into *err as (task << 8 | FBR_TASK_KEY) by atomicMin.  Returns the launch's cudaError_t.
template <class B>
int launch_keys(const void* values, uint64_t n, uint32_t n_keys, uint64_t first_task, uint32_t* keys, unsigned long long* err,
                void* sv) {
    if (n == 0) return (int)cudaSuccess;
    (void)cudaGetLastError();
    fbr::keys_kernel<B><<<(unsigned)std::min<uint64_t>((n + fbr::kThreads - 1) / fbr::kThreads, 8192), fbr::kThreads, 0, (cudaStream_t)sv>>>(
        (const uint8_t*)values, n, n_keys, first_task, keys, err);
    return (int)cudaGetLastError();
}
// tree() of each of the S segments [offsets[k], offsets[k + 1]) of the n key-ordered device records at `values` (folded in
// place) into dst[k], identity() for an empty segment.  offsets are S + 1 device words, non-decreasing, offsets[S] <= n.  Each
// level folds kFoldTile-record tiles aligned at every segment's start, then the next level folds the tile totals, until no
// segment has more than one record left (at most ceil(log_kFoldTile(n)) levels).  The tile numbering and the identity live in
// stream-ordered scratch.
template <class B>
int launch_fold_segments(void* values, uint64_t n, const uint64_t* offsets, uint32_t S, void* dst, void* sv) {
    constexpr uint64_t R = sizeof(typename B::Res), T = fbr::record::kFoldTile;
    const cudaStream_t s = (cudaStream_t)sv;
    if (S == 0) return (int)cudaSuccess;
    (void)cudaGetLastError();
    const uint64_t states = S / fbr::scan::kTile + 1;   // scan_counts_kernel: the tile holding index S writes the end
    // tiles[S] | tile_offs[S + 1] | tile_state[states] | total | ticket | identity
    const uint64_t o_offs = S, o_state = o_offs + S + 1, o_total = o_state + states, o_ticket = o_total + 1, o_id = o_ticket + 1;
    uint64_t* buf = nullptr;
    cudaError_t e = cudaMallocAsync((void**)&buf, o_id * 8 + R, s);
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        return (int)e;
    }
    uint8_t* const id = (uint8_t*)(buf + o_id);
    e = cudaMemcpyAsync(id, fold_identity<B>(), R, cudaMemcpyHostToDevice, s);
    const unsigned seg_grid = (unsigned)std::min<uint64_t>((S + fbr::kThreads - 1) / fbr::kThreads, 1024);
    for (uint64_t step = 1; e == cudaSuccess && step < n; step *= T) {
        e = cudaMemsetAsync(buf + o_state, 0, (states + 2) * 8, s);
        if (e != cudaSuccess) break;
        fbr::seg_tiles_kernel<<<seg_grid, fbr::kThreads, 0, s>>>(offsets, S, step, buf);
        fbr::scan_counts_kernel<<<(unsigned)states, fbr::scan::kThreads, 0, s>>>(buf, S, buf + o_offs, (unsigned long long*)(buf + o_state),
                                                                               (uint32_t*)(buf + o_ticket), buf + o_total);
        // at most one tile per kFoldTile records at this level, plus one partial tile per segment
        const uint64_t grid = std::min<uint64_t>((n + step * T - 1) / (step * T) + S, 1u << 16);
        fbr::fold_segments_kernel<B><<<(unsigned)grid, fbr::kThreads, 0, s>>>((uint8_t*)values, offsets, S, step, buf + o_offs);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        fbr::fold_segments_out_kernel<B><<<(unsigned)std::min<uint64_t>((S + 7) / 8, 8192), fbr::kThreads, 0, s>>>(
            (const uint8_t*)values, offsets, S, (uint8_t*)dst, id);
        e = cudaGetLastError();
    }
    cudaFreeAsync(buf, s);
    return (int)e;
}
template <class B>
constexpr int (*record_keys())(const void*, uint64_t, uint32_t, uint64_t, uint32_t*, unsigned long long*, void*) {
    if constexpr (fbr::record::KeyOf<B>::kOn) return launch_keys<B>;
    else return nullptr;
}
template <class B>
constexpr int (*record_fold_segments())(void*, uint64_t, const uint64_t*, uint32_t, void*, void*) {
    if constexpr (fbr::record::KeyOf<B>::kOn) return launch_fold_segments<B>;
    else return nullptr;
}
template <class B>
constexpr fbr_body_launch_fn record_launch() {
    if constexpr (fbr::record::EmitOf<B>::kOn) return launch_emit<B>;
    else if constexpr (fbr::record::FoldOf<B>::kOn) return launch_foldable<B>;
    else return launch_record<B>;
}
template <class B>
constexpr fbr_body_occupancy_fn record_occupancy() {
    if constexpr (fbr::record::EmitOf<B>::kOn) return occupancy_emit<B>;
    else if constexpr (fbr::record::FoldOf<B>::kOn) return occupancy_foldable<B>;
    else return occupancy_record<B>;
}
template <class B>
constexpr void (*record_fold())(void*, uint64_t, void*, void*) {
    if constexpr (fbr::record::FoldOf<B>::kOn) return launch_fold<B>;
    else return nullptr;
}
template <class B>
constexpr int (*record_scan())(void*, uint64_t, int, const void*, uint32_t, void*) {
    if constexpr (fbr::record::FoldOf<B>::kOn) return launch_scan<B>;
    else return nullptr;
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
           (fbr::record::ItemsOf<B>::kOn ? FBR_BODY_ITEMS : 0u) | (fbr::record::EmitOf<B>::kOn ? FBR_BODY_EMIT : 0u) |
           (fbr::record::FoldOf<B>::kOn ? (FBR_BODY_FOLD | FBR_BODY_SCAN) : 0u) | (fbr::record::KeyOf<B>::kOn ? FBR_BODY_KEYED : 0u);
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
// Items = fbr::ItemTypes<...> list) gets FBR_BODY_ITEMS, its item streams and their item sizes; a body with combine() gets
// FBR_BODY_FOLD | FBR_BODY_SCAN, its fold entry (fold_tree_kernel), its identity() and its scan entry (scan_level_kernel,
// scan_wrap_kernel); a fold body with key() also gets FBR_BODY_KEYED and its keys and fold_segments entries.
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
                                             fbr::record::ItemsOf<Body>::elem(3)},                               \
                                            fbr_body_export::record_fold<Body>(), fbr_body_export::fold_identity<Body>(), \
                                            fbr::record::FoldOf<Body>::kOn ? fbr::record::Layout<Body>::R : 0u,   \
                                            fbr_body_export::record_scan<Body>(),                                \
                                            fbr_body_export::record_keys<Body>(), fbr_body_export::record_fold_segments<Body>()}; \
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
