// kernels.cuh -- the sm_90a kernels of the Pool.map hot path.
//
//   dispatch_*_kernel  : persistent CTAs claim fixed-layout task records from the device task ring
//                        by atomic ticket, run the mapped body, and write the unit's results plus a
//                        16 B header into the paired slot of the result ring.
//                        Replaces _handle_tasks + PUSH/PULL + zpool_worker_core
//                        (fiber/pool.py:952-963, 783-824).
//   gather_ordered_kernel : result ring -> ordered output by index placement, optional sum
//                        epilogue.  Replaces result_conn.send xN + _res_get + Inventory.get
//                        (fiber/pool.py:814-824, 968-973, 666-679).
//   payload_fill_kernel : synthetic 4 KB records for BASELINE.json config 4.
//   fold_tree_kernel   : tree() over a fold body's records (a block's unit partials, block totals).
//
// Everything here is HBM-bound byte/integer work (no dense contraction => no tensor cores):
// 16 B vector accesses, fully coalesced, grids sized as (SM count x resident CTAs).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <type_traits>
#include <utility>

#include "bodies.cuh"

namespace fbr {

constexpr int kThreads = 256;

// One claim unit = `count` consecutive tasks of one map.  32 B, written by the host into the
// pinned task ring and copied to the device ring with cudaMemcpyAsync.  It is the fixed-layout
// stand-in for the reference's pickled task tuple (seq, batch_start, func, chunk, starmap)
// (fiber/pool.py:1181).
struct TaskRecord {
    uint32_t seq;       // map id (Inventory seq, fiber/pool.py:659-664), low 32 bits
    uint32_t count;     // tasks in this unit
    uint64_t first;     // index of the unit's first task inside the map (the reference's `batch`)
    uint64_t arg_off;   // byte offset of the unit's first argument record in the wave's arg ring
    uint32_t func_id;
    uint32_t attempt;   // re-dispatch count (resilient pool)
};
static_assert(sizeof(TaskRecord) == 32, "task record layout is part of the ABI");

// Header of a result-ring slot: the fixed-layout stand-in for the reference's per-item result
// message (seq, batch, batch + i, res) (fiber/pool.py:814,821), one per unit instead of per item.
struct SlotHeader {
    uint32_t seq;
    uint32_t count;     // bit 31: unit lost (its worker "died"), must be re-dispatched
    uint64_t first;
};
static_assert(sizeof(SlotHeader) == 16, "slot header layout is part of the ABI");
constexpr uint32_t kUnitLost = 0x80000000u;

// Item stream k >= 1 of a multi-stream items record body (stream 0 lives in WaveParams::items ...): the same fields, with
// the map index of offs[0] shared with stream 0 (item_first), since every stream is cut at the same tasks
struct ItemStream {
    const uint8_t* items;
    const uint64_t* offs;
    uint64_t base;              // item index of items[0]
    uint64_t count;             // offsets end here (the stream's n_items)
};
constexpr uint32_t kMaxItemStreams = 4;

struct WaveParams {
    const TaskRecord* records;  // device task ring window of this wave; nullptr: the wave is a contiguous,
                                // unshuffled block and unit t's record is computed from the syn_* fields below
                                // (an arithmetic progression needs no 32 B/unit of PCIe traffic)
    SlotHeader* headers;        // result ring headers (paired with records by ticket); nullptr: direct placement --
                                // `ring` IS the ordered output window and slot t lands at its final index, no gather
    uint8_t* ring;              // result ring payload arena (or the ordered output window, see headers)
    uint32_t* ticket;           // device counter, zero at launch
    uint32_t n_units;
    uint32_t slot_stride;       // bytes, multiple of 16
    const uint8_t* args;        // device argument ring window (arg_off is relative to it)
    uint32_t arg_stride;        // 0 => implicit index arguments
    int64_t index_start, index_step;
    uint64_t index_base;        // global index of the map's task 0
    const uint8_t* shared;      // broadcast argument block
    uint64_t shared_bytes;
    unsigned long long* err_word;
    uint32_t resilient;         // lost units are re-dispatched by the host (else a fault is an error)
    long long* sum;             // fold sum(results) here (nullptr: no fold); done where the values are in registers.
                                // 8-byte results: sum of the LOW 32-bit halves (as unsigned) ...
    long long* sum_hi;          // ... and sum of the high halves (arithmetic >> 32) here: the exact, unbounded sum
                                // is sum_hi * 2^32 + sum, whatever the int64 total would have wrapped to
    // synthesised records (records == nullptr): unit t = tasks [syn_first + t*syn_unit, ...) of map syn_seq
    uint64_t syn_first;         // map index of the wave's first task
    uint64_t syn_tasks;         // tasks in the wave
    uint64_t syn_arg_off;       // arg_off of unit 0
    uint32_t syn_unit;          // tasks per unit
    uint32_t syn_seq;
    uint32_t syn_func;
    uint32_t syn_attempt;       // re-dispatch count of the whole wave (a dead worker's block re-run elsewhere)
    uint64_t n_items;           // bodies whose task consumes several argument items (bit-packed bool twins: 8 per
                                // task): number of items of the whole map, items at or past it are not read
    // items record bodies (FBR_BODY_ITEMS): map task j reads items [o[j], o[j+1]) with o = item_offs - item_first, and
    // item k lies at items + (k - item_base) * item_bytes.  Offsets outside [item_base, item_count] are bad arguments
    const uint8_t* items;
    const uint64_t* item_offs;
    uint64_t item_first;        // map index of item_offs[0]
    uint64_t item_base;         // item index of items[0]
    uint64_t item_count;        // offsets end here (the map's n_items)
    // emit record bodies (FBR_BODY_EMIT): nullptr runs the count pass (each task's record is its value count).  Otherwise
    // the emit pass: task j writes its values at emit_values + o[j] * out_bytes with o = emit_offs - emit_first (the part's
    // exclusive offsets, o[j + 1] its end), and its record is its global end offset emit_base + o[j + 1]
    uint8_t* emit_values;
    const uint64_t* emit_offs;
    uint64_t emit_first;
    uint64_t emit_base;
    // items record bodies with K = 2 to 4 streams (Items = ItemTypes<...>): streams 1 .. K-1, read like stream 0 above.
    // Appended after every other field, so their offsets stay where one-stream kernels expect them
    ItemStream more_items[kMaxItemStreams - 1];
    // fold maps of record bodies with combine() (FoldPass): the unit of tasks [first, first + count) writes its tree to
    // fold_partials + (first - fold_first) / syn_unit * sizeof(Res) -- its place in its block, never its ticket (syn_unit
    // is a power of two)
    uint8_t* fold_partials;
    uint64_t fold_first;        // map index of the block's first task
};

// Task record of ticket t: from the device task ring, or computed (contiguous wave).
__device__ __forceinline__ TaskRecord wave_record(const WaveParams& wp, uint32_t t) {
    if (wp.records != nullptr) return wp.records[t];
    const uint64_t off = (uint64_t)t * wp.syn_unit;
    const uint64_t left = wp.syn_tasks - off;
    TaskRecord r;
    r.seq = wp.syn_seq;
    r.count = left < (uint64_t)wp.syn_unit ? (uint32_t)left : wp.syn_unit;
    r.first = wp.syn_first + off;
    r.arg_off = wp.syn_arg_off + off * (uint64_t)wp.arg_stride;
    r.func_id = wp.syn_func;
    r.attempt = wp.syn_attempt;
    return r;
}
__device__ __forceinline__ void put_header(const WaveParams& wp, uint32_t t, const SlotHeader& h) {
    if (wp.headers != nullptr) wp.headers[t] = h;
}

// ------------------------------------------------------------------------------------------------
// streaming 16 B accesses
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 ld_stream(const void* p) { return __ldcs(reinterpret_cast<const uint4*>(p)); }
__device__ __forceinline__ void st_vec(void* p, const uint4& v) { *reinterpret_cast<uint4*>(p) = v; }

// Ticket claim with prefetch: thread 0 holds the next ticket while the CTA works on the current
// one, so the ~700-cycle L2 atomic round trip is off the critical path.
struct TicketClaimer {
    uint32_t* counter;
    uint32_t next;  // valid in thread 0 only
    __device__ __forceinline__ void prime() {
        if (threadIdx.x == 0) next = atomicAdd(counter, 1u);
    }
    // returns the ticket for this iteration (uniform across the CTA) and prefetches the following one
    __device__ __forceinline__ uint32_t claim(uint32_t* s_slot) {
        __syncthreads();  // previous iteration's readers of *s_slot are done
        if (threadIdx.x == 0) {
            *s_slot = next;
            next = atomicAdd(counter, 1u);
        }
        __syncthreads();
        return *s_slot;
    }
    // Re-arm the counter for the wave that uses it next.  Every CTA draws exactly two tickets >= n_units (the
    // one that ends its loop and the one prefetched behind it), so n_units + 2*gridDim.x atomics happen in
    // all, and the highest value is always a prefetched, unused one: its holder knows every other atomic
    // has been performed and zeroes the counter (no memset node, no gather kernel needed for it).
    __device__ __forceinline__ void rearm(uint32_t n_units) {
        if (threadIdx.x == 0 && next == n_units + 2u * gridDim.x - 1u) *counter = 0u;
    }
    // one-barrier variant: `s_slots[2]` is indexed by iteration parity (see dispatch_thread_kernel)
    __device__ __forceinline__ uint32_t claim_db(uint32_t* s_slots, uint32_t iter) {
        if (threadIdx.x == 0) {
            s_slots[iter & 1] = next;
            next = atomicAdd(counter, 1u);
        }
        __syncthreads();
        return s_slots[iter & 1];
    }
};

// Fold one value per thread into a global accumulator: warp shuffle, then one atomic per warp (no
// block barrier: a __syncthreads() after the persistent loop made ptxas restructure the whole loop,
// +15 % instructions on the pi body).
// (unsigned arithmetic throughout: two's-complement wrap-around is defined, signed overflow is not)
__device__ __forceinline__ void warp_add(unsigned long long v, long long* target) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0 && v != 0) atomicAdd(reinterpret_cast<unsigned long long*>(target), v);
}

// ================================================================================================
// dispatch: ThreadBody -- one thread per task, V = 16/sizeof(Res) consecutive tasks per thread so
// each thread emits one 16 B store; a warp writes 512 contiguous bytes of the ring slot.
// ================================================================================================
// The slice of one unit that thread `vt` (0..kThreads-1) of the unit's thread grid owns: vectors
// vt, vt + kThreads, ...  Adds the slice's results to unit_acc / unit_acc32.
template <class B, bool kIndex>
__device__ __forceinline__ void run_unit_slice(const WaveParams& wp, const TaskRecord& rec, uint8_t* slot, uint32_t vt,
                                               const ErrSink& es, unsigned long long& unit_acc, unsigned long long& unit_hi,
                                               uint32_t& unit_acc32) {
    using Arg = typename B::Arg;
    using Res = typename B::Res;
    constexpr int V = (sizeof(Res) >= 16) ? 1 : (16 / (int)sizeof(Res));
    const uint8_t* uargs = wp.args + rec.arg_off;
    for (uint32_t base = vt * V; base < rec.count; base += kThreads * V) {
        // implicit range() argument: one multiply per thread, then strength-reduced adds
        // (keeps the integer-multiply pipe for the body: Philox needs 18 IMAD.WIDE per task)
        int64_t a_idx = 0;
        if constexpr (kIndex) a_idx = wp.index_start + (int64_t)(rec.first + base) * wp.index_step;
        const uint64_t gidx0 = wp.index_base + rec.first + base;
        uint8_t* dst = slot + (size_t)base * sizeof(Res);
        if (base + V <= rec.count) {
            // full vector: no per-task bounds checks (a branch per task cost 6 instructions and
            // serialised the tasks' dependency chains); results are packed into one 16 B
            // register vector (no local-memory staging)
            uint32_t pk[4] = {0u, 0u, 0u, 0u};
            if constexpr (kIndex && B::kVecIndex) {
                B::template run_index_vec<V>(a_idx, wp.index_step, pk);
            } else {
#pragma unroll
                for (int v = 0; v < V; ++v) {
                    Arg a;
                    if constexpr (kIndex) { a = (Arg)a_idx; a_idx += wp.index_step; }
                    else a = *reinterpret_cast<const Arg*>(uargs + (size_t)(base + v) * wp.arg_stride);
                    const Res r = B::run(a, gidx0 + v, es, rec.attempt);
                    if constexpr (sizeof(Res) == 1) {
                        pk[v >> 2] |= (uint32_t)(uint8_t)r << ((v & 3) * 8);
                    } else if constexpr (sizeof(Res) == 8) {
                        unsigned long long bits;
                        memcpy(&bits, &r, 8);
                        unit_acc += bits & 0xffffffffull;
                        unit_hi += (unsigned long long)((long long)bits >> 32);
                        pk[2 * v] = (uint32_t)bits;
                        pk[2 * v + 1] = (uint32_t)(bits >> 32);
                    } else {
                        static_assert(sizeof(Res) == 1 || sizeof(Res) == 8, "add a packing rule for this result size");
                    }
                }
            }
            if constexpr (sizeof(Res) == 1) {     // byte results: fold the packed words with dp4a
                uint32_t s4 = __dp4a(pk[0], 0x01010101u, 0u);
                s4 = __dp4a(pk[1], 0x01010101u, s4);
                s4 = __dp4a(pk[2], 0x01010101u, s4);
                s4 = __dp4a(pk[3], 0x01010101u, s4);
                unit_acc32 += s4;
            }
            st_vec(dst, make_uint4(pk[0], pk[1], pk[2], pk[3]));
        } else {
            // the unit's partial tail vector (at most one per unit): one task at a time, kept
            // rolled so the kernel holds a single copy of the unrolled body
#pragma unroll 1
            for (uint32_t i = base; i < rec.count; ++i) {
                Arg a;
                if constexpr (kIndex) { a = (Arg)a_idx; a_idx += wp.index_step; }
                else a = *reinterpret_cast<const Arg*>(uargs + (size_t)i * wp.arg_stride);
                const Res r = B::run(a, gidx0 + (i - base), es, rec.attempt);
                if constexpr (sizeof(Res) == 1) unit_acc32 += (uint32_t)(uint8_t)r;
                else if constexpr (sizeof(Res) == 8) {
                    unsigned long long bits;
                    memcpy(&bits, &r, 8);
                    unit_acc += bits & 0xffffffffull;
                    unit_hi += (unsigned long long)((long long)bits >> 32);
                }
                memcpy(dst + (size_t)(i - base) * sizeof(Res), &r, sizeof(Res));
            }
        }
    }
}

// kIndex: the task index itself is the argument (range()); a separate instantiation keeps each
// kernel to one copy of the unrolled body (the two-path version was 45 KB of SASS, beyond the 32 KB
// instruction cache level).
//
// One barrier per unit: the ticket slot (and, for bodies that can lose a unit, the fault flag) is
// double-buffered by iteration parity, so the write of iteration i+2 is ordered after the reads of
// iteration i by the barrier of iteration i+1.  (Warp-granular claims with no barrier at all were
// tried and dropped: the skew between a CTA's warps is not what limits this kernel.)
template <class B, bool kIndex>
__global__ void __launch_bounds__(kThreads) dispatch_thread_kernel(const WaveParams wp) {
    __shared__ uint32_t s_ticket[2];
    __shared__ int s_fault[2];
    if (threadIdx.x == 0) { s_fault[0] = 0; s_fault[1] = 0; }
    TicketClaimer tc{wp.ticket, 0u};
    tc.prime();
    unsigned long long acc = 0, acc_hi = 0;   // sums of this thread's results over every unit its CTA completed
    for (uint32_t iter = 0;; ++iter) {
        const uint32_t t = tc.claim_db(s_ticket, iter);
        if (t >= wp.n_units) break;
        int* const unit_fault = &s_fault[iter & 1];
        const ErrSink es{wp.err_word, unit_fault};
        const TaskRecord rec = wave_record(wp, t);
        unsigned long long unit_acc = 0, unit_hi = 0;
        uint32_t unit_acc32 = 0;
        run_unit_slice<B, kIndex>(wp, rec, wp.ring + (size_t)t * wp.slot_stride, threadIdx.x, es, unit_acc, unit_hi, unit_acc32);
        bool lost = false;
        if constexpr (B::kCanFault) {
            __syncthreads();      // every thread's fault reports for this unit are in
            lost = *unit_fault != 0;
            // re-arm the other flag for the next unit: its last readers ran before this barrier,
            // its next writers run after the next claim barrier
            if (threadIdx.x == 0) s_fault[(iter + 1) & 1] = 0;
        }
        if (!lost) {                                          // a lost unit is re-dispatched: never folded twice
            acc += unit_acc + unit_acc32;
            acc_hi += unit_hi;
        }
        if (threadIdx.x == 0) {
            // A dead worker loses its whole chunk.  ResilientZPool re-queues it; in the plain ZPool
            // the map would hang forever (fiber/pool.py:801-824 has no try/except) -- here it is
            // reported as a task error instead.
            if (lost && !wp.resilient)
                atomicMin(wp.err_word, (unsigned long long)(((wp.index_base + rec.first) << 8) | TASK_FAULT));
            put_header(wp, t, SlotHeader{rec.seq, rec.count | ((lost && wp.resilient) ? kUnitLost : 0u), rec.first});
        }
    }
    tc.rearm(wp.n_units);
    if (wp.sum != nullptr) {
        warp_add(acc, wp.sum);
        if constexpr (sizeof(typename B::Res) == 8) warp_add(acc_hi, wp.sum_hi);
    }
}

// ================================================================================================
// dispatch: pi_inside_bits8 -- task g is the 8 range() indices 8g..8g+7, its result one byte (bit k =
// is_inside(index 8g+k)).  A thread owns two consecutive bytes of the unit (16 indices, the same
// Philox vector as the byte-result kernel) and stores them as one uint16; a warp writes 64
// contiguous bytes.  Algorithmic bytes per index: 0 read + 1/8 written.
// ================================================================================================
__global__ void __launch_bounds__(kThreads) dispatch_pi_bits_kernel(const WaveParams wp) {
    __shared__ uint32_t s_ticket[2];
    TicketClaimer tc{wp.ticket, 0u};
    tc.prime();
    unsigned long long acc = 0;
    for (uint32_t iter = 0;; ++iter) {
        const uint32_t t = tc.claim_db(s_ticket, iter);
        if (t >= wp.n_units) break;
        const TaskRecord rec = wave_record(wp, t);
        uint8_t* slot = wp.ring + (size_t)t * wp.slot_stride;
        for (uint32_t b = threadIdx.x * 2; b < rec.count; b += kThreads * 2) {
            const int64_t a0 = wp.index_start + (int64_t)((rec.first + b) * 8ull) * wp.index_step;
            const uint32_t bits = PiInsideDet::run_index_bits16(a0, wp.index_step);
            if (b + 2 <= rec.count) {
                *reinterpret_cast<uint16_t*>(slot + b) = (uint16_t)bits;
                acc += __popc(bits);
            } else {                                  // odd byte count: the unit's last byte
                slot[b] = (uint8_t)bits;
                acc += __popc(bits & 0xffu);
            }
        }
        if (threadIdx.x == 0) put_header(wp, t, SlotHeader{rec.seq, rec.count, rec.first});
    }
    tc.rearm(wp.n_units);
    if (wp.sum != nullptr) warp_add(acc, wp.sum);
}

// ================================================================================================
// dispatch: bit-packed twin of ANY bool ThreadBody: 8 items per byte-task, items being explicit argument
// records (B::Arg, kIndex = false) or range() indices (kIndex = true: item i is index_start + i*index_step,
// no argument bytes).  A warp takes 512 consecutive items per pass: lane l evaluates items l, l+32, ...
// (each load instruction reads 32 consecutive records: fully coalesced), and the ballot of pass j IS word j
// of the warp's 64 output bytes (bit l = lane l's result = item 32j + l) -- no shuffles, no transposes.
// Lanes 0..15 store the 16 words: 64 contiguous bytes per warp.  Items at or past wp.n_items are not
// evaluated and leave zero bits.  Algorithmic bytes per item: sizeof(Arg) read + 1/8 written.
// ================================================================================================
template <class B, bool kIndex = false>
__global__ void __launch_bounds__(kThreads) dispatch_bits_items_kernel(const WaveParams wp) {
    using Arg = typename B::Arg;
    static_assert(!B::kCanFault, "bit-packed twins are for bodies that cannot lose a unit");
    __shared__ uint32_t s_ticket[2];
    __shared__ int s_fault;
    TicketClaimer tc{wp.ticket, 0u};
    tc.prime();
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const ErrSink es{wp.err_word, &s_fault};
    unsigned long long acc = 0;
    for (uint32_t iter = 0;; ++iter) {
        const uint32_t t = tc.claim_db(s_ticket, iter);
        if (t >= wp.n_units) break;
        const TaskRecord rec = wave_record(wp, t);
        uint8_t* slot = wp.ring + (size_t)t * wp.slot_stride;
        const uint8_t* uargs = wp.args + rec.arg_off;
        const uint64_t item0 = rec.first * 8ull;                       // map-level index of the unit's first item
        const uint32_t n_it = rec.count * 8u;                          // items covered by this unit's bytes
        for (uint32_t base = warp * 512u; base < n_it; base += (kThreads / 32) * 512u) {
            uint32_t mine = 0u;                                        // word `lane` of this pass block (lanes 0..15)
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const uint32_t i = base + 32u * j + lane;
                bool r = false;
                if (i < n_it && item0 + i < wp.n_items) {
                    Arg a;
                    if constexpr (kIndex) a = (Arg)(wp.index_start + (int64_t)(item0 + i) * wp.index_step);
                    else a = *reinterpret_cast<const Arg*>(uargs + (size_t)i * sizeof(Arg));
                    r = B::run(a, wp.index_base + item0 + i, es, rec.attempt) != 0;
                }
                const uint32_t word = __ballot_sync(0xffffffffu, r);
                if (lane == (uint32_t)j) mine = word;
            }
            if (lane < 16) {
                const uint32_t byte0 = (base >> 3) + lane * 4u;            // this word's first byte inside the slot
                if (byte0 + 4u <= rec.count) {
                    *reinterpret_cast<uint32_t*>(slot + byte0) = mine;
                } else {
                    for (uint32_t b = byte0; b < rec.count; ++b) slot[b] = (uint8_t)(mine >> ((b - byte0) * 8u));
                }
                acc += __popc(mine);
            }
        }
        if (threadIdx.x == 0) put_header(wp, t, SlotHeader{rec.seq, rec.count, rec.first});
    }
    tc.rearm(wp.n_units);
    if (wp.sum != nullptr) warp_add(acc, wp.sum);
}

// ================================================================================================
// dispatch: payload_map_4k -- a CTA streams its unit's 4 KB records: thread j owns the j-th 16 B
// column of every record, 4 records in flight per thread (16 KB per CTA in flight).
//   out[w] = in[w] * 2654435761 + t   (u32 wrap), t = global task index.
// Algorithmic bytes per task: 4096 read + 4096 written.
// ================================================================================================
__global__ void __launch_bounds__(kThreads) dispatch_payload_map_kernel(const WaveParams wp) {
    __shared__ uint32_t s_ticket;
    TicketClaimer tc{wp.ticket, 0u};
    tc.prime();
    constexpr int U = 4;
    for (;;) {
        const uint32_t t = tc.claim(&s_ticket);
        if (t >= wp.n_units) break;
        const TaskRecord rec = wave_record(wp, t);
        const uint8_t* src = wp.args + rec.arg_off + threadIdx.x * 16;
        uint8_t* dst = wp.ring + (size_t)t * wp.slot_stride + threadIdx.x * 16;
        const uint32_t tbase = (uint32_t)(wp.index_base + rec.first);
        uint32_t r = 0;
        for (; r + U <= rec.count; r += U) {
            uint4 v[U];
#pragma unroll
            for (int u = 0; u < U; ++u) v[u] = ld_stream(src + (size_t)(r + u) * wp.arg_stride);
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const uint32_t tt = tbase + r + u;
                v[u].x = v[u].x * kPayloadMul + tt;
                v[u].y = v[u].y * kPayloadMul + tt;
                v[u].z = v[u].z * kPayloadMul + tt;
                v[u].w = v[u].w * kPayloadMul + tt;
                st_vec(dst + (size_t)(r + u) * kPayloadBytes, v[u]);
            }
        }
        for (; r < rec.count; ++r) {
            uint4 v = ld_stream(src + (size_t)r * wp.arg_stride);
            const uint32_t tt = tbase + r;
            v.x = v.x * kPayloadMul + tt; v.y = v.y * kPayloadMul + tt;
            v.z = v.z * kPayloadMul + tt; v.w = v.w * kPayloadMul + tt;
            st_vec(dst + (size_t)r * kPayloadBytes, v);
        }
        if (threadIdx.x == 0) put_header(wp, t, SlotHeader{rec.seq, rec.count, rec.first});
    }
    tc.rearm(wp.n_units);
}

// ================================================================================================
// dispatch: payload_checksum_4k -- one warp per record, 8 coalesced 16 B loads per lane, shuffle
// reduce, lane 0 stores the u32.  Algorithmic bytes per task: 4096 read + 4 written.
// ================================================================================================
__global__ void __launch_bounds__(kThreads) dispatch_payload_checksum_kernel(const WaveParams wp) {
    __shared__ uint32_t s_ticket;
    TicketClaimer tc{wp.ticket, 0u};
    tc.prime();
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    unsigned long long acc = 0;
    for (;;) {
        const uint32_t t = tc.claim(&s_ticket);
        if (t >= wp.n_units) break;
        const TaskRecord rec = wave_record(wp, t);
        uint32_t* dst = reinterpret_cast<uint32_t*>(wp.ring + (size_t)t * wp.slot_stride);
        for (uint32_t r = warp; r < rec.count; r += kThreads / 32) {
            const uint8_t* src = wp.args + rec.arg_off + (size_t)r * wp.arg_stride + lane * 16;
            uint4 v[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] = ld_stream(src + k * 512);
            uint32_t s = 0;
#pragma unroll
            for (int k = 0; k < 8; ++k) s += v[k].x + v[k].y + v[k].z + v[k].w;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (lane == 0) { dst[r] = s; acc += s; }
        }
        if (threadIdx.x == 0) put_header(wp, t, SlotHeader{rec.seq, rec.count, rec.first});
    }
    tc.rearm(wp.n_units);
    if (wp.sum != nullptr) warp_add(acc, wp.sum);
}

// ================================================================================================
// dispatch: parzen -- a CTA per task: every thread tests samples j, j+256, ... against the window
// (samples are read from the broadcast block, L2-resident after the first task), block-reduce the
// count, thread 0 emits (h, (k/n)/h**power).  Algorithmic bytes per task: n*dims*sizeof(T) read
// (from L2), 16 written.
// ================================================================================================
template <typename T>
__global__ void __launch_bounds__(kThreads) dispatch_parzen_kernel(const WaveParams wp) {
    __shared__ uint32_t s_ticket;
    __shared__ uint32_t s_warp[kThreads / 32];
    TicketClaimer tc{wp.ticket, 0u};
    tc.prime();
    const ParzenShared sh = *reinterpret_cast<const ParzenShared*>(wp.shared);
    const T* samples = reinterpret_cast<const T*>(wp.shared + sizeof(ParzenShared));
    for (;;) {
        const uint32_t t = tc.claim(&s_ticket);
        if (t >= wp.n_units) break;
        const TaskRecord rec = wave_record(wp, t);
        double* dst = reinterpret_cast<double*>(wp.ring + (size_t)t * wp.slot_stride);
        for (uint32_t i = 0; i < rec.count; ++i) {
            const double h = *reinterpret_cast<const double*>(wp.args + rec.arg_off + (size_t)i * wp.arg_stride);
            const T hT = (T)h;
            uint32_t k = 0;
            if (sh.dims == 2) {
                // 4 independent sample loads in flight per thread (the block is L2-resident: ~40 dependent
                // L2 round trips per task otherwise), then the divides
                constexpr int U = 4;
                using V2 = typename std::conditional<sizeof(T) == 4, float2, double2>::type;
                const V2* s2 = reinterpret_cast<const V2*>(samples);
                uint32_t j = threadIdx.x;
                for (; j + (U - 1) * kThreads < sh.n_samples; j += U * kThreads) {
                    V2 v[U];
#pragma unroll
                    for (int u = 0; u < U; ++u) v[u] = s2[j + u * kThreads];
#pragma unroll
                    for (int u = 0; u < U; ++u) {
                        const T row[2] = {v[u].x, v[u].y};
                        k += parzen_inside<T>(row, sh, hT) ? 1u : 0u;
                    }
                }
                for (; j < sh.n_samples; j += kThreads) {
                    const V2 v = s2[j];
                    const T row[2] = {v.x, v.y};
                    k += parzen_inside<T>(row, sh, hT) ? 1u : 0u;
                }
            } else {
                for (uint32_t j = threadIdx.x; j < sh.n_samples; j += kThreads)
                    k += parzen_inside<T>(samples + (size_t)j * sh.dims, sh, hT) ? 1u : 0u;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) k += __shfl_xor_sync(0xffffffffu, k, o);
            if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = k;
            __syncthreads();
            if (threadIdx.x == 0) {
                uint32_t kn = 0;
                for (int w = 0; w < kThreads / 32; ++w) kn += s_warp[w];
                // (k_n / len(x_samples)) / (h ** point_x.shape[1]), float64 like the reference
                double hp = 1.0;
                for (uint32_t e = 0; e < sh.power; ++e) hp = __dmul_rn(hp, h);
                dst[2 * i] = h;
                dst[2 * i + 1] = __ddiv_rn(__ddiv_rn((double)kn, (double)sh.n_samples), hp);
            }
            __syncthreads();
        }
        if (threadIdx.x == 0) put_header(wp, t, SlotHeader{rec.seq, rec.count, rec.first});
    }
    tc.rearm(wp.n_units);
}

// ================================================================================================
// gather_ordered: result ring -> ordered output by index placement (fiber/pool.py:672).  The ring
// holds one slot per claim unit in task-record (arrival) order; each slot's header says which
// tasks it carries.  Three kernels, picked per wave by the host:
//
//   gather_bulk_kernel     TMA path (cp.async.bulk, UBLKCP in SASS) for slots of whole 16 KB chunks
//                          whose units are all valid: one elected thread per CTA pipelines
//                          ring --bulk load--> shared stage --bulk store--> output; no payload byte
//                          touches a register.  ONE CTA of one warp per SM keeps enough bulk
//                          copies in flight for big slots.
//   gather_rows_kernel     slots made of whole 4 KB rows, any unit state (lost units skipped and
//                          listed for re-dispatch, partial tail vector copied byte-wise).
//   gather_ordered_kernel  flat per-vector kernel for small or unaligned slots.
//
// The sum(results) fold lives in the dispatch kernels (where the values are in registers).
// Algorithmic bytes per task: R read + R written.
// ================================================================================================
struct LostUnit { uint64_t first; uint32_t count; uint32_t pad; };

struct GatherParams {
    const SlotHeader* headers;
    const uint8_t* ring;
    uint32_t n_units;
    uint32_t slot_stride;     // bytes, multiple of 16
    uint32_t result_bytes;    // R
    uint32_t pad;
    uint8_t* out;             // ordered output window
    uint64_t win_first;       // map index of out[0]
    uint32_t* ticket_to_reset;  // dispatch ticket of this wave, zeroed for its next use
    uint32_t* lost_count;     // device: number of lost units appended so far (nullable)
    LostUnit* lost_units;     // device: (first, count) of every lost unit, for re-dispatch
    uint32_t lost_capacity;
};

__device__ __forceinline__ SlotHeader ld_header(const SlotHeader* p) {
    const uint4 r = __ldg(reinterpret_cast<const uint4*>(p));
    SlotHeader h;
    h.seq = r.x; h.count = r.y; h.first = ((uint64_t)r.w << 32) | (uint64_t)r.z;
    return h;
}

__device__ __forceinline__ void copy_tail_bytes(uint8_t* dst, const uint4& data, uint32_t nb) {
    const uint32_t w[4] = {data.x, data.y, data.z, data.w};
    for (uint32_t b = 0; b < nb; ++b) dst[b] = (uint8_t)(w[b >> 2] >> ((b & 3) * 8));
}

// housekeeping shared by the gather kernels: re-arm the wave's dispatch ticket, list lost units
__device__ __forceinline__ void gather_epilogue(const GatherParams& gp, uint32_t tid, uint32_t nthreads) {
    if (tid == 0 && gp.ticket_to_reset) *gp.ticket_to_reset = 0u;
    if (gp.lost_count != nullptr) {
        for (uint32_t s = tid; s < gp.n_units; s += nthreads) {
            const SlotHeader h = gp.headers[s];
            if (h.count & kUnitLost) {
                const uint32_t k = atomicAdd(gp.lost_count, 1u);
                if (k < gp.lost_capacity) gp.lost_units[k] = LostUnit{h.first, h.count & ~kUnitLost, 0u};
            }
        }
    }
}

// ---- flat: one 16 B vector per thread-iteration ------------------------------------------------
__global__ void __launch_bounds__(kThreads) gather_ordered_kernel(const GatherParams gp) {
    // slot_stride == vps * 16, so ring vector v lives at ring + 16*v: the slot number is only
    // needed to find the header (destination), never for the source address.
    const uint32_t vps = gp.slot_stride >> 4;                   // vectors per slot
    const uint32_t total = gp.n_units * vps;                    // host guarantees < 2^32
    const int sh = (vps & (vps - 1)) == 0 ? (31 - __clz(vps)) : -1;
    constexpr int U = 4;
    constexpr uint32_t kTile = kThreads * U;                    // 16 KB of ring per CTA iteration

    // Resolve the destination while the data load is still in flight: per vector we keep only the
    // destination pointer and the number of valid bytes (0 = skip: lost unit / beyond the tail).
    auto resolve = [&](uint32_t v, uint8_t*& dst) -> uint32_t {
        const uint32_t slot = sh >= 0 ? (v >> sh) : (v / vps);
        const uint32_t within = v - slot * vps;
        const SlotHeader h = ld_header(gp.headers + slot);
        const uint64_t valid = (uint64_t)(h.count & ~kUnitLost) * gp.result_bytes;
        const uint64_t off = (uint64_t)within << 4;
        dst = gp.out + (h.first - gp.win_first) * gp.result_bytes + off;
        if ((h.count & kUnitLost) || off >= valid) return 0u;
        const uint32_t nb = (valid - off) < 16 ? (uint32_t)(valid - off) : 16u;
        // an unaligned destination takes the byte path as well (flagged in bit 8)
        return nb | (((reinterpret_cast<uintptr_t>(dst) & 15) != 0) ? 0x100u : 0u);
    };

    for (uint32_t base = blockIdx.x * kTile; base < total; base += gridDim.x * kTile) {
        uint4 data[U];
        uint8_t* dst[U];
        uint32_t nbf[U];
        const uint32_t v0 = base + threadIdx.x;
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const uint32_t v = v0 + u * kThreads;
            nbf[u] = 0u;
            if (v < total) {
                data[u] = ld_stream(gp.ring + ((size_t)v << 4));
                nbf[u] = resolve(v, dst[u]);
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (nbf[u] == 16u) st_vec(dst[u], data[u]);
            else if (nbf[u] != 0u) copy_tail_bytes(dst[u], data[u], nbf[u] & 0xffu);
        }
    }
    gather_epilogue(gp, blockIdx.x * kThreads + threadIdx.x, gridDim.x * kThreads);
}

// ---- rows: a CTA claims ~128 KB of ring by ticket and streams it as 4 KB rows ---------------------
// Thread j owns the j-th 16 B column of every row, 4 rows in flight.
__global__ void __launch_bounds__(kThreads) gather_rows_kernel(const GatherParams gp, uint32_t* ticket, uint32_t group_slots) {
    __shared__ uint32_t s_ticket;
    TicketClaimer tc{ticket, 0u};
    tc.prime();
    constexpr int U = 4;
    const uint32_t rps = gp.slot_stride >> 12;                          // 4 KB rows per slot
    const int sh = (rps & (rps - 1)) == 0 ? (31 - __clz(rps)) : -1;
    const uint32_t n_groups = (gp.n_units + group_slots - 1) / group_slots;

    auto place = [&](const uint4& data, uint32_t slot, uint32_t row_in_slot) {
        const SlotHeader h = ld_header(gp.headers + slot);
        const uint64_t valid = (uint64_t)(h.count & ~kUnitLost) * gp.result_bytes;
        const uint64_t off = ((uint64_t)row_in_slot << 12) + threadIdx.x * 16;
        if ((h.count & kUnitLost) || off >= valid) return;
        uint8_t* dst = gp.out + (h.first - gp.win_first) * gp.result_bytes + off;
        if (off + 16 <= valid) st_vec(dst, data);
        else copy_tail_bytes(dst, data, (uint32_t)(valid - off));
    };

    for (;;) {
        const uint32_t gt = tc.claim(&s_ticket);
        if (gt >= n_groups) break;
        // newest slots first: the dispatch kernel filled the ring in ticket order just before this
        // launch, so its tail is still in the L2 (50 MB on the H100) while its head has been written back
        const uint32_t g = n_groups - 1 - gt;
        const uint32_t slot0 = g * group_slots;
        const uint32_t nslots = min(group_slots, gp.n_units - slot0);
        const uint32_t nrows = nslots * rps;
        const uint8_t* src = gp.ring + (size_t)slot0 * gp.slot_stride + threadIdx.x * 16;
        uint32_t r = 0;
        for (; r + U <= nrows; r += U) {
            uint4 v[U];
#pragma unroll
            for (int u = 0; u < U; ++u) v[u] = ld_stream(src + ((size_t)(r + u) << 12));
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const uint32_t row = r + u;
                const uint32_t s = sh >= 0 ? (row >> sh) : (row / rps);
                place(v[u], slot0 + s, row - s * rps);
            }
        }
        for (; r < nrows; ++r) {
            const uint4 v = ld_stream(src + ((size_t)r << 12));
            const uint32_t s = sh >= 0 ? (r >> sh) : (r / rps);
            place(v, slot0 + s, r - s * rps);
        }
    }
    gather_epilogue(gp, blockIdx.x * kThreads + threadIdx.x, gridDim.x * kThreads);
}

// ---- bulk: TMA pipeline -------------------------------------------------------------------------------
namespace bulk {
constexpr uint32_t kChunk = 16384;     // bytes per bulk copy and per shared stage
constexpr int kStages = 6;             // 96 KB of shared memory per CTA
constexpr int kLag = 4;                // loads run this many chunks ahead of their store
constexpr uint32_t kGroup = 32;        // slots per ticket: their headers are prefetched by the 32 lanes

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bulk_store(void* gdst, const void* smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
}  // namespace bulk

// Requirements checked by the host: slot_stride a multiple of kChunk, R % 16 == 0 or every unit full,
// output window 16 B aligned, no lost units.
__global__ void __launch_bounds__(32) gather_bulk_kernel(const GatherParams gp, uint32_t* ticket, uint32_t group_slots /* <= kGroup */) {
    using namespace bulk;
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint64_t full[kStages];
    __shared__ SlotHeader s_hdr[kGroup];
    __shared__ uint32_t s_group;
    const uint32_t lane = threadIdx.x;
    if (lane == 0) {
        for (int s = 0; s < kStages; ++s) mbar_init(&full[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();

    const uint32_t n_groups = (gp.n_units + group_slots - 1) / group_slots;
    uint32_t it = 0, st = 0;                             // chunks loaded / stored so far (lane 0)
    uint8_t* pend_dst[kStages] = {};
    uint32_t pend_bytes[kStages] = {};

    auto store_one = [&]() {
        const int sg = st % kStages;
        mbar_wait(&full[sg], (st / kStages) & 1);
        bulk_store(pend_dst[sg], smem + (size_t)sg * kChunk, pend_bytes[sg]);
        ++st;
    };

    for (;;) {
        if (lane == 0) s_group = atomicAdd(ticket, 1u);
        __syncwarp();
        const uint32_t g = s_group;
        if (g >= n_groups) break;
        const uint32_t slot0 = g * group_slots;
        const uint32_t nslots = min(group_slots, gp.n_units - slot0);
        if (lane < nslots) s_hdr[lane] = ld_header(gp.headers + slot0 + lane);   // one coalesced 512 B read
        __syncwarp();
        if (lane == 0) {
            for (uint32_t s = 0; s < nslots; ++s) {
                const SlotHeader h = s_hdr[s];
                const uint32_t valid = (h.count & ~kUnitLost) * gp.result_bytes;   // < 4 GiB by construction
                const uint8_t* src = gp.ring + (size_t)(slot0 + s) * gp.slot_stride;
                uint8_t* dst = gp.out + (h.first - gp.win_first) * gp.result_bytes;
                // a tail unit whose byte count is not a multiple of 16: the last <16 bytes go by hand
                const uint32_t valid16 = valid & ~15u;
                for (uint32_t b = valid16; b < valid; ++b) dst[b] = src[b];
                for (uint32_t off = 0; off < valid16; off += kChunk) {
                    const uint32_t bytes = min(kChunk, valid16 - off);
                    const int sg = it % kStages;
                    // the stage was last used by chunk it-kStages, whose store was issued at least
                    // kStages-kLag-1 groups ago: wait until it has finished reading shared memory
                    if (it >= (uint32_t)kStages) bulk_wait_read<kStages - kLag - 1>();
                    pend_dst[sg] = dst + off;
                    pend_bytes[sg] = bytes;
                    mbar_expect_tx(&full[sg], bytes);
                    bulk_load(smem + (size_t)sg * kChunk, src + off, bytes, &full[sg]);
                    ++it;
                    while (it - st > (uint32_t)kLag) store_one();
                }
            }
        }
        __syncwarp();
    }
    if (lane == 0) {
        while (st < it) store_one();
        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
    gather_epilogue(gp, blockIdx.x * 32 + lane, gridDim.x * 32);
}

// ================================================================================================
// dispatch: payload_map_4k, TMA-staged (warp-specialised).  Same contract as
// dispatch_payload_map_kernel, for contiguous argument records (arg_stride == 4096):
//   warp 0 (one elected lane)  claims units by ticket, writes their slot headers, and bulk-loads the
//                              records in 16 KB chunks into shared-memory IN stages (mbarrier
//                              complete_tx); it waits on the stage's EMPTY barrier before reuse;
//   warps 1-4 (128 threads)    wait for a FULL stage, read it (LDS.128), apply out = in*K + t and
//                              write an OUT stage (STS.128); after a proxy fence + named barrier one
//                              of them bulk-stores the OUT stage into the result ring.
// Payload bytes cross registers only between two shared-memory stages; global traffic is TMA only.
// ================================================================================================
namespace tma_map {
constexpr uint32_t kMapChunk = 16384;
constexpr int kConsumers = 128;
struct ChunkDesc { uint8_t* dst; uint32_t bytes; uint32_t tbase; };
// 3 IN and 2 OUT stages at 2 CTAs per SM: 96 KB of loads in flight per SM from local HBM
constexpr int kInStages = 3, kOutStages = 2;
constexpr size_t kSmemBytes = (size_t)(kInStages + kOutStages) * kMapChunk;   // 80 KB
}  // namespace tma_map

__global__ void __launch_bounds__(160) dispatch_payload_map_tma_kernel(const WaveParams wp) {
    using namespace bulk;
    using namespace tma_map;
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint64_t full[kInStages], empty[kInStages];
    __shared__ ChunkDesc desc[kInStages];
    uint8_t* in_stage = smem;
    uint8_t* out_stage = smem + (size_t)kInStages * kMapChunk;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < kInStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kConsumers); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 0) {
        if (lane != 0) return;
        // ---------------- producer ----------------
        uint32_t seq = 0;
        auto acquire_stage = [&]() -> int {
            const int sg = seq % kInStages;
            mbar_wait(&empty[sg], ((seq / kInStages) & 1) ^ 1);   // fresh barrier: passes immediately
            return sg;
        };
        for (;;) {
            const uint32_t t = atomicAdd(wp.ticket, 1u);
            if (t >= wp.n_units) {
                // no prefetch here: each CTA draws exactly one ticket >= n_units; the highest re-arms the counter
                if (t == wp.n_units + gridDim.x - 1u) *wp.ticket = 0u;
                break;
            }
            const TaskRecord rec = wave_record(wp, t);
            put_header(wp, t, SlotHeader{rec.seq, rec.count, rec.first});
            const uint8_t* src = wp.args + rec.arg_off;
            uint8_t* dst = wp.ring + (size_t)t * wp.slot_stride;
            const uint32_t total = rec.count * kPayloadBytes;
            const uint32_t tbase = (uint32_t)(wp.index_base + rec.first);
            for (uint32_t off = 0; off < total; off += kMapChunk) {
                const uint32_t bytes = min(kMapChunk, total - off);
                const int sg = acquire_stage();
                desc[sg] = ChunkDesc{dst + off, bytes, tbase + off / kPayloadBytes};
                mbar_expect_tx(&full[sg], bytes);
                bulk_load(in_stage + (size_t)sg * kMapChunk, src + off, bytes, &full[sg]);
                ++seq;
            }
        }
        const int sg = acquire_stage();                 // end marker
        desc[sg] = ChunkDesc{nullptr, 0u, 0u};
        asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&full[sg])) : "memory");
        return;
    }

    // ---------------- consumers (threads 32..159) ----------------
    const uint32_t ct = threadIdx.x - 32;               // 0..127
    for (uint32_t seq = 0;; ++seq) {
        const int sg = seq % kInStages, og = seq % kOutStages;
        mbar_wait(&full[sg], (seq / kInStages) & 1);
        const ChunkDesc d = desc[sg];
        if (d.bytes == 0) break;
        // the bulk store that last read OUT stage `og` (chunk seq-kOutStages) must be done with it
        if (ct == 0 && seq >= (uint32_t)kOutStages) bulk_wait_read<kOutStages - 1>();
        asm volatile("bar.sync 1, 128;" ::: "memory");
        const uint8_t* in = in_stage + (size_t)sg * kMapChunk;
        uint8_t* out = out_stage + (size_t)og * kMapChunk;
        const uint32_t nvec = d.bytes >> 4;
#pragma unroll
        for (uint32_t k = 0; k < kMapChunk / 16 / kConsumers; ++k) {
            const uint32_t v = ct + k * kConsumers;
            if (v < nvec) {
                uint4 x = *reinterpret_cast<const uint4*>(in + ((size_t)v << 4));
                const uint32_t tt = d.tbase + (v >> 8);   // 256 vectors per 4 KB record
                x.x = x.x * kPayloadMul + tt; x.y = x.y * kPayloadMul + tt;
                x.z = x.z * kPayloadMul + tt; x.w = x.w * kPayloadMul + tt;
                *reinterpret_cast<uint4*>(out + ((size_t)v << 4)) = x;
            }
        }
        // IN stage consumed; make the generic-proxy writes to the OUT stage visible to the async proxy
        asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&empty[sg])) : "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        asm volatile("bar.sync 1, 128;" ::: "memory");
        if (ct == 0) bulk_store(d.dst, out, d.bytes);
    }
    if (ct == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// ================================================================================================
// dispatch: record bodies (FBR_BODY_RECORD) -- any trivially copyable Arg / Res of 4..4096 bytes (multiples
// of 4; up to 32768 for group bodies), staged through shared memory (warp-specialised, like
// dispatch_payload_map_tma_kernel):
//   warp 0 (one elected lane)  waits for an EMPTY IN stage, claims a unit by ticket and bulk-loads the unit's
//                              count * A argument bytes into it (cp.async.bulk + FULL mbarrier complete_tx);
//                              with two IN stages the next unit's load overlaps this unit's compute;
//   warps 1-8 (256 consumers)  copy whatever the bulk load could not take (see below), run B::run one task per
//                              thread from the IN stage into an OUT stage, then -- after a proxy fence and a
//                              named barrier -- one of them bulk-stores the unit's count * R result bytes to
//                              wp.ring + t * slot_stride (the ring slot, or the final index: direct placement).
// Fallbacks, chosen at run time per unit: argument bytes that are not contiguous (arg_stride != A), not 16 B
// aligned in global memory, or past the last multiple of 16 are copied by the consumers (16 B vectors where
// both sides allow it, else 4 B words); the same holds for the result bytes of an unaligned destination or a
// tail that is not a multiple of 16.  The body sees its argument and result as references into shared memory,
// so a 1 KB record is never copied into registers.  Known costs (DESIGN.md section 4): records are packed, so lane
// i's record starts at i * A -- a body that walks a large record word by word has every lane on the same bank
// (A = 1024: 32-way); reading it in 16 B vectors cuts that to 8-way.  A stage holds kStageBytes of the larger
// record, so for large records most consumers are idle during B::run (A = 1024: 32 tasks per unit).
// Group bodies (kGroup = G) answer both: G lanes run each task (run_unit), reading consecutive words of one
// record, and their records may fill a whole stage (32 KB, one task per unit).
// Bodies with a Shared element type also receive the map's broadcast block: one within the body's kSharedStage is
// bulk-loaded once per CTA into a region after the stages (DESIGN.md section 4 has the staged vs global measurement).
// ================================================================================================
// The map's broadcast block as a record body with a Shared element type sees it: n = shared_bytes / sizeof(T) elements,
// read-only, in shared memory when the block fits the body's kSharedStage, else in global memory.
template <class T>
struct Broadcast {
    const T* data;
    uint64_t n;
};

// What a group record body (kGroup = G) knows of the G threads that run each task together: G consecutive lanes of one
// warp.  `mask` names them for __shfl_*_sync; sync() is __syncwarp over them.
template <uint32_t G>
struct Group {
    uint32_t rank;                       // 0 .. G-1
    static constexpr uint32_t size = G;
    uint32_t mask;
    __device__ __forceinline__ void sync() const { __syncwarp(mask); }
};

// The variable-length items of one task of an items record body (`using Item = ...`): n elements, read-only, in global
// memory (through L1 / L2; DESIGN.md section 4 has the staged vs global measurement that chose this).
template <class T>
struct Items {
    const T* data;
    uint64_t n;
};

// The element types of a multi-stream items record body, one per stream: `using Items = fbr::ItemTypes<uint8_t, float>;`
template <class... T>
struct ItemTypes {};

// The Arg of an items record body without a fixed head record: run() then takes no argument record.
struct NoArg {};

// The Res of an emit record body (`using Out = ...`): its task returns a variable-length array instead of a record.
struct NoRes {};

// The result of one task of an emit body: run() appends values of type T.  The body runs twice per task: in the count pass
// data is nullptr and only n counts; in the emit pass data points at the task's place in the map's values and cap is the
// count the first pass gave (values past it are never written).  A one-thread body calls push(v); a group body (G > 1) calls
// the collective push_if(g, pred, v) on every lane of the group: lanes whose pred holds append their v in rank order, and
// every lane keeps the same n.
template <class T, uint32_t G = 1>
struct Emit {
    T* data;
    uint64_t cap;
    uint64_t n;
    __device__ __forceinline__ void push(const T& v) {
        static_assert(G == 1, "a group emitter has only the collective push_if(g, pred, v)");
        if (data != nullptr && n < cap) data[n] = v;
        ++n;
    }
    __device__ __forceinline__ void push_if(const Group<G>& g, bool pred, const T& v) {
        static_assert(G > 1, "push_if is the collective of a group emitter; a one-thread body calls push(v)");
        const uint32_t lanes = __ballot_sync(g.mask, pred) & g.mask;
        if (pred) {
            const uint64_t k = n + __popc(lanes & ((1u << (threadIdx.x & 31u)) - 1u));
            if (data != nullptr && k < cap) data[k] = v;
        }
        n += __popc(lanes);
    }
};

namespace record {
constexpr int kConsumers = 256;
constexpr int kThreads = 32 + kConsumers;
constexpr int kInStages = 2, kOutStages = 2;
constexpr uint32_t kStageBytes = 32768;   // per stage, for the larger of A and R
constexpr uint32_t kMaxUnit = 1024;       // tasks per unit: 4 per consumer thread
constexpr uint32_t kThreadRecordBytes = 4096;   // the largest record of a one-thread body (group bodies: kStageBytes)
constexpr uint64_t kSmemBudget = 200u << 10;    // dynamic shared memory: the stages plus the broadcast region

// tasks per unit that make count * A and count * R multiples of 16 (A and R are multiples of 4)
constexpr uint32_t align_tasks(uint32_t A, uint32_t R) {
    return (A % 16 == 0 && R % 16 == 0) ? 1u : (A % 8 == 0 && R % 8 == 0) ? 2u : 4u;
}
// dynamic shared memory of dispatch_record_kernel: the IN and OUT stages of `unit` tasks, then the broadcast region
// (A = 0: range() maps and NoArg bodies read no argument bytes)
constexpr uint64_t smem_bytes(uint32_t unit, uint32_t A, uint32_t R, uint32_t stage) {
    return (uint64_t)kInStages * unit * A + (uint64_t)kOutStages * unit * R + stage;
}
constexpr bool item_elem_ok(uint32_t e) { return e == 1 || e == 2 || (e % 4 == 0 && e >= 4 && e <= 4096); }
constexpr bool shared_elem_ok(uint32_t e) { return e != 0 && e % 4 == 0 && e <= 4096; }

// A record body opts into the broadcast block with `using Shared = <element>;` and `static constexpr uint32_t
// kSharedStage = <bytes>;`; its run() then takes a const Broadcast<Shared>& after the result.
template <class B, class = void>
struct BroadcastOf {
    static constexpr bool kOn = false;
    static constexpr uint32_t kElem = 0, kStage = 0;
};
template <class B>
struct BroadcastOf<B, std::void_t<typename B::Shared>> {
    using T = typename B::Shared;
    static constexpr bool kOn = true;
    static constexpr uint32_t kElem = (uint32_t)sizeof(T), kStage = B::kSharedStage;
    static_assert(std::is_trivially_copyable<T>::value, "broadcast bodies: Shared is trivially copyable");
    static_assert(shared_elem_ok(kElem), "broadcast bodies: sizeof(Shared) is a multiple of 4 up to 4096");
    static_assert(kStage % 16 == 0, "broadcast bodies: kSharedStage is a multiple of 16 (0: never stage)");
};

// A record body opts into groups with `static constexpr uint32_t kGroup = G;` (G = 2, 4, 8, 16 or 32): G threads run
// each task, and its run() takes a const Group<G>& after the result (after the broadcast block, if it has one).
template <class B, class = void>
struct GroupOf {
    static constexpr uint32_t kG = 1;
};
template <class B>
struct GroupOf<B, std::void_t<decltype(B::kGroup)>> {
    static constexpr uint32_t kG = B::kGroup;
    static_assert(kG == 2 || kG == 4 || kG == 8 || kG == 16 || kG == 32, "group record bodies: kGroup is 2, 4, 8, 16 or 32");
};

// A record body opts into variable-length items with `using Item = <element>;` (one stream) or `using Items =
// fbr::ItemTypes<T0, T1[, T2[, T3]]>;` (2 to 4 streams, each with its own element type and offsets): run() then takes a
// const Items<Tk>& per stream, in stream order, after the argument record (or first, when Arg is NoArg).  ItemsOf<B> is
// the one place the streams' element types and sizes are defined.
template <uint32_t k, class... T>
struct TypeAt;
template <uint32_t k, class T0, class... T>
struct TypeAt<k, T0, T...> {
    using type = typename TypeAt<k - 1, T...>::type;
};
template <class T0, class... T>
struct TypeAt<0, T0, T...> {
    using type = T0;
};
template <class B, class = void>
struct ItemDecl {                       // using Item = T: ItemTypes<T>
    static constexpr bool kOn = false;
    using type = ItemTypes<>;
};
template <class B>
struct ItemDecl<B, std::void_t<typename B::Item>> {
    static constexpr bool kOn = true;
    using type = ItemTypes<typename B::Item>;
};
template <class B, class = void>
struct ItemsDecl {                      // using Items = ItemTypes<...>
    static constexpr bool kOn = false;
    using type = ItemTypes<>;
};
template <class B>
struct ItemsDecl<B, std::void_t<typename B::Items>> {
    static constexpr bool kOn = true;
    using type = typename B::Items;
};
template <class L>
struct ItemList;
template <class... T>
struct ItemList<ItemTypes<T...>> {
    static constexpr uint32_t kStreams = (uint32_t)sizeof...(T);
    template <uint32_t k>
    using At = typename TypeAt<k, T...>::type;
    // element size of stream k < kMaxItemStreams (0 past the last stream)
    static constexpr uint32_t elem(uint32_t k) {
        constexpr uint32_t e[kMaxItemStreams + 1] = {(uint32_t)sizeof(T)...};
        return e[k];
    }
    static_assert((true && ... && std::is_trivially_copyable<T>::value), "items bodies: Item is trivially copyable");
    static_assert((true && ... && item_elem_ok((uint32_t)sizeof(T))), "items bodies: sizeof(Item) is 1, 2 or a multiple of 4 up to 4096");
};
template <class B>
struct ItemsOf : ItemList<typename std::conditional<ItemsDecl<B>::kOn, typename ItemsDecl<B>::type, typename ItemDecl<B>::type>::type> {
    using List = ItemList<typename std::conditional<ItemsDecl<B>::kOn, typename ItemsDecl<B>::type, typename ItemDecl<B>::type>::type>;
    static constexpr bool kOn = List::kStreams > 0;
    static constexpr uint32_t kElem = List::elem(0);   // stream 0
    static_assert(!(ItemDecl<B>::kOn && ItemsDecl<B>::kOn),
                  "items bodies declare `using Item = T;` (one stream) or `using Items = fbr::ItemTypes<...>;` (2 to 4), not both");
    static_assert(!ItemsDecl<B>::kOn || (List::kStreams >= 2 && List::kStreams <= kMaxItemStreams),
                  "items bodies: fbr::ItemTypes<...> lists 2 to 4 element types (one stream: `using Item = T;`)");
    static_assert(!kOn || !B::kIndexArg, "items bodies cannot take range() indices (kIndexArg)");
};

// A record body opts into variable-length results with `using Out = <element>;` and `using Res = NoRes;`: run() then takes
// an Emit<Out, G>& where other record bodies take Res&.  Its kernels are instantiated for EmitPass<B, false> (the count
// pass) and EmitPass<B, true> (the emit pass); in both, a task's fixed result record is one uint64 (its count, or its end
// offset), so the two passes share one claim plan.
template <class B, class = void>
struct EmitOf {
    static constexpr bool kOn = false;
    static constexpr uint32_t kElem = 0;
};
template <class B>
struct EmitOf<B, std::void_t<typename B::Out>> {
    using T = typename B::Out;
    static constexpr bool kOn = true;
    static constexpr uint32_t kElem = (uint32_t)sizeof(T);
    static_assert(std::is_trivially_copyable<T>::value, "emit bodies: Out is trivially copyable");
    static_assert(item_elem_ok(kElem), "emit bodies: sizeof(Out) is 1, 2 or a multiple of 4 up to 4096");
    static_assert(std::is_same<typename B::Res, NoRes>::value, "emit bodies have no fixed result record (Res = fbr::NoRes)");
};
// an emit body's optional `static uint64_t count(...)`: run()'s parameters without the emitter, es and attempt
template <class B, class = void>
struct HasCount : std::false_type {};
template <class B>
struct HasCount<B, std::void_t<decltype(&B::count)>> : std::true_type {};

template <class B, bool kValues>
struct EmitPass : B {
    static constexpr bool kEmitValues = kValues;
};
template <class B, class = void>
struct EmitModeOf {
    static constexpr bool kValues = false;
};
template <class B>
struct EmitModeOf<B, std::void_t<decltype(B::kEmitValues)>> {
    static constexpr bool kValues = B::kEmitValues;
};
// A record body opts into fold maps with `__host__ __device__ static Res identity();` and `__device__ static void
// combine(Res& acc, const Res& x);` (acc <- acc (+) x, called by one thread; either operand may be in shared or global
// memory).  A fold map reduces its results with
//     tree(x[0..c)): while c > 1: x[i] <- combine(x[2i], x[2i+1]) for every i with 2i+1 < c, an odd last element is
//                    carried to x[c/2]; c <- ceil(c/2)
// over each block's results in task order, then over the blocks' totals in block order; n = 0 gives identity().  Claim
// units of a fold map hold a power of two of tasks and start at a multiple of it within their block, so a unit's tree is
// an aligned subtree of its block's.  Its kernels are instantiated for FoldPass<B>.
template <class B, class = void>
struct FoldOf {
    static constexpr bool kOn = false;
};
template <class B>
struct FoldOf<B, std::void_t<decltype(&B::combine)>> {
    using Res = typename B::Res;
    static constexpr bool kOn = true;
    static_assert(std::is_same<decltype(&B::combine), void (*)(Res&, const Res&)>::value,
                  "fold bodies: combine is `static void combine(Res& acc, const Res& x)`");
    static_assert(std::is_same<decltype(B::identity()), Res>::value,
                  "fold bodies: `__host__ __device__ static Res identity()` is defined next to combine");
    static_assert(!EmitOf<B>::kOn, "emit bodies cannot fold (combine)");
    static_assert(std::is_default_constructible<Res>::value, "fold bodies: Res is default-constructible (the fold pass holds "
                  "results in registers)");
};
// a keyed fold body: a fold body that also defines `static uint32_t key(const Res&)` (FBR_BODY_KEYED)
template <class B, class = void>
struct KeyOf {
    static constexpr bool kOn = false;
};
template <class B>
struct KeyOf<B, std::void_t<decltype(&B::key)>> {
    static constexpr bool kOn = true;
    static_assert(FoldOf<B>::kOn, "keyed bodies: key() needs identity() and combine() (a keyed fold is a fold per key)");
    static_assert(std::is_same<decltype(&B::key), uint32_t (*)(const typename B::Res&)>::value,
                  "keyed bodies: key is `__device__ static uint32_t key(const Res& r)`");
};
template <class B>
struct FoldPass : B {
    static constexpr bool kFoldPass = true;
};
template <class B, class = void>
struct FoldModeOf {
    static constexpr bool kOn = false;
    static constexpr int kCtas = 0;
};
template <class B>
struct FoldModeOf<B, std::void_t<decltype(B::kFoldPass)>> {
    static constexpr bool kOn = B::kFoldPass;
    static constexpr int kCtas = sizeof(typename B::Res) > 16 ? 3 : 4;   // resident CTAs the fold pass asks ptxas for
};
// records per tile of fold_tree_kernel
constexpr uint32_t kFoldTile = 512;

// the fixed result record of one task: Res, or the uint64 count / end offset of an emit body
template <class B>
using ResultRecord = typename std::conditional<EmitOf<B>::kOn, uint64_t, typename B::Res>::type;

template <class B>
struct Layout {
    static constexpr bool kNoArg = std::is_same<typename B::Arg, NoArg>::value;
    static constexpr uint32_t A = kNoArg ? 0u : (uint32_t)sizeof(typename B::Arg), R = (uint32_t)sizeof(ResultRecord<B>);
    static_assert(!kNoArg || ItemsOf<B>::kOn, "record bodies: only an items body may have no argument record (NoArg)");
    static_assert(GroupOf<B>::kG > 1 || (A % 4 == 0 && R % 4 == 0 && (A >= 4 || kNoArg) && R >= 4 && A <= kThreadRecordBytes && R <= kThreadRecordBytes),
                  "record bodies: sizeof(Arg) and sizeof(Res) are multiples of 4 between 4 and 4096");
    static_assert(GroupOf<B>::kG == 1 || (A % 4 == 0 && R % 4 == 0 && (A >= 4 || kNoArg) && R >= 4 && A <= kStageBytes && R <= kStageBytes),
                  "group record bodies: sizeof(Arg) and sizeof(Res) are multiples of 4 between 4 and 32768");
    // the broadcast region after the IN / OUT stages (0 bytes for bodies without a Shared type)
    static constexpr uint32_t kShared = BroadcastOf<B>::kStage;
    static constexpr uint32_t kAlign = align_tasks(A, R);
    static_assert(GroupOf<B>::kG == 1 || kAlign * (A > R ? A : R) <= kStageBytes,
                  "group record bodies: one 16 B-aligned group of tasks fits a stage (kAlign * max(sizeof(Arg), sizeof(Res)) <= 32768)");
    static constexpr uint32_t unit() {
        const uint32_t w = A > R ? A : R;
        uint32_t u = kMaxUnit;
        while (u > kAlign && u * w > kStageBytes) u >>= 1;
        return u;
    }
    static constexpr uint32_t kUnit = unit();
    static constexpr uint32_t kInBytes = kUnit * A, kOutBytes = kUnit * R;   // multiples of 16
    // dynamic shared memory of an instantiation: range() maps (index) read no argument bytes and have no IN stages
    static constexpr size_t smem(bool index) { return smem_bytes(kUnit, index ? 0u : A, R, kShared); }
    static_assert(kInBytes % 16 == 0 && kOutBytes % 16 == 0 && smem(false) <= kSmemBudget, "record stage layout");
};

// contiguous copy by `n` threads; 16 B vectors while both sides are 16 B aligned, then 4 B words, then bytes
__device__ __forceinline__ void coop_copy(uint8_t* dst, const uint8_t* src, uint32_t bytes, uint32_t tid, uint32_t n) {
    const uintptr_t al = reinterpret_cast<uintptr_t>(dst) | reinterpret_cast<uintptr_t>(src);
    uint32_t off = 0;
    if ((al & 15) == 0) {
        const uint32_t nv = bytes >> 4;
        for (uint32_t v = tid; v < nv; v += n)
            reinterpret_cast<uint4*>(dst)[v] = reinterpret_cast<const uint4*>(src)[v];
        off = nv << 4;
    }
    if ((al & 3) == 0) {
        const uint32_t w1 = bytes >> 2;
        for (uint32_t w = (off >> 2) + tid; w < w1; w += n)
            reinterpret_cast<uint32_t*>(dst)[w] = reinterpret_cast<const uint32_t*>(src)[w];
        off = w1 << 2;
    }
    for (uint32_t b = off + tid; b < bytes; b += n) dst[b] = src[b];
}

// `count` records of A bytes, `stride` bytes apart in global memory (4 B aligned), packed into `dst`
template <uint32_t A>
__device__ __forceinline__ void gather_records(uint8_t* dst, const uint8_t* src, uint32_t stride, uint32_t count,
                                               uint32_t tid, uint32_t n) {
    constexpr uint32_t W = A / 4;
    for (uint32_t w = tid; w < count * W; w += n) {
        const uint32_t i = w / W, k = w - i * W;
        reinterpret_cast<uint32_t*>(dst)[w] = *reinterpret_cast<const uint32_t*>(src + (size_t)i * stride + 4 * k);
    }
}

// The G lanes that run consumer ct's task in a group body: ct is rank ct % G of group ct / G (consumers start at thread
// 32, so ct % 32 is the lane)
template <uint32_t G>
__device__ __forceinline__ Group<G> group_of(uint32_t ct) {
    return Group<G>{ct % G, (G == 32 ? 0xffffffffu : ((1u << G) - 1u) << ((ct & 31u) & ~(G - 1u)))};
}

// Stream k of an items map's wave: stream 0 from WaveParams::items ..., the others from more_items
template <uint32_t k>
__device__ __forceinline__ ItemStream item_stream(const WaveParams& wp) {
    if constexpr (k == 0) return ItemStream{wp.items, wp.item_offs, wp.item_base, wp.item_count};
    else return wp.more_items[k - 1];
}

// The item streams of a unit of an items body: o[k] are stream k's offsets from the unit's first task on
template <uint32_t K>
struct UnitItems {
    const uint64_t* o[K];
};
template <size_t... k>
__device__ __forceinline__ UnitItems<sizeof...(k)> unit_items(const WaveParams& wp, uint64_t first, std::index_sequence<k...>) {
    return UnitItems<sizeof...(k)>{{(item_stream<k>(wp).offs + (first - wp.item_first))...}};
}
// Task i's span [a[k], b[k]) in each stream k, read from the unit's offsets; true (a bad argument) when any stream's
// offsets decrease or leave [base, count]
template <uint32_t K>
struct TaskSpans {
    uint64_t a[K], b[K];
};
template <size_t... k>
__device__ __forceinline__ bool bad_spans(const WaveParams& wp, const UnitItems<sizeof...(k)>& u, uint32_t i, std::index_sequence<k...>,
                                           TaskSpans<sizeof...(k)>& t) {
    bool bad = false;
    ((t.a[k] = u.o[k][i], t.b[k] = u.o[k][i + 1],
      bad = bad || t.a[k] > t.b[k] || t.a[k] < item_stream<k>(wp).base || t.b[k] > item_stream<k>(wp).count), ...);
    return bad;
}
// f(the K views of task spans t, in stream order)
template <class B, class F, size_t... k>
__device__ __forceinline__ void with_items(const WaveParams& wp, const TaskSpans<sizeof...(k)>& t, std::index_sequence<k...>, F&& f) {
    using It = ItemsOf<B>;
    f(Items<typename It::template At<k>>{reinterpret_cast<const typename It::template At<k>*>(
                                             item_stream<k>(wp).items + (t.a[k] - item_stream<k>(wp).base) * sizeof(typename It::template At<k>)),
                                         t.b[k] - t.a[k]}...);
}

// One unit of a record body: group g = ct / G runs tasks g, g + C/G, ... (G = 1: one thread per task).  All G lanes of a
// group see the same i, so the group stays converged through B::run.  run() gets, in order: the head argument (a range()
// index, a record from `in`, or none for NoArg), the task's items (one view per stream), the result, the broadcast block
// `sh` (bodies that have one), the group (G > 1), then task_index, es and attempt.  An items task reads offsets o[i],
// o[i+1] of each stream and its items from global memory; one whose offsets decrease or leave [base, count] in any stream
// reports TASK_BADARG and its body is not called.
// An emit body's task that pushed another number of values than it counted lowers *emit_err (the unit's word, in shared
// memory) to its (task_index << 8 | TASK_EMIT): the kernel reports it only if the unit was not lost, since a faulting
// attempt's values are discarded.
template <class B, bool kIndex, class... Sh>
__device__ __forceinline__ void run_unit(const WaveParams& wp, const TaskRecord& rec, const uint8_t* in, uint8_t* out,
                                         uint32_t ct, const ErrSink& es, unsigned long long* emit_err, const Sh&... sh) {
    using L = Layout<B>;
    using Arg = typename B::Arg;
    using Res = ResultRecord<B>;
    constexpr uint32_t G = GroupOf<B>::kG, C = kConsumers;
    const uint64_t g0 = wp.index_base + rec.first;
    constexpr uint32_t K = ItemsOf<B>::kStreams > 0 ? ItemsOf<B>::kStreams : 1u;
    using Streams = std::make_index_sequence<K>;
    const UnitItems<K> u = unit_items(wp, rec.first, Streams{});   // items bodies: the unit's offsets in each stream
    for (uint32_t i = ct / G; i < rec.count; i += C / G) {
        auto res = [&]() -> Res& { return *reinterpret_cast<Res*>(out + (size_t)i * L::R); };
        auto call = [&](Res& r, const auto&... head) {  // head: the head argument, then the items of each stream
            if constexpr (EmitOf<B>::kOn) {
                // emit bodies: the count pass records the task's count, the emit pass its global end offset (the span the
                // count pass gave, so the offsets stay consistent); a task that pushed another number reports TASK_EMIT
                using O = typename EmitOf<B>::T;
                Emit<O, G> y{nullptr, 0, 0};
                uint64_t lo = 0;
                if constexpr (EmitModeOf<B>::kValues) {
                    const uint64_t* const e = wp.emit_offs + (rec.first + i - wp.emit_first);
                    lo = e[0];
                    y.cap = e[1] - lo;
                    y.data = reinterpret_cast<O*>(wp.emit_values) + lo;
                }
                if constexpr (!EmitModeOf<B>::kValues && HasCount<B>::value) {
                    static_assert(G == 1, "emit bodies: the count() hook is for one-thread bodies");
                    y.n = B::count(head..., sh..., g0 + i);
                } else if constexpr (G > 1) {
                    B::run(head..., y, sh..., group_of<G>(ct), g0 + i, es, rec.attempt);
                } else {
                    B::run(head..., y, sh..., g0 + i, es, rec.attempt);
                }
                if (ct % G == 0) {
                    if constexpr (EmitModeOf<B>::kValues) {
                        if (y.n != y.cap) atomicMin(emit_err, (unsigned long long)(((g0 + i) << 8) | TASK_EMIT));
                        r = wp.emit_base + lo + y.cap;
                    } else {
                        r = y.n;
                    }
                }
            } else if constexpr (G > 1) {
                B::run(head..., r, sh..., group_of<G>(ct), g0 + i, es, rec.attempt);
            } else {
                B::run(head..., r, sh..., g0 + i, es, rec.attempt);
            }
        };
        if constexpr (kIndex) {
            call(res(), (Arg)(wp.index_start + (int64_t)(rec.first + i) * wp.index_step));
        } else if constexpr (ItemsOf<B>::kOn) {
            TaskSpans<K> t;
            if (bad_spans(wp, u, i, Streams{}, t)) {
                if (ct % G == 0) es.report(TASK_BADARG, g0 + i);
                continue;
            }
            with_items<B>(wp, t, Streams{}, [&](const auto&... x) {
                if constexpr (L::kNoArg) call(res(), x...);
                else call(res(), *reinterpret_cast<const Arg*>(in + (size_t)i * L::A), x...);
            });
        } else {
            call(res(), *reinterpret_cast<const Arg*>(in + (size_t)i * L::A));
        }
    }
}
}  // namespace record

// (a fold pass asks ptxas for 4 resident CTAs, 3 when its Res is over 16 bytes: left to itself ptxas packs it into 32
// registers and spills, and a 24 B Res held in registers with its shuffled copy spills at the 56 registers of 4 CTAs)
template <class B, bool kIndex>
__global__ void __launch_bounds__(record::kThreads, record::FoldModeOf<B>::kCtas)
    dispatch_record_kernel(const WaveParams wp) {
    using namespace bulk;
    using L = record::Layout<B>;
    constexpr int kIn = record::kInStages, kOut = record::kOutStages;
    constexpr uint32_t C = record::kConsumers;
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint64_t full[kIn], empty[kIn];
    __shared__ TaskRecord s_rec[kIn];
    __shared__ uint32_t s_ticket[kIn];
    __shared__ uint32_t s_bulk[kIn];      // argument bytes of the unit the bulk load brings (the rest: consumers)
    __shared__ int s_fault[2];
    unsigned long long* s_emit_err = nullptr;   // emit bodies: per-unit count-mismatch word, by unit parity
    if constexpr (record::EmitOf<B>::kOn) {
        __shared__ unsigned long long s_emit_words[2];
        s_emit_err = s_emit_words;
    }
    uint8_t* const in_stage = smem;
    uint8_t* const out_stage = smem + (kIndex ? 0 : (size_t)kIn * L::kInBytes);   // L::smem(kIndex) bytes in all
    // broadcast bodies: the block is staged once per CTA into the region after the stages when it fits kSharedStage
    // (a run-time choice, uniform across the launch), else run() reads it from global memory
    using Bc = record::BroadcastOf<B>;
    uint64_t* bcast_full = nullptr;
    uint8_t* const bcast_stage = out_stage + (size_t)kOut * L::kOutBytes;   // after the IN and OUT stages
    bool staged = false;
    uint32_t bcast_bulk = 0;                           // bytes of the block the bulk load brings (the rest: consumers)
    if constexpr (Bc::kOn && Bc::kStage > 0) {
        __shared__ uint64_t s_bcast_full;
        bcast_full = &s_bcast_full;
        staged = wp.shared_bytes <= Bc::kStage;
        if ((reinterpret_cast<uintptr_t>(wp.shared) & 15) == 0) bcast_bulk = (uint32_t)wp.shared_bytes & ~15u;
    }
    constexpr bool kArgs = !kIndex && L::A > 0;          // NoArg items bodies have no argument records
    if (threadIdx.x == 0) {
        for (int s = 0; s < kIn; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], C); }
        if constexpr (Bc::kOn && Bc::kStage > 0) mbar_init(bcast_full, 1);
        s_fault[0] = 0; s_fault[1] = 0;
        if constexpr (record::EmitOf<B>::kOn) { s_emit_err[0] = ~0ull; s_emit_err[1] = ~0ull; }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (threadIdx.x < 32) {
        if (threadIdx.x != 0) return;
        // ---------------- producer ----------------
        if constexpr (Bc::kOn && Bc::kStage > 0) {
            // before the first claim: every consumer waits for the block once (also in a CTA that gets no unit, so no
            // bulk load is still in flight when the CTA exits)
            if (staged) {
                if (bcast_bulk) {
                    mbar_expect_tx(bcast_full, bcast_bulk);
                    bulk_load(bcast_stage, wp.shared, bcast_bulk, bcast_full);
                } else {
                    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bcast_full)) : "memory");
                }
            }
        }
        for (uint32_t seq = 0;; ++seq) {
            const int sg = seq % kIn;
            mbar_wait(&empty[sg], ((seq / kIn) & 1) ^ 1);      // fresh barrier: passes immediately
            const uint32_t t = atomicAdd(wp.ticket, 1u);
            if (t >= wp.n_units) {
                // each CTA draws exactly one ticket >= n_units; the highest re-arms the counter
                if (t == wp.n_units + gridDim.x - 1u) *wp.ticket = 0u;
                s_rec[sg].count = 0u;                            // end marker
                asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&full[sg])) : "memory");
                return;
            }
            const TaskRecord rec = wave_record(wp, t);
            s_rec[sg] = rec;
            s_ticket[sg] = t;
            uint32_t nb = 0;
            if constexpr (kArgs) {
                const uint8_t* src = wp.args + rec.arg_off;
                if (wp.arg_stride == L::A && (reinterpret_cast<uintptr_t>(src) & 15) == 0) nb = (rec.count * L::A) & ~15u;
                s_bulk[sg] = nb;
                if (nb) {
                    mbar_expect_tx(&full[sg], nb);
                    bulk_load(in_stage + (size_t)sg * L::kInBytes, src, nb, &full[sg]);
                }
            }
            if (nb == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&full[sg])) : "memory");
        }
    }

    // ---------------- consumers (threads 32..287) ----------------
    const uint32_t ct = threadIdx.x - 32;
    if constexpr (Bc::kOn && Bc::kStage > 0) {
        if (staged) {
            // the bytes the bulk load could not take (an unaligned base, a tail under 16 B) are copied by hand, never
            // reading past shared_bytes; the named barrier before the first run() publishes them to every consumer
            mbar_wait(bcast_full, 0);
            record::coop_copy(bcast_stage + bcast_bulk, wp.shared + bcast_bulk, (uint32_t)wp.shared_bytes - bcast_bulk, ct, C);
        }
    }
    for (uint32_t seq = 0;; ++seq) {
        const int sg = seq % kIn, og = seq % kOut;
        mbar_wait(&full[sg], (seq / kIn) & 1);
        const TaskRecord rec = s_rec[sg];
        if (rec.count == 0) break;
        const uint32_t t = s_ticket[sg];
        const uint8_t* in = in_stage + (size_t)sg * L::kInBytes;
        uint8_t* out = out_stage + (size_t)og * L::kOutBytes;
        if constexpr (kArgs) {
            const uint8_t* src = wp.args + rec.arg_off;
            uint8_t* stage = in_stage + (size_t)sg * L::kInBytes;
            if (wp.arg_stride == L::A) {
                const uint32_t nb = s_bulk[sg];
                record::coop_copy(stage + nb, src + nb, rec.count * L::A - nb, ct, C);
            } else {
                record::gather_records<L::A>(stage, src, wp.arg_stride, rec.count, ct, C);
            }
        }
        // the bulk store that last read OUT stage `og` (unit seq - kOut) must be done with it.  Thread 0 commits exactly
        // one bulk group per unit (see below), so "at most kOut - 1 groups still reading" means units seq-kOut+1 .. seq-1
        if (ct == 0 && seq >= (uint32_t)kOut) bulk_wait_read<kOut - 1>();
        asm volatile("bar.sync 1, %0;" ::"n"(C) : "memory");

        int* const unit_fault = &s_fault[seq & 1];
        const ErrSink es{wp.err_word, unit_fault};
        unsigned long long* const emit_err = s_emit_err != nullptr ? &s_emit_err[seq & 1] : nullptr;
        if constexpr (!Bc::kOn) {
            record::run_unit<B, kIndex>(wp, rec, in, out, ct, es, emit_err);
        } else {
            using T = typename Bc::T;
            const uint64_t n_elems = wp.shared_bytes / Bc::kElem;
            // one loop per placement of the block, so each sees its pointer's address space (shared or global loads);
            // an items body keeps one loop over a generic pointer, because two such loops made ptxas spill
            if constexpr (record::ItemsOf<B>::kOn) {
                const uint8_t* blk = staged ? bcast_stage : wp.shared;
                record::run_unit<B, kIndex>(wp, rec, in, out, ct, es, emit_err, Broadcast<T>{reinterpret_cast<const T*>(blk), n_elems});
            } else {
                auto run = [&](const Broadcast<T>& sh) { record::run_unit<B, kIndex>(wp, rec, in, out, ct, es, emit_err, sh); };
                if (staged) run(Broadcast<T>{reinterpret_cast<const T*>(bcast_stage), n_elems});
                else run(Broadcast<T>{reinterpret_cast<const T*>(wp.shared), n_elems});
            }
        }
        // generic-proxy writes of this unit's stages become visible to the async proxy (the bulk store below, the
        // next bulk load into the IN stage); then the IN stage goes back to the producer
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&empty[sg])) : "memory");
        asm volatile("bar.sync 1, %0;" ::"n"(C) : "memory");

        if constexpr (record::FoldModeOf<B>::kOn) {
            // fold pass: the unit's tree in place in its OUT stage -- level s combines x[j] and x[j + s] for every j that
            // is a multiple of 2s, which is tree()'s pairing, an odd last element staying where it is -- then its
            // partial at the unit's place in the block.  No bulk group is committed, so the wait above never waits.
            // Levels 1 and 2 stay within consumer ct's own records 4ct .. 4ct+3 (kMaxUnit = 4 * C), levels 4 .. 64 within
            // its warp's 128 records, so only the levels from 128 on take a named barrier.  A Res of at most 32 bytes is
            // folded in registers up to the warp's total (shuffles), which its lane 0 stores back in place of x[128 w].
            static_assert(record::kMaxUnit == 4 * C, "fold pass: four records per consumer");
            using Res = typename B::Res;
            const uint32_t n = rec.count, j0 = 4u * ct;
            auto x = [&](uint32_t j) -> Res& { return *reinterpret_cast<Res*>(out + (size_t)j * L::R); };
            if constexpr (sizeof(Res) <= 32) {
                constexpr uint32_t W = sizeof(Res) / 4;
                uint32_t w[W] = {};
                if (j0 < n) {
                    Res a = x(j0);
                    if (j0 + 1 < n) B::combine(a, x(j0 + 1));
                    if (j0 + 3 < n) {
                        Res b = x(j0 + 2);
                        B::combine(b, x(j0 + 3));
                        B::combine(a, b);
                    } else if (j0 + 2 < n) {
                        B::combine(a, x(j0 + 2));
                    }
                    memcpy(w, &a, sizeof(Res));
                }
                for (uint32_t d = 1; d < 32 && 4u * d < n; d <<= 1) {   // level 4d: lane l takes lane l + d's total
                    uint32_t v[W];
#pragma unroll
                    for (uint32_t k = 0; k < W; ++k) v[k] = __shfl_down_sync(0xffffffffu, w[k], d);
                    if ((ct & (2u * d - 1u)) == 0 && j0 + 4u * d < n) {
                        Res a, o;
                        memcpy(&a, w, sizeof(Res));
                        memcpy(&o, v, sizeof(Res));
                        B::combine(a, o);
                        memcpy(w, &a, sizeof(Res));
                    }
                }
                if ((ct & 31u) == 0 && j0 < n) memcpy(&x(j0), w, sizeof(Res));
            } else {
                if (j0 + 1 < n) B::combine(x(j0), x(j0 + 1));
                if (j0 + 3 < n) B::combine(x(j0 + 2), x(j0 + 3));
                if (j0 + 2 < n) B::combine(x(j0), x(j0 + 2));
                for (uint32_t s = 4; s < 128 && s < n; s <<= 1) {
                    __syncwarp();
                    if (j0 % (2u * s) == 0 && j0 + s < n) B::combine(x(j0), x(j0 + s));
                }
            }
            asm volatile("bar.sync 1, %0;" ::"n"(C) : "memory");
            for (uint32_t s = 128; s < n; s <<= 1) {
                for (uint32_t j = ct * 2u * s; j + s < n; j += C * 2u * s) B::combine(x(j), x(j + s));
                asm volatile("bar.sync 1, %0;" ::"n"(C) : "memory");
            }
            // (a fold map's unit is a power of two: a shift, not a 64-bit division)
            record::coop_copy(wp.fold_partials + ((rec.first - wp.fold_first) >> (__ffs(wp.syn_unit) - 1)) * L::R, out, L::R, ct, C);
        } else {
            uint8_t* dst = wp.ring + (size_t)t * wp.slot_stride;
            const uint32_t bytes = rec.count * L::R;
            const uint32_t nbs = (reinterpret_cast<uintptr_t>(dst) & 15) == 0 ? (bytes & ~15u) : 0u;
            if (ct == 0) {
                // one group per unit, empty when the unit's results are all copied by hand (fewer than 16 bytes, or an
                // unaligned destination): the wait above counts groups, and must count units
                if (nbs) bulk_store(dst, out, nbs);
                else asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
            if (nbs < bytes) record::coop_copy(dst + nbs, out + nbs, bytes - nbs, ct, C);
        }
        if (ct == 0) {
            bool lost = false;
            if constexpr (B::kCanFault) {
                lost = *unit_fault != 0;                  // every consumer's reports for this unit are in (barrier above)
                s_fault[(seq + 1) & 1] = 0;               // re-arm the next unit's flag: its writers start after the next barrier
            }
            if constexpr (record::EmitOf<B>::kOn) {
                // a count mismatch counts only in a unit that was not lost; re-arm the word like the fault flag
                if (!lost && s_emit_err[seq & 1] != ~0ull) atomicMin(wp.err_word, s_emit_err[seq & 1]);
                s_emit_err[seq & 1] = ~0ull;
            }
            // the thread kernel's protocol: a lost unit is re-dispatched (resilient) or a task error
            if (lost && !wp.resilient)
                atomicMin(wp.err_word, (unsigned long long)(((wp.index_base + rec.first) << 8) | TASK_FAULT));
            put_header(wp, t, SlotHeader{rec.seq, rec.count | ((lost && wp.resilient) ? kUnitLost : 0u), rec.first});
        }
    }
    if (ct == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// fold_tree_kernel: tree() over the n records x[k * stride], k < n, of a fold body.  CTA b folds tile b -- records
// [b * kFoldTile, (b + 1) * kFoldTile), an aligned subtree of the whole tree -- in place, leaving its total at the tile's
// first record; the host repeats with stride * kFoldTile over the tile totals, and the launch with a single tile copies
// the result to dst.  The records are folded where they lie in global memory (L1 / L2 resident), so records up to 32 KB
// need no shared-memory budget.
template <class B>
__global__ void __launch_bounds__(kThreads) fold_tree_kernel(uint8_t* x, uint64_t n, uint64_t stride, uint8_t* dst) {
    using Res = typename B::Res;
    constexpr uint32_t T = record::kFoldTile;
    const uint64_t tiles = (n + T - 1) / T;
    for (uint64_t b = blockIdx.x; b < tiles; b += gridDim.x) {
        uint8_t* const base = x + b * T * stride;
        const uint32_t c = (uint32_t)(n - b * T < T ? n - b * T : T);
        for (uint32_t s = 1; s < c; s <<= 1) {
            for (uint32_t j = threadIdx.x * 2u * s; j + s < c; j += kThreads * 2u * s)
                B::combine(*reinterpret_cast<Res*>(base + j * stride), *reinterpret_cast<const Res*>(base + (j + s) * stride));
            __syncthreads();
        }
        if (tiles == 1) record::coop_copy(dst, base, (uint32_t)sizeof(Res), threadIdx.x, kThreads);
    }
}

// ================================================================================================
// Prefix folds of a fold body (FBR_SCAN maps, fbr_scan_values).  y[i] = tree(x[0..i]) is computed without a running
// carry, whose bracketing would depend on scheduling: with F_1 .. F_k the aligned power-of-two pieces of [0, i) given by
// the set bits of i, largest first -- each the tree of a complete aligned subtree, so the same bits as tree()'s node --
//     y[i] = F_1 (+) (F_2 (+) ( ... (+) (F_k (+) x[i])))            (a (+) b = combine(acc = a, b))
// evaluated innermost first, popcount(i) combines per element.  scan_level_kernel builds one level of the complete
// subtrees from the level below it (level k holds the n >> k subtrees of 2^k records), scan_wrap_kernel wraps each element.
// Records of at most kScanRegBytes are combined in registers; larger ones in global memory, through one scratch record
// per thread, so no record is ever copied to the stack.
// ================================================================================================
constexpr uint32_t kScanRegBytes = 32;
constexpr int kScanMaxLevels = 64;
struct ScanLevels {
    const uint8_t* at[kScanMaxLevels];   // at[k]: level k (at[0] unused: level 0 is x itself)
};

namespace scan_detail {
// dst <- src, one record of R (a multiple of 4) bytes, by one thread
__device__ __forceinline__ void copy_record(uint8_t* dst, const uint8_t* src, uint32_t R) {
#pragma unroll 1
    for (uint32_t k = 0; k < R; k += 4) *reinterpret_cast<uint32_t*>(dst + k) = *reinterpret_cast<const uint32_t*>(src + k);
}
}  // namespace scan_detail

// scan_level_kernel: dst[j] = src[2j] (+) src[2j + 1] for j < n
template <class B>
__global__ void __launch_bounds__(kThreads) scan_level_kernel(const uint8_t* src, uint8_t* dst, uint64_t n) {
    using Res = typename B::Res;
    constexpr uint32_t R = sizeof(Res);
    for (uint64_t j = blockIdx.x * (uint64_t)kThreads + threadIdx.x; j < n; j += (uint64_t)gridDim.x * kThreads) {
        const Res* s = reinterpret_cast<const Res*>(src + 2 * j * R);
        Res* d = reinterpret_cast<Res*>(dst + j * R);
        if constexpr (R <= kScanRegBytes) {
            Res a = s[0];
            B::combine(a, s[1]);
            *d = a;
        } else {
            scan_detail::copy_record(dst + j * R, src + 2 * j * R, R);
            B::combine(*d, s[1]);
        }
    }
}

// scan_wrap_kernel: record i of x (n records, rewritten in place) becomes y[i] when `prefix` is set (lv holds levels 1 ..
// 63 - clz(n)), then is wrapped with the n_pieces records G_1 .. G_m at `pieces`, right-nested:
// G_1 (+) (G_2 (+) ( ... (+) (G_m (+) y[i]))).  An odd i starts from level 1's node i >> 1, which is x[i - 1] (+) x[i] by
// the same combine, so no thread reads another thread's element.  `tmp` holds one scratch record per thread of the grid
// when R > kScanRegBytes.
template <class B>
__global__ void __launch_bounds__(kThreads) scan_wrap_kernel(uint8_t* x, uint64_t n, int prefix, const ScanLevels lv,
                                                             const uint8_t* pieces, uint32_t n_pieces, uint8_t* tmp) {
    using Res = typename B::Res;
    constexpr uint32_t R = sizeof(Res);
    const uint64_t tid = blockIdx.x * (uint64_t)kThreads + threadIdx.x;
    for (uint64_t i = tid; i < n; i += (uint64_t)gridDim.x * kThreads) {
        uint8_t* const xi = x + i * R;
        const uint8_t* cur = xi;                   // where the element's value is so far
        uint64_t bits = prefix ? i : 0;            // set bits still to wrap
        if (bits & 1) {
            cur = lv.at[1] + (i >> 1) * R;
            bits &= ~1ull;
        }
        if constexpr (R <= kScanRegBytes) {
            Res a = *reinterpret_cast<const Res*>(cur);
            for (int k = 1; bits; ++k) {
                if (!((bits >> k) & 1)) continue;
                bits &= ~(1ull << k);
                Res b = *reinterpret_cast<const Res*>(lv.at[k] + ((i >> k) - 1) * R);
                B::combine(b, a);
                a = b;
            }
            for (uint32_t m = n_pieces; m-- > 0;) {
                Res b = *reinterpret_cast<const Res*>(pieces + (uint64_t)m * R);
                B::combine(b, a);
                a = b;
            }
            *reinterpret_cast<Res*>(xi) = a;
        } else {
            uint8_t* const t = tmp + tid * R;
            // each step writes F (+) cur to whichever of xi and t does not hold cur
            auto wrap = [&](const uint8_t* f) {
                uint8_t* const dst = cur == xi ? t : xi;
                scan_detail::copy_record(dst, f, R);
                B::combine(*reinterpret_cast<Res*>(dst), *reinterpret_cast<const Res*>(cur));
                cur = dst;
            };
            for (int k = 1; bits; ++k) {
                if (!((bits >> k) & 1)) continue;
                bits &= ~(1ull << k);
                wrap(lv.at[k] + ((i >> k) - 1) * R);
            }
            for (uint32_t m = n_pieces; m-- > 0;) wrap(pieces + (uint64_t)m * R);
            if (cur != xi) scan_detail::copy_record(xi, cur, R);
        }
    }
}

// ================================================================================================
// scan_counts_kernel: the emit pass's offsets from the count pass's counts -- offs[i] = counts[0] + ... + counts[i-1] for
// i = 0 .. n, and *total = offs[n] (mapped pinned memory: the host reads it once the kernel is done).  A single-pass
// exclusive scan with decoupled look-back: CTAs claim tiles of kScanTile counts by ticket, so tile t only ever waits for
// tiles claimed before it, which are running or done.  tile_state (one word per tile, zero at launch) holds a tile's
// aggregate (flag A) as soon as it is known, and its inclusive prefix (flag P) once the look-back has found it; counts
// and totals are below 2^62, so flag and value fit one 64-bit word that is written and read whole.
// ================================================================================================
namespace scan {
constexpr int kThreads = 256, kItems = 8;
constexpr uint32_t kTile = kThreads * kItems;
constexpr unsigned long long kFlagA = 1ull << 62, kFlagP = 2ull << 62, kValue = (1ull << 62) - 1;
}  // namespace scan

__global__ void __launch_bounds__(scan::kThreads) scan_counts_kernel(const uint64_t* counts, uint64_t n, uint64_t* offs,
                                                                    unsigned long long* tile_state, uint32_t* ticket,
                                                                    uint64_t* total) {
    using scan::kItems; using scan::kTile; using scan::kFlagA; using scan::kFlagP; using scan::kValue;
    constexpr int kThreads = scan::kThreads;
    __shared__ uint32_t s_tile;
    __shared__ uint64_t s_warp[kThreads / 32];
    __shared__ uint64_t s_prefix;
    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    if (tid == 0) s_tile = atomicAdd(ticket, 1u);
    __syncthreads();
    const uint32_t tile = s_tile;
    const uint64_t base = (uint64_t)tile * kTile + (uint64_t)tid * kItems;
    uint64_t v[kItems], mine = 0;
#pragma unroll
    for (int k = 0; k < kItems; ++k) {
        v[k] = base + k < n ? counts[base + k] : 0ull;
        mine += v[k];
    }
    // CTA-wide exclusive scan of the per-thread sums: warp shuffles, then the warp totals
    uint64_t incl = mine;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint64_t u = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= (uint32_t)d) incl += u;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    uint64_t before = incl - mine, tile_total = 0;
    for (uint32_t w = 0; w < kThreads / 32; ++w) {
        if (w < warp) before += s_warp[w];
        tile_total += s_warp[w];
    }
    if (tid == 0) {
        volatile unsigned long long* st = tile_state;
        uint64_t prefix = 0;
        if (tile == 0) {
            st[0] = kFlagP | tile_total;
        } else {
            st[tile] = kFlagA | tile_total;
            for (int64_t j = (int64_t)tile - 1; j >= 0;) {
                const unsigned long long s = st[j];
                if ((s & ~kValue) == 0) continue;              // tile j has not published its aggregate yet
                prefix += s & kValue;
                if (s & kFlagP) break;
                --j;
            }
            st[tile] = kFlagP | (prefix + tile_total);
        }
        s_prefix = prefix;
    }
    __syncthreads();
    uint64_t run = s_prefix + before;
#pragma unroll
    for (int k = 0; k < kItems; ++k) {
        if (base + k < n) offs[base + k] = run;
        run += v[k];
    }
    if (tile == (uint32_t)(n / kTile) && tid == kThreads - 1) {   // the tile holding index n writes the end and the total
        offs[n] = run;
        *total = run;
        __threadfence_system();
    }
}

// ================================================================================================
// Keyed folds (FBR_FOLD_KEYS).  After a block's last round its window holds its n results in task order; the body's keys
// entry (keys_kernel) writes key[i] for each, a stable LSD radix sort of (key, task) pairs puts the tasks in key order, the
// records are gathered into that order, and the body's fold_segments entry folds each key's run with tree().  The sort is
// body-independent: 8-bit digits, ceil(log2(n_keys) / 8) passes (0 for one key, 1 up to 256 keys, 2 up to 65536), each a
// per-tile digit histogram, an exclusive scan over (digit, tile) (scan_counts_kernel), and a stable scatter.  Tasks are
// uint32 within a block.
// ================================================================================================
namespace keyed {
constexpr int kThreads = 256, kItems = 16, kWarps = kThreads / 32;
constexpr uint32_t kTile = kThreads * kItems;   // keys per sort tile; warp w of a tile owns its w-th run of 32 * kItems
constexpr int kBins = 256;
}  // namespace keyed

// hist[d * n_tiles + t] = number of keys of tile t whose digit (key >> shift) & 255 is d
__global__ void __launch_bounds__(keyed::kThreads) radix_hist_kernel(const uint32_t* keys, uint32_t n, int shift,
                                                                     uint64_t* hist, uint32_t n_tiles) {
    __shared__ uint32_t s_bins[keyed::kBins];
    for (uint32_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        for (int d = threadIdx.x; d < keyed::kBins; d += keyed::kThreads) s_bins[d] = 0;
        __syncthreads();
        const uint32_t base = t * keyed::kTile;
#pragma unroll 4
        for (uint32_t k = threadIdx.x; k < keyed::kTile; k += keyed::kThreads)
            if (base + k < n) atomicAdd(&s_bins[(keys[base + k] >> shift) & 255u], 1u);
        __syncthreads();
        for (int d = threadIdx.x; d < keyed::kBins; d += keyed::kThreads) hist[(uint64_t)d * n_tiles + t] = s_bins[d];
        __syncthreads();
    }
}

// Stable scatter of one pass: the key at i goes to offs[d * n_tiles + t] (the exclusive scan of radix_hist_kernel's
// counts) plus its rank among the keys of digit d before it in tile t.  Each warp ranks its run 32 keys at a time with
// __match_any_sync and keeps one counter per digit; the warps' counts are scanned in warp order first.  idx_in == nullptr
// is the identity permutation (the first pass).
__global__ void __launch_bounds__(keyed::kThreads) radix_scatter_kernel(const uint32_t* keys_in, const uint32_t* idx_in,
                                                                        uint32_t* keys_out, uint32_t* idx_out, uint32_t n,
                                                                        int shift, const uint64_t* offs, uint32_t n_tiles) {
    using keyed::kWarps; using keyed::kBins; using keyed::kItems; using keyed::kTile;
    __shared__ uint32_t s_cnt[kWarps][kBins];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t lt = (1u << lane) - 1u;
    for (uint32_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        for (int d = lane; d < kBins; d += 32) s_cnt[warp][d] = 0;
        __syncwarp();
        const uint32_t base = t * kTile + warp * (32u * kItems);
        uint32_t key[kItems];
#pragma unroll
        for (int j = 0; j < kItems; ++j) {
            const uint32_t i = base + j * 32u + lane;
            key[j] = i < n ? keys_in[i] : 0u;
        }
        // this warp's count of each digit
#pragma unroll
        for (int j = 0; j < kItems; ++j) {
            const bool valid = base + j * 32u + lane < n;
            const uint32_t d = valid ? (key[j] >> shift) & 255u : 256u;
            const uint32_t peers = __match_any_sync(0xffffffffu, d);
            if (valid && (peers & lt) == 0) s_cnt[warp][d] += __popc(peers);
            __syncwarp();
        }
        __syncthreads();
        // each counter becomes where the warp's first key of that digit goes
        for (int d = threadIdx.x; d < kBins; d += keyed::kThreads) {
            uint64_t run = offs[(uint64_t)d * n_tiles + t];
            for (int w = 0; w < kWarps; ++w) {
                const uint32_t c = s_cnt[w][d];
                s_cnt[w][d] = (uint32_t)run;
                run += c;
            }
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < kItems; ++j) {
            const uint32_t i = base + j * 32u + lane;
            const bool valid = i < n;
            const uint32_t d = valid ? (key[j] >> shift) & 255u : 256u;
            const uint32_t peers = __match_any_sync(0xffffffffu, d);
            if (valid) {
                const uint32_t at = s_cnt[warp][d] + __popc(peers & lt);
                keys_out[at] = key[j];
                idx_out[at] = idx_in ? idx_in[i] : i;
            }
            __syncwarp();
            if (valid && (peers & lt) == 0) s_cnt[warp][d] += __popc(peers);
            __syncwarp();
        }
        __syncthreads();
    }
}

// offs[k] = the first place of key k in the n sorted keys (offs[n_keys] = n) and counts[k] = its number of tasks
__global__ void __launch_bounds__(kThreads) key_offsets_kernel(const uint32_t* sorted, uint32_t n, uint32_t n_keys,
                                                               uint64_t* offs, uint64_t* counts) {
    auto lower = [&](uint32_t k) {
        uint32_t lo = 0, hi = n;
        while (lo < hi) {
            const uint32_t mid = lo + (hi - lo) / 2;
            if (sorted[mid] < k) lo = mid + 1; else hi = mid;
        }
        return lo;
    };
    for (uint32_t k = blockIdx.x * kThreads + threadIdx.x; k <= n_keys; k += gridDim.x * kThreads) {
        const uint32_t a = lower(k);
        offs[k] = a;
        if (k < n_keys) counts[k] = lower(k + 1) - a;
    }
}

// Sparse keyed folds (FBR_FOLD_SPARSE_KEYS): the runs of equal keys of the n sorted keys.  run_heads_kernel flags the first
// task of each run; the exclusive scan of the flags (scan_counts_kernel) gives each head its run number and D, the number of
// runs, as its total; run_starts_kernel then writes run r's first place and key, and starts[D] = n.
__global__ void __launch_bounds__(kThreads) run_heads_kernel(const uint32_t* sorted, uint32_t n, uint64_t* head) {
    for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads)
        head[i] = i == 0 || sorted[i] != sorted[i - 1];
}

__global__ void __launch_bounds__(kThreads) run_starts_kernel(const uint32_t* sorted, uint32_t n, const uint64_t* run_of,
                                                              uint64_t* starts, uint32_t* keys) {
    for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) {
        const uint32_t k = sorted[i];
        if (i == 0 || k != sorted[i - 1]) {
            starts[run_of[i]] = i;
            keys[run_of[i]] = k;
        }
        if (i == 0) starts[run_of[n]] = n;
    }
}

// dst record j <- src record perm[j], records of `words` W-byte words (W = 16, 8 or 4, the widest that divides R)
template <class W>
__global__ void __launch_bounds__(kThreads) gather_records_kernel(const W* src, W* dst, const uint32_t* perm, uint64_t n,
                                                                  uint32_t words) {
    const uint64_t total = n * words;
    for (uint64_t v = blockIdx.x * (uint64_t)kThreads + threadIdx.x; v < total; v += (uint64_t)gridDim.x * kThreads) {
        const uint64_t j = v / words, w = v - j * words;
        dst[v] = src[(uint64_t)perm[j] * words + w];
    }
}

// keys_kernel: key[i] = B::key(x[i]) for the n records of a keyed fold body.  A key >= n_keys is stored as 0, so the sort
// stays in bounds, and min((first_task + i) << 8 | FBR_TASK_KEY) goes into *err (the block's error word).
template <class B>
__global__ void __launch_bounds__(kThreads) keys_kernel(const uint8_t* x, uint64_t n, uint32_t n_keys, uint64_t first_task,
                                                        uint32_t* key, unsigned long long* err) {
    using Res = typename B::Res;
    for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < n; i += (uint64_t)gridDim.x * kThreads) {
        const uint32_t k = B::key(*reinterpret_cast<const Res*>(x + i * sizeof(Res)));
        if (k >= n_keys) atomicMin(err, (unsigned long long)(((first_task + i) << 8) | TASK_KEY));
        key[i] = k < n_keys ? k : 0u;
    }
}

// Segmented tree(): segment k is records [offs[k], offs[k + 1]) of x.  At level `step` (1, kFoldTile, kFoldTile^2, ...)
// segment k holds c = ceil(size / step) partial records, step records apart, and is cut into tiles of kFoldTile of them
// aligned at its start -- aligned subtrees of its tree(), as fold_tree_kernel cuts one array.  seg_tiles_kernel counts
// each segment's tiles with more than one record; their exclusive scan (scan_counts_kernel) numbers the tiles, and
// fold_segments_kernel folds tile g of segment k in place, leaving its total at the tile's first record.
__global__ void __launch_bounds__(kThreads) seg_tiles_kernel(const uint64_t* offs, uint32_t S, uint64_t step, uint64_t* tiles) {
    for (uint32_t k = blockIdx.x * kThreads + threadIdx.x; k < S; k += gridDim.x * kThreads) {
        const uint64_t c = (offs[k + 1] - offs[k] + step - 1) / step;
        tiles[k] = c > 1 ? (c + record::kFoldTile - 1) / record::kFoldTile : 0;
    }
}

template <class B>
__global__ void __launch_bounds__(kThreads) fold_segments_kernel(uint8_t* x, const uint64_t* offs, uint32_t S, uint64_t step,
                                                                 const uint64_t* tile_offs) {
    using Res = typename B::Res;
    constexpr uint32_t T = record::kFoldTile;
    const uint64_t total = tile_offs[S];
    const uint64_t stride = step * sizeof(Res);
    for (uint64_t g = blockIdx.x; g < total; g += gridDim.x) {
        uint32_t lo = 0, hi = S - 1;   // the last segment whose first tile is <= g
        while (lo < hi) {
            const uint32_t mid = (lo + hi + 1) / 2;
            if (tile_offs[mid] <= g) lo = mid; else hi = mid - 1;
        }
        const uint64_t b = g - tile_offs[lo];
        const uint64_t c_seg = (offs[lo + 1] - offs[lo] + step - 1) / step;
        uint8_t* const base = x + offs[lo] * sizeof(Res) + b * T * stride;
        const uint32_t c = (uint32_t)(c_seg - b * T < T ? c_seg - b * T : T);
        for (uint32_t s = 1; s < c; s <<= 1) {
            for (uint32_t j = threadIdx.x * 2u * s; j + s < c; j += kThreads * 2u * s)
                B::combine(*reinterpret_cast<Res*>(base + j * stride), *reinterpret_cast<const Res*>(base + (j + s) * stride));
            __syncthreads();
        }
    }
}

// dst[k] <- segment k's total (its first record), or the identity record for an empty segment; one warp per segment
template <class B>
__global__ void __launch_bounds__(kThreads) fold_segments_out_kernel(const uint8_t* x, const uint64_t* offs, uint32_t S,
                                                                     uint8_t* dst, const uint8_t* identity) {
    constexpr uint32_t R = sizeof(typename B::Res);
    const uint32_t lane = threadIdx.x & 31u;
    for (uint64_t k = (blockIdx.x * (uint64_t)kThreads + threadIdx.x) / 32; k < S; k += (uint64_t)gridDim.x * (kThreads / 32)) {
        const uint8_t* src = offs[k + 1] > offs[k] ? x + offs[k] * R : identity;
        for (uint32_t w = lane * 4; w < R; w += 32 * 4)
            *reinterpret_cast<uint32_t*>(dst + k * R + w) = *reinterpret_cast<const uint32_t*>(src + w);
    }
}

// ================================================================================================
// payload_fill: w[t][j] = low32(splitmix64(SEED ^ (t*1024 + j))); each thread emits 16 B.
// ================================================================================================
__global__ void __launch_bounds__(kThreads) payload_fill_kernel(uint4* out, uint64_t t0, uint64_t n_vec) {
    const uint64_t gsize = (uint64_t)gridDim.x * kThreads;
    for (uint64_t v = (uint64_t)blockIdx.x * kThreads + threadIdx.x; v < n_vec; v += gsize) {
        const uint64_t w0 = t0 * kPayloadWords + v * 4;
        uint4 r;
        r.x = (uint32_t)splitmix64(kPayloadSeed ^ (w0 + 0));
        r.y = (uint32_t)splitmix64(kPayloadSeed ^ (w0 + 1));
        r.z = (uint32_t)splitmix64(kPayloadSeed ^ (w0 + 2));
        r.w = (uint32_t)splitmix64(kPayloadSeed ^ (w0 + 3));
        out[v] = r;
    }
}

}  // namespace fbr
