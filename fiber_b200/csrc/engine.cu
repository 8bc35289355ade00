// engine.cu -- host side of libfiber_b200.so: pool object, per-GPU workers, rings, wave pipeline,
// and the extern "C" entry points declared in include/fiber_b200.h.
//
// One worker == one CUDA device (the GPU analogue of one job-backed worker process,
// fiber/pool.py:1009-1057 + fiber/local_backend.py:37-42) with
//   * three streams: copy-in (task records + arguments), compute (dispatch + gather), copy-out;
//   * a pinned host task ring and its device mirror (fixed-layout TaskRecord, cudaMemcpyAsync);
//   * a device result ring (payload arena + one SlotHeader per claim unit);
//   * double-buffered device staging for host-resident arguments and ordered output.
// A map is cut into waves that fit the rings; wave w+1's copy-in and wave w-1's copy-out overlap
// wave w's kernels.  No host thread is needed: ordering is carried by stream events, completion
// by events the caller waits on (fbr_result_wait / fbr_result_poll).
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <deque>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/fiber_b200.h"
#include "../../include/fiber_b200_body.cuh"
#include "kernels.cuh"

using namespace fbr;
using fbr_body_export::occupancy_of;

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
static thread_local std::string g_err;

static int fail(int code, const char* fmt, ...);
const std::string& last_error_of_this_thread();
static std::string vstrf(const char* fmt, va_list ap) {
    char buf[512];
    vsnprintf(buf, sizeof buf, fmt, ap);
    return buf;
}
static std::string strf(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    std::string s = vstrf(fmt, ap);
    va_end(ap);
    return s;
}
static int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    g_err = vstrf(fmt, ap);
    va_end(ap);
    return code;
}
const std::string& last_error_of_this_thread() { return g_err; }
#define CK(call)                                                                                  \
    do {                                                                                          \
        cudaError_t e_ = (call);                                                                  \
        if (e_ != cudaSuccess)                                                                    \
            return fail(FBR_ECUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

struct SubmitThread;
void SubmitThread_loop_impl(SubmitThread* t);
// One host thread per worker for submissions: the CUDA calls of different devices (stream waits, launches,
// async copies, event records: tens of us per part of 8 waves) run side by side instead of one after the other,
// which is what an 8-GPU in-process pool needs to keep up with sub-millisecond kernels.
struct SubmitThread {
    std::mutex mu;
    std::condition_variable cv;
    std::function<int()> job;
    bool pending = false, finished = false, quit = false;
    int rc = 0;
    std::string err;
    std::thread th;             // declared LAST: it starts running in the constructor and uses every member above
    SubmitThread() : th([this] { loop(); }) {}
    ~SubmitThread() {
        { std::lock_guard<std::mutex> g(mu); quit = true; }
        cv.notify_all();
        if (th.joinable()) th.join();
    }
    void loop() { SubmitThread_loop_impl(this); }
    void post(std::function<int()> f) {
        { std::lock_guard<std::mutex> g(mu); job = std::move(f); pending = true; finished = false; }
        cv.notify_all();
    }
    int wait(std::string* msg) {
        std::unique_lock<std::mutex> g(mu);
        cv.wait(g, [this] { return finished; });
        if (msg) *msg = err;
        return rc;
    }
};

// ------------------------------------------------------------------------------------------------
// body table: the compiled-in bodies plus bodies registered at run time from separately compiled
// modules (fbr_register_body).  The reference ships ANY callable to its workers (fiber/pool.py:961,
// executed at :806,809,820); here a callable's device body may live outside this library.
// ------------------------------------------------------------------------------------------------
typedef void (*launch_fn)(const void* wave_params, int grid, void* stream);
typedef int (*occupancy_fn)(int index_mode);

static void launch_payload_map(const void* wpv, int grid, void* sv) {
    const WaveParams& wp = *(const WaveParams*)wpv;
    cudaStream_t s = (cudaStream_t)sv;
    // contiguous records: TMA-staged, warp-specialised kernel (2 CTAs of 5 warps per SM); strided
    // records (arg_stride > 4096) keep the register-streaming kernel
    if (wp.arg_stride == kPayloadBytes) {
        int sm = 132, dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, dev);
        int per_sm = 2;
        if (const char* e = getenv("FBR_DISPATCH_OCC")) per_sm = std::max(1, std::min(per_sm, atoi(e)));
        const int g = (int)std::min<uint32_t>(wp.n_units, (uint32_t)(sm * per_sm));
        dispatch_payload_map_tma_kernel<<<g, 160, tma_map::kSmemBytes, s>>>(wp);
        return;
    }
    dispatch_payload_map_kernel<<<grid, kThreads, 0, s>>>(wp);
}
static int occ_payload_map(int) {
    cudaFuncSetAttribute(dispatch_payload_map_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tma_map::kSmemBytes);
    cudaFuncAttributes at;
    cudaFuncGetAttributes(&at, (const void*)dispatch_payload_map_tma_kernel);   // force-load
    return occupancy_of((const void*)dispatch_payload_map_kernel, kThreads, 0);
}
static void launch_payload_checksum(const void* wpv, int grid, void* sv) {
    dispatch_payload_checksum_kernel<<<grid, kThreads, 0, (cudaStream_t)sv>>>(*(const WaveParams*)wpv);
}
static int occ_payload_checksum(int) { return occupancy_of((const void*)dispatch_payload_checksum_kernel, kThreads, 0); }
// bit-packed twin of a bool body: range() indices through the body's own 16-index vector routine,
// explicit argument items through the generic ballot kernel
static void launch_pi_bits(const void* wpv, int grid, void* sv) {
    const WaveParams& wp = *(const WaveParams*)wpv;
    if (wp.arg_stride == 0) dispatch_pi_bits_kernel<<<grid, kThreads, 0, (cudaStream_t)sv>>>(wp);
    else dispatch_bits_items_kernel<PiInsideDet><<<grid, kThreads, 0, (cudaStream_t)sv>>>(wp);
}
static int occ_pi_bits(int index_mode) {
    return index_mode ? occupancy_of((const void*)dispatch_pi_bits_kernel, kThreads, 0) : occupancy_of((const void*)dispatch_bits_items_kernel<PiInsideDet>, kThreads, 0);
}
template <typename T>
static void launch_parzen(const void* wpv, int grid, void* sv) {
    dispatch_parzen_kernel<T><<<grid, kThreads, 0, (cudaStream_t)sv>>>(*(const WaveParams*)wpv);
}
template <typename T>
static int occ_parzen(int) { return occupancy_of((const void*)dispatch_parzen_kernel<T>, kThreads, 0); }

struct BodyEntry {
    std::string name;
    uint32_t arg_bytes = 0, result_bytes = 0, result_kind = 0, flags = 0, unit_tasks = 0;
    launch_fn launch = nullptr;
    occupancy_fn occupancy = nullptr;
    int max_ctas_per_sm = 0;   // 0 = as many as fit; streaming read+write bodies run best with few, fat streams
    void* module = nullptr;    // dlopen handle of a registered body (never closed: kernels may be in flight)
    uint32_t shared_elem_bytes = 0, shared_stage_bytes = 0;   // FBR_BODY_BROADCAST record bodies
    uint32_t item_streams = 0;                                // FBR_BODY_ITEMS record bodies: 1 to 4 item streams ...
    uint32_t item_bytes[kMaxItemStreams] = {};                // ... and the element size of each
    uint32_t out_bytes = 0;                                   // FBR_BODY_EMIT record bodies
    void (*fold)(void*, uint64_t, void*, void*) = nullptr;    // FBR_BODY_FOLD record bodies: tree() over device records ...
    std::vector<uint8_t> identity;                            // ... and identity(), result_bytes bytes
    int (*scan)(void*, uint64_t, int, const void*, uint32_t, void*) = nullptr;   // FBR_BODY_SCAN: prefix folds, wraps
    int (*keys)(const void*, uint64_t, uint32_t, uint64_t, uint32_t*, unsigned long long*, void*) = nullptr;   // FBR_BODY_KEYED:
    int (*fold_segments)(void*, uint64_t, const uint64_t*, uint32_t, void*, void*) = nullptr;            // keys, segmented tree()
};

static std::mutex g_body_mu;
static std::deque<BodyEntry> g_bodies;   // append-only: references stay valid, func_id = position

static void builtin_bodies_once() {
    // caller holds g_body_mu
    if (!g_bodies.empty()) return;
    auto add = [](const char* name, uint32_t ab, uint32_t rb, uint32_t kind, uint32_t flags, uint32_t unit, launch_fn l,
                  occupancy_fn o, int max_ctas) {
        BodyEntry b;
        b.name = name; b.arg_bytes = ab; b.result_bytes = rb; b.result_kind = kind; b.flags = flags; b.unit_tasks = unit;
        b.launch = l; b.occupancy = o; b.max_ctas_per_sm = max_ctas;
        g_bodies.push_back(b);
    };
    // order == enum FuncId (bodies.cuh)
    add("square_i64", 8, 8, FBR_RES_I64, FBR_BODY_INDEX_ARG | FBR_BODY_SUMMABLE, 4096, fbr_body_export::launch<SquareI64>, fbr_body_export::occupancy<SquareI64>, 0);
    add("mul2_i64", 16, 8, FBR_RES_I64, FBR_BODY_SUMMABLE, 4096, fbr_body_export::launch<Mul2I64>, fbr_body_export::occupancy<Mul2I64>, 0);
    add("square_scale_i64", 16, 8, FBR_RES_I64, FBR_BODY_SUMMABLE, 4096, fbr_body_export::launch<SquareScaleI64>, fbr_body_export::occupancy<SquareScaleI64>, 0);
    add("identity_i64", 8, 8, FBR_RES_I64, FBR_BODY_INDEX_ARG | FBR_BODY_SUMMABLE, 4096, fbr_body_export::launch<IdentityI64>, fbr_body_export::occupancy<IdentityI64>, 0);
    add("pi_inside_det", 8, 1, FBR_RES_BOOL, FBR_BODY_INDEX_ARG | FBR_BODY_SUMMABLE, 4096, fbr_body_export::launch<PiInsideDet>, fbr_body_export::occupancy<PiInsideDet>, 0);
    add("parzen_f32", 8, 16, FBR_RES_F64X2, FBR_BODY_NEEDS_SHARED, 1, launch_parzen<float>, occ_parzen<float>, 0);
    add("parzen_f64", 8, 16, FBR_RES_F64X2, FBR_BODY_NEEDS_SHARED, 1, launch_parzen<double>, occ_parzen<double>, 0);
    add("payload_map_4k", 4096, 4096, FBR_RES_BYTES, 0, 32, launch_payload_map, occ_payload_map,
        3 /* few fat CTAs per SM stream read+write waves better than many thin ones */);
    add("payload_checksum_4k", 4096, 4, FBR_RES_U32, FBR_BODY_SUMMABLE, 256, launch_payload_checksum, occ_payload_checksum, 0);
    add("sleep_f64", 8, 1, FBR_RES_NONE, 0, 1, fbr_body_export::launch<SleepF64>, fbr_body_export::occupancy<SleepF64>, 0);
    add("fault_identity_i64", 8, 8, FBR_RES_I64, FBR_BODY_INDEX_ARG | FBR_BODY_SUMMABLE, 2, fbr_body_export::launch<FaultIdentityI64>, fbr_body_export::occupancy<FaultIdentityI64>, 0);
    // a byte-task = 8 items: 8 range() indices (arg_stride 0) or 8 int64 argument items (arg_stride 64)
    add("pi_inside_bits8", 64, 1, FBR_RES_BITS8, FBR_BODY_INDEX_ARG | FBR_BODY_SUMMABLE, 512, launch_pi_bits, occ_pi_bits, 0);
    add("trap_identity_i64", 8, 8, FBR_RES_I64, FBR_BODY_INDEX_ARG | FBR_BODY_SUMMABLE, 4096, fbr_body_export::launch<TrapIdentityI64>, fbr_body_export::occupancy<TrapIdentityI64>, 0);
}
static int body_count() {
    std::lock_guard<std::mutex> g(g_body_mu);
    builtin_bodies_once();
    return (int)g_bodies.size();
}
// nullptr if func_id is out of range
static const BodyEntry* body_of(int func_id) {
    std::lock_guard<std::mutex> g(g_body_mu);
    builtin_bodies_once();
    if (func_id < 0 || func_id >= (int)g_bodies.size()) return nullptr;
    return &g_bodies[func_id];
}

// ------------------------------------------------------------------------------------------------
// pool structures
// ------------------------------------------------------------------------------------------------
enum { ST_RUN = 0, ST_CLOSE = 1, ST_TERMINATE = 2 };
constexpr int kRecWindows = 4;         // task-ring windows in flight
constexpr uint32_t kRecCapacity = 65536;  // claim units per wave
constexpr int kCtrlSlots = 65536;      // maps in flight (submitted, not yet released) per worker
constexpr int kTickets = 64;

struct SeqCtrl {              // per (seq, worker) control block, device + pinned mirror
    long long sum;            // 8-byte results: sum of the low 32-bit halves; other kinds: the sum itself
    unsigned long long err;   // (task_index << 8 | code), ~0 = none
    uint32_t lost_count;
    uint32_t pad;
    long long sum_hi;         // 8-byte results: sum of the high halves (exact total = sum_hi * 2^32 + sum)
};
static_assert(sizeof(SeqCtrl) == 32, "");

struct Worker {
    int device = -1;
    bool dead = false;                     // the device's CUDA context took a sticky error: the worker process is gone
    int death_error = 0;                   // cudaError_t that killed it
    int numa_node = -1;                    // host NUMA node the GPU hangs off (-1 unknown)
    int sm_count = 0;
    cudaStream_t s_in = nullptr, s_comp = nullptr, s_out = nullptr;
    cudaStream_t s_gath = nullptr;         // higher-priority stream for gathers that overlap the next dispatch
    cudaStream_t s_fold = nullptr;         // fold_host_records and the wraps of queue_wrap: nothing there queues behind the maps
                                           // on the other streams, so a wait for it under the pool lock is short
    bool prev_wave_overlap = false;        // the previous wave used only its half of the ring
    cudaStream_t s_push = nullptr;         // a stream of the ROOT worker's device: its copy engine pushes this worker's argument waves
    cudaStream_t s_push2 = nullptr;        // (waves alternate between the two, like the copy-outs)
    cudaEvent_t ev_push[kRecWindows] = {}; // ... and these (root-device) events say when a pushed wave has landed
    int push_root_device = -1;
    uint32_t gath_hist = 0;                // bit k: wave wno-1-k ran its gather on s_gath (its ev_comp is not ordered by s_comp)
    TaskRecord* h_records = nullptr;   // pinned task ring: kRecWindows x kRecCapacity
    TaskRecord* d_records = nullptr;   // device mirror
    SlotHeader* d_headers = nullptr;   // kRecCapacity
    uint8_t* d_ring = nullptr;         // result ring arena (ring_bytes)
    uint8_t* d_args[2] = {nullptr, nullptr};
    uint8_t* d_items[2] = {nullptr, nullptr};   // items bodies, host-resident items: each stream's offsets slice, then its item span
    uint8_t* d_vals[2] = {nullptr, nullptr};    // emit bodies, host-resident values: a wave's values before their D2H copy
    uint8_t* d_out[2] = {nullptr, nullptr};
    uint32_t* d_tickets = nullptr;
    SeqCtrl* d_ctrl = nullptr;
    SeqCtrl* h_ctrl = nullptr;         // pinned: [0,kCtrlSlots) results, [kCtrlSlots] init pattern
    cudaEvent_t ev_rec_h2d[kRecWindows];   // window's H2D finished (host may rewrite the pinned window)
    cudaEvent_t ev_comp[kRecWindows];      // wave's kernels finished (device window / arg half reusable)
    cudaEvent_t ev_disp[kRecWindows];      // wave's dispatch kernel finished (its gather may start)
    cudaEvent_t ev_out[2];                 // out half's D2H finished
    uint64_t wave_no = 0;
    std::vector<int> occ, occ_index;   // per func_id: resident CTAs/SM of the explicit-argument / range() instantiation (0 = not asked yet)
    std::vector<int> occ_fold, occ_fold_index;   // ... and of the fold pass of a fold body
    int occ_gather = 1, occ_fill = 1, occ_gather_rows = 1;
    std::vector<int> ctrl_free;        // free-list of control-block slots
};

// resident CTAs per SM of body `func_id` on this worker's device (current device must be w.device)
static int worker_occ(Worker& w, int func_id, const BodyEntry& body, bool index_mode, bool fold) {
    std::vector<int>& v = fold ? (index_mode ? w.occ_fold_index : w.occ_fold) : (index_mode ? w.occ_index : w.occ);
    if ((int)v.size() <= func_id) v.resize(func_id + 1, 0);
    if (v[func_id] == 0) v[func_id] = std::max(1, body.occupancy((index_mode ? 1 : 0) | (fold ? 2 : 0)));
    return v[func_id];
}

struct TimedPair { cudaEvent_t a, b; };

// Where a block's results go (BlockPlan::sink):
//   Staged        the worker's out-staging halves, copied to the host segment wave by wave
//   StagedPeer    the out-staging halves, pushed wave by wave by this worker's copy engine to the ordered output on worker 0
//                 (another GPU): kernels storing over NVLink stay below what a copy engine pushes (FBR_PEER_OUT=0: CallerDevice)
//   CallerDevice  the caller's device output (FBR_OUT_DEVICE), stored in place
//   ZeroCopy      the pinned host segment, stored into over PCIe by the dispatch kernel itself (bit-packed bools)
//   WindowToHost  an engine window, copied to the host in one piece once no unit is lost (resilient, FBR_FULL_WINDOW)
//   WindowOnDevice  an engine window that stays on the device (FBR_RESULTS_ON_DEVICE)
//   ScanWindow    an engine window, rewritten into the block's prefix folds after its last round (FBR_SCAN)
//   KeyedWindow   an engine window, sorted by key and folded per key after its last round (FBR_FOLD_KEYS)
//   SparseKeyedWindow  an engine window, sorted by key and cut into runs of equal keys after its last round; the runs are
//                 folded at completion (FBR_FOLD_SPARSE_KEYS)
//   FoldPartials  each unit's tree, in d_fold: no result leaves the device (FBR_FOLD)
enum class Sink : uint8_t { Staged, StagedPeer, CallerDevice, ZeroCopy, WindowToHost, WindowOnDevice, ScanWindow, KeyedWindow,
                            SparseKeyedWindow, FoldPartials };
// Where a block's argument records come from: none (range() indices), the caller's device memory read in place
// (FBR_ARGS_DEVICE), a device copy of the block's records made once (Resident: a resilient unit may be re-dispatched at any
// time), the host wave by wave through the d_args staging halves, or device memory of worker 0 pushed wave by wave into the
// staging halves by worker 0's copy engine (FBR_PEER_PUSH=0: the kernel loads them itself, DeviceInPlace).
enum class ArgSource : uint8_t { None, DeviceInPlace, Resident, Staged, Pushed };
// Where an items body's items and offsets come from: the caller's device memory read in place, the host wave by wave
// through the d_items staging halves, or a device copy of the block's item span and offsets made once (resilient).
enum class ItemSource : uint8_t { None, DeviceInPlace, Staged, Resident };

// The placement of one worker's block of one map: decided once by plan_block, before anything is allocated, then acted on.
struct BlockPlan {
    uint32_t unit = 0, slot_stride = 0, R = 0, sum_kind = 0;
    Sink sink = Sink::Staged;
    ArgSource args = ArgSource::None;
    ItemSource items = ItemSource::None;
    bool resilient = false;
    bool direct = false;                  // contiguous, unshuffled, non-resilient block: the dispatch kernel stores every
                                          // unit at its final index (no ring, no task records, no gather launch)
    bool overlap = false;                 // gather(w) on s_gath concurrently with dispatch(w+1); ring used in halves
    uint64_t wave_tasks_cap = 0;          // tasks per regular wave (0: the ring holds no claim unit)
    uint64_t redispatch_units_cap = 0;    // claim units per re-dispatch wave
    uint64_t args_limit_bytes = 0;        // host arguments end here (n_items records); 0 = n_tasks * arg_stride
    // results pass through the out-staging halves; else they go to one window of the whole block (or d_fold)
    bool staged() const { return sink == Sink::Staged || sink == Sink::StagedPeer; }
    // the engine allocates the block's window on the device
    bool engine_window() const { return !staged() && sink != Sink::CallerDevice && sink != Sink::ZeroCopy && sink != Sink::FoldPartials; }
    // nothing of the block is final before its last round is: its results reach the host in one copy at the end, are
    // stored over PCIe by the kernel, or are rewritten (scan, keyed, fold) behind its last wave
    bool final_at_block_end() const { return !staged() && sink != Sink::CallerDevice && sink != Sink::WindowOnDevice; }
    // each wave copies its argument records in (from the host, or pushed by worker 0)
    bool args_streamed() const { return args == ArgSource::Staged || args == ArgSource::Pushed; }
    // the bytes of the argument records of tasks [first, first + n): a bit-packed map's last task may cover fewer items
    uint64_t arg_bytes(uint64_t first, uint64_t n, uint32_t stride) const {
        const uint64_t start = first * stride, bytes = n * stride;
        return !args_limit_bytes ? bytes : start >= args_limit_bytes ? 0 : std::min(bytes, args_limit_bytes - start);
    }
};

// The runtime state of a block's placement: the pointers its plan asked for, once they are allocated.
struct PartCtx {
    BlockPlan plan;
    uint8_t* fold_total = nullptr;        // FBR_FOLD: the block's total, in the map's pinned segment
    uint8_t* key_totals = nullptr;        // FBR_FOLD_KEYS: the block's n_keys totals and counts, in the map's pinned segment
    uint8_t* key_counts = nullptr;
    uint64_t* n_groups = nullptr;         // FBR_FOLD_SPARSE_KEYS: the block's D, its word of SeqState::sparse_words
    const uint8_t* d_shared = nullptr;
    uint8_t* window_base = nullptr;       // the block's window (BlockPlan::windowed)
    const uint8_t* args_full = nullptr;   // device-resident arguments of the whole map (DeviceInPlace / Resident)
    // items bodies: where the kernel finds the items and offsets of each stream for the whole map (WaveParams::items ...,
    // more_items), and the map index of the task offsets[0] belongs to
    ItemStream items[kMaxItemStreams] = {};
    uint64_t item_first = 0;
};

// A worker block of an emit map's emit pass: the part-local exclusive offsets its scan produced (count + 1 of them, the last
// is the block's total) and where its values go.  Blocks are contiguous, so block k's values start at the totals of the
// blocks before it (base).
// Where the emit pass writes a block's values:
//   - FBR_RESULTS_ON_DEVICE: d_values, an engine-owned device buffer of the block's exact size;
//   - host-resident values of a block that may re-dispatch units (resilient, FBR_FULL_WINDOW): d_values too, copied to the
//     pinned segment (host) in one piece once no unit is lost any more;
//   - other host-resident values: wave by wave into the worker's d_vals staging half, each wave's span copied to `host`
//     behind its kernel; h_offs (a pinned copy of the block's offsets) gives the host every wave's span before it launches.
struct EmitBlock {
    uint64_t* d_offs = nullptr;           // null: not an emit pass
    uint64_t* h_offs = nullptr;           // pinned: the block's count + 1 offsets (waves staged through d_vals)
    void* d_values = nullptr;
    uint8_t* host = nullptr;              // the block's first value in the pinned values segment (host-resident maps)
    uint64_t base = 0, total = 0;
};

struct SeqPart {
    int worker = 0;
    uint64_t first = 0, count = 0;        // task block of this worker inside the map
    int ctrl_slot = -1;
    cudaEvent_t done = nullptr;
    std::vector<cudaEvent_t> wave_done;
    std::vector<uint64_t> wave_cum;       // tasks finished once wave i is done
    std::vector<TimedPair> t_dispatch, t_gather;
    void* d_shared_tmp = nullptr;         // per-seq device copy of a host shared block
    void* d_window = nullptr;             // FULL_WINDOW device output
    void* d_args_full = nullptr;          // resilient: device copy of all argument records
    void* d_items[kMaxItemStreams] = {};      // resilient items bodies with host-resident items: each stream's item span ...
    void* d_item_offs[kMaxItemStreams] = {};  // ... and its count + 1 offsets, on the device for the part's whole life
    LostUnit* d_lost = nullptr;           // resilient: units whose worker "died" (filled by gather)
    LostUnit* h_lost = nullptr;           // pinned mirror
    uint32_t lost_cap = 0, attempt = 0;
    bool finalized = false;               // resilient: window copied back to the host
    bool first_wave_pending = true;       // the block's first wave must wait for what submit_part put on s_in
    void* d_fold = nullptr;               // FBR_FOLD: the partial of each claim unit, by its place in the block
    void* d_sparse = nullptr;             // FBR_FOLD_SPARSE_KEYS: gathered records, run starts, keys (sparse_keep_layout)
    PartCtx cx;
    EmitBlock emit;
};

struct SeqState {
    uint64_t seq = 0, n_tasks = 0;
    int func_id = 0;
    uint32_t flags = 0, result_bytes = 0, result_kind = 0;
    void* out = nullptr;
    bool own_out = false;
    bool finished = false;
    int64_t sum = 0;              // total wrapped to int64 ...
    uint64_t sum_lo = 0;          // ... and its exact form: sum_hi * 2^32 + sum_lo
    int64_t sum_hi = 0;
    bool sum_overflow = false;    // the exact total does not fit int64
    uint32_t err_code = 0;
    uint64_t err_task = 0;
    uint32_t n_waves = 0;
    uint32_t redispatched_units = 0;
    fbr_map_desc_t desc;
    fbr_items_desc_t items[kMaxItemStreams];   // items bodies (fbr_map_submit_items_n): one per stream; zero otherwise
    uint32_t n_item_streams = 0;
    std::vector<SeqPart> parts;
    std::vector<SeqPart> graveyard;        // parts that were running on a worker when it died (their blocks were re-dispatched)
    int waiters = 0;                       // threads inside fbr_result_wait for this seq (they hold event handles outside the lock)
    bool release_pending = false;          // fbr_result_release arrived while they were waiting: the last one out frees the seq
    int dead_worker = -1;                  // a worker died under this map and the map could not be re-dispatched
    int dead_error = 0;
    bool emit_pass = false;                // the emit pass of an emit map: its blocks carry the offsets their workers counted
    void* values = nullptr;                // emit pass: pinned values segment (host-resident results) ...
    uint64_t n_values = 0;                 // ... and the map's number of values
    bool completed = false;                // complete_map is done: the map is harvested, a fold map's result record (out) holds
                                           // tree() over the block totals, and a scan map's blocks after the first are wrapped
    std::vector<uint8_t> scan_totals;      // FBR_SCAN, several blocks: every block's total in block order, read before any
                                           // block is wrapped (the wrap rewrites the record that holds it)
    std::vector<cudaEvent_t> block_done;   // ... and block b's wrap (and D2H copy) once queued on its worker's s_fold; a sparse
                                           // keyed map's block b's run fold and D2H copy (sparse_keyed_finish)
    uint64_t* sparse_words = nullptr;      // FBR_FOLD_SPARSE_KEYS: each block's D, in pinned memory its run scan writes into
    std::vector<void*> sparse_host;        // ... block b's totals, keys and run starts once copied out (pinned, block order)
    std::vector<uint32_t> group_keys;      // ... and the result's distinct keys and counts (fbr_result_groups)
    std::vector<uint64_t> group_counts;
};

struct SharedBlock {
    uint64_t bytes = 0;
    std::vector<void*> d_ptr;  // per worker
};

struct fbr_pool {
    std::mutex mu;
    int state = ST_RUN;
    uint32_t flags = 0;
    uint64_t ring_bytes = 0;
    bool peer_ok = false;             // every worker can load/store every other worker's memory (NVLink P2P)
    bool peer_checked = false;        // ... decided (and enabled) by the first map with device-resident args / output
    std::vector<Worker> workers;
    uint64_t next_seq = 0;
    std::unordered_map<uint64_t, std::unique_ptr<SeqState>> seqs;
    std::unordered_map<uint64_t, SharedBlock> shared;
    uint64_t next_shared = 1;
    std::vector<std::unique_ptr<SubmitThread>> submitters;   // per worker, started with the first multi-worker map
    // pinned host segment cache (size class -> free blocks), and live blocks -> class
    std::unordered_map<uint64_t, std::vector<void*>> pin_free;
    std::unordered_map<void*, uint64_t> pin_live;
    uint64_t pin_cached_bytes = 0;    // bytes sitting in pin_free (bounded by kPinCacheCap)
    // NUMA-split result segments of multi-worker maps: exact byte size -> free blocks; live -> mapped bytes
    std::unordered_map<uint64_t, std::vector<void*>> numa_free;
    std::unordered_map<void*, std::pair<uint64_t, uint64_t>> numa_live;   // ptr -> (key bytes, mapped bytes)
    fbr_stats_t stats;
};

// ------------------------------------------------------------------------------------------------
// helpers
// ------------------------------------------------------------------------------------------------
// the parts of a multi-worker map are submitted from one host thread per worker: counters are added atomically
#define STAT_ADD(p, field, v) __atomic_fetch_add(&(p)->stats.field, (uint64_t)(v), __ATOMIC_RELAXED)

void SubmitThread_loop_impl(SubmitThread* t) {
    std::unique_lock<std::mutex> g(t->mu);
    for (;;) {
        t->cv.wait(g, [t] { return t->pending || t->quit; });
        if (t->quit) return;
        std::function<int()> f = std::move(t->job);
        t->pending = false;
        g.unlock();
        const int rc = f();
        const std::string msg = rc != FBR_OK ? last_error_of_this_thread() : std::string();
        g.lock();
        t->rc = rc;
        t->err = msg;
        t->finished = true;
        t->cv.notify_all();
    }
}

static uint64_t round_up(uint64_t x, uint64_t m) { return (x + m - 1) / m * m; }

static uint64_t pin_class(uint64_t bytes) {
    uint64_t c = 4096;
    while (c < bytes) c <<= 1;
    return c;
}

constexpr uint64_t kPinCacheCap = 24ull << 30;   // keep at most this much idle pinned memory per pool

static int pinned_acquire(fbr_pool* p, uint64_t bytes, void** out) {
    const uint64_t c = pin_class(bytes ? bytes : 1);
    auto& fl = p->pin_free[c];
    void* ptr = nullptr;
    if (!fl.empty()) {
        ptr = fl.back();
        fl.pop_back();
        p->pin_cached_bytes -= c;
    } else {
        CK(cudaHostAlloc(&ptr, c, cudaHostAllocPortable));
    }
    p->pin_live[ptr] = c;
    *out = ptr;
    return FBR_OK;
}

static void pinned_release(fbr_pool* p, void* ptr) {
    auto it = p->pin_live.find(ptr);
    if (it == p->pin_live.end()) return;
    const uint64_t c = it->second;
    p->pin_live.erase(it);
    if (p->pin_cached_bytes + c > kPinCacheCap) {
        cudaFreeHost(ptr);            // cache full: give the pages back
        return;
    }
    p->pin_free[c].push_back(ptr);
    p->pin_cached_bytes += c;
}

// ---- NUMA-split pinned segments ------------------------------------------------------------------
// One process driving several GPUs writes one ordered result segment; with a plain cudaHostAlloc the
// whole segment sits on the allocating thread's NUMA node and half of the GPUs push their D2H
// stream across the socket link, which caps the aggregate well below what socket-local blocks reach.  Here each worker's block of the segment is bound (mbind) to the node its
// GPU hangs off before the pages are faulted in by cudaHostRegister.
static int numa_node_of_device(int device) {
    char bdf[32] = {0};
    if (cudaDeviceGetPCIBusId(bdf, sizeof bdf, device) != cudaSuccess) { cudaGetLastError(); return -1; }
    for (char* c = bdf; *c; ++c) if (*c >= 'A' && *c <= 'F') *c = (char)(*c - 'A' + 'a');
    char path[128];
    snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bdf);
    FILE* f = fopen(path, "r");
    if (!f) return -1;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    return node;
}

static void bind_range_to_node(void* addr, uint64_t len, int node) {
    if (node < 0 || node >= 64 || len == 0) return;
    unsigned long mask = 1ul << node;
    // MPOL_BIND = 2; failure (no NUMA, no permission) only costs locality
    syscall(SYS_mbind, addr, (unsigned long)len, 2, &mask, 65ul, 0u);
}

struct NumaBlock { uint64_t off, len; int node; };

static int numa_pinned_acquire(fbr_pool* p, uint64_t bytes, const std::vector<NumaBlock>& blocks, void** out) {
    auto& fl = p->numa_free[bytes];
    if (!fl.empty()) {
        void* ptr = fl.back();
        fl.pop_back();
        p->numa_live[ptr].first = bytes;
        *out = ptr;
        return FBR_OK;
    }
    const uint64_t page = 1ull << 21;
    const uint64_t mapped = round_up(std::max<uint64_t>(bytes, 1), page);
    void* ptr = mmap(nullptr, mapped, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
    if (ptr == MAP_FAILED) return fail(FBR_ENOMEM, "mmap of %llu bytes failed", (unsigned long long)mapped);
    const uint64_t small = 4096;
    for (const NumaBlock& b : blocks) {
        const uint64_t lo = b.off / small * small, hi = std::min(mapped, round_up(b.off + b.len, small));
        bind_range_to_node((uint8_t*)ptr + lo, hi - lo, b.node);
    }
    cudaError_t e = cudaHostRegister(ptr, mapped, cudaHostRegisterPortable | cudaHostRegisterMapped);
    if (e != cudaSuccess) {
        munmap(ptr, mapped);
        return fail(FBR_ECUDA, "cudaHostRegister failed: %s", cudaGetErrorString(e));
    }
    p->numa_live[ptr] = {bytes, mapped};
    *out = ptr;
    return FBR_OK;
}

static bool numa_pinned_release(fbr_pool* p, void* ptr) {
    auto it = p->numa_live.find(ptr);
    if (it == p->numa_live.end()) return false;
    p->numa_free[it->second.first].push_back(ptr);
    return true;
}

static int worker_init(fbr_pool* p, Worker& w, int device) {
    w.device = device;
    CK(cudaSetDevice(device));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)     // sm_90a code loads on compute capability 9.0 and nothing else
        return fail(FBR_ENODEV, "device %d is sm_%d%d; this library is built for sm_90a (H100) only", device, prop.major, prop.minor);
    w.sm_count = prop.multiProcessorCount;
    w.numa_node = numa_node_of_device(device);
    {
        // stream-ordered allocations (per-map windows, shared blocks) come from the device's default pool: keep what is
        // freed cached instead of handing it back to the driver at every synchronisation (the default threshold is 0;
        // with 8 ranks on one box a 100 MB cudaMallocAsync/cudaFreeAsync pair per map then costs a millisecond)
        cudaMemPool_t mp = nullptr;
        if (cudaDeviceGetDefaultMemPool(&mp, device) == cudaSuccess) {
            uint64_t keep = ~0ull;
            cudaMemPoolSetAttribute(mp, cudaMemPoolAttrReleaseThreshold, &keep);
        }
        cudaGetLastError();
    }
    CK(cudaStreamCreateWithFlags(&w.s_in, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&w.s_comp, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&w.s_out, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&w.s_fold, cudaStreamNonBlocking));
    {
        int lo_prio = 0, hi_prio = 0;
        CK(cudaDeviceGetStreamPriorityRange(&lo_prio, &hi_prio));
        CK(cudaStreamCreateWithPriority(&w.s_gath, cudaStreamNonBlocking, hi_prio));
    }
    CK(cudaHostAlloc((void**)&w.h_records, sizeof(TaskRecord) * kRecCapacity * kRecWindows, cudaHostAllocPortable));
    CK(cudaMalloc((void**)&w.d_records, sizeof(TaskRecord) * kRecCapacity * kRecWindows));
    CK(cudaMalloc((void**)&w.d_headers, sizeof(SlotHeader) * kRecCapacity * 2));   // two halves (overlapped waves)
    CK(cudaMalloc((void**)&w.d_ring, p->ring_bytes));
    CK(cudaMalloc((void**)&w.d_tickets, sizeof(uint32_t) * kTickets * 2));
    CK(cudaMemsetAsync(w.d_tickets, 0, sizeof(uint32_t) * kTickets * 2, w.s_comp));
    CK(cudaMalloc((void**)&w.d_ctrl, sizeof(SeqCtrl) * kCtrlSlots));
    CK(cudaHostAlloc((void**)&w.h_ctrl, sizeof(SeqCtrl) * (kCtrlSlots + 1), cudaHostAllocPortable));
    w.h_ctrl[kCtrlSlots] = SeqCtrl{0, ~0ull, 0u, 0u, 0};
    w.ctrl_free.resize(kCtrlSlots);
    for (int i = 0; i < kCtrlSlots; ++i) w.ctrl_free[i] = kCtrlSlots - 1 - i;
    for (int i = 0; i < kRecWindows; ++i) {
        CK(cudaEventCreateWithFlags(&w.ev_rec_h2d[i], cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&w.ev_comp[i], cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&w.ev_disp[i], cudaEventDisableTiming));
    }
    for (int i = 0; i < 2; ++i) CK(cudaEventCreateWithFlags(&w.ev_out[i], cudaEventDisableTiming));
    // occupancy of every body known now (also force-loads their kernels: a lazy module load would
    // synchronise with resident device processes, queues.cu); bodies registered later are asked on first use
    for (int f = 0, n = body_count(); f < n; ++f) {
        const BodyEntry& b = *body_of(f);
        worker_occ(w, f, b, false, false);
        if (b.flags & FBR_BODY_INDEX_ARG) worker_occ(w, f, b, true, false);
    }
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&w.occ_gather, (const void*)gather_ordered_kernel, kThreads, 0));
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&w.occ_fill, (const void*)payload_fill_kernel, kThreads, 0));
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&w.occ_gather_rows, (const void*)gather_rows_kernel, kThreads, 0));
    if (w.occ_gather_rows < 1) w.occ_gather_rows = 1;
    CK(cudaFuncSetAttribute(gather_bulk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bulk::kStages * bulk::kChunk)));
    if (w.occ_gather < 1) w.occ_gather = 1;
    if (w.occ_fill < 1) w.occ_fill = 1;
    // no cudaDeviceSynchronize here: it would wait for resident device processes (queues.cu)
    CK(cudaStreamSynchronize(w.s_comp));
    return FBR_OK;
}

static void worker_destroy(Worker& w) {
    if (w.device < 0) return;
    if (w.dead) {                          // a corrupted context: every call on it fails; its memory goes with the process
        cudaGetLastError();
        w.device = -1;
        return;
    }
    cudaSetDevice(w.device);
    if (w.s_in) cudaStreamSynchronize(w.s_in);
    if (w.s_comp) cudaStreamSynchronize(w.s_comp);
    if (w.s_out) cudaStreamSynchronize(w.s_out);
    if (w.s_gath) { cudaStreamSynchronize(w.s_gath); cudaStreamDestroy(w.s_gath); }
    if (w.s_push) {                        // lives on the root worker's device
        cudaSetDevice(w.push_root_device);
        cudaStreamSynchronize(w.s_push);
        cudaStreamDestroy(w.s_push);
        if (w.s_push2) { cudaStreamSynchronize(w.s_push2); cudaStreamDestroy(w.s_push2); }
        for (int i = 0; i < kRecWindows; ++i) cudaEventDestroy(w.ev_push[i]);
        cudaGetLastError();
        cudaSetDevice(w.device);
        w.s_push = nullptr;
    }
    if (w.s_in) cudaStreamDestroy(w.s_in);
    if (w.s_comp) cudaStreamDestroy(w.s_comp);
    if (w.s_out) cudaStreamDestroy(w.s_out);
    if (w.s_fold) { cudaStreamSynchronize(w.s_fold); cudaStreamDestroy(w.s_fold); }
    cudaFreeHost(w.h_records);
    cudaFree(w.d_records);
    cudaFree(w.d_headers);
    cudaFree(w.d_ring);
    for (int i = 0; i < 2; ++i) {
        cudaFree(w.d_args[i]);
        cudaFree(w.d_items[i]);
        cudaFree(w.d_vals[i]);
        cudaFree(w.d_out[i]);
    }
    cudaFree(w.d_tickets);
    cudaFree(w.d_ctrl);
    cudaFreeHost(w.h_ctrl);
    for (int i = 0; i < kRecWindows; ++i) {
        cudaEventDestroy(w.ev_rec_h2d[i]);
        cudaEventDestroy(w.ev_comp[i]);
        cudaEventDestroy(w.ev_disp[i]);
    }
    for (int i = 0; i < 2; ++i) cudaEventDestroy(w.ev_out[i]);
    w.device = -1;
}

// Claim-unit size: near the body's preferred size, a multiple of the API chunksize when the chunk
// is smaller (so chunk boundaries coincide with unit boundaries), and a multiple of 16/R tasks so
// every full slot is 16 B aligned on both sides of the gather.
//
// Record bodies (FBR_BODY_RECORD): unit_tasks is what one shared-memory stage of dispatch_record_kernel holds, so the
// unit never exceeds it (rounded DOWN to the chunk and alignment multiples), and the alignment is the kernel's
// record::align_tasks(A, R): every full slot AND every unit's argument offset is 16 B aligned, which keeps both sides of
// the unit on the bulk-copy path (R = 12, 24, 40 need 4, 2, 2 tasks; 16/R would not do).
// Chunk boundaries coincide with unit boundaries only while lcm(chunksize, align) fits the stage: pick_unit may grow a
// unit to 2*pref for that, a record unit cannot, so with e.g. chunksize 1023 and align 4 the unit is the stage-sized
// pref and a chunk may straddle two units (which only changes how tasks are grouped, never a result).
static uint32_t gcd_u32(uint32_t a, uint32_t b) { while (b) { const uint32_t t = a % b; a = b; b = t; } return a; }
static uint32_t pick_unit_record(const BodyEntry& b, uint32_t chunksize, uint64_t n_tasks, int sm_count, uint64_t ring_bytes) {
    uint32_t pref = b.unit_tasks;
    if (const char* e = getenv("FBR_UNIT_TASKS")) pref = std::min<uint32_t>(pref, (uint32_t)std::max(16, atoi(e)));
    const uint64_t per_task = std::max(b.result_bytes, b.arg_bytes);
    while (pref > 1 && (uint64_t)pref * per_task > ring_bytes / 2) pref >>= 1;
    while (pref > 256 && (uint64_t)pref * (uint64_t)sm_count > n_tasks) pref >>= 1;
    const uint32_t align = record::align_tasks(b.arg_bytes, b.result_bytes);
    uint32_t unit = pref;
    if (chunksize <= pref) {
        const uint32_t m = chunksize / gcd_u32(chunksize, align) * align;   // lcm(chunksize, align)
        if (m <= pref) unit = pref / m * m;
    }
    unit = std::max(align, unit / align * align);
    // fold maps: a power of two (align is one), so every unit is an aligned subtree of its block's tree()
    if (chunksize == FBR_PLAN_FOLD) while (unit & (unit - 1)) unit &= unit - 1;
    return unit;
}

static uint32_t pick_unit(const BodyEntry& b, uint32_t chunksize, uint64_t n_tasks, int sm_count, uint64_t ring_bytes) {
    if (b.flags & FBR_BODY_RECORD) return pick_unit_record(b, chunksize, n_tasks, sm_count, ring_bytes);
    uint32_t pref = b.unit_tasks;
    if (pref == 1) return 1;
    if (const char* e = getenv("FBR_UNIT_TASKS")) pref = (uint32_t)std::max(16, atoi(e));   // tuning knob (profiles/pi_perf.py)
    // a unit's results (and its argument records) must fit the ring arenas
    const uint64_t per_task = std::max<uint64_t>(std::max(b.result_bytes, b.arg_bytes), 1);
    while (pref > 1 && (uint64_t)pref * per_task > ring_bytes / 2) pref >>= 1;
    // small maps: shrink the unit so the work still spreads over the SMs
    while (pref > 256 && (uint64_t)pref * (uint64_t)sm_count > n_tasks) pref >>= 1;
    const uint32_t align = b.result_bytes < 16 ? 16u / b.result_bytes : 1u;
    uint32_t unit = pref;
    if (chunksize <= pref) {
        uint32_t m = chunksize;  // lcm(chunksize, align)
        while (m % align) m += chunksize;
        if (m <= 2 * pref) unit = std::max(m, pref / m * m);
    }
    unit = (uint32_t)round_up(unit, align);
    while (unit > align && (uint64_t)unit * per_task > ring_bytes) unit -= align;   // chunk-aligned unit too big for the ring
    return unit;
}

// the chunksize a map's units are picked for: a fold map's units ignore it (FBR_PLAN_FOLD)
static uint32_t map_chunksize(const fbr_map_desc_t& d) {
    if (d.flags & (FBR_FOLD | FBR_SCAN | FBR_FOLD_KEYS | FBR_FOLD_SPARSE_KEYS)) return FBR_PLAN_FOLD;   // scan and keyed maps cut blocks as a fold
    return d.chunksize ? d.chunksize : 32u;
}

// The placement of tasks [first, first + count) of map `d` on worker `worker` (BlockPlan).  Pure: no CUDA call, no
// allocation.  host_out: the map has a pinned host result segment; root_alive: worker 0 is alive (it can push arguments);
// item_bytes_per_task: the mean bytes a task's host-resident items and offsets take of a staging half, over every stream.
static BlockPlan plan_block(const BodyEntry& body, const fbr_map_desc_t& d, uint32_t pool_flags, int worker, uint64_t first,
                            uint64_t count, bool host_out, int sm_count, uint64_t ring_bytes, bool root_alive,
                            uint64_t item_bytes_per_task) {
    BlockPlan pl;
    pl.R = body.result_bytes;
    pl.resilient = (d.flags & FBR_RESILIENT) != 0;
    pl.unit = pick_unit(body, map_chunksize(d), count, sm_count, ring_bytes);
    pl.slot_stride = (uint32_t)round_up((uint64_t)pl.unit * pl.R, 16);
    const uint32_t unit = pl.unit, R = pl.R;

    static const bool out_off = getenv("FBR_PEER_OUT") && atoi(getenv("FBR_PEER_OUT")) == 0;
    // Bit-packed bool results are small (1/8 B per task): instead of staging them in HBM and copying them out wave by wave
    // (6 x (2 MB D2H + copy set-up) = the critical path of the e2e step), the dispatch kernel stores them straight into the
    // pinned host segment (ZeroCopy): the PCIe writes spread over the whole kernel (FBR_NO_ZERO_COPY selects Staged).
    const bool zero_copy_ok = body.result_kind == FBR_RES_BITS8 && host_out && !pl.resilient &&
                              !(d.flags & (FBR_FULL_WINDOW | FBR_SHUFFLE | FBR_VIA_RING | FBR_NO_ZERO_COPY));
    if (d.flags & FBR_FOLD) pl.sink = Sink::FoldPartials;
    else if (d.flags & FBR_FOLD_KEYS) pl.sink = Sink::KeyedWindow;
    else if (d.flags & FBR_FOLD_SPARSE_KEYS) pl.sink = Sink::SparseKeyedWindow;
    else if (d.flags & FBR_SCAN) pl.sink = Sink::ScanWindow;
    else if (d.flags & FBR_OUT_DEVICE)
        pl.sink = worker != 0 && !pl.resilient && !out_off && !(d.flags & FBR_FULL_WINDOW) ? Sink::StagedPeer : Sink::CallerDevice;
    else if (d.flags & FBR_RESULTS_ON_DEVICE) pl.sink = Sink::WindowOnDevice;
    else if (zero_copy_ok) pl.sink = Sink::ZeroCopy;
    else if (pl.resilient || (d.flags & FBR_FULL_WINDOW)) pl.sink = Sink::WindowToHost;
    else pl.sink = Sink::Staged;

    static const bool push_off = getenv("FBR_PEER_PUSH") && atoi(getenv("FBR_PEER_PUSH")) == 0;
    if (d.flags & FBR_ARGS_DEVICE)
        pl.args = d.arg_stride != 0 && worker != 0 && !pl.resilient && !push_off && root_alive ? ArgSource::Pushed : ArgSource::DeviceInPlace;
    else if (d.arg_stride == 0) pl.args = ArgSource::None;
    else pl.args = pl.resilient ? ArgSource::Resident : ArgSource::Staged;
    if (d.n_items && d.arg_stride && body.result_kind == FBR_RES_BITS8)
        pl.args_limit_bytes = d.n_items * (uint64_t)(d.arg_stride / 8);   // a byte-task's record is 8 items
    if (body.flags & FBR_BODY_ITEMS)
        pl.items = (d.flags & FBR_ARGS_DEVICE) ? ItemSource::DeviceInPlace : pl.resilient ? ItemSource::Resident : ItemSource::Staged;

    // Opt-in (FBR_POOL_OVERLAP): gather(w) runs on a second, higher-priority stream while the next wave's / next map's
    // dispatch kernel computes; the ring is then used in alternating halves.  On the pi map (ALU-bound dispatch + HBM-bound
    // gather) the gather is a small share of the step and the two kernels contend for SM slots, so it is off by default.
    pl.overlap = !pl.staged() && !pl.resilient && (pool_flags & FBR_POOL_OVERLAP) != 0;
    // Direct placement: a contiguous, unshuffled, non-resilient block needs neither task records nor the ring -- unit t of
    // a wave is tasks [wave_first + t*unit, ...) and its results belong at exactly that index of the ordered window, so the
    // dispatch kernel stores them there and no gather is launched.  (Shuffled arrival, several attempts per unit and
    // FBR_VIA_RING keep the ring + gather path.)
    {
        const bool unit_ok = ((uint64_t)unit * R) % 16 == 0 || unit == 1;   // full vectors are stored 16 B at a time
        const bool base_ok = !(d.flags & FBR_OUT_DEVICE) || (((uintptr_t)d.out + first * R) & 15) == 0;
        pl.direct = !pl.resilient && !(d.flags & (FBR_SHUFFLE | FBR_VIA_RING)) && unit_ok && base_ok;
    }
    // wave capacity in claim units
    uint64_t units_cap = pl.direct ? (1ull << 31) :   // 32-bit unit counter; a direct wave needs no ring space
        std::min<uint64_t>(kRecCapacity, (pl.overlap ? ring_bytes / 2 : ring_bytes) / pl.slot_stride);
    if (pl.args_streamed()) units_cap = std::min<uint64_t>(units_cap, ring_bytes / ((uint64_t)unit * d.arg_stride));
    if (pl.staged()) units_cap = std::min<uint64_t>(units_cap, ring_bytes / ((uint64_t)unit * R));
    pl.wave_tasks_cap = units_cap * unit;
    // Host-resident output: cut large maps into ~8 waves (>= 8 MiB of results each) so the D2H of
    // wave w overlaps the kernels of wave w+1 instead of trailing one monolithic launch.
    if (pl.staged() || pl.args_streamed() || pl.items == ItemSource::Staged) {
        uint64_t bytes_per_task = std::max<uint64_t>(R, pl.args_streamed() ? d.arg_stride : 0);
        if (pl.items == ItemSource::Staged) bytes_per_task = std::max(bytes_per_task, item_bytes_per_task);
        // a wave must carry enough kernel time to hide its launches: 8 MiB of byte results is tens of us of
        // pi dispatch; a byte of bit-packed results stands for 8 tasks, so 1 MiB is the same work
        uint64_t min_wave_bytes = body.result_kind == FBR_RES_BITS8 ? (1ull << 20) : (8ull << 20);
        if (const char* e = getenv("FBR_MIN_WAVE_KB")) min_wave_bytes = std::max<uint64_t>(4096, (uint64_t)atoll(e) << 10);   // tuning knob
        const uint64_t min_wave_tasks = round_up(std::max<uint64_t>(1, min_wave_bytes / bytes_per_task), unit);
        // 8 waves for ~100 MB maps, up to 64 for multi-GB ones (~64 MiB per wave): the first wave's
        // H2D and the last wave's D2H are the only copies nothing overlaps with
        uint64_t n_waves = std::min<uint64_t>(64, std::max<uint64_t>(8, count * bytes_per_task / (64ull << 20)));
        // small outputs (bit-packed bools): per-copy set-up weighs more: T_kernel/n + n * T_setup is flattest at a few waves
        if (body.result_kind == FBR_RES_BITS8 && !pl.args_streamed()) n_waves = 6;
        if (const char* e = getenv("FBR_WAVES")) n_waves = std::max<uint64_t>(1, (uint64_t)atoll(e));                          // tuning knob
        const uint64_t share = round_up((count + n_waves - 1) / n_waves, unit);
        pl.wave_tasks_cap = std::min(pl.wave_tasks_cap, std::max(min_wave_tasks, share));
    }
    pl.redispatch_units_cap = std::max<uint64_t>(1, std::min<uint64_t>(kRecCapacity, ring_bytes / pl.slot_stride));
    pl.sum_kind = (d.flags & FBR_WANT_SUM) ? 1 : 0;   // the dispatch kernel folds sum(results) while they are in registers
    return pl;
}

// Worker i's block [b0, b1) of `count` tasks cut over n_workers: contiguous, in order, whole claim units of the map-level
// unit (every block gets the same number of units, the last ones may get fewer or none).
static void cut_block(const BodyEntry& body, uint32_t chunksize, uint64_t count, int n_workers, int i, int sm_count,
                      uint64_t ring_bytes, uint64_t* b0, uint64_t* b1) {
    const uint32_t unit = pick_unit(body, chunksize, (count + n_workers - 1) / n_workers, sm_count, ring_bytes);
    const uint64_t units_total = (count + unit - 1) / unit;
    const uint64_t units_per = (units_total + n_workers - 1) / n_workers;
    *b0 = std::min<uint64_t>(count, (uint64_t)i * units_per * unit);
    *b1 = std::min<uint64_t>(count, (uint64_t)(i + 1) * units_per * unit);
}

static void shuffle_records(TaskRecord* r, uint32_t n, uint64_t seed) {
    for (uint32_t i = n; i > 1; --i) {
        seed = splitmix64(seed);
        const uint32_t j = (uint32_t)(seed % i);
        std::swap(r[i - 1], r[j]);
    }
}

// ------------------------------------------------------------------------------------------------
// wave pipeline for one worker's block of one map
// ------------------------------------------------------------------------------------------------
// A variable-length stream of a block that travels wave by wave through a worker's two ring_bytes staging halves:
// host-resident items in (d_items: the n item streams of the map share each half), host-staged emit values out (d_vals).
// In a wave's half the n segments follow one another, each starting on a 256 B boundary: its 256 B-rounded header of
// wt + 1 offsets (items), then its data.
struct StagedStream {
    uint32_t n;                                 // segments sharing a half (1, or the K item streams of an items map)
    const uint64_t* offs[kMaxItemStreams];      // host offsets rebased to the block: offs[k][t] belongs to task part.first + t
    uint64_t elem_bytes[kMaxItemStreams];
    bool header;                // the wave's wt + 1 offsets travel ahead of each segment's data, in a 256 B-rounded header
    const char* too_large;      // error for a claim unit no half holds: its tasks [t0, t1), its data bytes, ring_bytes
    uint64_t seg_data(uint32_t k, uint64_t t0, uint64_t t1) const { return (offs[k][t1] - offs[k][t0]) * elem_bytes[k]; }
    uint64_t data_bytes(uint64_t t0, uint64_t t1) const {
        uint64_t b = 0;
        for (uint32_t k = 0; k < n; ++k) b += seg_data(k, t0, t1);
        return b;
    }
    uint64_t header_bytes(uint64_t t0, uint64_t t1) const { return header ? round_up((t1 - t0 + 1) * sizeof(uint64_t), 256) : 0; }
    // where segment k of the wave of tasks [t0, t1) starts in its half
    uint64_t seg_start(uint32_t k, uint64_t t0, uint64_t t1) const {
        uint64_t at = 0;
        for (uint32_t j = 0; j < k; ++j) at = round_up(at + header_bytes(t0, t1) + seg_data(j, t0, t1), 256);
        return at;
    }
    // what tasks [t0, t1) of the block take of a staging half
    uint64_t staged_bytes(uint64_t t0, uint64_t t1) const { return seg_start(n - 1, t0, t1) + header_bytes(t0, t1) + seg_data(n - 1, t0, t1); }
};

// the host-resident item streams of block `part` of an items map, as they are staged
static StagedStream staged_items(const SeqState& st, const SeqPart& part) {
    StagedStream s{st.n_item_streams, {}, {}, true,
                   "the claim unit of tasks [%llu, %llu) carries %llu item bytes, more than a staging half of "
                   "ring_bytes %llu holds with its offsets: raise ring_bytes or split the items"};
    for (uint32_t k = 0; k < s.n; ++k) {
        s.offs[k] = st.items[k].offsets + part.first;
        s.elem_bytes[k] = st.items[k].item_bytes;
    }
    return s;
}

// The most whole units (or the rest of the block) from task `done` on, at most `wt` tasks, whose wave fits one staging half
// in every stream; at least one unit (submit_part checked that each fits).  Binary search over the host offsets.
static uint64_t fit_staged_wave(const std::vector<StagedStream>& streams, uint64_t done, uint64_t wt, uint32_t unit,
                                uint64_t ring_bytes) {
    auto fits = [&](uint64_t tasks) {
        for (const StagedStream& s : streams)
            if (s.staged_bytes(done, done + tasks) > ring_bytes) return false;
        return true;
    };
    uint64_t lo_u = 0, hi_u = (wt + unit - 1) / unit;               // fits(lo_u units) holds (0 tasks always fit)
    while (lo_u < hi_u) {
        const uint64_t mid = (lo_u + hi_u + 1) / 2;
        if (fits(std::min<uint64_t>(mid * unit, wt))) lo_u = mid; else hi_u = mid - 1;
    }
    return std::min<uint64_t>(std::max<uint64_t>(lo_u, 1) * unit, wt);
}

// Grid of a wave's dispatch kernel: `occ` resident CTAs per SM of the body's kernel, at most the body's max_ctas_per_sm,
// one fewer for an overlapped wave (its gather CTAs run beside it), FBR_DISPATCH_OCC at most, no more CTAs than units.
static int dispatch_grid(const BodyEntry& body, int occ, bool overlapped, uint32_t n_units, int sm_count) {
    if (body.max_ctas_per_sm) occ = std::min(occ, body.max_ctas_per_sm);
    if (overlapped && occ > 1) occ -= 1;     // leave SM slots for the concurrently running gather CTAs
    if (const char* e = getenv("FBR_DISPATCH_OCC")) occ = std::max(1, std::min(occ, atoi(e)));
    return (int)std::min<uint64_t>(n_units, (uint64_t)sm_count * occ);
}

// How a wave's results reach their final place (kernels.cuh): the dispatch kernel stores them there itself (Direct), or a
// gather kernel moves them from the ring -- the TMA bulk pipeline (Bulk), row streaming (Rows) or the flat vector loop
// (Flat) -- on `grid` CTAs, Bulk and Rows in ticket groups of `group_slots` slots.
struct GatherChoice { enum Kind { Direct, Flat, Rows, Bulk } kind; int grid; uint32_t group_slots; };

// listed: the wave's units are task records (shuffled, re-dispatched), not its contiguous range; out: its ordered window.
static GatherChoice pick_gather(const BlockPlan& pl, const void* out, uint32_t n_units, bool listed, int sm_count, int occ_gather,
                                int occ_gather_rows) {
    if (pl.direct && !listed) return {GatherChoice::Direct, 0, 0};
    const bool aligned = pl.sink != Sink::FoldPartials && (((uintptr_t)out & 15) == 0) && (((uint64_t)pl.unit * pl.R) == pl.slot_stride);
    const bool rows_ok = aligned && (pl.slot_stride % 4096 == 0);
    const bool bulk_ok = rows_ok && !pl.resilient && pl.slot_stride % bulk::kChunk == 0;   // 4-12 KB slots: the rows kernel
    if (bulk_ok) {
        // ONE warp per SM keeps enough bulk copies in flight to saturate HBM
        int per_sm = 1;
        if (const char* e = getenv("FBR_GATHER_OCC")) per_sm = std::max(1, atoi(e));
        // ~256 KB of ring per ticket (<= 32 slots: one header per lane), >= ~8 tickets per CTA
        const uint64_t max_ctas = (uint64_t)sm_count * per_sm;
        uint32_t group_slots = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(
            std::min<uint64_t>(bulk::kGroup, (256u << 10) / pl.slot_stride), n_units / (8 * max_ctas)));
        if (const char* e = getenv("FBR_BULK_GROUP")) group_slots = std::max(1, std::min(32, atoi(e)));
        const uint32_t n_groups = (n_units + group_slots - 1) / group_slots;
        return {GatherChoice::Bulk, (int)std::min<uint64_t>(n_groups, max_ctas), group_slots};
    }
    if (rows_ok) {
        // ~128 KB of ring per ticket, but never fewer than ~4 tickets per resident CTA (small waves);
        // big slots (>= 32 KB): at most 4 fat streams per SM
        int occ_g = pl.slot_stride >= (32u << 10) ? std::min(occ_gather_rows, 4) : occ_gather_rows;
        if (const char* e = getenv("FBR_GATHER_OCC")) occ_g = std::max(1, std::min(occ_g, atoi(e)));
        const uint64_t max_ctas = (uint64_t)sm_count * occ_g;
        const uint32_t group_slots = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((128u << 10) / pl.slot_stride, n_units / (4 * max_ctas)));
        const uint32_t n_groups = (n_units + group_slots - 1) / group_slots;
        return {GatherChoice::Rows, (int)std::min<uint64_t>(n_groups, max_ctas), group_slots};
    }
    const uint64_t total_vec = (uint64_t)n_units * (pl.slot_stride >> 4);
    return {GatherChoice::Flat, (int)std::max<uint64_t>(1, std::min<uint64_t>((total_vec + kThreads * 4 - 1) / (kThreads * 4),
                                                                              (uint64_t)sm_count * occ_gather)), 0};
}

// One wave: `n_units` claim units -> copy-in, dispatch, gather, (streaming parts) copy-out.
// `wave_first`/`wt` describe the contiguous task window of a regular wave; a re-dispatch wave
// (arbitrary lost units) passes contiguous=false.  `have_records`: the caller wrote the wave's task
// records into the pinned window (shuffled, resilient or re-dispatch waves); otherwise the records
// are an arithmetic progression the kernels compute themselves.
static int run_wave(fbr_pool* p, SeqState& st, SeqPart& part, const BodyEntry& body, uint32_t n_units,
                    uint64_t wave_first, uint64_t wt, bool contiguous, bool have_records, uint64_t wno) {
    Worker& w = p->workers[part.worker];
    const PartCtx& cx = part.cx;
    const BlockPlan& pl = cx.plan;
    const fbr_map_desc_t& d = st.desc;
    const bool timing = (p->flags & FBR_POOL_TIMING) != 0;
    const int rw = (int)(wno % kRecWindows);
    const int half = (int)(wno & 1);
    const int slot = part.ctrl_slot;
    // the ordered output of this wave's window, and the map index of out_window[0]
    uint8_t* const out_window = pl.staged() ? w.d_out[half] : cx.window_base;
    const uint64_t out_first = pl.staged() ? wave_first : part.first;
    const GatherChoice gather = pick_gather(pl, out_window, n_units, !contiguous || have_records, w.sm_count, w.occ_gather,
                                            w.occ_gather_rows);
    const bool direct = gather.kind == GatherChoice::Direct;
    TaskRecord* hrec = w.h_records + (size_t)rw * kRecCapacity;
    TaskRecord* drec = w.d_records + (size_t)rw * kRecCapacity;

    // copy-in stream: wait until the device window / arg half were consumed, then H2D.  A wave that copies
    // nothing in (computed records, range() or device-resident arguments) skips the hop through s_in -- every
    // cross-stream event costs the GPU a few microseconds per wave -- except the first wave of a block, which
    // has to see the control block (and shared block) its submit_part put on s_in.
    const bool in_copies = have_records || pl.args_streamed() || pl.items == ItemSource::Staged || part.first_wave_pending;
    part.first_wave_pending = false;
    if (in_copies) {
        CK(cudaStreamWaitEvent(w.s_in, w.ev_comp[rw], 0));  // wave wno-4 kernels done (device window free)
        if (wno >= 2) CK(cudaStreamWaitEvent(w.s_in, w.ev_comp[(wno - 2) % kRecWindows], 0));  // arg half free
    }
    if (have_records) {
        CK(cudaMemcpyAsync(drec, hrec, sizeof(TaskRecord) * n_units, cudaMemcpyHostToDevice, w.s_in));
        STAT_ADD(p, h2d_bytes, sizeof(TaskRecord) * n_units);
        STAT_ADD(p, records_copied, n_units);
    }
    const uint8_t* wave_args = cx.args_full;
    bool pushed = false;
    if (pl.args_streamed()) {   // streaming arguments (contiguous waves only): from the host, or pushed by the root GPU
        const uint64_t bytes = pl.arg_bytes(wave_first, wt, d.arg_stride);
        const uint8_t* src = (const uint8_t*)d.args + wave_first * (uint64_t)d.arg_stride;
        if (pl.args == ArgSource::Pushed) {
            // The copy runs on a stream of the ROOT device, so the root's copy engine WRITES the wave into this
            // worker's staging half (posted NVLink writes, root TX), while this worker's kernels store their results
            // into the root's output (posted writes, root RX): both directions of the root's links carry payload at
            // the same time and neither carries read requests.  (Peer LOADS + peer stores from one kernel are the
            // FBR_PEER_PUSH=0 variant; see DESIGN.md section 6.)
            if (bytes) {
                CK(cudaSetDevice(w.push_root_device));
                cudaStream_t sp = half ? w.s_push2 : w.s_push;
                cudaError_t e = cudaStreamWaitEvent(sp, w.ev_comp[rw], 0);                 // device window free
                if (e == cudaSuccess && wno >= 2) e = cudaStreamWaitEvent(sp, w.ev_comp[(wno - 2) % kRecWindows], 0);   // staging half free
                if (e == cudaSuccess) e = cudaMemcpyPeerAsync(w.d_args[half], w.device, src, w.push_root_device, bytes, sp);
                if (e == cudaSuccess) e = cudaEventRecord(w.ev_push[rw], sp);
                cudaSetDevice(w.device);
                if (e != cudaSuccess) return fail(FBR_ECUDA, "peer push of wave %llu failed: %s", (unsigned long long)wno, cudaGetErrorString(e));
                pushed = true;
                STAT_ADD(p, peer_push_bytes, bytes);
            }
        } else {
            if (bytes) CK(cudaMemcpyAsync(w.d_args[half], src, bytes, cudaMemcpyHostToDevice, w.s_in));
            STAT_ADD(p, h2d_bytes, bytes);
        }
        wave_args = w.d_args[half];
    }
    // items of a streaming wave, stream by stream in the staging half (StagedStream): its wt + 1 offsets, then its item span
    // one 256 B-rounded header further on
    ItemStream wave_items[kMaxItemStreams];
    std::copy(cx.items, cx.items + kMaxItemStreams, wave_items);
    uint64_t item_first = cx.item_first;
    if (pl.items == ItemSource::Staged) {
        const StagedStream s = staged_items(st, part);
        const uint64_t t0 = wave_first - part.first, t1 = t0 + wt;
        const uint64_t obytes = (wt + 1) * sizeof(uint64_t), hbytes = s.header_bytes(t0, t1);
        for (uint32_t k = 0; k < s.n; ++k) {
            const fbr_items_desc_t& it = st.items[k];
            const uint64_t lo = it.offsets[wave_first], hi = it.offsets[wave_first + wt];
            const uint64_t at = s.seg_start(k, t0, t1), ibytes = s.seg_data(k, t0, t1);
            CK(cudaMemcpyAsync(w.d_items[half] + at, it.offsets + wave_first, obytes, cudaMemcpyHostToDevice, w.s_in));
            if (ibytes)
                CK(cudaMemcpyAsync(w.d_items[half] + at + hbytes, (const uint8_t*)it.items + lo * it.item_bytes, ibytes, cudaMemcpyHostToDevice, w.s_in));
            STAT_ADD(p, h2d_bytes, obytes + ibytes);
            wave_items[k] = ItemStream{w.d_items[half] + at + hbytes, (const uint64_t*)(w.d_items[half] + at), lo, hi};
        }
        item_first = wave_first;
    }
    if (in_copies) CK(cudaEventRecord(w.ev_rec_h2d[rw], w.s_in));

    // compute streams: dispatch on s_comp; gather on s_comp too, or -- overlapped waves -- on the
    // higher-priority s_gath so that it runs while the next wave's dispatch kernel computes.
    // Overlapped waves use alternating halves of the ring / header array.  Direct waves use neither.
    const bool ov = pl.overlap && !direct;
    cudaStream_t s_g = ov ? w.s_gath : w.s_comp;
    uint8_t* ring_base = ov ? w.d_ring + (size_t)half * (p->ring_bytes / 2) : w.d_ring;
    SlotHeader* hdr_base = ov ? w.d_headers + (size_t)half * kRecCapacity : w.d_headers;
    if (in_copies) CK(cudaStreamWaitEvent(w.s_comp, w.ev_rec_h2d[rw], 0));
    if (pushed) CK(cudaStreamWaitEvent(w.s_comp, w.ev_push[rw], 0));
    // the ring region this dispatch writes must have been drained by the gather that last read it (gathers on
    // s_comp itself are ordered by the stream: only a gather that ran on s_gath needs the event)
    if ((w.gath_hist & 3u) || ov) {
        if (wno >= 1 && !(ov && w.prev_wave_overlap)) CK(cudaStreamWaitEvent(w.s_comp, w.ev_comp[(wno - 1) % kRecWindows], 0));
        if (wno >= 2) CK(cudaStreamWaitEvent(w.s_comp, w.ev_comp[(wno - 2) % kRecWindows], 0));
    }
    w.prev_wave_overlap = ov;
    w.gath_hist = ((w.gath_hist << 1) | (ov ? 1u : 0u)) & 3u;
    if (pl.staged()) CK(cudaStreamWaitEvent(w.s_comp, w.ev_out[half], 0));  // out half drained
    WaveParams wp;
    memset(&wp, 0, sizeof wp);
    wp.records = have_records ? drec : nullptr;
    wp.headers = direct ? nullptr : hdr_base;
    wp.ring = direct ? out_window + (wave_first - out_first) * pl.R : ring_base;
    wp.ticket = w.d_tickets + (wno % kTickets);
    wp.n_units = n_units;
    wp.slot_stride = direct ? pl.unit * pl.R : pl.slot_stride;
    wp.args = wave_args;
    wp.arg_stride = d.arg_stride;
    wp.index_start = d.index_start;
    wp.index_step = d.index_step;
    wp.index_base = d.task_index_base;
    wp.shared = cx.d_shared;
    wp.shared_bytes = d.shared_bytes;
    wp.err_word = &w.d_ctrl[slot].err;
    wp.resilient = pl.resilient ? 1u : 0u;
    wp.sum = pl.sum_kind ? &w.d_ctrl[slot].sum : nullptr;
    wp.sum_hi = pl.sum_kind ? &w.d_ctrl[slot].sum_hi : nullptr;
    wp.syn_first = wave_first;
    wp.syn_tasks = wt;
    wp.syn_arg_off = pl.args_streamed() ? 0 : wave_first * (uint64_t)d.arg_stride;
    wp.syn_unit = pl.unit;
    wp.syn_seq = (uint32_t)st.seq;
    wp.syn_func = (uint32_t)st.func_id;
    wp.syn_attempt = part.attempt;
    wp.n_items = d.n_items ? d.n_items : ~0ull;
    wp.items = wave_items[0].items;
    wp.item_offs = wave_items[0].offs;
    wp.item_first = item_first;
    wp.item_base = wave_items[0].base;
    wp.item_count = wave_items[0].count;
    for (uint32_t k = 1; k < st.n_item_streams; ++k) wp.more_items[k - 1] = wave_items[k];
    const EmitBlock& emit = part.emit;
    uint64_t v_lo = 0, v_hi = 0;            // staged emit waves: the wave's span of the block's values
    if (emit.d_offs) {
        wp.emit_offs = emit.d_offs;
        wp.emit_first = part.first;
        wp.emit_base = emit.base;
        if (emit.h_offs) {
            v_lo = emit.h_offs[wave_first - part.first];
            v_hi = emit.h_offs[wave_first - part.first + wt];
            wp.emit_values = w.d_vals[half] - v_lo * body.out_bytes;     // the wave's first value lands at d_vals[half]
        } else {
            wp.emit_values = (uint8_t*)emit.d_values;
        }
    }
    const bool fold = pl.sink == Sink::FoldPartials;
    if (fold) {   // no unit stores results: each writes its tree to its place in d_fold
        wp.ring = nullptr;
        wp.fold_partials = (uint8_t*)part.d_fold;
        wp.fold_first = part.first;
    }
    const int grid_d = dispatch_grid(body, worker_occ(w, st.func_id, body, d.arg_stride == 0, fold), ov, n_units, w.sm_count);
    TimedPair td{nullptr, nullptr}, tg{nullptr, nullptr};
    if (timing) {
        CK(cudaEventCreate(&td.a)); CK(cudaEventCreate(&td.b));
        CK(cudaEventRecord(td.a, w.s_comp));
    }
    body.launch(&wp, grid_d, (void*)w.s_comp);
    CK(cudaGetLastError());
    if (timing) {
        CK(cudaEventRecord(td.b, w.s_comp));
        part.t_dispatch.push_back(td);
    }
    STAT_ADD(p, dispatch_launches, 1);
    STAT_ADD(p, units_dispatched, n_units);
    STAT_ADD(p, dispatch_bytes, wt * ((uint64_t)(d.arg_stride ? body.arg_bytes : 0) + pl.R));

    if (direct) {
        STAT_ADD(p, direct_waves, 1);
        CK(cudaEventRecord(w.ev_comp[rw], w.s_comp));
    } else {
        if (ov) {
            CK(cudaEventRecord(w.ev_disp[rw], w.s_comp));
            CK(cudaStreamWaitEvent(s_g, w.ev_disp[rw], 0));
        }
        if (timing) {
            CK(cudaEventCreate(&tg.a)); CK(cudaEventCreate(&tg.b));
            CK(cudaEventRecord(tg.a, s_g));
        }
        GatherParams gp;
        gp.headers = hdr_base;
        gp.ring = ring_base;
        gp.n_units = n_units;
        gp.slot_stride = fold ? 0u : pl.slot_stride;   // a fold wave's gather moves no payload, it only lists lost units
        gp.result_bytes = pl.R;
        gp.pad = 0;
        gp.out = out_window;
        gp.win_first = out_first;
        gp.ticket_to_reset = nullptr;     // dispatch kernels re-arm their own ticket (TicketClaimer::rearm)
        gp.lost_count = pl.resilient ? &w.d_ctrl[slot].lost_count : nullptr;
        gp.lost_units = part.d_lost;
        gp.lost_capacity = part.lost_cap;
        uint32_t* gticket = w.d_tickets + kTickets + (wno % kTickets);   // zero at launch, re-armed below
        if (gather.kind == GatherChoice::Bulk) {
            gather_bulk_kernel<<<gather.grid, 32, (size_t)bulk::kStages * bulk::kChunk, s_g>>>(gp, gticket, gather.group_slots);
            CK(cudaMemsetAsync(gticket, 0, sizeof(uint32_t), s_g));
        } else if (gather.kind == GatherChoice::Rows) {
            // newest slots first (see the kernel): the ring's most recently written part is still in the L2.  On the H100
            // (50 MB L2) this costs nothing for waves that fit the L2 and gains for larger ones -- 8-9 % at 95 MB, 4 % at
            // 190 MB per wave (profiles/r03_gather_order.txt) -- so it is the order at every size.
            gather_rows_kernel<<<gather.grid, kThreads, 0, s_g>>>(gp, gticket, gather.group_slots);
            CK(cudaMemsetAsync(gticket, 0, sizeof(uint32_t), s_g));
        } else {
            gather_ordered_kernel<<<gather.grid, kThreads, 0, s_g>>>(gp);
        }
        CK(cudaGetLastError());
        if (timing) {
            CK(cudaEventRecord(tg.b, s_g));
            part.t_gather.push_back(tg);
        }
        CK(cudaEventRecord(w.ev_comp[rw], s_g));
        STAT_ADD(p, gather_launches, 1);
        STAT_ADD(p, gather_bytes, 2 * wt * pl.R);
    }

    // copy-out stream (streaming parts): D2H of the ordered window of this wave
    if (contiguous) {
        cudaEvent_t wd;
        CK(cudaEventCreateWithFlags(&wd, cudaEventDisableTiming));
        if (pl.staged()) {
            CK(cudaStreamWaitEvent(w.s_out, w.ev_comp[rw], 0));
            if (pl.sink == Sink::StagedPeer) {      // this worker's copy engine writes the wave into the root's ordered output (posted NVLink writes)
                CK(cudaMemcpyPeerAsync((uint8_t*)st.out + wave_first * pl.R, p->workers[0].device, w.d_out[half], w.device, wt * pl.R, w.s_out));
                STAT_ADD(p, peer_push_bytes, wt * pl.R);
            } else {
                CK(cudaMemcpyAsync((uint8_t*)st.out + wave_first * pl.R, w.d_out[half], wt * pl.R, cudaMemcpyDeviceToHost, w.s_out));
                STAT_ADD(p, d2h_bytes, wt * pl.R);
            }
            if (v_hi > v_lo) {   // the wave's values, exactly its span, into the pinned segment
                const uint64_t ob = body.out_bytes;
                CK(cudaMemcpyAsync(emit.host + v_lo * ob, w.d_vals[half], (v_hi - v_lo) * ob, cudaMemcpyDeviceToHost, w.s_out));
                STAT_ADD(p, d2h_bytes, (v_hi - v_lo) * ob);
            }
            CK(cudaEventRecord(w.ev_out[half], w.s_out));
            CK(cudaEventRecord(wd, w.s_out));
        } else {
            CK(cudaEventRecord(wd, direct ? w.s_comp : s_g));
        }
        part.wave_done.push_back(wd);
    }
    __atomic_fetch_add(&st.n_waves, 1u, __ATOMIC_RELAXED);
    return FBR_OK;
}

// FBR_FOLD_KEYS, a block's last round, queued on its worker's s_out behind its last wave: the body's keys entry writes each
// task's key (a bad one goes into the block's error word), a stable LSD radix sort of (key, task) pairs puts the block's
// tasks in key order, the records are gathered into that order, key_offsets_kernel finds each key's run and count, and the
// body's fold_segments entry folds every run into the key's total.  Totals and counts are then copied into the block's area
// of the pinned segment.  With one key nothing is sorted or gathered: the window is folded in place.  Device scratch, all
// stream-ordered: 4 B per task of keys (16 B with a sort: keys and task indices, twice), a gathered copy of the window with
// a sort, the sort's (digit, tile) histogram and its scan (16 B per 256 bins per 4096 tasks), and n_keys * (R + 16) bytes.
static int fold_block_by_key(fbr_pool* p, SeqState& st, SeqPart& part) {
    Worker& w = p->workers[part.worker];
    const BodyEntry& body = *body_of(st.func_id);
    const PartCtx& cx = part.cx;
    const cudaStream_t s = w.s_out;
    const uint32_t K = st.desc.n_keys, n = (uint32_t)part.count;
    const uint64_t R = body.result_bytes;
    const int passes = K <= 1 ? 0 : K <= 256 ? 1 : 2;   // 8-bit digits of keys below K
    const uint32_t n_tiles = (n + keyed::kTile - 1) / keyed::kTile;
    const uint64_t H = (uint64_t)keyed::kBins * n_tiles, scan_tiles = H / scan::kTile + 1;
    uint64_t at = 0;
    auto take = [&](uint64_t bytes) { const uint64_t o = at; at = round_up(at + bytes, 256); return o; };
    const uint64_t o_keys0 = take(4ull * n), o_keys1 = passes ? take(4ull * n) : 0, o_idx0 = passes ? take(4ull * n) : 0,
                   o_idx1 = passes ? take(4ull * n) : 0, o_hist = passes ? take(8 * H) : 0, o_hoffs = passes ? take(8 * (H + 1)) : 0,
                   o_state = passes ? take(8 * (scan_tiles + 2)) : 0, o_gather = passes ? take(n * R) : 0;
    const uint64_t o_offs = take(8ull * (K + 1)), o_counts = take(8ull * K), o_totals = take(K * R);
    uint8_t* buf = nullptr;
    cudaError_t e = cudaMallocAsync((void**)&buf, at, s);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(e == cudaErrorMemoryAllocation ? FBR_ENOMEM : FBR_ECUDA, "keyed fold of body %s on worker %d: %llu bytes of device scratch: %s",
                    body.name.c_str(), part.worker, (unsigned long long)at, cudaGetErrorString(e));
    }
    uint32_t* keys[2] = {(uint32_t*)(buf + o_keys0), (uint32_t*)(buf + o_keys1)};
    uint32_t* idx[2] = {(uint32_t*)(buf + o_idx0), (uint32_t*)(buf + o_idx1)};
    uint64_t* const hist = (uint64_t*)(buf + o_hist);
    uint64_t* const hoffs = (uint64_t*)(buf + o_hoffs);
    uint64_t* const state = (uint64_t*)(buf + o_state);   // scan_counts_kernel: tile states, ticket, total
    uint64_t* const offs = (uint64_t*)(buf + o_offs);
    e = (cudaError_t)body.keys(cx.window_base, n, K, st.desc.task_index_base + part.first, keys[0], &w.d_ctrl[part.ctrl_slot].err, (void*)s);
    const unsigned sort_grid = (unsigned)std::min<uint32_t>(n_tiles, 1u << 16);
    int cur = 0;
    for (int pass = 0; pass < passes && e == cudaSuccess; ++pass, cur ^= 1) {
        radix_hist_kernel<<<sort_grid, keyed::kThreads, 0, s>>>(keys[cur], n, 8 * pass, hist, n_tiles);
        e = cudaMemsetAsync(state, 0, 8 * (scan_tiles + 2), s);
        if (e != cudaSuccess) break;
        scan_counts_kernel<<<(unsigned)scan_tiles, scan::kThreads, 0, s>>>(hist, H, hoffs, (unsigned long long*)state,
                                                                          (uint32_t*)(state + scan_tiles), state + scan_tiles + 1);
        radix_scatter_kernel<<<sort_grid, keyed::kThreads, 0, s>>>(keys[cur], pass ? idx[cur] : nullptr, keys[cur ^ 1], idx[cur ^ 1], n,
                                                                   8 * pass, hoffs, n_tiles);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        key_offsets_kernel<<<(unsigned)std::min<uint64_t>((K + kThreads) / kThreads, 1024), kThreads, 0, s>>>(
            keys[cur], n, K, offs, (uint64_t*)(buf + o_counts));
        e = cudaGetLastError();
    }
    uint8_t* src = cx.window_base;
    if (e == cudaSuccess && passes) {
        src = buf + o_gather;
        const uint32_t W = R % 16 == 0 ? 16 : R % 8 == 0 ? 8 : 4;
        const uint64_t words = R / W, grid = std::min<uint64_t>((n * words + kThreads - 1) / kThreads, 1u << 16);
        if (W == 16) gather_records_kernel<uint4><<<(unsigned)grid, kThreads, 0, s>>>((const uint4*)cx.window_base, (uint4*)src, idx[cur], n, (uint32_t)words);
        else if (W == 8) gather_records_kernel<uint2><<<(unsigned)grid, kThreads, 0, s>>>((const uint2*)cx.window_base, (uint2*)src, idx[cur], n, (uint32_t)words);
        else gather_records_kernel<uint32_t><<<(unsigned)grid, kThreads, 0, s>>>((const uint32_t*)cx.window_base, (uint32_t*)src, idx[cur], n, (uint32_t)words);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = (cudaError_t)body.fold_segments(src, n, offs, K, buf + o_totals, (void*)s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(cx.key_totals, buf + o_totals, K * R, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(cx.key_counts, buf + o_counts, 8ull * K, cudaMemcpyDeviceToHost, s);
    cudaFreeAsync(buf, s);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(FBR_ECUDA, "keyed fold of body %s on worker %d: %s", body.name.c_str(), part.worker, cudaGetErrorString(e));
    }
    STAT_ADD(p, d2h_bytes, K * (R + 8));
    return FBR_OK;
}

// Where a sparse keyed block keeps its gathered records (at 0), run starts (n + 1 words) and keys (n words) in d_sparse.
static uint64_t sparse_keep_layout(uint64_t n, uint64_t R, uint64_t* o_starts, uint64_t* o_keys) {
    *o_starts = round_up(n * R, 256);
    *o_keys = round_up(*o_starts + 8 * (n + 1), 256);
    return *o_keys + 4 * n;
}

// FBR_FOLD_SPARSE_KEYS, a block's last round, queued on its worker's s_out behind its last wave: the body's keys entry with
// n_keys = 0xFFFFFFFF writes each task's key (the reserved key goes into the block's error word), four LSD radix passes sort
// the (key, task) pairs -- always four: which digits a block uses is not known on the host without a synchronisation -- and
// the records are gathered into key order.  run_heads_kernel flags each run of equal keys, the scan of the flags numbers the
// runs and writes D, their number, into the block's pinned word, and run_starts_kernel writes each run's start and key.  The
// window and the sort's scratch (about 40 B per task) are freed here; the gathered records, starts and keys stay in
// part.d_sparse until sparse_keyed_finish folds the runs, since D is known on the host only then.
static int sparse_block_step(fbr_pool* p, SeqState& st, SeqPart& part) {
    Worker& w = p->workers[part.worker];
    const BodyEntry& body = *body_of(st.func_id);
    const PartCtx& cx = part.cx;
    const cudaStream_t s = w.s_out;
    const uint32_t n = (uint32_t)part.count;
    const uint64_t R = body.result_bytes;
    const uint32_t n_tiles = (n + keyed::kTile - 1) / keyed::kTile;
    const uint64_t H = (uint64_t)keyed::kBins * n_tiles, scan_tiles = H / scan::kTile + 1, run_tiles = n / scan::kTile + 1;
    uint64_t at = 0;
    auto take = [&](uint64_t bytes) { const uint64_t o = at; at = round_up(at + bytes, 256); return o; };
    const uint64_t o_keys0 = take(4ull * n), o_keys1 = take(4ull * n), o_idx0 = take(4ull * n), o_idx1 = take(4ull * n),
                   o_hist = take(8 * H), o_hoffs = take(8 * (H + 1)), o_state = take(8 * (scan_tiles + 2)),
                   o_head = take(8ull * n), o_run = take(8ull * (n + 1)), o_rstate = take(8 * (run_tiles + 2));
    uint64_t o_starts, o_dkeys;
    const uint64_t keep_bytes = sparse_keep_layout(n, R, &o_starts, &o_dkeys);
    uint8_t *buf = nullptr, *keep = nullptr;
    cudaError_t e = cudaMallocAsync((void**)&buf, at, s);
    if (e == cudaSuccess) e = cudaMallocAsync((void**)&keep, keep_bytes, s);
    if (e != cudaSuccess) {
        if (buf) cudaFreeAsync(buf, s);
        cudaGetLastError();
        return fail(e == cudaErrorMemoryAllocation ? FBR_ENOMEM : FBR_ECUDA, "sparse keyed fold of body %s on worker %d: %llu bytes "
                    "of device memory: %s", body.name.c_str(), part.worker, (unsigned long long)(at + keep_bytes), cudaGetErrorString(e));
    }
    part.d_sparse = keep;
    uint32_t* keys[2] = {(uint32_t*)(buf + o_keys0), (uint32_t*)(buf + o_keys1)};
    uint32_t* idx[2] = {(uint32_t*)(buf + o_idx0), (uint32_t*)(buf + o_idx1)};
    uint64_t* const hist = (uint64_t*)(buf + o_hist);
    uint64_t* const hoffs = (uint64_t*)(buf + o_hoffs);
    uint64_t* const state = (uint64_t*)(buf + o_state);   // scan_counts_kernel: tile states, ticket, total
    uint64_t* const head = (uint64_t*)(buf + o_head);
    uint64_t* const run = (uint64_t*)(buf + o_run);
    uint64_t* const rstate = (uint64_t*)(buf + o_rstate);
    e = (cudaError_t)body.keys(cx.window_base, n, 0xFFFFFFFFu, st.desc.task_index_base + part.first, keys[0],
                               &w.d_ctrl[part.ctrl_slot].err, (void*)s);
    const unsigned sort_grid = (unsigned)std::min<uint32_t>(n_tiles, 1u << 16);
    int cur = 0;
    for (int pass = 0; pass < 4 && e == cudaSuccess; ++pass, cur ^= 1) {
        radix_hist_kernel<<<sort_grid, keyed::kThreads, 0, s>>>(keys[cur], n, 8 * pass, hist, n_tiles);
        e = cudaMemsetAsync(state, 0, 8 * (scan_tiles + 2), s);
        if (e != cudaSuccess) break;
        scan_counts_kernel<<<(unsigned)scan_tiles, scan::kThreads, 0, s>>>(hist, H, hoffs, (unsigned long long*)state,
                                                                          (uint32_t*)(state + scan_tiles), state + scan_tiles + 1);
        radix_scatter_kernel<<<sort_grid, keyed::kThreads, 0, s>>>(keys[cur], pass ? idx[cur] : nullptr, keys[cur ^ 1], idx[cur ^ 1], n,
                                                                   8 * pass, hoffs, n_tiles);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        const uint32_t W = R % 16 == 0 ? 16 : R % 8 == 0 ? 8 : 4;
        const uint64_t words = R / W, grid = std::min<uint64_t>((n * words + kThreads - 1) / kThreads, 1u << 16);
        if (W == 16) gather_records_kernel<uint4><<<(unsigned)grid, kThreads, 0, s>>>((const uint4*)cx.window_base, (uint4*)keep, idx[cur], n, (uint32_t)words);
        else if (W == 8) gather_records_kernel<uint2><<<(unsigned)grid, kThreads, 0, s>>>((const uint2*)cx.window_base, (uint2*)keep, idx[cur], n, (uint32_t)words);
        else gather_records_kernel<uint32_t><<<(unsigned)grid, kThreads, 0, s>>>((const uint32_t*)cx.window_base, (uint32_t*)keep, idx[cur], n, (uint32_t)words);
        const unsigned grid_n = (unsigned)std::min<uint64_t>(((uint64_t)n + kThreads - 1) / kThreads, 1u << 16);
        run_heads_kernel<<<grid_n, kThreads, 0, s>>>(keys[cur], n, head);
        e = cudaMemsetAsync(rstate, 0, 8 * (run_tiles + 2), s);
        if (e == cudaSuccess) {
            scan_counts_kernel<<<(unsigned)run_tiles, scan::kThreads, 0, s>>>(head, n, run, (unsigned long long*)rstate,
                                                                             (uint32_t*)(rstate + run_tiles), cx.n_groups);
            run_starts_kernel<<<grid_n, kThreads, 0, s>>>(keys[cur], n, run, (uint64_t*)(keep + o_starts), (uint32_t*)(keep + o_dkeys));
            e = cudaGetLastError();
        }
    }
    cudaFreeAsync(buf, s);
    cudaFreeAsync(part.d_window, s);   // the window never leaves the device: the gathered copy replaces it
    part.d_window = nullptr;
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(FBR_ECUDA, "sparse keyed fold of body %s on worker %d: %s", body.name.c_str(), part.worker, cudaGetErrorString(e));
    }
    return FBR_OK;
}

// Control block (+ lost list) back to the pinned mirror, completion event.
static int finish_round(fbr_pool* p, SeqState& st, SeqPart& part, bool copy_window) {
    Worker& w = p->workers[part.worker];
    const PartCtx& cx = part.cx;
    const int slot = part.ctrl_slot;
    const int last_rw = (int)((w.wave_no - 1) % kRecWindows);
    // Every block finishes on s_out, behind its copy-outs, even one without any: finishing on the compute stream puts a
    // DMA hop between back-to-back kernels of pipelined maps, which costs them what a blocking map() gains.
    CK(cudaStreamWaitEvent(w.s_out, w.ev_comp[last_rw], 0));
    const BlockPlan& pl = cx.plan;
    if (copy_window && part.count) {   // the last round
        bool to_host = pl.sink == Sink::WindowToHost;
        if (pl.sink == Sink::ScanWindow) {   // the block's own prefix folds, in place in its window
            const cudaError_t e = (cudaError_t)body_of(st.func_id)->scan(cx.window_base, part.count, 1, nullptr, 0, (void*)w.s_out);
            if (e != cudaSuccess) return fail(FBR_ECUDA, "scan of body %s on worker %d: %s", body_of(st.func_id)->name.c_str(),
                                              part.worker, cudaGetErrorString(e));
            // a scan block after the first keeps its window on the device: scan_finish wraps it there, then copies it out once
            to_host = part.first == 0 && !(st.flags & FBR_RESULTS_ON_DEVICE);
        }
        if (to_host) {
            CK(cudaMemcpyAsync((uint8_t*)st.out + part.first * pl.R, cx.window_base, part.count * pl.R, cudaMemcpyDeviceToHost, w.s_out));
            STAT_ADD(p, d2h_bytes, part.count * pl.R);
        }
        if (pl.sink == Sink::FoldPartials) {   // the block's total from its units' partials
            body_of(st.func_id)->fold(part.d_fold, (part.count + pl.unit - 1) / pl.unit, cx.fold_total, (void*)w.s_out);
            CK(cudaGetLastError());
        }
        if (pl.sink == Sink::KeyedWindow) {
            const int rc = fold_block_by_key(p, st, part);
            if (rc != FBR_OK) return rc;
        }
        if (pl.sink == Sink::SparseKeyedWindow) {
            const int rc = sparse_block_step(p, st, part);
            if (rc != FBR_OK) return rc;
        }
    }
    const EmitBlock& e = part.emit;
    if (copy_window && e.host && e.d_values && e.total) {
        const uint64_t vbytes = e.total * body_of(st.func_id)->out_bytes;
        CK(cudaMemcpyAsync(e.host, e.d_values, vbytes, cudaMemcpyDeviceToHost, w.s_out));
        STAT_ADD(p, d2h_bytes, vbytes);
    }
    CK(cudaMemcpyAsync(&w.h_ctrl[slot], &w.d_ctrl[slot], sizeof(SeqCtrl), cudaMemcpyDeviceToHost, w.s_out));
    if (pl.resilient && part.lost_cap)
        CK(cudaMemcpyAsync(part.h_lost, part.d_lost, sizeof(LostUnit) * part.lost_cap, cudaMemcpyDeviceToHost, w.s_out));
    // one event per part for its whole life, re-recorded every round: another waiter may hold the handle
    // (fbr_result_wait blocks on it outside the pool lock), so it must never be destroyed under it
    if (!part.done) CK(cudaEventCreateWithFlags(&part.done, cudaEventDisableTiming));
    CK(cudaEventRecord(part.done, w.s_out));
    return FBR_OK;
}

static int submit_part(fbr_pool* p, SeqState& st, SeqPart& part, const BodyEntry& body) {
    Worker& w = p->workers[part.worker];
    const fbr_map_desc_t& d = st.desc;
    PartCtx& cx = part.cx;
    CK(cudaSetDevice(w.device));
    uint64_t item_bytes_per_task = 0;   // host-resident items: the mean item bytes and offsets of a task, over every stream
    if ((body.flags & FBR_BODY_ITEMS) && !(d.flags & FBR_ARGS_DEVICE) && part.count) {
        const StagedStream s = staged_items(st, part);
        item_bytes_per_task = s.data_bytes(0, part.count) / part.count + s.n * sizeof(uint64_t);
    }
    cx.plan = plan_block(body, d, p->flags, part.worker, part.first, part.count, st.out != nullptr, w.sm_count, p->ring_bytes,
                         !p->workers[0].dead, item_bytes_per_task);
    const BlockPlan& pl = cx.plan;
    if (pl.args == ArgSource::Pushed && w.s_push == nullptr) {
        const int root = p->workers[0].device;
        CK(cudaSetDevice(root));
        cudaError_t e = cudaStreamCreateWithFlags(&w.s_push, cudaStreamNonBlocking);
        if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&w.s_push2, cudaStreamNonBlocking);
        for (int i = 0; i < kRecWindows && e == cudaSuccess; ++i) e = cudaEventCreateWithFlags(&w.ev_push[i], cudaEventDisableTiming);
        cudaSetDevice(w.device);
        if (e != cudaSuccess) return fail(FBR_ECUDA, "creating the push stream on device %d failed: %s", root, cudaGetErrorString(e));
        w.push_root_device = root;
    }
    const uint32_t unit = pl.unit, R = pl.R;
    if ((body.flags & FBR_BODY_RECORD) && unit > body.unit_tasks)   // a unit must fit the kernel's shared-memory stage
        return fail(FBR_EINVAL, "record body %s: a claim unit of %u tasks exceeds its stage of %u", body.name.c_str(), unit, body.unit_tasks);

    // control block
    if (w.ctrl_free.empty()) return fail(FBR_ENOMEM, "more than %d maps in flight on worker %d", kCtrlSlots, part.worker);
    const int slot = w.ctrl_free.back();
    w.ctrl_free.pop_back();
    part.ctrl_slot = slot;
    CK(cudaMemcpyAsync(&w.d_ctrl[slot], &w.h_ctrl[kCtrlSlots], sizeof(SeqCtrl), cudaMemcpyHostToDevice, w.s_in));

    // shared (broadcast) block: with FBR_ARGS_DEVICE, d.shared is a device pointer too
    if (d.shared != nullptr && d.shared_bytes) {
        const bool dev_block = (d.flags & FBR_ARGS_DEVICE) != 0;
        if (d.flags & FBR_SHARED_HANDLE) {
            auto it = p->shared.find((uint64_t)(uintptr_t)d.shared);
            if (it == p->shared.end()) return fail(FBR_ENOENT, "unknown shared handle");
            cx.d_shared = (const uint8_t*)it->second.d_ptr[part.worker];
        } else if (dev_block && !((uintptr_t)d.shared & 15)) {
            cx.d_shared = (const uint8_t*)d.shared;
        } else if (dev_block && (body.flags & FBR_BODY_BROADCAST) && d.shared_bytes <= body.shared_stage_bytes) {
            // staged: the kernel copies whatever is not 16 B aligned into shared memory by hand
            cx.d_shared = (const uint8_t*)d.shared;
        } else if (dev_block) {
            // a caller's device block at a base that is not 16 B aligned, read in place by the kernel: a body may load its
            // elements as 8 or 16 B vectors (an alignas(16) struct, doubles), which would fault there.  Read an aligned copy.
            CK(cudaMallocAsync(&part.d_shared_tmp, d.shared_bytes, w.s_in));
            CK(cudaMemcpyAsync(part.d_shared_tmp, d.shared, d.shared_bytes, cudaMemcpyDefault, w.s_in));
            cx.d_shared = (const uint8_t*)part.d_shared_tmp;
        } else {
            CK(cudaMallocAsync(&part.d_shared_tmp, d.shared_bytes, w.s_in));
            CK(cudaMemcpyAsync(part.d_shared_tmp, d.shared, d.shared_bytes, cudaMemcpyHostToDevice, w.s_in));
            STAT_ADD(p, h2d_bytes, d.shared_bytes);
            cx.d_shared = (const uint8_t*)part.d_shared_tmp;
        }
    }

    // arguments that stay device-resident for the whole map
    if (pl.args == ArgSource::DeviceInPlace) {
        cx.args_full = (const uint8_t*)d.args;
    } else if (pl.args == ArgSource::Resident) {
        // lost units may be re-dispatched at any time: keep every argument record on the device
        CK(cudaMallocAsync(&part.d_args_full, std::max<uint64_t>(16, st.n_tasks * (uint64_t)d.arg_stride), w.s_in));
        const uint64_t abytes = pl.arg_bytes(part.first, part.count, d.arg_stride);
        if (abytes)
            CK(cudaMemcpyAsync((uint8_t*)part.d_args_full + part.first * (uint64_t)d.arg_stride,
                               (const uint8_t*)d.args + part.first * (uint64_t)d.arg_stride, abytes, cudaMemcpyHostToDevice, w.s_in));
        STAT_ADD(p, h2d_bytes, abytes);
        cx.args_full = (const uint8_t*)part.d_args_full;
    }

    // items: device-resident ones are read in place.  Host-resident ones (offsets checked by fbr_map_submit_items) stream
    // wave by wave through the worker's d_items staging halves (run_wave); a resilient map may re-dispatch any unit at
    // any time, so it copies its part's whole item span and count + 1 offsets to the device once, like d_args_full
    if (pl.items == ItemSource::DeviceInPlace) {
        for (uint32_t k = 0; k < st.n_item_streams; ++k) {
            const fbr_items_desc_t& it = st.items[k];
            cx.items[k] = ItemStream{(const uint8_t*)it.items, it.offsets, 0, it.n_items};
        }
        cx.item_first = 0;
    } else if (pl.items == ItemSource::Staged) {
        for (int i = 0; i < 2; ++i)
            if (!w.d_items[i]) CK(cudaMalloc((void**)&w.d_items[i], p->ring_bytes));
    } else if (pl.items == ItemSource::Resident) {
        for (uint32_t k = 0; k < st.n_item_streams; ++k) {
            const fbr_items_desc_t& it = st.items[k];
            const uint64_t lo = it.offsets[part.first], hi = it.offsets[part.first + part.count];
            const uint64_t ibytes = (hi - lo) * it.item_bytes, obytes = (part.count + 1) * sizeof(uint64_t);
            CK(cudaMallocAsync(&part.d_items[k], std::max<uint64_t>(16, ibytes), w.s_in));
            CK(cudaMallocAsync(&part.d_item_offs[k], obytes, w.s_in));
            if (ibytes) CK(cudaMemcpyAsync(part.d_items[k], (const uint8_t*)it.items + lo * it.item_bytes, ibytes, cudaMemcpyHostToDevice, w.s_in));
            CK(cudaMemcpyAsync(part.d_item_offs[k], it.offsets + part.first, obytes, cudaMemcpyHostToDevice, w.s_in));
            STAT_ADD(p, h2d_bytes, ibytes + obytes);
            cx.items[k] = ItemStream{(const uint8_t*)part.d_items[k], (const uint64_t*)part.d_item_offs[k], lo, hi};
        }
        cx.item_first = part.first;
    }

    if (pl.wave_tasks_cap == 0) return fail(FBR_ENOMEM, "ring_bytes=%llu too small for one claim unit of %u tasks", (unsigned long long)p->ring_bytes, unit);

    // staging
    if (pl.args_streamed())
        for (int i = 0; i < 2; ++i)
            if (!w.d_args[i]) CK(cudaMalloc((void**)&w.d_args[i], p->ring_bytes));
    if (pl.staged())
        for (int i = 0; i < 2; ++i)
            if (!w.d_out[i]) CK(cudaMalloc((void**)&w.d_out[i], p->ring_bytes));
    if (pl.sink == Sink::FoldPartials) {
        CK(cudaMallocAsync(&part.d_fold, std::max<uint64_t>(16, (part.count + unit - 1) / unit * R), w.s_in));
    } else if (pl.sink == Sink::CallerDevice) {
        cx.window_base = (uint8_t*)d.out + part.first * R;
    } else if (pl.sink == Sink::ZeroCopy) {
        cx.window_base = (uint8_t*)st.out + part.first * R;     // pinned host memory, mapped into the device's address space (UVA)
        STAT_ADD(p, d2h_bytes, part.count * (uint64_t)R);        // these bytes cross PCIe as the kernel's own stores
    } else if (pl.engine_window()) {
        CK(cudaMallocAsync(&part.d_window, std::max<uint64_t>(part.count * R, 16), w.s_in));
        cx.window_base = (uint8_t*)part.d_window;
    }
    if (pl.resilient) {
        part.lost_cap = (uint32_t)std::min<uint64_t>((part.count + unit - 1) / unit, 1u << 22);
        CK(cudaMallocAsync((void**)&part.d_lost, sizeof(LostUnit) * std::max<uint32_t>(1, part.lost_cap), w.s_in));
        CK(cudaHostAlloc((void**)&part.h_lost, sizeof(LostUnit) * std::max<uint32_t>(1, part.lost_cap), cudaHostAllocPortable));
    }

    if (pl.sum_kind && !(body.flags & FBR_BODY_SUMMABLE)) return fail(FBR_EINVAL, "body %s results cannot be summed", body.name.c_str());

    // before any wave launches: every claim unit of every staged stream must fit one staging half
    std::vector<StagedStream> streams;
    if (pl.items == ItemSource::Staged) streams.push_back(staged_items(st, part));
    if (part.emit.h_offs)
        streams.push_back({1, {part.emit.h_offs}, {body.out_bytes}, false,
                           "the claim unit of tasks [%llu, %llu) emits %llu value bytes, more than a staging half of "
                           "ring_bytes %llu holds: raise ring_bytes or use results=\"device\""});
    for (const StagedStream& s : streams)
        for (uint64_t t0 = 0; t0 < part.count; t0 += unit) {
            const uint64_t t1 = std::min<uint64_t>(t0 + unit, part.count);
            if (s.staged_bytes(t0, t1) > p->ring_bytes)
                return fail(FBR_EINVAL, s.too_large, (unsigned long long)(part.first + t0), (unsigned long long)(part.first + t1),
                            (unsigned long long)s.data_bytes(t0, t1), (unsigned long long)p->ring_bytes);
        }
    if (part.emit.h_offs)
        for (int i = 0; i < 2; ++i)
            if (!w.d_vals[i]) CK(cudaMalloc((void**)&w.d_vals[i], p->ring_bytes));
    uint64_t done_tasks = 0;
    while (done_tasks < part.count) {
        uint64_t wt = std::min<uint64_t>(pl.wave_tasks_cap, part.count - done_tasks);
        if (!streams.empty()) wt = fit_staged_wave(streams, done_tasks, wt, unit, p->ring_bytes);
        const uint32_t n_units = (uint32_t)((wt + unit - 1) / unit);
        const uint64_t wno = w.wave_no++;
        const int rw = (int)(wno % kRecWindows);
        const uint64_t wave_first = part.first + done_tasks;  // map index of the wave's first task

        // Task records go through the pinned ring window only when they are not an arithmetic
        // progression the kernels can compute (shuffled arrival).  (The host may not overwrite a window
        // whose previous H2D is in flight.)
        const bool have_records = (d.flags & FBR_SHUFFLE) != 0;
        if (have_records) {
            CK(cudaEventSynchronize(w.ev_rec_h2d[rw]));
            TaskRecord* hrec = w.h_records + (size_t)rw * kRecCapacity;
            for (uint32_t u = 0; u < n_units; ++u) {
                const uint64_t off = (uint64_t)u * unit;
                TaskRecord& r = hrec[u];
                r.seq = (uint32_t)st.seq;
                r.count = (uint32_t)std::min<uint64_t>(unit, wt - off);
                r.first = wave_first + off;
                r.arg_off = pl.args_streamed() ? off * (uint64_t)d.arg_stride : (wave_first + off) * (uint64_t)d.arg_stride;
                r.func_id = (uint32_t)st.func_id;
                r.attempt = part.attempt;
            }
            if (d.flags & FBR_SHUFFLE) shuffle_records(hrec, n_units, d.shuffle_seed ^ (wno * 0x9E3779B97F4A7C15ull));
        }
        int rc = run_wave(p, st, part, body, n_units, wave_first, wt, true, have_records, wno);
        if (rc != FBR_OK) return rc;
        done_tasks += wt;
        part.wave_cum.push_back(done_tasks);
    }
    // resilient parts copy the window back only once no unit is lost any more (resilient_advance)
    return finish_round(p, st, part, !pl.resilient);
}

// ResilientZPool semantics (fiber/pool.py:1612-1659): once a round has finished, re-queue the units
// whose worker died (their slot header carries kUnitLost; gather listed them) with attempt+1, until
// none is lost; then copy the ordered window back.  Returns 1 while more work was launched.
static int resilient_advance(fbr_pool* p, SeqState& st, SeqPart& part) {
    if (!part.cx.plan.resilient || part.finalized) return 0;
    Worker& w = p->workers[part.worker];
    CK(cudaSetDevice(w.device));
    const BodyEntry& body = *body_of(st.func_id);
    const uint32_t lost = std::min(w.h_ctrl[part.ctrl_slot].lost_count, part.lost_cap);
    if (lost == 0) {
        part.finalized = true;
        int rc = finish_round(p, st, part, true);
        return rc != FBR_OK ? rc : 1;
    }
    if (++part.attempt > 200) return fail(FBR_ETASK, "units still failing after 200 re-dispatch rounds");
    st.redispatched_units += lost;
    std::vector<LostUnit> todo(part.h_lost, part.h_lost + lost);
    // clear the device lost counter (sum/err keep accumulating: lost units were never placed)
    static const uint32_t kZero = 0;
    CK(cudaMemcpyAsync(&w.d_ctrl[part.ctrl_slot].lost_count, &kZero, sizeof(uint32_t), cudaMemcpyHostToDevice, w.s_in));
    const uint64_t units_cap = part.cx.plan.redispatch_units_cap;
    for (size_t i = 0; i < todo.size(); i += units_cap) {
        const uint32_t n_units = (uint32_t)std::min<uint64_t>(units_cap, todo.size() - i);
        const uint64_t wno = w.wave_no++;
        const int rw = (int)(wno % kRecWindows);
        CK(cudaEventSynchronize(w.ev_rec_h2d[rw]));
        TaskRecord* hrec = w.h_records + (size_t)rw * kRecCapacity;
        uint64_t wt = 0;
        for (uint32_t u = 0; u < n_units; ++u) {
            const LostUnit& l = todo[i + u];
            TaskRecord& r = hrec[u];
            r.seq = (uint32_t)st.seq;
            r.count = l.count;
            r.first = l.first;
            r.arg_off = l.first * (uint64_t)st.desc.arg_stride;
            r.func_id = (uint32_t)st.func_id;
            r.attempt = part.attempt;
            wt += l.count;
        }
        int rc = run_wave(p, st, part, body, n_units, 0, wt, false, true, wno);
        if (rc != FBR_OK) return rc;
    }
    int rc = finish_round(p, st, part, false);
    return rc != FBR_OK ? rc : 1;
}

// ------------------------------------------------------------------------------------------------
// fault domain: a worker is a CUDA device; it "dies" when its context takes a sticky error (a kernel that
// trapped, an illegal address, an ECC error, a lost device).  The reference notices dead worker processes by
// their exit code and re-queues their pending chunks on the other workers (fiber/pool.py:1623-1656).
// ------------------------------------------------------------------------------------------------
// Every call on a corrupted context returns its sticky error; a healthy stream answers Success / NotReady.
static bool worker_context_dead(Worker& w, cudaError_t* why) {
    if (w.dead) return true;
    cudaError_t e = cudaSetDevice(w.device);
    if (e == cudaSuccess) e = cudaStreamQuery(w.s_comp);
    cudaGetLastError();
    if (e == cudaSuccess || e == cudaErrorNotReady) return false;
    if (why) *why = e;
    return true;
}

static void on_worker_death(fbr_pool* p, int wi, cudaError_t err);

// After a failed CUDA call on worker wi: clears the error and, if the worker's context died, retires the worker
// (on_worker_death).  True if it did.
static bool retire_if_dead(fbr_pool* p, int wi) {
    cudaGetLastError();
    cudaError_t why = cudaErrorUnknown;
    if (!worker_context_dead(p->workers[wi], &why)) return false;
    on_worker_death(p, wi, why);
    return true;
}

// contiguous, claim-unit aligned sub-blocks of tasks [first, first + count) over `workers`
static void cut_blocks(fbr_pool* p, const BodyEntry& body, const fbr_map_desc_t& d, uint64_t first, uint64_t count,
                       const std::vector<int>& workers, uint32_t attempt, std::vector<SeqPart>& out) {
    const int nw = (int)workers.size();
    if (nw == 0 || count == 0) return;
    for (int i = 0; i < nw; ++i) {
        uint64_t b0, b1;
        cut_block(body, map_chunksize(d), count, nw, i, p->workers[workers[0]].sm_count, p->ring_bytes, &b0, &b1);
        if (b1 <= b0) continue;
        SeqPart part;
        part.worker = workers[i];
        part.first = first + b0;
        part.count = b1 - b0;
        part.attempt = attempt;
        out.push_back(std::move(part));
    }
}

// a map's blocks in task order
static std::vector<SeqPart*> parts_in_order(SeqState& st) {
    std::vector<SeqPart*> v;
    for (auto& part : st.parts) v.push_back(&part);
    std::sort(v.begin(), v.end(), [](const SeqPart* a, const SeqPart* b) { return a->first < b->first; });
    return v;
}

static int submit_part(fbr_pool* p, SeqState& st, SeqPart& part, const BodyEntry& body);

// Worker `wi` is dead.  Maps that asked for ResilientZPool semantics get the blocks it was working on cut
// over the surviving workers and re-dispatched with attempt + 1 (whole blocks: what a dead context had
// finished cannot be asked any more); other maps are failed (a plain ZPool map whose worker dies never
// returns, fiber/pool.py:801-824 -- here it raises).  The pool keeps serving on the survivors.
static void on_worker_death(fbr_pool* p, int wi, cudaError_t err) {
    Worker& w = p->workers[wi];
    if (w.dead) return;
    w.dead = true;
    w.death_error = (int)err;
    p->stats.workers_lost++;
    cudaGetLastError();
    std::vector<int> live;
    for (size_t i = 0; i < p->workers.size(); ++i)
        if (!p->workers[i].dead) live.push_back((int)i);
    std::vector<uint64_t> ids;
    for (auto& kv : p->seqs) ids.push_back(kv.first);
    for (uint64_t id : ids) {
        auto it = p->seqs.find(id);
        if (it == p->seqs.end()) continue;
        SeqState& st = *it->second;
        if (st.finished || st.dead_worker >= 0) continue;
        bool touched = false;
        for (auto& part : st.parts) touched |= part.worker == wi;
        if (!touched) continue;
        // device-resident arguments / outputs of a map live on worker 0
        const bool on_w0 = (st.flags & (FBR_ARGS_DEVICE | FBR_OUT_DEVICE)) != 0;
        // an emit pass's blocks carry the offsets of the workers that counted them, and a fold, scan or keyed map's order depends
        // on its block cut: both are failed, not re-cut
        if (!(st.flags & FBR_RESILIENT) || live.empty() || (on_w0 && p->workers[0].dead) || st.emit_pass ||
            (st.flags & (FBR_FOLD | FBR_SCAN | FBR_FOLD_KEYS | FBR_FOLD_SPARSE_KEYS))) {
            st.dead_worker = wi;
            st.dead_error = (int)err;
            continue;
        }
        const BodyEntry& body = *body_of(st.func_id);
        std::vector<SeqPart> next;
        for (auto& part : st.parts) {
            if (part.worker != wi) { next.push_back(std::move(part)); continue; }
            cut_blocks(p, body, st.desc, part.first, part.count, live, part.attempt + 1, next);
            st.redispatched_units += (uint32_t)((part.count + std::max<uint32_t>(1, part.cx.plan.unit) - 1) / std::max<uint32_t>(1, part.cx.plan.unit));
            st.graveyard.push_back(std::move(part));
        }
        st.parts.swap(next);
        for (size_t i = 0; i < st.parts.size(); ++i) {
            SeqPart& part = st.parts[i];
            if (part.ctrl_slot >= 0) continue;            // submitted before
            const int pw = part.worker;
            if (p->workers[pw].dead) continue;            // re-cut by a nested call below
            if (submit_part(p, st, part, body) != FBR_OK) {
                if (retire_if_dead(p, pw)) {              // a survivor turned out dead as well: cut again (st.parts changes)
                    i = (size_t)-1;                       // restart: submit whatever is still unsubmitted
                    if (st.dead_worker >= 0) break;
                } else {
                    st.dead_worker = wi;                  // a real submission error: fail the map
                    st.dead_error = (int)err;
                    break;
                }
            }
        }
    }
}

// A block's emit buffers.  The device ones go with a dead worker's context; the pinned offsets are host memory.
static void free_emit_block(fbr_pool* p, int worker, EmitBlock& e) {
    Worker& w = p->workers[worker];
    if (!w.dead) {
        cudaSetDevice(w.device);
        if (e.d_offs) cudaFreeAsync(e.d_offs, w.s_in);
        if (e.d_values) cudaFreeAsync(e.d_values, w.s_in);
    }
    if (e.h_offs) pinned_release(p, e.h_offs);
    e = EmitBlock();
}

static void free_seq(fbr_pool* p, SeqState& st) {
    // a scan map's wraps run on s_fold, its windows are freed on s_in: a wrap still in flight finishes first
    for (cudaEvent_t ev : st.block_done)
        if (ev) { cudaEventSynchronize(ev); cudaEventDestroy(ev); }
    cudaGetLastError();
    st.block_done.clear();
    for (auto& part : st.graveyard)        // device-side resources died with the worker's context
        if (part.h_lost) cudaFreeHost(part.h_lost);
    st.graveyard.clear();
    for (auto& part : st.parts) {
        Worker& w = p->workers[part.worker];
        if (w.dead) {                      // nothing on a dead context can be freed (or needs to be)
            if (part.h_lost) cudaFreeHost(part.h_lost);
            free_emit_block(p, part.worker, part.emit);
            continue;
        }
        cudaSetDevice(w.device);
        if (part.done) { cudaEventSynchronize(part.done); cudaEventDestroy(part.done); }
        for (auto e : part.wave_done) cudaEventDestroy(e);
        for (auto& t : part.t_dispatch) { cudaEventDestroy(t.a); cudaEventDestroy(t.b); }
        for (auto& t : part.t_gather) { cudaEventDestroy(t.a); cudaEventDestroy(t.b); }
        // stream-ordered frees: cudaFree would synchronise the whole device, i.e. wait for resident
        // device processes (queues.cu) that may themselves be waiting for this host thread
        if (part.d_shared_tmp) cudaFreeAsync(part.d_shared_tmp, w.s_in);
        if (part.d_window) cudaFreeAsync(part.d_window, w.s_in);
        if (part.d_args_full) cudaFreeAsync(part.d_args_full, w.s_in);
        for (uint32_t k = 0; k < kMaxItemStreams; ++k) {
            if (part.d_items[k]) cudaFreeAsync(part.d_items[k], w.s_in);
            if (part.d_item_offs[k]) cudaFreeAsync(part.d_item_offs[k], w.s_in);
        }
        if (part.d_lost) cudaFreeAsync(part.d_lost, w.s_in);
        if (part.d_fold) cudaFreeAsync(part.d_fold, w.s_in);
        if (part.d_sparse) cudaFreeAsync(part.d_sparse, w.s_in);
        free_emit_block(p, part.worker, part.emit);
        if (part.h_lost) cudaFreeHost(part.h_lost);
        if (part.ctrl_slot >= 0) w.ctrl_free.push_back(part.ctrl_slot);
    }
    if (st.values) pinned_release(p, st.values);
    st.values = nullptr;
    for (void* h : st.sparse_host)
        if (h) pinned_release(p, h);
    st.sparse_host.clear();
    if (st.sparse_words) pinned_release(p, st.sparse_words);
    st.sparse_words = nullptr;
    if (st.own_out && st.out && !numa_pinned_release(p, st.out)) pinned_release(p, st.out);
}

// ------------------------------------------------------------------------------------------------
// extern "C" API
// ------------------------------------------------------------------------------------------------
extern "C" {

int fbr_abi_version(void) { return FBR_ABI_VERSION; }

// Force-load every kernel of this library on `device`.  With CUDA's lazy module loading the first
// launch of a kernel may synchronise the context; if a resident device process (queues.cu) is
// spinning on a host message at that moment the two deadlock.  queues.cu calls this before it
// starts a resident kernel.  (Internal: not part of the public header.)
int fbr_internal_preload(int device) {
    if (cudaSetDevice(device) != cudaSuccess) return FBR_ECUDA;
    cudaFuncAttributes at;
    for (int f = 0, n = body_count(); f < n; ++f) {   // asking for the occupancy loads the kernels
        const BodyEntry& b = *body_of(f);
        b.occupancy(0);
        if (b.flags & FBR_BODY_INDEX_ARG) b.occupancy(1);
    }
    cudaFuncGetAttributes(&at, (const void*)gather_ordered_kernel);
    cudaFuncGetAttributes(&at, (const void*)gather_rows_kernel);
    cudaFuncGetAttributes(&at, (const void*)gather_bulk_kernel);
    cudaFuncGetAttributes(&at, (const void*)dispatch_payload_map_tma_kernel);
    cudaFuncGetAttributes(&at, (const void*)payload_fill_kernel);
    cudaGetLastError();
    return FBR_OK;
}
const char* fbr_last_error(void) { return g_err.c_str(); }

int fbr_device_count(int* n) {
    if (!n) return fail(FBR_EINVAL, "n is NULL");
    int c = 0;
    cudaError_t e = cudaGetDeviceCount(&c);
    if (e != cudaSuccess) {
        *n = 0;
        cudaGetLastError();
        return fail(FBR_ENODEV, "cudaGetDeviceCount: %s", cudaGetErrorString(e));
    }
    *n = c;
    return FBR_OK;
}

int fbr_body_count(int* n) {
    if (!n) return fail(FBR_EINVAL, "n is NULL");
    *n = body_count();
    return FBR_OK;
}

int fbr_body_info(int func_id, fbr_body_info_t* info) {
    const BodyEntry* bp = body_of(func_id);
    if (!info || !bp) return fail(FBR_EINVAL, "bad func_id %d", func_id);
    const BodyEntry& b = *bp;
    memset(info, 0, sizeof *info);
    info->func_id = func_id;
    info->arg_bytes = b.arg_bytes;
    info->result_bytes = b.result_bytes;
    info->result_kind = b.result_kind;
    info->flags = b.flags;
    info->unit_tasks = b.unit_tasks;
    snprintf(info->name, sizeof info->name, "%s", b.name.c_str());
    return FBR_OK;
}

int fbr_body_shared_info(int func_id, uint32_t* elem_bytes, uint32_t* stage_bytes) {
    const BodyEntry* bp = body_of(func_id);
    if (!elem_bytes || !stage_bytes || !bp) return fail(FBR_EINVAL, "bad func_id %d", func_id);
    *elem_bytes = bp->shared_elem_bytes;
    *stage_bytes = bp->shared_stage_bytes;
    return FBR_OK;
}

int fbr_body_items_info(int func_id, uint32_t* item_bytes) {
    const BodyEntry* bp = body_of(func_id);
    if (!item_bytes || !bp) return fail(FBR_EINVAL, "bad func_id %d", func_id);
    *item_bytes = bp->item_bytes[0];
    return FBR_OK;
}

int fbr_body_items_streams(int func_id, uint32_t* n_streams, uint32_t item_bytes[4]) {
    const BodyEntry* bp = body_of(func_id);
    if (!n_streams || !item_bytes || !bp) return fail(FBR_EINVAL, "bad func_id %d", func_id);
    *n_streams = bp->item_streams;
    for (uint32_t k = 0; k < kMaxItemStreams; ++k) item_bytes[k] = bp->item_bytes[k];
    return FBR_OK;
}

int fbr_body_emit_info(int func_id, uint32_t* out_bytes) {
    const BodyEntry* bp = body_of(func_id);
    if (!out_bytes || !bp) return fail(FBR_EINVAL, "bad func_id %d", func_id);
    *out_bytes = bp->out_bytes;
    return FBR_OK;
}

int fbr_body_fold_info(int func_id, void* identity, uint32_t* bytes) {
    const BodyEntry* bp = body_of(func_id);
    if (!bytes || !bp) return fail(FBR_EINVAL, "bad func_id %d", func_id);
    *bytes = (uint32_t)bp->identity.size();
    if (identity && !bp->identity.empty()) memcpy(identity, bp->identity.data(), bp->identity.size());
    return FBR_OK;
}

int fbr_body_lookup(const char* name, int* func_id) {
    if (!name || !func_id) return fail(FBR_EINVAL, "NULL argument");
    for (int f = 0, n = body_count(); f < n; ++f)
        if (body_of(f)->name == name) { *func_id = f; return FBR_OK; }
    return fail(FBR_ENOENT, "no device body named '%s' is compiled into libfiber_b200 or registered with fbr_register_body", name);
}

// Why the descriptor `m` of body `name` from `module_path` cannot be registered, or "" when it can.  The rules are checked
// in a fixed order, so a descriptor that breaks several always gets the same message.
static std::string descriptor_error(const fbr_body_module_t* m, const char* module_path, const char* name) {
    if (!m || m->abi != FBR_BODY_MODULE_ABI || m->wave_params_bytes != sizeof(WaveParams) || !m->launch || !m->occupancy || !m->name)
        return strf("module %s: descriptor ABI %u / wave-parameter size %u do not match this library (%u / %u); rebuild it against include/fiber_b200_body.cuh",
                    module_path, m ? m->abi : 0u, m ? m->wave_params_bytes : 0u, (unsigned)FBR_BODY_MODULE_ABI, (unsigned)sizeof(WaveParams));
    if (strcmp(m->name, name) != 0) return strf("module %s exports body '%s', not '%s'", module_path, m->name, name);
    const bool is_record = (m->flags & FBR_BODY_RECORD) != 0, bcast = (m->flags & FBR_BODY_BROADCAST) != 0;
    if (!bcast && (m->shared_elem_bytes || m->shared_stage_bytes))
        return strf("module %s: body '%s' describes a broadcast element but lacks FBR_BODY_BROADCAST", module_path, name);
    if (bcast && !is_record)
        return strf("module %s: body '%s': only record bodies take a broadcast block (FBR_BODY_BROADCAST)", module_path, name);
    const bool items = (m->flags & FBR_BODY_ITEMS) != 0;
    const char* why = nullptr;
    if (!items && m->item_bytes) why = "describes an item element but lacks FBR_BODY_ITEMS";
    else if (items && !is_record) why = "only record bodies take items (FBR_BODY_ITEMS)";
    else if (items && !record::item_elem_ok(m->item_bytes)) why = "the item size must be 1, 2 or a multiple of 4 up to 4096 bytes";
    else if (items && (m->flags & FBR_BODY_INDEX_ARG)) why = "an items body cannot take range() indices (FBR_BODY_INDEX_ARG)";
    else if (m->item_streams > kMaxItemStreams) why = "takes at most 4 item streams (item_streams)";
    else if (!items && m->item_streams > 1) why = "describes several item streams but lacks FBR_BODY_ITEMS";
    for (uint32_t k = 1; k < kMaxItemStreams && !why; ++k) {
        const uint32_t e = m->more_item_bytes[k - 1];
        if (k < m->item_streams && !record::item_elem_ok(e))
            why = "the item size of every stream must be 1, 2 or a multiple of 4 up to 4096 bytes";
        else if (k >= m->item_streams && e)
            why = "describes the item size of a stream past its item_streams";
    }
    const bool emit = (m->flags & FBR_BODY_EMIT) != 0;
    if (why) {
    } else if (!emit && m->out_bytes) {
        why = "describes an out element but lacks FBR_BODY_EMIT";
    } else if (emit && !is_record) {
        why = "only record bodies emit variable-length results (FBR_BODY_EMIT)";
    } else if (emit && (m->result_bytes != 8 || m->result_kind != FBR_RES_OFFSETS)) {
        why = "an emit body has no fixed result record (Res = fbr::NoRes): result_bytes 8 and result kind FBR_RES_OFFSETS";
    } else if (emit && !record::item_elem_ok(m->out_bytes)) {
        why = "the out size must be 1, 2 or a multiple of 4 up to 4096 bytes";
    } else if (emit && (m->flags & FBR_BODY_SUMMABLE)) {
        why = "an emit body's results cannot be folded on the device (FBR_BODY_SUMMABLE)";
    }
    const bool fold = (m->flags & FBR_BODY_FOLD) != 0;
    if (why) {
    } else if (fold != (m->fold != nullptr && m->identity != nullptr)) {
        why = fold ? "sets FBR_BODY_FOLD but its descriptor lacks the fold entry or the identity record"
                   : "describes a fold entry or an identity record but lacks FBR_BODY_FOLD";
    } else if (fold && !is_record) {
        why = "only record bodies fold their maps (FBR_BODY_FOLD)";
    } else if (fold && emit) {
        why = "an emit body cannot fold (FBR_BODY_FOLD with FBR_BODY_EMIT)";
    } else if (fold && (m->flags & FBR_BODY_SUMMABLE)) {
        why = "a fold body cannot also be FBR_BODY_SUMMABLE";
    } else if (fold ? m->identity_bytes != m->result_bytes : m->identity_bytes != 0) {
        why = fold ? "the identity record must be result_bytes long (identity_bytes)" : "describes an identity size but lacks FBR_BODY_FOLD";
    }
    // `scan` follows identity_bytes: it is read only from a descriptor that sets FBR_BODY_SCAN, so a fold descriptor that
    // ends before it stays valid
    const bool scan = (m->flags & FBR_BODY_SCAN) != 0;
    if (why) {
    } else if (scan && !fold) {
        why = "FBR_BODY_SCAN needs FBR_BODY_FOLD (a scan is a running fold)";
    } else if (scan && m->scan == nullptr) {
        why = "sets FBR_BODY_SCAN but its descriptor lacks the scan entry";
    }
    // `keys` and `fold_segments` follow `scan`, and are read only from a descriptor that sets FBR_BODY_KEYED
    const bool keyed = (m->flags & FBR_BODY_KEYED) != 0;
    if (why) {
    } else if (keyed && !fold) {
        why = "FBR_BODY_KEYED needs FBR_BODY_FOLD (a keyed fold is a fold per key)";
    } else if (keyed && (m->keys == nullptr || m->fold_segments == nullptr)) {
        why = "sets FBR_BODY_KEYED but its descriptor lacks the keys or the fold_segments entry";
    }
    if (why) return strf("module %s: body '%s' %s", module_path, name, why);
    const uint32_t group = m->group_threads;
    if (group > 1 && (group > 32 || (group & (group - 1)) != 0))
        return strf("module %s: body '%s': group_threads %u is not 0, 1, 2, 4, 8, 16 or 32", module_path, name, group);
    if (group > 1 && !is_record)
        return strf("module %s: body '%s': only record bodies run a task on a group of threads (group_threads %u)", module_path, name, group);
    if (!is_record) {
        if (m->result_bytes == 0 || m->unit_tasks == 0 || (m->arg_bytes % 8) != 0 || m->result_kind > FBR_RES_BITS8)
            return strf("module %s: body '%s' has an invalid record layout", module_path, name);
        return "";
    }
    // staged through shared memory by dispatch_record_kernel: sizes are free within its stages.  A group body's tasks must
    // also come in 16 B-aligned groups of kAlign that fit one 32 KB stage
    const uint32_t big = std::max(m->arg_bytes, m->result_bytes);
    if (m->arg_bytes == 0 && !items) why = "argument bytes may be 0 (no head record, fbr::NoArg) only for an items body (FBR_BODY_ITEMS)";
    else if (m->result_bytes == 0 || m->arg_bytes % 4 || m->result_bytes % 4) why = "argument and result bytes must be non-zero multiples of 4";
    else if (group <= 1 && big > record::kThreadRecordBytes) why = "argument and result records are at most 4096 bytes";
    else if (big > record::kStageBytes) why = "argument and result records of group bodies are at most 32768 bytes";
    else if ((uint64_t)record::align_tasks(m->arg_bytes, m->result_bytes) * big > record::kStageBytes)
        why = "one 16 B-aligned group of tasks must fit a 32768-byte stage: kAlign * max(arg_bytes, result_bytes) <= 32768, "
              "kAlign = 1 when both sizes are multiples of 16, 2 when both are multiples of 8, else 4";
    else if (m->result_kind != (emit ? (uint32_t)FBR_RES_OFFSETS : (uint32_t)FBR_RES_BYTES))
        why = "the result kind must be FBR_RES_BYTES (no bit-packed twin)";
    else if (m->flags & FBR_BODY_SUMMABLE) why = "results cannot be folded on the device (FBR_BODY_SUMMABLE)";
    else if ((m->flags & FBR_BODY_NEEDS_SHARED) && !bcast)
        why = "a body without a Shared element type receives no broadcast block (FBR_BODY_NEEDS_SHARED without FBR_BODY_BROADCAST)";
    else if (bcast && !(m->flags & FBR_BODY_NEEDS_SHARED)) why = "FBR_BODY_BROADCAST needs FBR_BODY_NEEDS_SHARED (its maps must pass a block)";
    else if (bcast && !record::shared_elem_ok(m->shared_elem_bytes)) why = "the broadcast element must be a non-zero multiple of 4 bytes up to 4096";
    else if (bcast && m->shared_stage_bytes % 16) why = "the broadcast staging budget must be a multiple of 16 bytes";
    else if (m->unit_tasks == 0) why = "unit_tasks is 0";
    else if (record::smem_bytes(m->unit_tasks, m->arg_bytes, m->result_bytes, m->shared_stage_bytes) > record::kSmemBudget)
        why = "the stages and the broadcast staging budget exceed 200 KB of shared memory";
    return why ? strf("module %s: record body '%s': %s", module_path, name, why) : "";
}

int fbr_register_body(const char* name, const char* module_path, const char* entry, int* func_id) {
    if (!name || !module_path || !entry || !func_id) return fail(FBR_EINVAL, "NULL argument");
    // RTLD_LOCAL: several body modules may define the same helper symbols
    void* h = dlopen(module_path, RTLD_NOW | RTLD_LOCAL);
    if (!h) return fail(FBR_ENOENT, "dlopen(%s) failed: %s", module_path, dlerror());
    fbr_body_entry_fn fn = (fbr_body_entry_fn)dlsym(h, entry);
    if (!fn) {
        dlclose(h);
        return fail(FBR_ENOENT, "module %s has no entry point '%s'", module_path, entry);
    }
    const fbr_body_module_t* m = fn();
    const std::string err = descriptor_error(m, module_path, name);
    if (!err.empty()) {
        dlclose(h);
        return fail(FBR_EINVAL, "%s", err.c_str());
    }
    std::lock_guard<std::mutex> g(g_body_mu);
    builtin_bodies_once();
    for (size_t f = 0; f < g_bodies.size(); ++f)
        if (g_bodies[f].name == name) {
            if (g_bodies[f].module == nullptr) { dlclose(h); return fail(FBR_EINVAL, "'%s' is a compiled-in body", name); }
            dlclose(h);             // same name registered before: idempotent, keep the first module
            *func_id = (int)f;
            return FBR_OK;
        }
    BodyEntry b;
    b.name = name;
    b.arg_bytes = m->arg_bytes; b.result_bytes = m->result_bytes; b.result_kind = m->result_kind;
    b.flags = m->flags; b.unit_tasks = m->unit_tasks;
    b.shared_elem_bytes = m->shared_elem_bytes; b.shared_stage_bytes = m->shared_stage_bytes;
    b.item_streams = (m->flags & FBR_BODY_ITEMS) ? std::max<uint32_t>(1, m->item_streams) : 0;
    b.item_bytes[0] = m->item_bytes;
    for (uint32_t k = 1; k < b.item_streams; ++k) b.item_bytes[k] = m->more_item_bytes[k - 1];
    b.out_bytes = m->out_bytes;
    if (m->flags & FBR_BODY_FOLD) {
        b.fold = m->fold;
        b.identity.assign((const uint8_t*)m->identity, (const uint8_t*)m->identity + m->result_bytes);
    }
    if (m->flags & FBR_BODY_SCAN) b.scan = m->scan;
    if (m->flags & FBR_BODY_KEYED) {
        b.keys = m->keys;
        b.fold_segments = m->fold_segments;
    }
    b.launch = m->launch; b.occupancy = m->occupancy;
    b.module = h;
    g_bodies.push_back(b);
    *func_id = (int)g_bodies.size() - 1;
    return FBR_OK;
}

int fbr_plan_query(int func_id, uint64_t n_tasks, uint32_t chunksize, uint64_t ring_bytes, int n_workers,
                   int worker, int sm_count, fbr_plan_t* plan) {
    if (!plan || !body_of(func_id) || n_workers < 1 || worker < 0 || worker >= n_workers)
        return fail(FBR_EINVAL, "bad arguments");
    const BodyEntry& body = *body_of(func_id);
    const uint64_t ring = round_up(ring_bytes ? ring_bytes : (256ull << 20), 4096);
    fbr_map_desc_t d{};
    d.chunksize = chunksize;   // map_chunksize: 0 is 32, FBR_PLAN_FOLD cuts as a fold map
    if (sm_count <= 0) sm_count = 132;
    // what fbr_map_submit does: cut_blocks, then plan_block of the worker's block
    uint64_t b0, b1;
    cut_block(body, map_chunksize(d), n_tasks, n_workers, worker, sm_count, ring, &b0, &b1);
    const BlockPlan pl = plan_block(body, d, 0, worker, b0, b1 - b0, true, sm_count, ring, true, 0);
    plan->block_first = b0;
    plan->block_count = b1 - b0;
    plan->unit_tasks = pl.unit;
    plan->slot_stride = pl.slot_stride;
    plan->n_units = plan->block_count ? (plan->block_count + plan->unit_tasks - 1) / plan->unit_tasks : 0;
    return FBR_OK;
}

int fbr_pool_create(int n_workers, const int* device_ids, uint64_t ring_bytes, uint32_t flags, fbr_pool_t** out) {
    if (!out || n_workers <= 0) return fail(FBR_EINVAL, "bad arguments");
    int ndev = 0;
    int rc = fbr_device_count(&ndev);
    if (rc != FBR_OK) return rc;
    if (ndev == 0) return fail(FBR_ENODEV, "no CUDA device visible; fiber_b200 has no CPU fallback");
    std::unique_ptr<fbr_pool> p(new fbr_pool());
    p->flags = flags;
    p->ring_bytes = round_up(ring_bytes ? ring_bytes : (256ull << 20), 4096);
    if (p->ring_bytes >= (1ull << 35)) return fail(FBR_EINVAL, "ring_bytes must be below 32 GiB (32-bit vector index in gather_ordered)");
    memset(&p->stats, 0, sizeof p->stats);
    p->workers.resize(n_workers);
    for (int i = 0; i < n_workers; ++i) {
        const int dev = device_ids ? device_ids[i] : (i % ndev);
        if (dev < 0 || dev >= ndev) return fail(FBR_EINVAL, "device id %d out of range (have %d)", dev, ndev);
        for (int j = 0; j < i; ++j)
            if (p->workers[j].device == dev) return fail(FBR_EINVAL, "device %d bound to two workers", dev);
        rc = worker_init(p.get(), p->workers[i], dev);
        if (rc != FBR_OK) {
            for (auto& w : p->workers) worker_destroy(w);
            return rc;
        }
    }
    // Peer access (NVLink P2P) is switched on by the first map that needs it (ensure_peer_access): contexts
    // with peer mappings between them share their fate -- a kernel fault on one device takes the peers' contexts
    // down with it -- so a pool that only runs host-resident maps keeps its workers' fault domains separate.
    *out = p.release();
    return FBR_OK;
}

// Peer access between all workers: lets one map keep its arguments / ordered output resident on worker 0
// while every worker's dispatch kernel loads its block from there and stores its results there, straight
// over NVLink (scatter + gather fused into the kernel, no separate collective).
static bool ensure_peer_access(fbr_pool* p) {
    if (p->peer_checked) return p->peer_ok;
    p->peer_checked = true;
    const int n = (int)p->workers.size();
    p->peer_ok = n > 1;
    for (int i = 0; i < n && p->peer_ok; ++i)
        for (int j = 0; j < n; ++j) {
            if (i == j) continue;
            int can = 0;
            cudaDeviceCanAccessPeer(&can, p->workers[i].device, p->workers[j].device);
            if (!can) { p->peer_ok = false; break; }
            cudaSetDevice(p->workers[i].device);
            cudaError_t e = cudaDeviceEnablePeerAccess(p->workers[j].device, 0);
            if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) p->peer_ok = false;
            cudaGetLastError();
        }
    return p->peer_ok;
}

int fbr_pool_n_workers(fbr_pool_t* p, int* n) {
    if (!p || !n) return fail(FBR_EINVAL, "NULL argument");
    *n = (int)p->workers.size();
    return FBR_OK;
}

int fbr_pool_worker_device(fbr_pool_t* p, int worker, int* dev) {
    if (!p || !dev || worker < 0 || worker >= (int)p->workers.size()) return fail(FBR_EINVAL, "bad worker");
    *dev = p->workers[worker].device;
    return FBR_OK;
}

int fbr_pool_close(fbr_pool_t* p) {
    if (!p) return fail(FBR_EINVAL, "NULL pool");
    std::lock_guard<std::mutex> g(p->mu);
    if (p->state == ST_RUN) p->state = ST_CLOSE;
    return FBR_OK;
}

int fbr_pool_terminate(fbr_pool_t* p) {
    if (!p) return fail(FBR_EINVAL, "NULL pool");
    std::lock_guard<std::mutex> g(p->mu);
    p->state = ST_TERMINATE;
    return FBR_OK;
}

int fbr_pool_join(fbr_pool_t* p) {
    if (!p) return fail(FBR_EINVAL, "NULL pool");
    std::lock_guard<std::mutex> g(p->mu);
    if (p->state == ST_RUN) return fail(FBR_ESTATE, "join() before close()/terminate()");
    for (auto& w : p->workers) {
        CK(cudaSetDevice(w.device));
        CK(cudaStreamSynchronize(w.s_in));
        CK(cudaStreamSynchronize(w.s_comp));
        CK(cudaStreamSynchronize(w.s_gath));
        CK(cudaStreamSynchronize(w.s_out));
    }
    return FBR_OK;
}

int fbr_pool_destroy(fbr_pool_t* p) {
    if (!p) return FBR_OK;
    {
        std::lock_guard<std::mutex> g(p->mu);
        p->submitters.clear();          // joins the submit threads
        for (auto& kv : p->seqs) free_seq(p, *kv.second);
        p->seqs.clear();
        for (auto& kv : p->shared)
            for (size_t i = 0; i < kv.second.d_ptr.size(); ++i) {
                cudaSetDevice(p->workers[i].device);
                cudaFreeAsync(kv.second.d_ptr[i], p->workers[i].s_comp);
            }
        for (auto& w : p->workers) worker_destroy(w);
        for (auto& kv : p->pin_free)
            for (void* q : kv.second) cudaFreeHost(q);
        for (auto& kv : p->pin_live) cudaFreeHost(kv.first);
        for (auto& kv : p->numa_live) { cudaHostUnregister(kv.first); munmap(kv.first, kv.second.second); }
    }
    delete p;
    return FBR_OK;
}

int fbr_shared_put(fbr_pool_t* p, const void* host, uint64_t bytes, uint64_t* handle) {
    if (!p || !host || !bytes || !handle) return fail(FBR_EINVAL, "bad arguments");
    std::lock_guard<std::mutex> g(p->mu);
    SharedBlock sb;
    sb.bytes = bytes;
    for (auto& w : p->workers) {
        CK(cudaSetDevice(w.device));
        void* dptr = nullptr;
        CK(cudaMallocAsync(&dptr, bytes, w.s_in));
        CK(cudaMemcpyAsync(dptr, host, bytes, cudaMemcpyHostToDevice, w.s_in));
        CK(cudaStreamSynchronize(w.s_in));
        sb.d_ptr.push_back(dptr);
        p->stats.h2d_bytes += bytes;
    }
    *handle = p->next_shared++;
    p->shared[*handle] = sb;
    return FBR_OK;
}

int fbr_shared_drop(fbr_pool_t* p, uint64_t handle) {
    if (!p) return fail(FBR_EINVAL, "NULL pool");
    std::lock_guard<std::mutex> g(p->mu);
    auto it = p->shared.find(handle);
    if (it == p->shared.end()) return fail(FBR_ENOENT, "unknown shared handle");
    for (size_t i = 0; i < it->second.d_ptr.size(); ++i) {
        Worker& w = p->workers[i];
        cudaSetDevice(w.device);
        cudaStreamSynchronize(w.s_comp);   // maps that read the block have been waited for by their owners
        cudaFreeAsync(it->second.d_ptr[i], w.s_comp);
    }
    p->shared.erase(it);
    return FBR_OK;
}

static int map_submit(fbr_pool_t* p, const fbr_map_desc_t* d, const fbr_items_desc_t* items, uint32_t n_streams, uint64_t* seq_out);

int fbr_map_submit(fbr_pool_t* p, const fbr_map_desc_t* d, uint64_t* seq_out) {
    if (!p || !d || !seq_out) return fail(FBR_EINVAL, "NULL argument");
    const BodyEntry* b = body_of(d->func_id);
    if (b && (b->flags & FBR_BODY_ITEMS))
        return fail(FBR_EINVAL, "body %s takes items: submit its maps with fbr_map_submit_items", b->name.c_str());
    return map_submit(p, d, nullptr, 0, seq_out);
}

int fbr_map_submit_items(fbr_pool_t* p, const fbr_map_desc_t* d, const fbr_items_desc_t* it, uint64_t* seq_out) {
    return fbr_map_submit_items_n(p, d, it, 1, seq_out);
}

int fbr_map_submit_items_n(fbr_pool_t* p, const fbr_map_desc_t* d, const fbr_items_desc_t* streams, uint32_t n_streams, uint64_t* seq_out) {
    if (!p || !d || !streams || !seq_out) return fail(FBR_EINVAL, "NULL argument");
    const BodyEntry* b = body_of(d->func_id);
    if (!b) return fail(FBR_EINVAL, "bad func_id %d", d->func_id);
    if (!(b->flags & FBR_BODY_ITEMS))
        return fail(FBR_EINVAL, "body %s takes no items: submit its maps with fbr_map_submit", b->name.c_str());
    if (n_streams != b->item_streams)
        return fail(FBR_EINVAL, "body %s takes %u item stream%s, not %u%s", b->name.c_str(), b->item_streams,
                    b->item_streams == 1 ? "" : "s", n_streams, n_streams == 1 ? " (fbr_map_submit_items_n submits several)" : "");
    for (uint32_t k = 0; k < n_streams; ++k) {
        const fbr_items_desc_t* it = &streams[k];
        // one-stream maps keep their messages; a multi-stream map's name the stream
        const std::string sk = n_streams > 1 ? strf("stream %u: ", k) : std::string();
        const char* sp = sk.c_str();
        if (it->item_bytes != b->item_bytes[k])
            return fail(FBR_EINVAL, "%sitem_bytes %u does not match body %s (%u)", sp, it->item_bytes, b->name.c_str(), b->item_bytes[k]);
        if (d->n_tasks && !it->offsets) return fail(FBR_EINVAL, "%soffsets is NULL", sp);
        if (it->n_items && !it->items) return fail(FBR_EINVAL, "%sitems is NULL", sp);
        if (d->flags & FBR_ARGS_DEVICE) {
            // a body may load its items as vectors as wide as the largest power of two dividing item_bytes, up to 16 B (a double,
            // a 16 B struct); this is the alignment required, which can be stricter than alignof(Item) (four floats: 16, not 4)
            const uint32_t e = it->item_bytes, align = std::min<uint32_t>(16u, e & (~e + 1u));
            if ((uintptr_t)it->items % align)
                return fail(FBR_EINVAL, "%sdevice-resident items of body %s must be %u-byte aligned", sp, b->name.c_str(), align);
            if ((uintptr_t)it->offsets % 8) return fail(FBR_EINVAL, "%sdevice-resident offsets must be 8-byte aligned", sp);
        } else if (d->n_tasks) {
            // the kernel trusts host-resident offsets: check them before anything launches
            const uint64_t* o = it->offsets;
            for (uint64_t j = 0; j < d->n_tasks; ++j)
                if (o[j] > o[j + 1])
                    return fail(FBR_EINVAL, "%soffsets decrease at task %llu (%llu > %llu)", sp, (unsigned long long)j,
                                (unsigned long long)o[j], (unsigned long long)o[j + 1]);
            if (o[d->n_tasks] > it->n_items)
                return fail(FBR_EINVAL, "%soffsets[%llu] = %llu is past n_items %llu", sp, (unsigned long long)d->n_tasks,
                            (unsigned long long)o[d->n_tasks], (unsigned long long)it->n_items);
        }
    }
    if (d->flags & FBR_ARGS_DEVICE) {
        int nw = 0;
        {
            std::lock_guard<std::mutex> g(p->mu);
            nw = (int)p->workers.size();
        }
        if (nw != 1)
            return fail(FBR_EINVAL, "device-resident items (FBR_ARGS_DEVICE) need a one-worker pool; this pool has %d workers", nw);
    }
    return map_submit(p, d, streams, n_streams, seq_out);
}

// Submits one map.  The emit pass of an emit map passes `counted`, the count pass's blocks with their emit state, and
// `values`, the pinned values segment of n_values values: it runs over exactly those blocks and takes both over.
static int map_submit_pass(fbr_pool_t* p, const fbr_map_desc_t* d, const fbr_items_desc_t* items, uint32_t n_streams, uint64_t* seq_out,
                           std::vector<SeqPart>* counted = nullptr, void** values = nullptr, uint64_t n_values = 0);
static int emit_submit(fbr_pool_t* p, const fbr_map_desc_t* d, const fbr_items_desc_t* items, uint32_t n_streams, uint64_t* seq_out);
static void harvest(fbr_pool* p, SeqState& st);

static int map_submit(fbr_pool_t* p, const fbr_map_desc_t* d, const fbr_items_desc_t* items, uint32_t n_streams, uint64_t* seq_out) {
    const BodyEntry* b = body_of(d->func_id);
    if (b && (b->flags & FBR_BODY_EMIT)) return emit_submit(p, d, items, n_streams, seq_out);
    return map_submit_pass(p, d, items, n_streams, seq_out);
}

// Emit map, step 2: scan_counts_kernel turns each block of the count pass `cseq` into an entry of `blocks` (task order)
// with its offsets and, in *totals, its total; `scanned` gets an event per scan.  With `host_offs` the host also gets a
// pinned copy of each block's offsets, to cut the emit pass's waves by.
static int emit_scan(fbr_pool_t* p, uint64_t cseq, bool host_offs, std::vector<SeqPart>& blocks, uint64_t** totals,
                     std::vector<std::pair<int, cudaEvent_t>>& scanned) {
    std::lock_guard<std::mutex> g(p->mu);
    auto it = p->seqs.find(cseq);
    if (it == p->seqs.end()) return fail(FBR_ENOENT, "count pass of an emit map was released");
    const std::vector<SeqPart*> parts = parts_in_order(*it->second);
    // one total per block, written by its scan into pinned memory (mapped into every device's address space)
    int rc = pinned_acquire(p, sizeof(uint64_t) * std::max<size_t>(1, parts.size()), (void**)totals);
    if (rc != FBR_OK) return rc;
    for (size_t k = 0; k < parts.size(); ++k) {
        const SeqPart& part = *parts[k];
        Worker& w = p->workers[part.worker];
        const uint64_t tiles = part.count / scan::kTile + 1;
        if (tiles >= (1ull << 31)) return fail(FBR_EINVAL, "emit map block of %llu tasks is too large to scan", (unsigned long long)part.count);
        const uint64_t obytes = (part.count + 1) * sizeof(uint64_t);
        SeqPart b;
        b.worker = part.worker;
        b.first = part.first;
        b.count = part.count;
        CK(cudaSetDevice(w.device));
        CK(cudaMallocAsync((void**)&b.emit.d_offs, obytes, w.s_comp));
        blocks.push_back(std::move(b));
        EmitBlock& e = blocks.back().emit;
        void* scratch = nullptr;
        CK(cudaMallocAsync(&scratch, (tiles + 1) * sizeof(uint64_t), w.s_comp));
        cudaMemsetAsync(scratch, 0, (tiles + 1) * sizeof(uint64_t), w.s_comp);
        scan_counts_kernel<<<(unsigned)tiles, scan::kThreads, 0, w.s_comp>>>(
            (const uint64_t*)part.cx.window_base, part.count, e.d_offs, (unsigned long long*)scratch,
            (uint32_t*)((uint64_t*)scratch + tiles), *totals + k);
        const cudaError_t launched = cudaGetLastError();
        cudaFreeAsync(scratch, w.s_comp);
        if (launched != cudaSuccess) return fail(FBR_ECUDA, "scan_counts_kernel: %s", cudaGetErrorString(launched));
        if (host_offs) {
            rc = pinned_acquire(p, obytes, (void**)&e.h_offs);
            if (rc != FBR_OK) return rc;
            CK(cudaMemcpyAsync(e.h_offs, e.d_offs, obytes, cudaMemcpyDeviceToHost, w.s_comp));
        }
        cudaEvent_t ev;
        CK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        scanned.push_back({w.device, ev});
        CK(cudaEventRecord(ev, w.s_comp));
    }
    return FBR_OK;
}

// Emit map, step 3: the blocks' totals give each block its base and the map its n_values.  Host-resident values go to
// one pinned segment (*values); a block whose values do not stream through the staging halves (no h_offs: values kept
// on the device, or units that may be re-dispatched) is written to a device buffer of its own.
static int emit_place(fbr_pool_t* p, const BodyEntry& body, bool on_device, std::vector<SeqPart>& blocks,
                      const uint64_t* totals, void** values, uint64_t* n_values) {
    std::lock_guard<std::mutex> g(p->mu);
    const uint64_t ob = body.out_bytes;
    for (size_t k = 0; k < blocks.size(); ++k) {
        blocks[k].emit.total = totals[k];
        blocks[k].emit.base = *n_values;
        *n_values += totals[k];
    }
    if (*n_values >= (1ull << 62) / std::max<uint32_t>(1, body.out_bytes))
        return fail(FBR_EINVAL, "body %s: the map's count pass gave %llu values, too many to place", body.name.c_str(),
                    (unsigned long long)*n_values);
    if (!on_device) {
        int rc = pinned_acquire(p, *n_values * ob, values);
        if (rc != FBR_OK) return rc;
        for (SeqPart& b : blocks) b.emit.host = (uint8_t*)*values + b.emit.base * ob;
    }
    for (SeqPart& b : blocks)
        if (!b.emit.h_offs) {
            Worker& w = p->workers[b.worker];
            CK(cudaSetDevice(w.device));
            CK(cudaMallocAsync(&b.emit.d_values, std::max<uint64_t>(16, b.emit.total * ob), w.s_comp));
        }
    return FBR_OK;
}

// An emit map: the count pass is an ordinary map of the body whose records (the tasks' counts) stay on the device; once it
// is done, scan_counts_kernel turns each block's counts into its offsets and total, the host sizes the values segment from
// the totals, and the emit pass runs as a second ordinary map over the same blocks.
static int emit_submit(fbr_pool_t* p, const fbr_map_desc_t* d, const fbr_items_desc_t* items, uint32_t n_streams, uint64_t* seq_out) {
    const BodyEntry& body = *body_of(d->func_id);
    if (d->out || (d->flags & FBR_OUT_DEVICE))
        return fail(FBR_EINVAL, "body %s emits variable-length results: its maps own their output (no out, no FBR_OUT_DEVICE)", body.name.c_str());
    const bool on_device = (d->flags & FBR_RESULTS_ON_DEVICE) != 0;
    const bool whole_block = (d->flags & (FBR_RESILIENT | FBR_FULL_WINDOW)) != 0;   // units may be re-dispatched: no waves
    // 1. the count pass
    fbr_map_desc_t cd = *d;
    cd.flags |= FBR_RESULTS_ON_DEVICE;
    uint64_t cseq = 0;
    int rc = map_submit_pass(p, &cd, items, n_streams, &cseq);
    if (rc != FBR_OK) return rc;
    fbr_result_t cres;
    rc = fbr_result_wait(p, cseq, -1, &cres);
    // 2. scan each block, then one wait per block outside the pool lock: then every total is in
    std::vector<SeqPart> blocks;                       // the count pass's blocks, each with its emit state
    uint64_t* totals = nullptr;
    std::vector<std::pair<int, cudaEvent_t>> scanned;  // (device, event after its block's scan)
    if (rc == FBR_OK) rc = emit_scan(p, cseq, !on_device && !whole_block, blocks, &totals, scanned);
    for (auto& s : scanned) {
        cudaSetDevice(s.first);
        if (rc == FBR_OK && cudaEventSynchronize(s.second) != cudaSuccess) rc = fail(FBR_ECUDA, "waiting for scan_counts_kernel failed");
        cudaEventDestroy(s.second);
    }
    // 3. size and place the values
    void* values = nullptr;
    uint64_t n_values = 0;
    if (rc == FBR_OK) rc = emit_place(p, body, on_device, blocks, totals, &values, &n_values);
    {
        // the count pass and the totals are done with; if the count pass failed, the map is born finished with its error
        // (fbr_result_wait reports it)
        std::lock_guard<std::mutex> g(p->mu);
        uint32_t err_code = 0;
        uint64_t err_task = 0;
        auto it = p->seqs.find(cseq);
        if (it != p->seqs.end()) {
            SeqState& cs = *it->second;
            err_code = cs.err_code;
            err_task = cs.err_task;
            if (rc != FBR_ETASK) harvest(p, cs);   // as fbr_result_release does (a no-op once the wait succeeded)
            free_seq(p, cs);
            p->seqs.erase(it);
        }
        if (totals) pinned_release(p, totals);
        if (rc == FBR_ETASK) {
            std::unique_ptr<SeqState> st(new SeqState());
            st->seq = ++p->next_seq;
            st->n_tasks = d->n_tasks;
            st->func_id = d->func_id;
            st->flags = d->flags;
            st->result_bytes = body.result_bytes;
            st->result_kind = body.result_kind;
            st->desc = *d;
            st->finished = true;
            st->err_code = err_code;
            st->err_task = err_task;
            p->stats.tasks_submitted += d->n_tasks;
            *seq_out = st->seq;
            p->seqs[st->seq] = std::move(st);
            return FBR_OK;
        }
    }
    // 4. the emit pass
    if (rc == FBR_OK) rc = map_submit_pass(p, d, items, n_streams, seq_out, &blocks, &values, n_values);
    if (rc != FBR_OK) {   // free what the emit pass did not take over
        const std::string msg = g_err;
        std::lock_guard<std::mutex> g(p->mu);
        for (SeqPart& b : blocks) free_emit_block(p, b.worker, b.emit);
        if (values) pinned_release(p, values);
        g_err = msg;
    }
    return rc;
}

static int map_submit_pass(fbr_pool_t* p, const fbr_map_desc_t* d, const fbr_items_desc_t* items, uint32_t n_streams, uint64_t* seq_out,
                           std::vector<SeqPart>* counted, void** values, uint64_t n_values) {
    std::lock_guard<std::mutex> g(p->mu);
    if (p->state != ST_RUN) return fail(FBR_ESTATE, "Pool is not running");
    if (!body_of(d->func_id)) return fail(FBR_EINVAL, "bad func_id %d", d->func_id);
    const BodyEntry& body = *body_of(d->func_id);
    const bool dev_mode = (d->flags & (FBR_ARGS_DEVICE | FBR_OUT_DEVICE)) != 0;
    if (dev_mode && p->workers.size() != 1 && !ensure_peer_access(p))
        return fail(FBR_EINVAL, "device-resident args/out on a multi-worker pool need peer access between all its GPUs");
    if ((body.flags & FBR_BODY_ITEMS) && body.arg_bytes == 0) {
        if (d->arg_stride != 0) return fail(FBR_EINVAL, "body %s has no head record (arg_stride must be 0)", body.name.c_str());
    } else if (d->arg_stride == 0) {
        if (!(body.flags & FBR_BODY_INDEX_ARG))
            return fail(FBR_EINVAL, "body %s needs explicit argument records (arg_stride=0)", body.name.c_str());
    } else if (body.flags & FBR_BODY_INDEX_ONLY) {
        return fail(FBR_EINVAL, "body %s takes range() arguments only (arg_stride must be 0)", body.name.c_str());
    } else if (body.flags & FBR_BODY_RECORD) {
        // dispatch_record_kernel copies argument records of any 4 B aligned layout (bulk loads where 16 B aligned)
        if (d->arg_stride < body.arg_bytes || (d->arg_stride % 4) != 0)
            return fail(FBR_EINVAL, "arg_stride %u invalid for body %s (arg_bytes %u)", d->arg_stride, body.name.c_str(), body.arg_bytes);
        if (d->n_tasks && !d->args) return fail(FBR_EINVAL, "args is NULL");
        if ((uintptr_t)d->args % 4) return fail(FBR_EINVAL, "argument records of body %s must be 4-byte aligned", body.name.c_str());
    } else {
        if (d->arg_stride < body.arg_bytes || (d->arg_stride % 8) != 0)
            return fail(FBR_EINVAL, "arg_stride %u invalid for body %s (arg_bytes %u)", d->arg_stride, body.name.c_str(), body.arg_bytes);
        if (d->n_tasks && !d->args) return fail(FBR_EINVAL, "args is NULL");
        if (body.arg_bytes >= 16 && body.result_kind != FBR_RES_BITS8 && (d->arg_stride % 16 || ((uintptr_t)d->args % 16)))
            return fail(FBR_EINVAL, "argument records of body %s must be 16-byte aligned", body.name.c_str());
    }
    if (body.flags & FBR_BODY_BROADCAST) {
        // run() iterates over shared_bytes / elem_bytes elements: the block must hold exactly that many
        if (!d->shared || d->shared_bytes == 0)
            return fail(FBR_EINVAL, "body %s needs a broadcast block", body.name.c_str());
        if (d->shared_bytes % body.shared_elem_bytes)
            return fail(FBR_EINVAL, "body %s: broadcast block of %llu bytes is not a whole number of %u-byte elements", body.name.c_str(),
                        (unsigned long long)d->shared_bytes, body.shared_elem_bytes);
    } else if ((body.flags & FBR_BODY_NEEDS_SHARED) && (!d->shared || d->shared_bytes < sizeof(ParzenShared))) {
        return fail(FBR_EINVAL, "body %s needs a shared argument block", body.name.c_str());
    }
    if (d->shared && d->shared_bytes && (d->flags & FBR_SHARED_HANDLE)) {
        // a kernel reads shared_bytes from the handle's allocation: it must not claim more than fbr_shared_put uploaded
        auto it = p->shared.find((uint64_t)(uintptr_t)d->shared);
        if (it == p->shared.end()) return fail(FBR_ENOENT, "unknown shared handle");
        if (d->shared_bytes > it->second.bytes)
            return fail(FBR_EINVAL, "shared_bytes %llu exceeds the %llu bytes of shared handle %llu", (unsigned long long)d->shared_bytes,
                        (unsigned long long)it->second.bytes, (unsigned long long)(uintptr_t)d->shared);
    }
    if ((d->flags & FBR_OUT_DEVICE) && !d->out) return fail(FBR_EINVAL, "FBR_OUT_DEVICE without out");
    if ((d->flags & FBR_RESULTS_ON_DEVICE) && ((d->flags & FBR_OUT_DEVICE) || d->out))
        return fail(FBR_EINVAL, "FBR_RESULTS_ON_DEVICE owns its output buffer: do not pass out / FBR_OUT_DEVICE");
    if ((d->flags & FBR_RESILIENT) && (d->flags & FBR_SHUFFLE)) return fail(FBR_EINVAL, "FBR_RESILIENT cannot be combined with FBR_SHUFFLE");
    if (d->flags & FBR_FOLD_SPARSE_KEYS) {
        if (!(body.flags & FBR_BODY_KEYED))
            return fail(FBR_EINVAL, "body %s has no key(): its maps cannot fold per key (FBR_FOLD_SPARSE_KEYS needs FBR_BODY_KEYED)", body.name.c_str());
        if (d->flags & (FBR_FOLD | FBR_SCAN | FBR_FOLD_KEYS))
            return fail(FBR_EINVAL, "FBR_FOLD_SPARSE_KEYS cannot be combined with FBR_FOLD, FBR_SCAN or FBR_FOLD_KEYS");
        if (d->out || (d->flags & (FBR_OUT_DEVICE | FBR_WANT_SUM | FBR_NO_ZERO_COPY)))
            return fail(FBR_EINVAL, "a sparse keyed fold map (FBR_FOLD_SPARSE_KEYS) of body %s owns its result records: no out, "
                        "FBR_OUT_DEVICE, FBR_WANT_SUM or FBR_NO_ZERO_COPY", body.name.c_str());
        if (d->n_keys != 0)
            return fail(FBR_EINVAL, "a sparse keyed fold map (FBR_FOLD_SPARSE_KEYS) takes no n_keys (%u): its keys are any uint32 "
                        "but 0xFFFFFFFF", d->n_keys);
        if (d->n_tasks > 0xffffffffull)   // a block's tasks are sorted as uint32 indices
            return fail(FBR_EINVAL, "a sparse keyed fold map takes fewer than 2^32 tasks (%llu)", (unsigned long long)d->n_tasks);
    }
    // (before the generic FBR_WANT_SUM check: a scan body is never summable, and the scan map says why)
    if (d->flags & FBR_SCAN) {
        if (!(body.flags & FBR_BODY_SCAN))
            return fail(FBR_EINVAL, "body %s exports no scan entry: its maps cannot return prefix folds (FBR_SCAN needs FBR_BODY_SCAN)", body.name.c_str());
        if (d->flags & FBR_FOLD) return fail(FBR_EINVAL, "FBR_SCAN returns every prefix of the fold: it cannot be combined with FBR_FOLD");
        if (d->out || (d->flags & FBR_OUT_DEVICE))
            return fail(FBR_EINVAL, "a scan map (FBR_SCAN) of body %s owns its result window: no out or FBR_OUT_DEVICE", body.name.c_str());
        if (d->flags & FBR_WANT_SUM) return fail(FBR_EINVAL, "a scan map (FBR_SCAN) has no sum of its results (FBR_WANT_SUM)");
        if (d->flags & FBR_NO_ZERO_COPY)
            return fail(FBR_EINVAL, "a scan map (FBR_SCAN) always stages its results on the device: FBR_NO_ZERO_COPY does not apply");
    }
    if (d->flags & FBR_FOLD_KEYS) {
        if (!(body.flags & FBR_BODY_KEYED))
            return fail(FBR_EINVAL, "body %s has no key(): its maps cannot fold per key (FBR_FOLD_KEYS needs FBR_BODY_KEYED)", body.name.c_str());
        if (d->flags & (FBR_FOLD | FBR_SCAN)) return fail(FBR_EINVAL, "FBR_FOLD_KEYS cannot be combined with FBR_FOLD or FBR_SCAN");
        if (d->out || (d->flags & (FBR_OUT_DEVICE | FBR_WANT_SUM | FBR_NO_ZERO_COPY)))
            return fail(FBR_EINVAL, "a keyed fold map (FBR_FOLD_KEYS) of body %s owns its result records: no out, FBR_OUT_DEVICE, "
                        "FBR_WANT_SUM or FBR_NO_ZERO_COPY", body.name.c_str());
        if (d->n_keys < 1 || d->n_keys > FBR_MAX_KEYS)
            return fail(FBR_EINVAL, "n_keys %u is not in 1 .. %u", d->n_keys, (unsigned)FBR_MAX_KEYS);
        if ((uint64_t)d->n_keys * body.result_bytes > p->ring_bytes)
            return fail(FBR_EINVAL, "n_keys %u records of %u bytes exceed ring_bytes %llu", d->n_keys, body.result_bytes,
                        (unsigned long long)p->ring_bytes);
        if (d->n_tasks > 0xffffffffull)   // a block's tasks are sorted as uint32 indices
            return fail(FBR_EINVAL, "a keyed fold map takes fewer than 2^32 tasks (%llu)", (unsigned long long)d->n_tasks);
    }
    if ((d->flags & FBR_WANT_SUM) && !(body.flags & FBR_BODY_SUMMABLE))
        return fail(FBR_EINVAL, "body %s results cannot be summed", body.name.c_str());
    if (d->flags & FBR_FOLD) {
        if (!(body.flags & FBR_BODY_FOLD)) return fail(FBR_EINVAL, "body %s has no combine(): its maps cannot fold (FBR_FOLD)", body.name.c_str());
        if (d->out || (d->flags & (FBR_OUT_DEVICE | FBR_WANT_SUM | FBR_NO_ZERO_COPY)))
            return fail(FBR_EINVAL, "a fold map (FBR_FOLD) of body %s owns its one result record: no out, FBR_OUT_DEVICE, "
                        "FBR_WANT_SUM or FBR_NO_ZERO_COPY", body.name.c_str());
    }

    // A submission can find out that a worker has died (its context rejects every call): the worker is
    // retired, maps in flight are re-dispatched or failed (on_worker_death) and this map is cut again over
    // the survivors -- at most once per worker.
    for (size_t round = 0; round <= p->workers.size(); ++round) {
        std::vector<int> live;
        for (size_t i = 0; i < p->workers.size(); ++i)
            if (!p->workers[i].dead) live.push_back((int)i);
        if (live.empty()) return fail(FBR_ECUDA, "every worker of this pool has died (last CUDA error: %s)",
                                      cudaGetErrorString((cudaError_t)p->workers[0].death_error));
        if (dev_mode && p->workers[0].dead)
            return fail(FBR_ECUDA, "worker 0, which holds the device-resident arguments / output, has died");
        std::unique_ptr<SeqState> st(new SeqState());
        st->seq = ++p->next_seq;
        st->n_tasks = d->n_tasks;
        st->func_id = d->func_id;
        st->flags = d->flags;
        st->result_bytes = body.result_bytes;
        st->result_kind = body.result_kind;
        st->out = d->out;
        st->desc = *d;
        memset(st->items, 0, sizeof st->items);
        st->n_item_streams = items ? n_streams : 0;
        for (uint32_t k = 0; k < st->n_item_streams; ++k) st->items[k] = items[k];
        const bool fold = (d->flags & FBR_FOLD) != 0, keyed = (d->flags & FBR_FOLD_KEYS) != 0;
        const bool sparse = (d->flags & FBR_FOLD_SPARSE_KEYS) != 0;
        const bool need_segment = !st->out && d->n_tasks && !(d->flags & FBR_RESULTS_ON_DEVICE) && !fold && !keyed && !sparse;
        // host allocations fail with the sticky error too once a context of this process has died: tell the two apart
        auto died_meanwhile = [&]() {
            bool any = false;
            for (int wi : live) any |= retire_if_dead(p, wi);
            return any;
        };
        if (need_segment && live.size() == 1) {
            int rc = pinned_acquire(p, d->n_tasks * body.result_bytes, &st->out);
            if (rc != FBR_OK) {
                const std::string msg = g_err;
                if (died_meanwhile()) continue;
                g_err = msg;
                return rc;
            }
            st->own_out = true;
        }
        // contiguous task blocks per live worker, cut on claim-unit boundaries (block partition ==
        // PUSH round-robin with chunk = block, SURVEY.md 8(e))
        cut_blocks(p, body, *d, 0, d->n_tasks, live, d->attempt, st->parts);
        if (fold) {
            // the result record, then each block's total in block order; pinned memory is mapped into every device, where
            // each block's fold_tree_kernel writes its total
            int rc = pinned_acquire(p, (1 + st->parts.size()) * (uint64_t)body.result_bytes, &st->out);
            if (rc != FBR_OK) return rc;
            st->own_out = true;
            for (size_t k = 0; k < st->parts.size(); ++k) st->parts[k].cx.fold_total = (uint8_t*)st->out + (1 + k) * body.result_bytes;
        }
        if (keyed) {
            // the result: n_keys records, then n_keys uint64 counts.  A single block writes its totals and counts there;
            // several each write theirs to an area of the same layout after it, combined by complete_map
            const uint64_t K = d->n_keys, area = K * (body.result_bytes + sizeof(uint64_t));
            const size_t nb = st->parts.size();
            int rc = pinned_acquire(p, (nb > 1 ? 1 + nb : 1) * area, &st->out);
            if (rc != FBR_OK) return rc;
            st->own_out = true;
            for (size_t k = 0; k < nb; ++k) {
                uint8_t* const a = (uint8_t*)st->out + (nb > 1 ? 1 + k : 0) * area;
                st->parts[k].cx.key_totals = a;
                st->parts[k].cx.key_counts = a + K * body.result_bytes;
            }
        }
        if (sparse && !st->parts.empty()) {
            // each block's D, written by its run scan; the result is sized at completion, once every D is known
            int rc = pinned_acquire(p, st->parts.size() * sizeof(uint64_t), (void**)&st->sparse_words);
            if (rc != FBR_OK) return rc;
            for (size_t k = 0; k < st->parts.size(); ++k) st->parts[k].cx.n_groups = st->sparse_words + k;
        }
        if (counted) {
            // the emit pass runs over the blocks the count pass counted
            bool same = counted->size() == st->parts.size();
            for (size_t k = 0; same && k < st->parts.size(); ++k) {
                const SeqPart& c = (*counted)[k];
                const SeqPart& part = st->parts[k];
                same = c.worker == part.worker && c.first == part.first && c.count == part.count;
            }
            if (!same) {
                free_seq(p, *st);
                return fail(FBR_ECUDA, "body %s: the pool's workers changed between the count and the emit pass", body.name.c_str());
            }
            for (size_t k = 0; k < st->parts.size(); ++k) st->parts[k].emit = (*counted)[k].emit;
            counted->clear();
            st->emit_pass = true;
            st->values = *values;
            *values = nullptr;
            st->n_values = n_values;
        }
        if (need_segment && live.size() > 1) {
            // several GPUs fill one segment: bind each worker's block to its GPU's NUMA node
            std::vector<NumaBlock> blocks;
            for (auto& part : st->parts)
                blocks.push_back({part.first * body.result_bytes, part.count * body.result_bytes, p->workers[part.worker].numa_node});
            int rc = numa_pinned_acquire(p, d->n_tasks * body.result_bytes, blocks, &st->out);
            if (rc != FBR_OK) {
                const std::string msg = g_err;
                if (died_meanwhile()) continue;
                g_err = msg;
                return rc;
            }
            st->own_out = true;
        }
        int failed_worker = -1, rc = FBR_OK;
        if (st->parts.size() > 1) {
            // one submit thread per worker (see SubmitThread); this thread holds the pool lock meanwhile
            if (p->submitters.size() < p->workers.size()) p->submitters.resize(p->workers.size());
            SeqState* stp = st.get();
            for (auto& part : st->parts) {
                auto& sub = p->submitters[part.worker];
                if (!sub) sub.reset(new SubmitThread());
                SeqPart* pp = &part;
                sub->post([p, stp, pp, &body] { return submit_part(p, *stp, *pp, body); });
            }
            for (auto& part : st->parts) {
                std::string msg;
                const int r = p->submitters[part.worker]->wait(&msg);
                if (r != FBR_OK && rc == FBR_OK) { rc = r; failed_worker = part.worker; g_err = msg; }
            }
        } else {
            for (auto& part : st->parts) {
                rc = submit_part(p, *st, part, body);
                if (rc != FBR_OK) { failed_worker = part.worker; break; }
            }
        }
        if (rc == FBR_OK) {
            p->stats.tasks_submitted += d->n_tasks;
            *seq_out = st->seq;
            p->seqs[st->seq] = std::move(st);
            return FBR_OK;
        }
        const std::string msg = g_err;
        const bool died = retire_if_dead(p, failed_worker);   // before free_seq: its parts on that worker are skipped
        free_seq(p, *st);
        if (!died) { g_err = msg; return rc; }
    }
    return fail(FBR_ECUDA, "submission kept failing while workers died");
}

static int first_live_worker(fbr_pool* p) {
    for (size_t i = 0; i < p->workers.size(); ++i)
        if (!p->workers[i].dead) return (int)i;
    return -1;
}

// tree() over n host records of fold body `body` into `out` (host), on the pool's first live worker; blocks until done.
// The caller holds the pool lock: the work goes to the worker's own s_fold, where no map's waves queue, so the wait is one
// small launch long.  A worker whose context died on the way is retired (on_worker_death), and the fold fails with FBR_ECUDA.
static int fold_host_records(fbr_pool* p, const BodyEntry& body, const void* values, uint64_t n, void* out) {
    const uint64_t R = body.result_bytes;
    if (n <= 1) {   // tree() of no record is the identity, of one record the record
        memmove(out, n ? values : body.identity.data(), R);
        return FBR_OK;
    }
    const int wi = first_live_worker(p);
    if (wi < 0) return fail(FBR_ECUDA, "every worker of this pool has died");
    Worker& w = p->workers[wi];
    uint8_t* d = nullptr;   // the n records, then the result
    cudaError_t e = cudaSetDevice(w.device);
    if (e == cudaSuccess) e = cudaMallocAsync((void**)&d, (n + 1) * R, w.s_fold);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d, values, n * R, cudaMemcpyHostToDevice, w.s_fold);
    if (e == cudaSuccess) {
        body.fold(d, n, d + n * R, (void*)w.s_fold);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(out, d + n * R, R, cudaMemcpyDeviceToHost, w.s_fold);
    if (d) cudaFreeAsync(d, w.s_fold);
    if (e == cudaSuccess) e = cudaStreamSynchronize(w.s_fold);
    if (e != cudaSuccess) {
        retire_if_dead(p, wi);
        return fail(FBR_ECUDA, "folding %llu records of body %s on worker %d: %s", (unsigned long long)n, body.name.c_str(), wi,
                    cudaGetErrorString(e));
    }
    p->stats.h2d_bytes += n * R;
    p->stats.d2h_bytes += R;
    return FBR_OK;
}

// tree() of each segment [offsets[k], offsets[k + 1]) of the host records `values` of keyed body `body` into out[k] (host),
// identity() for an empty segment, on the pool's first live worker's s_fold; blocks until done.  As fold_host_records.
static int fold_segments_host(fbr_pool* p, const BodyEntry& body, const void* values, const uint64_t* offsets, uint32_t S, void* out) {
    const uint64_t R = body.result_bytes, n = offsets[S];
    if (S == 0) return FBR_OK;
    const int wi = first_live_worker(p);
    if (wi < 0) return fail(FBR_ECUDA, "every worker of this pool has died");
    Worker& w = p->workers[wi];
    uint8_t* d = nullptr;   // the n records, the S results, the S + 1 offsets
    const uint64_t o_out = n * R, o_offs = round_up(o_out + S * R, 8);
    cudaError_t e = cudaSetDevice(w.device);
    if (e == cudaSuccess) e = cudaMallocAsync((void**)&d, o_offs + (S + 1) * 8ull, w.s_fold);
    if (e == cudaSuccess && n) e = cudaMemcpyAsync(d, values, n * R, cudaMemcpyHostToDevice, w.s_fold);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d + o_offs, offsets, (S + 1) * 8ull, cudaMemcpyHostToDevice, w.s_fold);
    if (e == cudaSuccess) e = (cudaError_t)body.fold_segments(d, n, (const uint64_t*)(d + o_offs), S, d + o_out, (void*)w.s_fold);
    if (e == cudaSuccess) e = cudaMemcpyAsync(out, d + o_out, S * R, cudaMemcpyDeviceToHost, w.s_fold);
    if (d) cudaFreeAsync(d, w.s_fold);
    if (e == cudaSuccess) e = cudaStreamSynchronize(w.s_fold);
    if (e != cudaSuccess) {
        retire_if_dead(p, wi);
        return fail(FBR_ECUDA, "folding %u segments of %llu records of body %s on worker %d: %s", S, (unsigned long long)n,
                    body.name.c_str(), wi, cudaGetErrorString(e));
    }
    p->stats.h2d_bytes += n * R + (S + 1) * 8ull;
    p->stats.d2h_bytes += S * R;
    return FBR_OK;
}

// FBR_FOLD_KEYS with several blocks, once every block is done: each block's totals and counts are in its area of the pinned
// segment.  Record k is tree() over the totals of the blocks where key k has tasks, in block order -- one fold_segments_host
// over the key-major sequence of those totals -- and count k the sum of the blocks' counts.
static int keyed_finish(fbr_pool* p, SeqState& st) {
    const BodyEntry& body = *body_of(st.func_id);
    const uint64_t K = st.desc.n_keys, R = body.result_bytes;
    const std::vector<SeqPart*> blocks = parts_in_order(st);
    std::vector<uint64_t> offs(K + 1, 0), counts(K, 0);
    std::vector<uint8_t> values;
    for (uint64_t k = 0; k < K; ++k) {
        offs[k] = values.size() / R;
        for (const SeqPart* b : blocks) {
            uint64_t c;
            memcpy(&c, b->cx.key_counts + k * 8, 8);
            if (!c) continue;
            values.insert(values.end(), b->cx.key_totals + k * R, b->cx.key_totals + (k + 1) * R);
            counts[k] += c;
        }
    }
    offs[K] = values.size() / R;
    const int rc = fold_segments_host(p, body, values.data(), offs.data(), (uint32_t)K, st.out);
    if (rc != FBR_OK) return rc;
    memcpy((uint8_t*)st.out + K * R, counts.data(), K * 8);
    return FBR_OK;
}

// Where sparse_keyed_finish puts block b's D totals, D keys and D + 1 run starts in its pinned buffer.
static uint64_t sparse_host_layout(uint64_t D, uint64_t R, uint64_t* o_keys, uint64_t* o_starts) {
    *o_keys = round_up(D * R, 8);
    *o_starts = round_up(*o_keys + 4 * D, 8);
    return *o_starts + 8 * (D + 1);
}

// FBR_FOLD_SPARSE_KEYS, once every block is done: block b's D_b is in its pinned word, and its gathered records, run starts
// and keys are on its worker's device (sparse_block_step).  The first call queues, for each block, the body's fold_segments
// entry over its D_b runs on its worker's s_fold, then the D2H copy of the D_b totals, keys and starts into pinned memory,
// behind the event st.block_done[b]; a call that failed part-way resumes at the first block without one.  Once every copy
// is in, one block's totals are the result.  Several blocks' sorted keys are merged on the host, stable by key with block
// order inside a key, which gives the key-major sequence of block totals and its offsets: one fold_segments_host folds it
// and the counts are summed.  The result records are sized exactly here.  With `block` the copies are waited for here;
// otherwise *ready tells whether they have all finished (fbr_result_wait waits for them outside the lock).
static int sparse_keyed_finish(fbr_pool* p, SeqState& st, bool block, bool* ready) {
    const BodyEntry& body = *body_of(st.func_id);
    const uint64_t R = body.result_bytes;
    const std::vector<SeqPart*> blocks = parts_in_order(st);
    const size_t nb = blocks.size();
    if (st.block_done.empty()) {
        st.block_done.assign(nb, nullptr);
        st.sparse_host.assign(nb, nullptr);
    }
    for (size_t b = 0; b < nb; ++b) {
        if (st.block_done[b]) continue;           // queued by an earlier call
        SeqPart& part = *blocks[b];
        Worker& w = p->workers[part.worker];
        if (w.dead) return fail(FBR_ECUDA, "worker %d died before its block of a sparse keyed fold map was folded", part.worker);
        const uint64_t D = *part.cx.n_groups;
        uint64_t o_starts, o_dkeys, h_keys, h_starts;
        sparse_keep_layout(part.count, R, &o_starts, &o_dkeys);
        const uint64_t hbytes = sparse_host_layout(D, R, &h_keys, &h_starts);
        if (!st.sparse_host[b]) {
            const int rc = pinned_acquire(p, hbytes, &st.sparse_host[b]);
            if (rc != FBR_OK) return rc;
        }
        uint8_t* const h = (uint8_t*)st.sparse_host[b];
        uint8_t* const keep = (uint8_t*)part.d_sparse;
        uint8_t* totals = nullptr;
        cudaError_t e = cudaSetDevice(w.device);
        if (e == cudaSuccess) e = cudaMallocAsync((void**)&totals, D * R, w.s_fold);
        if (e == cudaSuccess)
            e = (cudaError_t)body.fold_segments(keep, part.count, (const uint64_t*)(keep + o_starts), (uint32_t)D, totals, (void*)w.s_fold);
        if (e == cudaSuccess) e = cudaMemcpyAsync(h, totals, D * R, cudaMemcpyDeviceToHost, w.s_fold);
        if (e == cudaSuccess) e = cudaMemcpyAsync(h + h_keys, keep + o_dkeys, 4 * D, cudaMemcpyDeviceToHost, w.s_fold);
        if (e == cudaSuccess) e = cudaMemcpyAsync(h + h_starts, keep + o_starts, 8 * (D + 1), cudaMemcpyDeviceToHost, w.s_fold);
        if (totals) cudaFreeAsync(totals, w.s_fold);
        cudaEvent_t ev = nullptr;
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventRecord(ev, w.s_fold);
        if (e != cudaSuccess) {
            if (ev) cudaEventDestroy(ev);
            retire_if_dead(p, part.worker);
            return fail(FBR_ECUDA, "folding the runs of block %zu of a sparse keyed fold map of body %s on worker %d: %s", b,
                        body.name.c_str(), part.worker, cudaGetErrorString(e));
        }
        st.block_done[b] = ev;
        cudaFreeAsync(part.d_sparse, w.s_fold);   // behind the copies
        part.d_sparse = nullptr;
        p->stats.d2h_bytes += D * R + 4 * D + 8 * (D + 1);
    }
    for (size_t b = 0; b < nb; ++b) {
        const int wi = blocks[b]->worker;
        cudaError_t q = p->workers[wi].dead ? cudaErrorUnknown : cudaSetDevice(p->workers[wi].device);
        if (q == cudaSuccess) q = block ? cudaEventSynchronize(st.block_done[b]) : cudaEventQuery(st.block_done[b]);
        if (q == cudaErrorNotReady) { cudaGetLastError(); *ready = false; return FBR_OK; }
        if (q != cudaSuccess) {
            retire_if_dead(p, wi);
            return fail(FBR_ECUDA, "folding the runs of block %zu of a sparse keyed fold map on worker %d: %s", b, wi, cudaGetErrorString(q));
        }
    }
    *ready = true;
    // block b's totals, keys and counts (differences of its run starts)
    struct Run { uint32_t key; uint32_t block; uint64_t at; };   // the block's run number
    std::vector<Run> runs;
    std::vector<const uint64_t*> starts(nb);
    for (size_t b = 0; b < nb; ++b) {
        const uint64_t D = *blocks[b]->cx.n_groups;
        uint64_t h_keys, h_starts;
        sparse_host_layout(D, R, &h_keys, &h_starts);
        const uint8_t* h = (const uint8_t*)st.sparse_host[b];
        starts[b] = (const uint64_t*)(h + h_starts);
        for (uint64_t r = 0; r < D; ++r) runs.push_back({((const uint32_t*)(h + h_keys))[r], (uint32_t)b, r});
    }
    // stable: within one key the runs stay in block order
    if (nb > 1) std::stable_sort(runs.begin(), runs.end(), [](const Run& a, const Run& b) { return a.key < b.key; });
    std::vector<uint32_t> keys;
    std::vector<uint64_t> counts, offs;
    for (size_t i = 0; i < runs.size(); ++i) {
        const Run& r = runs[i];
        const uint64_t c = starts[r.block][r.at + 1] - starts[r.block][r.at];
        if (i == 0 || r.key != runs[i - 1].key) {
            keys.push_back(r.key);
            counts.push_back(0);
            offs.push_back(i);
        }
        counts.back() += c;
    }
    offs.push_back(runs.size());
    const uint64_t D = keys.size();
    void* out = nullptr;
    if (D) {
        int rc = pinned_acquire(p, D * R, &out);
        if (rc != FBR_OK) return rc;
        if (nb == 1) {
            memcpy(out, st.sparse_host[0], D * R);
        } else {
            std::vector<uint8_t> values(runs.size() * R);
            for (size_t i = 0; i < runs.size(); ++i)
                memcpy(&values[i * R], (const uint8_t*)st.sparse_host[runs[i].block] + runs[i].at * R, R);
            rc = fold_segments_host(p, body, values.data(), offs.data(), (uint32_t)D, out);
            if (rc != FBR_OK) {
                pinned_release(p, out);
                return rc;
            }
        }
    }
    st.out = out;
    st.own_out = out != nullptr;
    st.group_keys.swap(keys);
    st.group_counts.swap(counts);
    for (void*& h : st.sparse_host) {
        pinned_release(p, h);
        h = nullptr;
    }
    return FBR_OK;
}

// Queues on worker w's s_fold the wrap of the n records at `values` (w's device memory, rewritten in place) with the m host
// records `pieces`, right-nested: the body's scan entry without its prefix step.  With `host`, the wrapped records are then
// copied there; with `done`, an event is created there and recorded behind it all.  Nothing is waited for, but an upload
// from pageable memory is staged before it returns, so pageable `pieces` may be freed then.
static cudaError_t queue_wrap(Worker& w, const BodyEntry& body, const void* pieces, uint32_t m, uint8_t* values, uint64_t n,
                              void* host, cudaEvent_t* done) {
    const uint64_t R = body.result_bytes;
    uint8_t* d = nullptr;
    cudaError_t e = cudaSetDevice(w.device);
    if (e == cudaSuccess) e = cudaMallocAsync((void**)&d, m * R, w.s_fold);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d, pieces, m * R, cudaMemcpyHostToDevice, w.s_fold);
    if (e == cudaSuccess) e = (cudaError_t)body.scan(values, n, 0, d, m, (void*)w.s_fold);
    if (e == cudaSuccess && host) e = cudaMemcpyAsync(host, values, n * R, cudaMemcpyDeviceToHost, w.s_fold);
    if (d) cudaFreeAsync(d, w.s_fold);
    cudaEvent_t ev = nullptr;
    if (e == cudaSuccess && done) e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
    if (e == cudaSuccess && done) e = cudaEventRecord(ev, w.s_fold);
    if (e == cudaSuccess && done) *done = ev;
    else if (ev) cudaEventDestroy(ev);
    return e;
}

// FBR_SCAN, once every block is done: each block's window holds its own prefix folds (its last record is its total t_k),
// and every block but the first is still on its worker's device.  Block b > 0 is wrapped with the pieces G_1 .. G_m of
// t_0 .. t_{b-1} -- tree() over the aligned power-of-two ranges of block totals given by the set bits of b, largest first
// -- which gives tree(t_0, ..., t_{b-1}, p_i) (the same identity as within a block, over b + 1 elements).
//
// The caller holds the pool lock.  The first call reads every block's total into st.scan_totals (R bytes per block)
// before any block is wrapped: a wrap rewrites the record that holds its block's total.  Then, block by block, the pieces
// are folded from those totals and the wrap is queued on the block's own worker's s_fold (queue_wrap), host results with
// their one D2H copy into the pinned segment, behind the event st.block_done[b].  A call that failed part-way resumes at the
// first block without one and folds the same pieces from the kept totals.  With `block` the wraps are waited for here;
// otherwise *ready tells whether they have all finished (fbr_result_wait waits for them outside the lock).
static int scan_finish(fbr_pool* p, SeqState& st, bool block, bool* ready) {
    const BodyEntry& body = *body_of(st.func_id);
    const uint64_t R = body.result_bytes;
    const bool on_device = (st.flags & FBR_RESULTS_ON_DEVICE) != 0;
    const std::vector<SeqPart*> blocks = parts_in_order(st);
    const size_t nb = blocks.size();
    if (nb > 1 && st.scan_totals.empty()) {
        std::vector<uint8_t> totals(nb * R);
        for (size_t k = 0; k < nb; ++k) {
            const SeqPart& part = *blocks[k];
            Worker& w = p->workers[part.worker];
            if (w.dead) return fail(FBR_ECUDA, "worker %d died before its block of a scan map was wrapped", part.worker);
            cudaError_t e = cudaSetDevice(w.device);
            if (e == cudaSuccess) e = cudaMemcpyAsync(&totals[k * R], part.cx.window_base + (part.count - 1) * R, R, cudaMemcpyDeviceToHost, w.s_fold);
            if (e == cudaSuccess) e = cudaStreamSynchronize(w.s_fold);
            if (e != cudaSuccess) {
                retire_if_dead(p, part.worker);
                return fail(FBR_ECUDA, "reading the total of a scan block on worker %d: %s", part.worker, cudaGetErrorString(e));
            }
        }
        st.scan_totals.swap(totals);
        st.block_done.assign(nb, nullptr);
    }
    for (size_t b = 1; b < nb; ++b) {
        if (st.block_done[b]) continue;            // queued by an earlier call
        SeqPart& part = *blocks[b];
        Worker& w = p->workers[part.worker];
        if (w.dead) return fail(FBR_ECUDA, "worker %d died before its block of a scan map was wrapped", part.worker);
        std::vector<uint8_t> pieces;
        for (int k = 63; k >= 0; --k) {
            if (!((b >> k) & 1)) continue;
            const uint64_t lo = (b >> (k + 1)) << (k + 1);
            pieces.resize(pieces.size() + R);
            const int rc = fold_host_records(p, body, &st.scan_totals[lo * R], 1ull << k, &pieces[pieces.size() - R]);
            if (rc != FBR_OK) return rc;
        }
        const uint32_t m = (uint32_t)(pieces.size() / R);
        uint8_t* const host = on_device ? nullptr : (uint8_t*)st.out + part.first * R;
        const cudaError_t e = queue_wrap(w, body, pieces.data(), m, part.cx.window_base, part.count, host, &st.block_done[b]);
        if (e != cudaSuccess) {
            retire_if_dead(p, part.worker);
            return fail(FBR_ECUDA, "wrapping block %zu of a scan map of body %s on worker %d: %s", b, body.name.c_str(), part.worker,
                        cudaGetErrorString(e));
        }
        p->stats.h2d_bytes += m * R;
        if (host) p->stats.d2h_bytes += part.count * R;
    }
    for (size_t b = 1; b < nb; ++b) {
        const int wi = blocks[b]->worker;
        cudaError_t q = p->workers[wi].dead ? cudaErrorUnknown : cudaSetDevice(p->workers[wi].device);
        if (q == cudaSuccess) q = block ? cudaEventSynchronize(st.block_done[b]) : cudaEventQuery(st.block_done[b]);
        if (q == cudaErrorNotReady) { cudaGetLastError(); *ready = false; return FBR_OK; }
        if (q != cudaSuccess) {
            retire_if_dead(p, wi);
            return fail(FBR_ECUDA, "wrapping block %zu of a scan map on worker %d: %s", b, wi, cudaGetErrorString(q));
        }
    }
    *ready = true;
    return FBR_OK;
}

static void harvest(fbr_pool* p, SeqState& st) {
    if (st.finished) return;
    st.sum = 0;
    st.sum_lo = 0;
    st.sum_hi = 0;
    unsigned long long err = ~0ull;
    for (auto& part : st.parts) {
        Worker& w = p->workers[part.worker];
        const SeqCtrl& c = w.h_ctrl[part.ctrl_slot];
        st.sum_lo += (uint64_t)c.sum;       // < 2^32 per task: cannot wrap below 2^32 tasks
        st.sum_hi += c.sum_hi;
        err = std::min(err, c.err);
        for (auto& t : part.t_dispatch) {
            float ms = 0;
            if (cudaEventElapsedTime(&ms, t.a, t.b) == cudaSuccess) p->stats.dispatch_ms += ms;
        }
        for (auto& t : part.t_gather) {
            float ms = 0;
            if (cudaEventElapsedTime(&ms, t.a, t.b) == cudaSuccess) p->stats.gather_ms += ms;
        }
    }
    {
        const __int128 total = (__int128)st.sum_hi * ((__int128)1 << 32) + (__int128)st.sum_lo;
        st.sum = (int64_t)(uint64_t)total;
        st.sum_overflow = total != (__int128)st.sum;
    }
    if (err != ~0ull) {
        st.err_code = (uint32_t)(err & 0xff);
        st.err_task = (uint64_t)(err >> 8);
    }
    st.finished = true;
    p->stats.tasks_completed += st.n_tasks;
    p->stats.units_redispatched += st.redispatched_units;
}

// the map cannot complete: a worker died under it and it was not (or could not be) re-dispatched
static int dead_map_error(fbr_pool* p, const SeqState& st) {
    return fail(FBR_ECUDA, "worker %d (CUDA device %d) died under map %llu: %s; %s", st.dead_worker, p->workers[st.dead_worker].device,
                (unsigned long long)st.seq, cudaGetErrorString((cudaError_t)st.dead_error),
                (st.flags & FBR_RESILIENT) ? "no surviving worker could take its blocks over"
                                           : "the pool was created without error_handling, so its blocks are not re-dispatched");
}

// The completion step, once every part of the map is done: harvests the map and, unless a task failed (fbr_result_wait
// raises its error), gives a fold map its result record, tree() over the block totals that follow it in out, or wraps a
// scan map's blocks after the first (scan_finish).  Both run here rather than behind cross-device events, so no worker's
// stream waits on another device, and a dead worker fails the map before any other device depends on it.  *ready tells
// whether the map's results are final: without `block`, a scan map's queued wraps may still be running.  The caller holds
// the pool lock.
static int complete_map(fbr_pool* p, SeqState& st, bool block, bool* ready) {
    harvest(p, st);
    *ready = true;
    if (st.completed || st.err_code) return FBR_OK;
    const BodyEntry& body = *body_of(st.func_id);
    int rc = FBR_OK;
    if (st.flags & FBR_FOLD) rc = fold_host_records(p, body, (const uint8_t*)st.out + body.result_bytes, st.parts.size(), st.out);
    else if (st.flags & FBR_SCAN) rc = scan_finish(p, st, block, ready);
    else if ((st.flags & FBR_FOLD_KEYS) && st.parts.size() > 1) rc = keyed_finish(p, st);
    else if (st.flags & FBR_FOLD_SPARSE_KEYS) rc = sparse_keyed_finish(p, st, block, ready);
    if (rc != FBR_OK) return st.dead_worker >= 0 ? dead_map_error(p, st) : rc;
    st.completed = *ready;
    return FBR_OK;
}

static int result_wait_locked_out(fbr_pool_t* p, uint64_t seq, int timeout_ms, fbr_result_t* res);

// A waiter blocks on CUDA events OUTSIDE the pool lock; a concurrent fbr_result_release must not destroy them under it.
// Waiters are counted per seq; a release that arrives meanwhile is deferred to the last waiter leaving.
int fbr_result_wait(fbr_pool_t* p, uint64_t seq, int timeout_ms, fbr_result_t* res) {
    if (!p || !res) return fail(FBR_EINVAL, "NULL argument");
    {
        std::lock_guard<std::mutex> g(p->mu);
        auto it = p->seqs.find(seq);
        if (it == p->seqs.end()) return fail(FBR_ENOENT, "unknown seq %llu", (unsigned long long)seq);
        it->second->waiters++;
    }
    const int rc = result_wait_locked_out(p, seq, timeout_ms, res);
    const std::string msg = rc != FBR_OK ? g_err : std::string();
    {
        std::lock_guard<std::mutex> g(p->mu);
        auto it = p->seqs.find(seq);
        if (it != p->seqs.end() && --it->second->waiters == 0 && it->second->release_pending) {
            harvest(p, *it->second);
            free_seq(p, *it->second);
            p->seqs.erase(it);
        }
    }
    if (rc != FBR_OK) g_err = msg;
    return rc;
}

static int result_wait_locked_out(fbr_pool_t* p, uint64_t seq, int timeout_ms, fbr_result_t* res) {
    const auto deadline = std::chrono::steady_clock::now() + std::chrono::milliseconds(timeout_ms < 0 ? 0 : timeout_ms);
    for (;;) {
        struct Ev { int worker, device; cudaEvent_t ev; };
        std::vector<Ev> evs;
        {
            std::lock_guard<std::mutex> g(p->mu);
            auto it = p->seqs.find(seq);
            if (it == p->seqs.end()) return fail(FBR_ENOENT, "unknown seq %llu", (unsigned long long)seq);
            SeqState& st = *it->second;
            if (st.dead_worker >= 0) return dead_map_error(p, st);
            for (auto& part : st.parts) evs.push_back({part.worker, p->workers[part.worker].device, part.done});
            // FBR_SCAN: the wraps of blocks after the first; FBR_FOLD_SPARSE_KEYS: every block's run fold -- once queued
            // (block_done[b] belongs to the b-th block by start)
            const std::vector<SeqPart*> blocks = parts_in_order(st);
            for (size_t b = 0; b < st.block_done.size() && b < blocks.size(); ++b)
                if (st.block_done[b]) evs.push_back({blocks[b]->worker, p->workers[blocks[b]->worker].device, st.block_done[b]});
        }
        // block outside the pool lock so other threads can keep submitting
        bool again = false;
        for (auto& e : evs) {
            cudaError_t q = cudaSetDevice(e.device);
            if (q == cudaSuccess) {
                if (timeout_ms < 0) {
                    q = cudaEventSynchronize(e.ev);
                } else {
                    for (;;) {
                        q = cudaEventQuery(e.ev);
                        if (q != cudaErrorNotReady) break;
                        if (std::chrono::steady_clock::now() >= deadline) return fail(FBR_ETIMEOUT, "timeout waiting for seq %llu", (unsigned long long)seq);
                        std::this_thread::sleep_for(std::chrono::microseconds(50));
                    }
                }
            }
            if (q != cudaSuccess) {
                // watchdog: is it the worker (sticky context error) or just this call?
                std::lock_guard<std::mutex> g(p->mu);
                if (!retire_if_dead(p, e.worker))
                    return fail(FBR_ECUDA, "waiting for seq %llu on worker %d: %s", (unsigned long long)seq, e.worker, cudaGetErrorString(q));
                again = true;       // the map's parts changed (re-dispatched) or it is marked dead
                break;
            }
        }
        if (again) continue;
        std::lock_guard<std::mutex> g(p->mu);
        auto it = p->seqs.find(seq);
        if (it == p->seqs.end()) return fail(FBR_ENOENT, "seq released while waiting");
        SeqState& st = *it->second;
        if (st.dead_worker >= 0) return dead_map_error(p, st);
        // resilient maps: the round is over; re-dispatch what was lost, or copy the window back
        int more = 0;
        for (size_t i = 0; i < st.parts.size(); ++i) {
            SeqPart& part = st.parts[i];
            Worker& w = p->workers[part.worker];
            cudaError_t q = w.dead ? cudaErrorUnknown : cudaSetDevice(w.device);
            if (q == cudaSuccess) q = cudaEventQuery(part.done);
            if (q == cudaErrorNotReady) { cudaGetLastError(); more = 1; continue; }  // re-recorded by another waiter
            int rc = q == cudaSuccess ? resilient_advance(p, st, part) : FBR_ECUDA;
            if (rc < 0) {
                const std::string msg = g_err;
                if (!retire_if_dead(p, part.worker)) { g_err = msg; return rc; }
                more = 1;                                 // st.parts is a different vector now
                break;
            }
            more |= rc;
        }
        if (more) continue;
        bool ready = false;
        const int rc = complete_map(p, st, false, &ready);
        if (rc != FBR_OK) return rc;
        if (!ready) continue;                     // wait for the queued wraps outside the lock
        memset(res, 0, sizeof *res);
        res->seq = seq;
        res->n_tasks = st.n_tasks;
        res->result_bytes = st.result_bytes;
        res->result_kind = st.result_kind;
        res->data = st.out;
        res->sum = st.sum;
        res->sum_lo = st.sum_lo;
        res->sum_hi = st.sum_hi;
        res->sum_overflow = st.sum_overflow ? 1u : 0u;
        res->err_code = st.err_code;
        res->err_task = st.err_task;
        res->n_waves = st.n_waves;
        if (st.err_code) return fail(FBR_ETASK, "task %llu failed with code %u in body %s", (unsigned long long)st.err_task, st.err_code, body_of(st.func_id)->name.c_str());
        return FBR_OK;
    }
}

int fbr_result_poll(fbr_pool_t* p, uint64_t seq, uint64_t* n_done) {
    if (!p || !n_done) return fail(FBR_EINVAL, "NULL argument");
    std::lock_guard<std::mutex> g(p->mu);
    auto it = p->seqs.find(seq);
    if (it == p->seqs.end()) return fail(FBR_ENOENT, "unknown seq %llu", (unsigned long long)seq);
    SeqState& st = *it->second;
    if (st.dead_worker >= 0) return dead_map_error(p, st);
    if (st.finished && st.parts.empty()) {   // an emit map whose count pass failed: nothing more will come, wait reports why
        *n_done = st.n_tasks;
        return FBR_OK;
    }
    // ordered progress: tasks [0, n_done) are final.  Blocks are contiguous per worker, so count
    // complete waves worker by worker and stop at the first incomplete one.
    uint64_t done = 0;
    for (size_t pi = 0; pi < st.parts.size(); ++pi) {
        SeqPart& part = st.parts[pi];
        Worker& w = p->workers[part.worker];
        cudaError_t q = w.dead ? cudaErrorUnknown : cudaSetDevice(w.device);
        if (q == cudaSuccess) q = cudaEventQuery(part.done);
        if (q != cudaSuccess && q != cudaErrorNotReady) {
            // watchdog (same as fbr_result_wait): a dead worker's blocks move to the survivors
            if (!retire_if_dead(p, part.worker)) return fail(FBR_ECUDA, "polling seq %llu on worker %d: %s", (unsigned long long)seq, part.worker, cudaGetErrorString(q));
            if (st.dead_worker >= 0) return dead_map_error(p, st);
            break;                                        // progress so far stands; the next poll sees the new parts
        }
        cudaGetLastError();
        const bool part_finished = q == cudaSuccess;
        if (part.cx.plan.resilient) {
            // results become visible only once no unit is lost any more; polling drives the rounds
            if (part_finished) {
                if (part.finalized) { done += part.count; continue; }
                int rc = resilient_advance(p, st, part);
                if (rc < 0) {
                    const std::string msg = g_err;
                    if (!retire_if_dead(p, part.worker)) { g_err = msg; return rc; }
                    if (st.dead_worker >= 0) return dead_map_error(p, st);
                }
            }
            break;
        }
        uint64_t part_done = 0;
        if (part.cx.plan.final_at_block_end()) {
            // the window reaches the host in one copy at the end, or (a scan block, results on the device too) its prefix
            // folds are written in place behind its last wave: nothing is final before that
            if (part_finished) { done += part.count; continue; }
            break;
        }
        for (size_t i = 0; i < part.wave_done.size(); ++i) {
            if (cudaEventQuery(part.wave_done[i]) != cudaSuccess) break;
            part_done = part.wave_cum[i];
        }
        cudaGetLastError();
        done += part_done;
        if (part_done < part.count) break;
    }
    if (st.flags & (FBR_FOLD | FBR_SCAN | FBR_FOLD_KEYS | FBR_FOLD_SPARSE_KEYS)) {   // final once the map is complete: 0 tasks done until then
        bool ready = false;
        if (done >= st.n_tasks) {                 // every part is done: fold and scan blocks count only then (above)
            const int rc = complete_map(p, st, false, &ready);
            if (rc != FBR_OK) return rc;
        }
        if (!ready) done = 0;
    }
    *n_done = done;
    return FBR_OK;
}

int fbr_result_values(fbr_pool_t* p, uint64_t seq, void** values, uint64_t* n_values) {
    if (!p || !values || !n_values) return fail(FBR_EINVAL, "NULL argument");
    std::lock_guard<std::mutex> g(p->mu);
    auto it = p->seqs.find(seq);
    if (it == p->seqs.end()) return fail(FBR_ENOENT, "unknown seq %llu", (unsigned long long)seq);
    const SeqState& st = *it->second;
    if (!(body_of(st.func_id)->flags & FBR_BODY_EMIT)) return fail(FBR_EINVAL, "seq %llu is not a map of an emit body", (unsigned long long)seq);
    *values = st.values;
    *n_values = st.n_values;
    return FBR_OK;
}

int fbr_result_fetch_values(fbr_pool_t* p, uint64_t seq, uint64_t first, uint64_t count, void* host_dst) {
    if (!p || (!host_dst && count)) return fail(FBR_EINVAL, "NULL argument");
    std::lock_guard<std::mutex> g(p->mu);
    auto it = p->seqs.find(seq);
    if (it == p->seqs.end()) return fail(FBR_ENOENT, "unknown seq %llu", (unsigned long long)seq);
    SeqState& st = *it->second;
    if (!(body_of(st.func_id)->flags & FBR_BODY_EMIT) || !(st.flags & FBR_RESULTS_ON_DEVICE))
        return fail(FBR_EINVAL, "seq %llu is not an emit map that keeps its results on the device", (unsigned long long)seq);
    if (first + count > st.n_values || first + count < first) return fail(FBR_EINVAL, "range out of bounds");
    const uint64_t ob = body_of(st.func_id)->out_bytes;
    for (auto& part : st.parts) {
        CK(cudaSetDevice(p->workers[part.worker].device));
        CK(cudaEventSynchronize(part.done));
    }
    for (auto& part : st.parts) {
        const EmitBlock& e = part.emit;
        const uint64_t lo = std::max(first, e.base), hi = std::min(first + count, e.base + e.total);
        if (lo >= hi) continue;
        Worker& w = p->workers[part.worker];
        CK(cudaSetDevice(w.device));
        CK(cudaMemcpyAsync((uint8_t*)host_dst + (lo - first) * ob, (const uint8_t*)e.d_values + (lo - e.base) * ob, (hi - lo) * ob, cudaMemcpyDeviceToHost, w.s_out));
        p->stats.d2h_bytes += (hi - lo) * ob;
    }
    for (auto& part : st.parts) {
        CK(cudaSetDevice(p->workers[part.worker].device));
        CK(cudaStreamSynchronize(p->workers[part.worker].s_out));
    }
    return FBR_OK;
}

int fbr_result_data(fbr_pool_t* p, uint64_t seq, void** data) {
    if (!p || !data) return fail(FBR_EINVAL, "NULL argument");
    std::lock_guard<std::mutex> g(p->mu);
    auto it = p->seqs.find(seq);
    if (it == p->seqs.end()) return fail(FBR_ENOENT, "unknown seq %llu", (unsigned long long)seq);
    *data = it->second->out;
    return FBR_OK;
}

int fbr_result_fetch(fbr_pool_t* p, uint64_t seq, uint64_t first, uint64_t count, void* host_dst) {
    if (!p || (!host_dst && count)) return fail(FBR_EINVAL, "NULL argument");
    std::lock_guard<std::mutex> g(p->mu);
    auto it = p->seqs.find(seq);
    if (it == p->seqs.end()) return fail(FBR_ENOENT, "unknown seq %llu", (unsigned long long)seq);
    SeqState& st = *it->second;
    if (st.flags & FBR_FOLD) return fail(FBR_EINVAL, "seq %llu is a fold map: its one result record is fbr_result_t.data", (unsigned long long)seq);
    if (st.flags & FBR_FOLD_KEYS)
        return fail(FBR_EINVAL, "seq %llu is a keyed fold map: its records and counts are fbr_result_t.data", (unsigned long long)seq);
    if (st.flags & FBR_FOLD_SPARSE_KEYS)
        return fail(FBR_EINVAL, "seq %llu is a sparse keyed fold map: its records are fbr_result_t.data, its keys and counts "
                    "fbr_result_groups", (unsigned long long)seq);
    if (!(st.flags & FBR_RESULTS_ON_DEVICE)) return fail(FBR_EINVAL, "seq %llu does not keep its results on the device", (unsigned long long)seq);
    if (first + count > st.n_tasks) return fail(FBR_EINVAL, "range out of bounds");
    const uint64_t R = st.result_bytes;
    if ((st.flags & FBR_SCAN) && !st.completed) {   // blocks after the first hold their own prefixes until the map completes
        if (st.dead_worker >= 0) return dead_map_error(p, st);
        for (auto& part : st.parts) {
            CK(cudaSetDevice(p->workers[part.worker].device));
            CK(cudaEventSynchronize(part.done));
        }
        bool ready = false;
        const int rc = complete_map(p, st, true, &ready);   // a fetch reads the wrapped windows
        if (rc != FBR_OK) return rc;
    }
    for (auto& part : st.parts) {
        const uint64_t lo = std::max(first, part.first), hi = std::min(first + count, part.first + part.count);
        if (lo >= hi) continue;
        Worker& w = p->workers[part.worker];
        CK(cudaSetDevice(w.device));
        CK(cudaEventSynchronize(part.done));
        CK(cudaMemcpyAsync((uint8_t*)host_dst + (lo - first) * R, part.cx.window_base + (lo - part.first) * R, (hi - lo) * R,
                           cudaMemcpyDeviceToHost, w.s_out));
        p->stats.d2h_bytes += (hi - lo) * R;
    }
    for (auto& part : st.parts) {
        CK(cudaSetDevice(p->workers[part.worker].device));
        CK(cudaStreamSynchronize(p->workers[part.worker].s_out));
    }
    return FBR_OK;
}

int fbr_result_groups(fbr_pool_t* p, uint64_t seq, uint64_t* n_groups, const uint32_t** keys, const uint64_t** counts) {
    if (!p || !n_groups || !keys || !counts) return fail(FBR_EINVAL, "NULL argument");
    std::lock_guard<std::mutex> g(p->mu);
    auto it = p->seqs.find(seq);
    if (it == p->seqs.end()) return fail(FBR_ENOENT, "unknown seq %llu", (unsigned long long)seq);
    const SeqState& st = *it->second;
    if (!(st.flags & FBR_FOLD_SPARSE_KEYS))
        return fail(FBR_EINVAL, "seq %llu is not a sparse keyed fold map (FBR_FOLD_SPARSE_KEYS)", (unsigned long long)seq);
    if (!st.completed || st.err_code)
        return fail(FBR_EINVAL, "seq %llu has no groups before fbr_result_wait has succeeded", (unsigned long long)seq);
    *n_groups = st.group_keys.size();
    *keys = st.group_keys.data();
    *counts = st.group_counts.data();
    return FBR_OK;
}

int fbr_result_release(fbr_pool_t* p, uint64_t seq) {
    if (!p) return fail(FBR_EINVAL, "NULL pool");
    std::lock_guard<std::mutex> g(p->mu);
    auto it = p->seqs.find(seq);
    if (it == p->seqs.end()) return fail(FBR_ENOENT, "unknown seq %llu", (unsigned long long)seq);
    if (it->second->waiters > 0) {        // another thread is blocked on this map's events: it frees the seq when it leaves
        it->second->release_pending = true;
        return FBR_OK;
    }
    harvest(p, *it->second);  // keeps the timing statistics of maps released without a wait
    free_seq(p, *it->second);
    p->seqs.erase(it);
    return FBR_OK;
}

int fbr_fold_values(fbr_pool_t* p, int func_id, const void* values, uint64_t n, void* out) {
    if (!p || !out || (n && !values)) return fail(FBR_EINVAL, "NULL argument");
    const BodyEntry* bp = body_of(func_id);
    if (!bp) return fail(FBR_EINVAL, "bad func_id %d", func_id);
    if (!(bp->flags & FBR_BODY_FOLD)) return fail(FBR_EINVAL, "body %s has no combine(): it cannot fold", bp->name.c_str());
    std::lock_guard<std::mutex> g(p->mu);
    return fold_host_records(p, *bp, values, n, out);
}

int fbr_fold_segments(fbr_pool_t* p, int func_id, const void* values, const uint64_t* offsets, uint32_t n_segments, void* out) {
    if (!p || !offsets || (n_segments && !out)) return fail(FBR_EINVAL, "NULL argument");
    const BodyEntry* bp = body_of(func_id);
    if (!bp) return fail(FBR_EINVAL, "bad func_id %d", func_id);
    if (!(bp->flags & FBR_BODY_KEYED)) return fail(FBR_EINVAL, "body %s has no key(): it exports no fold_segments entry", bp->name.c_str());
    if (offsets[0] != 0) return fail(FBR_EINVAL, "offsets[0] must be 0");
    for (uint32_t k = 0; k < n_segments; ++k)
        if (offsets[k + 1] < offsets[k]) return fail(FBR_EINVAL, "offsets decrease at segment %u", k);
    if (offsets[n_segments] && !values) return fail(FBR_EINVAL, "NULL argument");
    std::lock_guard<std::mutex> g(p->mu);
    return fold_segments_host(p, *bp, values, offsets, n_segments, out);
}

int fbr_scan_values(fbr_pool_t* p, int func_id, const void* pieces, uint32_t n_pieces, void* values, uint64_t n) {
    if (!p || (n_pieces && !pieces) || (n && !values)) return fail(FBR_EINVAL, "NULL argument");
    const BodyEntry* bp = body_of(func_id);
    if (!bp) return fail(FBR_EINVAL, "bad func_id %d", func_id);
    if (!(bp->flags & FBR_BODY_SCAN)) return fail(FBR_EINVAL, "body %s exports no scan entry (FBR_BODY_SCAN)", bp->name.c_str());
    std::lock_guard<std::mutex> g(p->mu);
    const int wi = first_live_worker(p);
    if (wi < 0) return fail(FBR_ECUDA, "every worker of this pool has died");
    const uint64_t R = bp->result_bytes;
    if (n == 0 || n_pieces == 0) return FBR_OK;
    Worker& w = p->workers[wi];
    uint8_t* d = nullptr;   // the n records, wrapped in place
    cudaError_t e = cudaSetDevice(w.device);
    if (e == cudaSuccess) e = cudaMallocAsync((void**)&d, n * R, w.s_fold);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d, values, n * R, cudaMemcpyHostToDevice, w.s_fold);
    if (e == cudaSuccess) e = queue_wrap(w, *bp, pieces, n_pieces, d, n, values, nullptr);
    if (d) cudaFreeAsync(d, w.s_fold);
    if (e == cudaSuccess) e = cudaStreamSynchronize(w.s_fold);
    if (e != cudaSuccess) {
        retire_if_dead(p, wi);
        return fail(FBR_ECUDA, "wrapping %llu records of body %s on worker %d: %s", (unsigned long long)n, bp->name.c_str(), wi,
                    cudaGetErrorString(e));
    }
    p->stats.h2d_bytes += (n_pieces + n) * R;
    p->stats.d2h_bytes += n * R;
    return FBR_OK;
}

int fbr_host_alloc(fbr_pool_t* p, uint64_t bytes, void** ptr) {
    if (!p || !ptr) return fail(FBR_EINVAL, "NULL argument");
    std::lock_guard<std::mutex> g(p->mu);
    return pinned_acquire(p, bytes, ptr);
}

int fbr_host_free(fbr_pool_t* p, void* ptr) {
    if (!p) return fail(FBR_EINVAL, "NULL pool");
    std::lock_guard<std::mutex> g(p->mu);
    pinned_release(p, ptr);
    return FBR_OK;
}

int fbr_device_alloc(fbr_pool_t* p, int worker, uint64_t bytes, void** dptr) {
    if (!p || !dptr || worker < 0 || worker >= (int)p->workers.size()) return fail(FBR_EINVAL, "bad arguments");
    CK(cudaSetDevice(p->workers[worker].device));
    CK(cudaMalloc(dptr, bytes));
    return FBR_OK;
}

int fbr_device_free(fbr_pool_t* p, int worker, void* dptr) {
    if (!p || worker < 0 || worker >= (int)p->workers.size()) return fail(FBR_EINVAL, "bad arguments");
    CK(cudaSetDevice(p->workers[worker].device));
    CK(cudaFree(dptr));
    return FBR_OK;
}

int fbr_memcpy_h2d(fbr_pool_t* p, int worker, void* dptr, const void* src, uint64_t bytes) {
    if (!p || worker < 0 || worker >= (int)p->workers.size()) return fail(FBR_EINVAL, "bad arguments");
    Worker& w = p->workers[worker];
    CK(cudaSetDevice(w.device));
    CK(cudaMemcpyAsync(dptr, src, bytes, cudaMemcpyHostToDevice, w.s_in));
    CK(cudaStreamSynchronize(w.s_in));
    return FBR_OK;
}

int fbr_memcpy_d2h(fbr_pool_t* p, int worker, void* dst, const void* dptr, uint64_t bytes) {
    if (!p || worker < 0 || worker >= (int)p->workers.size()) return fail(FBR_EINVAL, "bad arguments");
    Worker& w = p->workers[worker];
    CK(cudaSetDevice(w.device));
    CK(cudaStreamSynchronize(w.s_comp));
    CK(cudaMemcpyAsync(dst, dptr, bytes, cudaMemcpyDeviceToHost, w.s_out));
    CK(cudaStreamSynchronize(w.s_out));
    return FBR_OK;
}

int fbr_payload_fill_device(fbr_pool_t* p, int worker, void* dptr, uint64_t t0, uint64_t n) {
    if (!p || !dptr || worker < 0 || worker >= (int)p->workers.size()) return fail(FBR_EINVAL, "bad arguments");
    std::lock_guard<std::mutex> g(p->mu);
    Worker& w = p->workers[worker];
    CK(cudaSetDevice(w.device));
    const uint64_t n_vec = n * (kPayloadBytes / 16);
    const int grid = (int)std::max<uint64_t>(1, std::min<uint64_t>((n_vec + kThreads - 1) / kThreads, (uint64_t)w.sm_count * w.occ_fill));
    payload_fill_kernel<<<grid, kThreads, 0, w.s_comp>>>((uint4*)dptr, t0, n_vec);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(w.s_comp));
    p->stats.fill_launches++;
    return FBR_OK;
}

int fbr_pool_stats(fbr_pool_t* p, fbr_stats_t* s) {
    if (!p || !s) return fail(FBR_EINVAL, "NULL argument");
    std::lock_guard<std::mutex> g(p->mu);
    *s = p->stats;
    return FBR_OK;
}

int fbr_pool_stats_reset(fbr_pool_t* p) {
    if (!p) return fail(FBR_EINVAL, "NULL pool");
    std::lock_guard<std::mutex> g(p->mu);
    memset(&p->stats, 0, sizeof p->stats);
    return FBR_OK;
}

}  // extern "C"
