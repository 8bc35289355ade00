/* fiber_b200.h -- C ABI of the H100-native Pool.map engine (libfiber_b200.so).
 *
 * This is the drop-in boundary for the ONE hot path of uber/fiber this repository replaces:
 * Pool.map / starmap / apply_async task scatter + result gather.  The reference is pure Python
 * and has no FFI of its own; each entry point below therefore cites the reference *interface* it
 * stands in for (paths relative to the reference checkout, fiber @ ad6faf02).  A reference
 * maintainer binds them with ctypes exactly as fiber_b200/_abi.py does (see INTEGRATION.md).
 *
 * Conventions: plain pointers and sizes only (no torch / C++ types); every function returns
 * FBR_OK (0) or a negative fbr_status; fbr_last_error() gives the thread-local message.  Blocking
 * calls (fbr_result_wait, fbr_pool_join) do not touch Python and are called with the GIL released.
 * The library never computes a task on the CPU: without a usable CUDA device fbr_pool_create
 * fails with FBR_ENODEV.
 */
#ifndef FIBER_B200_H_
#define FIBER_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FBR_ABI_VERSION 2

typedef enum fbr_status {
    FBR_OK = 0,
    FBR_EINVAL = -1,    /* bad argument */
    FBR_ECUDA = -2,     /* CUDA runtime error (message has the cudaError string) */
    FBR_ENOMEM = -3,
    FBR_ESTATE = -4,    /* pool not in RUN state: the ABI face of ValueError("Pool is not running"),
                           fiber/pool.py:1107-1108,1166-1167,1284-1285 */
    FBR_ETIMEOUT = -5,
    FBR_ETASK = -6,     /* a device body reported a task error (see fbr_result_t.err_*) */
    FBR_ENODEV = -7,    /* no CUDA device: there is no CPU fallback */
    FBR_ENOENT = -8     /* unknown body name / seq */
} fbr_status;

typedef struct fbr_pool fbr_pool_t;

/* ---- library ------------------------------------------------------------------------------ */
int fbr_abi_version(void);
const char* fbr_last_error(void);
/* fiber/context.py:61-62 cpu_count(): the engine's unit of parallel hardware is the GPU. */
int fbr_device_count(int* n);

/* ---- device-body registry -------------------------------------------------------------------
 * The reference ships `func` to workers by pickle reference (fiber/pool.py:961) and calls it at
 * fiber/pool.py:806,809,820.  A Python callable cannot run on a GPU, so callables are bound to a
 * compiled-in device body by name; unbound callables are rejected by the host layer. */
typedef enum fbr_result_kind {
    FBR_RES_BYTES = 0,   /* opaque fixed-size record */
    FBR_RES_BOOL = 1,    /* uint8 0/1  (Python bool) */
    FBR_RES_I64 = 2,     /* int64      (Python int) */
    FBR_RES_U32 = 3,     /* uint32     (Python int) */
    FBR_RES_F64X2 = 4,   /* two float64 (Python tuple of floats) */
    FBR_RES_NONE = 5,    /* body returns None; one pad byte per task */
    FBR_RES_BITS8 = 6,   /* one byte = the bool results of 8 consecutive items, bit k (LSB first) = item
                            8*task + k.  A map over N items is submitted as ceil(N/8) tasks: range() indices
                            (arg_stride 0) or 8 argument items per task record (arg_stride = 8 * item size,
                            fbr_map_desc_t.n_items = N so that items past N are never read).  For range()
                            indices the bits past N in the last byte are computed like any other index and
                            are masked by the caller (fiber_b200/pool.py does) */
    FBR_RES_OFFSETS = 7  /* emit bodies (FBR_BODY_EMIT): uint64 end offset of each task's values; task j's values are
                            [end[j-1], end[j]) of the map's values (fbr_result_values), end[-1] = 0 */
} fbr_result_kind;

#define FBR_BODY_INDEX_ARG 0x1u   /* body can take the task index itself as its int64 argument */
#define FBR_BODY_NEEDS_SHARED 0x2u /* body reads a shared (broadcast) argument block */
#define FBR_BODY_SUMMABLE 0x4u    /* the dispatch kernel can fold sum(results) (bool/int64/u32; popcount for bits) */
#define FBR_BODY_INDEX_ONLY 0x8u  /* body takes range() arguments only (arg_stride must be 0) */
#define FBR_BODY_RECORD 0x10u     /* argument and result records are staged through shared memory by dispatch_record_kernel
                                     (FBR_EXPORT_RECORD_BODY): arg_bytes and result_bytes are any multiples of 4 up to
                                     4096 -- up to 32768 for a group body (group_threads > 1 in its module descriptor)
                                     whose 16 B-aligned group of tasks fits one 32 KB stage --, arg_stride any multiple
                                     of 4 >= arg_bytes; result kind FBR_RES_BYTES, not SUMMABLE, no bit-packed twin;
                                     NEEDS_SHARED only together with BROADCAST */
#define FBR_BODY_BROADCAST 0x20u  /* record body whose run() receives the map's broadcast block as an array of its
                                     Shared element type (fbr_body_shared_info); always set with NEEDS_SHARED */
#define FBR_BODY_ITEMS 0x40u      /* record body whose task also takes a variable-length array of its Item element type
                                     (fbr_body_items_info); its maps go through fbr_map_submit_items.  arg_bytes may be 0
                                     (no head record, Arg = fbr::NoArg); never with FBR_BODY_INDEX_ARG */
#define FBR_BODY_EMIT 0x80u       /* record body whose task returns a variable-length array of its Out element type
                                     (fbr_body_emit_info) instead of a fixed record: result_bytes 8, result kind
                                     FBR_RES_OFFSETS.  Each map runs a count pass, a scan of the counts and an emit pass;
                                     never SUMMABLE, no bit-packed twin */
#define FBR_BODY_FOLD 0x100u      /* record body with identity() and combine(): its maps may fold their results on the device
                                     (FBR_FOLD, fbr_fold_values; fbr_body_fold_info).  Set exactly when the module
                                     descriptor has `fold` and `identity`, with identity_bytes = result_bytes; never
                                     with EMIT or SUMMABLE */
#define FBR_BODY_SCAN 0x200u      /* FBR_BODY_FOLD body whose descriptor exports `scan`: its maps may return every prefix of
                                     the fold (FBR_SCAN, fbr_scan_values).  Set exactly when `scan` is exported, and only
                                     with FBR_BODY_FOLD; `scan` is read only from descriptors that set it, so a fold
                                     descriptor that ends at identity_bytes stays a valid fold body */
#define FBR_BODY_KEYED 0x400u     /* FBR_BODY_FOLD body with key(): its maps may fold per key (FBR_FOLD_KEYS, fbr_fold_segments).
                                     Set exactly when the descriptor exports `keys` and `fold_segments`, and only with
                                     FBR_BODY_FOLD; both are read only from descriptors that set it */

typedef struct fbr_body_info {
    int32_t func_id;
    uint32_t arg_bytes;      /* fixed-layout per-task argument record */
    uint32_t result_bytes;   /* fixed-layout per-task result record */
    uint32_t result_kind;    /* fbr_result_kind */
    uint32_t flags;          /* FBR_BODY_* */
    uint32_t unit_tasks;     /* preferred claim-unit size (tasks per ring slot) */
    char name[40];
} fbr_body_info_t;

int fbr_body_count(int* n);
int fbr_body_info(int func_id, fbr_body_info_t* info);
int fbr_body_lookup(const char* name, int* func_id);

/* Out-of-tree device bodies.  The reference pickles ANY callable into the task tuple
 * (fiber/pool.py:961) and the worker calls it (fiber/pool.py:806,809,820); here the callable's device
 * code may be compiled separately from this library: a shared object built with nvcc for sm_90a from a
 * source that includes include/fiber_b200_body.cuh, defines a ThreadBody struct and exports it with
 * FBR_EXPORT_THREAD_BODY(Body, name, entry) (or a RecordBody over fixed-size structs with
 * FBR_EXPORT_RECORD_BODY(Body, name, entry, flags)).  fbr_register_body dlopen()s `module_path`, calls `entry`
 * to obtain the module descriptor below, checks its ABI stamp and appends the body to the table
 * (func_id >= the compiled-in count; the same name may be registered once).  The module's launch routine
 * receives the same wave parameters as the compiled-in kernels, so registered bodies run in the same
 * persistent-CTA dispatch kernels (direct placement, ring + gather_ordered, resilient re-dispatch). */
#define FBR_BODY_MODULE_ABI 4
typedef struct fbr_body_module {
    uint32_t abi;               /* FBR_BODY_MODULE_ABI */
    uint32_t wave_params_bytes; /* sizeof(fbr::WaveParams) the module was compiled against */
    const char* name;
    uint32_t arg_bytes, result_bytes, result_kind, flags, unit_tasks;
    void (*launch)(const void* wave_params, int grid, void* cuda_stream);
    int (*occupancy)(int index_mode);   /* resident CTAs per SM on the current device */
    /* FBR_BODY_BROADCAST record bodies: sizeof(Shared) (a multiple of 4 up to 4096) and the body's shared-memory
       budget for the block (a multiple of 16; 0 = always read it from global memory).  0, 0 for every other body */
    uint32_t shared_elem_bytes, shared_stage_bytes;
    /* record bodies only: threads that run each task together (the body's kGroup: 2, 4, 8, 16 or 32), which lets its
       records reach 32768 bytes (kAlign * max(arg_bytes, result_bytes) <= 32768, kAlign = 1, 2 or 4 tasks: both sizes
       multiples of 16, of 8, or neither).  0 or 1: one thread per task */
    uint32_t group_threads;
    /* FBR_BODY_ITEMS record bodies: sizeof(Item) (1, 2 or a multiple of 4 up to 4096).  0 (or left out of a hand-written
       descriptor) for every other body */
    uint32_t item_bytes;
    /* FBR_BODY_EMIT record bodies: sizeof(Out) (1, 2 or a multiple of 4 up to 4096).  0 (or left out of a hand-written
       descriptor) for every other body */
    uint32_t out_bytes;
    /* FBR_BODY_ITEMS record bodies: the number of item streams each task takes (the body's Items = fbr::ItemTypes<...>:
       2, 3 or 4; 0 or 1 = one stream, `using Item`), and the element sizes of streams 1 to 3 (stream 0's is item_bytes;
       each 1, 2 or a multiple of 4 up to 4096; 0 past the last stream).  0 (or left out of a hand-written descriptor) for
       every other body */
    uint32_t item_streams;
    uint32_t more_item_bytes[3];
    /* FBR_BODY_FOLD record bodies: tree() over n >= 1 device records at `values` (overwritten) into the record at `dst`
       (device-accessible), launched on `cuda_stream` (fold_tree_kernel), and the body's identity() evaluated on the host,
       identity_bytes (= result_bytes) bytes.  NULL, NULL, 0 (or left out of a hand-written descriptor) for every other
       body; the fold maps themselves go through `launch` like any map (WaveParams::fold_partials set) */
    void (*fold)(void* values, uint64_t n, void* dst, void* cuda_stream);
    const void* identity;
    uint32_t identity_bytes;
    /* FBR_BODY_SCAN bodies: the n device records at `values` (overwritten) become their prefix folds when `prefix` is
       set (record i <- tree(values[0..i]), see FBR_SCAN), then each is wrapped with the n_pieces device records at
       `pieces`, right-nested: pieces[0] (+) (pieces[1] (+) ( ... (+) (pieces[m-1] (+) record))).  Queued on `cuda_stream`
       (scan_level_kernel, scan_wrap_kernel, and stream-ordered scratch of fewer than n records); returns the launch's
       cudaError_t.  Left out of (or NULL in) a descriptor without FBR_BODY_SCAN */
    int (*scan)(void* values, uint64_t n, int prefix, const void* pieces, uint32_t n_pieces, void* cuda_stream);
    /* FBR_BODY_KEYED bodies, both queued on `cuda_stream` and returning the launch's cudaError_t.  `keys`: keys[i] = key() of
       the n device records at `values`; a key >= n_keys is stored as 0, and the lowest such task, first_task + i, goes into
       the device word *err as min(*err, (task << 8) | FBR_TASK_KEY).  `fold_segments`: the n device records at `values` are
       in key order (overwritten); dst[k] (device-accessible) <- tree() of records [offsets[k], offsets[k + 1]) for each of
       the n_segments segments, identity() for an empty one; `offsets` are n_segments + 1 non-decreasing device words.  Left
       out of (or NULL in) a descriptor without FBR_BODY_KEYED */
    int (*keys)(const void* values, uint64_t n, uint32_t n_keys, uint64_t first_task, uint32_t* keys, unsigned long long* err,
                void* cuda_stream);
    int (*fold_segments)(void* values, uint64_t n, const uint64_t* offsets, uint32_t n_segments, void* dst, void* cuda_stream);
} fbr_body_module_t;
typedef const fbr_body_module_t* (*fbr_body_entry_fn)(void);
int fbr_register_body(const char* name, const char* module_path, const char* entry, int* func_id);
/* Broadcast element size and staging budget of a FBR_BODY_BROADCAST body (0, 0 for other bodies).  A map of such a body
 * passes a block of shared_bytes > 0, a multiple of elem_bytes; blocks up to stage_bytes are staged into shared memory
 * once per CTA, larger ones are read from global memory. */
int fbr_body_shared_info(int func_id, uint32_t* elem_bytes, uint32_t* stage_bytes);
/* Item size of a FBR_BODY_ITEMS body (0 for other bodies; stream 0's for a multi-stream body).  The dispatch kernel reads
 * each task's items from global memory. */
int fbr_body_items_info(int func_id, uint32_t* item_bytes);
/* Item streams of a FBR_BODY_ITEMS body (1 to 4; 0 for other bodies) and the element size of each (item_bytes[k] for
 * stream k, 0 past the last stream). */
int fbr_body_items_streams(int func_id, uint32_t* n_streams, uint32_t item_bytes[4]);
/* Value size of a FBR_BODY_EMIT body (0 for other bodies). */
int fbr_body_emit_info(int func_id, uint32_t* out_bytes);
/* Identity record of a FBR_BODY_FOLD body: *bytes = result_bytes, and `identity` (if not NULL) gets that many bytes.
 * Other bodies: *bytes = 0. */
int fbr_body_fold_info(int func_id, void* identity, uint32_t* bytes);

/* ---- pool lifecycle -------------------------------------------------------------------------
 * fbr_pool_create   <- ZPool.__init__ (fiber/pool.py:888-943) + worker start
 *                      (_maintain_workers, fiber/pool.py:1009-1057) + local_backend.create_job
 *                      (fiber/local_backend.py:37-42): one worker == one CUDA device with its
 *                      three streams and its ring set, instead of one subprocess with two sockets.
 * fbr_pool_close    <- ZPool.close      (fiber/pool.py:1337-1353)
 * fbr_pool_terminate<- ZPool.terminate  (fiber/pool.py:1355-1388)
 * fbr_pool_join     <- ZPool.join       (fiber/pool.py:1390-1403); requires close/terminate first
 * fbr_pool_destroy  frees everything (the reference relies on process exit).
 * ring_bytes: size of each device ring arena per worker (result ring, and each half of the
 * argument / ordered-output staging rings); 0 selects the default (256 MiB). */
#define FBR_POOL_TIMING 0x1u  /* bracket every dispatch/gather launch with CUDA events (stats) */
#define FBR_POOL_OVERLAP 0x2u  /* run gather(w) on a second stream concurrently with the next dispatch
                                   (device-resident results only; ring used in halves) */
int fbr_pool_create(int n_workers, const int* device_ids, uint64_t ring_bytes, uint32_t flags,
                    fbr_pool_t** pool);
int fbr_pool_close(fbr_pool_t* pool);
int fbr_pool_terminate(fbr_pool_t* pool);
int fbr_pool_join(fbr_pool_t* pool);
int fbr_pool_destroy(fbr_pool_t* pool);
int fbr_pool_n_workers(fbr_pool_t* pool, int* n);
int fbr_pool_worker_device(fbr_pool_t* pool, int worker, int* device_id);

/* ---- map submission -------------------------------------------------------------------------
 * fbr_map_submit <- ZPool.map_async / starmap_async / apply_async (fiber/pool.py:1139-1184,
 * 1258-1305, 1089-1116) + _handle_tasks (fiber/pool.py:952-963): cut [0,n_tasks) into chunks,
 * write one fixed-layout task record per claim unit into the pinned task ring, cudaMemcpyAsync
 * them (and the argument records) to the worker's device ring, launch the persistent-CTA
 * dispatch kernel and the ordered gather.  Returns immediately with the map's `seq`
 * (Inventory.add, fiber/pool.py:659-664). */
#define FBR_MAP 0x0u            /* 5th task-tuple field False (fiber/pool.py:1181) */
#define FBR_STARMAP 0x1u        /* 5th field True, item = (args,)      (fiber/pool.py:1297-1301) */
#define FBR_APPLY 0x2u          /* 5th field True, item = (args, kwds) (fiber/pool.py:1112-1113) */
#define FBR_KIND_MASK 0x3u
#define FBR_ARGS_DEVICE 0x10u   /* args/shared are device pointers on worker 0; other workers of the pool read
                                   their block through NVLink peer loads inside the dispatch kernel */
#define FBR_OUT_DEVICE 0x20u    /* out is a device pointer on worker 0; other workers' gather kernels store
                                   their units into it through NVLink peer stores */
#define FBR_WANT_SUM 0x40u      /* fold sum(results) into fbr_result_t.sum (FBR_BODY_SUMMABLE) */
#define FBR_SHUFFLE 0x80u       /* permute task records inside each wave (arrival != index order;
                                   exercises placement-by-index, fiber/pool.py:672) */
#define FBR_FULL_WINDOW 0x100u  /* keep the whole ordered output resident on the device until the
                                   map completes (needed when units may be re-dispatched) */
#define FBR_SHARED_HANDLE 0x200u /* `shared` is a handle from fbr_shared_put, not a pointer */
#define FBR_RESULTS_ON_DEVICE 0x800u /* keep the ordered results in an engine-owned device buffer (per
                                   worker block); nothing but the 24-byte control block crosses PCIe
                                   until fbr_result_fetch asks for a range */
#define FBR_VIA_RING 0x1000u    /* always go through task records + result ring + gather_ordered, even for a
                                   contiguous block whose units could be stored at their final index by
                                   the dispatch kernel (direct placement) */
#define FBR_NO_ZERO_COPY 0x2000u /* results are wanted wave by wave (imap): stage and copy them out instead of letting the kernel
                                   store small results straight into the pinned segment */
#define FBR_RESILIENT 0x400u    /* ResilientZPool semantics (fiber/pool.py:1425-1688): a claim unit whose
                                   worker dies (FBR_TASK_FAULT) is re-dispatched until it completes */
#define FBR_FOLD 0x4000u        /* fold the map's results on the device (FBR_BODY_FOLD bodies): fbr_result_t.data points
                                   at ONE record of result_bytes, tree() over the totals of the map's non-empty blocks
                                   in block order, each block's total tree() over its tasks' results in task order:
                                       tree(x[0..c)): while c > 1: x[i] <- combine(x[2i], x[2i+1]) for every i with
                                       2i+1 < c, an odd last element is carried to x[c/2]; c <- ceil(c/2)
                                   and identity() for n_tasks = 0.  Claim units hold a power of two of tasks and start at
                                   a multiple of it in their block, so the result depends on the block cut only (the
                                   fold plan of fbr_plan_query), never on chunksize, ring_bytes, waves, FBR_SHUFFLE,
                                   FBR_VIA_RING or re-dispatched units.  Refused with out, FBR_OUT_DEVICE, FBR_WANT_SUM or
                                   FBR_NO_ZERO_COPY; FBR_RESULTS_ON_DEVICE changes nothing.  fbr_result_poll reports 0
                                   tasks done until the whole map is, fbr_result_fetch refuses the map, and a worker
                                   that dies under it fails it */
#define FBR_SCAN 0x8000u        /* every prefix of the fold (FBR_BODY_SCAN bodies): fbr_result_t.data holds n_tasks
                                   records, record i the fold of results 0 .. i under the fold plan's block cut.  Task i of
                                   the b-th non-empty block gets tree(t_0, ..., t_{b-1}, p_i), t_k block k's total and p_i
                                   tree() over block b's results from its first task to i; on one worker that is
                                   tree(x[0..i]), bit for bit the FBR_FOLD result of the first i + 1 tasks, and the last
                                   record is always the FBR_FOLD result.  Record 0 is the first result itself, never
                                   combine(identity(), x0).  Evaluated without a running carry, as
                                       y[i] = F_1 (+) (F_2 (+) ( ... (+) (F_k (+) x[i])))
                                   with F_1 .. F_k the aligned power-of-two pieces of [0, i) given by the set bits of i,
                                   largest first, each the tree() of a complete aligned subtree (across blocks the same
                                   form over the block totals, with p_i in place of x[i]).  Independent of chunksize,
                                   unit size, ring_bytes, waves, FBR_SHUFFLE, FBR_VIA_RING and re-dispatched units.
                                   Refused with FBR_FOLD, out, FBR_OUT_DEVICE, FBR_WANT_SUM or FBR_NO_ZERO_COPY; allowed
                                   with FBR_RESULTS_ON_DEVICE (fbr_result_fetch), FBR_RESILIENT and FBR_ARGS_DEVICE.
                                   Blocks after the first are wrapped once every block is done (from fbr_result_wait,
                                   fbr_result_poll or fbr_result_fetch), so fbr_result_poll reports 0 tasks done until
                                   the whole map is, and a worker that dies under it fails it */
#define FBR_FOLD_KEYS 0x10000u  /* fold per key (FBR_BODY_KEYED bodies): fbr_result_t.data holds n_keys records, then n_keys
                                   uint64 counts (tasks per key).  Record k is defined on the results whose key() is k, in
                                   task order (x_k): each block's total for k is tree() of its own x_k, and record k is
                                   tree() over those totals in block order, counting only blocks where k has a task (so one
                                   worker gives tree(x_k)); identity() for a key without tasks.  The block cut is the fold
                                   plan's (FBR_PLAN_FOLD); nothing else -- chunksize, unit size, ring_bytes, waves,
                                   FBR_SHUFFLE, FBR_VIA_RING, re-dispatched units -- changes a bit.  With n_keys = 1 it is
                                   FBR_FOLD's record.  desc.n_keys must be 1 .. 65536 with n_keys * result_bytes <= ring_bytes,
                                   and a block holds fewer than 2^32 tasks.  Refused with FBR_FOLD, FBR_SCAN, out,
                                   FBR_OUT_DEVICE, FBR_WANT_SUM or FBR_NO_ZERO_COPY; FBR_RESULTS_ON_DEVICE changes nothing.
                                   A task whose key() is >= n_keys fails the map with FBR_TASK_KEY.  Each block is a
                                   full-window map; after its last round it sorts its tasks by key on the device (a stable
                                   LSD radix sort), gathers its records into key order and folds each key's run, and only
                                   its n_keys totals and counts cross PCIe.  fbr_result_poll reports 0 tasks done until the
                                   whole map is, fbr_result_fetch refuses the map, and a worker that dies under it fails it */
#define FBR_MAX_KEYS 65536u
#define FBR_FOLD_SPARSE_KEYS 0x20000u  /* fold per distinct key (FBR_BODY_KEYED bodies), for any uint32 key() but 0xFFFFFFFF:
                                   fbr_result_t.data holds D records, one per distinct key some task produced, in ascending
                                   key order; fbr_result_groups gives D, the keys and the tasks per key.  Record k is
                                   FBR_FOLD_KEYS' record k with the keys without tasks left out: each block's total for k is
                                   tree() of its own x_k, record k tree() over the totals of the blocks where k has a task, in
                                   block order, under the fold plan's block cut (FBR_PLAN_FOLD).  One worker gives tree(x_k);
                                   with every key below K <= 65536 the records, keys and counts are FBR_FOLD_KEYS' over K keys
                                   without its empty keys, bit for bit.  Nothing else -- chunksize, unit size, ring_bytes,
                                   waves, FBR_SHUFFLE, FBR_VIA_RING, re-dispatched units -- changes a bit.  desc.n_keys must
                                   be 0, and a block holds fewer than 2^32 tasks.  Refused with FBR_FOLD, FBR_SCAN,
                                   FBR_FOLD_KEYS, out, FBR_OUT_DEVICE, FBR_WANT_SUM or FBR_NO_ZERO_COPY; FBR_RESULTS_ON_DEVICE
                                   changes nothing.  The key 0xFFFFFFFF is reserved: a task whose key() is 0xFFFFFFFF fails the
                                   map with FBR_TASK_KEY (the engine calls the body's keys entry with n_keys = 0xFFFFFFFF).
                                   Each block is a full-window map; after its last round it sorts its tasks by key on the
                                   device (four 8-bit LSD radix passes), gathers its records into key order and finds the
                                   runs of equal keys; its D, known only then, sizes the result at completion, where each
                                   block's runs are folded and, with several blocks, the blocks' sorted keys are merged on the
                                   host.  Only the D records, keys and run starts of each block cross PCIe.
                                   fbr_result_poll reports 0 tasks done until the whole map is, fbr_result_fetch refuses the
                                   map, and a worker that dies under it fails it */

typedef struct fbr_map_desc {
    int32_t func_id;
    uint32_t flags;
    uint64_t n_tasks;
    uint32_t chunksize;      /* 0 -> 32 (fiber/pool.py:1169-1170) */
    uint32_t arg_stride;     /* bytes between argument records; 0 -> implicit index arguments */
    const void* args;        /* n_tasks records of arg_stride bytes (host, ideally pinned; or device) */
    int64_t index_start;     /* implicit argument of task i = index_start + i*index_step (range()) */
    int64_t index_step;
    const void* shared;      /* broadcast argument block (e.g. parzen samples), may be NULL.  A FBR_ARGS_DEVICE block may
                                start at any address: one that is not 16 B aligned is read in place only when a broadcast
                                body stages it into shared memory, else from an aligned device copy made per map */
    uint64_t shared_bytes;
    void* out;               /* NULL: engine-owned pinned result segment; else n_tasks*result_bytes */
    uint64_t task_index_base;/* global index of task 0 (sharded maps: rank's block start) */
    uint64_t shuffle_seed;
    uint64_t n_items;        /* FBR_RES_BITS8 bodies with explicit arguments: number of argument items of the
                                whole map (the last task may cover fewer than 8); 0 = 8 * n_tasks */
    uint32_t attempt;        /* how many times this block of tasks has been dispatched before (a resilient pool that
                                re-queues a dead worker's chunk, fiber/pool.py:1635-1654, passes attempt + 1); bodies
                                see it as their `attempt` argument */
    uint32_t n_keys;         /* FBR_FOLD_KEYS: number of keys (1 .. FBR_MAX_KEYS); ignored without it */
} fbr_map_desc_t;

int fbr_map_submit(fbr_pool_t* pool, const fbr_map_desc_t* desc, uint64_t* seq);

/* Maps of FBR_BODY_ITEMS bodies: besides its head record (args / arg_stride, if the body has one; arg_stride 0 when
 * arg_bytes is 0), task j reads items [offsets[j], offsets[j+1]) of `items`.  offsets[0] may be non-zero (a slice of a
 * larger array).  Host-resident offsets are checked before anything launches; device-resident ones (FBR_ARGS_DEVICE:
 * items and offsets are device pointers on worker 0, one-worker pools only, offsets 8-byte aligned, items aligned to the
 * largest power of two that divides item_bytes, at most 16: 1, 2, 4, 8 or 16 bytes, so a body may load its items as
 * vectors that wide) are checked by the kernel, and a task whose offsets decrease or pass n_items fails with
 * FBR_TASK_BADARG.  Host-resident items and offsets stream to the device wave by wave through two staging halves of
 * ring_bytes each (a resilient map copies its whole block once); a claim unit whose offsets and items do not fit one
 * half is refused with FBR_EINVAL before anything launches.
 * fbr_map_submit refuses items bodies and fbr_map_submit_items every other body (FBR_EINVAL).
 *
 * One fbr_items_desc_t describes one item stream.  A body with K streams (fbr_body_items_streams) takes K of them, in
 * stream order, through fbr_map_submit_items_n: each has its own items, offsets, n_items and element size, all the checks
 * above apply to each, and task j reads [offsets[j], offsets[j+1]) of every stream.  FBR_ARGS_DEVICE applies to every
 * stream of the map.  Host-resident streams share the same two staging halves: in a wave's half, stream k's offsets and
 * item span follow stream k-1's, each stream starting on a 256 B boundary, and a claim unit whose K streams do not fit one
 * half together is refused.  fbr_map_submit_items is fbr_map_submit_items_n with n_streams = 1. */
typedef struct fbr_items_desc {
    const void* items;        /* item array: host, or device on worker 0 with FBR_ARGS_DEVICE */
    const uint64_t* offsets;  /* n_tasks + 1 non-decreasing item indices: task j reads items [offsets[j], offsets[j+1]) */
    uint64_t n_items;         /* items in `items`; every offset is <= n_items */
    uint32_t item_bytes;      /* must equal the body's element size of this stream */
    uint32_t pad;
} fbr_items_desc_t;
int fbr_map_submit_items(fbr_pool_t* pool, const fbr_map_desc_t* desc, const fbr_items_desc_t* items, uint64_t* seq);
int fbr_map_submit_items_n(fbr_pool_t* pool, const fbr_map_desc_t* desc, const fbr_items_desc_t* streams, uint32_t n_streams,
                           uint64_t* seq);

/* Broadcast argument blocks (initargs / arguments every task shares, e.g. the parzen sample array
 * the reference pickles into each of its 102 task messages, SURVEY.md 3.2): uploaded once to every
 * worker's device, then referenced by handle (desc.shared = (void*)handle + FBR_SHARED_HANDLE). */
int fbr_shared_put(fbr_pool_t* pool, const void* host, uint64_t bytes, uint64_t* handle);
int fbr_shared_drop(fbr_pool_t* pool, uint64_t handle);

/* Host-side planning of a map, without touching a device (pure function of its arguments): the claim
 * unit fbr_map_submit would pick, the resulting ring slot stride, and worker w's task block.  Lets
 * the chunking / alignment rules be checked against the reference's chunk plan
 * (fiber/pool.py:1084-1087) on a machine without a GPU. */
typedef struct fbr_plan {
    uint32_t unit_tasks;      /* tasks per claim unit (ring slot) */
    uint32_t slot_stride;     /* bytes per ring slot (multiple of 16) */
    uint64_t n_units;         /* claim units of the whole map */
    uint64_t block_first;     /* worker's block: first task */
    uint64_t block_count;     /*                 number of tasks */
} fbr_plan_t;
int fbr_plan_query(int func_id, uint64_t n_tasks, uint32_t chunksize, uint64_t ring_bytes, int n_workers,
                   int worker, int sm_count, fbr_plan_t* plan);
/* chunksize of fbr_plan_query for the plan of a FBR_FOLD map, which takes no chunksize: the record unit rounded down to
 * a power of two */
#define FBR_PLAN_FOLD 0xffffffffu

/* tree() (see FBR_FOLD) over n records of result_bytes each of FBR_BODY_FOLD body func_id, from host memory into `out`
 * (host), on the pool's first live worker; blocks until done.  n = 0 gives identity(). */
int fbr_fold_values(fbr_pool_t* pool, int func_id, const void* values, uint64_t n, void* out);
/* Wraps the n host records at `values` (result_bytes each, rewritten in place) of FBR_BODY_SCAN body func_id with the
 * n_pieces host records at `pieces`, right-nested: pieces[0] (+) (pieces[1] (+) ( ... (+) (pieces[n_pieces-1] (+) v))),
 * on the pool's first live worker; blocks until done.  With pieces G_1 .. G_m the tree() of the aligned power-of-two
 * ranges of block totals t_0 .. t_{b-1} given by the set bits of b (largest first, fbr_fold_values), this turns block b's
 * own prefix folds into the FBR_SCAN records of a map cut into blocks elsewhere (process-isolated pools). */
int fbr_scan_values(fbr_pool_t* pool, int func_id, const void* pieces, uint32_t n_pieces, void* values, uint64_t n);
/* tree() (see FBR_FOLD) of each segment [offsets[k], offsets[k + 1]) of the host records at `values` (result_bytes each) of
 * FBR_BODY_KEYED body func_id into out[k] (host), identity() for an empty segment, on the pool's first live worker; blocks
 * until done.  offsets are n_segments + 1 non-decreasing host words from 0.  A keyed map's blocks are combined this way. */
int fbr_fold_segments(fbr_pool_t* pool, int func_id, const void* values, const uint64_t* offsets, uint32_t n_segments, void* out);

/* ---- result collection ----------------------------------------------------------------------
 * fbr_result_wait    <- MapResult.get -> Inventory.get (fiber/pool.py:736-737, 666-679)
 * fbr_result_poll    <- Inventory.iget_ordered / iget_unordered progress (fiber/pool.py:681-728)
 * fbr_result_release <- `self._inventory[job_seq] = None` (fiber/pool.py:677-679) */
typedef struct fbr_result {
    uint64_t seq;
    uint64_t n_tasks;
    uint32_t result_bytes;
    uint32_t result_kind;
    void* data;              /* ordered results: pinned host (or the caller's `out`) */
    int64_t sum;             /* valid with FBR_WANT_SUM: sum(results), wrapped to int64 */
    uint32_t err_code;       /* 0, or fbr_task_error of the lowest failing task */
    uint32_t n_waves;
    uint64_t err_task;       /* index of that task */
    uint64_t sum_lo;         /* the exact sum is sum_hi * 2^32 + sum_lo (Python ints are unbounded: the device */
    int64_t sum_hi;          /* folds the two halves of int64 results separately, so nothing wraps silently) */
    uint32_t sum_overflow;   /* 1: the exact sum does not fit int64, `sum` is its low 64 bits */
    uint32_t pad;
} fbr_result_t;

typedef enum fbr_task_error {
    FBR_TASK_OK = 0,
    FBR_TASK_OVERFLOW = 1,   /* int64 result overflow (Python ints are unbounded: fail loudly) */
    FBR_TASK_BADARG = 2,
    FBR_TASK_FAULT = 3,      /* injected fault (resilient-pool tests) */
    FBR_TASK_EMIT = 4,       /* an emit body's task pushed another number of values than its count pass gave */
    FBR_TASK_KEY = 5         /* FBR_FOLD_KEYS: the task's key() is not below n_keys; FBR_FOLD_SPARSE_KEYS: it is 0xFFFFFFFF */
} fbr_task_error;

int fbr_result_wait(fbr_pool_t* pool, uint64_t seq, int timeout_ms, fbr_result_t* res);
/* A FBR_FOLD_SPARSE_KEYS map once fbr_result_wait has succeeded: *n_groups = D, the number of its records; *keys = its D
 * distinct keys in ascending order and *counts = the tasks of each (host memory owned by the map until its release). */
int fbr_result_groups(fbr_pool_t* pool, uint64_t seq, uint64_t* n_groups, const uint32_t** keys, const uint64_t** counts);
int fbr_result_poll(fbr_pool_t* pool, uint64_t seq, uint64_t* n_done);
/* Address of the map's ordered-result buffer without waiting: tasks [0, n_done) of it are final. */
int fbr_result_data(fbr_pool_t* pool, uint64_t seq, void** data);
/* Copy results [first, first+count) of a FBR_RESULTS_ON_DEVICE map to host memory (blocking). */
int fbr_result_fetch(fbr_pool_t* pool, uint64_t seq, uint64_t first, uint64_t count, void* host_dst);
int fbr_result_release(fbr_pool_t* pool, uint64_t seq);
/* Maps of FBR_BODY_EMIT bodies (fbr_map_submit / fbr_map_submit_items, neither `out` nor FBR_OUT_DEVICE): the result
 * records are the n_tasks uint64 end offsets, and the values live in a second segment of n_values elements of out_bytes
 * each, pinned host memory (fbr_result_values: valid from submission on, final where fbr_result_poll says the tasks are;
 * each wave's values reach it by one copy of exactly their span through a staging half of ring_bytes, so a claim unit
 * whose values exceed ring_bytes is refused with FBR_EINVAL)
 * or, with FBR_RESULTS_ON_DEVICE, engine-owned device memory (fbr_result_fetch_values, blocking).  Submission runs the
 * count pass and the scan and waits for them (a count pass that fails is reported by fbr_result_wait); the emit pass
 * then runs like any map.  A worker that dies under an emit map fails it. */
int fbr_result_values(fbr_pool_t* pool, uint64_t seq, void** values, uint64_t* n_values);
int fbr_result_fetch_values(fbr_pool_t* pool, uint64_t seq, uint64_t first, uint64_t count, void* host_dst);

/* ---- memory helpers ------------------------------------------------------------------------
 * Pinned host segments are the endpoints that replace LazyZConnection sockets
 * (fiber/queues.py:190-249): the host encodes argument records straight into them. */
int fbr_host_alloc(fbr_pool_t* pool, uint64_t bytes, void** ptr);
int fbr_host_free(fbr_pool_t* pool, void* ptr);
int fbr_device_alloc(fbr_pool_t* pool, int worker, uint64_t bytes, void** dptr);
int fbr_device_free(fbr_pool_t* pool, int worker, void* dptr);
int fbr_memcpy_h2d(fbr_pool_t* pool, int worker, void* dptr, const void* src, uint64_t bytes);
int fbr_memcpy_d2h(fbr_pool_t* pool, int worker, void* dst, const void* dptr, uint64_t bytes);
/* Fill device memory with the synthetic 4 KB payload records of tasks [t0, t0+n). */
int fbr_payload_fill_device(fbr_pool_t* pool, int worker, void* dptr, uint64_t t0, uint64_t n);

/* ---- statistics ------------------------------------------------------------------------------
 * ZPool keeps bare counters sent_tasks/recv_tasks (fiber/pool.py:902-903); these extend them. */
typedef struct fbr_stats {
    uint64_t tasks_submitted, tasks_completed;
    uint64_t units_dispatched;          /* task records claimed by persistent CTAs */
    uint64_t dispatch_launches, gather_launches, fill_launches;
    uint64_t h2d_bytes, d2h_bytes;
    double dispatch_ms, gather_ms;      /* summed CUDA-event time (FBR_POOL_TIMING only) */
    uint64_t gather_bytes;              /* algorithmic bytes moved by gather_ordered (read+write) */
    uint64_t dispatch_bytes;            /* algorithmic bytes of the dispatch kernels (args+results) */
    uint64_t units_redispatched;        /* lost units re-queued by resilient maps (pending-table resubmits) */
    uint64_t records_copied;            /* task records written to the pinned ring and copied to the device */
    uint64_t direct_waves;              /* waves whose dispatch kernel stored at the final index (no gather) */
    uint64_t peer_push_bytes;           /* argument bytes pushed from worker 0's memory into other workers' staging by
                                           worker 0's copy engine (root-resident maps over NVLink) */
    uint64_t workers_lost;              /* workers retired because their CUDA context died (sticky error); maps with
                                           FBR_RESILIENT had their blocks re-dispatched to the surviving workers */
} fbr_stats_t;
int fbr_pool_stats(fbr_pool_t* pool, fbr_stats_t* stats);
int fbr_pool_stats_reset(fbr_pool_t* pool);

/* ---- SimpleQueue / Pipe / device Process (fiber/queues.py:262-352, fiber/process.py:83-323) ---------
 * Every endpoint owns one SPSC lane of 64-byte records in pinned, device-mapped memory; a queue's
 * forwarder fair-queues its writer lanes into its reader lanes with strict round-robin (the
 * nn_device of fiber/socket.py:297-320; tests/test_queue.py:218-250 pins 600 of 2400 messages per
 * reader).  An endpoint is the host or a device process: a resident one-warp kernel that runs one
 * of the reference tests' process targets against its lanes. */
typedef struct fbr_queue fbr_queue_t;
typedef struct fbr_lane fbr_lane_t;
typedef struct fbr_process fbr_process_t;

typedef enum fbr_record_tag { FBR_REC_NONE = 0, FBR_REC_INT = 1, FBR_REC_FLOAT = 2, FBR_REC_BYTES = 3, FBR_REC_STR = 4 } fbr_record_tag;
typedef struct fbr_record {      /* fixed-layout message: what the reference pickles (queues.py:164-181) */
    uint32_t tag;                /* fbr_record_tag */
    uint32_t len;                /* payload bytes in use */
    uint8_t payload[56];
} fbr_record_t;

typedef enum fbr_process_kind {
    FBR_PROC_QUEUE_WORKER = 1,   /* worker(q_in, q_out, ident)      tests/test_queue.py:44-50 */
    FBR_PROC_PUT_QUEUE = 2,      /* put_queue(q, data)              tests/test_queue.py:23-33 */
    FBR_PROC_GET_QUEUE = 3,      /* get_queue(q_in, q_out, n)       tests/test_queue.py:36-42 */
    FBR_PROC_WRITE_PIPE = 4,     /* write_pipe(pipe, msg)           tests/test_queue.py:19-20 */
    FBR_PROC_PIPE_WORKER = 5     /* pipe_worker(conn)               tests/test_queue.py:53-57 */
} fbr_process_kind;

const char* fbr_queue_last_error(void);
int fbr_queue_create(fbr_queue_t** q);                                   /* SimpleQueuePush.__init__ / Pipe */
int fbr_queue_open_writer(fbr_queue_t* q, fbr_lane_t** lane);            /* LazyZConnection(("w", addr)) */
int fbr_queue_open_reader(fbr_queue_t* q, fbr_lane_t** lane);            /* LazyZConnection(("r", addr)) */
int fbr_lane_send(fbr_lane_t* lane, const fbr_record_t* rec, int timeout_ms);   /* ZConnection.send */
int fbr_lane_recv(fbr_lane_t* lane, fbr_record_t* rec, int timeout_ms);         /* ZConnection.recv */
int fbr_lane_poll(fbr_lane_t* lane, int* ready);                                 /* ZConnection._poll */
int fbr_queue_put(fbr_queue_t* q, const fbr_record_t* rec, int timeout_ms);     /* SimpleQueuePush.put */
int fbr_queue_get(fbr_queue_t* q, fbr_record_t* rec, int timeout_ms);           /* SimpleQueuePush.get */
int fbr_queue_stats(fbr_queue_t* q, uint64_t* forwarded, uint32_t* n_writers, uint32_t* n_readers);
int fbr_queue_destroy(fbr_queue_t* q);
/* Process.start / is_alive+exitcode / join / terminate (fiber/process.py:187-215, 217-262). */
int fbr_process_start(int device_id, int kind, fbr_lane_t* in, fbr_lane_t* out, int64_t ident,
                      const fbr_record_t* msg, const fbr_record_t* list, uint32_t list_len, int idle_timeout_ms,
                      fbr_process_t** proc);
int fbr_process_poll(fbr_process_t* proc, int* alive, int* exitcode);
int fbr_process_join(fbr_process_t* proc, int timeout_ms);
int fbr_process_terminate(fbr_process_t* proc);
int fbr_process_handled(fbr_process_t* proc, uint64_t* handled);
int fbr_process_destroy(fbr_process_t* proc);

/* ---- express lane: doorbell path for one-task submissions (apply / apply_async) --------------------
 * A resident one-warp kernel per device polls a pinned, device-mapped request lane, runs the body and
 * writes the result record into a pinned response lane the host polls: no kernel launch, copy or
 * event on the round trip (fiber/pool.py:1089-1116 pays a TCP round trip per apply).  The kernel exits
 * after `idle_timeout_us` without requests and is relaunched on demand.  Bodies whose argument and
 * result fit 48 bytes: square_i64, mul2_i64, square_scale_i64, identity_i64, pi_inside_det, sleep_f64. */
typedef struct fbr_express fbr_express_t;
const char* fbr_express_last_error(void);
int fbr_express_create(int device_id, int idle_timeout_us, fbr_express_t** x);
int fbr_express_submit(fbr_express_t* x, int func_id, const void* arg, uint32_t arg_bytes, uint64_t* ticket);
int fbr_express_wait(fbr_express_t* x, uint64_t ticket, void* result, uint32_t* result_bytes, uint32_t* err, int timeout_ms);
int fbr_express_discard(fbr_express_t* x, uint64_t ticket);   /* handle dropped without a wait: forget the response */
int fbr_express_stats(fbr_express_t* x, uint64_t* served, uint64_t* launches, int* resident);
int fbr_express_destroy(fbr_express_t* x);

/* ---- engine-level collectives: one process per GPU (SURVEY.md 8(e); fiber/experimental/ring.py:44-129) ---------
 * The map shards by contiguous task block with no data-path collective; what surrounds it does exchange data:
 * shared arguments that live on one rank (ncclBroadcast), an input array resident on one rank (scatter =
 * grouped ncclSend/ncclRecv: the fan-out of fiber/pool.py:910-914), the ordered result blocks (ncclAllGather, or
 * grouped send/recv to a root: the fan-in of fiber/pool.py:916-920), scalar folds (ncclAllReduce int64) and
 * experimental.Ring's all-reduce (examples/ring.py:81-86).  A communicator is bound to one CUDA device and owns
 * one stream; calls enqueue on it, fbr_comm_sync waits.  The 128-byte bootstrap id (ncclUniqueId) is what a ring
 * node publishes in the member table instead of the reference's ip/port.  NCCL is dlopen()ed on first use. */
typedef struct fbr_comm fbr_comm_t;
#define FBR_COMM_ID_BYTES 128
typedef enum fbr_dtype { FBR_DT_U8 = 0, FBR_DT_I32 = 1, FBR_DT_I64 = 2, FBR_DT_F32 = 3, FBR_DT_F64 = 4 } fbr_dtype;
typedef enum fbr_redop { FBR_OP_SUM = 0, FBR_OP_PROD = 1, FBR_OP_MAX = 2, FBR_OP_MIN = 3 } fbr_redop;
const char* fbr_comm_last_error(void);
int fbr_comm_load(const char* libnccl_path, int* version);          /* optional: pick the NCCL build; reports its version */
int fbr_comm_unique_id(void* id128);                                 /* rank 0: ncclGetUniqueId */
int fbr_comm_create(int device_id, int nranks, int rank, const void* id128, fbr_comm_t** comm);   /* ncclCommInitRank */
int fbr_comm_info(fbr_comm_t* comm, int* rank, int* nranks, int* device_id);
int fbr_comm_sync(fbr_comm_t* comm);
int fbr_comm_broadcast(fbr_comm_t* comm, void* dptr, uint64_t bytes, int root);
int fbr_comm_allgather(fbr_comm_t* comm, const void* send, void* recv, uint64_t bytes_per_rank);
int fbr_comm_gather(fbr_comm_t* comm, const void* send, void* recv_on_root, uint64_t bytes_per_rank, int root);
int fbr_comm_scatter(fbr_comm_t* comm, const void* send_on_root, void* recv, uint64_t bytes_per_rank, int root);
int fbr_comm_allreduce(fbr_comm_t* comm, const void* send, void* recv, uint64_t count, int dtype, int op);
int fbr_comm_allreduce_timed(fbr_comm_t* comm, void* buf, uint64_t count, int dtype, int op, int iters, float* ms_per_call);
int fbr_comm_allreduce_i64(fbr_comm_t* comm, int64_t* value);       /* host scalar in, global sum out (the pi count) */
int fbr_comm_allreduce_i64_begin(fbr_comm_t* comm, int64_t value);  /* the same, split: enqueue now ...               */
int fbr_comm_allreduce_i64_end(fbr_comm_t* comm, int64_t* sum);     /* ... collect later (overlaps the next map)      */
int fbr_comm_device_alloc(fbr_comm_t* comm, uint64_t bytes, void** dptr);
int fbr_comm_device_free(fbr_comm_t* comm, void* dptr);
int fbr_comm_memcpy_h2d(fbr_comm_t* comm, void* dptr, const void* src, uint64_t bytes);
int fbr_comm_memcpy_d2h(fbr_comm_t* comm, void* dst, const void* dptr, uint64_t bytes);
int fbr_comm_destroy(fbr_comm_t* comm);

#ifdef __cplusplus
}
#endif
#endif /* FIBER_B200_H_ */
