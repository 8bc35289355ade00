"""Generated record bodies, one per layout of dispatch_record_kernel: argument and result sizes at the edges of every
``kAlign`` class, group sizes 1 to 32, broadcast blocks at and around their staging limit, item streams of every element
size class and emit bodies of every ``Out`` size class.

Every body computes an integer hash of everything its task sees, so the GPU results are compared bit for bit with the
NumPy restatement below.  For result word ``j`` of ``Rw = R / 4`` words, argument words ``a[0 .. Aw)`` and task index
``t``::

    r[j] = ((a[j % Aw] * 0x9E3779B1 + rotl(a[(7j + 3) % Aw], 13)) ^ (lo32(t) + j * 0x85EBCA77))
           + sum over k = j, j + Rw, ... < Aw of (a[k] * (2k + 1) + k)

(``Aw = 0``, an items body without a head record: ``r[j] = lo32(t) + j * 0x85EBCA77``.)  So every result word depends on
the task index, and every argument word reaches a result word with a weight set by its position: a dropped, shifted or
swapped word changes the result.  A group body's lane ``rank`` writes words ``rank, rank + G, ...``.  On top of that:

- broadcast bodies add, to word ``j``, ``esum`` of element ``(t * 2654435761 + j) mod n`` of the block, and to word 0
  ``esum`` of the first element plus 3 ``esum`` of the last, so a wrong tail copy shows in every task
  (``esum(e) = sum of e's words w[m] * (2m + 1)``);
- items bodies add, for stream ``s``, to word ``s % Rw``: the element count plus the sum of the task's element words
  ``x[q] * (2q + 1)``, ``q`` counted from the task's first word (1- and 2-byte elements are widened to one word);
- emit bodies push ``c = mix32(seed ^ 0x5BD1E995) mod (cmax + 1)`` values, the ``w``-th word of value ``k`` being
  ``mix32(seed * 0x9E3779B1 + k * 0x85EBCA77 + w * 0xC2B2AE3D) ^ lo32(t)`` (1- and 2-byte values: its low bytes).  An
  index body's seed is ``lo32(a)``, and a negative index pushes nothing.  Group emit bodies test candidates
  ``q < c`` split by rank (``q = m + rank``) and push the ones with ``cand(seed, q) & 1`` in rank order.

Fault variants (``kCanFault``) report TASK_FAULT for about 5 % of tasks on attempts 0 and 1, seeded by (task, attempt):
a resilient map re-dispatches their units and must still place every result.

The bodies are generated into three translation units (fixed records, broadcast and items, emit), each compiled once with
``bodies.compile_module`` and registered with ``registry.register_module``.
"""
import numpy as np

from fiber_b200 import bodies, registry

# kStageBytes and kSmemBudget of dispatch_record_kernel (kernels.cuh, namespace record)
STAGE_BYTES = 32768
SMEM_BUDGET = 200 << 10
MAX_UNIT = 1024


class Layout:
    """One generated body.  A and R are the argument and result record sizes in bytes (A = 0: no head record; an emit
    body's R is its 8-byte end offset); ``index``: Arg = int64_t with kIndexArg; ``shared``: (element bytes, kSharedStage);
    ``items``: element sizes of its streams; ``out``: (Out bytes, cmax, defines count()); ``group``: kGroup (1: one
    thread per task)."""

    def __init__(self, name, A, R, group=1, index=False, fault=False, shared=None, items=(), out=None, module="fixed"):
        self.name, self.A, self.R, self.group, self.index, self.fault = name, A, R, group, index, fault
        self.shared, self.items, self.out, self.module = shared, tuple(items), out, module
        if out is not None:
            self.R = 8

    @property
    def k_align(self):
        return align_tasks(self.A, self.R)

    @property
    def k_unit(self):
        return stage_unit(self.A, self.R)

    @property
    def smem(self):
        return 2 * self.k_unit * self.A + 2 * self.k_unit * self.R + (self.shared[1] if self.shared else 0)


def align_tasks(A, R):
    """record::align_tasks: tasks per unit that keep count * A and count * R multiples of 16."""
    return 1 if (A % 16 == 0 and R % 16 == 0) else 2 if (A % 8 == 0 and R % 8 == 0) else 4


def stage_unit(A, R):
    """record::Layout<B>::kUnit: halved from 1024 until the larger record's stage fits 32 KB (not below kAlign)."""
    u, w, al = MAX_UNIT, max(A, R), align_tasks(A, R)
    while u > al and u * w > STAGE_BYTES:
        u >>= 1
    return u


L = Layout
SMALL_STAGE = SMEM_BUDGET - 4 * 1024 * 16          # next to 16 B / 16 B records (1024 tasks per unit: 64 KB of stages)
TINY_STAGE = SMEM_BUDGET - 4 * 1024 * 4            # next to 4 B / 4 B records
LAYOUTS = [
    # ---- fixed records: the largest of each kAlign class, R >> A and A >> R, every group size
    L("lay_a4_r4", 4, 4),
    L("lay_a4_r4096", 4, 4096),
    L("lay_a4092_r4", 4092, 4),
    L("lay_a8_r24", 8, 24),
    L("lay_a24_r8", 24, 8),
    L("lay_a12_r4096", 12, 4096),
    L("lay_a4096_r12", 4096, 12),
    L("lay_a2052_r2052", 2052, 2052),
    L("lay_a20_r20", 20, 20),
    L("lay_i8_r4096", 8, 4096, index=True),
    L("lay_i8_r12", 8, 12, index=True),
    L("lay_a8_r16384_g2", 8, 16384, group=2),
    L("lay_a16384_r8_g2", 16384, 8, group=2),
    L("lay_a4_r8188_g4", 4, 8188, group=4),
    L("lay_a8188_r4_g4", 8188, 4, group=4),
    L("lay_a32768_r32768_g32", 32768, 32768, group=32),
    L("lay_a16_r32768_g32", 16, 32768, group=32),
    L("lay_a32768_r16_g8", 32768, 16, group=8),
    L("lay_a20_r36_g16", 20, 36, group=16),
    L("lay_i8_r16384_g32", 8, 16384, group=32, index=True),
    L("lay_i8_r8184_g8", 8, 8184, group=8, index=True),
    # ---- kCanFault: one per gather route of a full unit (flat, rows, and a bulk-sized slot)
    L("flt_a2052_r2052", 2052, 2052, fault=True),
    L("flt_a4_r4", 4, 4, fault=True),
    L("flt_a4_r4096", 4, 4096, fault=True),
    L("flt_a20_r36_g16", 20, 36, group=16, fault=True),
    # ---- broadcast blocks: elements of 4, 12 and 4096 bytes; never staged, a 4 KB stage, and the largest stage
    L("bc_e4_s0", 12, 16, shared=(4, 0), module="shared"),
    L("bc_e4_s4096", 12, 16, shared=(4, 4096), module="shared"),
    L("bc_e12_s4096", 8, 8, shared=(12, 4096), module="shared"),
    L("bc_e12_big", 4, 4, shared=(12, TINY_STAGE), module="shared"),
    L("bc_e4096_big", 16, 16, shared=(4096, SMALL_STAGE), module="shared"),
    L("bc_e4_s4096_g8", 20, 36, group=8, shared=(4, 4096), module="shared"),
    # ---- items: one stream of each element size class, four streams, no head record or a 12 B one, groups of 8 and 32
    L("it_u1", 0, 8, items=(1,), module="shared"),
    L("it_u2", 0, 8, items=(2,), module="shared"),
    L("it_h12_u8", 12, 12, items=(8,), module="shared"),
    L("it_w12", 0, 16, items=(12,), module="shared"),
    L("it_h12_w4096_g8", 12, 8, group=8, items=(4096,), module="shared"),
    L("it_h12_u1_g32", 12, 4096, group=32, items=(1,), module="shared"),
    L("it4_g32", 0, 16, group=32, items=(1, 2, 12, 4096), module="shared"),
    L("it4_h12", 12, 20, items=(1, 2, 12, 4096), module="shared"),
    # ---- emit: Out of every size class, with and without count(), a G = 32 push_if body, and everything at once
    L("em_o1", 8, 0, index=True, out=(1, 9, True), module="emit"),
    L("em_o2", 8, 0, index=True, out=(2, 9, False), module="emit"),
    L("em_o8", 8, 0, index=True, out=(8, 9, True), module="emit"),
    L("em_o12", 8, 0, index=True, out=(12, 9, False), module="emit"),
    L("em_o4096", 8, 0, index=True, out=(4096, 3, True), module="emit"),
    L("em_o4_g32", 8, 0, group=32, index=True, out=(4, 70, False), module="emit"),
    L("em_mix_g8", 12, 0, group=8, items=(2,), shared=(4, 4096), out=(12, 20, False), module="emit"),
]
BY_NAME = {b.name: b for b in LAYOUTS}
MODULES = ("fixed", "shared", "emit")

PRELUDE = r'''
#include "fiber_b200_body.cuh"

namespace lb {
template <uint32_t N>
struct Words { uint32_t w[N]; };

__device__ __forceinline__ uint32_t rotl13(uint32_t x) { return (x << 13) | (x >> 19); }
__device__ __forceinline__ uint32_t mix32(uint32_t x) {
    x ^= x >> 16; x *= 0x85EBCA6Bu; x ^= x >> 13; x *= 0xC2B2AE35u; x ^= x >> 16;
    return x;
}
// result words rank, rank + G, ... of a task from its AW argument words (AW = 0: none)
template <uint32_t AW, uint32_t RW, uint32_t G>
__device__ __forceinline__ void fill(const uint32_t* a, uint32_t* r, uint64_t t, uint32_t rank) {
    for (uint32_t j = rank; j < RW; j += G) {
        uint32_t v = (uint32_t)t + j * 0x85EBCA77u;
        if constexpr (AW > 0) {
            v = (a[j % AW] * 0x9E3779B1u + rotl13(a[(7u * j + 3u) % AW])) ^ v;
            for (uint32_t k = j; k < AW; k += RW) v += a[k] * (2u * k + 1u) + k;
        }
        r[j] = v;
    }
}
template <class T>
__device__ __forceinline__ const uint32_t* words(const T& a) { return reinterpret_cast<const uint32_t*>(&a); }
// the weighted words of one element
template <class T>
__device__ __forceinline__ uint32_t esum(const T& e) {
    const uint32_t* w = words(e);
    uint32_t v = 0;
    for (uint32_t m = 0; m < sizeof(T) / 4; ++m) v += w[m] * (2u * m + 1u);
    return v;
}
// a broadcast block's share of result words rank, rank + G, ...
template <uint32_t RW, uint32_t G, class T>
__device__ __forceinline__ void add_block(uint32_t* r, const fbr::Broadcast<T>& sh, uint64_t t, uint32_t rank) {
    for (uint32_t j = rank; j < RW; j += G) r[j] += esum(sh.data[(t * 2654435761ull + j) % sh.n]);
    if (rank == 0) r[0] += esum(sh.data[0]) + 3u * esum(sh.data[sh.n - 1]);
}
// a task's items: their count plus their words weighted by position (1- and 2-byte elements widened)
template <class T>
__device__ __forceinline__ uint32_t items_sum(const fbr::Items<T>& x) {
    uint32_t v = (uint32_t)x.n;
    if constexpr (sizeof(T) <= 2) {
        for (uint64_t q = 0; q < x.n; ++q) v += (uint32_t)x.data[q] * (2u * (uint32_t)q + 1u);
    } else {
        const uint32_t* w = reinterpret_cast<const uint32_t*>(x.data);
        const uint64_t m = x.n * (sizeof(T) / 4);
        for (uint64_t q = 0; q < m; ++q) v += w[q] * (2u * (uint32_t)q + 1u);
    }
    return v;
}
template <uint32_t RW, uint32_t G, class T>
__device__ __forceinline__ void add_items(uint32_t* r, uint32_t s, const fbr::Items<T>& x, uint32_t rank) {
    if ((s % RW) % G == rank) r[s % RW] += items_sum(x);
}
__device__ __forceinline__ bool faults(uint64_t t, uint32_t attempt) {
    return attempt < 2 && mix32((uint32_t)t * 0x9E3779B1u ^ attempt * 0x85EBCA77u ^ 0xFA17u) % 100u < 5u;
}
// emit bodies
__device__ __forceinline__ uint32_t emit_n(uint32_t seed, uint32_t cmax) { return mix32(seed ^ 0x5BD1E995u) % (cmax + 1u); }
__device__ __forceinline__ uint32_t cand(uint32_t seed, uint32_t q) { return mix32(seed ^ (q * 0x27D4EB2Fu)); }
__device__ __forceinline__ uint32_t value_word(uint32_t seed, uint64_t t, uint32_t k, uint32_t w) {
    return mix32(seed * 0x9E3779B1u + k * 0x85EBCA77u + w * 0xC2B2AE3Du) ^ (uint32_t)t;
}
template <class T>
__device__ __forceinline__ T value(uint32_t seed, uint64_t t, uint32_t k) {
    T v;
    if constexpr (sizeof(T) <= 2) {
        v = (T)value_word(seed, t, k, 0);
    } else {
        uint32_t* w = reinterpret_cast<uint32_t*>(&v);
        for (uint32_t m = 0; m < sizeof(T) / 4; ++m) w[m] = value_word(seed, t, k, m);
    }
    return v;
}
__device__ __forceinline__ uint32_t index_seed(int64_t a) { return (uint32_t)(uint64_t)a; }
}  // namespace lb
'''


def _ctype(nbytes):
    return {1: "uint8_t", 2: "uint16_t"}.get(nbytes, "lb::Words<%d>" % (nbytes // 4))


def _source(b):
    """The CUDA struct and export of one layout."""
    s = b.name.upper()
    G, AW, RW = b.group, b.A // 4, b.R // 4
    rank = "g.rank" if G > 1 else "0u"
    lines = ["struct %s {" % s]
    if b.index:
        lines.append("    using Arg = int64_t;")
    elif b.A == 0:
        lines.append("    using Arg = fbr::NoArg;")
    else:
        lines.append("    using Arg = lb::Words<%d>;" % AW)
    if b.out is not None:
        lines += ["    using Out = %s;" % _ctype(b.out[0]), "    using Res = fbr::NoRes;"]
    else:
        lines.append("    using Res = lb::Words<%d>;" % RW)
    if len(b.items) == 1:
        lines.append("    using Item = %s;" % _ctype(b.items[0]))
    elif b.items:
        lines.append("    using Items = fbr::ItemTypes<%s>;" % ", ".join(_ctype(e) for e in b.items))
    if b.shared:
        lines += ["    using Shared = %s;" % _ctype(b.shared[0]), "    static constexpr uint32_t kSharedStage = %d;" % b.shared[1]]
    if G > 1:
        lines.append("    static constexpr uint32_t kGroup = %d;" % G)
    lines.append("    static constexpr bool kIndexArg = %s, kCanFault = %s;" % (str(b.index).lower(), str(b.fault).lower()))
    head = [] if b.A == 0 else ["const Arg& a"]
    xs = ["const fbr::Items<%s>& x%d" % (_ctype(e), k) for k, e in enumerate(b.items)]
    sh = ["const fbr::Broadcast<Shared>& sh"] if b.shared else []
    grp = ["const fbr::Group<%d>& g" % G] if G > 1 else []
    tail = ["uint64_t t", "const fbr::ErrSink& es", "uint32_t attempt"]
    if b.out is None:
        body = ["lb::fill<%d, %d, %d>(%s, r.w, t, %s);" % (AW, RW, G, "lb::words(a)" if AW else "nullptr", rank)]
        body += ["lb::add_items<%d, %d>(r.w, %d, x%d, %s);" % (RW, G, k, k, rank) for k in range(len(b.items))]
        if b.shared:
            body.append("lb::add_block<%d, %d>(r.w, sh, t, %s);" % (RW, G, rank))
        if b.fault:
            body.append("if (%s == %du && lb::faults(t, attempt)) es.report(fbr::TASK_FAULT, t);" % (rank, G - 1))
        params = head + xs + ["Res& r"] + sh + grp + tail
    else:
        ob, cmax, with_count = b.out
        if b.index:
            seed = "a < 0 ? 0u : lb::emit_n(lb::index_seed(a), %du)" % cmax
            body = ["const uint32_t seed = lb::index_seed(a);", "const uint32_t c = %s;" % seed]
        else:
            body = ["const uint32_t seed = a.w[0] ^ lb::items_sum(x0) ^ lb::esum(sh.data[t % sh.n]);",
                    "const uint32_t c = lb::emit_n(seed, %du);" % cmax]
        if G == 1:
            body.append("for (uint32_t k = 0; k < c; ++k) y.push(lb::value<Out>(seed, t, k));")
        else:
            body.append("for (uint32_t m = 0; m < c; m += %d) {" % G)
            body.append("    const uint32_t q = m + g.rank;")
            body.append("    y.push_if(g, q < c && (lb::cand(seed, q) & 1u), lb::value<Out>(seed, t, q));")
            body.append("}")
        if with_count:
            lines.append("    __device__ static __forceinline__ uint64_t count(%s) {" % ", ".join(head + xs + sh + ["uint64_t t"]))
            lines += ["        " + x for x in body[:2]]
            lines.append("        return c;")
            lines.append("    }")
        params = head + xs + ["fbr::Emit<Out%s>& y" % (", %d" % G if G > 1 else "")] + sh + grp + tail
    lines.append("    __device__ static __forceinline__ void run(%s) {" % ", ".join(params))
    lines += ["        " + x for x in body]
    lines += ["    }", "};"]
    lines.append('FBR_EXPORT_RECORD_BODY(%s, "%s", %s_entry, %s)' % (s, b.name, b.name, "FBR_BODY_INDEX_ARG" if b.index else "0"))
    return "\n".join(lines) + "\n"


def module_source(module):
    return PRELUDE + "\n".join(_source(b) for b in LAYOUTS if b.module == module)


def _dtypes(b):
    """(args, result, shared, items, out) keyword arguments of register_module."""
    kw = {"args": "<i8" if b.index else None if b.A == 0 else [("a", "<u4", (b.A // 4,))]}
    if b.out is None:
        kw["result"] = [("r", "<u4", (b.R // 4,))]
    else:
        kw["out"] = elem_dtype(b.out[0])
    if b.shared:
        kw["shared"] = ("block", elem_dtype(b.shared[0]))
    if len(b.items) == 1:
        kw["items"] = ("x0", elem_dtype(b.items[0]))
    elif b.items:
        kw["items"] = [("x%d" % k, elem_dtype(e)) for k, e in enumerate(b.items)]
    return kw


def elem_dtype(nbytes):
    """The NumPy dtype of an element the generated source declares: uint8, uint16, uint32 or lb::Words<nbytes / 4>."""
    return np.dtype({1: "<u1", 2: "<u2", 4: "<u4"}[nbytes] if nbytes <= 4 else [("w", "<u4", (nbytes // 4,))])


def register():
    for m in MODULES:
        path = bodies.compile_module("layout_" + m, module_source(m))
        for b in LAYOUTS:
            if b.module == m:
                kw = _dtypes(b)
                if kw["args"] is None:
                    del kw["args"]
                registry.register_module(b.name, path, b.name + "_entry", **kw)


register()


# ---- NumPy restatements ---------------------------------------------------------------------------------------------
M32 = np.uint64(0xFFFFFFFF)
_ZERO = np.zeros(1, np.uint64)


def _u32(x):
    return (np.asarray(x, np.uint64) & M32).astype(np.uint32)


def rotl13(x):
    return (x << np.uint32(13)) | (x >> np.uint32(19))


def mix32(x):
    x = np.asarray(x, np.uint32)
    x = x ^ (x >> np.uint32(16))
    x = x * np.uint32(0x85EBCA6B)
    x = x ^ (x >> np.uint32(13))
    x = x * np.uint32(0xC2B2AE35)
    return x ^ (x >> np.uint32(16))


def words_of(recs, nbytes):
    """(n, nbytes / 4) uint32 words of n records of nbytes (a structured array, or int64 indices)."""
    return np.ascontiguousarray(recs).view(np.uint32).reshape(len(recs), nbytes // 4)


def fill_np(aw, RW, t):
    """The result words of tasks t (uint64) from argument words aw ((n, Aw) uint32, or None)."""
    j = np.arange(RW, dtype=np.uint32)
    v = _u32(t)[:, None] + j[None, :] * np.uint32(0x85EBCA77)
    if aw is None:
        return v
    n, AW = aw.shape
    v = (aw[:, j % AW] * np.uint32(0x9E3779B1) + rotl13(aw[:, (7 * j.astype(np.uint64) + 3) % AW])) ^ v
    k = np.arange(AW, dtype=np.uint32)
    c = aw * (np.uint32(2) * k + np.uint32(1)) + k
    c = np.pad(c, ((0, 0), (0, (-AW) % RW))).reshape(n, -1, RW).sum(axis=1, dtype=np.uint64)
    return v + _u32(c)


def esum_np(block, E):
    w = words_of(block, E)
    m = np.arange(w.shape[1], dtype=np.uint64)
    return _u32((w * (2 * m + 1)).sum(axis=1, dtype=np.uint64))


def add_block_np(r, block, E, t):
    e = esum_np(block, E)
    n = np.uint64(len(e))
    j = np.arange(r.shape[1], dtype=np.uint64)
    idx = (t.astype(np.uint64)[:, None] * np.uint64(2654435761) + j[None, :]) % n
    r += e[idx]
    r[:, 0] += e[0] + np.uint32(3) * e[-1]
    return r


def item_words(values, E):
    """The word stream of an item array: 1- and 2-byte elements widened, larger ones as their uint32 words."""
    v = np.ascontiguousarray(values)
    return v.astype(np.uint32) if E <= 2 else v.view(np.uint32).reshape(-1)


def items_sum_np(values, offsets, E):
    """Per task [offsets[i], offsets[i+1]): count + sum of word q (from the task's first word) times 2q + 1."""
    ew = 1 if E <= 2 else E // 4
    w = item_words(values, E).astype(np.uint64)
    p = np.arange(len(w), dtype=np.uint64)
    s1 = np.concatenate([_ZERO, np.cumsum(w * (2 * p + 1), dtype=np.uint64)])
    s0 = np.concatenate([_ZERO, np.cumsum(w, dtype=np.uint64)])
    o = np.asarray(offsets, np.uint64)
    a, b = o[:-1] * np.uint64(ew), o[1:] * np.uint64(ew)
    with np.errstate(over="ignore"):
        v = (s1[b] - s1[a]) - np.uint64(2) * a * (s0[b] - s0[a]) + (o[1:] - o[:-1])
    return _u32(v)


def results_np(b, n, t0=0, args=None, block=None, streams=()):
    """Result records (n, R / 4) uint32 of a fixed-result layout for tasks t0 .. t0 + n - 1.  args: the argument
    records (or int64 indices); block: the broadcast block; streams: (values, offsets) per item stream."""
    t = np.arange(t0, t0 + n, dtype=np.uint64)
    aw = None if b.A == 0 else words_of(np.asarray(args, np.int64) if b.index else args, b.A)
    with np.errstate(over="ignore"):
        r = fill_np(aw, b.R // 4, t)
        for s, ((vals, offs), E) in enumerate(zip(streams, b.items)):
            r[:, s % (b.R // 4)] += items_sum_np(vals, offs, E)
        if b.shared:
            add_block_np(r, block, b.shared[0], t)
    return r


def _values(seed, t, k, ob):
    """Emitted values (len(k) elements of ob bytes) for task seeds / indices and value numbers k."""
    ow = max(1, ob // 4)
    w = np.arange(ow, dtype=np.uint32)
    v = mix32(seed[:, None] * np.uint32(0x9E3779B1) + k[:, None] * np.uint32(0x85EBCA77) + w[None, :] * np.uint32(0xC2B2AE3D))
    v = v ^ _u32(t)[:, None]
    if ob <= 2:
        return v[:, 0].astype(np.uint8 if ob == 1 else np.uint16)
    return np.ascontiguousarray(v).view(elem_dtype(ob)).reshape(-1)


def emit_np(b, n, t0=0, args=None, block=None, streams=()):
    """(end offsets from 0, values) of an emit layout."""
    ob, cmax, _ = b.out
    t = np.arange(t0, t0 + n, dtype=np.uint64)
    with np.errstate(over="ignore"):
        if b.index:
            a = np.asarray(args, np.int64)
            seed = _u32(a.view(np.uint64))
            c = np.where(a < 0, 0, mix32(seed ^ np.uint32(0x5BD1E995)) % np.uint32(cmax + 1)).astype(np.int64)
        else:
            vals, offs = streams[0]
            e = esum_np(block, b.shared[0])
            seed = words_of(args, b.A)[:, 0] ^ items_sum_np(vals, offs, b.items[0]) ^ e[(t % np.uint64(len(e)))]
            c = (mix32(seed ^ np.uint32(0x5BD1E995)) % np.uint32(cmax + 1)).astype(np.int64)
        task = np.repeat(np.arange(n), c)
        start = np.cumsum(c) - c
        k = (np.arange(len(task)) - start[task]).astype(np.uint32)
        if b.group > 1:                                    # candidates q < c whose cand bit is set, in rank order
            keep = (mix32(seed[task] ^ (k * np.uint32(0x27D4EB2F))) & np.uint32(1)) == 1
            task, k = task[keep], k[keep]
        vals = _values(seed[task], t[task], k, ob)
        ends = np.cumsum(np.bincount(task, minlength=n)).astype(np.uint64)
    return ends, vals


# ---- seeded inputs --------------------------------------------------------------------------------------------------
def arg_dtype(b):
    return registry.spec(b.name).arg_dtype


def make_args(b, n, seed):
    """n argument records of layout b: random words (int64 indices for an index body, some of them negative)."""
    rng = np.random.default_rng(seed)
    if b.index:
        return rng.integers(-2 ** 62, 2 ** 62, n, dtype=np.int64)
    a = np.empty(n, arg_dtype(b))
    a.view(np.uint32)[:] = rng.integers(0, 2 ** 32, n * (b.A // 4), dtype=np.uint32).reshape(a.view(np.uint32).shape)
    return a


def make_block(b, n_elems, seed):
    rng = np.random.default_rng(seed)
    E = b.shared[0]
    blk = np.empty(n_elems, elem_dtype(E))
    blk.view(np.uint32)[:] = rng.integers(1, 2 ** 32, blk.nbytes // 4, dtype=np.uint32)
    return blk


def make_items(E, counts, seed, first=0):
    """(values, offsets) of one stream: task i has counts[i] elements; offsets start at `first` (values before it are
    never read)."""
    rng = np.random.default_rng(seed)
    offs = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint64) + np.uint64(first)
    total = int(offs[-1])
    vals = np.empty(total, elem_dtype(E))
    v = vals.view(np.uint8)
    v[:] = rng.integers(0, 256, v.size, dtype=np.uint8)
    return vals, offs
