"""The kernel choice table: which gather and dispatch kernel each map of the kernel-choice suite is meant to reach.

The engine picks a gather kernel per wave (engine.cu ``pick_gather``, from the block's ``BlockPlan``) and the
payload body picks its dispatch kernel per launch (``launch_payload_map``), from the claim unit, the slot stride, the
output pointer and the map flags.  ``expected_kernel`` and ``expected_dispatch`` restate those rules;
``CASES`` lists the maps, each with the cell (kernel and the edge of its index arithmetic) it is meant to reach; ``CELLS``
says what each cell is and which task counts it must be run at.  tests/test_kernel_choice_cpu.py checks through
``fbr_plan_query`` that every case lands in its cell and that every cell is covered, so a change to the selection rule or to
the claim-unit planner fails there instead of silently thinning the GPU suite (tests/test_kernel_choice_gpu.py).

Task counts are named by their remainder against the claim unit of the map's own plan: ``one`` (n = 1), ``minus_one``
(n mod unit = unit - 1: one short unit at the end), ``exact`` (n mod unit = 0), ``plus_one`` (n mod unit = 1, n > 1: a
one-task tail unit), and ``waves``: at least four waves of a small ring (checked on the GPU from the result's wave count).
Bodies whose unit shrinks for small maps (pick_unit: units above 256 tasks halve until every SM gets one) reach a cell
only above 132 units, so their cases use k * unit - 1, k * unit and k * unit + 1 there.
"""
import contextlib
import ctypes
import os
from collections import namedtuple

from fiber_b200 import _abi, registry

from . import layout_bodies as LB

SM_COUNT = 132
CHUNK = 16384                      # bulk::kChunk
SMALL_RING = 1 << 20
DEFAULT_RING = 256 << 20
PAYLOAD = ("payload_map_4k", "payload_checksum_4k")

PLACE_FLAGS = {"direct": 0, "ring": _abi.FBR_VIA_RING, "shuffle": _abi.FBR_SHUFFLE, "resilient": _abi.FBR_RESILIENT,
               "out0": _abi.FBR_OUT_DEVICE, "out4": _abi.FBR_OUT_DEVICE}


@contextlib.contextmanager
def knobs(env):
    """Set the environment knobs of one map and restore the previous values afterwards.  The engine reads the per-call
    knobs at submit and at every wave, so no map may be in flight while they change."""
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


class Case(namedtuple("Case", "cell body n chunksize ring env place args stride want_sum waves")):
    """One map.  ring: the pool's ring_bytes (0: the default); env: per-call knobs; place: a key of PLACE_FLAGS; args:
    "host", "dev" or "range"; stride: arg_stride of a payload map (0: the body's record size)."""

    @property
    def id(self):
        knob = ",".join("%s=%s" % (k[4:], v) for k, v in sorted(self.env.items()))
        return "%s:%s:n=%d:cs=%d:ring=%dK:%s:%s%s%s" % (self.cell, self.body, self.n, self.chunksize, (self.ring or DEFAULT_RING) >> 10,
                                                   self.place, self.args, ":stride=%d" % self.stride if self.stride else "",
                                                   ":" + knob if knob else "")

    @property
    def flags(self):
        f = PLACE_FLAGS[self.place]
        if self.args == "dev":
            f |= _abi.FBR_ARGS_DEVICE
        if self.want_sum:
            f |= _abi.FBR_WANT_SUM
        return f

    @property
    def out_offset(self):
        return 4 if self.place == "out4" else 0

    @property
    def result_bytes(self):
        return registry.spec(self.body).result_bytes

    @property
    def arg_stride(self):
        if self.args == "range":
            return 0
        return self.stride or registry.spec(self.body).arg_bytes


def plan_of(body, n, chunksize=0, ring=0, env=None):
    """fbr_plan_query for a one-worker pool of 132 SMs under the given knobs."""
    p = _abi.Plan()
    with knobs(env or {}):
        _abi.check(_abi.load().fbr_plan_query(registry.spec(body).func_id, n, chunksize, ring, 1, 0, SM_COUNT, ctypes.byref(p)))
    return p


def case_plan(c):
    return plan_of(c.body, c.n, c.chunksize, c.ring, c.env)


def expected_kernel(plan, R, flags, out_ptr):
    """The kernel that places a wave's results (engine.cu pick_gather): "direct" (the dispatch kernel stores at the final
    index, no gather), or the gather kernel "bulk", "rows" or "flat".  out_ptr: the caller's device output (FBR_OUT_DEVICE)
    or 0."""
    unit, slot = plan.unit_tasks, plan.slot_stride
    resilient = bool(flags & _abi.FBR_RESILIENT)
    out_dev = bool(flags & _abi.FBR_OUT_DEVICE)
    unit_ok = (unit * R) % 16 == 0 or unit == 1
    base_ok = not out_dev or out_ptr % 16 == 0
    if not resilient and not flags & (_abi.FBR_SHUFFLE | _abi.FBR_VIA_RING) and unit_ok and base_ok:
        return "direct"
    # the gather writes into the caller's device output (FBR_OUT_DEVICE) or into a buffer of the engine (16 B aligned)
    aligned = (out_ptr if out_dev else 0) % 16 == 0 and unit * R == slot
    rows_ok = aligned and slot % 4096 == 0
    bulk_ok = rows_ok and not resilient and slot % CHUNK == 0
    return "bulk" if bulk_ok else "rows" if rows_ok else "flat"


def expected_dispatch(body, arg_stride):
    """The dispatch kernel of a payload body (engine.cu launch_payload_map / launch_payload_checksum): "tma"
    (dispatch_payload_map_tma_kernel), "regs" (dispatch_payload_map_kernel) or "checksum"."""
    if body == "payload_checksum_4k":
        return "checksum"
    return "tma" if arg_stride == 4096 else "regs"


def kernel_of(c):
    return expected_kernel(case_plan(c), c.result_bytes, c.flags, c.out_offset)


def kinds_of(c, plan):
    """The task-count kinds of a case (module docstring)."""
    unit, k = plan.unit_tasks, set()
    if c.n == 1:
        k.add("one")
    if unit > 1 and c.n % unit == unit - 1:
        k.add("minus_one")
    if c.n % unit == 0:
        k.add("exact")
    if c.n > 1 and c.n % unit == 1:
        k.add("plus_one")
    if c.waves:
        k.add("waves")
    return k


def _pow2(x):
    return x > 0 and x & (x - 1) == 0


ALL_KINDS = frozenset(("one", "minus_one", "exact", "plus_one", "waves"))


def _group_cell(g):
    return (lambda c, p, k: k == "bulk" and c.env.get("FBR_BULK_GROUP") == str(g) and (g == 1 or p.n_units % g != 0), ALL_KINDS)


# cell -> (predicate(case, plan, kernel), task-count kinds the cell must be run at)
CELLS = {
    "flat/stride_not_4k": (lambda c, p, k: k == "flat" and p.slot_stride % 4096 != 0, ALL_KINDS),
    "flat/vps_npot": (lambda c, p, k: k == "flat" and not _pow2(p.slot_stride // 16), ALL_KINDS),
    "flat/out_plus4": (lambda c, p, k: k == "flat" and c.place == "out4", ALL_KINDS),
    "rows/rps1": (lambda c, p, k: k == "rows" and p.slot_stride == 4096, ALL_KINDS),
    "rows/rps_npot": (lambda c, p, k: k == "rows" and not _pow2(p.slot_stride >> 12), ALL_KINDS),
    "rows/big_slot": (lambda c, p, k: k == "rows" and p.slot_stride >= 32768, ALL_KINDS),
    "rows/resilient_lost": (lambda c, p, k: k == "rows" and c.place == "resilient" and p.slot_stride % CHUNK == 0
                            and c.body.startswith("flt_"), ALL_KINDS),
    # several slots per ticket group (one CTA per SM, one wave): row / rps runs in the 4-rows-in-flight loop across slots
    "rows/grouped_npot": (lambda c, p, k: k == "rows" and not _pow2(p.slot_stride >> 12) and c.env.get("FBR_GATHER_OCC") == "1"
                          and c.env.get("FBR_WAVES") == "1" and min((128 << 10) // p.slot_stride, p.n_units // (4 * SM_COUNT)) >= 2,
                          frozenset(("minus_one", "exact", "plus_one"))),
    "bulk/16k": (lambda c, p, k: k == "bulk" and p.slot_stride == CHUNK, ALL_KINDS),
    "bulk/multi_chunk": (lambda c, p, k: k == "bulk" and p.slot_stride > CHUNK, ALL_KINDS),
    # a tail unit of count * R bytes, not a multiple of 16: no stable unit of a bulk slot has R % 16 != 0 at n = 1, and
    # a map of whole units has no tail
    "bulk/tail_bytes": (lambda c, p, k: k == "bulk" and (c.n % p.unit_tasks) * c.result_bytes % 16 != 0,
                        frozenset(("minus_one", "plus_one", "waves"))),
    "bulk/group_1": _group_cell(1),
    "bulk/group_3": _group_cell(3),
    "bulk/group_32": _group_cell(32),
    "bulk/occ1": (lambda c, p, k: k == "bulk" and c.env.get("FBR_GATHER_OCC") == "1", ALL_KINDS),
    "payload/tma": (lambda c, p, k: c.body == "payload_map_4k" and expected_dispatch(c.body, c.arg_stride) == "tma", ALL_KINDS),
    "payload/strided_map": (lambda c, p, k: c.body == "payload_map_4k" and c.arg_stride in (4112, 8192, 12288)
                            and expected_dispatch(c.body, c.arg_stride) == "regs", ALL_KINDS),
    "payload/strided_checksum": (lambda c, p, k: c.body == "payload_checksum_4k" and c.arg_stride in (4112, 8192, 12288)
                                 and c.want_sum, ALL_KINDS),
    "grid/occ1_record": (lambda c, p, k: c.env.get("FBR_DISPATCH_OCC") == "1" and c.body in LB.BY_NAME, ALL_KINDS),
    "grid/occ1_payload_tma": (lambda c, p, k: c.env.get("FBR_DISPATCH_OCC") == "1"
                              and expected_dispatch(c.body, c.arg_stride) == "tma", ALL_KINDS),
    # pi_inside_bits8 runs through Pool.map (8 indices per byte-task), so its kinds are not named by unit; its results
    # go straight into the pinned output (zero copy), which makes every such map one wave
    "grid/occ1_pi_bits": (lambda c, p, k: c.env.get("FBR_DISPATCH_OCC") == "1" and c.body == "pi_inside_bits8",
                          frozenset(("one",))),
    "waves/many_small": (lambda c, p, k: c.env.get("FBR_WAVES") == "64" and c.env.get("FBR_MIN_WAVE_KB") == "4", ALL_KINDS),
}


def _bytes_per_task(body, place, args, stride):
    s = registry.spec(body)
    a = 0 if args in ("range", "dev") or place == "resilient" else (stride or s.arg_bytes)
    return max(s.result_bytes, a)


def _cases(cell, body, chunksize=0, ring=0, env=None, place="ring", args="host", stride=0, want_sum=False, ns=None, wave_ring=None,
           waves_at=()):
    """Cases of one configuration: n = 1, unit - 1, unit, unit + 1 of the configuration's plan at a large map, and a map of
    at least four waves of ``wave_ring`` (the configuration's ring when it is small, else SMALL_RING).  ns: explicit
    task counts instead (for bodies whose unit shrinks on small maps); waves_at: task counts that take at least four waves
    of ``ring`` under the configuration's own knobs."""
    env = dict(env or {})
    out = []
    if ns is None:
        unit = plan_of(body, 10 ** 7, chunksize, ring, env).unit_tasks
        ns = sorted({1, unit - 1, unit, unit + 1} - {0})
    for n in ns:
        out.append(Case(cell, body, n, chunksize, ring, env, place, args, stride, want_sum, False))
    for n in waves_at:
        out.append(Case(cell, body, n, chunksize, ring, env, place, args, stride, want_sum, True))
    if wave_ring is None:
        wave_ring = ring if ring and ring <= SMALL_RING else SMALL_RING
    if wave_ring:
        n = 5 * wave_ring // _bytes_per_task(body, place, args, stride) + 3
        out.append(Case(cell, body, n, chunksize, wave_ring, env, place, args, stride, want_sum, True))
    return out


def _build():
    C = []
    # ---- flat: gather_ordered_kernel
    C += _cases("flat/stride_not_4k", "lay_a2052_r2052")                          # 8 x 2052 B = 16416 B slots
    C += _cases("flat/stride_not_4k", "payload_checksum_4k", place="shuffle")     # 256 x 4 B = 1 KB slots
    C += _cases("flat/vps_npot", "lay_a2052_r2052", place="shuffle")              # 1026 vectors per slot
    C += _cases("flat/vps_npot", "payload_checksum_4k", chunksize=3)              # 252 tasks: 63 vectors
    C += _cases("flat/out_plus4", "payload_map_4k", place="out4")
    C += _cases("flat/out_plus4", "payload_checksum_4k", place="out4", ns=[5, 1000])
    # ---- rows: gather_rows_kernel
    u256 = {"FBR_UNIT_TASKS": "256"}
    C += _cases("rows/rps1", "bc_e4_s0", env=u256)                                # 256 x 16 B: one row per slot
    big = 200 * 4096
    C += _cases("rows/rps1", "pi_inside_det", args="range", ns=[big - 1, big, big + 1])
    C += _cases("rows/rps1", "pi_inside_det", args="range", place="shuffle", ns=[big + 1])
    C += _cases("rows/rps_npot", "payload_map_4k", chunksize=3, ring=32 << 10)    # 3 tasks: 3 rows
    C += _cases("rows/rps_npot", "payload_map_4k", chunksize=3, ring=32 << 10, place="shuffle")
    C += _cases("rows/rps_npot", "lay_a8_r24", place="shuffle", ns=[200 * 1024 - 1, 200 * 1024 + 1], wave_ring=0)   # 6 rows
    C += _cases("rows/rps_npot", "lay_i8_r12", args="range", ns=[200 * 1024 + 1, 200 * 1024 + 5, 200 * 1024 - 1],
                wave_ring=0)                                                      # 12 KB slots, 12-byte records
    C += _cases("rows/rps_npot", "payload_map_4k", chunksize=9, place="shuffle")  # 27 tasks: 27 rows of 108 KB slots
    C += _cases("rows/rps_npot", "payload_map_4k", chunksize=9)
    C += _cases("rows/big_slot", "payload_map_4k", chunksize=3, place="shuffle")  # 30 tasks: 30 rows of 120 KB slots
    C += _cases("rows/big_slot", "payload_map_4k", chunksize=17)                  # 17 rows
    C += _cases("rows/big_slot", "lay_a12_r4096", place="resilient")              # 32 KB slots
    C += _cases("rows/resilient_lost", "flt_a4_r4096", place="resilient")         # 32 KB slots, ~5 % of the tasks lost twice
    grouped = {"FBR_GATHER_OCC": "1", "FBR_WAVES": "1"}
    C += _cases("rows/grouped_npot", "lay_a8_r24", env=grouped, ns=[1600 * 1024 - 1, 1600 * 1024, 1600 * 1024 + 1],
                wave_ring=0)                                                      # 24 KB slots
    C += _cases("rows/grouped_npot", "pi_inside_det", args="range", env=dict(grouped, FBR_UNIT_TASKS="12288"),
                ns=[2200 * 12288 + 1], wave_ring=0)                                                       # 12 KB slots
    # ---- bulk: gather_bulk_kernel
    C += _cases("bulk/16k", "payload_map_4k", ring=32 << 10)                      # 4 tasks of 4 KB
    C += _cases("bulk/16k", "lay_a4_r4096", ring=32 << 10, place="shuffle")
    C += _cases("bulk/multi_chunk", "payload_map_4k", place="shuffle")            # 128 KB: 8 chunks
    C += _cases("bulk/multi_chunk", "lay_a4_r4096")                               # 32 KB: 2 chunks
    u16k = {"FBR_UNIT_TASKS": "16384"}
    pi_u = 140 * 16384
    C += _cases("bulk/tail_bytes", "pi_inside_det", args="range", env=u16k, ns=[pi_u - 1, pi_u + 1, pi_u + 9])
    many = [1, 7, 8, 9, 8 * 96 + 1, 8 * 100 + 3, 8 * 101 + 2]                  # 1 .. 102 units of 8 tasks
    for g in (1, 3, 32):
        C += _cases("bulk/group_%d" % g, "lay_a4_r4096", env={"FBR_BULK_GROUP": str(g)}, ns=[n for n in many if g == 1 or -(-n // 8) % g])
    C += _cases("bulk/occ1", "lay_a4_r4096", env={"FBR_GATHER_OCC": "1"}, ns=many)
    C += _cases("bulk/occ1", "payload_map_4k", env={"FBR_GATHER_OCC": "1"}, place="shuffle")
    # ---- payload dispatch kernels
    C += _cases("payload/tma", "payload_map_4k", place="direct")
    C += _cases("payload/tma", "payload_map_4k", args="dev", place="shuffle", wave_ring=0)
    for i, stride in enumerate((4112, 8192, 12288)):
        for j, (args, place) in enumerate((a, p) for a in ("host", "dev") for p in ("direct", "ring", "shuffle")):
            n = (1, 31, 32, 33, 77, 5)[(i + j) % 6]
            C += _cases("payload/strided_map", "payload_map_4k", args=args, place=place, stride=stride, ns=[n], wave_ring=0)
            C += _cases("payload/strided_checksum", "payload_checksum_4k", args=args, place=place, stride=stride, want_sum=True,
                        ns=[(1, 255, 256, 257, 1000, 5)[(i + j) % 6]], wave_ring=0)
        C += _cases("payload/strided_map", "payload_map_4k", place=("direct", "ring", "shuffle")[i], stride=stride, ns=[],
                    wave_ring=4 << 20)
        C += _cases("payload/strided_checksum", "payload_checksum_4k", place=("direct", "ring", "shuffle")[i], stride=stride,
                    want_sum=True, ns=[], wave_ring=4 << 20)
    # ---- dispatch grids of one CTA per SM (each CTA claims many tickets)
    occ1 = {"FBR_DISPATCH_OCC": "1"}
    C += _cases("grid/occ1_record", "lay_a20_r36_g16", env=occ1, place="direct", ns=[1, 511, 512, 513, 200 * 512 + 1])
    C += _cases("grid/occ1_payload_tma", "payload_map_4k", env=occ1, place="direct")
    C += [Case("grid/occ1_pi_bits", "pi_inside_bits8", n, 0, 0, occ1, "direct", "range", 0, False, False)
          for n in (1, 4097, 3_000_001, 9_000_003)]
    # ---- many small waves
    tiny = {"FBR_WAVES": "64", "FBR_MIN_WAVE_KB": "4"}
    C += _cases("waves/many_small", "payload_map_4k", env=tiny, place="direct", ns=[1, 31, 32, 33], wave_ring=0,
                waves_at=[20 * 32 + 1])
    C += _cases("waves/many_small", "lay_a20_r20", env=tiny, place="ring", ns=[1, 200 * 1024 - 1, 200 * 1024],
                wave_ring=0, waves_at=[200 * 1024 + 1])
    return C


CASES = _build()
BY_ID = {c.id: c for c in CASES}


# ---- running a case on the GPU ---------------------------------------------------------------------------------------
def _payload_args(n, stride, seed):
    """cref's payload records, each at the start of a stride-byte row whose padding is noise (a load at the wrong stride
    reads noise)."""
    import numpy as np
    from oracle import cref
    recs = cref.payload_records(seed, n)
    if stride in (0, 4096):
        return recs, recs
    wide = np.random.default_rng(seed).integers(0, 2 ** 32, (n, stride // 4), dtype=np.uint32)
    wide[:, :1024] = recs
    return recs, wide


def _want(c, args, block):
    """(result bytes, sum or None) of a case, from the plain restatement: NumPy for the layout bodies, the C oracle
    for pi and the payload bodies."""
    import numpy as np
    from oracle import cref
    if c.body in LB.BY_NAME:
        b = LB.BY_NAME[c.body]
        return LB.results_np(b, c.n, 0, args, block).view(np.uint8).reshape(-1), None
    if c.body == "pi_inside_det":
        ref, count = cref.pi_inside_range(0, c.n)
        return ref, count
    if c.body == "payload_map_4k":
        return cref.payload_map(0, args).view(np.uint8).reshape(-1), None
    ck = cref.payload_checksum(args)
    return ck.view(np.uint8), int(ck.astype(np.int64).sum())


def run_case(pool, c):
    """Run case c on pool (a one-worker fiber_b200.Pool of ring_bytes c.ring) under its knobs.  Returns a list of
    mismatch messages (empty: every result byte and the sum agree with the restatement), the result's wave count and
    the pool's stats delta."""
    import numpy as np
    from oracle import cref
    eng, lib = pool._engine, pool._engine.lib
    before = pool.stats()
    bad = []
    if c.body == "pi_inside_bits8":                  # bit-packed pi through the public API (8 indices per byte-task)
        ref, count = cref.pi_inside_range(0, c.n)
        with knobs(c.env):
            res = pool.map(_is_inside(), range(c.n))
        if not np.array_equal(res.packed, np.packbits(ref, bitorder="little")) or res.sum() != count:
            bad.append("bit-packed results differ from the oracle")
        return bad, None, _delta(before, pool.stats())
    spec = registry.spec(c.body)
    R = spec.result_bytes
    bufs = []

    def dev_alloc(nbytes):
        p = ctypes.c_void_p()
        _abi.check(lib.fbr_device_alloc(eng.handle, 0, nbytes + 64, ctypes.byref(p)))
        bufs.append(p)
        return p.value

    try:
        d = _abi.MapDesc()
        d.func_id, d.flags, d.n_tasks, d.chunksize, d.shuffle_seed = spec.func_id, c.flags, c.n, c.chunksize, 0x5EED + c.n
        args = block = host = None
        if c.args == "range":
            d.index_start, d.index_step = 0, 1
            args = np.arange(c.n, dtype=np.int64)
        else:
            if c.body in PAYLOAD:
                args, host = _payload_args(c.n, c.arg_stride, c.n % 1000)
            else:
                args = host = LB.make_args(LB.BY_NAME[c.body], c.n, c.n)
            host = np.ascontiguousarray(host)
            d.arg_stride = c.arg_stride
            if c.args == "dev":
                d.args = dev_alloc(host.nbytes)
                _abi.check(lib.fbr_memcpy_h2d(eng.handle, 0, ctypes.c_void_p(d.args), host.ctypes.data, host.nbytes))
            else:
                d.args = host.ctypes.data
        b = LB.BY_NAME.get(c.body)
        if b is not None and b.shared:
            block = LB.make_block(b, 5, c.n)
            d.shared, d.shared_bytes = block.ctypes.data, block.nbytes
        out = None
        if c.flags & _abi.FBR_OUT_DEVICE:
            out = dev_alloc(c.n * R) + c.out_offset
            d.out = out
        seq = ctypes.c_uint64()
        res = _abi.Result()
        with knobs(c.env):
            _abi.check(lib.fbr_map_submit(eng.handle, ctypes.byref(d), ctypes.byref(seq)))
            try:
                _abi.check(lib.fbr_result_wait(eng.handle, seq.value, -1, ctypes.byref(res)))
            finally:
                data = np.zeros(c.n * R, np.uint8)
                if out is not None:
                    _abi.check(lib.fbr_memcpy_d2h(eng.handle, 0, data.ctypes.data, ctypes.c_void_p(out), data.nbytes))
                elif res.data:
                    ctypes.memmove(data.ctypes.data, res.data, data.nbytes)
                _abi.check(lib.fbr_result_release(eng.handle, seq.value))
        want, total = _want(c, args, block)
        if not np.array_equal(data, want):
            rows = np.nonzero((data.reshape(c.n, R) != want.reshape(c.n, R)).any(axis=1))[0]
            bad.append("%d of %d tasks differ, first %s" % (len(rows), c.n, rows[:8].tolist()))
        if c.want_sum and int(res.sum) != total:
            bad.append("sum %d != %d" % (res.sum, total))
        return bad, int(res.n_waves), _delta(before, pool.stats())
    finally:
        for p in bufs:
            lib.fbr_device_free(eng.handle, 0, p)


def _is_inside():
    from examples import workloads as W
    return W.is_inside


def _delta(a, b):
    return {k: b[k] - a[k] for k in b if isinstance(b[k], int)}


def check_stats(c, kernel, waves, st):
    """Messages for stats that contradict the path a case was meant to take: direct placement or a gather launch per
    wave, at least one dispatch launch per wave, and no task records copied for a map that is neither shuffled nor
    resilient."""
    bad = []
    if c.place not in ("shuffle", "resilient") and st["records_copied"] != 0:
        bad.append("records_copied %d on a map that is not shuffled" % st["records_copied"])
    if waves is not None and st["dispatch_launches"] < waves:
        bad.append("dispatch_launches %d < %d waves" % (st["dispatch_launches"], waves))
    if kernel == "direct" and not (st["direct_waves"] >= 1 and st["gather_launches"] == 0):
        bad.append("direct case: direct_waves %d gather_launches %d" % (st["direct_waves"], st["gather_launches"]))
    if kernel in ("flat", "rows", "bulk") and not (st["gather_launches"] >= 1 and st["direct_waves"] == 0):
        bad.append("gathered case: direct_waves %d gather_launches %d" % (st["direct_waves"], st["gather_launches"]))
    if c.waves and (st["dispatch_launches"] if waves is None else waves) < 4:
        bad.append("%s waves (%d dispatch launches), want >= 4" % (waves, st["dispatch_launches"]))
    return bad
