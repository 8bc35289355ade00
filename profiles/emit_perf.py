"""Emit record bodies (a variable-length result per task): count pass, scan and emit pass, against the hash-only floor, a
device-to-device copy and the padded fixed-capacity workaround.

    python profiles/emit_perf.py [--out profiles/r08_emit_perf.json] [--reps 10] [--rounds 3]

1. tokens_u32 over the fnv1a_bytes input of ragged_perf.py (8 Mi byte strings of seeded lengths 0 .. 512, mean 256 B):
   the 32-bit FNV-1a of every whitespace-separated token.  Beside it, fnv1a_bytes over the same strings (one 64-bit
   hash per string, a fixed 16 B result: one pass over the strings).
2. above_mask_f64 over the ragged_stats_f64 rows of ragged_perf.py (2 Mi float64 rows, lognormal lengths): the positions
   above 0.0, on a warp.
3. Against padding: tokens_u32 against a fixed-capacity record body (tokens_pad_u32: a count and at most 63 hashes, 256 B
   per task) plus the compaction of its padded records into values and offsets, on 1 Mi strings.
4. One host-resident Pool.map of tokens_u32 end to end (wall clock, 1 Mi strings from host memory, values in host memory).

Maps 1-3 are device-resident (FBR_ARGS_DEVICE, FBR_RESULTS_ON_DEVICE) with direct placement.  Each time is the median of
--reps maps after a warm-up, and the workloads are timed in turn for --rounds rounds.  Map time is the host clock around
submission (which runs the count pass and the scan and waits for them) and the wait; the kernels of one more map are split
into count, scan and emit with torch.profiler.  Beside each workload, a device-to-device copy of its algorithmic bytes.
The card's name and power limit are read in the same call.  Every map's values are checked against the Python
restatement on its first 4096 tasks.
"""
import argparse
import ctypes
import json
import os
import re
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import fiber_b200  # noqa: E402
from fiber_b200 import _abi, registry  # noqa: E402
from profiles.record_perf import card, time_copy  # noqa: E402
from tests import emit_bodies as EB  # noqa: E402
from tests import ragged_bodies as RB  # noqa: E402

PAD_CAP = 63
PAD_RES = np.dtype([("n", "<u4"), ("h", "<u4", (PAD_CAP,))])
PAD_SRC = EB.TOKENS_SRC.split("// the same, but")[0] + r'''
// tokens_u32 into a fixed-capacity record: the count, then at most 63 hashes (later tokens are dropped)
struct TokensPad {
    using Item = uint8_t;
    using Arg = fbr::NoArg;
    struct Res { uint32_t n; uint32_t h[63]; };
    static constexpr bool kIndexArg = false, kCanFault = false;
    struct Sink { Res& r; uint32_t n; __device__ void push(uint32_t v) { if (n < 63) r.h[n] = v; ++n; } };
    __device__ static __forceinline__ void run(const fbr::Items<Item>& x, Res& r, uint64_t, const fbr::ErrSink&, uint32_t) {
        Sink s{r, 0};
        uint32_t h = 0x811c9dc5u;
        bool in = false;
        for (uint64_t k = 0; k < x.n; ++k) {
            const uint8_t c = x.data[k];
            if (ascii_space(c)) { if (in) s.push(h); in = false; h = 0x811c9dc5u; }
            else { h = (h ^ c) * 0x01000193u; in = true; }
        }
        if (in) s.push(h);
        r.n = s.n < 63 ? s.n : 63;
    }
};
FBR_EXPORT_RECORD_BODY(TokensPad, "tokens_pad_u32", tokens_pad_entry, 0)
'''


@fiber_b200.device_body("tokens_pad_u32", source=PAD_SRC, entry="tokens_pad_entry", args=None, items=("doc", "u1"),
                        result=PAD_RES)
def tokens_pad_u32(doc):
    return EB.tokens_u32(doc)[:PAD_CAP]


def submit(pool, name, n, flags, values=None, offsets=None, args=None, arg_stride=0):
    spec = registry.spec(name)
    eng = pool._engine
    d = _abi.MapDesc()
    d.func_id, d.flags, d.n_tasks = spec.func_id, flags, n
    if args is not None:
        d.args, d.arg_stride = args.data_ptr(), arg_stride
    it = _abi.ItemsDesc()
    it.items, it.offsets, it.n_items, it.item_bytes = values.data_ptr(), offsets.data_ptr(), values.numel(), values.element_size()
    seq = ctypes.c_uint64()
    _abi.check(eng.lib.fbr_map_submit_items(eng.handle, ctypes.byref(d), ctypes.byref(it), ctypes.byref(seq)))
    res = _abi.Result()
    _abi.check(eng.lib.fbr_result_wait(eng.handle, seq.value, -1, ctypes.byref(res)))
    return seq.value


def fetch_head(pool, seq, n_head, out_dtype):
    """End offsets and values of the first n_head tasks of a device-resident emit map."""
    eng = pool._engine
    ends = np.zeros(n_head, np.uint64)
    _abi.check(eng.lib.fbr_result_fetch(eng.handle, seq, 0, n_head, ends.ctypes.data))
    vals = np.zeros(int(ends[-1]), out_dtype)
    if len(vals):
        _abi.check(eng.lib.fbr_result_fetch_values(eng.handle, seq, 0, len(vals), vals.ctypes.data))
    o = np.concatenate([[0], ends.astype(np.int64)])
    return [vals[o[i]:o[i + 1]].tolist() for i in range(n_head)]


def time_map(pool, run, reps):
    """Median host time of run() (a map submitted and waited for, then released)."""
    eng = pool._engine
    for _ in range(2):
        eng.lib.fbr_result_release(eng.handle, run())
    ms = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        seq = run()
        ms.append((time.perf_counter() - t0) * 1e3)
        eng.lib.fbr_result_release(eng.handle, seq)
    return statistics.median(ms), ms


def split_kernels(pool, run):
    """Device time of one map's kernels by pass: count (EmitPass<.., false>), scan, emit (EmitPass<.., true>), other."""
    eng = pool._engine
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        seq = run()
        torch.cuda.synchronize()
    eng.lib.fbr_result_release(eng.handle, seq)
    out = {"count_ms": 0.0, "scan_ms": 0.0, "emit_ms": 0.0, "other_ms": 0.0}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        ms = ev.device_time_total / 1e3 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1e3
        m = re.search(r"EmitPass<[^<>]*, *(true|false|\(bool\)[01])>", ev.name)
        key = ("scan_ms" if "scan_counts_kernel" in ev.name else "other_ms" if m is None else
               "emit_ms" if m.group(1) in ("true", "(bool)1") else "count_ms")
        out[key] += ms
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "emit_perf.json"))
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("emit_perf.py measures on a GPU; none is visible")
    pool = fiber_b200.Pool(1, devices=[0])
    pool.start_workers()
    dev = _abi.FBR_ARGS_DEVICE | _abi.FBR_RESULTS_ON_DEVICE
    head = 4096

    sv, so = RB.byte_strings(8 << 20, seed=22)
    rv, ro = RB.lognormal_rows(2_000_000, seed=21)
    n_s, n_r, n_p = len(so) - 1, len(ro) - 1, 1 << 20
    d_sv, d_so = torch.from_numpy(sv).cuda(), torch.from_numpy(so.astype(np.int64)).cuda()
    d_rv, d_ro = torch.from_numpy(rv).cuda(), torch.from_numpy(ro.astype(np.int64)).cuda()
    d_t = torch.zeros(n_r, dtype=torch.float64, device="cuda")
    d_pso = d_so[: n_p + 1].contiguous()
    pad_out = torch.empty(n_p * PAD_RES.itemsize, dtype=torch.uint8, device="cuda")

    def fnv():
        spec = registry.spec("fnv1a_bytes")
        d = _abi.MapDesc()
        d.func_id, d.flags, d.n_tasks = spec.func_id, _abi.FBR_ARGS_DEVICE | _abi.FBR_OUT_DEVICE, n_s
        d.out = fnv_out.data_ptr()
        it = _abi.ItemsDesc()
        it.items, it.offsets, it.n_items, it.item_bytes = d_sv.data_ptr(), d_so.data_ptr(), d_sv.numel(), 1
        seq = ctypes.c_uint64()
        _abi.check(pool._engine.lib.fbr_map_submit_items(pool._engine.handle, ctypes.byref(d), ctypes.byref(it), ctypes.byref(seq)))
        res = _abi.Result()
        _abi.check(pool._engine.lib.fbr_result_wait(pool._engine.handle, seq.value, -1, ctypes.byref(res)))
        return seq.value
    fnv_out = torch.empty(n_s * 16, dtype=torch.uint8, device="cuda")

    def padded():
        spec = registry.spec("tokens_pad_u32")
        d = _abi.MapDesc()
        d.func_id, d.flags, d.n_tasks = spec.func_id, _abi.FBR_ARGS_DEVICE | _abi.FBR_OUT_DEVICE, n_p
        d.out = pad_out.data_ptr()
        it = _abi.ItemsDesc()
        it.items, it.offsets, it.n_items, it.item_bytes = d_sv.data_ptr(), d_pso.data_ptr(), d_sv.numel(), 1
        seq = ctypes.c_uint64()
        _abi.check(pool._engine.lib.fbr_map_submit_items(pool._engine.handle, ctypes.byref(d), ctypes.byref(it), ctypes.byref(seq)))
        res = _abi.Result()
        _abi.check(pool._engine.lib.fbr_result_wait(pool._engine.handle, seq.value, -1, ctypes.byref(res)))
        # compaction: the counts' prefix sum and the kept hashes, as the caller of a fixed-capacity body has to do
        rec = pad_out.view(torch.int32).view(n_p, 1 + PAD_CAP)
        cnt = rec[:, 0].to(torch.int64)
        offs = torch.zeros(n_p + 1, dtype=torch.int64, device="cuda")
        torch.cumsum(cnt, 0, out=offs[1:])
        keep = torch.arange(PAD_CAP, device="cuda")[None, :] < cnt[:, None]
        vals = rec[:, 1:][keep]
        torch.cuda.synchronize()
        del offs, vals
        return seq.value

    work = {
        "tokens_u32": lambda: submit(pool, "tokens_u32", n_s, dev, d_sv, d_so),
        "fnv1a_bytes (floor)": fnv,
        "above_mask_f64": lambda: submit(pool, "above_mask_f64", n_r, dev, d_rv, d_ro, d_t, 8),
        "tokens_u32 (1 Mi strings)": lambda: submit(pool, "tokens_u32", n_p, dev, d_sv, d_pso),
        "tokens_pad_u32 + compaction (1 Mi strings)": padded,
    }
    rounds = {k: [] for k in work}
    for _ in range(args.rounds):
        for k, run in work.items():
            rounds[k].append(time_map(pool, run, args.reps)[0])

    # values and offsets of each emit map, checked on the first tasks
    checks = {}
    seq = work["tokens_u32"]()
    checks["tokens_u32"] = fetch_head(pool, seq, head, np.uint32) == [EB.tokens_u32(bytes(sv[so[i]:so[i + 1]])) for i in range(head)]
    ends = np.zeros(1, np.uint64)
    _abi.check(pool._engine.lib.fbr_result_fetch(pool._engine.handle, seq, n_s - 1, 1, ends.ctypes.data))
    total_tokens = int(ends[0])
    pool._engine.lib.fbr_result_release(pool._engine.handle, seq)
    seq = work["above_mask_f64"]()
    checks["above_mask_f64"] = fetch_head(pool, seq, head, np.uint32) == [np.flatnonzero(rv[ro[i]:ro[i + 1]] > 0.0).tolist() for i in range(head)]
    _abi.check(pool._engine.lib.fbr_result_fetch(pool._engine.handle, seq, n_r - 1, 1, ends.ctypes.data))
    total_above = int(ends[0])
    pool._engine.lib.fbr_result_release(pool._engine.handle, seq)

    splits = {k: split_kernels(pool, work[k]) for k in ("tokens_u32", "above_mask_f64")}

    def entry(k, algo):
        t = statistics.median(rounds[k])
        copy_ms, _ = time_copy(algo // 2, args.reps)
        return {"map_ms_median": t, "round_medians_ms": rounds[k], "round_spread": (max(rounds[k]) - min(rounds[k])) / t,
                "algorithmic_bytes": algo, "copy_ms_median": copy_ms, "of_copy": copy_ms / t}

    # algorithmic bytes: the items and offsets read (twice for an emit map: both passes), the counts and offsets written
    # and read back (8 B each per pass), the end offsets and the values written
    res = {
        "tokens_u32": dict(entry("tokens_u32", 2 * (sv.nbytes + so.nbytes) + 3 * 8 * n_s + 4 * total_tokens),
                           n_tasks=n_s, n_values=total_tokens, kernels_ms=splits["tokens_u32"], values_match=checks["tokens_u32"]),
        "fnv1a_bytes (floor)": dict(entry("fnv1a_bytes (floor)", sv.nbytes + so.nbytes + 16 * n_s), n_tasks=n_s),
        "above_mask_f64": dict(entry("above_mask_f64", 2 * (rv.nbytes + ro.nbytes + 8 * n_r) + 3 * 8 * n_r + 4 * total_above),
                               n_tasks=n_r, n_values=total_above, kernels_ms=splits["above_mask_f64"],
                               values_match=checks["above_mask_f64"]),
    }
    against = {"n_tasks": n_p, "capacity": PAD_CAP, "padded_record_bytes": PAD_RES.itemsize,
               "emit_ms_median": statistics.median(rounds["tokens_u32 (1 Mi strings)"]),
               "padded_plus_compaction_ms_median": statistics.median(rounds["tokens_pad_u32 + compaction (1 Mi strings)"]),
               "round_medians_ms": {k: rounds[k] for k in ("tokens_u32 (1 Mi strings)", "tokens_pad_u32 + compaction (1 Mi strings)")}}
    against["speedup"] = against["padded_plus_compaction_ms_median"] / against["emit_ms_median"]

    # one host-resident Pool.map end to end
    docs = fiber_b200.Ragged(sv[: int(so[n_p])], so[: n_p + 1])
    e2e = []
    for _ in range(args.rounds):
        t0 = time.perf_counter()
        r = pool.map(EB.tokens_u32, docs)
        e2e.append((time.perf_counter() - t0) * 1e3)
    host = {"n_tasks": n_p, "wall_ms": e2e, "wall_ms_median": statistics.median(e2e), "n_values": len(r.ragged.values),
            "values_match": r[:head] == [EB.tokens_u32(bytes(sv[so[i]:so[i + 1]])) for i in range(head)]}
    pool.terminate()
    pool.join()

    result = {"card": card(), "workloads": res, "against_padding": against, "host_pool_map": host}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(result, fh, indent=1)
    for k, v in res.items():
        print("%-22s %8.3f ms  copy %7.3f ms  spread %.1f %%  %s" % (k, v["map_ms_median"], v["copy_ms_median"],
              100 * v["round_spread"], v.get("kernels_ms", "")))
    print("padded + compaction %.3f ms  emit %.3f ms  (%.2fx)" % (against["padded_plus_compaction_ms_median"],
          against["emit_ms_median"], against["speedup"]))
    print("host Pool.map %.1f ms  values ok=%s  checks %s" % (host["wall_ms_median"], host["values_match"], checks))
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
