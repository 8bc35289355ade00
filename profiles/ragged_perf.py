"""Kernel rate of items record bodies (variable-length items per task) against a device-to-device copy, and against the
padded fixed-size workaround.

    python profiles/ragged_perf.py [--out profiles/ragged_perf.json] [--reps 10] [--rounds 3]

1. Rate: ragged_stats_f64 over 2 Mi float64 rows with seeded lognormal lengths (log-mean ln 64, sigma 1: a mean of about
   105 items, about 1.7 GB of items), and fnv1a_bytes
   over about 8 Mi byte strings with seeded lengths 0 .. 512 (tests/ragged_bodies.py).  The algorithmic bytes are the
   items, the offsets and the results; beside each map, in the same call, a device-to-device copy of that many bytes.
   Each map is timed --rounds times, so the run-to-run spread is reported beside the rate.
2. Against the workaround: 128 Ki rows of the same distribution, clipped to 1023 items, padded to 1023 float64 plus
   their length (8 KB records), through the equivalent group record body padded_stats_f64.

Every map is device-resident (FBR_ARGS_DEVICE | FBR_OUT_DEVICE) with direct placement; its kernel time comes from the
engine's CUDA events (FBR_POOL_TIMING), the median of --reps maps after a warm-up.  The card's name and power limit are
read in the same call.  The first 4096 results of every map are checked against the NumPy restatement.
"""
import argparse
import ctypes
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import fiber_b200  # noqa: E402
from fiber_b200 import _abi, registry  # noqa: E402
from profiles.record_perf import HBM_DATASHEET_TBS, card, time_copy  # noqa: E402
from tests import ragged_bodies as RB  # noqa: E402


def _ptr(t):
    return t.data_ptr()


def time_items(pool, name, values, offsets, n, reps, ref_head):
    """Median kernel time of a device-resident items map; checks the first 4096 results against ref_head."""
    spec = registry.spec(name)
    eng = pool._engine
    out = torch.empty(n * spec.result_bytes, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def one():
        d = _abi.MapDesc()
        d.func_id, d.flags, d.n_tasks = spec.func_id, _abi.FBR_ARGS_DEVICE | _abi.FBR_OUT_DEVICE, n
        d.out = _ptr(out)
        it = _abi.ItemsDesc()
        it.items, it.offsets, it.n_items, it.item_bytes = _ptr(values), _ptr(offsets), values.numel(), values.element_size()
        before = pool.stats()
        seq = ctypes.c_uint64()
        _abi.check(eng.lib.fbr_map_submit_items(eng.handle, ctypes.byref(d), ctypes.byref(it), ctypes.byref(seq)))
        res = _abi.Result()
        _abi.check(eng.lib.fbr_result_wait(eng.handle, seq.value, -1, ctypes.byref(res)))
        _abi.check(eng.lib.fbr_result_release(eng.handle, seq.value))
        st = pool.stats()
        assert st["gather_launches"] == before["gather_launches"] and res.err_code == 0
        return st["dispatch_ms"] - before["dispatch_ms"]
    for _ in range(2):
        one()
    ms = [one() for _ in range(reps)]
    head = out[: 4096 * spec.result_bytes].cpu().numpy()
    ok = bool(np.array_equal(head, np.ascontiguousarray(ref_head).view(np.uint8)))
    return {"kernel_ms_median": statistics.median(ms), "kernel_ms": ms, "results_match_numpy_head": ok}


def time_records(pool, name, args, n, reps, ref_head):
    spec = registry.spec(name)
    eng = pool._engine
    out = torch.empty(n * spec.result_bytes, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def one():
        d = _abi.MapDesc()
        d.func_id, d.flags, d.n_tasks = spec.func_id, _abi.FBR_ARGS_DEVICE | _abi.FBR_OUT_DEVICE, n
        d.args, d.arg_stride, d.out = _ptr(args), spec.arg_bytes, _ptr(out)
        before = pool.stats()
        seq = ctypes.c_uint64()
        _abi.check(eng.lib.fbr_map_submit(eng.handle, ctypes.byref(d), ctypes.byref(seq)))
        res = _abi.Result()
        _abi.check(eng.lib.fbr_result_wait(eng.handle, seq.value, -1, ctypes.byref(res)))
        _abi.check(eng.lib.fbr_result_release(eng.handle, seq.value))
        return pool.stats()["dispatch_ms"] - before["dispatch_ms"]
    for _ in range(2):
        one()
    ms = [one() for _ in range(reps)]
    head = out[: 4096 * spec.result_bytes].cpu().numpy()
    ok = bool(np.array_equal(head, np.ascontiguousarray(ref_head).view(np.uint8)))
    return {"kernel_ms_median": statistics.median(ms), "kernel_ms": ms, "results_match_numpy_head": ok}


def rate(name, n, algo, t_ms, copy_ms):
    return {"body": name, "n_tasks": n, "algorithmic_bytes": algo, "kernel_ms_median": t_ms, "kernel_GBps": algo / t_ms / 1e6,
            "copy_ms_median": copy_ms, "copy_GBps": algo / copy_ms / 1e6, "of_copy": copy_ms / t_ms,
            "of_datasheet_hbm": algo / t_ms / 1e6 / (HBM_DATASHEET_TBS * 1e3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "ragged_perf.json"))
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("ragged_perf.py measures on a GPU; none is visible")
    pool = fiber_b200.Pool(1, devices=[0], timing=True)
    pool.start_workers()

    workloads = []
    # float64 rows: ~1.7 GB of items
    rv, ro = RB.lognormal_rows(2_000_000, seed=21)
    workloads.append(("ragged_stats_f64", rv, ro, RB.ragged_stats_np))
    # byte strings: 8 Mi strings of 0 .. 512 bytes
    sv, so = RB.byte_strings(8 << 20, seed=22)
    workloads.append(("fnv1a_bytes", sv, so, RB.fnv1a_np))

    rates = []
    for name, vals, offs, ref in workloads:
        n = len(offs) - 1
        dv = torch.from_numpy(vals).cuda()
        do = torch.from_numpy(offs.astype(np.int64)).cuda()
        want = ref(vals[: int(offs[4096])], offs[:4097])
        rounds = [time_items(pool, name, dv, do, n, args.reps, want) for _ in range(args.rounds)]
        algo = vals.nbytes + offs.nbytes + n * registry.spec(name).result_bytes
        del dv, do
        torch.cuda.empty_cache()
        copy_ms, copy_all = time_copy(algo // 2, args.reps)
        meds = [r["kernel_ms_median"] for r in rounds]
        t = statistics.median(meds)
        r = rate(name, n, algo, t, copy_ms)
        r.update({"round_medians_ms": meds, "round_spread": (max(meds) - min(meds)) / t, "copy_ms": copy_all,
                  "mean_items_per_task": float(len(vals) / n),
                  "results_match_numpy_head": all(x["results_match_numpy_head"] for x in rounds)})
        rates.append(r)

    # the padded workaround against the items body on the same rows
    n = 128 << 10
    pv, po = RB.lognormal_rows(n, seed=23, max_len=RB.PADDED_LEN)
    padded = np.zeros(n, RB.PADDED_ARG)
    lens = np.diff(po)
    for i in range(n):
        padded["x"][i, : lens[i]] = pv[po[i]: po[i + 1]]
    padded["n"] = lens
    want = RB.ragged_stats_np(pv[: int(po[4096])], po[:4097])
    da = torch.from_numpy(padded.view(np.uint8)).cuda()
    pad = time_records(pool, "padded_stats_f64", da, n, args.reps, want)
    del da
    dv, do = torch.from_numpy(pv).cuda(), torch.from_numpy(po.astype(np.int64)).cuda()
    rag = time_items(pool, "ragged_stats_f64", dv, do, n, args.reps, want)
    del dv, do
    workaround = {"n_tasks": n, "mean_len": float(lens.mean()), "padded_len": RB.PADDED_LEN,
                  "padded_bytes": padded.nbytes, "items_bytes": pv.nbytes + po.nbytes,
                  "padded_stats_f64": pad, "ragged_stats_f64": rag,
                  "speedup": pad["kernel_ms_median"] / rag["kernel_ms_median"]}
    pool.terminate()
    pool.join()

    result = {"card": card(), "hbm_datasheet_TBps": HBM_DATASHEET_TBS, "rates": rates, "against_padding": workaround}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(result, fh, indent=1)
    for r in rates:
        print("%-24s n=%-8d %7.3f ms  %7.1f GB/s  copy %7.1f GB/s  (%.0f %% of copy)  spread %.1f %%  head ok=%s"
              % (r["body"], r["n_tasks"], r["kernel_ms_median"], r["kernel_GBps"], r["copy_GBps"], 100 * r["of_copy"],
                 100 * r["round_spread"], r["results_match_numpy_head"]))
    print("padded %.3f ms  ragged %.3f ms  (%.2fx)  head ok=%s/%s" % (pad["kernel_ms_median"], rag["kernel_ms_median"],
          workaround["speedup"], pad["results_match_numpy_head"], rag["results_match_numpy_head"]))
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
