"""Kernel rate of dispatch_record_kernel with a broadcast block: nearest_centroid_f32 over 16 Mi points.

    python profiles/broadcast_perf.py [--out profiles/r05_broadcast_perf.json] [--reps 10]

Device-resident maps (FBR_ARGS_DEVICE | FBR_OUT_DEVICE, one wave, direct placement) of nearest_centroid_f32 from
tests/broadcast_bodies.py: 16 Mi float32 points of 16 dimensions against K = 64, 256, 512 centroids (the block fits
the body's 32 KB budget and is staged in shared memory) and K = 513, 2048 (read from global memory).  At K = 256 the
same body built with kSharedStage = 0 (nearest_centroid_global_f32) runs on the same input, the two alternating map by
map, so staged and global reads are compared on identical work.  After a warm-up, each map's kernel time comes from the
engine's CUDA events (FBR_POOL_TIMING); the median of --reps maps is reported with points/s, FP32 operations/s
(N * K * 16 * 3: one sub, one mul and one add per dimension, separately rounded, so no FMA) against the 67 TFLOP/s
data-sheet figure (which counts an FMA as two), and HBM bytes/s (N * (64 + 8)) against 3.35 TB/s.  The card's name and
power limit are read in the same call; a sample of every map's results is checked against the NumPy restatement.
Writes one JSON object.
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
from profiles.record_perf import card  # noqa: E402
from tests import broadcast_bodies as BB  # noqa: E402

HBM_DATASHEET_TBS = 3.35       # H100 SXM data sheet
FP32_DATASHEET_TFLOPS = 67.0   # H100 SXM data sheet (FMA = 2 FLOP)
N = 16 << 20
SAMPLE = 2048


class Case:
    def __init__(self, pool, k, points):
        self.pool, self.k = pool, k
        C = BB.centroids(k, seed=k)
        self.C = C
        self.blk = torch.from_numpy(C.view(np.uint8).copy()).cuda()
        self.points = points
        self.out = torch.empty(N * 8, dtype=torch.uint8, device="cuda")

    def run(self, name):
        eng = self.pool._engine
        lib = eng.lib
        d = _abi.MapDesc()
        d.func_id = registry.spec(name).func_id
        d.flags = _abi.FBR_ARGS_DEVICE | _abi.FBR_OUT_DEVICE
        d.n_tasks, d.arg_stride, d.args = N, 64, self.points.data_ptr()
        d.shared, d.shared_bytes = self.blk.data_ptr(), self.blk.numel()
        d.out = self.out.data_ptr()
        _abi.check(lib.fbr_pool_stats_reset(eng.handle))
        seq = ctypes.c_uint64()
        _abi.check(lib.fbr_map_submit(eng.handle, ctypes.byref(d), ctypes.byref(seq)))
        res = _abi.Result()
        _abi.check(lib.fbr_result_wait(eng.handle, seq.value, -1, ctypes.byref(res)))
        _abi.check(lib.fbr_result_release(eng.handle, seq.value))
        st = self.pool.stats()
        assert st["dispatch_launches"] == 1 and st["gather_launches"] == 0, st
        return st["dispatch_ms"]

    def parity(self, head):
        got = self.out[: SAMPLE * 8].cpu().numpy()
        return bool(np.array_equal(got, BB.nearest_np(head, self.C).view(np.uint8)))


def row(case, name, ms, head):
    t = statistics.median(ms)
    flop = N * case.k * 16 * 3
    hbm = N * (64 + 8)
    flops, bps = flop / t / 1e9, hbm / t / 1e9
    of_fp32, of_hbm = flops / FP32_DATASHEET_TFLOPS, bps / HBM_DATASHEET_TBS
    return {"body": name, "K": case.k, "block_bytes": case.k * 64,
            "placement": "global" if name.endswith("global_f32") or case.k * 64 > 32768 else "shared (staged)",
            "n_points": N, "kernel_ms_median": t, "kernel_ms": ms, "spread_ms": max(ms) - min(ms),
            "points_per_s": N / t * 1e3, "fp32_TFLOPs": flops, "of_fp32_datasheet": of_fp32,
            "hbm_TBps": bps, "of_hbm_datasheet": of_hbm, "bound": "FP32 pipe" if of_fp32 > of_hbm else "HBM",
            "results_match_numpy_sample": case.parity(head)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r05_broadcast_perf.json"))
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("broadcast_perf.py measures on a GPU; none is visible")
    torch.cuda.init()
    head = BB.points(SAMPLE, seed=7)
    pts = torch.randn(N * 16, dtype=torch.float32, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    pts[: SAMPLE * 16].copy_(torch.from_numpy(head.view(np.float32).reshape(-1)))
    pool = fiber_b200.Pool(1, devices=[0], timing=True)
    pool.start_workers()
    rows = []
    for k in (64, 256, 512, 513, 2048):
        case = Case(pool, k, pts)
        if k == 256:
            # staged and global alternate map by map on the same input
            names = ("nearest_centroid_f32", "nearest_centroid_global_f32")
            for _ in range(2):
                for nm in names:
                    case.run(nm)
            ms = {nm: [] for nm in names}
            for _ in range(args.reps):
                for nm in names:
                    ms[nm].append(case.run(nm))
            for nm in names:
                case.run(nm)            # leaves this body's results in `out` for the parity check
                rows.append(row(case, nm, ms[nm], head))
        else:
            for _ in range(2):
                case.run("nearest_centroid_f32")
            rows.append(row(case, "nearest_centroid_f32", [case.run("nearest_centroid_f32") for _ in range(args.reps)], head))
        del case
        torch.cuda.empty_cache()
    pool.terminate()
    pool.join()
    staged, glob = [r for r in rows if r["K"] == 256]
    spread = max(staged["spread_ms"], glob["spread_ms"])
    gain = glob["kernel_ms_median"] - staged["kernel_ms_median"]
    result = {"card": card(), "fp32_datasheet_TFLOPs": FP32_DATASHEET_TFLOPS, "hbm_datasheet_TBps": HBM_DATASHEET_TBS,
              "cases": rows,
              "staged_vs_global_K256": {"staged_ms": staged["kernel_ms_median"], "global_ms": glob["kernel_ms_median"],
                                        "gain_ms": gain, "run_to_run_spread_ms": spread, "staging_faster": gain > spread}}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(result, fh, indent=1)
    for r in rows:
        print("%-28s K=%-5d %-16s %7.3f ms (spread %.3f)  %6.2f Gpts/s  %5.1f TFLOP/s (%.0f %%)  %5.2f TB/s (%.0f %%)  %s  ok=%s"
              % (r["body"], r["K"], r["placement"], r["kernel_ms_median"], r["spread_ms"], r["points_per_s"] / 1e9,
                 r["fp32_TFLOPs"], 100 * r["of_fp32_datasheet"], r["hbm_TBps"], 100 * r["of_hbm_datasheet"], r["bound"],
                 r["results_match_numpy_sample"]))
    print(json.dumps(result["staged_vs_global_K256"]))
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
