"""Accumulate maps on the H100: every prefix of a fold (FBR_SCAN) against the plain map of the same body, and against the
map followed by the prefix on the host.

    python profiles/scan_perf.py [--scale 1.0] [--out profiles/r11_scan_perf.json]

End to end (host-resident arguments and results; median of 5 timed calls after one warm-up):

  - ``sum_sq_idx_u64`` (8 B records) over range(n) and ``moments_f64`` (24 B records) over n float64, n = 1e6, 1e7, 1e8:
    ``Pool.accumulate``, ``Pool.map``, and ``Pool.map`` plus the host prefix -- ``np.cumsum`` for the u64 sums, a Python
    loop of Chan's merge for the moments (n = 1e6 only).

Kernel times (torch.profiler, one accumulate and one fold of each size): the scan kernels (``scan_level_kernel`` and
``scan_wrap_kernel``) against the fold pass (``dispatch_record_kernel`` of FoldPass and ``fold_tree_kernel``), and the wrap
kernel's achieved bytes/s, 2 n R over its time, against the H100 SXM data sheet's 3.35 TB/s.

``--scale`` shrinks every size.  The card's name and power limit are read in the same run and written beside the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import fiber_b200  # noqa: E402

from tests import fold_bodies as FB  # noqa: E402
from tests import scan_bodies  # noqa: E402,F401  (registers the scan test bodies next to the fold ones)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def median_ms(fn, reps=5):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def chan_prefix(res):
    out, acc = [], None
    for r in res.tolist():
        acc = tuple(r) if acc is None else FB.moments_combine(acc, tuple(r))
        out.append(acc)
    return out


def kernel_ms(fn):
    """Sum of the device time of each kernel family during fn(), by name."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        name = e.name
        for key in ("scan_level_kernel", "scan_wrap_kernel", "fold_tree_kernel", "FoldPass", "dispatch_record_kernel"):
            if key in name:
                out[key] = out.get(key, 0.0) + e.device_time / 1e3
                break
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r11_scan_perf.json"))
    a = ap.parse_args()
    rows = []
    pool = fiber_b200.Pool(1, devices=[0])
    try:
        for name in ("sum_sq_idx_u64", "moments_f64"):
            f = getattr(FB, name)
            R = 8 if name == "sum_sq_idx_u64" else 24
            for n0 in (10 ** 6, 10 ** 7, 10 ** 8):
                n = max(1, int(n0 * a.scale))
                xs = range(n) if name == "sum_sq_idx_u64" else np.random.default_rng(n).standard_normal(n) * 1e3
                row = {"body": name, "n": n, "record_bytes": R}
                row["accumulate_ms"] = median_ms(lambda: pool.accumulate(f, xs))
                row["map_ms"] = median_ms(lambda: pool.map(f, xs))
                if name == "sum_sq_idx_u64":
                    row["map_plus_np_cumsum_ms"] = median_ms(lambda: np.cumsum(np.asarray(pool.map(f, xs)), dtype=np.uint64))
                elif n0 == 10 ** 6:
                    row["map_plus_python_chan_ms"] = median_ms(lambda: chan_prefix(np.asarray(pool.map(f, xs))), reps=2)
                k_scan = kernel_ms(lambda: pool.accumulate(f, xs))
                k_fold = kernel_ms(lambda: pool.fold(f, xs))
                row["kernels_accumulate_ms"] = k_scan
                row["kernels_fold_ms"] = k_fold
                wrap = k_scan.get("scan_wrap_kernel", 0.0)
                if wrap:
                    row["wrap_tb_per_s"] = 2.0 * n * R / (wrap * 1e-3) / 1e12
                    row["wrap_fraction_of_3_35_tb_s"] = row["wrap_tb_per_s"] / 3.35
                print(json.dumps(row), flush=True)
                rows.append(row)
    finally:
        pool.terminate()
        pool.join()
    out = {"card": card(), "scale": a.scale, "rows": rows}
    with open(a.out, "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps({"card": out["card"]}))


if __name__ == "__main__":
    main()
