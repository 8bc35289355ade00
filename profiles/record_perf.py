"""Kernel rate of dispatch_record_kernel (record bodies) against a device-to-device copy of the same bytes.

    python profiles/record_perf.py [--out profiles/record_perf.json] [--reps 10]

Device-resident maps (FBR_ARGS_DEVICE | FBR_OUT_DEVICE, one wave, direct placement) of three record bodies from
tests/record_bodies.py: polar_f64 (16 B -> 16 B) and mix_i32x3 (12 B -> 12 B) at 64 Mi tasks, row_stats_u32
(1024 B -> 24 B) at 1 Mi tasks.  After a warm-up, the kernel time of each map comes from the engine's CUDA events
(FBR_POOL_TIMING); the algorithmic bytes are n * (A + R).  Beside each body, in the same call, a cudaMemcpy
device-to-device of n * (A + R) / 2 bytes (which reads and writes n * (A + R) bytes in all) is timed with CUDA
events.  The card's name and power limit are read in the same call.  A sample of every map's results is checked
against the NumPy restatement.  Writes one JSON object.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from fiber_b200 import registry  # noqa: E402
from tests import record_bodies as RB  # noqa: E402

HBM_DATASHEET_TBS = 3.35     # H100 SXM data sheet


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                                       "--format=csv,noheader"], text=True, timeout=30).strip()
        name, power, clk = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "sm_clock_max": clk}
    except Exception as e:      # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "power_limit": "unknown (%s)" % e}


def time_copy(nbytes, reps):
    src = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    dst = torch.empty_like(src)
    for _ in range(2):
        dst.copy_(src)
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        dst.copy_(src)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    del src, dst
    return statistics.median(ms), ms


def run_body(eng, name, n, make_sample, ref, reps):
    spec = registry.spec(name)
    A, R = spec.arg_bytes, spec.result_bytes
    args = torch.randint(-2 ** 31, 2 ** 31 - 1, (n * A // 4,), dtype=torch.int32, device="cuda")
    sample = make_sample(4096, seed=1)                      # a known head of the argument array, checked below
    args[: 4096 * A // 4].copy_(torch.from_numpy(sample.view(np.int32)))
    out = torch.empty(n * R, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def one():
        eng.stats(reset=True)
        eng.wait(eng.submit(name, n, ctypes_ptr(out), args_dev=ctypes_ptr(args), arg_stride=A, want_sum=False))
        st = eng.stats()
        assert st["dispatch_launches"] == 1 and st["gather_launches"] == 0, st
        return st["dispatch_ms"]
    for _ in range(2):
        one()
    ms = [one() for _ in range(reps)]
    head = out[: 4096 * R].cpu().numpy()
    ok = bool(np.array_equal(head, np.ascontiguousarray(ref(sample)).view(np.uint8)))
    del args, out
    torch.cuda.empty_cache()
    copy_ms, copy_all = time_copy(n * (A + R) // 2, reps)
    t = statistics.median(ms)
    algo = n * (A + R)
    return {"body": name, "n_tasks": n, "arg_bytes": A, "result_bytes": R, "algorithmic_bytes": algo,
            "kernel_ms_median": t, "kernel_ms": ms, "kernel_GBps": algo / t / 1e6,
            "copy_ms_median": copy_ms, "copy_ms": copy_all, "copy_GBps": algo / copy_ms / 1e6,
            "of_copy": copy_ms / t, "of_datasheet_hbm": algo / t / 1e6 / (HBM_DATASHEET_TBS * 1e3),
            "results_match_numpy_sample": ok}


def ctypes_ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "record_perf.json"))
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("record_perf.py measures on a GPU; none is visible")
    torch.cuda.init()
    eng = bench.RawEngine(0, 0)
    rows = [run_body(eng, "polar_f64", 64 << 20, RB.polar_args, RB.polar_np, args.reps),
            run_body(eng, "mix_i32x3", 64 << 20, RB.mix_args, RB.mix_np, args.reps),
            run_body(eng, "row_stats_u32", 1 << 20, RB.row_args, RB.row_stats_np, args.reps)]
    eng.close()
    result = {"card": card(), "hbm_datasheet_TBps": HBM_DATASHEET_TBS, "bodies": rows}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(result, fh, indent=1)
    for r in rows:
        print("%-14s n=%-9d %5.3f ms  %7.1f GB/s  copy %7.1f GB/s  (%.0f %% of copy, %.0f %% of data sheet)  sample ok=%s"
              % (r["body"], r["n_tasks"], r["kernel_ms_median"], r["kernel_GBps"], r["copy_GBps"], 100 * r["of_copy"],
                 100 * r["of_datasheet_hbm"], r["results_match_numpy_sample"]))
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
