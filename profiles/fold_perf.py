"""Fold maps on the H100: a map reduced on the device (FBR_FOLD) against the plain map of the same body.

    python profiles/fold_perf.py [--scale 1.0] [--out profiles/r10_fold_perf.json]

Workloads (each number is the median of 10 timed maps, over three rounds that alternate the variants, with the spread of
the three medians; device-resident arguments, results kept on the device for the plain maps):

  1. ``moments_f64`` over 256 Mi float64: the fold, the plain map (24 B of results per task), and a device-to-device copy of
     8 B per task (the arguments' bytes);
  2. the per-unit tree with a trivial body: ``sum_sq_idx_u64`` over range(2**30), fold against map;
  3. ``byte_hist_u8`` over 1 Mi byte strings of 0 to 512 bytes (the ``fnv1a_bytes`` inputs of r07): fold against map
     (1 KB of counts per task);
  4. end to end, host-resident: ``Pool.fold(moments_f64, x)`` against ``Pool.map`` plus the NumPy reduction of its results,
     for 64 Mi float64 (median of 3 per round).

``--scale`` shrinks every size (a rehearsal without a GPU fails at the first device call).  The card's name and power
limit are read in the same run and written beside the numbers."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import fiber_b200  # noqa: E402
from fiber_b200 import _abi, registry  # noqa: E402

from tests import fold_bodies as FB  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


class Device:
    def __init__(self, pool):
        self.eng = pool._engine
        self.ptrs = []

    def put(self, arr):
        p = ctypes.c_void_p()
        _abi.check(self.eng.lib.fbr_device_alloc(self.eng.handle, 0, max(16, arr.nbytes), ctypes.byref(p)))
        _abi.check(self.eng.lib.fbr_memcpy_h2d(self.eng.handle, 0, p, arr.ctypes.data, arr.nbytes))
        self.ptrs.append(p)
        return p.value

    def free(self):
        for p in self.ptrs:
            self.eng.lib.fbr_device_free(self.eng.handle, 0, p)


def run(pool, name, n, fold, args=None, stride=0, items=None):
    """One device-resident map submitted and waited for: (seconds, the fold's record or None)."""
    spec = registry.spec(name)
    eng = pool._engine
    d = _abi.MapDesc()
    d.func_id, d.n_tasks, d.chunksize = spec.func_id, n, 32
    d.flags = _abi.FBR_ARGS_DEVICE | (_abi.FBR_FOLD if fold else _abi.FBR_RESULTS_ON_DEVICE)
    if args is not None:
        d.args, d.arg_stride = args, stride
    else:
        d.index_start, d.index_step = 0, 1
    seq, res = ctypes.c_uint64(), _abi.Result()
    t0 = time.perf_counter()
    if items is not None:
        it = _abi.ItemsDesc()
        it.items, it.offsets, it.n_items, it.item_bytes = items[0], items[1], items[2], 1
        _abi.check(eng.lib.fbr_map_submit_items(eng.handle, ctypes.byref(d), ctypes.byref(it), ctypes.byref(seq)))
    else:
        _abi.check(eng.lib.fbr_map_submit(eng.handle, ctypes.byref(d), ctypes.byref(seq)))
    _abi.check(eng.lib.fbr_result_wait(eng.handle, seq.value, -1, ctypes.byref(res)))
    dt = time.perf_counter() - t0
    out = spec.unpack_result(ctypes.string_at(res.data, res.result_bytes)) if fold else None
    _abi.check(eng.lib.fbr_result_release(eng.handle, seq.value))
    return dt, out


def rounds_of(variants, reps=10, n_rounds=3):
    for f in variants.values():                      # warm-up
        f()
    out = {k: [] for k in variants}
    for _ in range(n_rounds):
        for k, f in variants.items():
            out[k].append(float(np.median([f() for _ in range(reps)])))
    return out


def stats(v):
    return {"median": float(np.median(v)), "rounds": v, "spread": float(max(v) - min(v))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r10_fold_perf.json"))
    a = ap.parse_args()
    import torch
    n_mom, n_idx, n_str, n_e2e = (max(1024, int(s * a.scale)) for s in (256 << 20, 1 << 30, 1 << 20, 64 << 20))
    rng = np.random.default_rng(7)
    x = rng.standard_normal(n_mom) * 100 + 3
    lens = rng.integers(0, 513, n_str)
    offs = np.zeros(n_str + 1, np.uint64)
    np.cumsum(lens, out=offs[1:])
    strs = rng.integers(0, 256, int(offs[-1]), dtype=np.uint8)
    pool = fiber_b200.Pool(1, devices=[0])
    pool.start_workers()
    dev = Device(pool)
    out = {"card": card()}
    try:
        dx, ds, do = dev.put(x), dev.put(strs), dev.put(offs)
        src = torch.empty(n_mom * 8, dtype=torch.uint8, device="cuda:0")
        dst = torch.empty_like(src)

        def d2d():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            dst.copy_(src)
            e1.record()
            e1.synchronize()
            return e0.elapsed_time(e1) / 1e3

        # results first: each fold equals its restatement (bit for bit where the restatement is cheap enough)
        _, got = run(pool, "sum_sq_idx_u64", n_idx, True)
        assert got == (sum(i * i for i in range(n_idx)) if n_idx < 1 << 20 else (n_idx - 1) * n_idx * (2 * n_idx - 1) // 6) & FB.M64
        _, got = run(pool, "byte_hist_u8", n_str, True, items=(ds, do, len(strs)))
        assert list(got) == np.bincount(strs, minlength=256).tolist()
        _, got = run(pool, "moments_f64", n_mom, True, args=dx, stride=8)
        assert got[0] == n_mom and abs(got[1] - x.mean()) < 1e-9 * abs(x.mean()) + 1e-9
        mom = rounds_of({
            "fold": lambda: run(pool, "moments_f64", n_mom, True, args=dx, stride=8)[0],
            "map": lambda: run(pool, "moments_f64", n_mom, False, args=dx, stride=8)[0],
            "d2d_copy_8B_per_task": d2d,
        })
        idx = rounds_of({
            "fold": lambda: run(pool, "sum_sq_idx_u64", n_idx, True)[0],
            "map": lambda: run(pool, "sum_sq_idx_u64", n_idx, False)[0],
        })
        hist = rounds_of({
            "fold": lambda: run(pool, "byte_hist_u8", n_str, True, items=(ds, do, len(strs)))[0],
            "map": lambda: run(pool, "byte_hist_u8", n_str, False, items=(ds, do, len(strs)))[0],
        })
        xe = x[:n_e2e].copy()

        def e2e_fold():
            t = time.perf_counter()
            r = pool.fold(FB.moments_f64, xe)
            return time.perf_counter() - t, r

        def e2e_map():
            t = time.perf_counter()
            arr = np.asarray(pool.map(FB.moments_f64, xe))
            mean = float(arr["mean"].mean())
            r = (float(arr["n"].sum()), mean, float(((arr["mean"] - mean) ** 2).sum() + arr["m2"].sum()))
            return time.perf_counter() - t, r

        rf, rm = e2e_fold()[1], e2e_map()[1]
        assert rf[0] == rm[0] == n_e2e and abs(rf[1] - rm[1]) < 1e-9 * abs(rm[1]) and abs(rf[2] - rm[2]) < 1e-6 * rm[2]
        e2e = {"fold": [], "map_plus_numpy": []}
        for _ in range(3):
            e2e["fold"].append(float(np.median([e2e_fold()[0] for _ in range(3)])))
            e2e["map_plus_numpy"].append(float(np.median([e2e_map()[0] for _ in range(3)])))
    finally:
        dev.free()
        pool.terminate()
        pool.join()
    out["workloads"] = {
        "moments_f64_device": {"tasks": n_mom, "seconds": {k: stats(v) for k, v in mom.items()}},
        "sum_sq_idx_u64_range": {"tasks": n_idx, "seconds": {k: stats(v) for k, v in idx.items()}},
        "byte_hist_u8_strings": {"tasks": n_str, "string_bytes": int(len(strs)), "seconds": {k: stats(v) for k, v in hist.items()}},
        "moments_f64_host_e2e": {"tasks": n_e2e, "seconds": {k: stats(v) for k, v in e2e.items()}},
    }
    for w in out["workloads"].values():
        s = w["seconds"]
        other = "map" if "map" in s else "map_plus_numpy"
        w["fold_over_" + other] = s["fold"]["median"] / s[other]["median"]
    out["conditions"] = ("device-resident arguments, chunksize 32 for the plain maps (FBR_RESULTS_ON_DEVICE), median of 10, "
                         "3 alternating rounds; the host end-to-end pair: median of 3 per round")
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
