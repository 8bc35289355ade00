"""Keyed folds on the H100 (Pool.fold_by_key, FBR_FOLD_KEYS) against the ways to get the same groups without them.

    python profiles/keyed_perf.py [--scale 1.0] [--out profiles/r12_keyed_perf.json]

End to end (host-resident arguments and results, one worker; three rounds, the variants alternating inside each round, the
median of each round's calls and the spread over the rounds):

  - ``label_sum_u64`` (8 B arguments, 16 B records) at n = 1e8 with K = 1, 256 and 65536 keys: ``Pool.fold_by_key``,
    ``Pool.fold`` of the same body (K = 1 only: the same bits), and ``Pool.map`` followed by the host reduction
    (``np.bincount`` of the labels and ``np.add.at`` of the values).
  - ``kmeans_step_f32`` at 16 Mi points, K = 64 centroids: ``Pool.fold_by_key`` against ``Pool.map(nearest_centroid_f32)``
    followed by the NumPy update (``np.add.at`` of the points per centroid, ``np.bincount`` of the counts).

Kernel split (torch.profiler, one keyed fold of label_sum_u64 per K): the dispatch kernel, ``keys_kernel``, each sort pass
(``radix_hist_kernel``, ``scan_counts_kernel``, ``radix_scatter_kernel``), ``key_offsets_kernel``, ``gather_records_kernel``
and the segmented tree (``seg_tiles_kernel``, ``fold_segments_kernel``, ``fold_segments_out_kernel``).  The sort's bytes
-- per pass the histogram's 4 n reads and the scatter's keys and indices, 4 n (first pass) or 8 n read and 8 n written --
over the sort kernels' time, as a share of the H100 SXM data sheet's 3.35 TB/s.

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

from tests import broadcast_bodies as BB  # noqa: E402
from tests import keyed_bodies as KB  # noqa: E402

HBM_TBS = 3.35
SORT_KERNELS = ("radix_hist_kernel", "scan_counts_kernel", "radix_scatter_kernel")
KERNELS = ("dispatch_record_kernel", "keys_kernel") + SORT_KERNELS + (
    "key_offsets_kernel", "gather_records_kernel", "seg_tiles_kernel", "fold_segments_out_kernel", "fold_segments_kernel")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    if not q:
        raise RuntimeError("nvidia-smi found no GPU: keyed_perf.py measures the H100 and has no CPU mode")
    return q[0]


def rounds(variants, rounds=3, reps=1):
    """Each variant warmed up once, then ``rounds`` rounds in which the variants alternate, ``reps`` timed calls each; per
    variant the median of each round (ms), their median and their spread (max - min)."""
    for fn in variants.values():
        fn()
    per = {name: [] for name in variants}
    for _ in range(rounds):
        for name, fn in variants.items():
            ts = []
            for _ in range(reps):
                t0 = time.perf_counter()
                fn()
                ts.append((time.perf_counter() - t0) * 1e3)
            per[name].append(float(np.median(ts)))
    return {name: {"rounds_ms": v, "median_ms": float(np.median(v)), "spread_ms": float(max(v) - min(v))} for name, v in per.items()}


def kernel_split(fn):
    """Device time (ms) of each kernel family during fn(), by name, and the number of launches."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        for key in KERNELS:
            if key in e.name:
                ms, k = out.get(key, (0.0, 0))
                out[key] = (ms + e.device_time / 1e3, k + 1)
                break
    return {k: {"ms": v[0], "launches": v[1]} for k, v in out.items()}


def sort_bytes(n, n_keys):
    passes = 0 if n_keys <= 1 else 1 if n_keys <= 256 else 2
    return sum(4 * n + (4 * n if p == 0 else 8 * n) + 8 * n for p in range(passes)), passes


def label_sum(pool, n, n_keys_list):
    rng = np.random.default_rng(1)
    args = np.zeros(n, KB.LABEL_ARG)
    args["v"] = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    out = {}
    for K in n_keys_list:
        args["label"] = rng.integers(0, K, n)

        def host_reduce(K=K):
            r = pool.map(KB.label_sum_u64, args)
            a = np.asarray(r.array)
            sums = np.zeros(K, np.uint64)
            np.add.at(sums, a["key"], a["sum"])
            return sums, np.bincount(a["key"], minlength=K)

        variants = {"fold_by_key": lambda K=K: pool.fold_by_key(KB.label_sum_u64, args, K), "map_plus_numpy": host_reduce}
        if K == 1:
            variants["fold"] = lambda: pool.fold(KB.label_sum_u64, args)
        got = pool.fold_by_key(KB.label_sum_u64, args, K)
        sums, counts = host_reduce()
        same = bool(np.array_equal(np.asarray(got.array)["sum"], sums) and np.array_equal(got.counts, counts))
        split = kernel_split(lambda K=K: pool.fold_by_key(KB.label_sum_u64, args, K))
        nbytes, passes = sort_bytes(n, K)
        sort_ms = sum(split.get(k, {"ms": 0.0})["ms"] for k in SORT_KERNELS)
        out["K=%d" % K] = {
            "n": n, "n_keys": K, "times": rounds(variants), "same_result_as_map_plus_numpy": same, "kernels": split,
            "sort": {"passes": passes, "bytes": nbytes, "ms": sort_ms,
                     "tb_per_s": nbytes / sort_ms / 1e9 if sort_ms else None,
                     "share_of_3_35_tbs": nbytes / sort_ms / 1e9 / HBM_TBS if sort_ms else None},
        }
    return out


def kmeans(n, K):
    rng = np.random.default_rng(2)
    cents = rng.standard_normal((K, 16)).astype(np.float32)
    pts = np.zeros(n, KB.POINT)
    pts["p"] = rng.standard_normal((n, 16)).astype(np.float32)
    keyed = fiber_b200.Pool(1, devices=[0], initializer=KB.set_centroids, initargs=(cents,))
    plain = fiber_b200.Pool(1, devices=[0], initializer=BB.set_centroids, initargs=(cents,))
    try:
        p2 = pts["p"].reshape(n, 16)

        def map_plus_numpy():
            k = np.asarray(plain.map(BB.nearest_centroid_f32, pts).array)["k"]
            sums = np.zeros((K, 16), np.float32)
            np.add.at(sums, k, p2)
            return sums, np.bincount(k, minlength=K)

        got = keyed.fold_by_key(KB.kmeans_step_f32, pts, K)
        _, counts = map_plus_numpy()
        return {"n": n, "n_keys": K, "same_counts_as_map_plus_numpy": bool(np.array_equal(got.counts, counts)),
                "note": "the float32 sums differ in order from np.add.at's, so only the counts are compared",
                "times": rounds({"fold_by_key": lambda: keyed.fold_by_key(KB.kmeans_step_f32, pts, K),
                                 "map_plus_numpy": map_plus_numpy})}
    finally:
        for p in (keyed, plain):
            p.terminate()
            p.join()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r12_keyed_perf.json"))
    a = ap.parse_args()
    rec = {"gpu": card(), "workers": 1, "results": "host"}
    pool = fiber_b200.Pool(1, devices=[0])
    try:
        rec["label_sum_u64"] = label_sum(pool, max(1, int(1e8 * a.scale)), (1, 256, 65536))
    finally:
        pool.terminate()
        pool.join()
    rec["kmeans_step_f32"] = kmeans(max(1, int((16 << 20) * a.scale)), 64)
    rec["gpu_after"] = card()
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
