"""Sparse keyed folds on the H100 (Pool.fold_by_sparse_key, FBR_FOLD_SPARSE_KEYS) against the ways to get the same groups
without them.

    python profiles/sparse_keyed_perf.py [--scale 1.0] [--out profiles/r13_sparse_keyed_perf.json]

End to end (host-resident arguments and results, one worker; three rounds, the variants alternating inside each round, the
median of each round's calls and the spread over the rounds):

  - ``label_sum_u64`` (8 B arguments, 16 B records) at n = 1e8 with D ~ 1e3, 1e6 and ~ n distinct keys (uniform over 32
    bits): ``Pool.starfold_by_sparse_key`` against ``Pool.map`` followed by the host reduction (``np.unique(...,
    return_inverse=True)`` and ``np.add.reduceat`` of the values in key order); at D ~ 1e3 also ``fold_by_key`` over the
    same data with the labels mapped to their ranks (the mapping is not timed).
  - A word count over 8 Mi strings: ``Pool.map(tokens_u32)`` then ``starfold_by_sparse_key(label_sum_u64)`` of the hashes
    against the same map followed by ``np.unique(..., return_counts=True)`` of the hashes.

Kernel split (torch.profiler, one sparse keyed fold per D): ``keys_kernel``, the four sort passes (``radix_hist_kernel``,
``scan_counts_kernel``, ``radix_scatter_kernel``), ``gather_records_kernel``, the runs (``run_heads_kernel``,
``run_starts_kernel``) and the segmented fold (``seg_tiles_kernel``, ``fold_segments_kernel``, ``fold_segments_out_kernel``).
``scan_counts_kernel`` serves both the sort and the runs; its launches are reported together.

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

from tests import emit_bodies as EB  # noqa: E402
from tests import keyed_bodies as KB  # noqa: E402

KERNELS = ("dispatch_record_kernel", "keys_kernel", "radix_hist_kernel", "scan_counts_kernel", "radix_scatter_kernel",
           "gather_records_kernel", "run_heads_kernel", "run_starts_kernel", "seg_tiles_kernel", "fold_segments_out_kernel",
           "fold_segments_kernel")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    if not q:
        raise RuntimeError("nvidia-smi found no GPU: sparse_keyed_perf.py measures the H100 and has no CPU mode")
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


def host_reduce(labels, vals):
    keys, inv = np.unique(labels, return_inverse=True)
    order = np.argsort(inv, kind="stable")
    starts = np.flatnonzero(np.concatenate([[True], np.diff(inv[order]) != 0]))
    return keys, np.add.reduceat(vals[order].astype(np.uint64), starts), np.diff(np.concatenate([starts, [len(inv)]]))


def label_sum(pool, n):
    rng = np.random.default_rng(1)
    vals = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    out = {}
    for name, D in (("D~1e3", 1000), ("D~1e6", 1_000_000), ("D~n", None)):
        if D is None:
            labels = rng.integers(0, 0xFFFFFFFF, n, dtype=np.uint64).astype(np.uint32)
        else:
            labels = rng.choice(rng.integers(0, 0xFFFFFFFF, D, dtype=np.uint64).astype(np.uint32), n)
        cols = fiber_b200.Columns(labels, vals)

        def map_plus_numpy():
            a = np.asarray(pool.starmap(KB.label_sum_u64, cols).array)
            return host_reduce(a["key"], a["sum"])

        variants = {"fold_by_sparse_key": lambda: pool.starfold_by_sparse_key(KB.label_sum_u64, cols),
                    "map_plus_numpy": map_plus_numpy}
        if D is not None and D <= 65536:
            ranks = np.unique(labels, return_inverse=True)[1].astype(np.uint32)
            rcols = fiber_b200.Columns(ranks, vals)
            n_ranks = int(ranks.max()) + 1
            variants["fold_by_key_of_ranks"] = lambda: pool.starfold_by_key(KB.label_sum_u64, rcols, n_ranks)
        got = pool.starfold_by_sparse_key(KB.label_sum_u64, cols)
        keys, sums, counts = host_reduce(labels, vals)
        same = bool(np.array_equal(got.keys, keys) and np.array_equal(np.asarray(got.array)["sum"], sums)
                    and np.array_equal(got.counts, counts))
        out[name] = {"n": n, "distinct_keys": len(got), "times": rounds(variants), "same_result_as_map_plus_numpy": same,
                     "kernels": kernel_split(lambda: pool.starfold_by_sparse_key(KB.label_sum_u64, cols))}
    return out


def word_count(pool, n_docs):
    rng = np.random.default_rng(3)
    vocab = [bytes(rng.integers(97, 123, rng.integers(1, 12), dtype=np.uint8)) for _ in range(200_000)]
    words = np.minimum(rng.zipf(1.2, n_docs * 8), len(vocab)) - 1
    docs = [b" ".join(vocab[i] for i in words[8 * d:8 * d + 8]) for d in range(n_docs)]

    def device():
        h = pool.map(EB.tokens_u32, docs).ragged.values
        return pool.starfold_by_sparse_key(KB.label_sum_u64, fiber_b200.Columns(h, np.ones(len(h), np.uint32)))

    def host():
        return np.unique(pool.map(EB.tokens_u32, docs).ragged.values, return_counts=True)

    got, (keys, counts) = device(), host()
    return {"strings": n_docs, "tokens": int(counts.sum()), "distinct": len(keys),
            "same_counts": bool(np.array_equal(got.keys, keys) and np.array_equal(got.counts, counts)),
            "times": rounds({"map_then_fold_by_sparse_key": device, "map_then_np_unique": host})}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r13_sparse_keyed_perf.json"))
    a = ap.parse_args()
    rec = {"gpu": card(), "workers": 1, "results": "host"}
    pool = fiber_b200.Pool(1, devices=[0])
    try:
        rec["label_sum_u64"] = label_sum(pool, max(1, int(1e8 * a.scale)))
        rec["word_count"] = word_count(pool, max(1, int((8 << 20) * a.scale)))
    finally:
        pool.terminate()
        pool.join()
    rec["gpu_after"] = card()
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
