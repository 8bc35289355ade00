"""Kernel rate of group record bodies (kGroup) against one-thread record bodies and a device-to-device copy.

    python profiles/group_perf.py [--out profiles/group_perf.json] [--reps 10] [--rounds 3]

1. 4 KB rows, one thread against a group: three bodies reduce the same float x[1024] rows to (max, min) --
   row4k_word_f32 (one thread per task, word by word: the 32 lanes of a warp read words 4 KB apart, one shared-memory
   bank), row4k_vec_f32 (one thread, 16 B vectors) and row4k_group_f32 (a warp per task, lane k reads x[k + 32 j]).
   max and min do not depend on the order, so all three give the same results.  The three are timed in turn, --rounds
   times, so the spread between rounds is measured beside the differences between bodies.
2. The new sizes: row_moments_f64 (8 KB rows, four tasks per unit) and wide_row_max_f32 (32 KB rows: one task per
   unit, so one of the eight consumer warps runs it while seven wait) from tests/group_bodies.py.

Every map is device-resident (FBR_ARGS_DEVICE | FBR_OUT_DEVICE) with direct placement; its kernel time comes from the
engine's CUDA events (FBR_POOL_TIMING), the median of --reps maps after a warm-up.  The algorithmic bytes are
n * (A + R).  Beside each body, in the same call, a device-to-device copy that reads and writes the same bytes is timed
with CUDA events.  The card's name and power limit are read in the same call.  The first 4096 results of every map are
checked against the NumPy restatement.  Writes one JSON object.
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

import bench  # noqa: E402
import fiber_b200  # noqa: E402
from fiber_b200 import registry  # noqa: E402
from profiles.record_perf import HBM_DATASHEET_TBS, card, time_copy  # noqa: E402
from tests import group_bodies as GB  # noqa: E402

ROW4K_ARG = np.dtype([("x", "<f4", (1024,))])
ROW4K_RES = np.dtype([("max", "<f4"), ("min", "<f4")])

ROW4K_SRC = r'''
#include "fiber_b200_body.cuh"

// a row of 1024 float32 -> (max, min), three ways
struct Row4kWord {               // one thread, word by word
    struct Arg { float x[1024]; };
    struct Res { float mx, mn; };
    static constexpr bool kIndexArg = false;
    static constexpr bool kCanFault = false;
    __device__ static __forceinline__ void run(const Arg& a, Res& r, uint64_t, const fbr::ErrSink&, uint32_t) {
        float mx = a.x[0], mn = a.x[0];
#pragma unroll 8
        for (uint32_t k = 1; k < 1024; ++k) { mx = fmaxf(mx, a.x[k]); mn = fminf(mn, a.x[k]); }
        r.mx = mx; r.mn = mn;
    }
};
FBR_EXPORT_RECORD_BODY(Row4kWord, "row4k_word_f32", row4k_word_entry, 0)

struct Row4kVec {                // one thread, 16 B vectors (records start at multiples of 4 KB in the stage)
    using Arg = Row4kWord::Arg;
    using Res = Row4kWord::Res;
    static constexpr bool kIndexArg = false;
    static constexpr bool kCanFault = false;
    __device__ static __forceinline__ void run(const Arg& a, Res& r, uint64_t, const fbr::ErrSink&, uint32_t) {
        const float4* v = reinterpret_cast<const float4*>(a.x);
        float mx = a.x[0], mn = a.x[0];
#pragma unroll 4
        for (uint32_t k = 0; k < 256; ++k) {
            const float4 q = v[k];
            mx = fmaxf(fmaxf(mx, q.x), fmaxf(q.y, fmaxf(q.z, q.w)));
            mn = fminf(fminf(mn, q.x), fminf(q.y, fminf(q.z, q.w)));
        }
        r.mx = mx; r.mn = mn;
    }
};
FBR_EXPORT_RECORD_BODY(Row4kVec, "row4k_vec_f32", row4k_vec_entry, 0)

struct Row4kGroup {              // a warp per task: lane k reads x[k], x[k + 32], ...
    using Arg = Row4kWord::Arg;
    using Res = Row4kWord::Res;
    static constexpr uint32_t kGroup = 32;
    static constexpr bool kIndexArg = false;
    static constexpr bool kCanFault = false;
    __device__ static __forceinline__ void run(const Arg& a, Res& r, const fbr::Group<32>& g, uint64_t,
                                               const fbr::ErrSink&, uint32_t) {
        float mx = a.x[g.rank], mn = mx;
#pragma unroll 8
        for (uint32_t k = g.rank + 32; k < 1024; k += 32) { mx = fmaxf(mx, a.x[k]); mn = fminf(mn, a.x[k]); }
#pragma unroll
        for (uint32_t o = 16; o > 0; o >>= 1) {
            mx = fmaxf(mx, __shfl_xor_sync(g.mask, mx, o));
            mn = fminf(mn, __shfl_xor_sync(g.mask, mn, o));
        }
        if (g.rank == 0) { r.mx = mx; r.mn = mn; }
    }
};
FBR_EXPORT_RECORD_BODY(Row4kGroup, "row4k_group_f32", row4k_group_entry, 0)
'''

for _name in ("row4k_word_f32", "row4k_vec_f32", "row4k_group_f32"):
    fiber_b200.device_body(_name, source=ROW4K_SRC, entry=_name.replace("_f32", "_entry"), args=ROW4K_ARG,
                           result=ROW4K_RES)


def row4k_np(args):
    out = np.empty(len(args), ROW4K_RES)
    out["max"] = args["x"].max(axis=1)
    out["min"] = args["x"].min(axis=1)
    return out


def ctypes_ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def make_args(dtype, n):
    """n records of `dtype` (float fields only) filled with standard normal values on the device."""
    base = dtype.fields[dtype.names[0]][0].base
    tdt = {np.dtype("<f4"): torch.float32, np.dtype("<f8"): torch.float64}[base]
    return torch.randn(n * dtype.itemsize // base.itemsize, dtype=tdt, device="cuda")


def time_body(eng, name, args, n, reps):
    spec = registry.spec(name)
    out = torch.empty(n * spec.result_bytes, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def one():
        eng.stats(reset=True)
        eng.wait(eng.submit(name, n, ctypes_ptr(out), args_dev=ctypes_ptr(args), arg_stride=spec.arg_bytes, want_sum=False))
        st = eng.stats()
        assert st["gather_launches"] == 0, st
        return st["dispatch_ms"], st["dispatch_launches"]
    for _ in range(2):
        one()
    runs = [one() for _ in range(reps)]
    head = np.frombuffer(args[: 4096 * spec.arg_bytes // args.element_size()].cpu().numpy().tobytes(), spec.arg_dtype)
    ok = bool(np.array_equal(out[: 4096 * spec.result_bytes].cpu().numpy(), np.ascontiguousarray(REF[name](head)).view(np.uint8)))
    del out
    ms = [r[0] for r in runs]
    return {"kernel_ms_median": statistics.median(ms), "kernel_ms": ms, "launches": runs[0][1],
            "results_match_numpy_head": ok}


REF = {"row4k_word_f32": row4k_np, "row4k_vec_f32": row4k_np, "row4k_group_f32": row4k_np,
       "row_moments_f64": GB.row_moments_np, "wide_row_max_f32": GB.wide_row_max_np}


def rates(name, n, t_ms, copy_ms):
    spec = registry.spec(name)
    algo = n * (spec.arg_bytes + spec.result_bytes)
    return {"body": name, "n_tasks": n, "arg_bytes": spec.arg_bytes, "result_bytes": spec.result_bytes,
            "algorithmic_bytes": algo, "kernel_GBps": algo / t_ms / 1e6, "copy_ms_median": copy_ms,
            "copy_GBps": algo / copy_ms / 1e6, "of_copy": copy_ms / t_ms,
            "of_datasheet_hbm": algo / t_ms / 1e6 / (HBM_DATASHEET_TBS * 1e3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "group_perf.json"))
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("group_perf.py measures on a GPU; none is visible")
    torch.cuda.init()
    eng = bench.RawEngine(0, 0)

    # 1. 4 KB rows: the three bodies over the same 1 GiB of rows, in turn, --rounds times
    n4 = 1 << 18
    a4 = make_args(ROW4K_ARG, n4)
    trio = ("row4k_word_f32", "row4k_vec_f32", "row4k_group_f32")
    rounds = {name: [] for name in trio}
    for _ in range(args.rounds):
        for name in trio:
            rounds[name].append(time_body(eng, name, a4, n4, args.reps))
    del a4
    torch.cuda.empty_cache()
    copy4, copy4_all = time_copy(n4 * (4096 + 8) // 2, args.reps)
    four_kb = []
    for name in trio:
        meds = [r["kernel_ms_median"] for r in rounds[name]]
        t = statistics.median(meds)
        row = rates(name, n4, t, copy4)
        row.update({"kernel_ms_median": t, "round_medians_ms": meds,
                    "round_spread": (max(meds) - min(meds)) / t, "rounds": rounds[name],
                    "results_match_numpy_head": all(r["results_match_numpy_head"] for r in rounds[name])})
        four_kb.append(row)

    # 2. the new sizes
    new_sizes = []
    for name, dtype, n in (("row_moments_f64", GB.MOMENTS_ARG, 1 << 17), ("wide_row_max_f32", GB.WIDE_ARG, 1 << 15)):
        a = make_args(dtype, n)
        r = time_body(eng, name, a, n, args.reps)
        del a
        torch.cuda.empty_cache()
        spec = registry.spec(name)
        copy_ms, copy_all = time_copy(n * (spec.arg_bytes + spec.result_bytes) // 2, args.reps)
        row = rates(name, n, r["kernel_ms_median"], copy_ms)
        row.update(r)
        row["copy_ms"] = copy_all
        new_sizes.append(row)
    eng.close()

    result = {"card": card(), "hbm_datasheet_TBps": HBM_DATASHEET_TBS, "copy_4kb_ms": copy4_all,
              "four_kb_rows": four_kb, "new_sizes": new_sizes}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(result, fh, indent=1)
    for r in four_kb + new_sizes:
        print("%-18s n=%-7d %6.3f ms  %7.1f GB/s  copy %7.1f GB/s  (%.0f %% of copy)  spread %s  head ok=%s"
              % (r["body"], r["n_tasks"], r["kernel_ms_median"], r["kernel_GBps"], r["copy_GBps"], 100 * r["of_copy"],
                 "%.1f %%" % (100 * r["round_spread"]) if "round_spread" in r else "-", r["results_match_numpy_head"]))
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
