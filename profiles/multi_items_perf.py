"""Multi-stream items bodies on the H100: what a second offsets stream costs, against the workaround it replaces.

    python profiles/multi_items_perf.py [--pairs N] [--out profiles/r09_multi_items_perf.json]

Workload: N (default 8 Mi) pairs of seeded sorted uint32 lists with skewed lengths (geometric, mean about 4 and 6), the
inputs of ``intersect_count_u32``.  Device-resident items, direct placement, engine-owned pinned results; each number is
the median of 10 timed maps, over three rounds that alternate the variants, with the spread of the three medians.

  - two_streams: ``intersect_count_u32`` through fbr_map_submit_items_n, both lists as their own stream;
  - concat_one_stream: the workaround -- one stream holding a then b per task, the split point in a head record
    (``concat_intersect_count_u32`` below), the same algorithm;
  - d2d_copy: a device-to-device copy of the map's algorithmic bytes (both item arrays, both offset arrays, the results);
  - host_concat_build: the host NumPy time to build the workaround's input from the two Raggeds (not a GPU time);
  - starmap_columns_e2e: ``Pool.starmap(f, Columns(ra, rb))`` from host-resident Raggeds, end to end.

The card's name and power limit are read in the same run and written beside the numbers."""
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
from fiber_b200 import Columns, Ragged, _abi, registry  # noqa: E402

from tests import multi_items_bodies as M  # noqa: E402

CONCAT_SRC = r'''
#include "fiber_b200_body.cuh"

// the one-stream workaround: a task's items are a then b, the head record says where a ends
struct ConcatIntersectCount {
    using Item = uint32_t;
    struct Arg { uint64_t split; };
    struct Res { uint32_t common, na, nb; };
    static constexpr bool kIndexArg = false, kCanFault = false;
    __device__ static __forceinline__ void run(const Arg& s, const fbr::Items<uint32_t>& x, Res& r, uint64_t, const fbr::ErrSink&,
                                               uint32_t) {
        const fbr::Items<uint32_t> a{x.data, s.split}, b{x.data + s.split, x.n - s.split};
        uint64_t i = 0, j = 0;
        uint32_t c = 0;
        while (i < a.n && j < b.n) {
            const uint32_t p = a.data[i], q = b.data[j];
            c += p == q;
            i += p <= q;
            j += q <= p;
        }
        r.common = c; r.na = (uint32_t)a.n; r.nb = (uint32_t)b.n;
    }
};
FBR_EXPORT_RECORD_BODY(ConcatIntersectCount, "concat_intersect_count_u32", concat_entry, 0)
'''
fiber_b200.device_body("concat_intersect_count_u32", source=CONCAT_SRC, entry="concat_entry", args=[("split", "<u8")],
                       items=("ab", "<u4"), result=M.COUNT_RES)


def sorted_lists(n, seed, mean):
    rng = np.random.default_rng(seed)
    lens = np.minimum(rng.geometric(1.0 / (mean + 1), n) - 1, 64 * mean)
    offs = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=offs[1:])
    vals = rng.integers(0, 64, int(offs[-1]), dtype=np.uint32)
    task = np.repeat(np.arange(n), lens)
    vals = vals[np.lexsort((vals, task))]
    return Ragged(vals, offs)


def concat(ra, rb):
    """The workaround's input: per task a's items then b's, the new offsets and the split of each task."""
    oa, ob = np.asarray(ra.offsets, np.int64), np.asarray(rb.offsets, np.int64)
    la, lb = np.diff(oa), np.diff(ob)
    offs = np.zeros(len(la) + 1, np.int64)
    np.cumsum(la + lb, out=offs[1:])
    vals = np.empty(int(offs[-1]), ra.values.dtype)
    ta, tb = np.repeat(np.arange(len(la)), la), np.repeat(np.arange(len(lb)), lb)
    vals[offs[:-1][ta] + (np.arange(len(ta)) - oa[:-1][ta])] = ra.values
    vals[offs[:-1][tb] + la[tb] + (np.arange(len(tb)) - ob[:-1][tb])] = rb.values
    return Ragged(vals, offs), la.astype(np.uint64)


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


def run_map(pool, name, n, streams, args=None):
    """One device-resident map (direct placement) submitted and waited for: (seconds, result bytes)."""
    spec = registry.spec(name)
    eng = pool._engine
    d = _abi.MapDesc()
    d.func_id, d.flags, d.n_tasks, d.chunksize = spec.func_id, _abi.FBR_ARGS_DEVICE, n, 32
    if args is not None:
        d.args, d.arg_stride = args, 8
    its = (_abi.ItemsDesc * len(streams))()
    for it, (items, offs, n_items), dt in zip(its, streams, spec.item_dtypes):
        it.items, it.offsets, it.n_items, it.item_bytes = items, offs, n_items, dt.itemsize
    seq, res = ctypes.c_uint64(), _abi.Result()
    t0 = time.perf_counter()
    _abi.check(eng.lib.fbr_map_submit_items_n(eng.handle, ctypes.byref(d), its, len(its), ctypes.byref(seq)))
    _abi.check(eng.lib.fbr_result_wait(eng.handle, seq.value, -1, ctypes.byref(res)))
    dt = time.perf_counter() - t0
    out = np.frombuffer((ctypes.c_char * (n * spec.result_bytes)).from_address(res.data), np.uint8).copy()
    _abi.check(eng.lib.fbr_result_release(eng.handle, seq.value))
    return dt, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=8 << 20)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r09_multi_items_perf.json"))
    a = ap.parse_args()
    import torch
    n = a.pairs
    ra, rb = sorted_lists(n, 1, 4), sorted_lists(n, 2, 6)
    t0 = time.perf_counter()
    rc, split = concat(ra, rb)
    host_build = time.perf_counter() - t0
    pool = fiber_b200.Pool(1, devices=[0])
    pool.start_workers()
    dev = Device(pool)
    try:
        oa, ob, oc = (np.asarray(r.offsets).astype(np.uint64) for r in (ra, rb, rc))
        two = [(dev.put(ra.values), dev.put(oa), len(ra.values)), (dev.put(rb.values), dev.put(ob), len(rb.values))]
        one = [(dev.put(rc.values), dev.put(oc), len(rc.values))]
        dsplit = dev.put(split)
        res_bytes = n * registry.spec("intersect_count_u32").result_bytes
        alg_bytes = ra.values.nbytes + rb.values.nbytes + oa.nbytes + ob.nbytes + res_bytes
        src = torch.empty(alg_bytes, dtype=torch.uint8, device="cuda:0")
        dst = torch.empty_like(src)

        def d2d():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            dst.copy_(src)
            e1.record()
            e1.synchronize()
            return e0.elapsed_time(e1) / 1e3

        variants = {
            "two_streams": lambda: run_map(pool, "intersect_count_u32", n, two),
            "concat_one_stream": lambda: run_map(pool, "concat_intersect_count_u32", n, one, args=dsplit),
        }
        # the same results, bit for bit, from both maps (and, on a sample, from the restatement)
        _, r2 = variants["two_streams"]()
        _, r1 = variants["concat_one_stream"]()
        assert np.array_equal(r1, r2)
        k = 2000
        assert np.array_equal(r2[:k * 12].view(M.COUNT_RES), M.intersect_count_np(ra[:k], rb[:k]))
        for f in list(variants.values()) + [d2d]:      # warm-up
            f()
        rounds = {name: [] for name in list(variants) + ["d2d_copy"]}
        for _ in range(3):
            for name, f in variants.items():
                rounds[name].append(float(np.median([f()[0] for _ in range(10)])))
            rounds["d2d_copy"].append(float(np.median([d2d() for _ in range(10)])))
        # host-resident starmap over Columns, end to end
        f = M.intersect_count_u32
        e2e = []
        for _ in range(3):
            ts = []
            for _ in range(3):
                t = time.perf_counter()
                r = pool.starmap(f, Columns(ra, rb))
                ts.append(time.perf_counter() - t)
            e2e.append(float(np.median(ts)))
        assert np.array_equal(np.asarray(r).view(np.uint8).reshape(-1), r2)
        rounds["starmap_columns_e2e"] = e2e
    finally:
        dev.free()
        pool.terminate()
        pool.join()
    out = {
        "card": card(),
        "workload": {"pairs": n, "items_a": int(len(ra.values)), "items_b": int(len(rb.values)),
                     "algorithmic_bytes": int(alg_bytes), "conditions": "device-resident, direct placement, median of 10, "
                     "3 alternating rounds (starmap_columns_e2e: host-resident, median of 3 per round)"},
        "seconds": {k: {"median": float(np.median(v)), "rounds": v, "spread": float(max(v) - min(v))} for k, v in rounds.items()},
        "host_concat_build_seconds": host_build,
    }
    out["two_streams_over_concat"] = out["seconds"]["two_streams"]["median"] / out["seconds"]["concat_one_stream"]["median"]
    out["two_streams_over_d2d"] = out["seconds"]["two_streams"]["median"] / out["seconds"]["d2d_copy"]["median"]
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
