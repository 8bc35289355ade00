"""Child process of tests/test_kernel_choice_gpu.py: a fixed battery of maps under the knobs the engine reads once per
process (FBR_DIRECT, FBR_RECORDS, FBR_ZERO_COPY, FBR_SERIAL_SUBMIT, FBR_DISPATCH_TMA, FBR_TMA_DEEP), set by the parent in
this process's environment.  Prints one JSON line: "ok" or the mismatches of every case, a digest of every result that
only a restatement of the whole map's order could check (accumulate), the summed stats of its pools, and the task
records copied for maps that are not shuffled.  Exits when the battery is done; its pools are joined before it does."""
import hashlib
import json

import numpy as np

import fiber_b200
from examples import workloads as W
from oracle import cref

from . import fold_bodies as FB
from . import keyed_bodies as KB
from . import kernel_choice_cases as K

SMALL = 1 << 20


def _case(cell, body, n, ring=0, place="ring", args="host", stride=0, want_sum=False, chunksize=0):
    return K.Case(cell, body, n, chunksize, ring, {}, place, args, stride, want_sum, False)


# one map per gather kernel and payload dispatch path; "direct" maps are unshuffled, so FBR_RECORDS=1 shows on them
BATTERY = [
    _case("flat", "lay_a2052_r2052", 1001, SMALL),
    _case("flat_direct", "lay_a2052_r2052", 1001, SMALL, place="direct"),
    _case("rows", "payload_map_4k", 43, 32 << 10, chunksize=3),
    _case("bulk", "lay_a4_r4096", 803, SMALL),
    _case("bulk_direct", "lay_a4_r4096", 803, SMALL, place="direct"),
    _case("payload_tma", "payload_map_4k", 301, SMALL, place="direct"),
    _case("payload_tma_shuffled", "payload_map_4k", 97, 0, place="shuffle", args="dev"),
    _case("payload_strided", "payload_map_4k", 301, 4 << 20, place="direct", stride=8192),
    _case("payload_strided_dev", "payload_map_4k", 97, 0, place="ring", args="dev", stride=4112),
    _case("checksum_strided", "payload_checksum_4k", 3001, 4 << 20, place="direct", stride=12288, want_sum=True),
    _case("pi_rows", "pi_inside_det", 2_000_001, SMALL, args="range"),
    _case("pi_direct", "pi_inside_det", 2_000_001, SMALL, place="direct", args="range"),
]


def main():
    out = {"cases": {}, "digests": {}, "stats": {}, "unshuffled_records": 0}
    pools = {}

    def pool(ring, results="host"):
        key = (ring, results)
        if key not in pools:
            pools[key] = fiber_b200.Pool(1, devices=[0], ring_bytes=ring, results=results)
            pools[key].start_workers()
        return pools[key]

    def record(name, ok, why=""):
        out["cases"][name] = "ok" if ok else (why or "mismatch")

    try:
        for c in BATTERY:
            bad, waves, st = K.run_case(pool(c.ring), c)
            record(c.cell, not bad, "; ".join(bad))
            if c.place != "shuffle":
                out["unshuffled_records"] += st["records_copied"]
        # pi through the public API: one byte per task, and bit-packed (zero copy unless FBR_ZERO_COPY=0)
        n = 3_000_017
        ref, count = cref.pi_inside_range(0, n)
        r = pool(SMALL, "bytes").map(W.is_inside, range(n))
        record("pi_bytes", np.array_equal(np.asarray(r).view(np.uint8), ref) and r.sum() == count)
        r = pool(SMALL).map(W.is_inside, range(n))
        record("pi_bits", np.array_equal(r.packed, np.packbits(ref, bitorder="little")) and r.sum() == count)
        # fold and accumulate of moments_f64, keyed fold of class_moments_f64
        xs = np.random.default_rng(5).standard_normal(70_001) * 1e3 + 7.0
        p = pool(SMALL)
        want = FB.fold_of([FB.moments_run(x) for x in xs.tolist()], FB.moments_combine, FB.MOMENTS_ID)
        got = p.fold(FB.moments_f64, xs)
        record("fold", tuple(got) == tuple(want), "%s != %s" % (got, want))
        acc = np.ascontiguousarray(np.asarray(p.accumulate(FB.moments_f64, xs)))
        record("accumulate_last", tuple(acc[-1].tolist()) == tuple(want))
        out["digests"]["accumulate"] = hashlib.sha256(acc.tobytes()).hexdigest()
        a = np.zeros(50_003, KB.MOMENTS_ARG)
        rng = np.random.default_rng(6)
        a["x"] = rng.standard_normal(len(a)) * 1e3
        a["label"] = rng.integers(0, 37, len(a))
        want, counts = KB.keyed_tree([KB.class_moments_f64(float(x), int(k)) for x, k in zip(a["x"], a["label"])],
                                     KB.KEY_OF["class_moments_f64"], KB.moments_combine, KB.MOMENTS_ID, 37)
        try:
            r = p.fold_by_key(KB.class_moments_f64, a, 37)
            record("keyed_fold", r.tolist() == want and r.counts.tolist() == counts)
        except ValueError as e:
            record("keyed_fold", False, str(e))
        for q in pools.values():
            for k, v in q.stats().items():
                if isinstance(v, int):
                    out["stats"][k] = out["stats"].get(k, 0) + v
    finally:
        for q in pools.values():
            q.terminate()
            q.join()
    print(json.dumps(out, sort_keys=True), flush=True)


if __name__ == "__main__":
    main()
