#!/usr/bin/env python
"""Record tests/golden/placement_stats.json: what every map of the placement matrix (tests/placement_cases.py) does to the
pool's counters, its wave count and a fingerprint of its result bytes, on one GPU.

Run it on an H100, from the repository root, with the library built:

    python tests/golden/make_placement_stats.py [--out PATH]

Record it at a commit whose placement is known to be right: tests/test_placement_stats_gpu.py then checks that later
commits place every block exactly as that one did.  The counts depend on the device's SM count (claim units shrink for
small maps until every SM gets one), which the file records.
"""
import argparse
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)


def main():
    from tests import placement_cases as P
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(HERE, P.GOLDEN))
    a = ap.parse_args()
    doc = {"sm_count": P.sm_count(), "cases": P.run_all()}
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
        json.dump(doc, fh, indent=1, sort_keys=True)
        fh.write("\n")
    print("wrote %d cases to %s" % (len(doc["cases"]), a.out))


if __name__ == "__main__":
    main()
