"""GPU: every map of the placement matrix (tests/placement_cases.py) -- each argument source and result sink a block can
take, over range, bit-packed, payload, broadcast, items, emit, fold, scan and keyed-fold bodies -- copies, launches and
produces exactly what tests/golden/placement_stats.json recorded: the same stats delta, wave count and result bytes."""
import json
import os

import pytest

from . import placement_cases as P

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", P.GOLDEN)


def test_placement_stats():
    with open(GOLDEN) as fh:
        golden = json.load(fh)
    sm = P.sm_count()
    if sm != golden["sm_count"]:
        pytest.skip("the golden was recorded on a device of %d SMs and this one has %d: claim units, and with them the "
                    "counts, depend on the SM count" % (golden["sm_count"], sm))
    assert sorted(golden["cases"]) == sorted(P.BY_ID), "the matrix and the golden list different maps"
    got = P.run_all()
    bad = []
    for cid, want in sorted(golden["cases"].items()):
        g = got[cid]
        diff = {k: (g["stats"][k], v) for k, v in want["stats"].items() if g["stats"][k] != v}
        if diff:
            bad.append("%s: stats (got, want) %s" % (cid, diff))
        if g["n_waves"] != want["n_waves"]:
            bad.append("%s: n_waves %d, want %d" % (cid, g["n_waves"], want["n_waves"]))
        if g["fingerprint"] != want["fingerprint"]:
            bad.append("%s: result bytes differ" % cid)
    assert not bad, "\n".join(bad)
