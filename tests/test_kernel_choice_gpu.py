"""GPU: every case of the kernel choice table (tests/kernel_choice_cases.py) -- each gather kernel (flat, rows, TMA bulk)
and payload dispatch kernel at the edges of its index arithmetic, reached through the map flags and the per-call
environment knobs -- compared byte for byte with the plain restatement (NumPy for the layout bodies, the C oracle for pi
and the payload bodies, and the oracle's sum), with the stats confirming the placement path."""
import pytest

import fiber_b200

from . import kernel_choice_cases as K

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pools():
    """One-worker pools by ring size, created on first use."""
    made = {}

    def get(ring):
        if ring not in made:
            made[ring] = fiber_b200.Pool(1, devices=[0], ring_bytes=ring)
            made[ring].start_workers()
        return made[ring]
    yield get
    for p in made.values():
        p.terminate()
        p.join()


@pytest.mark.parametrize("cid", [c.id for c in K.CASES])
def test_case(pools, cid):
    c = K.BY_ID[cid]
    kernel = K.kernel_of(c)
    bad, waves, st = K.run_case(pools(c.ring), c)
    bad += K.check_stats(c, kernel, waves, st)
    if c.cell == "rows/resilient_lost" and c.waves:
        if not st["units_redispatched"] > 0:
            bad.append("no unit was lost and re-dispatched")
    assert not bad, "%s (%s): %s" % (cid, kernel, "; ".join(bad))

