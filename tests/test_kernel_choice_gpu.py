"""GPU: every case of the kernel choice table (tests/kernel_choice_cases.py) -- each gather kernel (flat, rows, TMA bulk)
and payload dispatch kernel at the edges of its index arithmetic, reached through the map flags and the per-call
environment knobs -- compared byte for byte with the plain restatement (NumPy for the layout bodies, the C oracle for pi
and the payload bodies, and the oracle's sum), with the stats confirming the placement path.  The knobs read once per
process (FBR_DIRECT, FBR_RECORDS, FBR_ZERO_COPY, FBR_SERIAL_SUBMIT, FBR_DISPATCH_TMA, FBR_TMA_DEEP) are exercised in
child processes (tests/_kernel_choice_child.py)."""
import json
import os
import subprocess
import sys

import pytest

import fiber_b200

from . import kernel_choice_cases as K

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


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


# ---- knobs read once per process: one child process per setting ------------------------------------------------------
SETTINGS = {
    "baseline": {},
    "dispatch_tma_0": {"FBR_DISPATCH_TMA": "0"},
    "tma_deep_1": {"FBR_TMA_DEEP": "1"},
    "direct_0": {"FBR_DIRECT": "0"},
    "records_1": {"FBR_RECORDS": "1"},
    "zero_copy_0": {"FBR_ZERO_COPY": "0"},
    "serial_submit_1": {"FBR_SERIAL_SUBMIT": "1"},
    "direct_0_records_1": {"FBR_DIRECT": "0", "FBR_RECORDS": "1"},
}


def _child(env):
    e = {k: v for k, v in os.environ.items() if not k.startswith("FBR_")}
    e.update(env)
    r = subprocess.run([sys.executable, "-m", "tests._kernel_choice_child"], cwd=ROOT, env=e, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.fixture(scope="module")
def baseline():
    return _child({})


@pytest.mark.parametrize("setting", sorted(SETTINGS))
def test_static_knob_in_child(baseline, setting):
    out = baseline if setting == "baseline" else _child(SETTINGS[setting])
    failed = {k: v for k, v in out["cases"].items() if v != "ok"}
    assert not failed, (setting, failed)
    # every setting computes what the default computes, bit for bit (folds and scans included)
    assert out["digests"] == baseline["digests"], setting
    st, env = out["stats"], SETTINGS[setting]
    if env.get("FBR_DIRECT") == "0" or env.get("FBR_RECORDS") == "1":   # explicit records take every wave through the ring
        assert st["direct_waves"] == 0, st
    else:
        assert st["direct_waves"] > 0, st
    if env.get("FBR_RECORDS") == "1":
        assert out["unshuffled_records"] > 0, out      # task records on maps that are not shuffled
    else:
        assert out["unshuffled_records"] == 0, out
    # FBR_ZERO_COPY=0 has no stat of its own (d2h_bytes counts zero-copy stores and staged copies alike): the pi bits
    # of the battery, equal to the oracle's, are its check
