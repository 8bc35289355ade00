"""GPU: every map kind through both isolations and every result placement gives the same values, result types and task
counters.  Kinds: plain results (square_i64), bit-packed bool results (pi_inside_det through its bits twin), emit results
(tokens_u32 / prime_factors_i64), folds and accumulates (sum_sq_idx_u64 / pair_overlap_u32); each in its map and its star
form.  imap on a thread pool runs with a ring small enough that the map streams over several waves."""
import numpy as np
import pytest

import fiber_b200
from examples import workloads as W
from fiber_b200.pool import ResultArray

from . import emit_bodies as EB
from . import fold_bodies as FB

pytestmark = pytest.mark.gpu

RING = 1 << 20
STREAM_RING = 64 << 10
ISOLATIONS = ["thread", "process"]
RESULTS = ["host", "bytes", "device"]
KINDS = ["plain", "bits", "emit", "fold", "accumulate"]
FORMS = ["map", "star"]


def _columns(n, seed):
    rng = np.random.default_rng(seed)
    cols = []
    for _ in range(2):
        lens = rng.integers(0, 16, n)
        offs = np.zeros(n + 1, np.int64)
        np.cumsum(lens, out=offs[1:])
        vals = rng.integers(0, 30, int(offs[-1]), dtype=np.uint32)
        for i in range(n):
            vals[offs[i]:offs[i + 1]].sort()
        cols.append(fiber_b200.Ragged(vals, offs))
    return fiber_b200.Columns(*cols)


# (callable, items, empty items) per kind and form; folds and accumulates over 50 000 tasks cover two process-pool blocks
CASES = {
    ("plain", "map"): (W.f, list(range(-60_000, 60_000)), []),
    ("plain", "star"): (W.f, [(x,) for x in range(-30_000, 30_000)], []),
    ("bits", "map"): (W.is_inside, range(1_000_003), range(0)),
    ("bits", "star"): (W.is_inside, [(i,) for i in range(70_001)], []),
    ("emit", "map"): (EB.prime_factors_i64, range(2, 60_000), range(2, 2)),
    ("emit", "star"): (EB.tokens_u32, [(d,) for d in EB.documents(5_000, seed=3, empty_every=7)], []),
    ("fold", "map"): (FB.sum_sq_idx_u64, range(5, 5 + 3 * 50_000, 3), range(0)),
    ("fold", "star"): (FB.pair_overlap_u32, _columns(50_000, seed=43), []),
    ("accumulate", "map"): (FB.sum_sq_idx_u64, range(5, 5 + 3 * 50_000, 3), range(0)),
    ("accumulate", "star"): (FB.pair_overlap_u32, _columns(50_000, seed=44), []),
}


def run(pool, kind, form, items):
    f = CASES[(kind, form)][0]
    if kind == "fold":
        return pool.fold(f, items) if form == "map" else pool.starfold(f, items)
    if kind == "accumulate":
        return pool.accumulate(f, items) if form == "map" else pool.staraccumulate(f, items)
    return pool.map(f, items) if form == "map" else pool.starmap(f, items)


def plain(r):
    """(result type, values) of a map's result; a fold's value as it is."""
    return (type(r), r.tolist()) if isinstance(r, ResultArray) else (type(r), r)


@pytest.fixture(scope="module")
def pools():
    made = {}

    def get(isolation, results):
        if (isolation, results) not in made:
            if isolation in ("thread", "stream"):
                ring = RING if isolation == "thread" else STREAM_RING
                made[(isolation, results)] = fiber_b200.Pool(1, devices=[0], ring_bytes=ring, results=results)
            else:
                made[(isolation, results)] = fiber_b200.Pool(1, devices=[0], isolation="process", results=results)
        return made[(isolation, results)]
    yield get
    for p in made.values():
        p.terminate()
        p.join()


@pytest.fixture(scope="module")
def want(pools):
    cache = {}

    def get(kind, form, empty=False):
        if (kind, form, empty) not in cache:
            items = CASES[(kind, form)][2 if empty else 1]
            cache[(kind, form, empty)] = plain(run(pools("thread", "host"), kind, form, items))
        return cache[(kind, form, empty)]
    return get


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("results", RESULTS)
@pytest.mark.parametrize("isolation", ISOLATIONS)
def test_same_results(pools, want, isolation, results, kind, form):
    got = plain(run(pools(isolation, results), kind, form, CASES[(kind, form)][1]))
    assert got == want(kind, form)


@pytest.mark.parametrize("kind", ["plain", "bits", "emit"])
@pytest.mark.parametrize("results", RESULTS)
@pytest.mark.parametrize("isolation", ISOLATIONS)
def test_imap_streams_the_map(pools, want, isolation, results, kind):
    f, items, _ = CASES[(kind, "map")]
    p = pools("stream" if isolation == "thread" else isolation, results)
    assert list(p.imap(f, items)) == want(kind, "map")[1]
    assert list(p.imap_unordered(f, items, chunksize=7)) == want(kind, "map")[1]
    if isolation == "thread" and results != "device":        # results kept on the device are handed out after the map
        r = p.map_async(f, items, 1, _streaming=True)          # the map imap iterates
        assert list(r.iget_ordered()) == want(kind, "map")[1]
        assert r.n_waves > 1


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("results", RESULTS)
@pytest.mark.parametrize("isolation", ISOLATIONS)
def test_empty(pools, want, isolation, results, kind, form):
    got = plain(run(pools(isolation, results), kind, form, CASES[(kind, form)][2]))
    assert got == want(kind, form, empty=True)
    if kind != "fold":
        assert got[1] == []


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("results", RESULTS)
@pytest.mark.parametrize("isolation", ISOLATIONS)
def test_task_counters(pools, isolation, results, kind, form):
    p = pools(isolation, results)
    items = CASES[(kind, form)][1]
    sent, recv = p.sent_tasks, p.recv_tasks
    run(p, kind, form, items)
    assert p.sent_tasks - sent == len(items)
    if isolation == "thread":
        assert p.recv_tasks - recv == len(items)
