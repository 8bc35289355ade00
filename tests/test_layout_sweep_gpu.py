"""GPU: every generated layout of tests/layout_bodies.py through dispatch_record_kernel, compared bit for bit with its
NumPy restatement.  Each layout runs at n = 1, kAlign + 1, unit - 1, unit, unit + 1, 3 unit + kAlign - 1 and one size
that takes at least four waves of a 1 MiB ring (4 MiB for 4 KB emitted values); the placement (direct, result ring, shuffled, resilient, device-resident
results fetched in unaligned ranges), the chunksize and the argument buffer (contiguous, a strided field, a host buffer
at byte offset 4, device-resident at offsets 0 and 4) of each map are drawn from an RNG seeded by the layout's name, so
a failure reproduces; every assertion message names the combination."""
import ctypes
import zlib

import numpy as np
import pytest

import fiber_b200
from fiber_b200 import _abi, registry

from . import layout_bodies as LB

pytestmark = pytest.mark.gpu

SMALL_RING = 1 << 20
PLACEMENTS = {"direct": 0, "ring": _abi.FBR_VIA_RING, "shuffle": _abi.FBR_SHUFFLE, "resilient": _abi.FBR_RESILIENT,
              "device": _abi.FBR_RESULTS_ON_DEVICE}


def _pool(ring=0):
    p = fiber_b200.Pool(1, devices=[0], ring_bytes=ring)
    p.start_workers()
    return p


@pytest.fixture(scope="module")
def pool():
    p = _pool()
    yield p
    p.terminate()
    p.join()


@pytest.fixture(scope="module")
def small_pool():
    p = _pool(SMALL_RING)
    yield p
    p.terminate()
    p.join()


def _plan(b, n, chunksize, ring=0):
    p = _abi.Plan()
    _abi.check(_abi.load().fbr_plan_query(registry.spec(b.name).func_id, n, chunksize, ring, 1, 0, 132, ctypes.byref(p)))
    return p


class _Device:
    """Device buffers of one map (freed by close())."""

    def __init__(self, pool):
        self.eng, self.bufs = pool._engine, []

    def put(self, a, off):
        p = ctypes.c_void_p()
        _abi.check(self.eng.lib.fbr_device_alloc(self.eng.handle, 0, a.nbytes + 64, ctypes.byref(p)))
        self.bufs.append(p)
        _abi.check(self.eng.lib.fbr_memcpy_h2d(self.eng.handle, 0, ctypes.c_void_p(p.value + off), a.ctypes.data, a.nbytes))
        return p.value + off

    def close(self):
        for p in self.bufs:
            self.eng.lib.fbr_device_free(self.eng.handle, 0, p)


def _map(pool, b, n, flags, chunksize, args=None, arg_stride=0, block=None, streams=(), seed=11):
    """One map through the C ABI.  args: a pointer (None: range(n)); block: (pointer, bytes); streams: (values,
    offsets) host arrays.  Returns (result bytes, emitted value bytes or None, waves)."""
    spec = registry.spec(b.name)
    eng = pool._engine
    d = _abi.MapDesc()
    d.func_id, d.flags, d.n_tasks, d.chunksize, d.shuffle_seed = spec.func_id, flags, n, chunksize, seed
    if args is None:
        d.index_start, d.index_step = 0, 1
    else:
        d.args, d.arg_stride = args, arg_stride
    if block is not None:
        d.shared, d.shared_bytes = block
    seq = ctypes.c_uint64()
    if streams:
        its = (_abi.ItemsDesc * len(streams))()
        for it, (vals, offs), e in zip(its, streams, b.items):
            it.items, it.offsets, it.n_items, it.item_bytes = vals.ctypes.data, offs.ctypes.data, len(vals), e
        if len(streams) == 1:
            _abi.check(eng.lib.fbr_map_submit_items(eng.handle, ctypes.byref(d), its, ctypes.byref(seq)))
        else:
            _abi.check(eng.lib.fbr_map_submit_items_n(eng.handle, ctypes.byref(d), its, len(its), ctypes.byref(seq)))
    else:
        _abi.check(eng.lib.fbr_map_submit(eng.handle, ctypes.byref(d), ctypes.byref(seq)))
    res = _abi.Result()
    try:
        _abi.check(eng.lib.fbr_result_wait(eng.handle, seq.value, -1, ctypes.byref(res)))
        data = np.zeros(n * b.R, np.uint8)
        if flags & _abi.FBR_RESULTS_ON_DEVICE:
            # unaligned ranges first (one task, a range across 4 KB, the last task), then everything
            for lo, cnt in ((min(3, n - 1), 1), (n // 3, min(n - n // 3, 37)), (n - 1, 1), (0, n)):
                part = np.zeros(cnt * b.R, np.uint8)
                _abi.check(eng.lib.fbr_result_fetch(eng.handle, seq.value, lo, cnt, part.ctypes.data))
                data[lo * b.R:(lo + cnt) * b.R] = part
        else:
            ctypes.memmove(data.ctypes.data, res.data, data.nbytes)
        values = None
        if b.out is not None:
            nv = int(data.view(np.uint64)[-1]) if n else 0
            values = np.zeros(nv * b.out[0], np.uint8)
            if flags & _abi.FBR_RESULTS_ON_DEVICE:
                if nv:
                    _abi.check(eng.lib.fbr_result_fetch_values(eng.handle, seq.value, 0, nv, values.ctypes.data))
            else:
                vp, cnt = ctypes.c_void_p(), ctypes.c_uint64()
                _abi.check(eng.lib.fbr_result_values(eng.handle, seq.value, ctypes.byref(vp), ctypes.byref(cnt)))
                assert cnt.value == nv
                if nv:
                    ctypes.memmove(values.ctypes.data, vp.value, values.nbytes)
        return data, values, res.n_waves
    finally:
        _abi.check(eng.lib.fbr_result_release(eng.handle, seq.value))


def _counts(rng, n, E, big=None):
    """Items per task: many empty tasks, short ones, and (big) one task at index big[0] with big[1] items."""
    c = rng.integers(0, 9 if E < 4096 else 3, n)
    c[rng.random(n) < 0.3] = 0
    if big is not None:
        c[big[0]] = big[1]
    return c


def _run(pool, b, n, place, chunksize, argmode, rng, what, big=None, block_elems=None):
    """Map layout b over n tasks with the given combination and compare with the restatement."""
    flags = PLACEMENTS[place]
    dev = _Device(pool)
    try:
        args = ptr = None
        stride = 0
        if b.index:
            args = rng.integers(-2 ** 40, 2 ** 40, n, dtype=np.int64) if argmode == "host" else np.arange(n, dtype=np.int64)
            if argmode == "host":
                ptr, stride = args.ctypes.data, 8
        elif b.A:
            args = LB.make_args(b, n, int(rng.integers(2 ** 31)))
            stride = b.A
            if argmode == "strided":
                wide = np.zeros(n, [("rec", args.dtype), ("pad", "<u4")])
                wide["rec"] = args
                ptr, stride = wide.ctypes.data, wide.itemsize
            elif argmode == "offset4":
                raw = np.zeros(n * b.A + 16, np.uint8)
                raw[4:4 + n * b.A] = args.view(np.uint8)
                ptr = raw.ctypes.data + 4
            elif argmode in ("dev0", "dev4"):
                ptr = dev.put(np.ascontiguousarray(args), 4 if argmode == "dev4" else 0)
                flags |= _abi.FBR_ARGS_DEVICE
            else:
                ptr = args.ctypes.data
        block = blk = None
        if b.shared:
            E, stage = b.shared
            n_el = int(rng.choice(_block_sizes(E, stage))) if block_elems is None else block_elems
            blk = LB.make_block(b, n_el, int(rng.integers(2 ** 31)))
            block = (blk.ctypes.data, blk.nbytes)
            if flags & _abi.FBR_ARGS_DEVICE:                # the block is a device pointer too, at the arguments' offset
                block = (dev.put(blk, 4 if argmode == "dev4" else 0), blk.nbytes)
        streams = []
        for k, E in enumerate(b.items):
            first = int(rng.integers(0, 5))
            streams.append(LB.make_items(E, _counts(rng, n, E, big if k == 0 else None), int(rng.integers(2 ** 31)), first))
        data, values, waves = _map(pool, b, n, flags, chunksize, ptr, stride, block, streams)
        if b.out is None:
            want = LB.results_np(b, n, 0, args, blk, streams)
            ok = np.array_equal(data.view(np.uint32).reshape(n, -1), want)
            if not ok:
                bad = np.nonzero((data.view(np.uint32).reshape(n, -1) != want).any(axis=1))[0]
                what += " first bad tasks %s of %d" % (bad[:8].tolist(), len(bad))
            assert ok, what
        else:
            ends, vals = LB.emit_np(b, n, 0, args, blk, streams)
            assert np.array_equal(data.view(np.uint64), ends), what + " (end offsets)"
            assert np.array_equal(values, np.ascontiguousarray(vals).view(np.uint8)), what + " (values)"
        return waves
    finally:
        dev.close()


def _block_sizes(E, stage):
    """Broadcast blocks (in elements) just under, at and just over the body's stage, and sizes not a multiple of 16."""
    at = stage // E
    sizes = {1, 3, 5, at - 1, at, at + 1} if stage else {1, 3, 5, 4096 // E + 1}
    return sorted(s for s in sizes if s >= 1)


def _arg_modes(b):
    if b.index:
        return ["range", "host"]
    if b.items or b.out is not None:
        return ["host", "strided"] if b.A else ["none"]
    return ["host", "strided", "offset4", "dev0", "dev4"]


def _placements(b):
    if b.fault:
        return ["resilient"]
    return ["direct", "ring", "shuffle", "resilient", "device"]


def _bytes_per_task(b):
    """A low estimate of the staged bytes of one task: its records, its items (_counts: about 2.8 elements, 0.7 of
    4096 bytes) and its emitted values."""
    per = max(b.A, b.R) + sum(e // 2 if e == 4096 else 2 * e for e in b.items)
    if b.out is not None:
        per += b.out[0] * b.out[1] // (4 if b.group == 1 else 8)
    return per


@pytest.mark.parametrize("name", [b.name for b in LB.LAYOUTS])
def test_layout(pool, small_pool, name):
    b = LB.BY_NAME[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    modes, places = _arg_modes(b), _placements(b)
    kinds = [lambda u: 1, lambda u: b.k_align + 1, lambda u: u - 1, lambda u: u, lambda u: u + 1,
             lambda u: 3 * u + b.k_align - 1]
    for kind in kinds:
        cs = int(rng.choice([1, 3, 7, 0]))
        unit = _plan(b, 10 ** 6, cs).unit_tasks
        n = kind(unit)
        place, mode = str(rng.choice(places)), str(rng.choice(modes))
        if n < 1:
            continue
        _run(pool, b, n, place, cs, mode, rng, "%s n=%d unit=%d chunksize=%d %s args=%s" % (name, n, unit, cs, place, mode))
    if b.shared:                                    # every block size next to the stage, at n = unit + 1
        for n_el in _block_sizes(*b.shared):
            cs = int(rng.choice([1, 3, 7, 0]))
            n = _plan(b, 10 ** 6, cs).unit_tasks + 1
            place, mode = str(rng.choice(places)), str(rng.choice(modes))
            _run(pool, b, n, place, cs, mode, rng, "%s n=%d chunksize=%d %s args=%s block=%d elements" % (name, n, cs, place, mode, n_el),
                 block_elems=n_el)
    # at least four waves of a 1 MiB ring through the result ring (resilient for the fault variants)
    # (4 MiB for 4 KB values: a claim unit of up to 3 of them per task must fit a staging half)
    place = "resilient" if b.fault else "ring"
    ring = 4 * SMALL_RING if b.out is not None and b.out[0] >= 4096 else SMALL_RING
    n = min(8 * ring // _bytes_per_task(b) + 3, 1 << 21)
    mode = modes[0]                                 # host arguments (or range()): their staging cuts waves too
    what = "%s n=%d chunksize=0 %s args=%s ring=%d" % (name, n, place, mode, ring)
    p = small_pool if ring == SMALL_RING else _pool(ring)
    try:
        waves = _run(p, b, n, place, 0, mode, rng, what)
    finally:
        if p is not small_pool:
            p.terminate()
            p.join()
    assert waves >= 4, what + " waves=%d" % waves


@pytest.mark.parametrize("name", ["it_u1", "it_h12_u8", "em_mix_g8"])
def test_items_staging_half(small_pool, name):
    """The last task, alone in its claim unit, carries as many items as a staging half holds next to its 256 B-rounded
    offsets header, after many short and empty tasks."""
    b = LB.BY_NAME[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()) + 1)
    unit = _plan(b, 5000, 0, SMALL_RING).unit_tasks
    n = 3 * unit + 1
    assert _plan(b, n, 0, SMALL_RING).unit_tasks == unit
    big = (SMALL_RING - 256) // b.items[0]
    _run(small_pool, b, n, "direct", 0, _arg_modes(b)[0], rng, "%s n=%d big=%d" % (name, n, big), big=(n - 1, big))


def test_emit_all_empty_and_many_scan_tiles(pool):
    """Index maps over negative indices push nothing; 3 scan tiles (2048 counts each) plus a partial one, placed every way."""
    for b in (LB.BY_NAME["em_o2"], LB.BY_NAME["em_o4_g32"]):
        for place in ("direct", "ring", "device"):
            n = 3 * 2048 + 77
            args = -np.arange(1, n + 1, dtype=np.int64)
            data, values, _ = _map(pool, b, n, PLACEMENTS[place], 0, args.ctypes.data, 8)
            assert not data.view(np.uint64).any() and len(values) == 0, (b.name, place)
            args = np.arange(n, dtype=np.int64) * 7919
            ends, vals = LB.emit_np(b, n, 0, args)
            data, values, _ = _map(pool, b, n, PLACEMENTS[place], 0, args.ctypes.data, 8)
            assert np.array_equal(data.view(np.uint64), ends) and np.array_equal(values, vals.view(np.uint8)), (b.name, place)


def _smallest_ring(b):
    """The smallest ring_bytes a map of b through the result ring with host arguments is accepted on: the units_cap
    arithmetic of the wave planner (ring / slot_stride and ring / (unit * arg_stride) at least 1), with the unit the
    planner picks for that ring."""
    for ring in range(4096, 1 << 22, 4096):
        p = _plan(b, 10 ** 4, 0, ring)
        if ring // p.slot_stride >= 1 and ring // (p.unit_tasks * b.A) >= 1 and ring // (p.unit_tasks * b.R) >= 1:
            return ring
    raise AssertionError(b.name)


def test_ring_too_small_is_refused_then_the_pool_goes_on():
    big, small = LB.BY_NAME["lay_a32768_r32768_g32"], LB.BY_NAME["lay_a4_r4"]
    p = _pool(4096)
    try:
        args = LB.make_args(big, 3, 1)
        with pytest.raises(_abi.EngineError, match=r"ring_bytes=4096 too small for one claim unit of 1 tasks"):
            _map(p, big, 3, _abi.FBR_VIA_RING, 0, args.ctypes.data, big.A)
        rng = np.random.default_rng(5)
        _run(p, small, 5000, "ring", 0, "host", rng, "lay_a4_r4 after a refused map")
    finally:
        p.terminate()
        p.join()


@pytest.mark.parametrize("name", ["lay_a2052_r2052", "lay_a32768_r32768_g32", "lay_a4092_r4"])
def test_smallest_accepted_ring(name):
    b = LB.BY_NAME[name]
    ring = _smallest_ring(b)
    rng = np.random.default_rng(9)
    if ring > 4096:
        p = _pool(ring - 4096)
        try:
            args = LB.make_args(b, 50, 1)
            with pytest.raises(_abi.EngineError, match="too small for one claim unit"):
                _map(p, b, 50, _abi.FBR_VIA_RING, 0, args.ctypes.data, b.A)
        finally:
            p.terminate()
            p.join()
    p = _pool(ring)
    try:
        waves = _run(p, b, 50, "ring", 0, "host", rng, "%s ring=%d" % (name, ring))
        assert waves > 1
    finally:
        p.terminate()
        p.join()
