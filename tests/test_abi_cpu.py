"""CPU: the C-ABI library loads, exports exactly what include/fiber_b200.h declares, describes its
device bodies, and refuses to run without a GPU (no CPU fallback).  Plus the host-side logic that
needs no device: record encoders, the callable registry, Pool argument validation."""
import ctypes
import os
import re

import numpy as np
import pytest

import fiber_b200
from fiber_b200 import _abi, registry

from . import workloads as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gpu_present():
    n = ctypes.c_int(0)
    return _abi.load().fbr_device_count(ctypes.byref(n)) == 0 and n.value > 0


def test_library_exports_every_declared_symbol():
    header = open(os.path.join(ROOT, "include", "fiber_b200.h")).read()
    declared = sorted(set(re.findall(r"^(?:int|const char\*)\s+(fbr_\w+)\s*\(", header, flags=re.M)))
    assert declared == sorted(_abi.SYMBOLS), set(declared) ^ set(_abi.SYMBOLS)
    lib = ctypes.CDLL(_abi.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), name
    assert _abi.load().fbr_abi_version() == _abi.FBR_ABI_VERSION == int(re.search(r"#define FBR_ABI_VERSION (\d+)", header).group(1))


def test_header_constants_match_binding():
    header = open(os.path.join(ROOT, "include", "fiber_b200.h")).read()
    for name in ("FBR_STARMAP", "FBR_APPLY", "FBR_ARGS_DEVICE", "FBR_OUT_DEVICE", "FBR_WANT_SUM", "FBR_SHUFFLE",
                 "FBR_FULL_WINDOW", "FBR_SHARED_HANDLE", "FBR_POOL_TIMING", "FBR_BODY_INDEX_ARG", "FBR_BODY_SUMMABLE"):
        m = re.search(r"#define %s (0x[0-9a-fA-F]+)u" % name, header)
        assert m and int(m.group(1), 16) == getattr(_abi, name), name
    for name in ("FBR_EINVAL", "FBR_ESTATE", "FBR_ETASK", "FBR_ENODEV", "FBR_ENOENT"):
        m = re.search(r"%s = (-\d+)" % name, header)
        assert m and int(m.group(1)) == getattr(_abi, name), name
    # struct sizes the C side static_asserts / the binding mirrors
    assert ctypes.sizeof(_abi.MapDesc) == 104 and ctypes.sizeof(_abi.Result) == 80 and ctypes.sizeof(_abi.Stats) == 136 and ctypes.sizeof(_abi.BodyInfo) == 64


def test_body_table():
    names = fiber_b200.body_names()
    assert set(names) >= {"square_i64", "mul2_i64", "square_scale_i64", "identity_i64", "pi_inside_det", "parzen_f32",
                          "parzen_f64", "payload_map_4k", "payload_checksum_4k", "sleep_f64", "fault_identity_i64"}
    s = registry.spec("pi_inside_det")
    assert (s.arg_bytes, s.result_bytes, s.result_kind) == (8, 1, _abi.FBR_RES_BOOL)
    assert s.flags & _abi.FBR_BODY_INDEX_ARG and s.flags & _abi.FBR_BODY_SUMMABLE
    s = registry.spec("payload_map_4k")
    assert (s.arg_bytes, s.result_bytes) == (4096, 4096) and s.result_dtype() == (np.dtype(np.uint32), (1024,))
    fid = ctypes.c_int(-1)
    lib = _abi.load()
    assert lib.fbr_body_lookup(b"parzen_f64", ctypes.byref(fid)) == 0 and fid.value == registry.spec("parzen_f64").func_id
    assert lib.fbr_body_lookup(b"no_such_body", ctypes.byref(fid)) == _abi.FBR_ENOENT
    assert b"no_such_body" in lib.fbr_last_error()
    with pytest.raises(KeyError):
        registry.spec("no_such_body")


@pytest.mark.skipif(_gpu_present(), reason="checks the no-GPU failure mode")
def test_no_gpu_means_hard_failure_not_cpu_fallback():
    lib = _abi.load()
    h = ctypes.c_void_p()
    rc = lib.fbr_pool_create(1, None, 0, 0, ctypes.byref(h))
    assert rc == _abi.FBR_ENODEV and not h.value
    pool = fiber_b200.Pool(2)
    with pytest.raises(_abi.EngineError) as ei:
        pool.map(W.f, [1, 2, 3])
    assert ei.value.status == _abi.FBR_ENODEV


def test_missing_library_is_a_hard_error(monkeypatch):
    monkeypatch.setattr(_abi, "_lib", None)
    monkeypatch.setattr(_abi, "LIB_PATH", "/nonexistent/libfiber_b200.so")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        _abi.load()


# ---- host logic: registry + encoders (what replaces pickling, fiber/pool.py:961,1181) -----------------
def test_registry_binding_and_meta():
    assert registry.body_name_of(W.f) == "square_i64"
    assert W.f.__fiber_meta__ == {"gpu": 1}                      # fiber/meta.py:53-56 storage attribute

    @fiber_b200.meta(cpu=4, memory=1000, gpu=1)
    def g():
        pass
    assert g.__fiber_meta__ == {"cpu": 4, "mem": 1000, "gpu": 1}  # memory -> mem (fiber/meta.py:19-25)
    with pytest.raises(AssertionError):
        fiber_b200.meta(disk=1)
    with pytest.raises(TypeError, match="no CPU fallback"):
        registry.body_name_of(W.unbound)
    with pytest.raises(TypeError):
        registry.body_name_of(print)
    with pytest.raises(KeyError):
        fiber_b200.bind(lambda x: x, "not_a_body")
    fiber_b200.bind(abs, "identity_i64")                          # builtins cannot carry attributes
    assert registry.body_name_of(abs) == "identity_i64"


def test_encoders_unary():
    s = registry.spec("square_i64")
    e = s.encode_map(range(5, 500, 7))
    assert (e.n, e.arg_stride, e.index_start, e.index_step, e.args) == (71, 0, 5, 7, None)
    e = s.encode_map([3, -4, 5])
    assert e.arg_stride == 8 and e.args.dtype == np.int64 and e.args.tolist() == [3, -4, 5]
    e = s.encode_starmap([(x,) for x in range(4)])
    assert e.args.tolist() == [0, 1, 2, 3]
    e = s.encode_apply((42,), {})
    assert e.n == 1 and e.args.tolist() == [42]
    assert s.encode_map([]).n == 0
    with pytest.raises(OverflowError):
        s.encode_map([2 ** 70])
    with pytest.raises(TypeError):
        s.encode_map([1.5])
    with pytest.raises(TypeError):
        s.encode_starmap([(1, 2)])
    with pytest.raises(TypeError):
        s.encode_apply((1,), {"y": 2})


def test_encoders_binary_and_kwds():
    s = registry.spec("square_scale_i64")
    assert s.encode_apply((36,), {"y": 2}).args.tolist() == [[36, 2]]       # tests/test_pool.py:115
    assert s.encode_apply((36,), {}).args.tolist() == [[36, 1]]             # default y=1
    assert s.encode_starmap([(3,), (4, 5)]).args.tolist() == [[3, 1], [4, 5]]
    m = registry.spec("mul2_i64")
    assert m.encode_starmap([(x, x) for x in range(3)]).args.tolist() == [[0, 0], [1, 1], [2, 2]]
    with pytest.raises(TypeError):
        m.encode_starmap([(1,)])
    with pytest.raises(TypeError):
        m.encode_apply((1, 2), {"y": 3})


def test_encoder_parzen_shared_block():
    from oracle import bodies as B
    xs, px, widths = B.parzen_example_inputs()
    s = registry.spec("parzen_f32")
    e = s.encode_starmap([(xs, px, w) for w in widths])
    assert e.n == 102 and e.arg_stride == 8 and e.args.tolist() == [float(w) for w in widths]
    hdr = np.frombuffer(e.shared[:80], dtype=s.HEADER)[0]
    assert (hdr["n_samples"], hdr["dims"], hdr["power"], hdr["elem_bytes"]) == (10000, 2, 1, 4)
    assert len(e.shared) == 80 + 10000 * 2 * 4
    assert np.array_equal(np.frombuffer(e.shared[80:], dtype=np.float32).reshape(10000, 2), xs.astype(np.float32))
    e64 = registry.spec("parzen_f64").encode_apply((xs, px, 0.5), {})
    assert len(e64.shared) == 80 + 10000 * 2 * 8
    with pytest.raises(ValueError):                   # reference: ambiguous truth value for p != 1
        s.encode_apply((xs, np.zeros((2, 2)), 0.5), {})
    with pytest.raises(ValueError):
        s.encode_starmap([(xs, px, 0.1), (xs[:100], px, 0.2)])


def test_encoder_parzen_empty_samples_divide_by_zero():
    """The reference divides k_n by len(x_samples): an empty sample set raises ZeroDivisionError, on the encoder's
    side here, before any block is built or any task runs (the kernel would compute 0.0 / 0.0)."""
    from oracle import bodies as B
    px = np.array([[0.1], [0.2], [0.3]])
    with pytest.raises(ZeroDivisionError):
        B.parzen_estimation(np.zeros((0, 3)), px, 0.5)
    for name in ("parzen_f64", "parzen_f32"):
        s = registry.spec(name)
        with pytest.raises(ZeroDivisionError, match="division by zero"):
            s.encode_apply((np.zeros((0, 3)), px, 0.5), {})
        with pytest.raises(ZeroDivisionError):
            s.encode_starmap([(np.zeros((0, 3)), px, w) for w in (0.5, 1.0)])
        with pytest.raises(ZeroDivisionError):
            s.shared_block(np.zeros((0, 3)), px)
        assert len(s.encode_apply((np.zeros((1, 3)), px, 0.5), {}).shared) == 80 + 3 * s.elem.itemsize


def test_encoder_payload():
    from oracle import cref
    recs = cref.payload_records(10, 4)
    s = registry.spec("payload_map_4k")
    e = s.encode_map(recs)
    assert (e.n, e.arg_stride, e.task_index_base) == (4, 4096, 0) and e.args.ctypes.data == recs.ctypes.data
    e = s.encode_starmap([(10 + i, recs[i]) for i in range(4)])
    assert e.task_index_base == 10 and np.array_equal(e.args, recs)
    with pytest.raises(ValueError):
        s.encode_starmap([(0, recs[0]), (2, recs[1])])
    with pytest.raises(TypeError):
        s.encode_map(np.zeros((3, 100), dtype=np.uint32))


def test_pool_argument_validation_without_device():
    with pytest.raises(NotImplementedError):
        fiber_b200.Pool(2, initializer=print)
    with pytest.raises(ValueError):
        fiber_b200.Pool(0)
    p = fiber_b200.Pool()                                    # processes=None -> 1 (fiber/pool.py:894)
    assert p._processes == 1
    with pytest.raises(NotImplementedError):
        p.map_async(W.f, [1], error_callback=print)           # fiber/pool.py:1162-1164
    with pytest.raises(TypeError):
        p.map(W.unbound, [1])                                 # rejected before any device work
    p.close()
    with pytest.raises(ValueError, match="Pool is not running"):
        p.map(W.f, [1, 2, 3])                                 # fiber/pool.py:1166-1167
    with pytest.raises(ValueError):
        p.apply_async(W.f, (1,))
    with pytest.raises(ValueError):
        p.starmap(W.f, [(1,)])
    p.join()
    assert fiber_b200.active_children() == []


def test_affinity_helpers_degrade_gracefully():
    """No NVML / no GPU: device_cpus is empty and bind_to_device leaves the process untouched."""
    import os
    from fiber_b200 import affinity
    before = os.sched_getaffinity(0)
    cpus = affinity.device_cpus(0)
    assert isinstance(cpus, list)
    if not cpus:
        assert affinity.bind_to_device(0) == [] and os.sched_getaffinity(0) == before
    p = fiber_b200.Pool(1, bind_cpu=True, results="device", express=False)
    assert p.bound_cpus == [] and p._results_on_device and not p._use_express


def test_express_and_queue_symbols_need_a_gpu_to_start():
    lib = _abi.load()
    if _gpu_present():
        pytest.skip("checks the no-GPU failure mode")
    x = ctypes.c_void_p()
    assert lib.fbr_express_create(0, 0, ctypes.byref(x)) == _abi.FBR_ENODEV
    assert b"no CPU fallback" in lib.fbr_express_last_error()


def _plan(body, n, cs=0, ring=0, nw=1, w=0, sms=132):
    p = _abi.Plan()
    _abi.check(_abi.load().fbr_plan_query(registry.spec(body).func_id, n, cs, ring, nw, w, sms, ctypes.byref(p)))
    return p


def test_claim_unit_planning_rules():
    """Host logic of fbr_map_submit without a device: claim units vs the reference's chunk plan."""
    from oracle.zpool_port import chunk_plan
    # default chunksize 32 (fiber/pool.py:1169-1170): every reference chunk lies inside one claim unit
    for body, n in (("pi_inside_det", 10 ** 8), ("square_i64", 10 ** 6), ("payload_map_4k", 10 ** 6), ("payload_checksum_4k", 10 ** 5)):
        p = _plan(body, n)
        spec = registry.spec(body)
        assert p.unit_tasks % 32 == 0 and p.block_first == 0 and p.block_count == n
        assert p.slot_stride % 16 == 0 and p.slot_stride == p.unit_tasks * spec.result_bytes
        assert p.n_units == -(-n // p.unit_tasks)
        for start, count in chunk_plan(min(n, 50000))[::97]:
            assert start // p.unit_tasks == (start + count - 1) // p.unit_tasks
    assert _plan("pi_inside_det", 10 ** 8).unit_tasks == 4096 and _plan("payload_map_4k", 10 ** 6).unit_tasks == 32
    # odd chunk sizes keep slots 16-byte aligned (unit is a multiple of lcm(chunksize, 16/R))
    for cs in (1, 3, 7, 100, 1000):
        p = _plan("pi_inside_det", 10 ** 7, cs)
        assert p.unit_tasks % 16 == 0 and (cs > 4096 or p.unit_tasks % cs == 0)
        p = _plan("square_i64", 10 ** 6, cs)
        assert (p.unit_tasks * 8) % 16 == 0
    # one-task bodies dispatch task by task (tests/test_pool.py:179-234: chunksize 1 must not batch)
    assert _plan("parzen_f64", 102, 1).unit_tasks == 1 and _plan("sleep_f64", 9, 1).unit_tasks == 1
    # small maps shrink the unit so the work still spreads over the SMs; tiny rings clamp it
    assert _plan("pi_inside_det", 20000).unit_tasks < 4096
    p = _plan("payload_map_4k", 1000, ring=64 << 10)
    assert p.unit_tasks * 4096 <= 64 << 10
    # contiguous, complete, unit-aligned blocks per worker (PUSH round-robin with chunk = block)
    n = 10 ** 6
    blocks = [_plan("payload_map_4k", n, nw=8, w=w) for w in range(8)]
    assert blocks[0].block_first == 0 and sum(b.block_count for b in blocks) == n
    assert all(blocks[i].block_first + blocks[i].block_count == blocks[i + 1].block_first for i in range(7))
    assert all(b.block_first % 32 == 0 for b in blocks)
    assert _abi.load().fbr_plan_query(999, 1, 0, 0, 1, 0, 0, ctypes.byref(_abi.Plan())) == _abi.FBR_EINVAL


def test_bits_body_and_bit_backed_result_array():
    """pi_inside_bits8 is in the body table; a bit-backed ResultArray behaves like the list of bools."""
    from fiber_b200.pool import ResultArray
    s = registry.spec("pi_inside_bits8")
    assert (s.result_bytes, s.result_kind) == (1, _abi.FBR_RES_BITS8)
    assert s.flags & _abi.FBR_BODY_INDEX_ARG and s.flags & _abi.FBR_BODY_SUMMABLE and s.arg_bytes == 64
    assert registry.BITS_TWIN["pi_inside_det"] == "pi_inside_bits8"
    e = s.encode_range(range(3, 1003, 5))
    assert (e.n, e.arg_stride, e.index_start, e.index_step, e.n_items) == (25, 0, 3, 5, 200)
    # explicit arguments: 8 int64 items per byte-task, the map's item count travels in n_items
    base = registry.spec("pi_inside_det")
    e = s.from_encoded(base.encode_map([5, 6, 7, 8, 9, 10, 11, 12, 13]))
    assert (e.n, e.arg_stride, e.n_items) == (2, 64, 9) and e.args.tolist() == list(range(5, 14))
    e = s.from_encoded(base.encode_starmap([(x,) for x in range(16)]))
    assert (e.n, e.arg_stride, e.n_items) == (2, 64, 16)
    e = s.from_encoded(base.encode_map(range(10, 110)))
    assert (e.n, e.arg_stride, e.index_start, e.n_items) == (13, 0, 10, 100)
    assert s.encode_range(range(0)).n == 0 and s.encode_range(range(8)).n == 1 and s.encode_range(range(9)).n == 2
    with pytest.raises(TypeError):
        s.encode_range([1, 2, 3])
    rng = np.random.default_rng(5)
    for n in (1, 7, 8, 9, 1000, 65537):
        want = rng.integers(0, 2, n).astype(bool)
        ra = ResultArray(registry.spec("pi_inside_det"), None, None, n=n, bits=np.packbits(want, bitorder="little"))
        assert len(ra) == n and ra.tolist() == want.tolist() and ra == want.tolist() and ra.sum() == int(want.sum())
        assert ra[0] == bool(want[0]) and ra[-1] == bool(want[-1]) and ra[n // 2] == bool(want[n // 2])
        assert ra[1:n - 1] == want[1:n - 1].tolist() and ra[::3] == want[::3].tolist()
        assert list(ra) == want.tolist() and np.array_equal(np.asarray(ra), want)
        with pytest.raises(IndexError):
            ra[n]


def test_out_of_tree_body_registration():
    """fbr_register_body: a body module compiled outside the library is loaded, ABI-checked and appended to
    the body table (no device needed for that); its encoders follow the declared argument layout."""
    from . import device_bodies as D
    lib = _abi.load()
    n = ctypes.c_int(0)
    assert lib.fbr_body_count(ctypes.byref(n)) == 0 and n.value >= 16
    s = registry.spec("collatz_steps")
    assert s.func_id >= 13 and (s.arg_bytes, s.result_bytes, s.result_kind) == (8, 8, _abi.FBR_RES_I64)
    assert s.flags & _abi.FBR_BODY_INDEX_ARG and registry.body_name_of(D.collatz_steps) == "collatz_steps"
    assert s.encode_map(range(1, 10)).arg_stride == 0 and s.encode_map([3, 4]).args.tolist() == [3, 4]
    b = registry.spec("odd_bits")
    assert (b.arg_bytes, b.result_bytes, b.result_kind) == (8, 1, _abi.FBR_RES_BOOL)
    t = registry.spec("odd_bits_bits8")                   # the module's bit-packed twin, registered with it
    assert (t.arg_bytes, t.result_bytes, t.result_kind) == (64, 1, _abi.FBR_RES_BITS8) and registry.BITS_TWIN["odd_bits"] == "odd_bits_bits8"
    assert registry.module_of("odd_bits")[3] == "odd_bits_bits_entry"
    fid = ctypes.c_int(-1)
    assert lib.fbr_body_lookup(b"odd_bits", ctypes.byref(fid)) == 0 and fid.value == b.func_id
    assert lib.fbr_register_body(b"x", b"/nonexistent.so", b"e", ctypes.byref(fid)) == _abi.FBR_ENOENT
    # a compiled-in name cannot be taken over by a module
    from fiber_b200 import bodies
    so = bodies.compile_module("collatz_steps", D.COLLATZ_SRC)
    assert lib.fbr_register_body(b"square_i64", so.encode(), b"fbr_body_entry", ctypes.byref(fid)) == _abi.FBR_EINVAL
    with pytest.raises(RuntimeError, match="nvcc failed"):
        bodies.compile_module("broken", "#include \"fiber_b200_body.cuh\"\nthis is not CUDA\n")


def test_initializer_binding_and_result_layout_options():
    with pytest.raises(NotImplementedError):
        fiber_b200.Pool(1, initializer=print)
    p = fiber_b200.Pool(1, initializer=W.set_parzen_samples, initargs=(np.zeros((4, 2)), np.zeros((2, 1))))
    assert p._initializer.__fbr_init_body__ == "parzen_f64"
    for mode in ("host", "bytes", "bits", "device"):
        fiber_b200.Pool(1, results=mode)
    with pytest.raises(ValueError):
        fiber_b200.Pool(1, results="disk")
    # parzen items may carry only h (samples from the initializer block) -- but not a mix
    s = registry.spec("parzen_f64")
    e = s.encode_map([0.1, 0.2])
    assert e.shared is None and e.args.tolist() == [0.1, 0.2]
    e = s.encode_starmap([(0.5,), (0.7,)])
    assert e.shared is None and e.n == 2
    xs, px = np.zeros((4, 2)), np.zeros((2, 1))
    with pytest.raises(TypeError):
        s.encode_starmap([(0.5,), (xs, px, 0.7)])


def test_parzen_block_cache_and_isolation_argument():
    """The parzen encoder re-uses the broadcast block of the previous call when the arrays compare equal (the example
    issues 102 apply_async calls with the same 160 KB array) and rebuilds it when they do not; Pool validates `isolation`."""
    s = registry.spec("parzen_f32")
    xs, px = np.random.default_rng(0).standard_normal((500, 2)), np.zeros((2, 1))
    b1 = s.shared_block(xs, px)
    assert s.shared_block(xs.copy(), px.copy()) is b1             # equal content: the very same bytes object
    xs2 = xs.copy()
    xs2[17, 1] += 1.0
    b2 = s.shared_block(xs2, px)
    assert b2 is not b1 and b2 != b1 and len(b2) == len(b1) == 80 + 500 * 2 * 4
    assert s.shared_block(xs, px) == b1                            # and back again (rebuilt, same content)
    e = s.encode_apply((xs, px, 0.5), {})
    assert e.n == 1 and e.shared is s.shared_block(xs, px)
    with pytest.raises(ValueError, match="isolation"):
        fiber_b200.Pool(2, isolation="container")
    p = fiber_b200.Pool(2, error_handling=True, isolation="process")
    assert p._isolation == "process" and p._proc is None          # worker processes start lazily, like the reference's
