"""Callable -> device-body registry and fixed-layout record encoders.

The reference ships the mapped callable to its workers by pickle reference and calls it there
(fiber/pool.py:961, 806-820).  A Python callable cannot execute on a GPU, so a callable has to be
*bound* to one of the device bodies compiled into libfiber_b200 (``fbr_body_lookup``).  The hook is
the one the reference already inspects when it starts workers: ``func.__fiber_meta__``
(fiber/meta.py:53-56, fiber/pool.py:1122-1137).  ``device_body`` / ``bind`` add ``__fbr_body__``.

An unbound callable raises ``TypeError`` -- there is no CPU fallback.

Encoders turn the Python-level task arguments (what the reference would pickle,
fiber/pool.py:1181,1297-1301,1112-1113) into fixed-layout argument records.
"""
import hashlib
import operator
import struct

import numpy as np

from . import _abi

_BOUND = {}  # callables that cannot carry attributes (builtins) -> body name


def device_body(name, source=None, entry="fbr_body_entry", args="i64", bits_entry=None, result=None, shared=None, items=None,
                out=None, out_as="list", **meta):
    """Decorator: ``@device_body("pi_inside_det")`` binds ``func`` to the device body ``name`` and sets
    ``func.__fiber_meta__`` (``gpu=1`` unless overridden), like ``fiber.meta``.

    ``source=`` makes it an OUT-OF-TREE body: CUDA source of a translation unit that includes
    ``fiber_b200_body.cuh``, defines a ThreadBody and exports it with
    ``FBR_EXPORT_THREAD_BODY(Body, "<name>", <entry>, kind, flags)``.  It is compiled for sm_90a with
    nvcc (cached by content hash under ``fiber_b200/_lib/bodies/``) and registered with
    ``fbr_register_body`` -- the reference ships any callable to its workers (fiber/pool.py:961); this is
    how a callable that is not compiled into libfiber_b200 gets its device code there.  ``args`` names the
    argument record layout: ``"i64"`` (one int) or ``"i64x2"`` (two ints).  A bool body may also export its
    bit-packed twin (``FBR_EXPORT_BOOL_BODY_BITS(Body, "<name>_bits8", <bits_entry>, flags)``): pass ``bits_entry``
    and its results travel one bit each, like the compiled-in bool body's.

    A RECORD body (``FBR_EXPORT_RECORD_BODY``: any fixed-size argument and result structs) describes both records
    with NumPy dtypes: ``args`` and ``result`` take anything ``np.dtype()`` accepts, e.g. ``"<f8"`` or
    ``[("x", "<f8"), ("y", "<f8")]``, sub-array fields included.  The field names are the function's parameter
    names; a one-field (or plain scalar) result is returned as that value, several fields as a tuple.

    A record body with a broadcast element (``using Shared = ...`` in its struct) also reads one array every task of a
    map shares: ``shared=("centroids", <element dtype>)`` names the function's FIRST parameter and describes one
    element of that array; the ``args`` fields are the parameters after it.  Tasks pass the array as that parameter, or
    leave it out and read the block of the pool's initializer (``device_initializer``).

    A GROUP record body (``static constexpr uint32_t kGroup = G;`` in its struct, G = 2, 4, 8, 16 or 32) runs each task on
    G lanes of one warp, and its records may reach 32 KB (INTEGRATION.md has the size rules).  Nothing changes here:
    ``kGroup`` lives in the CUDA source, and ``map(f, rows)`` over a plain ``(n, k)`` array of a one-field body with a
    ``(k,)`` sub-array passes the rows without a copy, e.g. ``args=[("x", "<f8", (1024,))]`` for 8 KB rows.

    An ITEMS record body (``using Item = ...`` in its struct) also takes one variable-length array per task:
    ``items=("doc", "u1")`` names that parameter and describes one element.  The parameters are the broadcast parameter
    (if any), then the items parameter, then the ``args`` fields; ``args=None`` means no head record (``fbr::NoArg``).
    A task's items are a 1-D array of the element dtype (or a 1-D array / list whose values the dtype holds exactly: floats
    into an integer dtype or integers out of its range raise ``TypeError``), or, for a 1-byte
    element, ``bytes`` / ``bytearray`` / ``memoryview`` / ``str`` (sent as UTF-8).  ``map(f, Ragged(values, offsets))``
    passes a whole ragged array without a copy.  A body with 2 to 4 item streams (``using Items = fbr::ItemTypes<...>;``)
    takes a list of pairs, one per stream in order, e.g. ``items=[("a", "u1"), ("b", "u1")]``: the item parameters then
    come in that order after the broadcast parameter, each stream with its own element dtype and the same rules, and
    ``starmap(f, Columns(ra, rb))`` passes two ``Ragged`` columns without a copy.

    An EMIT record body (``using Out = ...;`` and ``using Res = fbr::NoRes;`` in its struct) returns a variable-length array
    per task: ``out="<u4"`` describes one element (``result=`` is not passed).  A task's value reads as a list, or, with
    ``out_as="bytes"`` / ``out_as="str"`` (UTF-8) and a 1-byte element, as ``bytes`` / ``str``; ``result.ragged`` is the
    whole map as one ``Ragged(values, offsets)``, which an items body can map over directly."""
    from .meta import VALID_META_KEYS
    for k in meta:
        assert k in VALID_META_KEYS, "Invalid meta argument \"{}\"".format(k)
    md = {"gpu": 1}
    md.update(meta)
    if source is not None:
        from . import bodies
        register_module(name, bodies.compile_module(name, source), entry, args, bits_entry, result, shared, items, out, out_as)

    def decorator(func):
        bind(func, name, **md)
        return func
    return decorator


_MODULES = {}   # body name -> (module path, entry, argument layout, bits entry, result layout, broadcast parameter, items
                # parameter) of bodies registered from their own module


def module_of(name):
    """Where an out-of-tree body came from (worker processes of a process-isolated pool register it themselves)."""
    return _MODULES.get(name)


def register_module(name, module_path, entry="fbr_body_entry", args="i64", bits_entry=None, result=None, shared=None, items=None,
                    out=None, out_as="list"):
    """``fbr_register_body`` + the host-side encoder for the body's argument records (and, with ``bits_entry``, the
    body's bit-packed twin ``<name>_bits8``).  Record bodies (``FBR_BODY_RECORD``) take NumPy dtypes for ``args`` and
    ``result``; their sizes must be the module's ``arg_bytes`` / ``result_bytes`` (``ValueError`` otherwise).
    Broadcast bodies (``FBR_BODY_BROADCAST``) also take ``shared=(parameter name, element dtype)``, whose size must be
    the module's element size; ``shared`` is refused for every other body (``ValueError``).  A group record body
    (``group_threads`` > 1 in its module descriptor: several threads per task, records up to 32 KB) registers like any
    other record body.  Items bodies (``FBR_BODY_ITEMS``) take ``items=(parameter name, element dtype)``, whose size must
    be the module's item size, and ``args=None`` when they have no head record; ``items`` is refused for every other
    body (``ValueError``).  A body with several item streams takes ``items=[(name, dtype), ...]``, one pair per stream
    in order: the count and every size must match ``fbr_body_items_streams`` (``ValueError``).  Emit bodies (``FBR_BODY_EMIT``) take ``out=<element dtype>``, whose size must be the module's
    out size, and ``out_as`` ("list", or "bytes" / "str" for 1-byte elements) instead of ``result``; ``out`` is refused for
    every other body (``ValueError``)."""
    import ctypes
    specs = _load_specs()           # the table as it was: the body registered below gets the encoder its layout asks for
    if bits_entry is not None:
        twin = name + "_bits8"
        register_module(twin, module_path, bits_entry, "bits8")
        _MODULES.pop(twin, None)
        BITS_TWIN[name] = twin
    L = _abi.load()
    fid = ctypes.c_int(-1)
    _abi.check(L.fbr_register_body(name.encode(), str(module_path).encode(), entry.encode(), ctypes.byref(fid)))
    info = _abi.BodyInfo()
    _abi.check(L.fbr_body_info(fid.value, ctypes.byref(info)))
    has_items, has_shared = info.flags & _abi.FBR_BODY_ITEMS, info.flags & _abi.FBR_BODY_BROADCAST
    out_dtype = None
    if out is not None and not info.flags & _abi.FBR_BODY_EMIT:
        raise ValueError("body %s returns a fixed-size result (its record struct has no Out element type): out= is for emit "
                         "bodies only" % name)
    if info.flags & _abi.FBR_BODY_EMIT:
        if out is None:
            raise ValueError("emit body %s: pass out=<element dtype> (each task returns a variable-length array)" % name)
        if result is not None:
            raise ValueError("emit body %s returns a variable-length array of out=: result= is for fixed-size results" % name)
        ob = ctypes.c_uint32(0)
        _abi.check(L.fbr_body_emit_info(fid.value, ctypes.byref(ob)))
        out_dtype = _record_dtype(out, "out", name)
        if out_dtype.itemsize != ob.value:
            raise ValueError("%s: out dtype %s is %d bytes, the body's Out is %d" % (name, out_dtype, out_dtype.itemsize, ob.value))
        if out_as not in ("list", "bytes", "str"):
            raise ValueError("%s: out_as is 'list', 'bytes' or 'str', got %r" % (name, out_as))
        if out_as != "list" and out_dtype.itemsize != 1:
            raise ValueError("%s: out_as=%r needs a 1-byte out element, the body's is %s" % (name, out_as, out_dtype))
        result = "<u8"                  # the engine's result record of an emit body: each task's end offset
    if items is not None and not has_items:
        raise ValueError("body %s takes no items (its record struct has no Item element type): items= is for items bodies "
                         "only" % name)
    if has_items and (result is None or items is None):
        raise ValueError("items body %s: pass result=<dtype> and items=(<parameter name>, <element dtype>)" % name)
    if has_shared and (result is None or shared is None):
        raise ValueError(("items body %s reads a broadcast block: pass shared=(<parameter name>, <element dtype>)" if has_items
                          else "broadcast body %s: pass result=<dtype> and shared=(<parameter name>, <element dtype>)") % name)
    if shared is not None and not has_shared:
        raise ValueError("body %s reads no broadcast block (its record struct has no Shared element type): shared= is "
                         "for broadcast bodies only" % name)
    record = None
    if info.flags & _abi.FBR_BODY_RECORD:
        if result is None:
            raise ValueError("record body %s: pass result=<dtype> (its %d-byte result record)" % (name, info.result_bytes))
        elem, stage = ctypes.c_uint32(0), ctypes.c_uint32(0)
        if has_shared:
            _abi.check(L.fbr_body_shared_info(fid.value, ctypes.byref(elem), ctypes.byref(stage)))
        if has_items:
            ns, ib = ctypes.c_uint32(0), (ctypes.c_uint32 * _abi.MAX_ITEM_STREAMS)()
            _abi.check(L.fbr_body_items_streams(fid.value, ctypes.byref(ns), ib))
            # args left at its default means no head record for a body that has none
            head = None if (isinstance(args, str) and args == "i64" and info.arg_bytes == 0) else args
            record = _Items(info, items, head, result, shared, list(ib)[:ns.value], elem.value, stage.value)
            items = record.layouts()[3]
        elif has_shared:
            record = _Broadcast(info, args, result, shared, elem.value, stage.value)
        else:
            record = _Record(info, args, result)        # validates the layouts against the module
        args, result = record.arg_dtype, record.res_dtype
        if shared is not None:
            shared = (record.shared_name, record.shared_dtype)
    elif result is not None:
        raise ValueError("body %s is not a record body (FBR_EXPORT_RECORD_BODY): its result layout is fixed" % name)
    old = specs.get(name)
    if record is not None and isinstance(old, _Record) and old.layouts() != record.layouts():
        raise ValueError("record body %s is registered already with %s; a name keeps its layouts"
                         % (name, ", ".join("%s=%s" % kv for kv in zip(("args", "result", "shared", "items"), old.layouts()))))
    if record is not None:
        record.out_dtype, record.out_as = out_dtype, out_as
    # the engine keeps the first module registered under a name (fbr_register_body is idempotent): so do worker processes
    _MODULES.setdefault(name, (str(module_path), entry, args, bits_entry, None if out_dtype is not None else result, shared,
                               items, out_dtype, out_as))
    if name not in specs:
        if record is not None:
            specs[name] = record
        elif args == "i64":
            specs[name] = _UnaryI64(info)
        elif args == "i64x2":
            specs[name] = _BinaryI64(info)
        elif args == "bits8":
            specs[name] = _Bits8(info)
        else:
            raise ValueError("unknown argument layout %r (have: i64, i64x2, bits8)" % (args,))
    return specs[name]


def device_initializer(body_name):
    """Bind a pool ``initializer`` to the broadcast block of device body ``body_name``.

    The reference runs ``initializer(*initargs)`` once in every worker process (fiber/pool.py:858-859),
    the idiom for giving all tasks the same large arguments without pickling them per task.  A host
    callable cannot run inside a GPU worker; what the idiom *means* maps exactly onto the engine's
    broadcast blocks: ``Pool(initializer=f, initargs=(...))`` with ``f`` decorated here uploads
    ``spec(body_name).shared_block(*initargs)`` once to every worker (``fbr_shared_put``), and tasks of that
    body submitted without their own shared arguments read it."""
    def decorator(func):
        spec(body_name)
        func.__fbr_init_body__ = body_name
        return func
    return decorator


def bind(func, name, **meta):
    """Bind an existing callable to device body ``name`` (see ``device_body``)."""
    from .meta import post_process
    spec(name)  # validate early: unknown names fail at bind time
    md = post_process(dict(meta) if meta else {"gpu": 1})
    try:
        func.__fbr_body__ = name
        func.__fiber_meta__ = md
    except (AttributeError, TypeError):
        _BOUND[func] = name
    return func


def body_name_of(func):
    name = getattr(func, "__fbr_body__", None)
    if name is None:
        try:
            name = _BOUND.get(func)
        except TypeError:
            name = None
    if name is None:
        raise TypeError(
            "fiber_b200.Pool: %r is not bound to a device body. Mapped functions execute on the GPU; "
            "bind one with @fiber_b200.device_body(name) or fiber_b200.bind(func, name) "
            "(available: %s). There is no CPU fallback." % (func, ", ".join(sorted(body_names()))))
    return name


# ------------------------------------------------------------------------------------------------
class Encoded:
    """Fixed-layout form of one map's arguments."""
    __slots__ = ("n", "args", "arg_stride", "index_start", "index_step", "shared", "task_index_base", "keepalive", "n_items",
                 "streams")

    def __init__(self, n, args=None, arg_stride=0, index_start=0, index_step=1, shared=None, task_index_base=0, n_items=0):
        self.n, self.args, self.arg_stride = n, args, arg_stride
        self.index_start, self.index_step = index_start, index_step
        self.shared, self.task_index_base = shared, task_index_base
        self.n_items = n_items     # bit-packed twins: argument items of the whole map (8 per task, the last may be short)
        self.streams = None        # items bodies: per stream (values, uint64 offsets) -- task j reads values[offsets[j]:offsets[j+1]]

    @property
    def items(self):
        """Stream 0 of an items body's map (its only stream for a one-stream body), or None."""
        return self.streams[0] if self.streams else None


def _as_i64(values, what):
    try:
        a = np.asarray(values)
    except OverflowError as e:
        raise OverflowError("%s: Python int too large for the int64 task record" % what) from e
    if a.size == 0:
        return np.zeros(a.shape if a.ndim else (0,), dtype=np.int64)
    if a.dtype == object:
        raise OverflowError("%s: arguments do not fit the int64 task record (got %r...)" % (what, values[:1]))
    if a.dtype.kind not in "iub":
        raise TypeError("%s: expected integer arguments, got dtype %s" % (what, a.dtype))
    if a.dtype.kind == "u" and a.dtype.itemsize == 8 and a.size and int(a.max()) > 2 ** 63 - 1:
        raise OverflowError("%s: argument exceeds int64" % what)
    return np.ascontiguousarray(a, dtype=np.int64)


class BodySpec:
    """One compiled-in device body plus the encoders for its argument records."""

    def __init__(self, info):
        self.name = info.name.decode()
        self.func_id = info.func_id
        self.arg_bytes = info.arg_bytes
        self.result_bytes = info.result_bytes
        self.result_kind = info.result_kind
        self.flags = info.flags

    # ---- argument encoders ---------------------------------------------------------------------
    def encode_map(self, items):
        """``map(func, items)``: one positional argument per task (fiber/pool.py:819-821)."""
        if self._fast_map_ok(items):
            return self._encode(items, fast=True)
        return self._encode([(it,) for it in items], fast=False)

    def encode_starmap(self, items):
        """``starmap(func, items)``: items are argument tuples (fiber/pool.py:807-809)."""
        return self._encode(list(items), fast=False)

    def encode_apply(self, args, kwds):
        """``apply_async(func, args, kwds)``: one task (fiber/pool.py:804-806)."""
        return self._encode([(tuple(args), dict(kwds))], fast=False, apply=True)

    def _fast_map_ok(self, items):
        return False

    def _encode(self, items, fast, apply=False):
        raise NotImplementedError

    @staticmethod
    def _split(item, apply):
        """-> (args tuple, kwds dict) of one starmap/apply item; mirrors the arity rules at
        fiber/pool.py:803-812."""
        if apply:
            return item
        if not isinstance(item, (tuple, list)):
            raise TypeError("starmap items must be argument tuples, got %r" % (item,))
        return tuple(item), {}

    # ---- single-record fast path (doorbell lane): no NumPy on the round trip ---------------------
    def pack_apply(self, args, kwds):
        """One task's argument record as bytes (default: through the array encoder)."""
        enc = self.encode_apply(args, kwds)
        return np.ascontiguousarray(enc.args).tobytes()

    def unpack_result(self, raw):
        k = self.result_kind
        if k == _abi.FBR_RES_NONE:
            return None
        if k == _abi.FBR_RES_BOOL:
            return raw[0] != 0
        if k == _abi.FBR_RES_I64:
            return struct.unpack_from("<q", raw)[0]
        if k == _abi.FBR_RES_U32:
            return struct.unpack_from("<I", raw)[0]
        if k == _abi.FBR_RES_F64X2:
            return struct.unpack_from("<dd", raw)
        return list(raw)

    # ---- result decoding -----------------------------------------------------------------------
    def result_dtype(self):
        k = self.result_kind
        if k == _abi.FBR_RES_BOOL:
            return np.dtype(np.bool_), ()
        if k == _abi.FBR_RES_I64:
            return np.dtype(np.int64), ()
        if k == _abi.FBR_RES_U32:
            return np.dtype(np.uint32), ()
        if k == _abi.FBR_RES_F64X2:
            return np.dtype(np.float64), (2,)
        if k == _abi.FBR_RES_NONE:
            return np.dtype(np.uint8), ()
        return np.dtype(np.uint8), (self.result_bytes,)

    def to_python(self, row):
        """One result element as the Python object the reference would have returned."""
        k = self.result_kind
        if k == _abi.FBR_RES_NONE:
            return None
        if k == _abi.FBR_RES_F64X2:
            return (float(row[0]), float(row[1]))
        if k == _abi.FBR_RES_BYTES:
            return row.tolist()
        return row.item()

    def rows_to_list(self, arr):
        k = self.result_kind
        if k == _abi.FBR_RES_NONE:
            return [None] * len(arr)
        if k == _abi.FBR_RES_F64X2:
            return [tuple(r) for r in arr.tolist()]
        return arr.tolist()

    def sum_rows(self, arr):
        """``sum()`` of the reference's result list, from the result array."""
        if arr.dtype.kind in "iu" and arr.dtype.itemsize == 8:
            # int64 results: NumPy's sum wraps silently, Python's sum of the reference's list does not
            lo = int((arr.view(np.uint64) & np.uint64(0xFFFFFFFF)).sum(dtype=np.uint64))
            hi = int((arr.view(np.int64) >> np.int64(32)).sum(dtype=np.int64))
            return hi * (1 << 32) + lo
        return int(arr.sum())


class _UnaryI64(BodySpec):
    """f(x) with one int argument: square_i64, identity_i64, pi_inside_det, fault_identity_i64."""

    def pack_apply(self, args, kwds):
        if len(args) != 1 or kwds or type(args[0]) is not int:
            return super().pack_apply(args, kwds)       # full validation / error messages
        try:
            return struct.pack("<q", args[0])
        except struct.error:
            raise OverflowError("%s: Python int too large for the int64 task record" % self.name) from None

    def _fast_map_ok(self, items):
        return True

    def _encode(self, items, fast, apply=False):
        if fast:
            if isinstance(items, range):
                # a range() chunk stays a range in the reference too (76 B pickled, BASELINE.md):
                # here it needs no argument records at all, the task index is the argument.
                if len(items) and not (-2 ** 63 <= items[0] <= 2 ** 63 - 1 and -2 ** 63 <= items[-1] <= 2 ** 63 - 1):
                    raise OverflowError("range() bounds exceed the int64 task record")
                return Encoded(len(items), index_start=items.start, index_step=items.step)
            a = _as_i64(items if isinstance(items, np.ndarray) else list(items), self.name)
            if a.ndim != 1:
                raise TypeError("%s: expected a flat sequence of ints" % self.name)
            return Encoded(len(a), args=a, arg_stride=8)
        xs = []
        for it in items:
            args, kwds = self._split(it, apply)
            if len(args) != 1 or kwds:
                raise TypeError("%s() takes exactly one positional argument" % self.name)
            xs.append(args[0])
        a = _as_i64(xs, self.name)
        return Encoded(len(a), args=a, arg_stride=8)


class _Bits8(BodySpec):
    """``pi_inside_bits8``: task g = items 8g..8g+7 (range() indices or int64 arguments), result = one byte
    (bit k = item 8g+k).  Not bound to a callable: ``Pool`` routes maps of the bool body here
    (``BITS_TWIN``) and presents the bytes as a bit-backed ``ResultArray``."""

    def from_encoded(self, enc):
        """Re-express the bool body's encoded map (one int64 record or range() index per task) as byte-tasks."""
        n = enc.n
        if enc.arg_stride == 0:
            return Encoded((n + 7) // 8, index_start=enc.index_start, index_step=enc.index_step, n_items=n)
        return Encoded((n + 7) // 8, args=enc.args, arg_stride=64, n_items=n)

    def result_dtype(self):
        return np.dtype(np.uint8), ()

    def encode_range(self, items):
        """``range`` of n indices -> ceil(n/8) byte tasks (the body walks the same start/step)."""
        if not isinstance(items, range):
            raise TypeError("%s takes range() arguments only" % self.name)
        if len(items) and not (-2 ** 63 <= items[0] <= 2 ** 63 - 1 and -2 ** 63 <= items[-1] + 7 * items.step <= 2 ** 63 - 1
                               and -2 ** 63 <= items[-1] <= 2 ** 63 - 1):
            raise OverflowError("range() bounds exceed the int64 task record")
        return Encoded((len(items) + 7) // 8, index_start=items.start, index_step=items.step, n_items=len(items))


# bool bodies that have a bit-packed twin: 8 consecutive range() indices per result byte
BITS_TWIN = {"pi_inside_det": "pi_inside_bits8"}


class _BinaryI64(BodySpec):
    """f(x, y) / f(x, y=default) with int arguments: mul2_i64, square_scale_i64."""

    def __init__(self, info, y_default=None):
        super().__init__(info)
        self.y_default = y_default

    def pack_apply(self, args, kwds):
        if not kwds and len(args) == 2 and type(args[0]) is int and type(args[1]) is int:
            try:
                return struct.pack("<qq", args[0], args[1])
            except struct.error:
                raise OverflowError("%s: Python int too large for the int64 task record" % self.name) from None
        return super().pack_apply(args, kwds)

    def _encode(self, items, fast, apply=False):
        rows = []
        for it in items:
            args, kwds = self._split(it, apply)
            vals = dict(zip(("x", "y"), args))
            if len(args) > 2:
                raise TypeError("%s() takes at most 2 positional arguments" % self.name)
            for k, v in kwds.items():
                if k not in ("x", "y") or k in vals:
                    raise TypeError("%s() got an unexpected or duplicate keyword argument %r" % (self.name, k))
                vals[k] = v
            if "y" not in vals and self.y_default is not None:
                vals["y"] = self.y_default
            if "x" not in vals or "y" not in vals:
                raise TypeError("%s() missing required arguments" % self.name)
            rows.append((vals["x"], vals["y"]))
        a = _as_i64(rows, self.name).reshape(len(rows), 2)
        return Encoded(len(rows), args=a, arg_stride=16)


_LAYOUT_ALIASES = {"i64": "<i8", "i64x2": [("x", "<i8"), ("y", "<i8")]}


def _record_dtype(layout, what, name):
    """``np.dtype(layout)``, refused when a field holds Python objects (``TypeError``) or is big-endian (the device is
    little-endian: ``TypeError``)."""
    dt = np.dtype(_LAYOUT_ALIASES.get(layout, layout) if isinstance(layout, str) else layout)

    def check(d):
        if d.hasobject:
            raise TypeError("%s: the %s layout %s holds Python objects; records are fixed-size bytes" % (name, what, dt))
        if d.names is not None:
            for f in d.names:
                check(d.fields[f][0])
        elif d.subdtype is not None:
            check(d.subdtype[0])
        elif d.byteorder == ">" or (d.byteorder == "=" and np.little_endian is False):
            raise TypeError("%s: the %s layout %s is big-endian; the device reads little-endian records" % (name, what, dt))
    check(dt)
    return dt


_MISSING = object()


class _Record(BodySpec):
    """A record body (``FBR_BODY_RECORD``): argument and result records described by NumPy dtypes.

    The argument dtype's field names are the function's parameter names (a dtype without fields is one positional
    parameter).  ``map(f, array)`` with exactly the argument dtype -- or, for a one-parameter body, an array of the
    parameter's own dtype and shape -- is passed to the engine without a copy; lists, ``starmap`` tuples and
    ``apply_async(args, kwds)`` are bound to the fields the way Python binds a call.  Results come back as a structured
    view of the pinned segment; one value per task (a scalar or one-field dtype) reads as that value, several fields
    as a tuple."""

    def __init__(self, info, args, result):
        super().__init__(info)
        # args=None for a body without argument bytes: an items body with no head record (fbr::NoArg), no argument fields
        self.arg_dtype = None if args is None and not self.arg_bytes else _record_dtype(args, "argument", self.name)
        self.res_dtype = _record_dtype(result, "result", self.name)
        if self.arg_dtype is not None and self.arg_dtype.itemsize != self.arg_bytes:
            raise ValueError("%s: argument dtype %s is %d bytes, the body's argument record is %d"
                             % (self.name, self.arg_dtype, self.arg_dtype.itemsize, self.arg_bytes))
        if self.res_dtype.itemsize != self.result_bytes:
            raise ValueError("%s: result dtype %s is %d bytes, the body's result record is %d"
                             % (self.name, self.res_dtype, self.res_dtype.itemsize, self.result_bytes))
        if self.arg_dtype is None:
            self.params, self._sdt, self._fields = None, None, ()
            return
        self.params = self.arg_dtype.names                 # None: one positional-only parameter
        # the argument records as a structured array with named fields (one field "_0" when the dtype has none)
        self._sdt = self.arg_dtype if self.params else np.dtype([("_0", self.arg_dtype)])
        self._fields = self._sdt.names

    def layouts(self):
        """What a name keeps once registered: the argument and result dtypes."""
        return (self.arg_dtype, self.res_dtype)

    # ---- arguments ------------------------------------------------------------------------------------------------
    def _fast_map_ok(self, items):
        return True

    def _bind(self, args, kwds):
        """Field values of one call ``f(*args, **kwds)``, with Python's TypeErrors for a bad argument list."""
        names = self.params or ("",)
        if len(args) > len(names):
            raise TypeError("%s() takes %d positional argument%s but %d %s given"
                            % (self.name, len(names), "" if len(names) == 1 else "s", len(args), "was" if len(args) == 1 else "were"))
        vals = list(args) + [_MISSING] * (len(names) - len(args))
        for k, v in kwds.items():
            if self.params is None or k not in self.params:
                raise TypeError("%s() got an unexpected keyword argument %r" % (self.name, k))
            j = self.params.index(k)
            if vals[j] is not _MISSING:
                raise TypeError("%s() got multiple values for argument %r" % (self.name, k))
            vals[j] = v
        _check_missing(self.name, [names[j] for j, v in enumerate(vals) if v is _MISSING])
        return vals

    def _columns(self, columns):
        arr = np.empty(len(columns[0]) if columns else 0, self._sdt)
        for f, col in zip(self._fields, columns):
            arr[f] = col
        return Encoded(len(arr), args=arr, arg_stride=self.arg_bytes)

    def _encode(self, items, fast, apply=False):
        if fast:
            if isinstance(items, range) and self.flags & _abi.FBR_BODY_INDEX_ARG:
                if len(items) and not (-2 ** 63 <= items[0] <= 2 ** 63 - 1 and -2 ** 63 <= items[-1] <= 2 ** 63 - 1):
                    raise OverflowError("range() bounds exceed the int64 task record")
                return Encoded(len(items), index_start=items.start, index_step=items.step)
            if isinstance(items, np.ndarray):
                if items.ndim == 1 and items.dtype == self.arg_dtype:
                    a = np.ascontiguousarray(items)         # zero-copy when it already is
                    return Encoded(len(a), args=a, arg_stride=self.arg_bytes)
                one = self._sdt.fields[self._fields[0]][0]
                if len(self._fields) == 1 and items.ndim >= 1 and items.dtype == one.base and items.shape[1:] == one.shape:
                    a = np.ascontiguousarray(items)
                    return Encoded(len(a), args=a.reshape(len(a), -1).view(self._sdt).reshape(len(a)), arg_stride=self.arg_bytes)
            if len(self._fields) == 1:
                return self._columns([list(items)])
            items = [(it,) for it in items]                 # map() passes one argument: f(item) must bind
        rows = [self._bind(*self._split(it, apply)) for it in items]
        return self._columns([list(c) for c in zip(*rows)] if rows else [[] for _ in self._fields])

    # ---- results --------------------------------------------------------------------------------------------------
    def result_dtype(self):
        d = self.res_dtype
        if d.names is None and d.subdtype is not None:
            return d.subdtype[0], d.subdtype[1]
        return d, ()

    def to_python(self, row):
        names = self.res_dtype.names
        if names is None:
            return row.tolist()
        if len(names) == 1:
            return row[names[0]].tolist()
        return tuple(row[n].tolist() for n in names)

    def rows_to_list(self, arr):
        names = self.res_dtype.names
        if names is None:
            return arr.tolist()
        if len(names) == 1:
            return arr[names[0]].tolist()
        return list(zip(*(arr[n].tolist() for n in names)))

    def unpack_result(self, raw):
        return self.to_python(np.frombuffer(raw, self.res_dtype)[0])

    def sum_rows(self, arr):
        names = self.res_dtype.names
        if names is not None and len(names) > 1:
            raise TypeError("unsupported operand type(s) for +: 'int' and 'tuple' (%s returns %d fields)" % (self.name, len(names)))
        vals = arr[names[0]] if names else arr
        if vals.ndim > 1:
            raise TypeError("unsupported operand type(s) for +: 'int' and 'list' (%s returns an array per task)" % self.name)
        if vals.dtype.kind in "iub" and vals.dtype.itemsize <= 4:
            return int(vals.sum(dtype=np.int64))         # exact: fewer than 2^31 values of at most 32 bits
        return sum(vals.tolist())                        # Python's left-to-right sum, as over the reference's list


def _check_missing(name, missing):
    """Python's TypeError for a call of ``name`` that leaves the parameters ``missing`` without a value."""
    if missing:
        missing = [repr(m) for m in missing]
        listed = missing[0] if len(missing) == 1 else "%s and %s" % (", ".join(missing[:-1]) + ("," if len(missing) > 2 else ""), missing[-1])
        raise TypeError("%s() missing %d required positional argument%s: %s"
                        % (name, len(missing), "" if len(missing) == 1 else "s", listed))


def _same_bytes(a, b):
    """Whether two arrays are the same block: equal dtype and shape and the same bytes.  Comparing values would call
    -0.0 and +0.0 (or two NaNs with different payloads) the same while their blocks differ, and never call an array
    holding a NaN equal to its own copy."""
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    return np.array_equal(np.ascontiguousarray(a).reshape(-1).view(np.uint8), np.ascontiguousarray(b).reshape(-1).view(np.uint8))


class _LastBlock:
    """The broadcast block built from the last arguments, reused while new arguments compare equal to them.  A map's
    tasks usually all pass the same array (the reference pickles it into every task message), and an exact comparison
    with a kept copy is far cheaper than building the block again.  Returning the very same bytes object also lets
    ``Pool`` skip fingerprinting it before the upload-cache lookup."""

    def __init__(self):
        self._last = None         # (copies of the arguments, block)

    def get(self, arrays, build):
        last = self._last
        if last is not None and all(_same_bytes(a, b) for a, b in zip(last[0], arrays)):
            return last[1]
        blob = build(*arrays)
        self._last = ([a.copy() for a in arrays], blob)
        return blob


def _block_bytes(a):
    return np.ascontiguousarray(a).tobytes()


class _Broadcast(_Record):
    """A record body whose run() also reads the map's broadcast block (``FBR_BODY_BROADCAST``): an array of
    ``shared_dtype`` elements that every task shares, uploaded once per worker.

    The function's first parameter (``shared_name``) is that array, the argument dtype's fields are the parameters
    after it: ``starmap(f, [(C, p0), (C, p1)])``, ``apply_async(f, (C, p))`` and ``apply_async(f, (p,), {name: C})`` pass
    it with every task (the same array each time); ``map(f, points)`` and items without it read the pool's initializer
    block (``Pool(initializer=<@device_initializer(body)>, initargs=(C,))``)."""

    def __init__(self, info, args, result, shared, elem_bytes, stage_bytes):
        super().__init__(info, args, result)
        self._init_shared(shared, elem_bytes, stage_bytes)

    def _init_shared(self, shared, elem_bytes, stage_bytes):
        if not (isinstance(shared, (tuple, list)) and len(shared) == 2 and isinstance(shared[0], str) and shared[0].isidentifier()):
            raise ValueError("%s: shared= is (<parameter name>, <element dtype>), got %r" % (self.name, shared))
        self.shared_name = shared[0]
        if self.params is not None and self.shared_name in self.params:
            raise ValueError("%s: the broadcast parameter %r is also an argument field" % (self.name, self.shared_name))
        self.shared_dtype = _record_dtype(shared[1], "broadcast element", self.name)
        if self.shared_dtype.itemsize != elem_bytes:
            raise ValueError("%s: broadcast element dtype %s is %d bytes, the body's Shared element is %d"
                             % (self.name, self.shared_dtype, self.shared_dtype.itemsize, elem_bytes))
        self.elem_bytes, self.stage_bytes = elem_bytes, stage_bytes
        # the element as a plain array's trailing shape and base type: (K, 16) float32 for ("c", "<f4", (16,))
        d = self.shared_dtype
        if d.names is not None and len(d.names) == 1:
            d = d.fields[d.names[0]][0]
        self._plain = (d.subdtype[0], d.subdtype[1]) if d.subdtype is not None else (d, ())
        self._blocks = _LastBlock()

    def layouts(self):
        return (self.arg_dtype, self.res_dtype, (self.shared_name, self.shared_dtype))

    def _block_array(self, x):
        """The broadcast array as a contiguous array of elements: exactly the element dtype (1-D), or a plain array whose
        trailing shape and base type are the element's (viewed, not converted)."""
        a = np.asarray(x)
        base, shape = self._plain
        if a.dtype == self.shared_dtype and a.ndim == 1:
            pass
        elif a.dtype == base and a.ndim == 1 + len(shape) and a.shape[1:] == shape:
            if self.shared_dtype.names is not None and len(a):
                # the same elements as a 1-D array of the element dtype (a view when `a` is contiguous), so a plain array
                # and its structured twin find the same kept block
                a = np.ascontiguousarray(a).reshape(len(a), -1).view(self.shared_dtype).reshape(len(a))
        else:
            raise TypeError("%s: %s must be a 1-D array of %s or an array of shape (n,) + %s and dtype %s, got shape %s "
                            "and dtype %s" % (self.name, self.shared_name, self.shared_dtype, shape, base, a.shape, a.dtype))
        if len(a) == 0:
            raise ValueError("%s: %s is empty; the broadcast block needs at least one element" % (self.name, self.shared_name))
        return a

    def shared_block(self, *initargs):
        """The broadcast block of ``initializer(array)``: the array's bytes, kept while later arrays compare equal."""
        if len(initargs) != 1:
            raise TypeError("%s: the initializer takes exactly one argument (%s), got %d" % (self.name, self.shared_name, len(initargs)))
        return self._blocks.get((self._block_array(initargs[0]),), _block_bytes)

    def _calls(self, items, apply, n_rest):
        """Each item's ``(args, kwds)`` without the broadcast array, with the array's element view so far (None until an
        item passes it).  An item passes the array by keyword, or first when it has one more argument than the ``n_rest``
        other parameters take.  Every item of a map passes it or none does, and all pass the same elements."""
        first = block = carried = None      # first: the first item's array; block: its element view
        for it in items:
            args, kwds = self._split(it, apply)
            if self.shared_name is None:    # an items body without a broadcast block
                yield args, kwds, None
                continue
            if self.shared_name in kwds:
                kwds = dict(kwds)
                b = kwds.pop(self.shared_name)
            elif args and len(args) + len(kwds) > n_rest:
                b, args = args[0], tuple(args[1:])
            else:
                b = _MISSING
            has = b is not _MISSING
            if carried is None:
                carried = has
            elif carried != has:
                raise TypeError("%s: mixed items with and without %s in one map" % (self.name, self.shared_name))
            if has:
                # the same object as the first item's: nothing to check; else the same elements, byte for byte, in
                # either of the accepted forms (C and C["c"] are one block)
                if first is None:
                    first, block = b, self._block_array(b)
                elif b is not first and not _same_bytes(self._block_array(b), block):
                    raise ValueError("%s: all tasks of one map must share %s" % (self.name, self.shared_name))
            yield args, kwds, block

    def _encode(self, items, fast, apply=False):
        if fast:
            return super()._encode(items, fast)              # map(f, points): the block is the initializer's
        rows, block = [], None
        for args, kwds, block in self._calls(items, apply, len(self._fields)):
            rows.append(self._bind(args, kwds))
        enc = self._columns([list(c) for c in zip(*rows)] if rows else [[] for _ in self._fields])
        enc.shared = self._blocks.get((block,), _block_bytes) if block is not None else None
        return enc


class Ragged:
    """A sequence of variable-length 1-D arrays in two arrays: ``r[i]`` is ``values[offsets[i]:offsets[i+1]]``.

    ``map(f, Ragged(values, offsets))`` over an items body passes both arrays to the engine without a copy (when
    ``values`` is contiguous with the body's element dtype and ``offsets`` contiguous 64-bit integers).  ``offsets`` are
    n + 1 non-decreasing indices, all within ``values``; ``offsets[0]`` need not be 0.  Slicing gives a Ragged over the
    slice's values with rebased offsets."""

    def __init__(self, values, offsets):
        values, offsets = np.asarray(values), np.asarray(offsets)
        if values.ndim != 1:
            raise ValueError("Ragged: values must be 1-D, got shape %s" % (values.shape,))
        if offsets.ndim != 1 or len(offsets) == 0 or offsets.dtype.kind not in "iu":
            raise ValueError("Ragged: offsets must be a non-empty 1-D integer array (n + 1 entries)")
        if len(offsets) > 1 and bool(np.any(offsets[1:] < offsets[:-1])):
            raise ValueError("Ragged: offsets must not decrease")
        if (offsets.dtype.kind == "i" and int(offsets[0]) < 0) or int(offsets[-1]) > len(values):
            raise ValueError("Ragged: offsets must lie in [0, len(values)] (last offset %d, %d values)" % (int(offsets[-1]), len(values)))
        self.values, self.offsets = values, offsets

    def __len__(self):
        return len(self.offsets) - 1

    def __getitem__(self, i):
        if isinstance(i, slice):
            start, stop, step = i.indices(len(self))
            if step != 1:
                raise ValueError("Ragged: only contiguous slices")
            o = self.offsets[start:max(start, stop) + 1]
            return Ragged(self.values[int(o[0]):int(o[-1])], o.astype(np.int64) - int(o[0]))
        i = operator.index(i)
        n = len(self)
        if i < 0:
            i += n
        if not 0 <= i < n:
            raise IndexError("Ragged index out of range")
        return self.values[int(self.offsets[i]):int(self.offsets[i + 1])]

    def __reduce__(self):
        return (Ragged, (self.values, self.offsets))


def _item_array(name, dtype, x):
    """One task's items as a 1-D array of `dtype`.  Values the dtype cannot hold exactly -- floats into an integer dtype,
    integers out of its range, text or objects -- are refused (TypeError) rather than truncated or wrapped."""
    try:
        a = np.asarray(x)
    except (ValueError, TypeError, OverflowError) as e:
        raise TypeError("%s: an item is not convertible to a 1-D array of %s (%s)" % (name, dtype, e)) from None
    if a.ndim != 1:
        raise TypeError("%s: every item must be 1-D, got shape %s" % (name, a.shape))
    if a.dtype == dtype:
        return a
    kind = dtype.kind
    if a.dtype.kind in "OUSV" or (a.dtype.kind in "fc" and kind in "iub") or (a.dtype.kind == "c" and kind == "f"):
        raise TypeError("%s: an item of %s is not convertible to a 1-D array of %s without loss" % (name, a.dtype, dtype))
    out = a.astype(dtype)
    if a.dtype.kind in "iub" and kind in "iu" and not np.array_equal(out, a):
        raise TypeError("%s: an item holds integers outside the range of %s" % (name, dtype))
    return out


def _encode_items(name, dtype, xs):
    """One map's items as (values, uint64 offsets): a Ragged as it is, else the concatenation of every task's items.  Byte
    strings are joined in one call (no NumPy call per item)."""
    if isinstance(xs, Ragged):
        v, o = xs.values, xs.offsets
        if v.dtype != dtype:
            raise TypeError("%s: Ragged values are %s, the body's items are %s" % (name, v.dtype, dtype))
        if o.dtype == np.int64:
            o = o.view(np.uint64)                 # validated non-negative by Ragged
        return np.ascontiguousarray(v), np.ascontiguousarray(o, dtype=np.uint64)
    xs = list(xs)
    byteish = [isinstance(x, (bytes, bytearray, memoryview, str)) for x in xs]
    if any(byteish):
        if dtype.itemsize != 1:
            raise TypeError("%s: bytes and str items need a 1-byte item dtype, the body's is %s" % (name, dtype))
        if not all(byteish):
            raise TypeError("%s: mixed byte strings and arrays in one map" % name)
        parts = [x.encode("utf-8") if isinstance(x, str) else bytes(x) for x in xs]
        lens = np.fromiter(map(len, parts), dtype=np.uint64, count=len(parts))
        values = np.frombuffer(b"".join(parts), dtype=dtype)
    else:
        arrays = [_item_array(name, dtype, x) for x in xs]
        lens = np.fromiter(map(len, arrays), dtype=np.uint64, count=len(arrays))
        values = np.concatenate(arrays) if arrays else np.empty(0, dtype)
    offsets = np.zeros(len(lens) + 1, np.uint64)
    np.cumsum(lens, out=offsets[1:])
    return values, offsets


class Columns:
    """``n`` argument tuples held as columns: ``starmap(f, Columns(ra, rb, thresholds))`` calls ``f(ra[i], rb[i],
    thresholds[i])`` for every i.  Column k is the function's parameter k after the broadcast parameter (tasks under
    Columns read the pool initializer's block): a ``Ragged`` for an items parameter, passed to the engine without a copy
    where ``zip(ra, rb)`` would build a tuple and an array per task, or a 1-D array or list for a head-record field.  All
    columns have the same length.  A slice is the Columns of the columns' slices (a Ragged's offsets rebased), and a
    Columns pickles, so process-isolated pools ship each block's slice."""

    def __init__(self, *columns):
        if not columns:
            raise ValueError("Columns: pass at least one column")
        n = len(columns[0])
        for k, c in enumerate(columns):
            if len(c) != n:
                raise ValueError("Columns: column %d has %d entries, column 0 has %d" % (k, len(c), n))
        self.columns = columns

    def __len__(self):
        return len(self.columns[0])

    def __getitem__(self, i):
        if isinstance(i, slice):
            return Columns(*(c[i] for c in self.columns))
        return tuple(c[i] for c in self.columns)

    def __iter__(self):
        return (self[i] for i in range(len(self)))

    def __reduce__(self):
        return (Columns, self.columns)


def _is_item_pair(x):
    return isinstance(x, (tuple, list)) and len(x) == 2 and isinstance(x[0], str) and x[0].isidentifier()


class _Items(_Broadcast):
    """A record body whose task also takes 1 to 4 variable-length arrays (``FBR_BODY_ITEMS``), one per item stream:
    ``item_names`` are their parameters and ``item_dtypes`` their elements, in stream order (``item_name`` /
    ``item_dtype``: stream 0).  The parameters are the broadcast parameter (bodies with a Shared type), the items of each
    stream, then the argument dtype's fields (none when ``args`` is None: the body has no head record).  ``map(f, xs)``
    passes one items array per task (one-stream bodies without a head record); ``starmap`` / ``apply_async`` bind the
    items like any other parameter, and ``starmap(f, Columns(...))`` takes whole columns."""

    def __init__(self, info, items, args, result, shared, item_bytes, shared_elem=0, shared_stage=0):
        # item_bytes: the element size of each of the body's streams
        if args is None and info.arg_bytes:
            raise ValueError("%s: args=None, but the body's head record is %d bytes" % (info.name.decode(), info.arg_bytes))
        _Record.__init__(self, info, args, result)
        self.shared_name = self.shared_dtype = None
        if shared is not None:
            self._init_shared(shared, shared_elem, shared_stage)
        k = len(item_bytes)
        pairs = [items] if _is_item_pair(items) else list(items) if isinstance(items, (tuple, list)) else []
        if not pairs or not all(_is_item_pair(p) for p in pairs):
            raise ValueError(("%s: items= is (<parameter name>, <element dtype>), got %r" if k == 1 else
                              "%s: items= is a list of (<parameter name>, <element dtype>) pairs, one per item stream, got %r")
                             % (self.name, items))
        if len(pairs) != k:
            raise ValueError("%s: items= describes %d item stream%s, the body takes %d"
                             % (self.name, len(pairs), "" if len(pairs) == 1 else "s", k))
        self.item_names = tuple(p[0] for p in pairs)
        for j, n in enumerate(self.item_names):
            if n == self.shared_name or (self.params is not None and n in self.params) or n in self.item_names[:j]:
                raise ValueError("%s: the items parameter %r is also another parameter" % (self.name, n))
        self.item_dtypes = tuple(_record_dtype(p[1], "item", self.name) for p in pairs)
        for j, (d, b) in enumerate(zip(self.item_dtypes, item_bytes)):
            if d.itemsize != b:
                raise ValueError(("%s: item dtype %s is %d bytes, the body's Item is %d" if k == 1 else
                                  "%%s: item dtype %%s is %%d bytes, the body's stream %d item is %%d" % j)
                                 % (self.name, d, d.itemsize, b))
        self.item_name, self.item_dtype = self.item_names[0], self.item_dtypes[0]

    def layouts(self):
        shared = (self.shared_name, self.shared_dtype) if self.shared_name is not None else None
        items = tuple(zip(self.item_names, self.item_dtypes))
        return (self.arg_dtype, self.res_dtype, shared, items[0] if len(items) == 1 else items)

    def _with_items(self, enc, columns):
        enc.streams = [_encode_items(self.name, d, xs) for d, xs in zip(self.item_dtypes, columns)]
        enc.n = len(enc.streams[0][1]) - 1
        return enc

    def encode_starmap(self, items):
        if isinstance(items, Columns):
            return self._encode_columns(items)
        return super().encode_starmap(items)

    def _encode_columns(self, c):
        k, want = len(self.item_names), len(self.item_names) + len(self._fields)
        if len(c.columns) != want:
            raise TypeError("%s() takes %d argument%s after the broadcast parameter, got %d columns"
                            % (self.name, want, "" if want == 1 else "s", len(c.columns)))
        enc = Encoded(0) if self.arg_dtype is None else self._columns(list(c.columns[k:]))
        return self._with_items(enc, c.columns[:k])

    def _encode(self, items, fast, apply=False):
        k = len(self.item_names)
        if fast:
            if self.arg_dtype is None and k == 1:   # map(f, xs): each item is one task's items; a broadcast block is the initializer's
                return self._with_items(Encoded(0), [items])
            items = [(it,) for it in items]
        xs, rows, block = [[] for _ in range(k)], [], None
        for args, kwds, block in self._calls(items, apply, k + len(self._fields)):    # the items and the record's fields
            kwds = dict(kwds)
            missing = []
            for j, name in enumerate(self.item_names):
                if name in kwds:
                    xs[j].append(kwds.pop(name))
                elif args:
                    xs[j].append(args[0])
                    args = tuple(args[1:])
                else:
                    missing.append(name)
            _check_missing(self.name, missing)
            if self.arg_dtype is None:
                if args or kwds:
                    n = k + (self.shared_name is not None)
                    raise TypeError("%s() takes %d positional argument%s but more were given (unexpected %s)"
                                    % (self.name, n, "" if n == 1 else "s",
                                       ", ".join([repr(a) for a in args] + list(map(repr, kwds)))))
            else:
                rows.append(self._bind(args, kwds))
        if self.arg_dtype is None:
            enc = Encoded(0)
        else:
            enc = self._columns([list(c) for c in zip(*rows)] if rows else [[] for _ in self._fields])
        enc.shared = self._blocks.get((block,), _block_bytes) if block is not None else None
        return self._with_items(enc, xs)


class _SleepF64(BodySpec):
    def _fast_map_ok(self, items):
        return True

    def _encode(self, items, fast, apply=False):
        if fast:
            a = np.ascontiguousarray(list(items), dtype=np.float64)
        else:
            vals = []
            for it in items:
                args, kwds = self._split(it, apply)
                if len(args) != 1 or kwds:
                    raise TypeError("sleep body takes exactly one positional argument")
                vals.append(args[0])
            a = np.ascontiguousarray(vals, dtype=np.float64)
        return Encoded(len(a), args=a, arg_stride=8)


class _Parzen(BodySpec):
    """parzen_estimation(x_samples, point_x, h) (examples/parzen_estimation.py:6-15).

    ``x_samples`` and ``point_x`` are identical for every task of a map: they become the broadcast
    block (uploaded once per distinct array instead of pickled into every task message,
    SURVEY.md 3.2); the per-task record is ``h``."""
    HEADER = np.dtype([("n_samples", "<u4"), ("dims", "<u4"), ("power", "<u4"), ("elem_bytes", "<u4"),
                       ("point_x", "<f8", (8,))])

    def __init__(self, info, elem):
        super().__init__(info)
        self.elem = np.dtype(elem)
        self._blocks = _LastBlock()

    def shared_block(self, x_samples, point_x):
        """The broadcast block for (x_samples, point_x).  The reference pickles both into every one of its task
        messages; the example submits 102 ``apply_async`` calls with the same arrays, so the last block is kept
        and reused when the arguments compare equal (an exact memcmp of 160 KB, ~10 us, instead of casting and
        serialising them again)."""
        return self._blocks.get((np.asarray(x_samples), np.asarray(point_x)), self._build_block)

    def _build_block(self, xs, px):
        if xs.ndim != 2 or px.ndim != 2 or px.shape[0] != xs.shape[1]:
            raise TypeError("parzen_estimation: x_samples must be (n, d) and point_x (d, p)")
        if px.shape[0] > 8:
            raise TypeError("parzen_estimation: at most 8 dimensions are supported by the device body")
        if px.shape[1] != 1:
            # the reference evaluates `np.abs(row) > 1/2` on a length-p row, which raises for p != 1
            raise ValueError("The truth value of an array with more than one element is ambiguous")
        if xs.shape[0] == 0:
            # the reference's `k_n / len(x_samples)` (examples/parzen_estimation.py:15); the kernel would return 0.0 / 0.0
            raise ZeroDivisionError("division by zero")
        hdr = np.zeros((), dtype=self.HEADER)
        hdr["n_samples"], hdr["dims"], hdr["power"], hdr["elem_bytes"] = xs.shape[0], xs.shape[1], px.shape[1], self.elem.itemsize
        hdr["point_x"][: px.shape[0]] = px[:, 0].astype(np.float64)
        body = np.ascontiguousarray(xs, dtype=self.elem)  # the one cast to fp32 for parzen_f32
        return hdr.tobytes() + body.tobytes()

    def _fast_map_ok(self, items):
        # map(func, widths): the samples come from the pool's broadcast block (Pool(initializer=, initargs=))
        return True

    def _encode(self, items, fast, apply=False):
        if fast:
            return Encoded(len(items), args=np.ascontiguousarray(list(items), dtype=np.float64), arg_stride=8)
        hs, first = [], None
        for it in items:
            args, kwds = self._split(it, apply)
            if len(args) == 1 and not kwds:        # (h,): samples from the broadcast block
                if first is not None:
                    raise TypeError("parzen_estimation: mixed (h,) and (x_samples, point_x, h) items in one map")
                hs.append(float(args[0]))
                continue
            if hs and first is None:
                raise TypeError("parzen_estimation: mixed (h,) and (x_samples, point_x, h) items in one map")
            vals = dict(zip(("x_samples", "point_x", "h"), args))
            vals.update(kwds)
            if set(vals) != {"x_samples", "point_x", "h"}:
                raise TypeError("parzen_estimation(x_samples, point_x, h): bad arguments")
            if first is None:
                first = (vals["x_samples"], vals["point_x"])
            elif not (vals["x_samples"] is first[0] and vals["point_x"] is first[1]):
                if not (np.array_equal(vals["x_samples"], first[0]) and np.array_equal(vals["point_x"], first[1])):
                    raise ValueError("parzen_estimation: all tasks of one map must share x_samples and point_x")
            hs.append(float(vals["h"]))
        a = np.ascontiguousarray(hs, dtype=np.float64)
        enc = Encoded(len(a), args=a, arg_stride=8)
        enc.shared = self.shared_block(*first) if first is not None else None
        return enc


class _Payload4K(BodySpec):
    """Synthetic 4 KB payload bodies.  ``map(func, records)`` with a ``(n, 1024)`` uint32 array, or
    ``starmap(func, [(t, rec), ...])`` with consecutive ``t`` (the task's global index)."""

    def _fast_map_ok(self, items):
        return isinstance(items, np.ndarray)

    def result_dtype(self):
        if self.result_kind == _abi.FBR_RES_BYTES:
            return np.dtype(np.uint32), (1024,)
        return super().result_dtype()

    def _encode(self, items, fast, apply=False):
        if fast:
            recs, base = items, 0
        else:
            ts, rows = [], []
            for it in items:
                args, kwds = self._split(it, apply)
                if len(args) != 2 or kwds:
                    raise TypeError("%s(t, rec): bad arguments" % self.name)
                ts.append(int(args[0]))
                rows.append(args[1])
            base = ts[0] if ts else 0
            if ts != list(range(base, base + len(ts))):
                raise ValueError("%s: task indices must be consecutive" % self.name)
            recs = np.asarray(rows, dtype=np.uint32)
        recs = np.ascontiguousarray(recs, dtype=np.uint32)
        if recs.ndim != 2 or recs.shape[1] != 1024:
            raise TypeError("%s: records must be (n, 1024) uint32" % self.name)
        return Encoded(recs.shape[0], args=recs, arg_stride=4096, task_index_base=base)


_SPECS = None


def _load_specs():
    global _SPECS
    if _SPECS is not None:
        return _SPECS
    import ctypes
    L = _abi.load()
    n = ctypes.c_int(0)
    _abi.check(L.fbr_body_count(ctypes.byref(n)))
    specs = {}
    for fid in range(n.value):
        info = _abi.BodyInfo()
        _abi.check(L.fbr_body_info(fid, ctypes.byref(info)))
        name = info.name.decode()
        if name in ("square_i64", "identity_i64", "pi_inside_det", "fault_identity_i64", "trap_identity_i64"):
            s = _UnaryI64(info)
        elif name == "mul2_i64":
            s = _BinaryI64(info)
        elif name == "square_scale_i64":
            s = _BinaryI64(info, y_default=1)
        elif name == "sleep_f64":
            s = _SleepF64(info)
        elif name == "parzen_f32":
            s = _Parzen(info, np.float32)
        elif name == "parzen_f64":
            s = _Parzen(info, np.float64)
        elif name in ("payload_map_4k", "payload_checksum_4k"):
            s = _Payload4K(info)
        elif name == "pi_inside_bits8":
            s = _Bits8(info)
        else:
            s = BodySpec(info)
        specs[name] = s
    _SPECS = specs
    return specs


def body_names():
    return list(_load_specs())


def spec(name):
    specs = _load_specs()
    if name not in specs:
        raise KeyError("no device body named %r is compiled into libfiber_b200 (have: %s)" % (name, ", ".join(sorted(specs))))
    return specs[name]


def fingerprint(buf):
    return hashlib.blake2b(buf, digest_size=16).digest()
