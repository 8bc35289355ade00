"""``fiber_b200.Pool`` -- the reference's ``ZPool`` / ``ResilientZPool`` surface
(fiber/pool.py:881-1422, 1425-1688) on the GPU engine.

Same constructor, method names, defaults and exceptions as the reference:

* ``Pool(processes=None, initializer=None, initargs=(), maxtasksperchild=None, error_handling=False)``
  (fiber/context.py:38-45); ``processes=None`` means 1 (fiber/pool.py:894);
* ``map / map_async / starmap / starmap_async / apply / apply_async / imap / imap_unordered /
  close / terminate / join / start_workers / wait_until_workers_up``;
* ``chunksize=None`` -> 32 (fiber/pool.py:1169-1170), ``imap`` default chunksize 1 (:1218);
* ``ValueError("Pool is not running")`` once closed (:1107-1108, 1166-1167, 1284-1285);
  ``NotImplementedError`` for ``error_callback`` (:1162-1164); ``RuntimeError`` when a function
  with different ``__fiber_meta__`` arrives after the workers started (:1128-1133);
* workers start lazily on the first submission (:1122-1137).

What differs, by construction: a worker is a CUDA device, the mapped callable must be bound to a
compiled-in device body (``fiber_b200.device_body``), results come back as a buffer-backed
``ResultArray`` (list-like; ``.tolist()`` materialises the reference's list) instead of 1e8 Python
objects, and nothing on this path executes tasks on the CPU.
"""
import collections.abc
import ctypes
import math
import operator
import threading
import time

import numpy as np

from . import _abi, registry

RUN, CLOSE, TERMINATE = 0, 1, 2
DEFAULT_CHUNKSIZE = 32


class _Engine:
    """Owner of one ``fbr_pool_t``.  Destroyed when the last Python reference (pool or result
    segment) goes away, so result buffers never dangle."""

    def __init__(self, n_workers, devices, ring_bytes, timing):
        self.lib = _abi.load()
        ids = (ctypes.c_int * n_workers)(*devices)
        handle = ctypes.c_void_p()
        _abi.check(self.lib.fbr_pool_create(n_workers, ids, ring_bytes, _abi.FBR_POOL_TIMING if timing else 0,
                                            ctypes.byref(handle)))
        self.handle = handle
        self.n_workers = n_workers
        self.devices = list(devices)
        self.lock = threading.Lock()

    def __del__(self):
        h, self.handle = getattr(self, "handle", None), None
        if h:
            self.lib.fbr_pool_destroy(h)


class _Segment:
    """Owner of one map's engine state (its seq: control slots, events, pinned result segment) from the
    moment it is submitted.  Once the map has finished, ``bind`` exposes the pinned segment through
    ``__array_interface__`` so NumPy views keep it (and through it the engine) alive.  Dropping the last
    reference -- a fetched result going away, but also a fire-and-forget ``map_async`` or an abandoned
    ``imap`` generator -- releases the seq (``self._inventory[job_seq] = None``, fiber/pool.py:677-679)."""

    def __init__(self, engine, seq):
        self.engine, self.seq, self.ptr, self.nbytes = engine, seq, None, 0

    def bind(self, ptr, nbytes):
        self.ptr, self.nbytes = ptr, nbytes
        self.__array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr or 0, False), "version": 3}
        return self

    def __del__(self):
        eng = getattr(self, "engine", None)
        if eng is not None and eng.handle:
            eng.lib.fbr_result_release(eng.handle, self.seq)


class _PinnedBlock:
    """Pinned host block from the engine's segment cache (``fbr_host_alloc``): NumPy views keep it
    alive, garbage collection returns it.  Arguments that live here are DMA'd straight to the device
    (no staging copy) -- the host end of the pinned task ring."""

    def __init__(self, engine, nbytes):
        self.engine = engine
        ptr = ctypes.c_void_p()
        _abi.check(engine.lib.fbr_host_alloc(engine.handle, max(1, nbytes), ctypes.byref(ptr)))
        self.ptr = ptr.value
        self.__array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (self.ptr, False), "version": 3}

    def __del__(self):
        eng = getattr(self, "engine", None)
        if eng is not None and eng.handle and getattr(self, "ptr", None):
            eng.lib.fbr_host_free(eng.handle, ctypes.c_void_p(self.ptr))


class ResultArray(collections.abc.Sequence):
    """Ordered results of one map, backed by the pinned result segment (no per-item Python
    objects).  Behaves like the list the reference returns: indexing, slicing, iteration, ``len``,
    ``==`` against lists; ``tolist()`` materialises it; ``sum()`` returns the device-side sum folded
    by ``gather_ordered`` when available.

    With ``Pool(results="device")`` the ordered results stay in HBM: ``sum()`` and ``len()`` cost
    nothing, indexing fetches just the requested range, and the full array crosses PCIe only when
    something needs all of it (``array``, ``tolist()``, iteration, ``==``)."""

    def __init__(self, spec, array, device_sum=None, n=None, fetch=None, bits=None):
        self._spec = spec
        self._arr = array
        self._sum = device_sum
        self._n = len(array) if array is not None else n
        self._fetch = fetch            # (lo, hi) -> ndarray, for device-resident results
        self._bits = bits              # Pool(results="bits"): uint8[ceil(n/8)], bit k of byte j = result 8j+k

    @property
    def _a(self):
        if self._arr is None:
            if self._bits is not None:
                self._arr = np.unpackbits(self._bits, count=self._n, bitorder="little").view(np.bool_)
            else:
                self._arr = self._fetch(0, self._n)
        return self._arr

    @property
    def packed(self):
        """The bit-packed results (``Pool(results="bits")``): zero-copy uint8 view of the pinned
        segment, result i at bit ``i & 7`` of byte ``i >> 3``; ``None`` for byte-per-result maps."""
        return self._bits

    @property
    def on_device(self):
        return self._arr is None and self._bits is None

    def __len__(self):
        return self._n

    def __getitem__(self, i):
        if self._arr is None and self._bits is not None:
            # bit-backed: single results and contiguous ranges are read straight from the packed bytes
            if isinstance(i, slice):
                lo, hi, step = i.indices(self._n)
                if step == 1:
                    hi = max(lo, hi)
                    part = np.unpackbits(self._bits[lo >> 3:(hi + 7) >> 3], bitorder="little")
                    return part[lo & 7:(lo & 7) + hi - lo].view(np.bool_).tolist()
            else:
                j = i + self._n if i < 0 else i
                if not 0 <= j < self._n:
                    raise IndexError("ResultArray index out of range")
                return bool((int(self._bits[j >> 3]) >> (j & 7)) & 1)
        elif self._arr is None:
            if isinstance(i, slice):
                lo, hi, step = i.indices(self._n)
                if step == 1:
                    return self._spec.rows_to_list(self._fetch(lo, max(lo, hi)))
            else:
                j = i + self._n if i < 0 else i
                if not 0 <= j < self._n:
                    raise IndexError("ResultArray index out of range")
                return self._spec.to_python(self._fetch(j, j + 1)[0])
        if isinstance(i, slice):
            return self._spec.rows_to_list(self._a[i])
        return self._spec.to_python(self._a[i])

    def __iter__(self):
        step = 1 << 16
        for s in range(0, self._n, step):
            yield from self[s:s + step]

    def __eq__(self, other):
        if isinstance(other, ResultArray):
            if self._bits is not None and other._bits is not None:
                return self._n == other._n and np.array_equal(self._bits, other._bits)
            return np.array_equal(self._a, other._a)
        if isinstance(other, (list, tuple)):
            return len(other) == len(self) and self.tolist() == list(other)
        return NotImplemented

    def __repr__(self):
        n = len(self)
        head = self[:6]
        return "ResultArray(%s%s, len=%d, body=%s%s)" % (head, "..." if n > 6 else "", n, self._spec.name,
                                                         ", bit-packed" if self._bits is not None else
                                                         ", on device" if self.on_device else "")

    def __array__(self, dtype=None, copy=None):
        a = self._a
        return a.astype(dtype) if dtype is not None else a

    @property
    def array(self):
        """Zero-copy NumPy view of the pinned result segment (fetches device-resident results)."""
        return self._a

    def tolist(self):
        return self._spec.rows_to_list(self._a)

    def sum(self):
        if self._sum is not None:
            return self._sum
        if self._bits is not None:
            return int(np.unpackbits(self._bits).sum())   # the bits past n are zero
        return self._spec.sum_rows(self._a)              # what sum() of the reference's list gives, per result layout

    def sort(self):
        raise TypeError("ResultArray is read-only; use sorted(result) or result.tolist()")


class _View:
    """A NumPy-visible block of engine memory that keeps its owner (a map's _Segment) alive."""

    def __init__(self, owner, ptr, nbytes):
        self.owner = owner
        self.__array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr or 0, False), "version": 3}


def _emit_value(spec, arr):
    """One task's values as Python sees them: a list, or bytes / str (device_body(out_as=))."""
    if spec.out_as == "bytes":
        return arr.tobytes()
    if spec.out_as == "str":
        return arr.tobytes().decode("utf-8")
    return arr.tolist()


class EmitResultArray(ResultArray):
    """Ordered results of a map of an emit body: task i's value is a variable-length array, read as a list (or ``bytes`` /
    ``str``, see ``device_body(out_as=)``).  ``ends`` are the n end offsets and ``values`` every task's values back to back,
    both views of the map's pinned segments; ``ragged`` is the whole map as one ``Ragged``.  With ``Pool(results="device")``
    both stay in HBM and ranges are fetched on demand."""

    def __init__(self, spec, ends, values, n=None, fetch=None, fetch_values=None):
        super().__init__(spec, ends, None, n=n, fetch=fetch)
        self._values = values
        self._fetch_values = fetch_values    # (lo, hi) -> ndarray of values [lo, hi), device-resident maps

    def _span(self, lo, hi):
        """End offsets of tasks [lo - 1, hi) (the first is 0 for lo = 0) and the values of tasks [lo, hi)."""
        if self._arr is not None:
            ends = self._arr[max(0, lo - 1):hi]
        else:
            ends = self._fetch(max(0, lo - 1), hi)
        ends = np.concatenate([np.zeros(1, np.uint64), ends]) if lo == 0 else ends
        v0, v1 = int(ends[0]), int(ends[-1])
        vals = self._values[v0:v1] if self._values is not None else self._fetch_values(v0, v1)
        return ends - np.uint64(v0), vals

    def __getitem__(self, i):
        if isinstance(i, slice):
            lo, hi, step = i.indices(self._n)
            if step != 1:
                return [self[j] for j in range(lo, hi, step)]
            hi = max(lo, hi)
            o, vals = self._span(lo, hi)
            return [_emit_value(self._spec, vals[int(o[k]):int(o[k + 1])]) for k in range(hi - lo)]
        j = operator.index(i)
        j = j + self._n if j < 0 else j
        if not 0 <= j < self._n:
            raise IndexError("ResultArray index out of range")
        o, vals = self._span(j, j + 1)
        return _emit_value(self._spec, vals[int(o[0]):int(o[1])])

    def __eq__(self, other):
        if isinstance(other, EmitResultArray):
            return len(self) == len(other) and self.tolist() == other.tolist()
        if isinstance(other, (list, tuple)):
            return len(other) == len(self) and self.tolist() == list(other)
        return NotImplemented

    @property
    def ragged(self):
        """The map's values as ``Ragged(values, offsets)``: values without a copy, offsets = 0 then the end offsets."""
        if self._values is None:
            self._values = self._fetch_values(0, int(self._a[-1]) if self._n else 0)
        return registry.Ragged(self._values, np.concatenate([np.zeros(1, np.uint64), self._a]))

    def tolist(self):
        return self[:]

    def sum(self):
        raise TypeError("unsupported operand type(s) for +: 'int' and 'list' (%s returns a variable-length array per task)"
                        % self._spec.name)


class KeyedResultArray(ResultArray):
    """The result of a keyed fold (``Pool.fold_by_key``): record k is the fold of the results whose ``key()`` is k, read like
    a map result, and ``counts`` (uint64 per key) the number of tasks of each key."""

    def __init__(self, spec, array, counts):
        super().__init__(spec, array)
        self._counts = counts

    @property
    def counts(self):
        return self._counts

    def __repr__(self):
        return "KeyedResultArray(%s%s, n_keys=%d, body=%s)" % (self[:6], "..." if len(self) > 6 else "", len(self), self._spec.name)


class SparseKeyedResultArray(ResultArray):
    """The result of a sparse keyed fold (``Pool.fold_by_sparse_key``): one record per distinct key some task produced, in
    ascending key order, read like a map result; ``keys`` (uint32) are those keys and ``counts`` (uint64) their tasks."""

    def __init__(self, spec, array, keys, counts):
        super().__init__(spec, array)
        self._keys, self._counts = keys, counts

    @property
    def keys(self):
        return self._keys

    @property
    def counts(self):
        return self._counts

    def get(self, key, default=None):
        """The record of ``key``, or ``default`` when no task produced it."""
        i = int(np.searchsorted(self._keys, key))
        return self[i] if i < len(self._keys) and int(self._keys[i]) == key else default

    def __repr__(self):
        return "SparseKeyedResultArray(%s%s, n_groups=%d, body=%s)" % (self[:6], "..." if len(self) > 6 else "", len(self),
                                                                      self._spec.name)


def host_result(spec, kind, data, n=0, total=None, values=None):
    """What a finished map whose results are in host memory returns, in either isolation.  ``kind`` is "plain", "bits"
    (one bit per bool result), "emit" (variable-length results), "fold", "keyed" or "sparse"; ``spec`` is the body the
    caller mapped; ``n`` the number of results the caller sees (a keyed fold's n_keys, a sparse keyed fold's D).  ``data``
    holds the result records as uint8 (the bit-packed bytes, the end offsets of an emit map, a fold's one record, a keyed
    fold's n records then n uint64 counts, a sparse keyed fold's n records, n uint64 counts, then n uint32 keys), or is None
    for a map over no tasks; ``values`` are an emit map's values; ``total`` is the device-side sum, or None."""
    if kind == "sparse":
        dtype, sub = spec.result_dtype()
        R = spec.result_bytes
        if data is None:        # no task: no key
            return SparseKeyedResultArray(spec, np.empty((0,) + sub, dtype), np.empty(0, np.uint32), np.empty(0, np.uint64))
        records = data[:n * R]
        counts = data[n * R:n * (R + 8)].copy().view(np.uint64)
        keys = data[n * (R + 8):n * (R + 12)].copy().view(np.uint32)
        return SparseKeyedResultArray(spec, records.view(dtype).reshape((n,) + sub), keys, counts)
    if kind == "fold":
        return spec.unpack_result(fold_identity(spec) if data is None else bytes(data))
    if kind == "keyed":
        dtype, sub = spec.result_dtype()
        if data is None:        # no task: every key gets identity()
            records = np.frombuffer(fold_identity(spec) * n, np.uint8)
            counts = np.zeros(n, np.uint64)
        else:
            records = data[:n * spec.result_bytes]
            counts = data[n * spec.result_bytes:n * (spec.result_bytes + 8)].copy().view(np.uint64)
        return KeyedResultArray(spec, records.view(dtype).reshape((n,) + sub), counts)
    if kind == "emit":
        if data is None:
            return EmitResultArray(spec, np.empty(0, np.uint64), np.empty(0, spec.out_dtype))
        return EmitResultArray(spec, data.view(np.uint64), values)
    if kind == "bits" and data is not None:
        return ResultArray(spec, None, total, n=n, bits=data)
    dtype, sub = spec.result_dtype()
    if data is None:
        return ResultArray(spec, np.empty((0,) + sub, dtype), 0)
    return ResultArray(spec, data.view(dtype).reshape((n,) + sub), total)


def _n_keys(n_keys):
    """``n_keys`` of a keyed fold as an int in 1 .. FBR_MAX_KEYS: any integer (a NumPy one too), never a bool."""
    try:
        k = operator.index(n_keys) if not isinstance(n_keys, (bool, np.bool_)) else None
    except TypeError:
        k = None
    if k is None or not 1 <= k <= _abi.FBR_MAX_KEYS:
        raise ValueError("n_keys must be an int in 1 .. %d, not %r" % (_abi.FBR_MAX_KEYS, n_keys))
    return k


def _raise_task_error(name, code, task, emit_count=None, n_keys=None):
    """Raise the exception of a map's first failed task (``err_code`` / ``err_task`` of its fbr_result_t) for body
    ``name``; ``emit_count(task)`` gives the number of values an emit body's task was counted to push, and ``n_keys`` is a
    keyed fold's number of keys (0 for a sparse keyed fold)."""
    if code == _abi.FBR_TASK_KEY and not n_keys:
        raise ValueError("%s: key() of task %d is 0xffffffff, which fold_by_sparse_key reserves" % (name, task))
    if code == _abi.FBR_TASK_KEY:
        raise ValueError("%s: key() of task %d is not below n_keys=%d" % (name, task, n_keys))
    if code == _abi.FBR_TASK_EMIT:
        raise RuntimeError("%s: task %d emitted another number of values than the %d its count pass gave"
                           % (name, task, emit_count(task)))
    if code == _abi.FBR_TASK_OVERFLOW:
        raise OverflowError("%s: result of task %d does not fit int64 (Python ints are unbounded; "
                            "the device body refuses to wrap)" % (name, task))
    if code == _abi.FBR_TASK_BADARG:
        raise ValueError("%s: bad argument in task %d" % (name, task))
    raise RuntimeError("%s: task %d failed with device error code %d" % (name, task, code))


class MapResult:
    """Handle of an asynchronous map (fiber/pool.py:731-743)."""

    def __init__(self, pool, engine, spec, seq, n, keepalive, flags=0, user_spec=None, n_items=None, n_keys=0):
        """``flags``: the map's FBR_* flags.  A bit-packed map runs ``spec``, the bit-packed twin of the bool body
        ``user_spec`` the caller mapped, over ``n`` = ceil(n_items / 8) byte tasks.  ``n_keys``: a keyed fold's keys."""
        self._pool, self._engine, self._spec, self._seq, self._n = pool, engine, spec, seq, n
        self._keepalive = keepalive   # argument buffers must outlive the asynchronous H2D copies
        self._flags = flags
        self._user_spec = user_spec or spec
        self._n_items = n if n_items is None else n_items      # the items the caller mapped
        self._n_keys = n_keys
        self._kind = "fold" if flags & _abi.FBR_FOLD else "keyed" if flags & _abi.FBR_FOLD_KEYS else \
            "sparse" if flags & _abi.FBR_FOLD_SPARSE_KEYS else \
            "bits" if user_spec is not None else "emit" if spec.flags & _abi.FBR_BODY_EMIT else "plain"
        self._result = None
        self._exc = None              # a task error is raised again by every later get()
        self._segment = _Segment(engine, seq) if n else None   # owns the seq from submission on

    # -- internal ----------------------------------------------------------------------------
    def _wait(self, timeout=None):
        if self._result is not None:
            return self._result
        if self._exc is not None:
            raise self._exc
        if self._n == 0:
            self._result = host_result(self._user_spec, self._kind, None, self._n_keys)
            return self._result
        res = self._engine_wait(timeout)
        # exact, unbounded sum: the device folds the two halves of int64 results separately (nothing wraps)
        dsum = (int(res.sum_hi) * (1 << 32) + int(res.sum_lo)) if (self._flags & _abi.FBR_WANT_SUM) else None
        self.n_waves = res.n_waves
        if self._kind == "fold":
            self.raw = ctypes.string_at(res.data, res.result_bytes)     # process-isolated pools ship these bytes
            self._result = host_result(self._spec, "fold", self.raw)
        elif self._kind == "keyed":         # n_keys records, then n_keys uint64 counts
            self.raw = ctypes.string_at(res.data, self._n_keys * (res.result_bytes + 8))
            self._result = host_result(self._spec, "keyed", np.frombuffer(self.raw, np.uint8), self._n_keys)
        elif self._kind == "sparse":        # D records (fbr_result_t.data), then D counts and D keys (fbr_result_groups)
            eng, d = self._engine, ctypes.c_uint64(0)
            keys, counts = ctypes.c_void_p(), ctypes.c_void_p()
            _abi.check(eng.lib.fbr_result_groups(eng.handle, self._seq, ctypes.byref(d), ctypes.byref(keys), ctypes.byref(counts)))
            D = d.value
            self.raw = ctypes.string_at(res.data, D * res.result_bytes) + ctypes.string_at(counts, 8 * D) + \
                ctypes.string_at(keys, 4 * D)
            self._result = host_result(self._spec, "sparse", np.frombuffer(self.raw, np.uint8), D)
        elif self._flags & _abi.FBR_RESULTS_ON_DEVICE:
            self._result = self._device_result(res, dsum)
        else:
            data = np.asarray(self._segment.bind(res.data, res.n_tasks * res.result_bytes))
            values = self._values_view() if self._kind == "emit" else None
            if self._kind == "bits" and self._n_items % 8:
                # `data` holds ceil(n/8) bytes.  The body evaluated all 8 indices of the last byte; the ones past the
                # end of the range are dropped here, from the byte and from the folded count.
                last = int(data[-1])
                keep = last & (0xFF >> (-self._n_items) % 8)
                if dsum is not None:
                    dsum -= bin(last ^ keep).count("1")
                data[-1] = keep
            self._result = host_result(self._user_spec, self._kind, data, self._n_items, dsum, values)
        return self._result

    def _device_result(self, res, dsum):
        """A finished map whose results stay in HBM: ranges of its results (and an emit map's values) are fetched on demand."""
        eng, seq, seg = self._engine, self._seq, self._segment       # the segment owns the seq (device buffer) until GC

        def fetcher(call, itemsize, dtype, sub=()):
            def fetch(lo, hi, seg=seg):
                block = _PinnedBlock(eng, max(1, (hi - lo) * itemsize))
                if hi > lo:
                    _abi.check(call(eng.handle, seq, lo, hi - lo, ctypes.c_void_p(block.ptr)))
                return np.asarray(block)[: (hi - lo) * itemsize].view(dtype).reshape((hi - lo,) + sub)
            return fetch
        n = int(res.n_tasks)
        if self._kind == "emit":
            od = self._spec.out_dtype
            return EmitResultArray(self._spec, None, None, n=n, fetch=fetcher(eng.lib.fbr_result_fetch, 8, np.uint64),
                                   fetch_values=fetcher(eng.lib.fbr_result_fetch_values, od.itemsize, od))
        dtype, sub = self._spec.result_dtype()
        return ResultArray(self._spec, None, dsum, n=n, fetch=fetcher(eng.lib.fbr_result_fetch, res.result_bytes, dtype, sub))

    def _engine_wait(self, timeout):
        """fbr_result_wait for a map of n > 0 tasks: its fbr_result_t, or the map's task error raised."""
        res = _abi.Result()
        eng = self._engine
        tmo = -1 if timeout is None else int(timeout * 1000)
        rc = eng.lib.fbr_result_wait(eng.handle, self._seq, tmo, ctypes.byref(res))
        if rc == _abi.FBR_ETIMEOUT:
            raise TimeoutError("map %d not finished" % self._seq)
        if rc == _abi.FBR_ETASK:
            try:
                _raise_task_error(self._user_spec.name, res.err_code, res.err_task, lambda task: self._emit_count(res, task),
                                  self._n_keys)
            except Exception as e:      # noqa: BLE001 -- remembered: later get() calls raise it without touching the engine
                self._exc = e
                raise
        _abi.check(rc)
        self._keepalive = None
        self._pool.recv_tasks += self._n_items
        return res

    def _values_view(self):
        eng, ptr, nv = self._engine, ctypes.c_void_p(), ctypes.c_uint64(0)
        _abi.check(eng.lib.fbr_result_values(eng.handle, self._seq, ctypes.byref(ptr), ctypes.byref(nv)))
        od = self._spec.out_dtype
        return np.asarray(_View(self._segment, ptr.value, nv.value * od.itemsize)).view(od)

    def _emit_count(self, res, task):
        """The number of values task `task` of a failed emit map was counted to push: the difference of its end offsets."""
        lo = max(0, task - 1)
        ends = np.zeros(task + 1 - lo, np.uint64)
        if self._flags & _abi.FBR_RESULTS_ON_DEVICE:
            eng = self._engine
            _abi.check(eng.lib.fbr_result_fetch(eng.handle, self._seq, lo, len(ends), ends.ctypes.data))
        else:
            ctypes.memmove(ends.ctypes.data, res.data + lo * 8, ends.nbytes)
        return int(ends[-1]) - (int(ends[0]) if task > 0 else 0)

    # -- reference surface -------------------------------------------------------------------
    def get(self, timeout=None):
        return self._wait(timeout)

    def _iter_ready(self):
        """Yield results as ordered prefixes become final (per-wave completion events)."""
        if self._n == 0:
            return
        if self._flags & _abi.FBR_RESULTS_ON_DEVICE:
            yield from self._wait()
            return
        eng, values = self._engine, None
        done, emitted, items = ctypes.c_uint64(0), 0, 0
        # peek at the segment: results land in it wave by wave
        while emitted < self._n:
            _abi.check(eng.lib.fbr_result_poll(eng.handle, self._seq, ctypes.byref(done)))
            if done.value >= self._n:
                break
            if done.value > emitted:
                # an ordered prefix is final but the map is not: hand it out from the live segment (an emit map's values
                # of a finished wave are final in its values segment)
                values = self._values_view() if self._kind == "emit" and values is None else values
                part = self._live_prefix(done.value, values)[items:]
                yield from part
                items += len(part)
                emitted = done.value
            else:
                time.sleep(0.0002)
        yield from self._wait()[items:]

    def _live_prefix(self, rows, values):
        """The results of the first ``rows`` result rows of the live segment, read as the finished map reads them.  A
        bit-packed map's row is a byte of 8 results: every byte of a finished wave is a full byte, the (masked) last byte
        of the map only comes from _wait()."""
        eng, ptr = self._engine, ctypes.c_void_p()
        _abi.check(eng.lib.fbr_result_data(eng.handle, self._seq, ctypes.byref(ptr)))   # the engine-owned pinned segment
        data = np.asarray(_View(self._segment, ptr.value, rows * self._spec.result_bytes))
        return host_result(self._user_spec, self._kind, data, 8 * rows if self._kind == "bits" else rows, None, values)

    def iget_ordered(self):
        return self._iter_ready()

    def iget_unordered(self):
        # arrival order == ring order; ordered prefixes are a valid "unordered" stream
        return self._iter_ready()


def fold_identity(spec):
    """The identity() record of fold body ``spec`` as bytes (the result of a fold over no tasks)."""
    lib = _abi.load()
    nb = ctypes.c_uint32(0)
    _abi.check(lib.fbr_body_fold_info(spec.func_id, None, ctypes.byref(nb)))
    buf = ctypes.create_string_buffer(max(1, nb.value))
    _abi.check(lib.fbr_body_fold_info(spec.func_id, buf, ctypes.byref(nb)))
    return buf.raw[:nb.value]


class FoldResult(MapResult):
    """Handle of an asynchronous fold (``Pool.fold_async``): ``get()`` returns tree() over the map's results (FBR_FOLD in
    include/fiber_b200.h), read like one task's result."""

    def _iter_ready(self):
        raise TypeError("%s: a fold has one result, not one per task: use get()" % self._spec.name)


class KeyedFoldResult(MapResult):
    """Handle of an asynchronous keyed fold (``Pool.fold_by_key_async``): ``get()`` returns a KeyedResultArray of n_keys
    records and their counts (FBR_FOLD_KEYS in include/fiber_b200.h)."""

    def _iter_ready(self):
        raise TypeError("%s: a keyed fold has one result per key, not one per task: use get()" % self._spec.name)


class SparseKeyedFoldResult(MapResult):
    """Handle of an asynchronous sparse keyed fold (``Pool.fold_by_sparse_key_async``): ``get()`` returns a
    SparseKeyedResultArray of one record per distinct key, with its keys and counts (FBR_FOLD_SPARSE_KEYS in
    include/fiber_b200.h)."""

    def _iter_ready(self):
        raise TypeError("%s: a sparse keyed fold has one result per distinct key, not one per task: use get()" % self._spec.name)


class ApplyResult(MapResult):
    """fiber/pool.py:746-757: ``get()`` returns the single element."""

    def get(self, timeout=None):
        return self._wait(timeout)[0]


class _Express:
    """Owner of one ``fbr_express_t``: the doorbell lane of one device (resident one-warp kernel)."""
    BODIES = ("square_i64", "mul2_i64", "square_scale_i64", "identity_i64", "pi_inside_det", "sleep_f64")

    def __init__(self, device, idle_us):
        self.lib = _abi.load()
        h = ctypes.c_void_p()
        _abi.xcheck(self.lib.fbr_express_create(device, idle_us, ctypes.byref(h)))
        self.handle = h

    def stats(self):
        served, launches, resident = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_int()
        _abi.xcheck(self.lib.fbr_express_stats(self.handle, ctypes.byref(served), ctypes.byref(launches), ctypes.byref(resident)))
        return {"served": served.value, "kernel_launches": launches.value, "resident": bool(resident.value)}

    def __del__(self):
        h, self.handle = getattr(self, "handle", None), None
        if h:
            self.lib.fbr_express_destroy(h)


class ExpressResult:
    """``ApplyResult`` (fiber/pool.py:746-757) of a task sent through the doorbell lane."""

    def __init__(self, pool, express, spec, ticket):
        self._pool, self._x, self._spec, self._ticket = pool, express, spec, ticket
        self._done, self._value, self._exc = False, None, None

    def __del__(self):
        # handle dropped without a get(): tell the lane to forget the response instead of parking it forever
        x = getattr(self, "_x", None)
        if x is not None and not getattr(self, "_done", True) and x.handle:
            x.lib.fbr_express_discard(x.handle, self._ticket)

    def get(self, timeout=None):
        if self._done:
            if self._exc is not None:
                raise self._exc
            return self._value
        buf = (ctypes.c_uint8 * 48)()
        nbytes, err = ctypes.c_uint32(), ctypes.c_uint32()
        rc = self._x.lib.fbr_express_wait(self._x.handle, self._ticket, buf, ctypes.byref(nbytes), ctypes.byref(err),
                                          -1 if timeout is None else int(timeout * 1000))
        if rc == _abi.FBR_ETIMEOUT:
            raise TimeoutError("apply %d not finished" % self._ticket)
        if rc == _abi.FBR_ETASK:
            self._done = True
            try:
                _raise_task_error(self._spec.name, err.value, 0)
            except Exception as e:      # noqa: BLE001 -- remembered so that a second get() raises again
                self._exc = e
                raise
        _abi.xcheck(rc)
        self._value, self._done = self._spec.unpack_result(bytes(buf[: nbytes.value])), True
        self._pool.recv_tasks += 1
        return self._value


class Pool:
    """H100-native drop-in for ``fiber.Pool`` on the map/starmap/apply path."""

    def __init__(self, processes=None, initializer=None, initargs=(), maxtasksperchild=None,
                 error_handling=False, *, devices=None, ring_bytes=0, timing=False, results="host", express=True,
                 express_idle_us=2000, bind_cpu=False, isolation="thread"):
        self._processes = processes if processes is not None else 1   # fiber/pool.py:894
        if self._processes < 1:
            raise ValueError("Number of processes must be at least 1")
        if initializer is not None and getattr(initializer, "__fbr_init_body__", None) is None:
            # the reference runs initializer(*initargs) inside every worker process
            # (fiber/pool.py:858-859); a host callable cannot run inside a GPU worker.  What the idiom is
            # for -- giving every task the same large arguments once -- is the engine's broadcast block:
            # see fiber_b200.device_initializer.
            raise NotImplementedError("fiber_b200.Pool: Python initializers cannot run on GPU workers; bind the "
                                      "initializer with @fiber_b200.device_initializer(body) to upload initargs as "
                                      "the body's broadcast block")
        self._initializer, self._initargs = initializer, initargs
        self._init_block = None   # (body name, blob, handle): initargs uploaded once per worker at start
        self._maxtasksperchild = maxtasksperchild
        self._error_handling = bool(error_handling)
        self._devices = list(devices) if devices is not None else None
        self._ring_bytes = int(ring_bytes)
        self._timing = bool(timing)
        if results not in ("host", "bytes", "device", "bits"):
            raise ValueError("results must be 'host' (pinned result segment; bool results packed one bit each), "
                             "'bytes' (pinned result segment, one byte per bool), 'device' (stay in HBM, fetched "
                             "lazily) or 'bits' (same as 'host')")
        self._results_on_device = results == "device"
        # A bool needs one bit: bool bodies with a bit-packed twin run through it by default, so the ring, the
        # ordered output and the D2H copy move n/8 bytes.  ResultArray hides the layout; 'bytes' opts out.
        self._results_bits = results in ("host", "bits")
        self._use_express = bool(express) and not self._error_handling
        self._express_idle_us = int(express_idle_us)
        self._express = None
        # concurrent first apply calls must create ONE lane: unserialised, two threads could each create one, submit on
        # one and wait on the other ("unknown express ticket"; tests/test_fuzz_gpu.py::test_concurrent_submitters_share_one_pool)
        self._express_lock = threading.Lock()
        if isolation not in ("thread", "process"):
            raise ValueError("isolation must be 'thread' (workers are devices of this process) or 'process' (one worker process "
                             "per GPU: the only fault domain CUDA offers -- see fiber_b200/procpool.py)")
        self._isolation = isolation
        self._proc = None                    # ProcessPool when isolation == "process"
        self._attempt = 0                    # re-dispatch count stamped on submitted blocks (set by process-pool workers)
        self._bind_cpu = bool(bind_cpu)      # one process per GPU: keep pinned segments on the GPU's NUMA node
        self.bound_cpus = []
        self._state = RUN
        self._engine = None
        self._worker_handler_started = False
        self._meta = None
        self._live = {}         # seq -> data pointer of the engine-owned segment (for imap peeks)
        self._shared_cache = collections.OrderedDict()
        self.sent_tasks = 0     # fiber/pool.py:902-903
        self.recv_tasks = 0

    def __repr__(self):
        return "<{}({}, {})>".format(type(self).__name__, self._processes,
                                     self._engine.devices if self._engine else None)

    # -- workers (fiber/pool.py:1118-1137, 1405-1422) ---------------------------------------------
    def start_workers(self):
        if self._isolation == "process":
            if self._proc is None:
                from .procpool import ProcessPool
                init = None
                if self._initializer is not None:
                    # every worker process runs the initializer (fiber/pool.py:858-859): it uploads initargs itself.
                    # Bad initargs raise here, as with thread isolation, instead of killing every worker process at start
                    body = self._initializer.__fbr_init_body__
                    registry.spec(body).shared_block(*self._initargs)
                    init = (body, tuple(self._initargs), registry.module_of(body))
                lib = _abi.load()
                n = ctypes.c_int(0)
                _abi.check(lib.fbr_device_count(ctypes.byref(n)))            # counts devices, creates no context
                if n.value == 0:
                    raise _abi.EngineError(_abi.FBR_ENODEV, "no CUDA device visible; fiber_b200 has no CPU fallback")
                devs = self._devices if self._devices is not None else list(range(n.value))
                self._proc = ProcessPool(self._processes, devs, results="bytes" if not self._results_bits else "host",
                                         redispatch=self._error_handling, init=init)
            self._proc.start()
            self._worker_handler_started = True
            return
        if self._engine is None:
            lib = _abi.load()
            n = ctypes.c_int(0)
            _abi.check(lib.fbr_device_count(ctypes.byref(n)))
            if self._devices is not None:
                devs = self._devices
            else:
                # one worker per GPU; more requested processes than GPUs fold onto the GPUs we have
                devs = list(range(min(self._processes, n.value)))
            if self._bind_cpu and len(devs) == 1:
                from .affinity import bind_to_device
                self.bound_cpus = bind_to_device(devs[0])
            self._engine = _Engine(len(devs), devs, self._ring_bytes, self._timing)
            if self._initializer is not None:
                # initializer(*initargs) in every worker (fiber/pool.py:858-859) == one broadcast block per device
                body = self._initializer.__fbr_init_body__
                blob = registry.spec(body).shared_block(*self._initargs)
                self._init_block = (body, blob, self._shared_handle(blob))
        self._worker_handler_started = True

    def lazy_start_workers(self, func):
        meta = getattr(func, "__fiber_meta__", None)
        if meta is not None and meta != self._meta:
            if self._worker_handler_started and self._meta is not None:
                raise RuntimeError(
                    "Cannot run function that has different resource "
                    "requirements acceptable by this pool. Try creating a "
                    "different pool for it.")
            self._meta = meta
        if not self._worker_handler_started:
            self.start_workers()

    def wait_until_workers_up(self):
        self.start_workers()
        if self._proc is not None:
            self._proc.wait_until_workers_up()

    @property
    def n_jobs(self):
        """Jobs the reference would start for this pool: ceil(processes / cpu_per_job)
        (fiber/pool.py:1405-1408)."""
        from . import config
        return n_jobs(self._processes, config.cpu_per_job)

    @property
    def n_workers(self):
        self.start_workers()
        return self._engine.n_workers

    # -- submission ----------------------------------------------------------------------------------
    def _check_running(self):
        if self._state != RUN:
            raise ValueError("Pool is not running")

    def _shared_handle(self, blob):
        # the very same bytes object as last time (the encoder's block cache): no need to fingerprint 80-160 KB again
        last = getattr(self, "_last_shared", None)
        if last is not None and last[0] is blob and last[1] in self._shared_cache:
            return self._shared_cache[last[1]]
        key = registry.fingerprint(blob)
        self._last_shared = (blob, key)
        hit = self._shared_cache.get(key)
        if hit is not None:
            self._shared_cache.move_to_end(key)
            return hit
        eng = self._engine
        buf = np.frombuffer(blob, dtype=np.uint8)
        h = ctypes.c_uint64(0)
        _abi.check(eng.lib.fbr_shared_put(eng.handle, buf.ctypes.data, buf.nbytes, ctypes.byref(h)))
        self._shared_cache[key] = h.value
        while len(self._shared_cache) > 8:
            _, old = self._shared_cache.popitem(last=False)
            eng.lib.fbr_shared_drop(eng.handle, old)
        return h.value

    def _submit(self, func, enc, kind, chunksize, cls=MapResult, want_sum=True, extra_flags=0, spec=None, user_spec=None,
                n_keys=0):
        spec = spec or registry.spec(registry.body_name_of(func))
        eng = self._engine
        d = _abi.MapDesc()
        d.func_id = spec.func_id
        flags = kind | extra_flags
        if self._results_on_device:
            flags |= _abi.FBR_RESULTS_ON_DEVICE
        if self._error_handling:
            # ResilientZPool (fiber/context.py:42-43): units whose worker dies are re-dispatched
            flags |= _abi.FBR_RESILIENT
        if want_sum and (spec.flags & _abi.FBR_BODY_SUMMABLE):
            flags |= _abi.FBR_WANT_SUM
        d.n_tasks = enc.n
        d.chunksize = chunksize
        d.arg_stride = enc.arg_stride
        keep = [enc.args]
        if enc.args is not None and enc.n:
            d.args = enc.args.ctypes.data
        d.index_start, d.index_step = enc.index_start, enc.index_step
        if enc.shared is not None:
            d.shared = self._shared_handle(enc.shared)
            d.shared_bytes = len(enc.shared)
            flags |= _abi.FBR_SHARED_HANDLE
        elif spec.flags & _abi.FBR_BODY_NEEDS_SHARED:
            # tasks without their own shared arguments read the block the pool's initializer uploaded
            if self._init_block is None or self._init_block[0] != spec.name:
                raise TypeError("%s: tasks carry no shared arguments and the pool has no initializer block for this "
                                "body (Pool(initializer=<@device_initializer(%r)>, initargs=...))" % (spec.name, spec.name))
            d.shared = self._shared_handle(self._init_block[1])
            d.shared_bytes = len(self._init_block[1])
            flags |= _abi.FBR_SHARED_HANDLE
        d.n_items = enc.n_items
        d.task_index_base = enc.task_index_base
        d.attempt = self._attempt
        d.n_keys = n_keys
        d.flags = flags
        seq = ctypes.c_uint64(0)
        if enc.n and enc.streams is not None:
            streams = (_abi.ItemsDesc * len(enc.streams))()
            for it, (values, offsets) in zip(streams, enc.streams):
                keep += [values, offsets]
                it.items, it.offsets = values.ctypes.data, offsets.ctypes.data
                it.n_items, it.item_bytes = len(values), values.dtype.itemsize
            _abi.check(eng.lib.fbr_map_submit_items_n(eng.handle, ctypes.byref(d), streams, len(streams), ctypes.byref(seq)))
        elif enc.n:
            _abi.check(eng.lib.fbr_map_submit(eng.handle, ctypes.byref(d), ctypes.byref(seq)))
        n_items = enc.n if user_spec is None else enc.n_items
        self.sent_tasks += n_items
        return cls(self, eng, spec, seq.value, enc.n, keep, flags, user_spec, n_items, n_keys)

    @staticmethod
    def _spec_of(func):
        return registry.spec(registry.body_name_of(func))

    def _start(self, func, iterable, *, star, mode, chunksize=None, streaming=False, n_keys=0):
        """The one submission path of maps (``mode`` "map"), folds, keyed folds ("fold_by_key"), sparse keyed folds
        ("fold_by_sparse_key") and accumulates of ``func`` over ``iterable``, whose items are argument tuples with ``star``:
        a MapResult, a FoldResult for a fold, a KeyedFoldResult for a keyed fold or a SparseKeyedFoldResult for a sparse one."""
        self._check_running()
        if chunksize is None:
            chunksize = DEFAULT_CHUNKSIZE if mode == "map" else 0     # a fold's order does not depend on a chunksize
        spec = self._spec_of(func) if mode == "map" else \
            self._fold_spec(func, scan=mode == "accumulate", keyed=mode in ("fold_by_key", "fold_by_sparse_key"))
        if mode == "fold_by_key":
            n_keys = _n_keys(n_keys)
        if not hasattr(iterable, "__len__"):
            iterable = list(iterable)
        self.lazy_start_workers(func)
        if self._proc is not None:
            return self._submit_proc(spec, ("star" if star else "") + mode, iterable, chunksize, n_keys)
        # imap wants ordered prefixes as they complete: results are staged and copied out wave by wave instead of being
        # stored straight into the pinned segment by one kernel (zero copy, final only when the whole block is)
        cls, want_sum, flags = {"map": (MapResult, True, _abi.FBR_NO_ZERO_COPY if streaming else 0),
                                "fold": (FoldResult, False, _abi.FBR_FOLD),
                                "fold_by_key": (KeyedFoldResult, False, _abi.FBR_FOLD_KEYS),
                                "fold_by_sparse_key": (SparseKeyedFoldResult, False, _abi.FBR_FOLD_SPARSE_KEYS),
                                "accumulate": (MapResult, False, _abi.FBR_SCAN)}[mode]
        if mode != "map" and len(iterable) == 0:          # identity() / no prefixes: nothing to bind or submit
            return cls(self, self._engine, spec, 0, 0, None, flags, n_keys=n_keys)
        enc = spec.encode_starmap(iterable) if star else spec.encode_map(iterable)
        kind = _abi.FBR_STARMAP if star else _abi.FBR_MAP
        if mode == "map" and self._results_bits and spec.name in registry.BITS_TWIN:
            # A bool needs one bit: the twin body evaluates 8 consecutive items (range() indices or argument
            # records) per result byte, so the ring, the ordered output and the D2H copy move n/8 bytes.
            twin = registry.spec(registry.BITS_TWIN[spec.name])
            return self._submit(func, twin.from_encoded(enc), kind, max(1, chunksize // 8), extra_flags=flags, spec=twin,
                                user_spec=spec)
        return self._submit(func, enc, kind, chunksize, cls=cls, want_sum=want_sum, extra_flags=flags, spec=spec, n_keys=n_keys)

    def _submit_proc(self, spec, kind, items, chunksize, n_keys=0):
        """Process-isolated workers: the map is cut into blocks that worker processes pull (procpool.py).  ``kind`` is the
        block kind: "map", "apply", "fold", "fold_by_key" (with ``n_keys``), "fold_by_sparse_key" or "accumulate", with "star" in front for
        argument tuples."""
        if (kind.startswith("star") and not isinstance(items, registry.Columns)) or \
                not isinstance(items, (range, list, np.ndarray, registry.Ragged, registry.Columns)):
            items = list(items)         # a Ragged (or Columns) stays one: its blocks are slices with rebased offsets
        if kind == "map" and len(items):
            spec.encode_map(items[:1] if not isinstance(items, range) else items)      # argument validation up front
        twin = registry.BITS_TWIN.get(spec.name) if self._results_bits and kind in ("map", "starmap") else None
        r = self._proc.submit(spec, twin, kind, items, chunksize, single=kind in ("apply", "fold", "starfold"), n_keys=n_keys)
        self.sent_tasks += len(items)
        return r

    def map_async(self, func, iterable, chunksize=None, callback=None, error_callback=None, _streaming=False):
        if error_callback:
            raise NotImplementedError
        return self._start(func, iterable, star=False, mode="map", chunksize=chunksize, streaming=_streaming)

    def map(self, func, iterable, chunksize=None):
        return self.map_async(func, iterable, chunksize).get()

    def starmap_async(self, func, iterable, chunksize=None, callback=None, error_callback=None):
        return self._start(func, iterable, star=True, mode="map", chunksize=chunksize)

    def starmap(self, func, iterable, chunksize=None):
        return self.starmap_async(func, iterable, chunksize).get()

    # -- folds: a map reduced on the device with the body's combine() ------------------------------------------------
    def _fold_spec(self, func, scan=False, keyed=False):
        spec = self._spec_of(func)
        if not spec.flags & _abi.FBR_BODY_FOLD:
            if not spec.flags & _abi.FBR_BODY_RECORD:
                hint = "thread bodies do not fold; sum(pool.map(f, xs)) sums their results on the device"
            else:
                hint = "a record body folds when it defines identity() and combine() next to run()"
            raise TypeError("%s cannot fold: it has no combine() (%s)" % (spec.name, hint))
        if scan and not spec.flags & _abi.FBR_BODY_SCAN:
            raise TypeError("%s cannot accumulate: its module exports no scan entry (rebuild it with "
                            "FBR_EXPORT_RECORD_BODY)" % spec.name)
        if keyed and not spec.flags & _abi.FBR_BODY_KEYED:
            raise TypeError("%s cannot fold by key: it has no key() (a fold body groups its results when it defines "
                            "`__device__ static uint32_t key(const Res& r)` next to combine())" % spec.name)
        return spec

    def fold_async(self, func, iterable):
        """``functools.reduce(combine, map(func, iterable))`` on the device, in the fixed order tree() of FBR_FOLD
        (include/fiber_b200.h): a FoldResult.  There is no chunksize, since the order does not depend on one."""
        return self._start(func, iterable, star=False, mode="fold")

    def fold(self, func, iterable):
        return self.fold_async(func, iterable).get()

    def starfold_async(self, func, iterable):
        """``fold_async`` over argument tuples, bound as ``starmap`` binds them."""
        return self._start(func, iterable, star=True, mode="fold")

    def starfold(self, func, iterable):
        return self.starfold_async(func, iterable).get()

    # -- keyed folds: a fold per key() of the results, on the device -------------------------------------------------
    def fold_by_key_async(self, func, iterable, n_keys):
        """A fold of the results of each key: a KeyedFoldResult whose ``get()`` gives a KeyedResultArray of ``n_keys``
        records, record k the fold of the results whose body ``key()`` is k in the order of FBR_FOLD_KEYS
        (include/fiber_b200.h) -- on one worker ``fold(func, [x for x in iterable if key(func(x)) == k])`` bit for bit, and
        identity() for a key without tasks -- and ``counts``, the tasks of each key.  There is no chunksize, as for
        ``fold``.  A task whose key is not below ``n_keys`` raises ValueError."""
        return self._start(func, iterable, star=False, mode="fold_by_key", n_keys=n_keys)

    def fold_by_key(self, func, iterable, n_keys):
        return self.fold_by_key_async(func, iterable, n_keys).get()

    def starfold_by_key_async(self, func, iterable, n_keys):
        """``fold_by_key_async`` over argument tuples, bound as ``starmap`` binds them."""
        return self._start(func, iterable, star=True, mode="fold_by_key", n_keys=n_keys)

    def starfold_by_key(self, func, iterable, n_keys):
        return self.starfold_by_key_async(func, iterable, n_keys).get()

    # -- sparse keyed folds: a fold per distinct uint32 key() of the results, on the device -----------------------------
    def fold_by_sparse_key_async(self, func, iterable):
        """A fold of the results of each distinct key: a SparseKeyedFoldResult whose ``get()`` gives a
        SparseKeyedResultArray with one record per key some task produced, in ascending key order -- record k the fold of
        the results whose body ``key()`` is k in the order of FBR_FOLD_SPARSE_KEYS (include/fiber_b200.h), on one worker
        ``fold(func, [x for x in iterable if key(func(x)) == k])`` bit for bit -- with ``keys`` and ``counts``.  Keys are
        any uint32 but 0xFFFFFFFF, which is reserved: a task whose key is 0xFFFFFFFF raises ValueError.  There is no
        chunksize, as for ``fold``."""
        return self._start(func, iterable, star=False, mode="fold_by_sparse_key")

    def fold_by_sparse_key(self, func, iterable):
        return self.fold_by_sparse_key_async(func, iterable).get()

    def starfold_by_sparse_key_async(self, func, iterable):
        """``fold_by_sparse_key_async`` over argument tuples, bound as ``starmap`` binds them."""
        return self._start(func, iterable, star=True, mode="fold_by_sparse_key")

    def starfold_by_sparse_key(self, func, iterable):
        return self.starfold_by_sparse_key_async(func, iterable).get()

    # -- accumulates: every prefix of a fold, on the device ------------------------------------------------------------
    def accumulate_async(self, func, iterable):
        """``itertools.accumulate(map(func, iterable), combine)`` on the device: a MapResult whose record i is the fold of
        results 0 .. i in the order of FBR_SCAN (include/fiber_b200.h) -- on one worker ``fold(func, iterable[:i + 1])``
        bit for bit, and the last record is always ``fold(func, iterable)``.  There is no chunksize, as for ``fold``."""
        return self._start(func, iterable, star=False, mode="accumulate")

    def accumulate(self, func, iterable):
        return self.accumulate_async(func, iterable).get()

    def staraccumulate_async(self, func, iterable):
        """``accumulate_async`` over argument tuples, bound as ``starmap`` binds them."""
        return self._start(func, iterable, star=True, mode="accumulate")

    def staraccumulate(self, func, iterable):
        return self.staraccumulate_async(func, iterable).get()

    def apply_async(self, func, args=(), kwds={}, callback=None, error_callback=None):
        self._check_running()
        spec = self._spec_of(func)
        self.lazy_start_workers(func)
        if self._proc is not None:
            return self._submit_proc(spec, "apply", [(tuple(args), dict(kwds))], 1)
        if self._use_express and spec.name in _Express.BODIES:
            # one task whose record fits the doorbell lane: no kernel launch / copy on the round trip
            rec = spec.pack_apply(args, kwds)
            with self._express_lock:
                if self._express is None:
                    self._express = _Express(self._engine.devices[0], self._express_idle_us)
                x = self._express
            ticket = ctypes.c_uint64()
            _abi.xcheck(x.lib.fbr_express_submit(x.handle, spec.func_id, rec, len(rec), ctypes.byref(ticket)))
            self.sent_tasks += 1
            return ExpressResult(self, x, spec, ticket.value)
        return self._submit(func, spec.encode_apply(args, kwds), _abi.FBR_APPLY, 1, cls=ApplyResult, want_sum=False)

    def apply(self, func, args=(), kwds={}):
        return self.apply_async(func, args, kwds).get()

    def imap(self, func, iterable, chunksize=1):
        r = self.map_async(func, iterable, chunksize, _streaming=True)
        return iter(r.get()) if self._proc is not None else r.iget_ordered()

    def imap_unordered(self, func, iterable, chunksize=1):
        return self.imap(func, iterable, chunksize)     # arrival order == ring order: ordered prefixes are a valid "unordered" stream

    # -- shutdown (fiber/pool.py:1332-1403) -----------------------------------------------------------
    def close(self):
        if self._state == RUN:
            self._state = CLOSE
            if self._proc is not None:
                self._proc.close()
            if self._engine is not None:
                self._engine.lib.fbr_pool_close(self._engine.handle)

    def terminate(self):
        self._state = TERMINATE
        if self._proc is not None:
            self._proc.terminate()
        if self._engine is not None:
            self._engine.lib.fbr_pool_terminate(self._engine.handle)

    def join(self):
        assert self._state in (TERMINATE, CLOSE)
        if self._proc is not None:
            self._proc.join()
        if self._engine is not None:
            _abi.check(self._engine.lib.fbr_pool_join(self._engine.handle))

    # -- extras ------------------------------------------------------------------------------------------
    def pinned_empty(self, shape, dtype=np.uint8):
        """NumPy array in pinned host memory owned by this pool: argument records built in it are
        copied to the GPU by DMA without an intermediate staging copy."""
        self.start_workers()
        dtype = np.dtype(dtype)
        shape = (shape,) if isinstance(shape, int) else tuple(shape)
        nbytes = int(np.prod(shape, dtype=np.int64)) * dtype.itemsize
        block = _PinnedBlock(self._engine, nbytes)
        return np.asarray(block).view(dtype).reshape(shape)

    def stats(self):
        """``fbr_pool_stats`` as a dict (extends the reference's sent_tasks/recv_tasks counters)."""
        self.start_workers()
        if self._proc is not None:
            return dict(self._proc.stats)
        s = _abi.Stats()
        _abi.check(self._engine.lib.fbr_pool_stats(self._engine.handle, ctypes.byref(s)))
        d = s.as_dict()
        if self._express is not None:
            d["express"] = self._express.stats()
        return d

    def reset_stats(self):
        self.start_workers()
        _abi.check(self._engine.lib.fbr_pool_stats_reset(self._engine.handle))


def n_jobs(processes, cpu_per_job=1):
    """Number of job-backed workers the reference would start (fiber/pool.py:1405-1408)."""
    return math.ceil(float(processes) / cpu_per_job)
