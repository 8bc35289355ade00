"""Process-isolated workers: the resilient pool's real fault domain.

The reference's ``ResilientZPool`` survives the death of a worker *process*: the master notices the exit
(fiber/pool.py:1623-1656), re-queues the chunks that worker had pending (``:1635-1654``) and a fresh worker is started
(``_maintain_workers``, ``:1009-1057``).  On a GPU the matching fault is a kernel that traps, touches an illegal
address or hits an ECC error -- and CUDA makes such an error sticky for the whole *process*: every context the process
holds, on every device, rejects all further work (a ``trap`` on device 0 of an in-process ``Pool(2)`` takes device 1
down with "unspecified launch failure" too, with or without peer access).  The only fault domain CUDA
offers is therefore the process, exactly as in the reference.

``Pool(processes, error_handling=True, isolation="process")`` gives every worker its own process (``spawn``), each with
its own engine (``fiber_b200.Pool(1, devices=[k])``).  The master holds no CUDA context.  A map is cut into blocks
(the reference's chunks, ``:1084-1087``); idle workers pull blocks (REQ/REP dispatch, ``:1526-1542``); a block's ordered
results land in a shared-memory segment at their final offset (placement by index, ``:672``); a worker that dies --
its engine reports ``FBR_ECUDA``, or the process just disappears -- has its block re-queued with ``attempt + 1`` and is
replaced by a fresh process.  Everything a worker computes still runs through the C ABI on its GPU; there is no CPU
fallback here either.
"""
import collections
import contextlib
import mmap
import multiprocessing as mp
import multiprocessing.connection as mpc
import os
import pickle
import sys
import threading
import time
import weakref

import numpy as np

from . import _abi

BLOCK_ALIGN = 32768          # tasks: a multiple of every claim unit and of 8 (bit-packed bytes stay whole)
MAX_ATTEMPTS = 6
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class WorkerDied(RuntimeError):
    pass


class SharedSegment:
    """A result segment every worker process can write into: a file in /dev/shm, mmap()ed by the master and by
    the workers (plain POSIX shared memory; ``multiprocessing.shared_memory`` would hand the segment to a resource
    tracker that unlinks it when the first worker exits)."""

    def __init__(self, name, size=None):
        self.name = name
        path = os.path.join("/dev/shm", name)
        if size is not None:                                     # create (master)
            fd = os.open(path, os.O_CREAT | os.O_EXCL | os.O_RDWR, 0o600)
            os.ftruncate(fd, max(1, size))
            self.owner = True
        else:                                                    # attach (worker)
            fd = os.open(path, os.O_RDWR)
            self.owner = False
        try:
            self.map = mmap.mmap(fd, 0)
        finally:
            os.close(fd)
        self.array = np.frombuffer(self.map, dtype=np.uint8)

    def release(self):
        if self.owner:
            try:
                os.unlink(os.path.join("/dev/shm", self.name))
            except FileNotFoundError:
                pass
            self.owner = False


def values_name(shm_name, blk):
    """The /dev/shm name of block ``blk``'s values in a map of an emit body (variable-length results): each block's end
    offsets land in the map's segment like any result records (block-local: they start from 0), its values in a file of
    their own, which the master concatenates in block order, rebasing the offsets, at get()."""
    return "%s_v%d" % (shm_name, blk)


def put_values(name, values):
    """Worker side: write a block's values (a 1-D array) to /dev/shm under ``name``.  Written to a private name, then
    renamed, so a re-dispatched block replaces an earlier attempt's file whole."""
    path = os.path.join("/dev/shm", name)
    tmp = "%s.%d.tmp" % (path, os.getpid())
    np.ascontiguousarray(values).tofile(tmp)
    os.replace(tmp, path)


def _unlink_values(shm_name, n_blocks):
    for b in range(n_blocks):
        try:
            os.unlink(os.path.join("/dev/shm", values_name(shm_name, b)))
        except FileNotFoundError:
            pass


# ------------------------------------------------------------------------------------------------
# worker side
# ------------------------------------------------------------------------------------------------
def _proxy_for(body):
    """A callable bound to device body ``body`` (the worker maps by body name, like the reference's workers call
    the function they unpickled by reference)."""
    from . import registry

    def proxy(*a, **k):
        raise RuntimeError("bound to device body %s" % body)
    registry.bind(proxy, body)
    return proxy


def _initializer_for(body):
    """A pool initializer bound to the broadcast block of device body ``body`` (the worker runs the master's initializer,
    like every worker of the reference runs ``initializer(*initargs)``)."""
    from . import registry

    def initializer(*a):
        raise RuntimeError("bound to the broadcast block of device body %s" % body)
    return registry.device_initializer(body)(initializer)


def _register(body, module):
    """Register device body ``body`` from ``module`` (``registry.module_of`` in the master) if this process lacks it."""
    from . import registry
    if module is not None and body not in registry.body_names():
        registry.register_module(body, *module)


def _attach(segments, name):
    """This worker's mapping of the map segment ``name``: one live segment per worker is enough."""
    seg = segments.get(name)
    if seg is None:
        segments.clear()
        seg = segments[name] = SharedSegment(name)
    return seg


@contextlib.contextmanager
def _reporting(conn, job, blk):
    """One step of map ``job`` (block ``blk``, -1 for a map's last step) in a worker: a failure is sent to the master as
    "error", except a lost CUDA context, which is sent as "dead" and ends the process."""
    try:
        yield
    except _abi.EngineError as e:
        if e.status == _abi.FBR_ECUDA:
            # the CUDA context of this process is gone for good: report and die, the master re-queues the work
            try:
                conn.send(("dead", job, blk, str(e)))
            finally:
                os._exit(3)
        conn.send(("error", job, blk, "EngineError", str(e)))
    except (OverflowError, ValueError, TypeError, RuntimeError, KeyError, OSError) as e:   # OSError: the segment of a failed map is gone
        conn.send(("error", job, blk, type(e).__name__, str(e)))


def gpu_worker_main(device, conn, results, sys_path, init=None):
    """Worker process: one engine on one GPU, blocks in, ordered result bytes out (into shared memory).  ``init``:
    (body, initargs, module) of the pool's initializer, or None."""
    for p in sys_path:
        if p not in sys.path:
            sys.path.insert(0, p)
    import fiber_b200
    from fiber_b200 import registry
    kw = {}
    if init is not None:
        body, initargs, module = init
        _register(body, module)
        kw = {"initializer": _initializer_for(body), "initargs": initargs}
    pool = fiber_b200.Pool(1, devices=[device], express=False, results=results, **kw)
    pool.start_workers()
    proxies, segments = {}, {}
    conn.send(("ready", os.getpid()))
    while True:
        msg = conn.recv()
        if msg is None:
            break
        if msg[0] == "fold":
            _fold_totals_in_worker(pool, conn, segments, msg)
            continue
        if msg[0] == "scan":
            _scan_blocks_in_worker(pool, conn, segments, msg)
            continue
        _, job, blk, body, kind, chunksize, payload, shm_name, off, attempt, module = msg
        with _reporting(conn, job, blk):
            _register(body, module)
            spec = registry.spec(body)
            f = proxies.get(body) or proxies.setdefault(body, _proxy_for(body))
            items = range(*payload[1]) if payload[0] == "range" else pickle.loads(payload[1])
            pool._attempt = attempt
            # the block runs as the same kind of map of a thread-isolated pool: an accumulate block gives its own prefix folds
            mode = kind.removeprefix("star")
            if mode == "apply":
                handle = pool.apply_async(f, items[0][0], items[0][1])
            else:
                handle = pool._start(f, items, star=mode != kind, mode=mode, chunksize=chunksize)
            res = handle._wait()
            if mode == "fold":                                     # the block's total, R bytes
                raw = np.frombuffer(handle.raw, np.uint8)
            else:
                raw = res.packed if res.packed is not None else np.ascontiguousarray(np.asarray(res)).view(np.uint8).reshape(-1)
            _attach(segments, shm_name).array[off:off + raw.nbytes] = raw      # placement by index (fiber/pool.py:672), block-wise
            if spec.flags & _abi.FBR_BODY_EMIT:
                put_values(values_name(shm_name, blk), res.ragged.values)   # an emit body: the block's values beside it
            total = res.sum() if (spec.flags & _abi.FBR_BODY_SUMMABLE) else None
            del res, raw
            conn.send(("done", job, blk, total))
    os._exit(0)


def _fold_values(pool, spec, records, count):
    """tree() over ``count`` result records of body ``spec`` (uint8, back to back) in their order, by fbr_fold_values."""
    out = np.zeros(spec.result_bytes, np.uint8)
    src = np.ascontiguousarray(records)
    _abi.check(pool._engine.lib.fbr_fold_values(pool._engine.handle, spec.func_id, src.ctypes.data, count, out.ctypes.data))
    return out


def _scan_pieces(fold, totals, b):
    """The pieces G_1 .. G_m of block b (largest first): fold(lo, count) over the aligned power-of-two ranges of the block
    totals before it given by the set bits of b."""
    return [fold((b >> (k + 1)) << (k + 1), 1 << k) for k in range(b.bit_length() - 1, -1, -1) if (b >> k) & 1]


def _scan_blocks_in_worker(pool, conn, segments, msg):
    """An accumulate map's last step, in the worker the master picked: each listed block b > 0 of the map's segment (its own
    prefix folds) is wrapped with the pieces of the block totals before it (fbr_fold_values), right-nested
    (fbr_scan_values).  The totals come from the master, read before any block was wrapped, so a step sent again after a
    death wraps the blocks still listed exactly as the first attempt would have.  Each block is wrapped in a private copy,
    placed, and reported ("scanned"), so the master never lists a placed block again."""
    from fiber_b200 import registry
    _, job, ranges, todo, totals, body, shm_name, module = msg
    with _reporting(conn, job, -1):
        _register(body, module)
        spec = registry.spec(body)
        R = spec.result_bytes
        seg = _attach(segments, shm_name)
        eng = pool._engine
        tot = np.frombuffer(totals, np.uint8)

        def fold(k, count):
            return _fold_values(pool, spec, tot[k * R:(k + count) * R], count)

        for b in todo:
            lo, hi = ranges[b]
            pieces = np.concatenate(_scan_pieces(fold, tot, b))
            recs = np.array(seg.array[lo * R:hi * R])
            _abi.check(eng.lib.fbr_scan_values(eng.handle, spec.func_id, pieces.ctypes.data, len(pieces) // R,
                                               recs.ctypes.data, hi - lo))
            seg.array[lo * R:hi * R] = recs
            conn.send(("scanned", job, b))
        conn.send(("folded", job))


def _fold_totals_in_worker(pool, conn, segments, msg):
    """A fold map's last step, in the worker the master picked: the n_blocks totals after the result record in the map's
    segment, folded in block order by fbr_fold_values into the result record (the segment's first R bytes)."""
    from fiber_b200 import registry
    _, job, n_blocks, body, shm_name, module = msg
    with _reporting(conn, job, -1):
        _register(body, module)
        spec = registry.spec(body)
        R = spec.result_bytes
        seg = _attach(segments, shm_name)
        seg.array[:R] = _fold_values(pool, spec, seg.array[R:(1 + n_blocks) * R], n_blocks)
        conn.send(("folded", job))


# ------------------------------------------------------------------------------------------------
# master side
# ------------------------------------------------------------------------------------------------
class _Worker:
    def __init__(self, index, device):
        self.index, self.device = index, device
        self.proc = self.conn = None
        self.block = None          # (job, blk) in flight
        self.ready = False


class _Job:
    def __init__(self, jid, body, kind, chunksize, n, result_bytes, bits, blocks, payload_of, module, out_dtype=None):
        self.id, self.body, self.kind, self.chunksize, self.n = jid, body, kind, chunksize, n
        # fold maps: the segment holds the result record, then each block's total in block order
        self.fold = kind in ("fold", "starfold")
        # accumulate maps: each block places its own prefix folds like a map; blocks after the first are wrapped at the end
        self.scan = kind in ("accumulate", "staraccumulate")
        self.scan_wrapped = set()                     # blocks (b > 0) already wrapped and placed
        self.scan_totals = None                       # every block's total, read once before the first wrap
        self.result_bytes, self.bits = result_bytes, bits
        self.out_dtype = out_dtype                    # emit bodies: the values' dtype (blocks put them in files of their own)
        self.ranges = [(lo, hi) for _, lo, hi, _ in blocks]
        self.blocks = collections.deque(blocks)       # (blk id, lo, hi, attempt)
        self.n_blocks, self.done_blocks = len(blocks), 0
        self.payload_of, self.module = payload_of, module
        nbytes = ((n + 7) // 8) if bits else ((1 + len(blocks)) * result_bytes if self.fold else n * result_bytes)
        self.shm = SharedSegment("fbr_%d_%d_%d" % (os.getpid(), jid, int(time.time() * 1e6) & 0xFFFFFF), nbytes) if n else None
        self.nbytes = nbytes
        self.sum, self.error = 0, None
        self.event = threading.Event()
        if self.shm is not None:            # the /dev/shm name never outlives the job object (fire-and-forget maps, failed maps)
            weakref.finalize(self, _release_shm, self.shm)
            if out_dtype is not None:
                weakref.finalize(self, _unlink_values, self.shm.name, len(blocks))

    def offset(self, lo, blk):
        if self.fold:
            return (1 + blk) * self.result_bytes
        return lo // 8 if self.bits else lo * self.result_bytes


def _release_shm(shm):
    shm.release()                   # unlink the name; the mapping lives as long as NumPy views of it do


# the exceptions a worker's "error" message names that the master raises as they are; any other becomes RuntimeError
_ERRORS = {"OverflowError": OverflowError, "ValueError": ValueError, "TypeError": TypeError}


def _receive(w, ready, when=""):
    """What worker ``w`` has to say, given the objects ``mpc.wait`` found ``ready``: (message, None); (message or None,
    reason) when the worker is dead -- it reported its CUDA context lost, its pipe broke or its process exited; or
    (None, None) when it has nothing to say.  ``when`` is put after "connection lost" in the reason."""
    if w.conn in ready:
        try:
            msg = w.conn.recv()
        except (EOFError, OSError):
            return None, "connection lost%s (exit code %s)" % (when, w.proc.exitcode)
        return msg, (msg[3] if msg[0] == "dead" else None)
    if w.proc is not None and w.proc.sentinel in ready and not w.proc.is_alive():
        return None, "process exited with code %s" % w.proc.exitcode
    return None, None


class ProcessResult:
    """Handle of an asynchronous map on the process pool (``MapResult``, fiber/pool.py:731-743)."""

    def __init__(self, pool, job, spec, single=False):
        self._pool, self._job, self._spec, self._single = pool, job, spec, single
        self._result = None

    def _emit_parts(self):
        """An emit map: the blocks' end offsets rebased by the values of the blocks before them, and their values
        concatenated in block order."""
        job = self._job
        ends = job.shm.array[:job.nbytes].view(np.uint64).copy()
        parts, base = [], 0
        for b, (lo, hi) in enumerate(job.ranges):
            path = os.path.join("/dev/shm", values_name(job.shm.name, b))
            k = int(ends[hi - 1]) if hi > lo else 0
            vals = np.fromfile(path, dtype=job.out_dtype)
            if len(vals) != k:
                raise RuntimeError("%s: block %d of map %d holds %d values, its offsets say %d" % (job.body, b, job.id, len(vals), k))
            parts.append(vals)
            ends[lo:hi] += np.uint64(base)
            base += k
        _unlink_values(job.shm.name, len(job.ranges))
        return ends, np.concatenate(parts)

    def get(self, timeout=None):
        from .pool import host_result
        if self._result is None:
            job = self._job
            if not job.event.wait(timeout):
                raise TimeoutError("map %d not finished" % job.id)
            if job.error is not None:
                raise job.error
            kind = "fold" if job.fold else "emit" if job.out_dtype is not None else "bits" if job.bits else "plain"
            data = values = None
            if kind == "emit" and job.n:
                data, values = self._emit_parts()
            elif job.n:
                data = job.shm.array[:job.result_bytes if job.fold else job.nbytes]
            total = job.sum if (self._spec.flags & _abi.FBR_BODY_SUMMABLE) else None
            result = host_result(self._spec, kind, data, job.n, total, values)
            if job.shm is not None:
                if not job.fold:
                    result._shm = job.shm    # the mapping lives as long as the result; workers are done with the name
                job.shm.release()
            self._result = (result,) if job.fold else result
        return self._result[0] if self._single else self._result


class ProcessPool:
    """One worker process per GPU slot; pull dispatch of blocks; dead workers are replaced and their blocks re-queued."""

    def __init__(self, processes, devices, results="host", redispatch=True, worker_main=gpu_worker_main, block_tasks=None,
                 init=None):
        self._n = processes
        self._init = init            # (initializer body, initargs, module) every worker process starts with, or None
        self._devices = list(devices)
        self._results = results
        self._redispatch = redispatch
        self._worker_main = worker_main
        self._block_tasks = block_tasks
        self._ctx = mp.get_context("spawn")
        self._workers = [_Worker(i, self._devices[i % len(self._devices)]) for i in range(processes)]
        self._jobs = collections.deque()
        self._cv = threading.Condition()
        self._next_job = 0
        self._closing = False
        self._terminated = False     # terminate(): work still queued is abandoned (close() lets it finish)
        self._thread = None
        self.stats = {"workers_lost": 0, "workers_started": 0, "blocks_dispatched": 0, "blocks_redispatched": 0, "maps": 0}

    # -- workers -----------------------------------------------------------------------------------------
    def _spawn(self, w):
        parent, child = self._ctx.Pipe()
        kw = {"init": self._init} if self._init is not None else {}
        w.proc = self._ctx.Process(target=self._worker_main, args=(w.device, child, self._results, [ROOT]), kwargs=kw, daemon=True)
        w.proc.start()
        child.close()
        w.conn, w.block, w.ready = parent, None, False
        self.stats["workers_started"] += 1

    def start(self):
        for w in self._workers:
            if w.proc is None:
                self._spawn(w)
        if self._thread is None:
            self._thread = threading.Thread(target=self._run, daemon=True)
            self._thread.start()

    def wait_until_workers_up(self, timeout=120):
        self.start()
        t0 = time.time()
        while not all(w.ready for w in self._workers):
            if time.time() - t0 > timeout:
                raise TimeoutError("worker processes did not come up")
            time.sleep(0.01)

    # -- submission --------------------------------------------------------------------------------------
    def fold_blocks(self, n):
        """The task blocks [lo, hi) a map of n tasks is cut into, in block order (a fold map's result is tree() over their
        totals in this order)."""
        per = self._block_tasks or max(BLOCK_ALIGN, -(-n // (4 * self._n) // BLOCK_ALIGN) * BLOCK_ALIGN)
        return [(lo, min(n, lo + per)) for lo in range(0, n, per)]

    def submit_fold(self, spec, kind, items):
        """A fold map (``kind`` "map" or "starmap"): each block runs ``Pool.fold`` in its worker and places its total;
        once every block is in, one live worker folds the totals in block order."""
        return self.submit(spec, None, "fold" if kind == "map" else "starfold", items, 0, single=True)

    def submit_accumulate(self, spec, kind, items):
        """An accumulate map (``kind`` "map" or "starmap"): each block runs ``Pool.accumulate`` in its worker and places its
        own prefix folds; once every block is in, one live worker wraps blocks 1, 2, ... with the pieces of the block totals
        before them, so record i of block b is tree(t_0, ..., t_{b-1}, p_i) over the blocks of ``fold_blocks``."""
        return self.submit(spec, None, "accumulate" if kind == "map" else "staraccumulate", items, 0)

    def submit(self, spec, twin, kind, items, chunksize, single=False):
        """items: a ``range`` or a list/array of per-task items (tuples for starmap)."""
        from . import registry
        n = len(items)
        bits = twin is not None
        blocks = [(i, lo, hi, 0) for i, (lo, hi) in enumerate(self.fold_blocks(n))]
        if isinstance(items, range):
            def payload_of(lo, hi, r=items):
                sub = r[lo:hi]
                return ("range", (sub.start, sub.stop, sub.step))
        else:
            def payload_of(lo, hi, seq=items):
                return ("items", pickle.dumps(seq[lo:hi], protocol=pickle.HIGHEST_PROTOCOL))
        with self._cv:
            if self._closing:
                raise ValueError("Pool is not running")
            self._next_job += 1
            job = _Job(self._next_job, spec.name, kind, chunksize, n, spec.result_bytes, bits, blocks, payload_of,
                       registry.module_of(spec.name), getattr(spec, "out_dtype", None))
            if n == 0:
                job.event.set()
            else:
                self._jobs.append(job)
            self.stats["maps"] += 1
            self._cv.notify_all()
        self.start()
        return ProcessResult(self, job, spec, single)

    # -- dispatcher thread (the master's _handle_tasks + _handle_workers + _res_get in one loop) -----------
    def _fail(self, job, exc):
        job.error = exc
        job.blocks.clear()
        job.event.set()
        # (the segment's name is unlinked when the job object goes away: blocks of this map may still be running)

    def _on_death(self, w, reason):
        self.stats["workers_lost"] += 1
        blk = w.block
        try:
            w.conn.close()
        except OSError:
            pass
        if w.proc is not None:
            w.proc.join(timeout=5)
        if blk is not None:
            job, (bid, lo, hi, attempt) = blk
            if job.error is None:
                if not self._redispatch:
                    self._fail(job, WorkerDied("worker %d (CUDA device %d) died under map %d: %s; the pool was created without "
                                               "error_handling, so its block is not re-dispatched" % (w.index, w.device, job.id, reason)))
                elif attempt + 1 >= MAX_ATTEMPTS:
                    self._fail(job, WorkerDied("block %d of map %d killed its worker %d times: %s" % (bid, job.id, attempt + 1, reason)))
                else:
                    job.blocks.appendleft((bid, lo, hi, attempt + 1))      # re-queue (fiber/pool.py:1635-1654)
                    self.stats["blocks_redispatched"] += 1
        if not self._closing:
            self._spawn(w)                                                  # _maintain_workers: a fresh worker takes its place

    def _pump_idle(self):
        """No map in flight: take "ready" notes from fresh workers, replace workers that died while idle."""
        waitables = [w.conn for w in self._workers if w.conn is not None]
        ready = mpc.wait(waitables, timeout=0) if waitables else []
        for w in self._workers:
            msg, dead_reason = _receive(w, ready, " while idle")
            if msg is not None and msg[0] == "ready":
                w.ready = True
            if dead_reason is not None:
                self._on_death(w, dead_reason)

    def _run(self):
        while True:
            with self._cv:
                while not self._jobs and not self._closing:
                    self._cv.wait(0.02)
                    self._pump_idle()
                if self._closing and not self._jobs:
                    return
                job = self._jobs[0]
            self._run_job(job)
            with self._cv:
                if self._jobs and self._jobs[0] is job:
                    self._jobs.popleft()

    def _run_job(self, job):
        inflight = 0
        while (job.blocks or inflight) and job.error is None:
            for w in self._workers:                                        # idle workers pull the next block
                if w.ready and w.block is None and job.blocks:
                    bid, lo, hi, attempt = job.blocks.popleft()
                    try:
                        w.conn.send(("block", job.id, bid, job.body, job.kind, job.chunksize, job.payload_of(lo, hi), job.shm.name,
                                     job.offset(lo, bid), attempt, job.module))
                    except (OSError, ValueError):
                        job.blocks.appendleft((bid, lo, hi, attempt))
                        w.block = None
                        self._on_death(w, "pipe closed")
                        continue
                    w.block = (job, (bid, lo, hi, attempt))
                    inflight += 1
                    self.stats["blocks_dispatched"] += 1
            waitables = [w.conn for w in self._workers if w.conn is not None] + [w.proc.sentinel for w in self._workers if w.proc is not None]
            ready = mpc.wait(waitables, timeout=0.5)
            for w in self._workers:
                if w.conn is None:
                    continue
                msg, dead_reason = _receive(w, ready)
                if msg is not None:
                    # a block of an EARLIER map (one that failed while this block was still running) reports late:
                    # the worker becomes idle again, the current map's accounting is not touched
                    mine = w.block is not None and w.block[0] is job and msg[0] != "ready" and msg[1] == job.id
                    if msg[0] == "ready":
                        w.ready = True
                    elif not mine:
                        w.block = None
                    elif msg[0] == "done":
                        job.sum += msg[3] or 0
                        job.done_blocks += 1
                        w.block = None
                        inflight -= 1
                    elif msg[0] == "error":
                        w.block = None
                        inflight -= 1
                        self._fail(job, _ERRORS.get(msg[3], RuntimeError)(msg[4]))
                if dead_reason is not None:
                    if w.block is not None and w.block[0] is job:
                        inflight -= 1
                    self._on_death(w, dead_reason)
        if (job.fold or (job.scan and job.n_blocks > 1)) and job.n and job.error is None:
            self._fold_totals(job)
        job.event.set()

    def _fold_totals(self, job):
        """A fold map whose blocks have all placed their totals: one live worker folds them in block order into the result
        record; an accumulate map's wraps every block after the first (_scan_blocks_in_worker).  This runs after close()
        too, like the blocks of queued maps; terminate() abandons it.  A worker that dies meanwhile is replaced and the fold goes to the next live one, as a block would be re-queued: without error_handling
        the first death fails the map, and MAX_ATTEMPTS deaths fail it in any case.  The map always ends folded or failed."""
        deaths = 0
        while job.error is None:
            if self._terminated:
                self._fail(job, RuntimeError("map %d: the pool was terminated before its block totals were folded" % job.id))
                return
            live = [w for w in self._workers if w.conn is not None and w.proc is not None and w.proc.is_alive()]
            w = next((w for w in live if w.ready and w.block is None), None)
            if w is None:
                if not live and self._closing:                  # a closed pool replaces no worker
                    self._fail(job, WorkerDied("map %d: no live worker is left to fold its block totals" % job.id))
                    return
                self._pump_idle()
                time.sleep(0.01)
                continue
            dead_reason = None
            try:
                if job.scan:
                    R = job.result_bytes
                    if job.scan_totals is None:
                        job.scan_totals = b"".join(bytes(job.shm.array[(hi - 1) * R:hi * R]) for _, hi in job.ranges)
                    todo = [b for b in range(1, job.n_blocks) if b not in job.scan_wrapped]
                    w.conn.send(("scan", job.id, job.ranges, todo, job.scan_totals, job.body, job.shm.name, job.module))
                else:
                    w.conn.send(("fold", job.id, job.n_blocks, job.body, job.shm.name, job.module))
            except (OSError, ValueError):
                dead_reason = "pipe closed"
            while dead_reason is None:
                msg, dead_reason = _receive(w, mpc.wait([w.conn, w.proc.sentinel], timeout=0.5))
                if msg is not None and msg[0] == "ready":
                    w.ready = True
                elif msg is not None and msg[1] == job.id:
                    if msg[0] == "scanned":
                        job.scan_wrapped.add(msg[2])
                    elif msg[0] == "folded":
                        return
                    elif msg[0] == "error":
                        self._fail(job, _ERRORS.get(msg[3], RuntimeError)(msg[4]))
                        return
            deaths += 1
            self._on_death(w, dead_reason)                      # no block of its own: nothing is re-queued
            if self._terminated:
                continue
            if not self._redispatch:
                self._fail(job, WorkerDied("worker %d (CUDA device %d) died folding the block totals of map %d: %s; the pool was "
                                           "created without error_handling, so the fold is not sent again"
                                           % (w.index, w.device, job.id, dead_reason)))
            elif deaths >= MAX_ATTEMPTS:
                self._fail(job, WorkerDied("folding the block totals of map %d killed its worker %d times: %s"
                                           % (job.id, deaths, dead_reason)))

    # -- shutdown ----------------------------------------------------------------------------------------
    def close(self):
        with self._cv:
            self._closing = True
            self._cv.notify_all()

    def terminate(self):
        self._terminated = True
        self.close()
        for w in self._workers:
            if w.conn is not None:
                try:
                    w.conn.send(None)
                except (OSError, ValueError):
                    pass

    def join(self, timeout=30):
        if self._thread is not None:
            self._thread.join(timeout)
        for w in self._workers:
            if w.conn is not None:
                try:
                    w.conn.send(None)
                except (OSError, ValueError):
                    pass
            if w.proc is not None:
                w.proc.join(timeout=10)
                if w.proc.is_alive():
                    w.proc.terminate()
