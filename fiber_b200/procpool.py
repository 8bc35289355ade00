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


def gpu_worker_main(device, conn, results, sys_path, init=None):
    """Worker process: one engine on one GPU, blocks in, ordered result bytes out (into shared memory).  ``init``:
    (body, initargs, module) of the pool's initializer, or None."""
    for p in sys_path:
        if p not in sys.path:
            sys.path.insert(0, p)
    import fiber_b200
    from fiber_b200 import _abi, registry
    kw = {}
    if init is not None:
        body, initargs, module = init
        if module is not None and body not in registry.body_names():
            registry.register_module(body, *module)
        kw = {"initializer": _initializer_for(body), "initargs": initargs}
    pool = fiber_b200.Pool(1, devices=[device], express=False, results=results, **kw)
    pool.start_workers()
    proxies, segments = {}, {}
    conn.send(("ready", os.getpid()))
    while True:
        msg = conn.recv()
        if msg is None:
            break
        _, job, blk, body, kind, chunksize, payload, shm_name, off, attempt, module = msg
        try:
            if module is not None and body not in registry.body_names():
                registry.register_module(body, *module)
            f = proxies.get(body) or proxies.setdefault(body, _proxy_for(body))
            items = range(*payload[1]) if payload[0] == "range" else pickle.loads(payload[1])
            pool._attempt = attempt
            if kind == "starmap":
                res = pool.starmap(f, items, chunksize)
            elif kind == "apply":
                res = pool.apply_async(f, items[0][0], items[0][1])._wait()
            else:
                res = pool.map(f, items, chunksize)
            raw = res.packed if res.packed is not None else np.ascontiguousarray(np.asarray(res)).view(np.uint8).reshape(-1)
            seg = segments.get(shm_name)
            if seg is None:
                segments.clear()                                   # one live segment per worker is enough
                seg = segments.setdefault(shm_name, SharedSegment(shm_name))
            seg.array[off:off + raw.nbytes] = raw                  # placement by index (fiber/pool.py:672), block-wise
            total = res.sum() if (registry.spec(body).flags & _abi.FBR_BODY_SUMMABLE) else None
            del res, raw
            conn.send(("done", job, blk, total))
        except _abi.EngineError as e:
            if e.status == _abi.FBR_ECUDA:
                # the CUDA context of this process is gone for good: report and die, the master re-queues the block
                try:
                    conn.send(("dead", job, blk, str(e)))
                finally:
                    os._exit(3)
            conn.send(("error", job, blk, "EngineError", str(e)))
        except (OverflowError, ValueError, TypeError, RuntimeError, KeyError, OSError) as e:   # OSError: the segment of a failed map is gone
            conn.send(("error", job, blk, type(e).__name__, str(e)))
    os._exit(0)


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
    def __init__(self, jid, body, kind, chunksize, n, result_bytes, bits, blocks, payload_of, module):
        self.id, self.body, self.kind, self.chunksize, self.n = jid, body, kind, chunksize, n
        self.result_bytes, self.bits = result_bytes, bits
        self.blocks = collections.deque(blocks)       # (blk id, lo, hi, attempt)
        self.n_blocks, self.done_blocks = len(blocks), 0
        self.payload_of, self.module = payload_of, module
        nbytes = ((n + 7) // 8) if bits else n * result_bytes
        self.shm = SharedSegment("fbr_%d_%d_%d" % (os.getpid(), jid, int(time.time() * 1e6) & 0xFFFFFF), nbytes) if n else None
        self.nbytes = nbytes
        self.sum, self.error = 0, None
        self.event = threading.Event()
        if self.shm is not None:            # the /dev/shm name never outlives the job object (fire-and-forget maps, failed maps)
            weakref.finalize(self, _release_shm, self.shm)

    def offset(self, lo):
        return lo // 8 if self.bits else lo * self.result_bytes


def _release_shm(shm):
    shm.release()                   # unlink the name; the mapping lives as long as NumPy views of it do


class ProcessResult:
    """Handle of an asynchronous map on the process pool (``MapResult``, fiber/pool.py:731-743)."""

    def __init__(self, pool, job, spec, single=False):
        self._pool, self._job, self._spec, self._single = pool, job, spec, single
        self._result = None

    def get(self, timeout=None):
        from .pool import ResultArray
        if self._result is None:
            job = self._job
            if not job.event.wait(timeout):
                raise TimeoutError("map %d not finished" % job.id)
            if job.error is not None:
                raise job.error
            dtype, sub = self._spec.result_dtype()
            total = job.sum if (self._spec.flags & 0x4) else None
            if job.n == 0:
                self._result = ResultArray(self._spec, np.empty((0,) + sub, dtype), 0)
            elif job.bits:
                self._result = ResultArray(self._spec, None, total, n=job.n, bits=job.shm.array[:job.nbytes])
            else:
                arr = job.shm.array[:job.nbytes].view(dtype).reshape((job.n,) + sub)
                self._result = ResultArray(self._spec, arr, total)
            if job.shm is not None:
                self._result._shm = job.shm      # the mapping lives as long as the result; workers are done with the name
                job.shm.release()
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
    def submit(self, spec, twin, kind, items, chunksize, single=False):
        """items: a ``range`` or a list/array of per-task items (tuples for starmap)."""
        from . import registry
        n = len(items)
        bits = twin is not None
        per = self._block_tasks or max(BLOCK_ALIGN, -(-n // (4 * self._n) // BLOCK_ALIGN) * BLOCK_ALIGN)
        blocks = [(i, lo, min(n, lo + per), 0) for i, lo in enumerate(range(0, n, per))]
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
                       registry.module_of(spec.name))
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
        for c in mpc.wait(waitables, timeout=0) if waitables else []:
            for w in self._workers:
                if w.conn is c:
                    try:
                        msg = c.recv()
                        if msg and msg[0] == "ready":
                            w.ready = True
                    except (EOFError, OSError):
                        self._on_death(w, "connection lost while idle (exit code %s)" % w.proc.exitcode)

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
                                     job.offset(lo), attempt, job.module))
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
                dead_reason = None
                if w.conn in ready:
                    try:
                        msg = w.conn.recv()
                    except (EOFError, OSError):
                        msg, dead_reason = None, "connection lost (exit code %s)" % w.proc.exitcode
                    if msg is not None:
                        # a block of an EARLIER map (one that failed while this block was still running) reports late:
                        # the worker becomes idle again, the current map's accounting is not touched
                        mine = w.block is not None and w.block[0] is job and msg[0] != "ready" and msg[1] == job.id
                        if msg[0] == "ready":
                            w.ready = True
                        elif not mine:
                            if msg[0] == "dead":
                                w.block = None
                                dead_reason = msg[3]
                            else:
                                w.block = None
                        elif msg[0] == "done":
                            job.sum += msg[3] or 0
                            job.done_blocks += 1
                            w.block = None
                            inflight -= 1
                        elif msg[0] == "error":
                            w.block = None
                            inflight -= 1
                            exc = {"OverflowError": OverflowError, "ValueError": ValueError, "TypeError": TypeError}.get(msg[3], RuntimeError)
                            self._fail(job, exc(msg[4]))
                        elif msg[0] == "dead":
                            dead_reason = msg[3]
                elif w.proc is not None and w.proc.sentinel in ready and not w.proc.is_alive():
                    dead_reason = "process exited with code %s" % w.proc.exitcode
                if dead_reason is not None:
                    if w.block is not None and w.block[0] is job:
                        inflight -= 1
                    self._on_death(w, dead_reason)
        job.event.set()

    # -- shutdown ----------------------------------------------------------------------------------------
    def close(self):
        with self._cv:
            self._closing = True
            self._cv.notify_all()

    def terminate(self):
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
