"""fiber_b200 -- H100-native engine behind uber/fiber's ``Pool.map`` hot path.

Public surface mirrors ``fiber/__init__.py:65-67`` / ``fiber/context.py:20-69`` for the path this
repository replaces: ``Pool`` (``ZPool`` / ``ResilientZPool`` semantics), ``meta``, ``cpu_count``,
``current_process``, ``active_children``, plus the binding helpers ``device_body`` / ``bind`` that
attach a compiled-in device body to a Python callable.

Importing the package does not touch CUDA; the shared library ``fiber_b200/_lib/libfiber_b200.so``
is loaded on first use and its absence is a hard error (no CPU fallback).
"""
import multiprocessing as _mp

from .meta import meta  # noqa: F401
from .pool import ApplyResult, FoldResult, MapResult, Pool, ResultArray  # noqa: F401
from .process import Process, active_children, device_process  # noqa: F401
from . import config  # noqa: F401
from .config import init, reset  # noqa: F401
from .queues import Connection, Pipe  # noqa: F401
from .queues import SimpleQueuePush as _SimpleQueuePush
from .registry import Columns, Ragged, bind, body_names, device_body, device_initializer, register_module  # noqa: F401

__version__ = "0.1.0"


def cpu_count():
    """fiber/context.py:61-62 returns ``os.cpu_count()``; the unit of parallel hardware here is the
    GPU, so this is the number of visible CUDA devices."""
    import ctypes
    from . import _abi
    n = ctypes.c_int(0)
    _abi.check(_abi.load().fbr_device_count(ctypes.byref(n)))
    return n.value


def current_process():
    """fiber/context.py:24: GPU workers are not OS processes, the caller is always the master."""
    return _mp.current_process()


def SimpleQueue():
    """fiber/context.py:47-54: the push queue, unless ``use_push_queue`` was switched off."""
    if config.use_push_queue:
        return _SimpleQueuePush()
    raise NotImplementedError
