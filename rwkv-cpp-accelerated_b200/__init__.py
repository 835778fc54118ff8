"""rwkv-cpp-accelerated_b200 — H100 (sm_90a) RWKV-v4 uint8 decode engine.

The product is the CUDA library in ``csrc/`` behind the C ABI of ``include/rwkv_b200.h``;
this package is the thin Python side used by tests and ``bench.py`` (ctypes over that
ABI) plus build helpers. The directory name contains a hyphen, so import it with::

    import importlib
    pkg = importlib.import_module("rwkv-cpp-accelerated_b200")
"""
from .engine import Batcher, Engine, EngineError, PrefixCache, Sampler, StateIndex, lib_path, load_library  # noqa: F401
from . import build as build  # noqa: F401
from . import constrain as constrain  # noqa: F401
from . import tp as tp  # noqa: F401
