"""Loader for the in-tree sm_90a extension ``relora_b200/_C.so`` (built by ``__graft_entry__.build``
or ``python -m relora_b200.csrc.build``).  The shared object is kept in the source tree so it travels
with the repository snapshot to the GPU box; nothing is JIT-compiled at import time.
"""
from __future__ import annotations

import importlib
import os
import threading

_lock = threading.Lock()
_mod = None
_err = None


def _try_load():
    global _mod, _err
    if _mod is not None or _err is not None:
        return
    with _lock:
        if _mod is not None or _err is not None:
            return
        try:
            import torch  # noqa: F401  (libtorch must be loaded before the extension)

            _mod = importlib.import_module("relora_b200._C")
        except Exception as e:  # ImportError, OSError (missing libcuda on CPU boxes), ...
            _err = e


def available() -> bool:
    _try_load()
    return _mod is not None


def module():
    _try_load()
    if _mod is None:
        raise RuntimeError(f"relora_b200 native extension is not available: {_err!r}")
    return _mod


def require():
    """Fail loudly when running on a GPU without the extension (no silent eager fallback)."""
    _try_load()
    if _mod is None:
        raise RuntimeError(
            "relora_b200._C (sm_90a kernels) could not be loaded on a CUDA device: "
            f"{_err!r}. Build it with `python -c 'import __graft_entry__ as g; g.build()'`."
        )
    return _mod


def so_path():
    m = module()
    return os.path.abspath(m.__file__)
