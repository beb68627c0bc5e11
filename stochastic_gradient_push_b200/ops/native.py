"""
Loader for the in-tree sm_90a extension (``stochastic_gradient_push_b200/_C*.so``).

The extension is never silently replaced by a PyTorch fallback: on a machine
with a CUDA device ``load()`` either returns the native module or raises.  If
the shared object is missing or stale it is (re)built in-tree with nvcc (see
``ops/build.py``); CPU-only hosts can still build (cross-compile) but cannot
run the kernels.
"""

from __future__ import annotations

import importlib
import os
import threading

_lock = threading.Lock()
_mod = None


def available() -> bool:
    """True iff the native module can be imported (does not build)."""
    try:
        load(build_if_missing=False)
        return True
    except Exception:
        return False


def load(build_if_missing: bool = True):
    global _mod
    if _mod is not None:
        return _mod
    with _lock:
        if _mod is not None:
            return _mod
        import torch  # noqa: F401  (libtorch must be loaded before the extension)
        from . import build as _build
        so = _build.so_path()
        if not os.path.exists(so):
            if not build_if_missing:
                raise ImportError('native extension not built: %s' % so)
            _build.build()
        try:
            _mod = importlib.import_module('stochastic_gradient_push_b200._C')
        except ImportError:
            if not build_if_missing:
                raise
            _build.build(force=True)
            _mod = importlib.import_module('stochastic_gradient_push_b200._C')
        return _mod
