"""Loader for the native extension.  ``get()`` imports the in-tree ``_C`` module, building it first if
it is missing (machines without a GPU can build: nvcc cross-compiles sm_90a).  On a GPU machine a
missing extension is a hard error for every CUDA op - there is no silent PyTorch fallback."""
from __future__ import annotations

import importlib
import importlib.util
import os
import sys
import threading

_lock = threading.Lock()
_mod = None
_err = None


def _import_built():
    from .build import ext_path
    path = ext_path()
    if not path.exists():
        return None
    import torch  # noqa: F401  (libtorch must be loaded before the extension)
    name = __package__ + "._C"
    spec = importlib.util.spec_from_file_location(name, str(path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    sys.modules[name] = mod
    return mod


def get(build_if_missing: bool = True):
    """Return the extension module or raise."""
    global _mod, _err
    if _mod is not None:
        return _mod
    with _lock:
        if _mod is not None:
            return _mod
        try:
            mod = _import_built()
            if mod is None and build_if_missing and os.environ.get("B200DDP_NO_BUILD") != "1":
                from .build import build
                build(verbose=True)
                mod = _import_built()
            if mod is None:
                raise ImportError("b200ddp native extension is not built; run `python -m b200ddp.build`")
            _mod = mod
            return mod
        except Exception as exc:  # remember: later callers get the same diagnosis, not a rebuild storm
            _err = exc
            raise


def available() -> bool:
    try:
        get(build_if_missing=False)
        return True
    except Exception:
        return False


def require_for(device) -> None:
    """CUDA tensors must hit native kernels: fail loudly instead of falling back."""
    import torch
    if torch.device(device).type == "cuda":
        get()
