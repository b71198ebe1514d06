"""Builds and loads the native sm_90a extension (``pytorch_distributed_b200/_C*.so``, in-tree).

* ``build()`` compiles every source under ``csrc/`` with
  ``-gencode arch=compute_90a,code=sm_90a -lineinfo`` (nvcc cross-compiles without a GPU) and drops the shared
  object next to this file, so it travels with the source tree.  A content hash of the sources is stored beside it;
  a stale or missing build is redone on import when a compiler is available.
* ``lib()`` returns the module or raises.  On a CUDA machine a missing extension is a hard error - there is no
  silent PyTorch fallback for the GPU paths.
"""
from __future__ import annotations

import hashlib
import importlib.util
import os
import shutil
import sys
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_HERE, "csrc")
_NAME = "_C"
_SO = os.path.join(_HERE, _NAME + ".so")
_STAMP = os.path.join(_HERE, _NAME + ".hash")
_SOURCES = ["bindings.cpp", "symm.cpp", "hvd_core.cpp", "collectives.cu", "optim.cu", "bn_act.cu", "data_ops.cu", "gemm_bnstats.cu", "stem_conv.cu",
            "resample.cu", "sync_bn.cu", "mix.cu", "augment.cu"]
_lock = threading.Lock()
_mod = None
_err = None

CUDA_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "--use_fast_math", "-std=c++17",
              "--expt-relaxed-constexpr", "-Xptxas", "-v"]


def source_hash() -> str:
    h = hashlib.sha256()
    for fn in sorted(os.listdir(_CSRC)):
        if fn.endswith((".cu", ".cpp", ".h", ".cuh")):
            with open(os.path.join(_CSRC, fn), "rb") as f:
                h.update(fn.encode())
                h.update(f.read())
    h.update(" ".join(CUDA_FLAGS).encode())
    return h.hexdigest()


def is_built() -> bool:
    if not (os.path.exists(_SO) and os.path.exists(_STAMP)):
        return False
    with open(_STAMP) as f:
        return f.read().strip() == source_hash()


def build(verbose: bool = False, force: bool = False) -> str:
    """Compile the extension in-tree for sm_90a. Returns the path of the shared object."""
    with _lock:
        if is_built() and not force:
            return _SO
        from torch.utils import cpp_extension
        build_dir = os.path.join(_CSRC, "build")
        os.makedirs(build_dir, exist_ok=True)
        os.environ.setdefault("MAX_JOBS", str(max(2, min(8, (os.cpu_count() or 4)))))
        cpp_extension.load(
            name=_NAME,
            sources=[os.path.join(_CSRC, s) for s in _SOURCES],
            extra_cflags=["-O3", "-std=c++17"],
            extra_cuda_cflags=CUDA_FLAGS,
            extra_include_paths=[_CSRC],
            build_directory=build_dir,
            verbose=verbose,
            is_python_module=False,
        )
        built = os.path.join(build_dir, _NAME + ".so")
        shutil.copyfile(built, _SO + ".tmp")
        os.replace(_SO + ".tmp", _SO)
        with open(_STAMP, "w") as f:
            f.write(source_hash())
        return _SO


def _import_so():
    import torch  # noqa: F401  (libtorch must be loaded before the extension)
    spec = importlib.util.spec_from_file_location("pytorch_distributed_b200." + _NAME, _SO)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    sys.modules["pytorch_distributed_b200." + _NAME] = mod
    return mod


def lib(build_if_missing: bool = True):
    """The loaded native module (building it first if needed and possible)."""
    global _mod, _err
    if _mod is not None:
        return _mod
    if _err is not None:
        raise _err
    try:
        if not is_built():
            if not build_if_missing or os.environ.get("PTD_NO_BUILD") == "1":
                raise RuntimeError("native extension is not built (run `python -c 'import __graft_entry__ as g; g.build()'`)")
            build()
        _mod = _import_so()
        return _mod
    except Exception as e:  # remember: do not retry a failing build on every call
        _err = RuntimeError("pytorch_distributed_b200 native extension unavailable: %s" % (e,))
        raise _err from e


def available() -> bool:
    try:
        lib()
        return True
    except Exception:
        return False


def require_on_cuda() -> None:
    """Fail loudly when a GPU is present but the native kernels are not."""
    import torch
    if torch.cuda.is_available():
        lib()


# ---------------------------------------------------------------------- launch accounting (bench.py "gpu_launches")
launches = 0


def note_launch(n: int = 1) -> None:
    """Python wrappers of the native kernels call this once per kernel they enqueue."""
    global launches
    launches += n
