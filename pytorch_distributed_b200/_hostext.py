"""Builds and loads the host-only native module (``pytorch_distributed_b200/_L.so``): the C++ shard loader.

Kept apart from ``_C`` (the sm_90a extension) on purpose: it has no CUDA or libtorch dependency, compiles with plain
``g++`` in a few seconds, and is usable on machines without nvcc.  Same in-tree + content-hash scheme as ``_ext``.
"""
from __future__ import annotations

import hashlib
import importlib.util
import os
import subprocess
import sys
import sysconfig
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "csrc", "host", "loader.cpp")
_NAME = "_L"
_SO = os.path.join(_HERE, _NAME + ".so")
_STAMP = os.path.join(_HERE, _NAME + ".hash")
# -ffp-contract=off: resample() must round every multiply and add on its own, like the device kernel
# (csrc/resample.cu), also with compilers that contract to FMA by default (GCC on aarch64)
_FLAGS = ["-O3", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden", "-pthread", "-ffp-contract=off"]
_lock = threading.Lock()
_mod = None


def source_hash() -> str:
    h = hashlib.sha256()
    with open(_SRC, "rb") as f:
        h.update(f.read())
    h.update(" ".join(_FLAGS).encode())
    return h.hexdigest()


def is_built() -> bool:
    if not (os.path.exists(_SO) and os.path.exists(_STAMP)):
        return False
    with open(_STAMP) as f:
        return f.read().strip() == source_hash()


def build(force: bool = False) -> str:
    with _lock:
        if is_built() and not force:
            return _SO
        import pybind11
        cxx = os.environ.get("CXX", "g++")
        cmd = [cxx] + _FLAGS + ["-I" + pybind11.get_include(), "-I" + sysconfig.get_paths()["include"], _SRC, "-o", _SO + ".tmp"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("building %s failed:\n%s" % (_NAME, r.stderr[-4000:]))
        os.replace(_SO + ".tmp", _SO)
        with open(_STAMP, "w") as f:
            f.write(source_hash())
        return _SO


def lib():
    global _mod
    if _mod is not None:
        return _mod
    if not is_built():
        if os.environ.get("PTD_NO_BUILD") == "1":
            raise RuntimeError("host extension is not built (run `python -c 'import __graft_entry__ as g; g.build()'`)")
        build()
    spec = importlib.util.spec_from_file_location("pytorch_distributed_b200." + _NAME, _SO)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    sys.modules["pytorch_distributed_b200." + _NAME] = mod
    _mod = mod
    return mod
