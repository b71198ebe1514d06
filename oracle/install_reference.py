"""Install the UNMODIFIED reference scripts into ``oracle/_ref`` (git-ignored) for ``bench.py --impl reference``.

The reference is a set of scripts without ``setup.py`` / ``pyproject.toml``, so it cannot be pip-installed: the install
is a byte-for-byte copy of every file of the reference checkout, verified against the sha256 manifest below.  The checkout
is looked for in ``PTD_REFERENCE_DIR`` first, then at its default location ``DEFAULT_DIRS``.
Called by ``__graft_entry__.build()`` and, as a last resort, by ``bench.py --impl reference`` itself.
"""
from __future__ import annotations

import hashlib
import os
import shutil

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")
ENV = "PTD_REFERENCE_DIR"
DEFAULT_DIRS = ["/root/reference"]       # where the reference checkout lives next to this repository's build

# sha256 of the reference scripts (integrity check of the copy, nothing else)
MANIFEST = {
    "apex_distributed.py": "f17d6bc0749db6267c8116b01bc84dd06ee98fdc83016c23d3a338490523bc1e",
    "dataparallel.py": "683f9c1bab9ede3fc9443cda9ff9c462a2eccecedf766dc7aa286e7de56a7d50",
    "distributed.py": "37b20448988adc04e4306e696e2a6f9d05cfef6874fc1614e05df48c8f171cb2",
    "distributed_slurm_main.py": "0cd7298ef6163573bd6e6e1f69554d10f03086cd1f62ea92f7e705122783cbc2",
    "horovod_distributed.py": "ae6bd717a5c3b65d550690da8a1d578a2cd5ecf6a0922a729ac8bd0835bc38f7",
    "multiprocessing_distributed.py": "3dc54e8a4cbdc8de92a82255d311ba4af2d8e50f1219df798dac6799e919a4a4",
    "start.sh": "2a60fba72e6897241c7f77e5d1c4cbd516716f2dc14ef5fa8522ce6b84c9f25c",
    "statistics.sh": "e8fe1eca45bfe86cad5b9b246d98936d447a794b61a639b85c3acd07f5a8e575",
    "requirements.txt": "11767ec0796a7709ead1019560e7cd916c06d7f51f61ff1fcb1703639862dbde",
}


def sha256(path: str) -> str:
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def verify(directory: str = None) -> list:
    """Names of manifest files that are missing from ``directory`` (default: ``REF_DIR``) or differ from the reference."""
    directory = directory or REF_DIR
    bad = []
    for fn, h in MANIFEST.items():
        p = os.path.join(directory, fn)
        if not os.path.exists(p) or sha256(p) != h:
            bad.append(fn)
    return bad


def install(force: bool = False) -> str:
    """Copy the reference tree into oracle/_ref.  Returns a one-line status; raises only if a copy was attempted and
    produced files that do not match the manifest."""
    if not force and os.path.isdir(REF_DIR) and not verify():
        return "oracle/_ref present (%d files verified)" % len(MANIFEST)
    candidates = [os.environ.get(ENV, "")] + DEFAULT_DIRS
    src = next((c for c in candidates if c and os.path.exists(os.path.join(c, "distributed.py"))), None)
    if src is None:
        return "NOT INSTALLED: no reference checkout in %s or %s" % (ENV, ", ".join(DEFAULT_DIRS))
    os.makedirs(REF_DIR, exist_ok=True)
    n = 0
    for root, dirs, files in os.walk(src):
        dirs[:] = [d for d in dirs if d not in (".git", "__pycache__")]
        rel = os.path.relpath(root, src)
        for fn in files:
            dst_dir = os.path.join(REF_DIR, rel) if rel != "." else REF_DIR
            os.makedirs(dst_dir, exist_ok=True)
            shutil.copyfile(os.path.join(root, fn), os.path.join(dst_dir, fn))
            n += 1
    bad = verify()
    if bad:
        raise RuntimeError("reference copy does not match the sha256 manifest: %s" % bad)
    return "installed %d files from %s into oracle/_ref (sha256 verified)" % (n, src)


if __name__ == "__main__":
    print(install(force=True))
