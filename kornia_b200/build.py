"""In-tree build of the CUDA shared library for sm_90a (nvcc cross-compiles without a GPU)."""
from __future__ import annotations

import os
import shutil
import subprocess
import time

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
OUT_DIR = os.path.join(_HERE, "_C")
OUT = os.path.join(OUT_DIR, "libkornia_b200.so")

NVCC_FLAGS = [
    "-Xfatbin", "-compress-all",
    "-O3", "-std=c++17",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo",
    "-Xcompiler", "-fPIC",
]


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stale() -> bool:
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(os.path.dirname(_HERE), "include", "kornia_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def _deps_of(dep_file: str):
    """Prerequisites listed in a make-style dependency file written by ``nvcc -MD`` (None if unreadable)."""
    try:
        text = open(dep_file).read()
    except OSError:
        return None
    body = text.split(":", 1)[1] if ":" in text else ""
    return [tok for tok in body.replace("\\\n", " ").split() if tok != "\\"]


def _object_is_current(obj: str, dep_file: str) -> bool:
    """True when ``obj`` is newer than every file its translation unit read the last time it was compiled."""
    if not os.path.exists(obj):
        return False
    deps = _deps_of(dep_file)
    if not deps:
        return False
    t = os.path.getmtime(obj)
    deps = [d if os.path.isabs(d) else os.path.join(CSRC, d) for d in deps]  # nvcc runs in CSRC (compile_one)
    return all(os.path.exists(d) and os.path.getmtime(d) <= t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile kornia_b200/csrc/*.cu (one object per file, in parallel) and link
    kornia_b200/_C/libkornia_b200.so; returns the path.  Objects and their ``nvcc -MD`` dependency files stay in
    kornia_b200/_C/obj (git- and gpurun-ignored), so a later build recompiles only the translation units whose sources or
    headers changed; ``force`` recompiles everything."""
    if not force and not _stale():
        return OUT
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("kornia_b200.build: nvcc not found; cannot build the CUDA library")
    started = time.time()
    os.makedirs(OUT_DIR, exist_ok=True)
    obj_dir = os.path.join(OUT_DIR, "obj")
    os.makedirs(obj_dir, exist_ok=True)
    from concurrent.futures import ThreadPoolExecutor

    def compile_one(src):
        stem = os.path.join(obj_dir, os.path.basename(src)[:-3])
        obj, dep = stem + ".o", stem + ".d"
        if not force and not verbose and _object_is_current(obj, dep):
            return obj
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-MD", "-MF", dep, "-c", "-o", obj, src]
        started = time.time()
        proc = subprocess.run(cmd, capture_output=True, text=True, cwd=CSRC)
        if proc.returncode != 0:
            for stale in (obj, dep):
                if os.path.exists(stale):
                    os.remove(stale)
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + proc.stdout + proc.stderr)
        os.utime(obj, (started, started))  # a source edited while this ran is newer than the object, as it should be
        if verbose:
            print(proc.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as pool:
        objs = list(pool.map(compile_one, _sources()))
    known = {os.path.basename(o) for o in objs}
    for f in os.listdir(obj_dir):  # objects of sources that no longer exist must not be linked by a later glob or linger
        if f.endswith(".o") and f not in known:
            os.remove(os.path.join(obj_dir, f))
    cmd = [nvcc, "-shared", "-Xfatbin", "-compress-all", "-gencode", "arch=compute_90a,code=sm_90a", "-o", OUT] + objs
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError("link failed:\n" + " ".join(cmd) + "\n" + proc.stdout + proc.stderr)
    os.utime(OUT, (started, started))  # same rule for the library: _stale() compares source times with the build's START
    return OUT
