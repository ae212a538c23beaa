"""Build libbioreason_b200.so in-tree with nvcc for sm_90a (no JIT cache: the shared object is built once, next to the sources)."""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT_DIR = os.path.join(HERE, "_C")
LIB = os.path.join(OUT_DIR, "libbioreason_b200.so")
NVCC = os.environ.get("NVCC", shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v"]
FLAGS += os.environ.get("BR_NVCC_EXTRA", "").split()          # experiments only (extra nvcc flags); part of the object digests


def _nccl_include():
    try:
        import nvidia.nccl  # type: ignore
        return os.path.join(os.path.dirname(nvidia.nccl.__path__[0] + "/"), "include")
    except Exception:
        return None


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(path, extra):
    h = hashlib.sha1()
    h.update(open(path, "rb").read())
    for e in extra:
        h.update(open(e, "rb").read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def build(verbose: bool = False, force: bool = False) -> str:
    os.makedirs(OUT_DIR, exist_ok=True)
    headers = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h")))
    headers.append(os.path.join(os.path.dirname(HERE), "include", "bioreason_b200.h"))
    inc = []
    ni = _nccl_include()
    if ni and os.path.isdir(ni):
        inc += ["-I", ni]
    objs, todo = [], []
    for src in sources():
        obj = os.path.join(OUT_DIR, os.path.basename(src)[:-3] + ".o")
        stamp = obj + ".sha1"
        dig = _digest(src, headers)
        objs.append(obj)
        if force or not os.path.exists(obj) or not os.path.exists(stamp) or open(stamp).read() != dig:
            todo.append((src, obj, stamp, dig))

    def compile_one(job):
        src, obj, stamp, dig = job
        cmd = [NVCC, *FLAGS, *inc, "-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = r.stdout + r.stderr
        with open(obj + ".log", "w") as f:
            f.write(log)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{log}")
        if "bytes spill stores" in log and verbose:
            for line in log.splitlines():
                if "spill" in line and " 0 bytes spill stores" not in line:
                    print(os.path.basename(src), line.strip())
        open(stamp, "w").write(dig)
        return src

    if todo:
        with ThreadPoolExecutor(max_workers=min(8, len(todo))) as ex:
            for s in ex.map(compile_one, todo):
                if verbose:
                    print("compiled", os.path.relpath(s, HERE))
    if todo or not os.path.exists(LIB):
        cmd = [NVCC, "-shared", "-o", LIB, *objs, "-lcudart", "-ldl"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
        if verbose:
            print("linked", LIB)
    return LIB


def ensure_built() -> str:
    """Build once if the shared object is missing (safe under torchrun: an exclusive lock file serialises the ranks)."""
    if os.path.exists(LIB):
        return LIB
    import fcntl
    os.makedirs(OUT_DIR, exist_ok=True)
    with open(os.path.join(OUT_DIR, ".build.lock"), "w") as lk:
        fcntl.flock(lk, fcntl.LOCK_EX)
        try:
            if not os.path.exists(LIB):
                build()
        finally:
            fcntl.flock(lk, fcntl.LOCK_UN)
    return LIB


if __name__ == "__main__":
    build(verbose=True, force="--force" in sys.argv)
