"""cffi (ABI mode) binding of libbioreason_b200.so.  No fallback: if the library is missing this raises."""
from __future__ import annotations

import os
import re

import cffi

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(os.path.dirname(HERE), "include", "bioreason_b200.h")
LIB_PATH = os.path.join(HERE, "_C", "libbioreason_b200.so")

ffi = cffi.FFI()
_lib = None


def _cdef_text() -> str:
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    out = []
    for line in src.splitlines():
        s = line.strip()
        if s.startswith("#define BR_"):
            out.append(line)
        elif s.startswith("#") or s.startswith('extern "C"') or s == "}":
            continue
        else:
            out.append(line)
    return "\n".join(out)


def exported_symbols() -> list[str]:
    """Every function the header declares (used by the CPU-side ABI test)."""
    return sorted(set(re.findall(r"\b(br_[a-z0-9_]+)\s*\(", _cdef_text())))


ffi.cdef(_cdef_text())       # declarations only; the shared object is opened on first use


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -m bioreason_b200.build` "
                "(there is no CPU / PyTorch fallback for the hot path)")
        _lib = ffi.dlopen(LIB_PATH)
    return _lib


def last_error() -> str:
    buf = ffi.new("char[1024]")
    lib().br_last_error(buf, 1024)
    return ffi.string(buf).decode()


_KERNELS_PER_CALL = {"lmhead_logprob_fwd": 2, "lmhead_logprob_entropy_fwd": 2, "attn_bwd": 2, "sample_next_2stage": 2, "sample_next_2stage_logp": 2,
                     "sample_next_2stage_proc": 2,
                     "quantize_rows_e4m3": 2}
COUNTER = [0]


def check(rc: int, what: str = ""):
    COUNTER[0] += _KERNELS_PER_CALL.get(what, 1)
    if rc != 0:
        raise RuntimeError(f"libbioreason_b200 {what} failed ({rc}): {last_error()}")


def ptr(t, ctype: str = "void*"):
    """Device pointer of a torch tensor (or NULL)."""
    if t is None:
        return ffi.NULL
    return ffi.cast(ctype, t.data_ptr())
