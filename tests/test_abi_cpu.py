"""CPU-side checks of the C-ABI boundary: the library builds, loads, and exports every declared symbol."""
import ctypes
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built_lib():
    from bioreason_b200 import build
    return build.build()


def test_library_exports_every_declared_symbol(built_lib):
    from bioreason_b200 import _lib
    dll = ctypes.CDLL(built_lib)
    names = _lib.exported_symbols()
    assert len(names) >= 15
    missing = [n for n in names if not hasattr(dll, n)]
    assert not missing, f"declared in include/bioreason_b200.h but not exported: {missing}"


def test_cffi_parses_header_and_loads(built_lib):
    from bioreason_b200 import _lib
    lib = _lib.lib()
    assert lib.br_version() >= 100
    buf = _lib.ffi.new("char[64]")
    assert lib.br_last_error(buf, 64) >= 0


def test_ops_refuse_cpu_tensors():
    import torch
    from bioreason_b200 import ops
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.grpo_advantages(torch.zeros(8, 2), 4)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.gemm(torch.zeros(8, 8, dtype=torch.bfloat16), torch.zeros(8, 8, dtype=torch.bfloat16))


def test_sass_is_hopper_native(built_lib):
    """Every contraction must be a warpgroup MMA fed by TMA, not a recompiled mma.sync kernel."""
    import shutil, subprocess
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    # every contraction of the path -- GEMMs, decode weight streaming, flash attention forward / backward, LoRA gradients -- must be
    # wgmma (HGMMA) fed by TMA (UTMALDG), and must NOT contain the legacy mma.sync path (HMMA)
    objs = ("gemm_tc5.o", "decode_gemm_tc5.o", "attn_fwd_tc5.o", "attn_bwd_tc5.o", "lora_grad_tc5.o")
    for name in objs:
        sass = subprocess.run([cuobjdump, "-sass", os.path.join(os.path.dirname(built_lib), name)], capture_output=True, text=True).stdout
        for mnemonic in ("HGMMA", "UTMALDG"):
            assert mnemonic in sass, (name, mnemonic)
        assert "HMMA." not in sass, f"{name} still contains mma.sync (HMMA)"
    # ... and nothing else on the dense path may carry mma.sync: the round-1 attention and x^T y kernels are gone
    for name in ("attn_fwd.o", "attn_bwd.o", "backward_rows.o", "elementwise.o", "grpo_loss.o"):
        sass = subprocess.run([cuobjdump, "-sass", os.path.join(os.path.dirname(built_lib), name)], capture_output=True, text=True).stdout
        assert "HMMA." not in sass, f"{name} contains mma.sync (HMMA)"
    # P / dS / P^T stay in registers: the probability tiles feed the register-A form of the warpgroup MMA
    for name in ("attn_fwd_tc5.o", "attn_bwd_tc5.o"):
        sass = subprocess.run([cuobjdump, "-sass", os.path.join(os.path.dirname(built_lib), name)], capture_output=True, text=True).stdout
        assert "HGMMA.64x128x16.F32.BF16 R" in sass, name


def test_product_never_imports_the_oracle():
    """oracle/ is test infrastructure: only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline leg may touch it."""
    import re
    bad = []
    for base in ("bioreason_b200", "compat"):
        for dirpath, _, files in os.walk(os.path.join(ROOT, base)):
            for f in files:
                if f.endswith(".py"):
                    src = open(os.path.join(dirpath, f)).read()
                    if re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M):
                        bad.append(os.path.join(dirpath, f))
    assert not bad, bad
    bench = open(os.path.join(ROOT, "bench.py")).read()
    b200_arm = bench[bench.index("def run_b200"):bench.index("# CPU reference arm")]
    assert "oracle" not in b200_arm.replace("oracle's", "")           # the timed arm is oracle-free
