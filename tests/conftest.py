import os, sys
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); run with -m gpu")
    config.addinivalue_line("markers", "needs_lib: CPU test that loads libbioreason_b200.so (symbols only, no compute)")


_BUILT = []


@pytest.fixture(autouse=True)
def _built_library(request):
    """GPU tests (and the ABI test, which asks for it explicitly) need libbioreason_b200.so to match the sources (hash-checked,
    a no-op when up to date).  CPU tests that mock the ops must run on a box without nvcc: nothing is built for them."""
    if request.node.get_closest_marker("gpu") is None and request.node.get_closest_marker("needs_lib") is None:
        return
    if not _BUILT:
        import shutil
        from bioreason_b200 import build
        if not (shutil.which("nvcc") or os.path.exists(build.NVCC)):
            if os.path.exists(build.LIB):
                _BUILT.append(build.LIB)
                return
            pytest.skip("nvcc not available and libbioreason_b200.so not built")
        _BUILT.append(build.build())


@pytest.fixture(scope="session")
def golden():
    import torch
    return torch.load(os.path.join(ROOT, "tests", "golden", "reference_tiny.pt"), weights_only=True)


@pytest.fixture(scope="session")
def tiny_oracle(golden):
    """Oracle DNA-LLM carrying exactly the weights the reference run used."""
    import torch
    from bioreason_b200.configs import text_config, dna_config
    from oracle.models import build_oracle
    m = build_oracle(text_config("tiny"), dna_config("tiny"), seed=99)   # different seed on purpose
    missing, unexpected = m.load_state_dict({k: v.float() for k, v in golden["weights"].items()}, strict=False)
    assert not unexpected and all("inv_freq" in k or "position_ids" in k for k in missing), (missing, unexpected)
    return m.eval()
