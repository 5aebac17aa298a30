import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


# Property tests draw the SAME examples on every run of the suite (what passed here is what runs elsewhere);
# HYPOTHESIS_PROFILE=explore draws fresh ones.
try:
    from hypothesis import settings as _hyp_settings

    _hyp_settings.register_profile("suite", derandomize=True, deadline=None)
    _hyp_settings.register_profile("explore", deadline=None)
    _hyp_settings.load_profile(os.environ.get("HYPOTHESIS_PROFILE", "suite"))
except ImportError:  # hypothesis is optional for the GPU box
    pass


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs at least one CUDA GPU (run with -m gpu on an H100)")


def _gpu_count() -> int:
    try:
        import torch

        return torch.cuda.device_count() if torch.cuda.is_available() else 0
    except Exception:
        return 0


@pytest.fixture(scope="session")
def gpu_count() -> int:
    return _gpu_count()


@pytest.fixture(scope="session")
def native():
    import hpc_patterns_b200

    if not hpc_patterns_b200.native_available():
        # Build in-tree once (CPU box: nvcc cross-compiles sm_90a without a GPU).
        from hpc_patterns_b200 import _build

        _build.build(cli=True)
    return hpc_patterns_b200.native()


@pytest.fixture(scope="session")
def bin_dir(native) -> str:
    d = os.path.join(ROOT, "bin")
    if not os.path.exists(os.path.join(d, "concurency")):
        from hpc_patterns_b200 import _build

        _build.build(cli=True)
    return d


def pytest_collection_modifyitems(config, items):
    if _gpu_count() > 0:
        return
    skip = pytest.mark.skip(reason="no CUDA GPU in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
