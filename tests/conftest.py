import os
import sys
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


_HAS_GPU = None


def has_gpu():
    """True iff libb200reg can create a handle on device 0 (no torch import needed)."""
    global _HAS_GPU
    if _HAS_GPU is None:
        try:
            import hdl_graph_slam_b200 as pkg
            from hdl_graph_slam_b200 import _capi
            r = pkg.Registration(pkg.default_config(pkg.B2R_METHOD_GICP))
            r.close()
            _HAS_GPU = True
        except Exception as e:  # noqa: BLE001
            code = getattr(e, "code", None)
            if code == -2:  # B2R_ENODEVICE
                _HAS_GPU = False
            else:
                raise
    return _HAS_GPU


def pytest_collection_modifyitems(config, items):
    # GPU tests are skipped ONLY when there is no CUDA device at all; a missing/broken library on a GPU box is an error.
    gpu_items = [it for it in items if "gpu" in it.keywords]
    if not gpu_items:
        return
    if not has_gpu():
        skip = pytest.mark.skip(reason="no CUDA device on this machine")
        for it in gpu_items:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as orc
    orc.build()
    orc.lib()
    return orc


@pytest.fixture(scope="session")
def synth():
    from hdl_graph_slam_b200 import build as b
    b.build_synth()
    from hdl_graph_slam_b200 import synth as s
    return s
