import os, sys
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")
    # the CUDA library is a build artefact (git-ignored): compile it when the tree is fresh, so the host-side tests that load
    # it (symbol exports, module mirrors) and the GPU tests never depend on an earlier manual build
    lib = os.path.join(ROOT, "nope_nerf_b200", "libnope_nerf_b200.so")
    if not os.path.exists(lib):
        import __graft_entry__
        __graft_entry__.build()
