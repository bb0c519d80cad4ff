"""pytest configuration: markers and import paths."""

import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
for p in (ROOT, ROOT / "tests"):
    if str(p) not in sys.path:
        sys.path.insert(0, str(p))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


import pytest


@pytest.fixture(params=["exact", "fast"])
def coords(request):
    """K1 coordinate mode of fp32 trilinear resampling: "exact" keeps the reference's fp32
    rounding chain on every voxel (TIO_EXACT_COORDS), "fast" is the default one-fma form for
    voxels whose taps are all inside the volume.  Yields the tolerance against the oracle."""
    from torchio_b200 import ops

    previous = ops.set_exact_coords(request.param == "exact")
    try:
        yield request.param
    finally:
        ops.set_exact_coords(previous)
