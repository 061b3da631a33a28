"""GPU tier of one image over ranks, by row regions and by tiles (tests/test_regions.py and tests/test_sharding.py hold
the CPU tiers and the workers): the nvcc-built library with two processes on ONE device.  The file sorts last on
purpose -- it holds the only GPU tests that spawn processes and talk over sockets, and `pytest -x` should have run
everything else by the time they start."""
import pytest
from test_regions import _run
from test_sharding import TILE_CASES, _native_worker


@pytest.mark.gpu
def test_gpu_row_regions_two_processes_one_device(ref):
    """the nvcc-built library: two processes share cuda:0 and exchange through the callback transport (gloo, staged
    through host memory) -- the same C++ and kernels as the NCCL path of tools/region_check.py, inside `pytest -m gpu`"""
    _run(2, [0, 1, 2], timeout=240, gpu=True)


@pytest.mark.gpu
def test_gpu_tile_partition_two_processes_one_device(ref):
    """the tile partition on the device, two processes on cuda:0 through the callback transport: byte-identical
    codestream on the writer (5/3; 9/7: same length and main header) and the reference's samples back, lossless for 5/3
    -- including the six 256x256 tiles of a 700x500 12-bit RGB frame with TLM"""
    _run(2, list(range(len(TILE_CASES))), timeout=240, gpu=True, worker=_native_worker)
