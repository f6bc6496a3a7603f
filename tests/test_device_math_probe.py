"""CPU: the device-math probe of tests/test_gpu_device_math.py still compiles for sm_90a with the library's nvcc flags,
so a change to the names or signatures of the primitives it calls (csrc/mppi_math.cuh, csrc/mppi_mlp_tc.cuh) fails
without a GPU."""
import os
import shutil

import pytest

from tests import device_math_probe as probe


@pytest.mark.skipif(shutil.which(os.environ.get("NVCC", "nvcc")) is None, reason="nvcc not found")
def test_device_math_probe_compiles_for_sm90a(tmp_path):
    assert os.path.getsize(probe.build(tmp_path)) > 0
