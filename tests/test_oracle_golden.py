"""CPU: properties of the golden fixtures and the oracle that the replay (tests/test_golden_replay.py) does not check."""
import numpy as np
import torch

from tests.golden.replay import load


def test_fp32_noise_floor_documented():
    """The reference's own fp32-vs-fp64 gap on identical draws at the north-star config — the
    yardstick the 1e-5 target is read against (SURVEY.md §7 'hard parts')."""
    _, g32 = load("pendulum_c2_f32")
    _, g64 = load("pendulum_c2_f64")
    gap = np.abs(g32["U_0"].astype(np.float64) - g64["U_0"]).max()
    assert 1e-7 < gap < 2e-4, gap


def test_rbf_closed_form():
    # reference tests/test_mppi.py:560-570 pins exp(-0.5) for unit-distance points at sigma=1
    from oracle.mppi_oracle import rbf_kernel
    t = torch.tensor([[0.0], [1.0]], dtype=torch.double)
    k = rbf_kernel(t, t, 1.0)
    assert abs(k[0, 1].item() - np.exp(-0.5)) < 1e-6 and abs(k[0, 0].item() - 1.0) < 1e-12
