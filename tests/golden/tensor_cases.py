"""Golden cases of a model that reads device tensors (tests/tensor_models.py: bilinear costmap lookup + a reference path
indexed by the horizon step) under MPPI and KMPPI.  Fixtures tests/golden/tens_*.npz, produced by the live reference with
the torch twins (tests/golden/make_golden_tensors.py); each holds the costmap and the path it was made with."""
import functools

import numpy as np
import torch

from oracle import mppi_oracle as orc
from tests import tensor_models as tm
from tests.golden.cases import _DT
from tests.golden.replay import Stream
from tests.golden.step_cases import HorizonClock

TENSOR_CASES = {
    "tens_mppi_f64": dict(variant="mppi", dtype="f64", K=512, T=20, lambda_=1.0, noise_sigma=1.0, u_max=3.0,
                          x0=[-1.2, -0.9], map_hw=[64, 64], map_seed=11, steps=3, seed=901),
    "tens_kmppi_f32": dict(variant="kmppi", dtype="f32", K=2048, T=24, lambda_=1.0, noise_sigma=1.0, u_max=3.0,
                           x0=[-1.5, -1.0], map_hw=[64, 64], map_seed=12, kernel=dict(S=5, sigma=2.0), steps=3, seed=902),
}


def case_tensors(case):
    """(costmap (H, W) float32, path (T, 2) float64) of a case, on the CPU."""
    return (tm.make_costmap(torch.float32, tuple(case["map_hw"]), device="cpu", seed=case["map_seed"]),
            tm.make_path(case["T"], device="cpu"))


def callables(costmap, path, params=tm.NAV_PARAMS):
    """The step-dependent (dynamics, running_cost) twins on these tensors: f(state, u, t)."""
    return (functools.partial(tm.nav_dyn, p=params),
            lambda s, a, t: tm.nav_cost(s, a, t, params, costmap, path))


class TensorOracleRunner:
    """Steps the oracle through a tensor case on the fixture's injected draws."""

    def __init__(self, case, costmap, path):
        self.case = case
        dt = _DT[case["dtype"]]
        f, c = callables(costmap, path)
        self.f = f
        clock = HorizonClock(f, c, case["T"])
        self.prob = orc.Problem(clock.dynamics, clock.running_cost, 2, case["noise_sigma"] * torch.eye(2, dtype=dt),
                                K=case["K"], T=case["T"], lambda_=case["lambda_"],
                                u_max=torch.full((2,), case["u_max"], dtype=dt))
        self.stream = Stream(case, self.prob)
        self.U = self.stream.U0.clone()
        if case["variant"] == "kmppi":
            S, sig = case["kernel"]["S"], case["kernel"]["sigma"]
            self.theta = torch.zeros(S, 2, dtype=dt)
            self.W, self.Wshift = orc.kernel_matrices(case["T"], S, lambda a, b: orc.rbf_kernel(a, b, sig), dt)

    def step(self, x, z):
        if self.case["variant"] == "kmppi":
            r = orc.kmppi_command(self.prob, self.U, self.theta, x, z, self.W, self.Wshift)
            self.theta = r["theta"]
        else:
            r = orc.mppi_command(self.prob, self.U, x, z)
        self.U = r["U"]
        return r

    def advance(self, x, action):
        return self.f(x.view(1, -1), action.view(1, -1), 0).view(-1)


def fixture_tensors(gold, device):
    """The costmap and path a fixture was made with, on `device`."""
    return (torch.from_numpy(np.asarray(gold["costmap"])).to(device).contiguous(),
            torch.from_numpy(np.asarray(gold["path"])).to(device).contiguous())
