"""Golden cases of a model that reads device tensors (tests/tensor_models.py: bilinear costmap lookup + a reference path
indexed by the horizon step) under MPPI and KMPPI.  Fixtures tests/golden/tens_*.npz, produced by the live reference with
the torch twins (tests/golden/make_golden.py); each holds the costmap and the path it was made with."""
import functools

import numpy as np
import torch

from oracle import mppi_oracle as orc
from tests import tensor_models as tm
from tests.golden.cases import _DT, Family, controller, took_route
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


def _fixture(case):
    costmap, path = case_tensors(case)
    return {"costmap": costmap.numpy(), "path": path.numpy()}


def _model(case, fixture):
    """The oracle's problem on the fixture's costmap and path; the closed loop's simulated system is the dynamics at
    t = 0."""
    dt = _DT[case["dtype"]]
    f, c = callables(*fixture_tensors(fixture, "cpu"))
    clock = HorizonClock(f, c, case["T"])
    prob = orc.Problem(clock.dynamics, clock.running_cost, 2, case["noise_sigma"] * torch.eye(2, dtype=dt),
                       K=case["K"], T=case["T"], lambda_=case["lambda_"], u_max=torch.full((2,), case["u_max"], dtype=dt))
    return prob, lambda x, u: f(x, u, 0)


def _reference(case, prob, fixture):
    dt = _DT[case["dtype"]]
    return (*callables(*fixture_tensors(fixture, "cpu")),
            dict(noise_sigma=case["noise_sigma"] * torch.eye(2, dtype=dt), u_max=torch.full((2,), case["u_max"], dtype=dt),
                 step_dependent_dynamics=True))


def fixture_tensors(gold, device):
    """The costmap and path a fixture was made with, on `device`."""
    return (torch.from_numpy(np.asarray(gold["costmap"])).to(device).contiguous(),
            torch.from_numpy(np.asarray(gold["path"])).to(device).contiguous())


def _engine(case, gold, U0, route, copy_rows=None, **controller_kw):
    """The CudaModel of tests/tensor_models.py on the fixture's costmap and path, on the fused route."""
    dt = _DT[case["dtype"]]
    m = tm.nav_model(*fixture_tensors(gold, "cuda"))
    c = controller(case, m.dynamics, m.running_cost, 2, case["noise_sigma"] * torch.eye(2, dtype=dt), U0,
                   u_max=torch.full((2,), case["u_max"], dtype=dt), step_dependent_dynamics=True, **controller_kw)
    return took_route(c, m, route)


def _check_costs(name, case, route, got, want, tol):
    rtol = 1e-10 if case["dtype"] == "f64" else 5e-6          # the base family's
    np.testing.assert_allclose(got, want, rtol=rtol, atol=rtol)


TENSORS = Family("tensors", TENSOR_CASES, _model, _reference, _fixture, scalars=False, engine=_engine,
                 check_costs=_check_costs, lockable=lambda case: case["K"] <= 2048)
