"""Golden cases of step-dependent dynamics and cost (step_dependent_dynamics=True, reference mppi.py:147-157): the model
of tests/step_models.py under MPPI, KMPPI and MPPI_Batched.  Fixtures tests/golden/stepint_*.npz, produced by the live
reference (tests/golden/make_golden.py); kept apart from cases.CASES so that the tests parametrised over those do not see
them.

The oracle (oracle/mppi_oracle.py) calls its plugins as `dynamics(state, u)` / `running_cost(state, u)`.  Its rollouts,
like the reference's (mppi.py:312-319, 849-853), call dynamics and then running_cost exactly once per horizon step,
t = 0, ..., T-1, in order, once per command; `HorizonClock` relies on that order to hand the step-dependent callables
their t, and refuses any other call sequence."""
import functools

import numpy as np
import torch

import pytorch_mppi_b200 as eng
from oracle import mppi_oracle as orc
from tests import step_models as sm
from tests.golden.cases import _DT, U_TOL, Family, controller, took_route

STEPINT = {"kind": "step_integrator", "params": list(sm.SD_PARAMS), "terminal": True}
STEP_CASES = {
    "stepint_mppi_f64": dict(variant="mppi", model=STEPINT, dtype="f64", K=512, T=20, lambda_=1.0, noise_sigma=1.0,
                             u_max=3.0, x0=[0.0, 0.0], steps=3, seed=801),
    "stepint_kmppi_f32": dict(variant="kmppi", model=STEPINT, dtype="f32", K=2048, T=24, lambda_=1.0, noise_sigma=2.0,
                              u_max=3.0, x0=[0.2, -0.1], kernel=dict(S=6, sigma=2.0), steps=3, seed=802),
}
STEP_BATCHED_CASES = {
    "stepint_batched_f64": dict(model=dict(STEPINT, terminal=False), dtype="f64", N=3, K=384, T=15, lambda_=0.8,
                                noise_sigma=1.0, u_max=3.0, x0=[[0.0, 0.0], [1.0, -0.5], [-1.0, 0.5]], steps=3, seed=803),
}


class HorizonClock:
    """dynamics(state, u) / running_cost(state, u) for the oracle, calling f(state, u, t) / c(state, u, t) with the
    horizon index of the step the rollout is at (see the module docstring)."""

    def __init__(self, f, c, T):
        self.f, self.c, self.T = f, c, T
        self.t, self.stepped = 0, False

    def dynamics(self, state, u):
        assert not self.stepped, "dynamics called twice without the running cost of the step in between"
        self.stepped = True
        return self.f(state, u, self.t)

    def running_cost(self, state, u):
        assert self.stepped, "running cost called before the dynamics of its step"
        self.stepped = False
        cost = self.c(state, u, self.t)
        self.t = (self.t + 1) % self.T
        return cost


def callables(case):
    """The step-dependent (dynamics, running_cost, terminal cost or None) of a case: f(state, u, t) etc."""
    m = case["model"]
    p = m["params"]
    term = functools.partial(sm.sd_term, p=p) if m["terminal"] else None
    return functools.partial(sm.sd_dyn, p=p), functools.partial(sm.sd_cost, p=p), term


def step_problem(case, dynamics=None, running_cost=None):
    """The oracle's Problem of a case; `dynamics` / `running_cost` (f(state, u, t)) replace the case's own."""
    dt = _DT[case["dtype"]]
    f, c, term = callables(case)
    clock = HorizonClock(dynamics or f, running_cost or c, case["T"])
    return orc.Problem(clock.dynamics, clock.running_cost, 2, torch.tensor(case["noise_sigma"], dtype=dt), K=case["K"],
                       T=case["T"], lambda_=case["lambda_"], u_max=torch.tensor(case["u_max"], dtype=dt),
                       terminal_state_cost=term)


def _model(case, fixture):
    """The oracle's problem, and the closed loop's simulated system: the model at t = 0, the horizon index of the step
    being applied."""
    return step_problem(case), lambda x, u: sm.sd_dyn(x, u, 0, case["model"]["params"])


def _reference(case, prob, fixture):
    f, c, term = callables(case)
    dt = _DT[case["dtype"]]
    kw = dict(noise_sigma=torch.tensor(case["noise_sigma"], dtype=dt), u_max=torch.tensor(case["u_max"], dtype=dt),
              step_dependent_dynamics=True)
    if term is not None:
        kw["terminal_state_cost"] = term
    return f, c, kw


def _engine(case, gold, U0, route, copy_rows=None, **controller_kw):
    """The CudaModel of tests/step_models.py (step_dependent=True) on the fused route."""
    dt = _DT[case["dtype"]]
    m = sm.step_dependent_user_model(case["model"]["params"], terminal=case["model"]["terminal"])
    sigma, u_max = torch.tensor(case["noise_sigma"], dtype=dt), torch.tensor(case["u_max"], dtype=dt)
    if "N" in case:
        c = eng.MPPI_Batched(m.dynamics, m.running_cost, 2, sigma, case["N"], num_samples=case["K"], horizon=case["T"],
                             lambda_=case["lambda_"], u_max=u_max, step_dependent_dynamics=True, device="cuda", **controller_kw)
        c.U = U0.clone()
    else:
        c = controller(case, m.dynamics, m.running_cost, 2, sigma, U0, u_max=u_max, terminal_state_cost=m.terminal_cost,
                       step_dependent_dynamics=True, **controller_kw)
    return took_route(c, m, route)


# stepint_kmppi_f32: the force sin(0.7 t) is CUDA's sinf in the kernel and numpy's float32 sin in the reference (1-ulp
# differences, as the pendulum's sin: cases.U_TOL_OVERRIDE); measured 1.2e-5 on H100, bound 2e-5.  The costs, too.
_F32_TOL = 2e-5


def _check_costs(name, case, route, got, want, tol):
    rtol = 1e-10 if case["dtype"] == "f64" else _F32_TOL
    np.testing.assert_allclose(got, want, rtol=rtol, atol=rtol)


STEP = Family("step", dict(STEP_CASES, **STEP_BATCHED_CASES), _model, _reference, engine=_engine,
              u_tol=lambda name, case, route: U_TOL["f64"] if case["dtype"] == "f64" else _F32_TOL,
              check_costs=_check_costs, lockable=lambda case: "N" not in case and case["K"] <= 2048)
