"""Golden cases of rollout_samples M > 1 with copies that differ (reference mppi.py:334-373): the models of
tests/ensemble_models.py under MPPI, SMPPI and KMPPI.  Fixtures tests/golden/ens_*.npz, produced by the live reference
(tests/golden/make_golden.py); kept apart from cases.CASES so that the tests parametrised over those do not see them.
The step-dependent case hands the oracle its callables through step_cases.HorizonClock: an M-copy rollout also calls
dynamics, then the running cost, once per horizon step."""
import functools

import numpy as np
import torch

from oracle import mppi_oracle as orc
from tests import ensemble_models as em
from tests.golden.cases import _DT, Family, controller, plain, took_route
from tests.golden.step_cases import HorizonClock

ENSEMBLE_CASES = {
    "ens_pend_mppi_f64": dict(variant="mppi", model="pendulum", dtype="f64", M=4, K=512, T=20, lambda_=1.0,
                              noise_sigma=1.0, u_max=2.0, x0=[2.5, 0.5], var_cost=0.5, var_discount=0.9, steps=3, seed=901),
    "ens_pend_smppi_f32": dict(variant="smppi", model="pendulum", dtype="f32", M=3, K=1024, T=16, lambda_=1.0,
                               noise_sigma=0.5, u_max=2.0, x0=[2.0, -0.3], var_cost=0.8, var_discount=0.95,
                               smooth=dict(w=0.5, delta_t=0.5, action_max=2.0), steps=3, seed=902),
    "ens_pend_kmppi_f64": dict(variant="kmppi", model="pendulum", dtype="f64", M=8, K=256, T=16, lambda_=1.0,
                               noise_sigma=1.0, u_max=2.0, x0=[2.8, 0.0], var_cost=0.3, var_discount=0.85,
                               kernel=dict(S=5, sigma=2.0), steps=3, seed=903),
    "ens_stepint_mppi_f64": dict(variant="mppi", model="scenario_integrator", dtype="f64", M=4, K=384, T=15, lambda_=1.0,
                                 noise_sigma=1.0, u_max=3.0, x0=[0.0, 0.0], var_cost=1.0, var_discount=0.9, steps=3,
                                 seed=904),
}


def case_params(case):
    if case["model"] == "pendulum":
        return em.pendulum_params(case["M"])
    return em.scenario_params(case["M"], case["T"])


def callables(case, params=None):
    """(dynamics, running_cost, terminal cost) the reference is given for these parameters (default: the case's);
    the scenario integrator's take t."""
    p = case_params(case) if params is None else params
    M, K, T = case["M"], case["K"], case["T"]
    if case["model"] == "pendulum":
        return (functools.partial(em.pend_dyn, p=p, M=M, K=K), functools.partial(em.pend_cost, p=p),
                functools.partial(em.pend_term, p=p, M=M))
    return (functools.partial(em.si_dyn, p=p, M=M, T=T, K=K), functools.partial(em.si_cost, p=p),
            functools.partial(em.si_term, p=p, M=M))


def shifted_params(case, shift):
    """The case's parameters with copy m's values at copy m - shift: what a twin whose copy index is off by `shift`
    reads.  (Every copy's rollout is then another copy's, so only a twin that also evaluates a copy-dependent cost with
    the right index, as the terminal costs here, can tell.)"""
    p, M, T = case_params(case), case["M"], case["T"]
    perm = [(m + shift) % M for m in range(M)]
    if case["model"] == "pendulum":
        return p[:6] + [p[6 + j] for j in perm] + [p[6 + M + j] for j in perm]
    return p[:3 + M] + sum((p[3 + M + j * T:3 + M + (j + 1) * T] for j in perm), [])


def ensemble_problem(case, dyn_params=None):
    """The oracle's Problem of a case; with `dyn_params`, its dynamics read those parameters instead of the case's."""
    dt = _DT[case["dtype"]]
    f, c, term = callables(case)
    if dyn_params is not None:
        f = callables(case, dyn_params)[0]
    if case["model"] == "scenario_integrator":
        clock = HorizonClock(f, c, case["T"])
        f, c = clock.dynamics, clock.running_cost
    return orc.Problem(f, c, 2, torch.tensor(case["noise_sigma"], dtype=dt), K=case["K"], T=case["T"],
                       lambda_=case["lambda_"], u_max=torch.tensor(case["u_max"], dtype=dt), terminal_state_cost=term,
                       rollout_samples=case["M"], rollout_var_cost=case["var_cost"],
                       rollout_var_discount=case["var_discount"])


def plant_step(case, x, u):
    """The closed loop's simulated system: copy 0 (at t = 0)."""
    f, _, _ = callables(case)
    return f(x, u) if case["model"] == "pendulum" else f(x, u, 0)


def _model(case, fixture):
    return ensemble_problem(case), functools.partial(plant_step, case)


def _reference(case, prob, fixture):
    dt = _DT[case["dtype"]]
    f, c, term = callables(case)
    return f, c, dict(noise_sigma=torch.tensor(case["noise_sigma"], dtype=dt), u_max=torch.tensor(case["u_max"], dtype=dt),
                      terminal_state_cost=term, rollout_samples=case["M"], rollout_var_cost=case["var_cost"],
                      rollout_var_discount=case["var_discount"],
                      step_dependent_dynamics=case["model"] == "scenario_integrator")


def engine_model(case, K=None, params=None):
    """The case's CudaModel(copies=M) for `K` samples per copy (default the case's), with `params` (default the case's)."""
    K, p = K or case["K"], params or case_params(case)
    if case["model"] == "pendulum":
        return em.pendulum_ensemble(case["M"], K, p)
    return em.scenario_integrator(case["M"], case["T"], K, p)


def ensemble_controller(case, m, route="fused", U0=None, **kw):
    """The controller of a case around the model `m`: on the fused route, or on the stepped route with m's torch twins
    (the reference's M-copy T-loop)."""
    dt = _DT[case["dtype"]]
    c = controller(case, plain(m.dynamics) if route == "stepped" else m.dynamics, m.running_cost, 2,
                   torch.tensor(case["noise_sigma"], dtype=dt), U0, **dict(dict(
                       u_max=torch.tensor(case["u_max"], dtype=dt), terminal_state_cost=m.terminal_cost,
                       rollout_samples=case["M"], rollout_var_cost=case["var_cost"],
                       rollout_var_discount=case["var_discount"],
                       step_dependent_dynamics=case["model"] == "scenario_integrator"), **kw))
    return took_route(c, m, route)


def _engine(case, gold, U0, route, copy_rows=None, **controller_kw):
    return ensemble_controller(case, engine_model(case, K=copy_rows), route, U0, **controller_kw)


def _check_costs(name, case, route, got, want, tol):
    np.testing.assert_allclose(got, want, rtol=0, atol=tol * max(1.0, float(np.abs(want).max())))


ENSEMBLE = Family("ensemble", ENSEMBLE_CASES, _model, _reference, smooth_key="action_sequence", scalars=False,
                  engine=_engine, check_costs=_check_costs)
