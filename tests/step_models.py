"""A step-dependent user-written CUDA model used by the tests (CudaModel(step_dependent=True); its cubins are compiled by
`__graft_entry__.build()`, so the GPU tests load them without compiling).

A double integrator driven by u plus the time-varying force p[1] sin(p[2] t), tracking the moving target p[3] + p[4] t,
with a terminal cost towards p[7].  The force and the target change enough from one step to the next that a cost or a
step evaluated at t +- 1 misses the golden fixtures by far more than any parity tolerance
(tests/test_step_dependent.py)."""
import numpy as np
import torch

import pytorch_mppi_b200 as eng

SD_PARAMS = [0.1, 4.0, 0.7, 0.5, 0.3, 0.05, 4.0, 4.0]     # dt, force amplitude, force frequency, target c0 c1, w_vel, w_T, x_T
SD_STEP = """
    real f = O::mul(p[1], O::sin_(O::mul(p[2], (real)t)));
    real v = O::add(x[1], O::mul(p[0], O::add(u[0], f)));
    x[0] = O::add(x[0], O::mul(p[0], v));
    x[1] = v;
"""
SD_COST = """
    real d = O::sub(x[0], O::add(p[3], O::mul(p[4], (real)t)));
    return O::add(O::mul(d, d), O::mul(p[5], O::mul(x[1], x[1])));
"""
SD_TERM = "real d = O::sub(x[0], p[7]); return O::mul(p[6], O::mul(d, d));"


def _real(like):
    """The scalar type of `like`'s dtype: the t-dependent scalars are computed with the kernel's roundings."""
    return np.float32 if like.dtype == torch.float32 else np.float64


def sd_dyn(s, a, t, p=SD_PARAMS):
    r = _real(s)
    f = float(r(p[1]) * np.sin(r(p[2]) * r(t)))
    dt = float(r(p[0]))
    v = s[:, 1] + dt * (a[:, 0] + f)
    return torch.stack((s[:, 0] + dt * v, v), dim=1)


def sd_cost(s, a, t, p=SD_PARAMS):
    r = _real(s)
    d = s[:, 0] - float(r(p[3]) + r(p[4]) * r(t))
    return d * d + float(r(p[5])) * (s[:, 1] * s[:, 1])


def sd_term(states, actions, p=SD_PARAMS):
    d = states[..., -1, 0] - float(_real(states)(p[7]))
    return float(_real(states)(p[6])) * (d * d)


def step_dependent_user_model(params=SD_PARAMS, terminal=True):
    """The torch twins read `m.params`, so they follow `set_params` as the compiled bodies do."""
    m = eng.CudaModel(2, 1, SD_STEP, SD_COST, params=params, terminal_code=SD_TERM if terminal else None, step_dependent=True,
                      dynamics=lambda s, a, t: sd_dyn(s, a, t, m.params),
                      running_cost=lambda s, a, t: sd_cost(s, a, t, m.params),
                      terminal_cost=(lambda states, actions: sd_term(states, actions, m.params)) if terminal else None)
    return m
