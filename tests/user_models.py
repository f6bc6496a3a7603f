"""User-written CUDA models used by the tests (compiled with NVRTC by `__graft_entry__.build()`, cubins cached in-tree,
so the GPU tests load them without compiling)."""
import torch

import pytorch_mppi_b200 as eng

PEND_STEP = """
    real uc = clamp<real>(u[0], -p[4], p[4]);
    real acc = O::add(O::mul((real)(3 * 10.0 / 2), O::sin_(x[0])), O::mul((real)3.0, uc));
    real thd = clamp<real>(O::add(x[1], O::mul(acc, p[3])), -p[5], p[5]);
    x[0] = O::add(x[0], O::mul(thd, p[3]));
    x[1] = thd;
"""
PEND_COST = """
    const real pi = (real)3.141592653589793, two_pi = (real)(2 * 3.141592653589793);
    real an = O::sub(remainder<real>(O::add(x[0], pi), two_pi), pi);
    return O::add(O::mul(an, an), O::mul(p[6], O::mul(x[1], x[1])));
"""


def pendulum_user_model():
    ref = eng.Pendulum()
    return eng.CudaModel(2, 1, PEND_STEP, PEND_COST, params=[10.0, 1.0, 1.0, 0.05, 2.0, 8.0, 0.1],
                         dynamics=ref.dynamics, running_cost=ref.running_cost)


# a model that exists nowhere else: x = (pos, vel); vel' = vel + dt (u - c vel); pos' = pos + dt vel'
DT_, DRAG, GOAL, WV, WT = 0.1, 0.3, 1.5, 0.05, 4.0
INT_STEP = "real v = O::add(x[1], O::mul(p[0], O::sub(u[0], O::mul(p[1], x[1])))); x[0] = O::add(x[0], O::mul(p[0], v)); x[1] = v;"
INT_COST = "real d = O::sub(x[0], p[2]); return O::add(O::mul(d, d), O::mul(p[3], O::mul(x[1], x[1])));"
INT_TERM = "real d = O::sub(x[0], p[2]); return O::mul(p[4], O::mul(d, d));"


def int_dyn(s, a):
    v = s[:, 1] + DT_ * (a[:, 0] - DRAG * s[:, 1])
    return torch.stack((s[:, 0] + DT_ * v, v), dim=1)


def int_cost(s, a):
    return (s[:, 0] - GOAL) ** 2 + WV * s[:, 1] ** 2


def int_term(states, actions):
    return WT * (states[..., -1, 0] - GOAL) ** 2


def integrator_user_model():
    return eng.CudaModel(2, 1, INT_STEP, INT_COST, params=[DT_, DRAG, GOAL, WV, WT], terminal_code=INT_TERM,
                         dynamics=int_dyn, running_cost=int_cost, terminal_cost=int_term)
