"""User-written CUDA models whose rollout copies differ (CudaModel(copies=M), rollout_samples=M), used by the tests; their
cubins are compiled by `__graft_entry__.build()`, so the GPU tests load them without compiling.

* A pendulum ensemble (domain randomisation): copy m has its own mass p[6 + m] and length p[6 + M + m]; the terminal
  cost is weighted by the copy's length, so the terminal cost of every copy differs too.
* The linear point of the reference's M > 1 fixtures (tests/golden/cases.py: copy m is pushed by m * copy_offset every
  step), for replaying them on the fused route.
* A step- and copy-dependent double integrator (scenario disturbances): copy m is pushed by w[m][t] = p[3 + M + m*T + t]
  at horizon step t, and its terminal cost has its own weight p[3 + m].  The table goes past MPPI_MODEL_PARAM_DOUBLES
  into model_params_ext.

The torch twins are called as the reference calls an M-copy rollout (mppi.py:348-364): M*K rows, copy-major, so row r
belongs to copy r // K.  They read `model.params`, so they follow `set_params` as the compiled bodies do, and they have to
know K (the controller's num_samples)."""
import torch

import pytorch_mppi_b200 as eng

# g, dt, max_torque, max_speed, w_thdot, w_terminal, then masses[M], lengths[M]
PEND_BASE = [10.0, 0.05, 2.0, 8.0, 0.1, 2.0]
PEND_MASSES = [1.0, 0.8, 1.3, 1.1, 0.9, 1.2, 0.7, 1.4]
PEND_LENGTHS = [1.0, 1.2, 0.9, 0.8, 1.1, 1.05, 0.95, 1.3]
PEND_STEP = """
    const real mass = p[6 + m], len = p[6 + COPIES + m];
    real uc = clamp<real>(u[0], -p[2], p[2]);
    real a_g = O::div(O::mul((real)3, p[0]), O::mul((real)2, len));
    real a_u = O::div((real)3, O::mul(mass, O::mul(len, len)));
    real acc = O::add(O::mul(a_g, O::sin_(x[0])), O::mul(a_u, uc));
    real thd = clamp<real>(O::add(x[1], O::mul(acc, p[1])), -p[3], p[3]);
    x[0] = O::add(x[0], O::mul(thd, p[1]));
    x[1] = thd;
"""
PEND_COST = "return O::add(O::mul(x[0], x[0]), O::mul(p[4], O::mul(x[1], x[1])));"
PEND_TERM = "return O::mul(O::mul(p[5], p[6 + COPIES + m]), O::mul(x[0], x[0]));"


def pendulum_params(M, masses=PEND_MASSES, lengths=PEND_LENGTHS):
    return PEND_BASE + list(masses[:M]) + list(lengths[:M])


def _copy_of_row(n, K, device):
    """Copy index of each of n rows: the reference's (M,K) copy-major flattening."""
    return torch.div(torch.arange(n, device=device), K, rounding_mode="floor")


def pend_dyn(s, a, p, M, K):
    g, dt, mt, ms = (torch.tensor(v, dtype=s.dtype, device=s.device) for v in p[:4])
    tab = torch.tensor(p[6:6 + 2 * M], dtype=s.dtype, device=s.device)
    idx = _copy_of_row(s.shape[0], K, s.device)
    mass, length = tab[idx], tab[M + idx]
    three = torch.tensor(3.0, dtype=s.dtype, device=s.device)      # a tensor numerator: `3 / x` multiplies by 1 / x
    uc = torch.clamp(a[:, 0], -mt, mt)
    acc = (3 * g) / (2 * length) * torch.sin(s[:, 0]) + three / (mass * (length * length)) * uc
    thd = torch.clamp(s[:, 1] + acc * dt, -ms, ms)
    return torch.stack((s[:, 0] + thd * dt, thd), dim=1)


def pend_cost(s, a, p):
    w = torch.tensor(p[4], dtype=s.dtype, device=s.device)
    return s[:, 0] * s[:, 0] + w * (s[:, 1] * s[:, 1])


def pend_term(states, actions, p, M):
    """states (M,K,T,nx) -> (M,K)"""
    w = torch.tensor(p[5], dtype=states.dtype, device=states.device)
    length = torch.tensor(p[6 + M:6 + 2 * M], dtype=states.dtype, device=states.device)
    th = states[..., -1, 0]
    return (w * length).unsqueeze(1) * (th * th)


def pendulum_ensemble(M, K, params=None):
    m = eng.CudaModel(2, 1, PEND_STEP, PEND_COST, params=params or pendulum_params(M), terminal_code=PEND_TERM, copies=M,
                      dynamics=lambda s, a: pend_dyn(s, a, m.params, M, K),
                      running_cost=lambda s, a: pend_cost(s, a, m.params),
                      terminal_cost=lambda states, actions: pend_term(states, actions, m.params, M))
    return m


# dt, w_vel, goal, then the terminal weights w_T[M], then the disturbance scenarios w[m][t] (M x T)
SI_BASE = [0.1, 0.05, 1.0]
SI_TERMINAL_WEIGHTS = [3.0, 1.0, 5.0, 2.0, 4.0, 1.5, 2.5, 3.5]


def scenario_params(M, T, seed=7):
    g = torch.Generator().manual_seed(seed)
    return SI_BASE + SI_TERMINAL_WEIGHTS[:M] + (0.8 * torch.randn(M * T, generator=g, dtype=torch.float64)).tolist()


def _si_step(T):
    return f"""
    real v = O::add(x[1], O::mul(p[0], O::add(u[0], p[3 + COPIES + m * {T} + t])));
    x[0] = O::add(x[0], O::mul(p[0], v));
    x[1] = v;
"""


SI_COST = "real d = O::sub(x[0], p[2]); return O::add(O::mul(d, d), O::mul(p[1], O::mul(x[1], x[1])));"
SI_TERM = "real d = O::sub(x[0], p[2]); return O::mul(p[3 + m], O::mul(d, d));"


def si_dyn(s, a, t, p, M, T, K):
    dt = torch.tensor(p[0], dtype=s.dtype, device=s.device)
    w = torch.tensor(p[3 + M:3 + M + M * T], dtype=s.dtype, device=s.device).view(M, T)[:, t]
    v = s[:, 1] + dt * (a[:, 0] + w[_copy_of_row(s.shape[0], K, s.device)])
    return torch.stack((s[:, 0] + dt * v, v), dim=1)


def si_cost(s, a, t, p):
    wv, goal = (torch.tensor(v, dtype=s.dtype, device=s.device) for v in (p[1], p[2]))
    d = s[:, 0] - goal
    return d * d + wv * (s[:, 1] * s[:, 1])


def si_term(states, actions, p, M):
    """states (M,K,T,nx) -> (M,K)"""
    goal = torch.tensor(p[2], dtype=states.dtype, device=states.device)
    wt = torch.tensor(p[3:3 + M], dtype=states.dtype, device=states.device)
    d = states[..., -1, 0] - goal
    return wt.unsqueeze(1) * (d * d)


def scenario_integrator(M, T, K, params=None):
    m = eng.CudaModel(2, 1, _si_step(T), SI_COST, params=params or scenario_params(M, T), terminal_code=SI_TERM, copies=M,
                      step_dependent=True,
                      dynamics=lambda s, a, t: si_dyn(s, a, t, m.params, M, T, K),
                      running_cost=lambda s, a, t: si_cost(s, a, t, m.params),
                      terminal_cost=lambda states, actions: si_term(states, actions, m.params, M))
    return m


# x' = x + B u + m * offset; cost |goal - x|^2; terminal terminal_scale |goal - x_T|^2 (oracle LinearPointModel, Q = I)
LIN_STEP = """
    x[0] = O::add(O::add(x[0], O::add(O::mul(u[0], p[0]), O::mul(u[1], p[1]))), O::mul((real)m, p[6]));
    x[1] = O::add(O::add(x[1], O::add(O::mul(u[0], p[2]), O::mul(u[1], p[3]))), O::mul((real)m, p[7]));
"""
LIN_COST = "real d0 = O::sub(p[4], x[0]), d1 = O::sub(p[5], x[1]); return O::add(O::mul(d0, d0), O::mul(d1, d1));"
LIN_TERM = ("real d0 = O::sub(p[4], x[0]), d1 = O::sub(p[5], x[1]); "
            "return O::mul(p[8], O::add(O::mul(d0, d0), O::mul(d1, d1)));")


def copy_offset_linear(M, B, goal, offset, terminal_scale=0.0, terminal_cost=None):
    """Compiled only (the replay test feeds the fixture's draws; no torch twins for dynamics and running cost)."""
    params = [float(v) for row in B for v in row] + list(goal) + list(offset) + [terminal_scale]
    return eng.CudaModel(2, 2, LIN_STEP, LIN_COST, params=params, terminal_code=LIN_TERM if terminal_scale else None,
                         terminal_cost=terminal_cost, copies=M)


def prebuilt():
    """(model, dtype, variant) of every ensemble kernel the GPU tests and scripts/time_ensemble.py load."""
    f32, f64 = torch.float32, torch.float64
    out = [(pendulum_ensemble(4, 1), f64, 0), (pendulum_ensemble(3, 1), f32, 1), (pendulum_ensemble(8, 1), f64, 2),
           (scenario_integrator(4, 15, 1), f64, 0)]
    out += [(pendulum_ensemble(M, 1), f32, 0) for M in (2, 4, 8)]
    out += [(copy_offset_linear(3, [[1.0, 0.0], [0.0, -1.0]], [2.0, 2.0], [0.05, -0.03], 1.0), f64, 0),
            (copy_offset_linear(4, [[1.0, 0.0], [0.0, -1.0]], [2.0, 2.0], [0.04, 0.02]), f32, 0)]
    return out
