"""User-written CUDA models at the edges of the model envelope (nx, nu) = (1,1), (3,3) and (8,4) (MPPI_MAX_NX = 8,
MPPI_MAX_NU = 4), with torch twins that do the same individually rounded operations in the same order, so that the
fused route, the stepped route and the reference agree at the fp32 noise floor.  Their cubins are compiled by
`__graft_entry__.build()`, so the GPU tests load them without compiling.

Every state and action component reaches the cost through its own coefficient, so a swapped index, a skipped component
or a transposed matrix in a kernel changes the result instead of cancelling out:
    s        = x_0 / (1 + x_0^2)                                  (bounded, nonlinear, exactly rounded on both sides)
    drive    = a s - damp x_{nx-1} + sum_j b_j u_j
    x_i     += dt (x_{i+1} + c_i u_i)        i < nx-1             (u_i only for i < nu; x_{i+1} before its own update)
    x_{nx-1} += dt (drive + c_{nx-1} u_{nx-1})                    (u term only if nx-1 < nu)
    cost     = w x_0 x_{nx-1} + sum_i q_i (x_i - g_i)^2 + sum_j r_j u_j^2
    terminal = wT sum_i q_i (x_i - g_i)^2
"""
import numpy as np
import torch

import pytorch_mppi_b200 as eng

SHAPES = ((1, 1), (3, 3), (8, 4))
_DT, _A, _DAMP, _W, _WT = 0, 1, 2, 3, 4


def layout(nx, nu):
    """Index of each coefficient group in the parameter vector."""
    b = 5
    c = b + nu
    r = c + nu
    q = r + nu
    g = q + nx
    return dict(b=b, c=c, r=r, q=q, g=g, n=g + nx)


def default_params(nx, nu):
    L = layout(nx, nu)
    p = [0.0] * L["n"]
    p[_DT], p[_A], p[_DAMP], p[_W], p[_WT] = 0.1, 1.7, 0.35, 0.15, 3.0
    for j in range(nu):
        p[L["b"] + j] = (0.9 - 0.45 * j) if j % 2 == 0 else (-0.6 - 0.2 * j)
        p[L["c"] + j] = 0.25 + 0.2 * j
        p[L["r"] + j] = 0.03 + 0.02 * j
    for i in range(nx):
        p[L["q"] + i] = 1.0 + 0.35 * i
        p[L["g"] + i] = 0.4 - 0.15 * i
    return p


def step_code(nx, nu):
    L = layout(nx, nu)
    last = nx - 1
    lines = ["real s = O::div(x[0], O::add((real)1, O::mul(x[0], x[0])));",
             f"real d = O::sub(O::mul(p[{_A}], s), O::mul(p[{_DAMP}], x[{last}]));"]
    lines += [f"d = O::add(d, O::mul(p[{L['b'] + j}], u[{j}]));" for j in range(nu)]
    for i in range(nx - 1):
        inc = f"x[{i + 1}]" if i >= nu else f"O::add(x[{i + 1}], O::mul(p[{L['c'] + i}], u[{i}]))"
        lines.append(f"x[{i}] = O::add(x[{i}], O::mul(p[{_DT}], {inc}));")
    inc = "d" if last >= nu else f"O::add(d, O::mul(p[{L['c'] + last}], u[{last}]))"
    lines.append(f"x[{last}] = O::add(x[{last}], O::mul(p[{_DT}], {inc}));")
    return "\n    ".join(lines)


def _state_terms(nx, nu, first):
    L = layout(nx, nu)
    out = []
    for i in range(nx):
        out.append(f"real e{i} = O::sub(x[{i}], p[{L['g'] + i}]);")
        term = f"O::mul(p[{L['q'] + i}], O::mul(e{i}, e{i}))"
        out.append(f"real c = {term};" if (i == 0 and first) else f"c = O::add(c, {term});")
    return out


def cost_code(nx, nu):
    L = layout(nx, nu)
    lines = [f"real c = O::mul(p[{_W}], O::mul(x[0], x[{nx - 1}]));"] + _state_terms(nx, nu, first=False)
    lines += [f"c = O::add(c, O::mul(p[{L['r'] + j}], O::mul(u[{j}], u[{j}])));" for j in range(nu)]
    lines.append("return c;")
    return "\n    ".join(lines)


def terminal_code(nx, nu):
    return "\n    ".join(_state_terms(nx, nu, first=True) + [f"return O::mul(p[{_WT}], c);"])


def _cast(p, like):
    """The parameters as the controller dtype rounds them (the kernel reads (real)p[i])."""
    r = np.float32 if like.dtype == torch.float32 else np.float64
    return [float(r(v)) for v in p]


def dynamics(nx, nu, p, state, action):
    P, L = _cast(p, state), layout(nx, nu)
    x = [state[:, i] for i in range(nx)]
    u = [action[:, j] for j in range(nu)]
    last = nx - 1
    s = x[0] / (1.0 + x[0] * x[0])
    d = P[_A] * s - P[_DAMP] * x[last]
    for j in range(nu):
        d = d + P[L["b"] + j] * u[j]
    out = list(x)
    for i in range(nx - 1):
        inc = x[i + 1] if i >= nu else x[i + 1] + P[L["c"] + i] * u[i]
        out[i] = x[i] + P[_DT] * inc
    inc = d if last >= nu else d + P[L["c"] + last] * u[last]
    out[last] = x[last] + P[_DT] * inc
    return torch.stack(out, dim=1)


def _state_cost(nx, nu, P, x):
    L = layout(nx, nu)
    c = None
    for i in range(nx):
        e = x[..., i] - P[L["g"] + i]
        term = P[L["q"] + i] * (e * e)
        c = term if c is None else c + term
    return c


def running_cost(nx, nu, p, state, action):
    P, L = _cast(p, state), layout(nx, nu)
    c = P[_W] * (state[:, 0] * state[:, nx - 1])
    for i in range(nx):
        e = state[:, i] - P[L["g"] + i]
        c = c + P[L["q"] + i] * (e * e)
    for j in range(nu):
        c = c + P[L["r"] + j] * (action[:, j] * action[:, j])
    return c


def terminal_cost(nx, nu, p, states, actions):
    P = _cast(p, states)
    return P[_WT] * _state_cost(nx, nu, P, states[..., -1, :])


def twins(nx, nu, p=None):
    """(dynamics, running_cost, terminal_cost) torch callables of the (nx, nu) model."""
    p = default_params(nx, nu) if p is None else p
    return (lambda s, a: dynamics(nx, nu, p, s, a), lambda s, a: running_cost(nx, nu, p, s, a),
            lambda st, ac: terminal_cost(nx, nu, p, st, ac))


def shape_model(nx, nu, terminal=True):
    p = default_params(nx, nu)
    f, c, t = twins(nx, nu, p)
    return eng.CudaModel(nx, nu, step_code(nx, nu), cost_code(nx, nu), params=p,
                         terminal_code=terminal_code(nx, nu) if terminal else None,
                         dynamics=f, running_cost=c, terminal_cost=t if terminal else None)


def prebuilt():
    """(model, dtype, variant) of every shape-model kernel the GPU tests load: all variants in both dtypes, and the
    terminal-free (3,3) form the MPPI_Batched tests take, in both dtypes."""
    out = [(shape_model(nx, nu), dt, v) for nx, nu in SHAPES for dt in (torch.float32, torch.float64) for v in (0, 1, 2)]
    out += [(shape_model(3, 3, terminal=False), dt, 0) for dt in (torch.float32, torch.float64)]
    return out
