"""A tracking problem with a step-dependent user model (tests/step_models.py: double integrator with a time-varying force,
moving target) at K=16384, T=30, fp32, with `set_params` moving the target before every control step: time per step of
the fused `command()` (back to back), the fused `command_host()` (the action back on the
host every step) and the stepped route (the same torch twins in a Python T-loop).  Prints one JSON line with the card
name and power limit."""
import itertools
import os
import sys

import torch

import timing

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402
from tests import step_models as um  # noqa: E402

K, T = 16384, 30


def make(m, stepped):
    dyn, cost, term = m.dynamics, m.running_cost, m.terminal_cost
    if stepped:
        dyn, cost, term = (lambda s, a, t: m.dynamics(s, a, t)), (lambda s, a, t: m.running_cost(s, a, t)), (lambda s, a: m.terminal_cost(s, a))
    c = eng.MPPI(dyn, cost, 2, torch.tensor(1.0), num_samples=K, horizon=T, U_init=torch.zeros(T, 1), u_max=torch.tensor(3.0),
                 terminal_state_cost=term, step_dependent_dynamics=True, device="cuda", rng_seed=1)
    assert (c._model is None) == stepped
    return c


def per_step_us(m, c, call, n):
    p = list(m.params)
    i = itertools.count()

    def step():
        p[3] = 0.5 + 0.03 * (next(i) % n)           # the target moves every control step
        m.set_params(p)
        return call(c, [0.0, 0.0])

    return timing.back_to_back_us(step, n)


def main():
    m = um.step_dependent_user_model()
    fused, stepped = make(m, False), make(m, True)
    out = {
        "fused_command_us": per_step_us(m, fused, lambda c, x: c.command(x), 2000),
        "fused_command_host_us": per_step_us(m, fused, lambda c, x: c.command_host(x), 2000),
        "stepped_command_us": per_step_us(m, stepped, lambda c, x: c.command(x), 100),
        "split_cost": int(fused.launch_info.split_cost),
    }
    out["config"] = f"K={K} T={T} fp32, set_params before every step"
    timing.emit(out)


if __name__ == "__main__":
    main()
