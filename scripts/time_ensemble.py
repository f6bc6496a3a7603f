"""Ensemble controllers (tests/ensemble_models.py: pendulum with a mass and length per copy, terminal cost) at K=16384,
T=30, fp32, for rollout_samples M in {1, 2, 4, 8}: time per command of the fused `command()` back to back, of the
fused `command()` with L2 flushed before each command, and of the stepped route (the same torch twins in the
reference's M-copy Python T-loop).  M = 1 is the same pendulum compiled without copies, on the single-loop kernel
(the one copies use) and on the split-cost kernel (the default for one copy at this size).  Prints one JSON line with
the card name and power limit."""
import os
import sys

import torch

import timing

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402
from tests import ensemble_models as em  # noqa: E402

K, T = 16384, 30
X0 = [2.5, 0.5]


def model(M):
    if M > 1:
        return em.pendulum_ensemble(M, K)
    one = "const int m = 0, COPIES = 1; (void)m; (void)COPIES;\n"      # the same bodies for a model without copies
    m = eng.CudaModel(2, 1, one + em.PEND_STEP, em.PEND_COST, params=em.pendulum_params(1), terminal_code=one + em.PEND_TERM,
                      dynamics=lambda s, a: em.pend_dyn(s, a, m.params, 1, K),
                      running_cost=lambda s, a: em.pend_cost(s, a, m.params),
                      terminal_cost=lambda states, actions: em.pend_term(states, actions, m.params, 1))
    return m


def make(m, M, stepped=False, split=True):
    dyn = (lambda s, a: m.dynamics(s, a)) if stepped else m.dynamics
    c = eng.MPPI(dyn, m.running_cost, 2, torch.tensor(1.0), num_samples=K, horizon=T, U_init=torch.zeros(T, 1),
                 u_max=torch.tensor(2.0), terminal_state_cost=m.terminal_cost, rollout_samples=M, rollout_var_cost=0.5,
                 rollout_var_discount=0.9, device="cuda", rng_seed=1)
    c._split_cost = split
    c.refresh()
    assert (c._model is None) == stepped
    return c


def main():
    out = {}
    for M in (1, 2, 4, 8):
        m = model(M)
        fused = make(m, M)
        out[f"M{M}_fused_command_us"] = timing.back_to_back_us(lambda: fused.command(X0), 2000)
        out[f"M{M}_fused_command_l2_flushed_us"] = timing.median(timing.flushed_us(lambda: fused.command(X0), 200))
        out[f"M{M}_split_cost"] = int(fused.launch_info.split_cost)
        out[f"M{M}_regs"] = int(fused.launch_info.regs_per_thread)
        if M == 1:
            single = make(m, M, split=False)
            out["M1_single_loop_command_us"] = timing.back_to_back_us(lambda: single.command(X0), 2000)
            out["M1_single_loop_command_l2_flushed_us"] = timing.median(timing.flushed_us(lambda: single.command(X0), 200))
        stepped = make(m, M, stepped=True)
        out[f"M{M}_stepped_command_us"] = timing.back_to_back_us(lambda: stepped.command(X0), 50)
    out["config"] = f"K={K} T={T} fp32, pendulum ensemble with terminal cost, rollout_var_cost=0.5"
    timing.emit(out)


if __name__ == "__main__":
    main()
