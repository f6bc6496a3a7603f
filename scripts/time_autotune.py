"""Time of one CMA-ES generation of the tuner, and of the per-environment-horizon command it runs.

1. ms per generation of `BatchedAutotune` over sigma, lambda and horizon: 16 candidates + the incumbent, 4 start states
   (68 environments), 200-step closed loops of the pendulum, K = 4096, max horizon T = 30, fp32: one launch sequence per
   generation.
2. The same generation through the sequential `Autotune`, whose evaluate_fn runs one `run_closed_loop` (the 4 starts)
   per candidate, and once more for the best point, as the reference does.
3. µs per back-to-back `MPPI_Batched.command()` at N = 16, K = 4096, T = 30 with mixed horizons (5..30) against every
   environment at T (best of 5 windows per round), the two alternating within each round.

Prints one JSON line with the card name and power limit.
usage: python scripts/time_autotune.py [--generations 5] [--commands 1000] [--rounds 3]"""
import argparse
import math
import os
import sys

import torch

import timing

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402
from pytorch_mppi_b200 import autotune  # noqa: E402

K, T, S, STEPS, POP = 4096, 30, 4, 200, 16
START = [[math.pi, 0.0], [math.pi - 0.4, 0.0], [math.pi + 0.3, 0.5], [2.5, -0.5]]


def pendulum_ctrl():
    pend = eng.Pendulum()
    return eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(1.0), num_samples=K, horizon=20, lambda_=1.0,
                    u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda", rng_seed=3)


def params(ctrl):
    ps = [autotune.SigmaParameter(ctrl), autotune.LambdaParameter(ctrl), autotune.HorizonParameter(ctrl)]
    ps[2].max_horizon = T
    return ps


def batched_tuner():
    torch.manual_seed(0)
    ctrl = pendulum_ctrl()
    ev = autotune.ClosedLoopEvaluation(ctrl, torch.tensor(START, device="cuda"), STEPS, max_horizon=T)
    return autotune.BatchedAutotune(params(ctrl), ev, optimizer=autotune.CMAESOpt(POP, 1.0, seed=0))


def sequential_tuner():
    torch.manual_seed(0)
    ctrl = pendulum_ctrl()
    ev = autotune.ClosedLoopEvaluation(ctrl, torch.tensor(START, device="cuda"), STEPS, max_horizon=T)

    def evaluate():           # one run_closed_loop of the 4 starts with the controller's current settings
        settings = {"lambda_": torch.tensor([ctrl.lambda_], dtype=torch.float64),
                    "noise_sigma": ctrl.noise_sigma.reshape(1, 1, 1), "horizon": torch.tensor([ctrl.T], dtype=torch.int32)}
        costs, states = ev.evaluate(1, settings)
        return autotune.EvaluationResult(costs[0], states[:, 0].transpose(0, 1))
    return autotune.Autotune(params(ctrl), evaluate, optimizer=autotune.CMAESOpt(POP, 1.0, seed=0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--generations", type=int, default=5)
    ap.add_argument("--commands", type=int, default=1000)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    out = {"generation": {"candidates": POP, "starts": S, "steps": STEPS, "K": K, "max_horizon": T, "dtype": "float32"}}
    for name, make_tuner in (("batched", batched_tuner), ("sequential", sequential_tuner)):
        # one window of the generations after one warm-up generation (plans, module loads)
        us = timing.back_to_back_us(make_tuner().optimize_step, args.generations, warm=1, reps=1)
        out[f"{name}_ms_per_generation"] = round(us / 1e3, 1)

    N = 16
    pend = eng.Pendulum()
    make = lambda: eng.MPPI_Batched(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), N, num_samples=K, horizon=T,
                                    device="cuda", u_max=torch.tensor(2.0), rng_seed=1)
    uniform, mixed = make(), make()
    mixed.set_env_horizon(torch.linspace(5, T, N).round().to(torch.int32))
    x0 = torch.tensor([[math.pi, 0.0]] * N, device="cuda")
    res = timing.alternate_us({"uniform_T": (lambda: uniform.command(x0), args.commands),
                               "mixed_5_to_30": (lambda: mixed.command(x0), args.commands)}, args.rounds, reps=5)
    out["command_us_N16"] = {k: [round(v, 2) for v in x] for k, x in res.items()}
    timing.emit(out)


if __name__ == "__main__":
    main()
