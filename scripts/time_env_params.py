"""Microseconds per command of MPPI_Batched (N=16, K=4096, T=30, fp32; the closed-loop shape) with shared settings, with
per-environment noise only (lambda, Sigma, mu: set_env_params on the plan's own batched kernel) and with per-environment
noise plus model parameters (the batched kernel that reads one parameter block per environment), for the pendulum and
for LinearPoint.toy2d_nav() (without its terminal cost) with one goal per environment.  Each variant is timed back to
back (best of 5 windows of `--commands` commands), with the L2 flushed before every command (median of 200) and per
control step of `run_closed_loop` (best of 3 episodes of `--steps`), the variants alternating within each of `--rounds`
rounds.  Prints one JSON line with the card name and power limit.

usage: python scripts/time_env_params.py [--commands 1000] [--steps 500]"""
import argparse
import math
import os
import sys

import torch

import timing

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402

N, K, T = 16, 4096, 30


def make(model, variant):
    m = eng.Pendulum() if model == "pendulum" else eng.LinearPoint.toy2d_nav(terminal_scale=0.0)
    nu = 1 if model == "pendulum" else 2
    sigma = torch.tensor(10.0) if nu == 1 else torch.eye(2)
    c = eng.MPPI_Batched(m.dynamics, m.running_cost, 2, sigma, N, num_samples=K, horizon=T, device="cuda",
                         u_max=torch.full((nu,), 2.0), rng_seed=1)
    if variant != "shared":
        lams = torch.linspace(0.5, 2.0, N, dtype=torch.float64)
        sig = (sigma.reshape(nu, nu) * torch.linspace(0.5, 1.5, N).view(N, 1, 1)).contiguous()
        kw = dict(lambda_=lams, noise_sigma=sig, noise_mu=torch.zeros(N, nu))
        if variant == "noise_and_model":
            if model == "pendulum":
                rows = [eng.Pendulum(m=1.0 + 0.05 * e).param_blob() for e in range(N)]
            else:
                rows = []
                for e in range(N):
                    g = eng.LinearPoint.toy2d_nav(terminal_scale=0.0)
                    g.goal = [2.0 - 0.2 * e, 2.0 - 0.1 * e]
                    rows.append(g.param_blob())
            kw["model_params"] = rows
        c.set_env_params(**kw)
    x0 = torch.tensor([[math.pi, 0.0]] * N if nu == 1 else [[-3.0, -2.0]] * N, device="cuda")
    return c, x0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--commands", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=500)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    out = {"shape": {"N": N, "K": K, "T": T, "dtype": "float32"}}
    variants = ("shared", "noise", "noise_and_model")
    for model in ("pendulum", "toy2d_nav"):
        ctrls = {v: make(model, v) for v in variants}
        for c, x0 in ctrls.values():           # warm-up: plans, module loads
            c.run_closed_loop(x0, 20)
            for _ in range(50):
                c.command(x0)
        res = {v: {"b2b_us": [], "cold_us": [], "closed_loop_us": []} for v in variants}
        for _ in range(args.rounds):           # the variants alternate within each round
            for v in variants:
                c, x0 = ctrls[v]
                res[v]["b2b_us"].append(timing.back_to_back_us(lambda: c.command(x0), args.commands, warm=0))
                res[v]["cold_us"].append(timing.median(timing.flushed_us(lambda: c.command(x0), 200, warm=0)))
                closed = timing.back_to_back_us(lambda: c.run_closed_loop(x0, args.steps), 1, warm=0, reps=3)
                res[v]["closed_loop_us"].append(closed / args.steps)
        out[model] = {v: {k: round(min(x), 2) for k, x in r.items()} for v, r in res.items()}
        out[model]["grid"] = ctrls["shared"][0].launch_info.grid_blocks
        out[model]["block_threads"] = ctrls["shared"][0].launch_info.block_threads
    timing.emit(out)


if __name__ == "__main__":
    main()
