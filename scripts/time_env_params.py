"""Microseconds per command of MPPI_Batched (N=16, K=4096, T=30, fp32; the closed-loop shape) with shared settings, with
per-environment noise only (lambda, Sigma, mu: set_env_params on the plan's own batched kernel) and with per-environment
noise plus model parameters (the batched kernel that reads one parameter block per environment), for the pendulum and
for LinearPoint.toy2d_nav() (without its terminal cost) with one goal per environment.  Each variant is timed back to back (best of 5 windows of
`--commands` commands, CUDA events) and with the L2 flushed before every command (a 100 MB write between commands, CUDA
events around the command alone, median), alternating the variants within one run; and per control step of
`run_closed_loop` (best of 3).  Prints one JSON line with the card name and power limit.

usage: python scripts/time_env_params.py [--commands 1000] [--steps 500]"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

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


def b2b(c, x0, n, reps=5):
    best = float("inf")
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        for _ in range(n):
            c.command(x0)
        b.record()
        torch.cuda.synchronize()
        best = min(best, a.elapsed_time(b) * 1e3 / n)
    return best


def cold(c, x0, n, flush):
    ts = []
    for _ in range(n):
        flush.fill_(1.0)                           # evicts the L2 (50 MB) between commands
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        c.command(x0)
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    return sorted(ts)[len(ts) // 2]


def closed(c, x0, steps, reps=3):
    best = float("inf")
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        c.run_closed_loop(x0, steps)
        b.record()
        torch.cuda.synchronize()
        best = min(best, a.elapsed_time(b) * 1e3 / steps)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--commands", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=500)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out = {"gpu": q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(),
           "shape": {"N": N, "K": K, "T": T, "dtype": "float32"}}
    flush = torch.empty(100 * 2 ** 20 // 4, device="cuda")
    variants = ("shared", "noise", "noise_and_model")
    for model in ("pendulum", "toy2d_nav"):
        ctrls = {v: make(model, v) for v in variants}
        for c, x0 in ctrls.values():           # warm-up: plans, module loads
            c.run_closed_loop(x0, 20)
            b2b(c, x0, 50, reps=1)
        res = {v: {"b2b_us": [], "cold_us": [], "closed_loop_us": []} for v in variants}
        for _ in range(args.rounds):           # the variants alternate within each round
            for v in variants:
                c, x0 = ctrls[v]
                res[v]["b2b_us"].append(b2b(c, x0, args.commands))
                res[v]["cold_us"].append(cold(c, x0, 200, flush))
                res[v]["closed_loop_us"].append(closed(c, x0, args.steps))
        out[model] = {v: {k: round(min(x), 2) for k, x in r.items()} for v, r in res.items()}
        out[model]["grid"] = ctrls["shared"][0].launch_info.grid_blocks
        out[model]["block_threads"] = ctrls["shared"][0].launch_info.block_threads
    print(json.dumps(out))


if __name__ == "__main__":
    main()
