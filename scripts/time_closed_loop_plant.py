"""Microseconds per control step of closed-loop episodes against a plant named apart from the controller's model
(`run_closed_loop(steps, plant=...)`), over 1000-step episodes.

* C4 shape: PendulumMLP, K=32768, T=30, fp32, on the wgmma kernel, with a `Pendulum` plant — `run_closed_loop(plant=)`
  against back-to-back `command()` on a device state (no plant) and against the Python loop it replaces
  (`u = command(x)`, `x = P.get_rollouts(x, U=u[None])[0, 0]` with P a controller on the plant).
* C2 pendulum (MPPI, K=16384, T=30, fp32): `plant=Pendulum()` against `plant=None` (the same plant step).

Warm-up first; the variants of each shape alternate within a repetition, CUDA events around each (best of 5).  Prints
one JSON line with the card name and power limit.

usage: python scripts/time_closed_loop_plant.py [--steps 1000]"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402


def c4():
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(3, 32), torch.nn.Tanh(), torch.nn.Linear(32, 32), torch.nn.Tanh(),
                              torch.nn.Linear(32, 2))
    m = eng.PendulumMLP(net)
    return eng.MPPI(m.dynamics, m.running_cost, 2, torch.tensor(1.0), num_samples=32768, horizon=30, device="cuda",
                    u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), U_init=torch.zeros(30, 1), rng_seed=1)


def c2():
    m = eng.Pendulum()
    return eng.MPPI(m.dynamics, m.running_cost, 2, torch.tensor(10.0), num_samples=16384, horizon=30, device="cuda",
                    u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), U_init=torch.zeros(30, 1), rng_seed=1)


def time_once(fn, steps):
    """us per step of fn() (which runs `steps` control steps), CUDA events around it"""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / steps


def alternate(variants, steps, reps=5):
    """best us per step of each variant, the variants interleaved within every repetition"""
    for fn in variants.values():                      # warm-up: plans, module loads, caches
        fn(50)
        fn(50)
    best = {k: float("inf") for k in variants}
    for _ in range(reps):
        for k, fn in variants.items():
            best[k] = min(best[k], time_once(lambda: fn(steps), steps))
    return {k: round(v, 2) for k, v in best.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1000)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out = {"gpu": q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(),
           "steps": args.steps}
    plant = eng.Pendulum()
    pc = eng.MPPI(plant.dynamics, plant.running_cost, 2, torch.tensor(1.0), num_samples=64, horizon=5, device="cuda")

    x4 = torch.tensor([math.pi, 1.0], device="cuda")
    c = c4()

    def host_loop(n):
        x = x4
        for _ in range(n):
            u = c.command(x)
            x = pc.get_rollouts(x, U=u[None])[0, 0]

    def back_to_back(n):
        for _ in range(n):
            c.command(x4)

    t = alternate({"closed_loop_plant_us": lambda n: c.run_closed_loop(x4, n, plant=plant),
                   "command_b2b_us": back_to_back, "host_loop_us": host_loop}, args.steps)
    t["closed_loop_minus_command_us"] = round(t["closed_loop_plant_us"] - t["command_b2b_us"], 2)
    c.command(x4)
    t["route"] = {"block_threads": c.launch_info.block_threads, "threads_per_sample": c.launch_info.threads_per_sample}
    out["c4_mlp_wgmma_K32768_T30_f32_pendulum_plant"] = t

    x2 = torch.tensor([math.pi, 0.0], device="cuda")
    d = c2()
    out["c2_pendulum_K16384_T30_f32"] = alternate({"plant_pendulum_us": lambda n: d.run_closed_loop(x2, n, plant=plant),
                                                   "plant_none_us": lambda n: d.run_closed_loop(x2, n)}, args.steps)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
