"""Microseconds per control step of closed-loop episodes against a plant named apart from the controller's model
(`run_closed_loop(steps, plant=...)`), over 1000-step episodes.

* C4 shape: PendulumMLP, K=32768, T=30, fp32, on the wgmma kernel, with a `Pendulum` plant — `run_closed_loop(plant=)`
  against back-to-back `command()` on a device state (no plant) and against the Python loop it replaces
  (`u = command(x)`, `x = P.get_rollouts(x, U=u[None])[0, 0]` with P a controller on the plant).
* C2 pendulum (MPPI, K=16384, T=30, fp32): `plant=Pendulum()` against `plant=None` (the same plant step).

The variants of each shape alternate within a repetition, an episode of warm-up before each (best of 5).  Prints
one JSON line with the card name and power limit.

usage: python scripts/time_closed_loop_plant.py [--steps 1000]"""
import argparse
import math
import os
import sys

import torch

import timing

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


def alternate(variants, steps, reps=5):
    """best us per step of each variant fn(n), which runs n control steps: episodes of `steps`, interleaved"""
    samples = timing.alternate_us({k: ((lambda fn=fn: fn(steps)), 1) for k, fn in variants.items()}, reps, warm=1)
    return {k: round(min(v) / steps, 2) for k, v in samples.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1000)
    args = ap.parse_args()
    out = {"steps": args.steps}
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
    timing.emit(out)


if __name__ == "__main__":
    main()
