"""Microseconds per control step of a closed-loop episode: `run_closed_loop(steps=1000)` (commands and plant steps
enqueued from C, chained with programmatic dependent launch) against back-to-back `command()` on a device state (no
plant) and the Python host loop it replaces (`u = command(x)`, `x = get_rollouts(x, U=u[None])[0, 0]`).  Shapes: the C2
pendulum (MPPI, K=16384, T=30, fp32) and MPPI_Batched N=16, K=4096, T=30 (fp32 pendulum).  Two episodes of warm-up, then
each timed over whole episodes (best of 3).  Prints one JSON line with the card name and power limit.

usage: python scripts/time_closed_loop.py [--steps 1000] [--trace DIR]   (--trace: a torch.profiler trace of a 50-step
episode of each shape, for launch gaps)"""
import argparse
import math
import os
import sys

import torch

import timing

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402


def c2():
    m = eng.Pendulum()
    return eng.MPPI(m.dynamics, m.running_cost, 2, torch.tensor(10.0), num_samples=16384, horizon=30, device="cuda",
                    u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), U_init=torch.zeros(30, 1), rng_seed=1)


def batched():
    m = eng.Pendulum()
    return eng.MPPI_Batched(m.dynamics, m.running_cost, 2, torch.tensor(10.0), 16, num_samples=4096, horizon=30,
                            device="cuda", u_max=torch.tensor(2.0), rng_seed=1)


def host_loop(c, x0, steps):
    """The Python loop; MPPI_Batched: one get_rollouts of the N states (get_rollouts replays one sequence for every
    start state, so this applies environment 0's action to all: the same calls and launches, not the same physics)"""
    x = x0
    for _ in range(steps):
        u = c.command(x)
        x = c.get_rollouts(x, num_rollouts=x.shape[0], U=u[:1])[:, 0] if x.dim() == 2 else c.get_rollouts(x, U=u[None])[0, 0]


def back_to_back(c, x0, steps):
    for _ in range(steps):
        c.command(x0)


def measure(name, make, x0, steps):
    c = make()
    # each a window of one episode of `steps` control steps, after two such episodes of warm-up; best of 3
    out = {k: timing.back_to_back_us(fn, 1, warm=2, reps=3) / steps
           for k, fn in (("closed_loop_us", lambda: c.run_closed_loop(x0, steps)),
                         ("command_b2b_us", lambda: back_to_back(c, x0, steps)),
                         ("host_loop_us", lambda: host_loop(c, x0, steps)))}
    # what the plant step adds to a control step over back-to-back commands
    out["closed_loop_minus_command_us"] = out["closed_loop_us"] - out["command_b2b_us"]
    info = c.launch_info
    out["route"] = {"split_cost": info.split_cost, "ll_tail": info.ll_tail, "cluster": info.cluster_size,
                    "grid": info.grid_blocks}
    return {name: {k: (round(v, 2) if isinstance(v, float) else v) for k, v in out.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--trace", default=None)
    args = ap.parse_args()
    out = {"steps": args.steps}
    x_c2 = torch.tensor([math.pi, 0.0], device="cuda")
    x_b = torch.tensor([[math.pi, 0.0]] * 16, device="cuda")
    out.update(measure("c2_pendulum_K16384_T30_f32", c2, x_c2, args.steps))
    out.update(measure("batched_N16_K4096_T30_f32", batched, x_b, args.steps))
    if args.trace:
        from torch.profiler import ProfilerActivity, profile
        os.makedirs(args.trace, exist_ok=True)
        for name, make, x0 in (("c2", c2, x_c2), ("batched", batched, x_b)):
            c = make()
            c.run_closed_loop(x0, 50)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                c.run_closed_loop(x0, 50)
                torch.cuda.synchronize()
            prof.export_chrome_trace(os.path.join(args.trace, f"closed_loop_{name}.json"))
            ev = sorted((e for e in prof.events() if e.device_type.name == "CUDA"), key=lambda e: e.time_range.start)
            gaps = [b.time_range.start - a.time_range.end for a, b in zip(ev, ev[1:])]
            plant = [e.time_range.elapsed_us() for e in ev if "plant_step" in e.name]
            out[f"trace_{name}"] = {"kernels": len(ev), "plant_kernel_us_median": sorted(plant)[len(plant) // 2] if plant else None,
                                    "gap_us_median": sorted(gaps)[len(gaps) // 2] if gaps else None}
    timing.emit(out)


if __name__ == "__main__":
    main()
