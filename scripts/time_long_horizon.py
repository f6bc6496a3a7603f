"""Microseconds per command of the global-tile kernels (tile_memory="global") against the stepped route past the
shared-memory edge, and against the shared-memory kernels at a horizon where both plan.  (8,4) shape model, fp64,
K = 2048; CUDA events around N back-to-back commands after a warm-up (the stepped route: 2 commands), in R windows per
case with the cases interleaved; prints min / median / max per case.  usage: time_long_horizon.py [N [R]]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import pytorch_mppi_b200 as eng  # noqa: E402
from tests import shape_models as shm  # noqa: E402


def ctrl(variant, T, route, tm):
    nx, nu, dtype = 8, 4, torch.float64
    m = shm.shape_model(nx, nu)
    f, c, t = shm.twins(nx, nu)
    dyn, cost, term = (m.dynamics, m.running_cost, m.terminal_cost) if route == "fused" else (f, c, t)
    kw = {"smppi": dict(w_action_seq_cost=2.0, delta_t=0.5),
          "kmppi": dict(num_support_pts=T // 2, kernel=eng.RBFKernel(sigma=2.0))}.get(variant, {})
    cls = {"mppi": eng.MPPI, "smppi": eng.SMPPI, "kmppi": eng.KMPPI}[variant]
    sigma = torch.tensor(np.eye(nu) * 0.7 + 0.1, dtype=dtype)
    return cls(dyn, cost, nx, sigma, num_samples=2048, horizon=T, terminal_state_cost=term,
               u_max=torch.full((nu,), 1.2, dtype=dtype), device="cuda", rng_seed=1, tile_memory=tm, **kw)


def time_us(c, n):
    x = torch.linspace(-0.5, 0.5, 8, dtype=torch.float64)
    for _ in range(3):
        c.command(x)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        c.command(x)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1000.0 / n


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    cases = {}
    for v in ("mppi", "smppi", "kmppi"):
        Ts = 150 if v == "mppi" else 90          # within the shared-memory edge of each variant (185 / 97 / 99)
        cases[f"{v} T=512 fused global"] = (ctrl(v, 512, "fused", "global"), n)
        cases[f"{v} T=512 stepped global"] = (ctrl(v, 512, "stepped", "global"), 2)
        cases[f"{v} T={Ts} fused shared"] = (ctrl(v, Ts, "fused", "shared"), n)
        cases[f"{v} T={Ts} fused global"] = (ctrl(v, Ts, "fused", "global"), n)
    runs = {k: [] for k in cases}
    for _ in range(reps):                     # the cases interleaved, so that a slow phase of the host hits all of them
        for k, (c, m) in cases.items():
            runs[k].append(time_us(c, m))
    out = {"gpu": gpu, "K": 2048, "shape": "(8,4) fp64", "commands_per_window": n, "windows": reps,
           "us_per_command": {k: {"min": min(r), "median": sorted(r)[len(r) // 2], "max": max(r)} for k, r in runs.items()}}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
