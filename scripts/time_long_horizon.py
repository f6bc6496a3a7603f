"""Microseconds per command of the global-tile kernels (tile_memory="global") against the stepped route past the
shared-memory edge, and against the shared-memory kernels at a horizon where both plan.  (8,4) shape model, fp64,
K = 2048; windows of N back-to-back commands (the stepped route: 2 commands) after a warm-up, R windows per case with
the cases interleaved; prints min / median / max per case.  usage: time_long_horizon.py [N [R]]"""
import os
import sys

import numpy as np
import torch

import timing

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


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    x = torch.linspace(-0.5, 0.5, 8, dtype=torch.float64)
    cases = {}
    for v in ("mppi", "smppi", "kmppi"):
        Ts = 150 if v == "mppi" else 90          # within the shared-memory edge of each variant (185 / 97 / 99)
        cases[f"{v} T=512 fused global"] = (ctrl(v, 512, "fused", "global"), n)
        cases[f"{v} T=512 stepped global"] = (ctrl(v, 512, "stepped", "global"), 2)
        cases[f"{v} T={Ts} fused shared"] = (ctrl(v, Ts, "fused", "shared"), n)
        cases[f"{v} T={Ts} fused global"] = (ctrl(v, Ts, "fused", "global"), n)
    runs = timing.alternate_us({k: ((lambda c=c: c.command(x)), m) for k, (c, m) in cases.items()}, reps, warm=3)
    out = {"K": 2048, "shape": "(8,4) fp64", "commands_per_window": n, "windows": reps,
           "us_per_command": {k: {"min": min(r), "median": sorted(r)[len(r) // 2], "max": max(r)} for k, r in runs.items()}}
    timing.emit(out)


if __name__ == "__main__":
    main()
