"""The C3 shape (2-D navigation, KMPPI S=5, K=8192, T=40, fp32) with a user model whose cost reads a 256 x 256 fp32
costmap with bilinear interpolation and a reference path by t (tests/tensor_models.py), against
`LinearPoint.toy2d_nav()` (analytic hills) on the same controller shape.  Times per command: the fused `command()` back
to back (one synchronise at the end) and L2-flushed (a 256 MB write before each command, CUDA events around the command
alone), and the tensor model on the stepped route (its torch twins in a Python T-loop).  Prints one JSON line with the
card name and power limit, and the registers per thread of each fused kernel."""
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402
from tests import tensor_models as tm  # noqa: E402

K, T, S = 8192, 40, 5


def make(dyn, cost, term=None, sd=True):
    c = eng.KMPPI(dyn, cost, 2, torch.eye(2), num_samples=K, horizon=T, U_init=torch.zeros(T, 2), u_max=torch.full((2,), 3.0),
                  terminal_state_cost=term, step_dependent_dynamics=sd, num_support_pts=S, kernel=eng.RBFKernel(sigma=2.0),
                  device="cuda", rng_seed=1)
    return c


def back_to_back_us(c, n):
    x = [-1.2, -0.9]
    for _ in range(20):
        c.command(x)
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(3):
        t0 = time.perf_counter()
        for _ in range(n):
            c.command(x)
        torch.cuda.synchronize()
        best = min(best, (time.perf_counter() - t0) / n * 1e6)
    return best


def flushed_us(c, n):
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device="cuda")
    x = [-1.2, -0.9]
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n)]
    for _ in range(10):
        c.command(x)
    for a, b in ev:
        flush.zero_()
        a.record()
        c.command(x)
        b.record()
    torch.cuda.synchronize()
    ts = sorted(a.elapsed_time(b) * 1e3 for a, b in ev)
    return ts[len(ts) // 2]


def main():
    m = tm.nav_model(tm.make_costmap(hw=(256, 256)), tm.make_path(T))
    fused = make(m.dynamics, m.running_cost)
    stepped = make(lambda s, a, t: m.dynamics(s, a, t), lambda s, a, t: m.running_cost(s, a, t))
    hills = eng.LinearPoint.toy2d_nav()
    ref = make(hills.dynamics, hills.running_cost, hills.terminal_cost, sd=False)
    assert fused._model is m and stepped._model is None and ref._model is hills
    out = {
        "tensor_fused_command_us": back_to_back_us(fused, 2000),
        "tensor_fused_command_l2_flushed_us": flushed_us(fused, 500),
        "tensor_stepped_command_us": back_to_back_us(stepped, 50),
        "toy2d_nav_fused_command_us": back_to_back_us(ref, 2000),
        "toy2d_nav_fused_command_l2_flushed_us": flushed_us(ref, 500),
        "regs_per_thread": {"tensor": int(fused.launch_info.regs_per_thread), "toy2d_nav": int(ref.launch_info.regs_per_thread)},
        "split_cost": {"tensor": int(fused.launch_info.split_cost), "toy2d_nav": int(ref.launch_info.split_cost)},
    }
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out["gpu"] = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()
    out["config"] = f"KMPPI S={S} K={K} T={T} fp32; costmap 256x256 fp32 bilinear + (T,2) fp64 path"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
