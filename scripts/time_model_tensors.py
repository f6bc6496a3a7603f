"""The C3 shape (2-D navigation, KMPPI S=5, K=8192, T=40, fp32) with a user model whose cost reads a 256 x 256 fp32
costmap with bilinear interpolation and a reference path by t (tests/tensor_models.py), against
`LinearPoint.toy2d_nav()` (analytic hills) on the same controller shape.  Times per command: the fused `command()` back
to back and with the L2 flushed before each command, and the tensor model on the stepped route (its torch twins in a
Python T-loop).  Prints one JSON line with the card name and power limit, and the registers per thread of each fused
kernel."""
import os
import sys

import torch

import timing

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402
from tests import tensor_models as tm  # noqa: E402

K, T, S = 8192, 40, 5
X0 = [-1.2, -0.9]


def make(dyn, cost, term=None, sd=True):
    c = eng.KMPPI(dyn, cost, 2, torch.eye(2), num_samples=K, horizon=T, U_init=torch.zeros(T, 2), u_max=torch.full((2,), 3.0),
                  terminal_state_cost=term, step_dependent_dynamics=sd, num_support_pts=S, kernel=eng.RBFKernel(sigma=2.0),
                  device="cuda", rng_seed=1)
    return c


def main():
    m = tm.nav_model(tm.make_costmap(hw=(256, 256)), tm.make_path(T))
    fused = make(m.dynamics, m.running_cost)
    stepped = make(lambda s, a, t: m.dynamics(s, a, t), lambda s, a, t: m.running_cost(s, a, t))
    hills = eng.LinearPoint.toy2d_nav()
    ref = make(hills.dynamics, hills.running_cost, hills.terminal_cost, sd=False)
    assert fused._model is m and stepped._model is None and ref._model is hills
    out = {
        "tensor_fused_command_us": timing.back_to_back_us(lambda: fused.command(X0), 2000),
        "tensor_fused_command_l2_flushed_us": timing.median(timing.flushed_us(lambda: fused.command(X0), 500)),
        "tensor_stepped_command_us": timing.back_to_back_us(lambda: stepped.command(X0), 50),
        "toy2d_nav_fused_command_us": timing.back_to_back_us(lambda: ref.command(X0), 2000),
        "toy2d_nav_fused_command_l2_flushed_us": timing.median(timing.flushed_us(lambda: ref.command(X0), 500)),
        "regs_per_thread": {"tensor": int(fused.launch_info.regs_per_thread), "toy2d_nav": int(ref.launch_info.regs_per_thread)},
        "split_cost": {"tensor": int(fused.launch_info.split_cost), "toy2d_nav": int(ref.launch_info.split_cost)},
    }
    out["config"] = f"KMPPI S={S} K={K} T={T} fp32; costmap 256x256 fp32 bilinear + (T,2) fp64 path"
    timing.emit(out)


if __name__ == "__main__":
    main()
