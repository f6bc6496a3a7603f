"""BASELINE config 3 (2-D navigation, KMPPI, RBF(sigma=2), 5 support points, K=8192, T=40, fp32; SURVEY 8d /
reference tests/smooth_mppi.py:539-560): device time per command for the three controllers on the same model,
fused route (both rollouts) and stepped route.  Not under ncu."""
import os
import sys

import torch

import timing

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402

K, T, S = 8192, 40, 5


def make(nav, kind, split, stepped=False):
    os.environ["MPPI_B200_SPLIT_COST"] = "1" if split else "0"
    dyn, cost, term = nav.dynamics, nav.running_cost, nav.terminal_cost
    if stepped:
        dyn, cost, term = (lambda s, a: nav.dynamics(s, a)), (lambda s, a: nav.running_cost(s, a)), (lambda s, a: nav.terminal_cost(s, a))
    kw = dict(num_samples=K, horizon=T, device="cuda", lambda_=1.0, terminal_state_cost=term, u_max=torch.tensor([1.0, 1.0]), rng_seed=1)
    if kind == "mppi":
        return eng.MPPI(dyn, cost, 2, torch.eye(2), **kw)
    if kind == "smppi":
        return eng.SMPPI(dyn, cost, 2, torch.eye(2), w_action_seq_cost=10.0, action_max=torch.tensor([1.0, 1.0]), **kw)
    return eng.KMPPI(dyn, cost, 2, torch.eye(2), num_support_pts=S, kernel=eng.RBFKernel(sigma=2), **kw)


def main():
    print(timing.card(), flush=True)
    nav = eng.LinearPoint.toy2d_nav(terminal_scale=10.0)
    x0 = torch.tensor([-3.0, -2.0], device="cuda")
    for kind in ("kmppi", "mppi", "smppi"):
        for split in (0, 1):
            c = make(nav, kind, split)
            t_us = timing.back_to_back_us(lambda: c.command(x0), 500)
            li = c.launch_info   # set when the first command packs the launch parameters
            print(f"{kind:5s} fused split={li.split_cost} grid={li.grid_blocks} block={li.block_threads} tps={li.threads_per_sample} "
                  f"regs={li.regs_per_thread} smem={li.smem_bytes}: {t_us:.2f} us/command back to back", flush=True)
        c = make(nav, kind, 0, stepped=True)
        print(f"{kind:5s} stepped (Python T-loop + kernels): {timing.back_to_back_us(lambda: c.command(x0), 20):.1f} us/command", flush=True)
        c.compile()
        print(f"{kind:5s} stepped + compile() (CUDA graph): {timing.back_to_back_us(lambda: c.command(x0), 50):.1f} us/command", flush=True)


if __name__ == "__main__":
    main()
