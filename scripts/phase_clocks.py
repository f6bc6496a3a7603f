"""Phase timeline of the fused kernel from %globaltimer stamps (debug aid).
usage: phase_clocks.py K T [bt] [tps] [model] [variant]
  model   pendulum (default) | nav   (LinearPoint.toy2d_nav with terminal cost: BASELINE config 3's model)
  variant mppi (default) | smppi | kmppi
e.g. config 3:  phase_clocks.py 8192 40 0 0 nav kmppi        (MPPI_B200_SPLIT_COST=0/1 selects the rollout)"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402


def main():
    K, T = int(sys.argv[1]), int(sys.argv[2])
    bt = int(sys.argv[3]) if len(sys.argv) > 3 else 0
    tps = int(sys.argv[4]) if len(sys.argv) > 4 else 0
    model = sys.argv[5] if len(sys.argv) > 5 else "pendulum"
    variant = sys.argv[6] if len(sys.argv) > 6 else "mppi"
    geom = dict(block_threads=bt, threads_per_sample=tps)
    if model == "pendulum":
        pend = eng.Pendulum()
        ctrl = eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), num_samples=K, horizon=T,
                        u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda", rng_seed=1, **geom)
    else:
        nav = eng.LinearPoint.toy2d_nav(terminal_scale=10.0)
        kw = dict(num_samples=K, horizon=T, device="cuda", lambda_=1.0, terminal_state_cost=nav.terminal_cost,
                  u_max=torch.tensor([1.0, 1.0]), rng_seed=1, **geom)
        if variant == "mppi":
            ctrl = eng.MPPI(nav.dynamics, nav.running_cost, 2, torch.eye(2), **kw)
        elif variant == "smppi":
            ctrl = eng.SMPPI(nav.dynamics, nav.running_cost, 2, torch.eye(2), w_action_seq_cost=10.0, action_max=torch.tensor([1.0, 1.0]), **kw)
        else:
            ctrl = eng.KMPPI(nav.dynamics, nav.running_cost, 2, torch.eye(2), num_support_pts=5, kernel=eng.RBFKernel(sigma=2), **kw)
    x = [3.14159, 1.0] if model == "pendulum" else [-3.0, -2.0]
    for _ in range(5):
        ctrl.command(x)
    nb = ctrl.launch_info.grid_blocks
    dbg = torch.zeros(nb, 16, dtype=torch.int64, device="cuda")
    ctrl._debug_clocks = dbg
    ctrl._dirty = True
    names = ["start", "staged", "filled", "transformed", "rolled", "folded", "tail entered", "CTA exit", "L:published", "combined#1", "L:combined#2", "L:numer", "L:collected"]
    for rep in range(3):
        dbg.zero_()
        torch.cuda.synchronize()
        ctrl.command(x)
        torch.cuda.synchronize()
        d = dbg.cpu().numpy().astype(np.int64)
        t0 = d[:, 0].min()
        print(f"rep {rep}: {model}/{variant} K={K} T={T} grid={nb} block={ctrl.launch_info.block_threads} tps={ctrl.launch_info.threads_per_sample} split={ctrl.launch_info.split_cost}")
        for i, n in enumerate(names):
            col = d[:, i]
            col = col[col > 0]
            if len(col):
                print(f"  {n:12s} min {(col.min()-t0)/1e3:7.2f} us  median {(np.median(col)-t0)/1e3:7.2f}  max {(col.max()-t0)/1e3:7.2f}")


if __name__ == "__main__":
    main()
