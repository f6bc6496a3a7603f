"""Tiny driver for ncu: N commands of the pendulum fused kernel.  usage: prof_cmd.py K T [n] [bt]"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402


def main():
    K, T = int(sys.argv[1]), int(sys.argv[2])
    n = int(sys.argv[3]) if len(sys.argv) > 3 else 10
    bt = int(sys.argv[4]) if len(sys.argv) > 4 else 0
    pend = eng.Pendulum()
    ctrl = eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), num_samples=K, horizon=T,
                    u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda", rng_seed=1, block_threads=bt)
    x = [3.14159, 1.0]
    for _ in range(n):
        a = ctrl.command(x)
    torch.cuda.synchronize()
    print("done", a)


if __name__ == "__main__":
    main()
