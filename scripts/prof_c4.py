"""Tiny driver for ncu: n commands of the learned-dynamics (MLP) fused kernel.
usage: prof_c4.py K T mode(off|bf16x3|bf16) fast(0|1) [n]"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402


def main():
    K, T = int(sys.argv[1]), int(sys.argv[2])
    mode = {"off": False}.get(sys.argv[3], sys.argv[3])
    fast = bool(int(sys.argv[4]))
    n = int(sys.argv[5]) if len(sys.argv) > 5 else 4
    torch.manual_seed(25)
    net = torch.nn.Sequential(torch.nn.Linear(3, 32), torch.nn.Tanh(), torch.nn.Linear(32, 32), torch.nn.Tanh(), torch.nn.Linear(32, 2)).cuda()
    m = eng.PendulumMLP(net, fast_tanh=fast, tensor_cores=mode)
    c = eng.MPPI(m.dynamics, m.running_cost, 2, torch.tensor(1.0), num_samples=K, horizon=T, u_min=torch.tensor(-2.0),
                 u_max=torch.tensor(2.0), device="cuda", rng_seed=1)
    x = [3.0, 0.5]
    for _ in range(n):
        a = c.command(x)
    torch.cuda.synchronize()
    print("done", a)


if __name__ == "__main__":
    main()
