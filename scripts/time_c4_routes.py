"""Learned-dynamics rollout (BASELINE config 4 network), fp32: FFMA kernel vs wgmma kernel over K — picks the
crossover of the automatic route (PendulumMLP(tensor_cores="auto")).  Device time per command, back to back."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402

torch.manual_seed(25)
net = torch.nn.Sequential(torch.nn.Linear(3, 32), torch.nn.Tanh(), torch.nn.Linear(32, 32), torch.nn.Tanh(), torch.nn.Linear(32, 2)).cuda()
T = 30


def run(K, mode):
    m = eng.PendulumMLP(net, tensor_cores=mode)
    c = eng.MPPI(m.dynamics, m.running_cost, 2, torch.tensor(1.0), num_samples=K, horizon=T, u_min=torch.tensor(-2.0),
                 u_max=torch.tensor(2.0), device="cuda", rng_seed=1)
    x = [3.0, 0.5]
    for _ in range(5):
        c.command(x)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 100
    e0.record()
    for _ in range(n):
        c.command(x)
    e1.record()
    torch.cuda.synchronize()
    info = c.launch_info
    return e0.elapsed_time(e1) / n * 1e3, info.grid_blocks, info.block_threads


for K in (1024, 2048, 4096, 8192, 16384, 32768, 65536, 131072):
    row = [f"K={K:6d}"]
    for mode in (False, "bf16x3", "bf16"):
        us, g, b = run(K, mode)
        row.append(f"{str(mode):6s} {us:7.1f} us (grid {g} x {b})")
    print("  ".join(row))
