"""BASELINE config 4 (learned pendulum dynamics: a 3-32-32-2 tanh MLP, T=30, fp32): device time per command, back to
back, of every route at each K — the FFMA kernel (tensor_cores=False) and the wgmma kernel with hi/lo-split (bf16x3,
what the default tensor_cores="auto" runs) and plain bf16 operands, each with exact and MUFU tanh; the stepped route
(the torch MLP in a Python T-loop), and the same under compile() (CUDA graph replay).  The FFMA / wgmma rows over K
show where the tensor cores pay off.
usage: time_c4.py [--K 1024 2048 ...]"""
import argparse
import os
import sys

import torch

import timing

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402

T = 30
X = [3.0, 0.5]


def run(name, K, dyn, cost, n, compile=False):
    c = eng.MPPI(dyn, cost, 2, torch.tensor(1.0), num_samples=K, horizon=T, u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0),
                 device="cuda", rng_seed=1)
    if compile:
        c.compile()
    us = timing.back_to_back_us(lambda: c.command(X), n)
    row = f"K={K} {name}: {us:.1f} us/command -> {K*T/us/1e3:.2f} G rollout-steps/s, {2368*K*T/us/1e6:.2f} TFLOP/s of MLP math"
    if c._model is not None:
        i = c.launch_info
        row += (f" grid={i.grid_blocks} block={i.block_threads} regs={i.regs_per_thread} smem={i.smem_bytes} "
                f"occ={i.max_blocks_per_sm} tps={i.threads_per_sample} cost_mean={float(c.cost_total.mean()):.4f}")
    print(row, flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--K", type=int, nargs="+", default=[1024, 2048, 4096, 8192, 16384, 32768, 65536, 131072])
    args = ap.parse_args()
    print(timing.card(), flush=True)
    torch.manual_seed(25)
    net = torch.nn.Sequential(torch.nn.Linear(3, 32), torch.nn.Tanh(), torch.nn.Linear(32, 32), torch.nn.Tanh(),
                              torch.nn.Linear(32, 2)).cuda()
    for K in args.K:
        for mode, route in ((False, "fp32 FFMA"), ("bf16x3", "wgmma bf16x3"), ("bf16", "wgmma bf16")):
            for fast in (False, True):
                m = eng.PendulumMLP(net, fast_tanh=fast, tensor_cores=mode)
                run(f"fused   {route} fast_tanh={fast}", K, m.dynamics, m.running_cost, 50)
        m = eng.PendulumMLP(net)
        stepped = (lambda s, a: m.dynamics(s, a)), (lambda s, a: m.running_cost(s, a))
        run("stepped fp32 (torch MLP, Python T-loop)", K, *stepped, 10)
        run("stepped fp32 + compile() (CUDA graph replay)", K, *stepped, 20, compile=True)


if __name__ == "__main__":
    main()
