"""Ensembles of learned pendulum networks (PendulumMLPEnsemble: M networks of BASELINE config 4's shape, one per rollout
copy) at K=32768, T=30, fp32, for rollout_samples M in {2, 4, 8}: time per command of the fused wgmma kernel (hi/lo-split
bf16 operands, the default) back to back (one synchronise at the end) and with L2 flushed before each command (CUDA events
around the command alone), of the fused FFMA kernel (tensor_cores=False) back to back, and of the stepped route (the same
torch twin in the reference's M-copy Python T-loop).  M = 1 is one PendulumMLP on the same two kernels.  Prints one JSON
line with the card name and power limit."""
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402
from tests.golden.cases import make_mlp_net  # noqa: E402

K, T = 32768, 30
X0 = [2.5, 0.5]


def model(M, tc):
    nets = [make_mlp_net(40 + m, torch.float32).cuda() for m in range(M)]
    return eng.PendulumMLP(nets[0], tensor_cores=tc) if M == 1 else eng.PendulumMLPEnsemble(nets, tensor_cores=tc)


def make(m, M, stepped=False):
    dyn = (lambda s, a: m.dynamics(s, a)) if stepped else m.dynamics
    c = eng.MPPI(dyn, m.running_cost, 2, torch.tensor(1.0), num_samples=K, horizon=T, U_init=torch.zeros(T, 1),
                 u_max=torch.tensor(2.0), rollout_samples=M, rollout_var_cost=0.5 if M > 1 else 0.0,
                 rollout_var_discount=0.9, device="cuda", rng_seed=1)
    assert (c._model is None) == stepped
    return c


def back_to_back_us(c, n):
    for _ in range(10):
        c.command(X0)
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(3):
        t0 = time.perf_counter()
        for _ in range(n):
            c.command(X0)
        torch.cuda.synchronize()
        best = min(best, (time.perf_counter() - t0) / n * 1e6)
    return best


def flushed_us(c, n, flush):
    for _ in range(5):
        c.command(X0)
    ts = []
    for _ in range(n):
        flush.zero_()                               # 256 MB: evicts the 50 MB L2
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        c.command(X0)
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def main():
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    out = {}
    for M in (1, 2, 4, 8):
        wg = make(model(M, "bf16x3"), M)
        out[f"M{M}_wgmma_command_us"] = back_to_back_us(wg, 500)
        out[f"M{M}_wgmma_command_l2_flushed_us"] = flushed_us(wg, 100, flush)
        out[f"M{M}_wgmma_regs"] = int(wg.launch_info.regs_per_thread)
        out[f"M{M}_wgmma_smem_bytes"] = int(wg.launch_info.smem_bytes)
        out[f"M{M}_wgmma_ctas_per_sm"] = int(wg.launch_info.max_blocks_per_sm)
        ff = make(model(M, False), M)
        out[f"M{M}_ffma_command_us"] = back_to_back_us(ff, 200)
        out[f"M{M}_ffma_regs"] = int(ff.launch_info.regs_per_thread)
        if M > 1:
            out[f"M{M}_stepped_command_us"] = back_to_back_us(make(model(M, False), M, stepped=True), 10)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out["gpu"] = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()
    out["config"] = f"K={K} T={T} fp32, MPPI, rollout_var_cost=0.5, networks of pendulum_approximate.py's shape"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
