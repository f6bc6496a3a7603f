"""Ensembles of learned pendulum networks (PendulumMLPEnsemble: M networks of BASELINE config 4's shape, one per rollout
copy) at K=32768, T=30, fp32, for rollout_samples M in {2, 4, 8}: time per command of the fused wgmma kernel (hi/lo-split
bf16 operands, the default) back to back and with L2 flushed before each command, of the fused FFMA kernel
(tensor_cores=False) back to back, and of the stepped route (the same torch twin in the reference's M-copy Python
T-loop).  M = 1 is one PendulumMLP on the same two kernels.  Prints one JSON
line with the card name and power limit."""
import os
import sys

import torch

import timing

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


def main():
    out = {}
    for M in (1, 2, 4, 8):
        wg = make(model(M, "bf16x3"), M)
        out[f"M{M}_wgmma_command_us"] = timing.back_to_back_us(lambda: wg.command(X0), 500)
        out[f"M{M}_wgmma_command_l2_flushed_us"] = timing.median(timing.flushed_us(lambda: wg.command(X0), 100))
        out[f"M{M}_wgmma_regs"] = int(wg.launch_info.regs_per_thread)
        out[f"M{M}_wgmma_smem_bytes"] = int(wg.launch_info.smem_bytes)
        out[f"M{M}_wgmma_ctas_per_sm"] = int(wg.launch_info.max_blocks_per_sm)
        ff = make(model(M, False), M)
        out[f"M{M}_ffma_command_us"] = timing.back_to_back_us(lambda: ff.command(X0), 200)
        out[f"M{M}_ffma_regs"] = int(ff.launch_info.regs_per_thread)
        if M > 1:
            stepped = make(model(M, False), M, stepped=True)
            out[f"M{M}_stepped_command_us"] = timing.back_to_back_us(lambda: stepped.command(X0), 10)
    out["config"] = f"K={K} T={T} fp32, MPPI, rollout_var_cost=0.5, networks of pendulum_approximate.py's shape"
    timing.emit(out)


if __name__ == "__main__":
    main()
