"""Ensemble controllers (tests/ensemble_models.py: pendulum with a mass and length per copy, terminal cost) at K=16384,
T=30, fp32, for rollout_samples M in {1, 2, 4, 8}: time per command of the fused `command()` back to back (one
synchronise at the end), of the fused `command()` with L2 flushed before each command (CUDA events around the command
alone), and of the stepped route (the same torch twins in the reference's M-copy Python T-loop).  M = 1 is the same
pendulum compiled without copies, on the single-loop kernel (the one copies use) and on the split-cost kernel (the
default for one copy at this size).  Prints one JSON line with the card name and power limit."""
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402
from tests import ensemble_models as em  # noqa: E402

K, T = 16384, 30
X0 = [2.5, 0.5]


def model(M):
    if M > 1:
        return em.pendulum_ensemble(M, K)
    one = "const int m = 0, COPIES = 1; (void)m; (void)COPIES;\n"      # the same bodies for a model without copies
    m = eng.CudaModel(2, 1, one + em.PEND_STEP, em.PEND_COST, params=em.pendulum_params(1), terminal_code=one + em.PEND_TERM,
                      dynamics=lambda s, a: em.pend_dyn(s, a, m.params, 1, K),
                      running_cost=lambda s, a: em.pend_cost(s, a, m.params),
                      terminal_cost=lambda states, actions: em.pend_term(states, actions, m.params, 1))
    return m


def make(m, M, stepped=False, split=True):
    dyn = (lambda s, a: m.dynamics(s, a)) if stepped else m.dynamics
    c = eng.MPPI(dyn, m.running_cost, 2, torch.tensor(1.0), num_samples=K, horizon=T, U_init=torch.zeros(T, 1),
                 u_max=torch.tensor(2.0), terminal_state_cost=m.terminal_cost, rollout_samples=M, rollout_var_cost=0.5,
                 rollout_var_discount=0.9, device="cuda", rng_seed=1)
    c._split_cost = split
    c.refresh()
    assert (c._model is None) == stepped
    return c


def back_to_back_us(c, n):
    for _ in range(20):
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
        m = model(M)
        fused = make(m, M)
        out[f"M{M}_fused_command_us"] = back_to_back_us(fused, 2000)
        out[f"M{M}_fused_command_l2_flushed_us"] = flushed_us(fused, 200, flush)
        out[f"M{M}_split_cost"] = int(fused.launch_info.split_cost)
        out[f"M{M}_regs"] = int(fused.launch_info.regs_per_thread)
        if M == 1:
            single = make(m, M, split=False)
            out["M1_single_loop_command_us"] = back_to_back_us(single, 2000)
            out["M1_single_loop_command_l2_flushed_us"] = flushed_us(single, 200, flush)
        out[f"M{M}_stepped_command_us"] = back_to_back_us(make(m, M, stepped=True), 50)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out["gpu"] = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()
    out["config"] = f"K={K} T={T} fp32, pendulum ensemble with terminal cost, rollout_var_cost=0.5"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
