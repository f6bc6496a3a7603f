"""A/B of the fused kernel's rollout variants — single loop (64 registers) and split-cost rollout (MPPI_B200_SPLIT_COST=1,
problems with helper threads) — back-to-back device time, L2-flushed per-command time (the bench's `value` protocol) and
the host round trip, pendulum fp32.
usage: ab_split.py [K T]...   (default: the north-star C2 size, two smaller ones and two mid-size ones)"""
import os
import sys

import torch

import timing

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402


VARIANTS = {"loop": "0", "split": "1"}     # name: MPPI_B200_SPLIT_COST


def make(K, T, variant):
    os.environ["MPPI_B200_SPLIT_COST"] = VARIANTS[variant]
    pend = eng.Pendulum()
    torch.manual_seed(0)
    U0 = torch.randn(T, 1) * 3.0
    return eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), num_samples=K, horizon=T, U_init=U0,
                    u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda", rng_seed=7)


def main():
    sizes = [(16384, 30), (4096, 30), (1024, 15), (32768, 30), (65536, 30)]
    if len(sys.argv) > 2:
        sizes = [(int(sys.argv[i]), int(sys.argv[i + 1])) for i in range(1, len(sys.argv) - 1, 2)]
    print(timing.card(), flush=True)
    xh = [3.14159, 1.0]
    x = torch.tensor(xh, dtype=torch.float32, device="cuda")
    for K, T in sizes:
        ctrls = {v: make(K, T, v) for v in VARIANTS}
        # same seed, same counter -> same draws: the kernels must agree to the bit
        acts = {}
        for _ in range(3):
            for v, c in ctrls.items():
                acts[v] = c.command(x)
        ref = ctrls["loop"]
        same = all(torch.equal(ref.U, c.U) and torch.equal(ref.cost_total, c.cost_total) and torch.equal(acts["loop"], acts[v])
                   for v, c in ctrls.items())
        for s, c in ctrls.items():
            t_b2b = timing.back_to_back_us(lambda: c.command(x), 500)
            ts = timing.flushed_us(lambda: c.command(x), 300)
            t_host = timing.host_us(lambda: c.command_host(xh), 2000, warm=50)
            li = c.launch_info
            print(f"K={K} T={T} {s:5s} split={li.split_cost} grid={li.grid_blocks} block={li.block_threads} tps={li.threads_per_sample} "
                  f"regs={li.regs_per_thread} smem={li.smem_bytes}: b2b {t_b2b:.2f} us | flushed mean {sum(ts) / len(ts):.2f} "
                  f"median {timing.median(ts):.2f} us | command_host {t_host:.2f} us | all variants bit-identical: {same}", flush=True)


if __name__ == "__main__":
    main()
