"""Geometry sweep: b2b device time per command for (K, T) x (block_threads, threads_per_sample)."""
import os
import sys

import torch

import timing

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402


def main():
    print(timing.card(), flush=True)
    pend = eng.Pendulum()
    x = [3.14159, 1.0]
    for K, T in ((16384, 30), (32768, 30), (65536, 30), (131072, 50), (262144, 50), (1 << 20, 50)):
        res = []
        for bt in (64, 128, 192, 256, 320, 384, 448, 512):
            for tps in (1, 2, 4):
                if bt * tps > 512:
                    continue
                try:
                    c = eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), num_samples=K, horizon=T,
                                 u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda", rng_seed=1, block_threads=bt, threads_per_sample=tps)
                    best = timing.back_to_back_us(lambda: c.command(x), 100 if K <= 131072 else 30)
                    i = c.launch_info
                    res.append((best, bt, tps, i.grid_blocks, i.max_blocks_per_sm))
                    del c
                except Exception as e:
                    res.append((1e9, bt, tps, -1, str(e)[:40]))
        res.sort()
        print(f"K={K} T={T}: " + " | ".join(f"{t:.1f}us bs={bt} tps={tps} g={g} occ={o}" for t, bt, tps, g, o in res[:6]), flush=True)
        print("      worst: " + " | ".join(f"{t:.1f}us bs={bt} tps={tps} g={g}" for t, bt, tps, g, o in res[-3:]), flush=True)


if __name__ == "__main__":
    main()
