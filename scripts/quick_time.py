"""Quick A/B timing: back-to-back device time per command + host-side cost of one command() call.
usage: quick_time.py K T [bt] [tps]   (MPPI_B200_LIB selects a library variant)"""
import os
import sys

import torch

import timing

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402


def main():
    K, T = int(sys.argv[1]), int(sys.argv[2])
    bt = int(sys.argv[3]) if len(sys.argv) > 3 else 0
    tps = int(sys.argv[4]) if len(sys.argv) > 4 else 0
    print(timing.card())
    pend = eng.Pendulum()
    ctrl = eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), num_samples=K, horizon=T,
                    u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda", rng_seed=1, block_threads=bt, threads_per_sample=tps)
    x = [3.14159, 1.0]
    best = timing.back_to_back_us(lambda: ctrl.command(x), 500)
    # the issue rate of command() from an empty queue: the GPU soon saturates, so this is a wall time, not a call cost
    host = timing.host_us(lambda: ctrl.command(x), 2000, warm=0)
    torch.cuda.synchronize()
    e2e = timing.host_us(lambda: ctrl.command_host(x), 2000, warm=0)
    info = ctrl.launch_info
    print(f"{os.environ.get('MPPI_B200_LIB', 'default'):28s} K={K} T={T} grid={info.grid_blocks} block={info.block_threads} tps={info.threads_per_sample} regs={info.regs_per_thread}: "
          f"b2b {best:.2f} us/cmd; issue-rate-limited wall {host:.2f} us; command_host {e2e:.2f} us")


if __name__ == "__main__":
    main()
