"""Fixed overhead of the host round trip: command_host on a tiny problem vs the north-star one."""
import os
import sys

import torch

import timing

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402


def main():
    print(timing.card())
    pend = eng.Pendulum()
    n = 3000
    for K, T in ((32, 2), (1024, 5), (16384, 30)):
        c = eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), num_samples=K, horizon=T,
                     u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda", rng_seed=1)
        x = [3.14159, 1.0]
        e2e = timing.host_us(lambda: c.command_host(x), n, warm=300)
        # pieces: python-only cost (no launch) approximated by timing the pre/post code paths
        pre = timing.host_us(lambda: (c._host_state(x), c._noise_source(), torch._C._cuda_getCurrentRawStream(0)), n)
        post = timing.host_us(lambda: torch.empty_like(c._host_template).data_ptr(), n)
        # device-side: launch + sync round trip without mailbox
        sync = timing.host_us(lambda: (c.command(x), torch.cuda.synchronize()), n)
        print(f"K={K} T={T}: command_host {e2e:.2f} us | python pre {pre:.2f} post {post:.2f} | command()+synchronize {sync:.2f} us")


if __name__ == "__main__":
    main()
