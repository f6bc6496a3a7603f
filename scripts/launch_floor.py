"""Launch+sync latency floor on this box: trivial kernel vs tiny fused command (PDL on/off)."""
import os
import sys

import torch

import timing

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402
from pytorch_mppi_b200 import _cabi  # noqa: E402


def main():
    print(timing.card())
    lib = _cabi.load()
    a = torch.zeros(32, device="cuda")
    b = torch.ones(32, device="cuda")
    n = 3000
    s = torch.cuda.current_stream().cuda_stream

    def triv():
        lib.mppi_cost_accumulate(a.data_ptr(), b.data_ptr(), None, 1, 32, 1.0, 0, s)
        torch.cuda.synchronize()
    print(f"trivial kernel (ctypes) + synchronize: {timing.host_us(triv, n, warm=300):.2f} us")
    print(f"torch add_ + synchronize: {timing.host_us(lambda: (a.add_(1), torch.cuda.synchronize()), n, warm=300):.2f} us")
    print(f"synchronize only: {timing.host_us(torch.cuda.synchronize, n, warm=300):.2f} us")
    pend = eng.Pendulum()
    for pdl in ("1", "0"):
        os.environ["MPPI_B200_PDL"] = pdl
        c = eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), num_samples=32, horizon=2,
                     u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda", rng_seed=1)
        x = [3.0, 1.0]
        sync = timing.host_us(lambda: (c.command(x), torch.cuda.synchronize()), n, warm=300)
        print(f"tiny fused PDL={pdl}: command+sync {sync:.2f} us; command_host {timing.host_us(lambda: c.command_host(x), n, warm=300):.2f} us")
        print(f"   tiny fused b2b device: {timing.back_to_back_us(lambda: c.command(x), 1000):.2f} us per command")


if __name__ == "__main__":
    main()
