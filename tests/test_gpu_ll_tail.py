"""GPU: the split-cost kernel specialised for one GPU in LL mode (fused_command_kernel_ll, csrc/mppi_fused.cuh).

A single-GPU split-cost plan whose cluster records all go through the GPU's own mailbox runs the instantiation with the
inlined tail; launch_info.ll_tail says so.  Its tail runs the same combines in the same order as the general tail, so
its commands must EQUAL those of the resident kernel (csrc/mppi_resident.cuh), which runs the general, out-of-line
tail on the same grid and cluster size.  Checked for the built-in pendulum at bench.py's C2 size and for a user model
compiled with NVRTC."""
import pytest
import torch

import pytorch_mppi_b200 as eng
from tests import user_models

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(120)]


def _controller(model, dtype):
    T = 30
    torch.manual_seed(0)
    return eng.MPPI(model.dynamics, model.running_cost, 2, torch.tensor(10.0, dtype=dtype), num_samples=16384, horizon=T,
                    U_init=torch.randn(T, 1, dtype=dtype) * 3.0, u_min=torch.tensor(-2.0, dtype=dtype),
                    u_max=torch.tensor(2.0, dtype=dtype), device="cuda", rng_seed=11)


@pytest.mark.parametrize("name", ["pendulum_f32", "pendulum_f64", "user_pendulum_f32"])
def test_ll_tail_route_equals_the_general_tail(name):
    model = user_models.pendulum_user_model() if name.startswith("user") else eng.Pendulum()
    dtype = torch.float64 if name.endswith("f64") else torch.float32
    a, b = _controller(model, dtype), _controller(model, dtype)
    x = [3.14159, 1.0]
    with b.resident(idle_us=500000):
        for i in range(4):
            ua, ub = a.command_host(x), b.command_host(x)
            assert torch.equal(ua, ub), (name, i, ua, ub)
            x = [x[0] + 0.05 * x[1], x[1] + 0.1 * float(ua[0])]
        assert torch.equal(a.U, b.U) and torch.equal(a.cost_total, b.cost_total), name
    info = a.launch_info
    assert info.split_cost == 1 and info.grid_blocks // info.cluster_size > 1
    assert info.ll_tail == 1, (name, info.grid_blocks, info.cluster_size)


def test_ll_tail_only_on_split_cost_plans(monkeypatch):
    monkeypatch.setenv("MPPI_B200_SPLIT_COST", "0")
    c = _controller(eng.Pendulum(), torch.float32)
    c.command([3.14159, 1.0])
    assert c.launch_info.split_cost == 0 and c.launch_info.ll_tail == 0
