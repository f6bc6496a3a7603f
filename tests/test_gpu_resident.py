"""GPU: resident mode (csrc/mppi_resident.cuh) — command_host() served by a grid that stays on the GPU.

The contract is bit-identity with the launch route: the resident kernel runs the same stage functions on the same
(state, seed, Philox counter, flags), so every action, the nominal sequence and cost_total must be EQUAL, not close.

A resident kernel is a spin-waiting kernel, so
every test carries a timeout, the host side gives up after 10 s, and the kernel itself leaves after `idle_us` without a
command.
"""
import time

import pytest
import torch

import pytorch_mppi_b200 as eng
from tests import reports

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(120)]


def _pendulum(K=2048, T=15, dtype=torch.float32, seed=11):
    torch.manual_seed(5)                      # U_init is drawn from the global generator (mppi.py:145)
    m = eng.Pendulum()
    return eng.MPPI(m.dynamics, m.running_cost, 2, torch.tensor(4.0, dtype=dtype), num_samples=K, horizon=T, device="cuda",
                    lambda_=1.0, u_min=torch.tensor(-2.0, dtype=dtype), u_max=torch.tensor(2.0, dtype=dtype), rng_seed=seed)


def _nav(cls, dtype, **kw):
    torch.manual_seed(3)
    nav = eng.LinearPoint.toy2d_nav()
    return cls(nav.dynamics, nav.running_cost, 2, torch.eye(2, dtype=dtype), num_samples=1024, horizon=20, device="cuda",
               terminal_state_cost=nav.terminal_cost, u_max=torch.tensor([1.0, 1.0], dtype=dtype), rng_seed=7, u_per_command=2, **kw)


def _pend_step(x, u):
    """host-side closed loop (tests/pendulum.py:30-48 in plain floats)"""
    import math
    th, thd = x
    u = max(-2.0, min(2.0, float(u)))
    thd = max(-8.0, min(8.0, thd + (15.0 * math.sin(th) + 3.0 * u) * 0.05))
    return [th + thd * 0.05, thd]


def test_resident_equals_launch_route_pendulum_closed_loop():
    a, b = _pendulum(), _pendulum()
    xa, xb = [3.0, 1.0], [3.0, 1.0]
    with b.resident(idle_us=500000):             # long idle clock: the launch count below must not depend on host jitter
        for i in range(40):
            ua, ub = a.command_host(xa), b.command_host(xb)
            assert torch.equal(ua, ub), (i, ua, ub)
            xa, xb = _pend_step(xa, ua[0]), _pend_step(xb, ub[0])
        assert b.resident_launches == 1                    # forty commands, one kernel launch
        assert a.launch_info.split_cost == 1 and b.launch_info.split_cost == 1
        assert torch.equal(a.U, b.U)
        assert torch.equal(a.cost_total, b.cost_total)
        assert torch.equal(a.omega, b.omega)
    assert torch.equal(a.command_host(xa), b.command_host(xb))      # back on the launch route


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("kind", ["mppi", "smppi", "kmppi"])
def test_resident_equals_launch_route_all_variants(kind, dtype):
    cls, kw = {"mppi": (eng.MPPI, {}),
               "smppi": (eng.SMPPI, dict(w_action_seq_cost=10.0, action_max=torch.tensor([1.0, 1.0], dtype=dtype))),
               "kmppi": (eng.KMPPI, dict(num_support_pts=5, kernel=eng.RBFKernel(sigma=2)))}[kind]
    a, b = _nav(cls, dtype, **kw), _nav(cls, dtype, **kw)
    x = [-3.0, -2.0]
    b.start_resident(idle_us=20000)
    try:
        for i in range(6):
            shift = i % 3 != 2                             # every third command contradicts the predicted shift flag
            ua, ub = a.command_host(x, shift_nominal_trajectory=shift), b.command_host(x, shift_nominal_trajectory=shift)
            assert ua.shape == (2, 2) and torch.equal(ua, ub), (kind, i)
            x = [x[0] + 0.5 * float(ua[0, 0]), x[1] - 0.5 * float(ua[0, 1])]
        assert torch.equal(a.U, b.U) and torch.equal(a.cost_total, b.cost_total)
        if kind == "smppi":
            assert torch.equal(a.action_sequence, b.action_sequence)
        if kind == "kmppi":
            assert torch.equal(a.theta, b.theta)
        assert torch.equal(a.noise, b.noise)               # lazily materialised from the last command's counter
    finally:
        b.stop_resident()


def test_resident_wakes_up_after_idle_exit_and_after_writes():
    a, b = _pendulum(K=1024), _pendulum(K=1024)
    x = [3.0, 1.0]
    b.start_resident(idle_us=300)
    try:
        assert torch.equal(a.command_host(x), b.command_host(x))
        time.sleep(0.05)                                   # far beyond idle_us: the grid has left
        torch.cuda.synchronize()                           # ... so this returns
        assert torch.equal(a.command_host(x), b.command_host(x))
        assert b.resident_launches == 2
        # a write through the setter makes the grid leave; the next command_host brings it back
        newU = torch.zeros_like(a.U)
        a.U, b.U = newU, newU
        assert torch.equal(a.command_host(x), b.command_host(x))
        # a launch-route command in between
        assert torch.equal(a.command(x).cpu(), b.command(x).cpu())
        assert torch.equal(a.command_host(x), b.command_host(x))
        # a parameter change repacks the plan (the resident grid's arguments are frozen at launch)
        a.lambda_, b.lambda_ = 0.5, 0.5
        assert torch.equal(a.command_host(x), b.command_host(x))
        assert torch.equal(a.U, b.U)
    finally:
        b.stop_resident()


def test_resident_refuses_what_it_cannot_run():
    big = _pendulum(K=131072, T=15)                        # many tiles per SM: not the split-cost geometry
    with pytest.raises(eng._cabi.MppiLibraryError):
        big.start_resident()
    lin = torch.nn.Linear(3, 2).cuda()
    stepped = eng.MPPI(lambda s, a: s + lin(torch.cat((s, a), 1)), lambda s, a: (s ** 2).sum(1), 2, torch.tensor(1.0),
                       num_samples=256, horizon=5, device="cuda")
    with pytest.raises(eng._cabi.MppiLibraryError):
        stepped.start_resident()


def test_resident_latency_report():
    """Not an assertion about speed — writes the host-loop time per command of both routes (C2 shape) to
    tests/_reports/resident_latency.txt."""
    lines = []
    for K, T in ((16384, 30), (4096, 30)):
        res = {}
        for mode in ("launch", "resident"):
            c = _pendulum(K=K, T=T)
            if mode == "resident":
                c.start_resident(idle_us=5000)
            x = [3.0, 1.0]
            for _ in range(200):
                u = c.command_host(x)
                x = _pend_step(x, u[0])
            t0 = time.perf_counter()
            n = 3000
            for _ in range(n):
                u = c.command_host(x)
                x = _pend_step(x, u[0])
            res[mode] = (time.perf_counter() - t0) / n * 1e6
            if mode == "resident":
                lines.append(f"K={K} T={T} resident launches: {c.resident_launches}")
                c.stop_resident()
        lines.append(f"K={K} T={T} command_host: launch route {res['launch']:.2f} us, resident {res['resident']:.2f} us per command "
                     f"(Python host loop, pendulum stepped on the host)")
    reports.write("resident_latency.txt", "\n".join(lines) + "\n")
    print("\n".join(lines))
