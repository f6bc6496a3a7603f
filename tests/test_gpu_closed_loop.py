"""GPU: closed-loop episodes (`run_closed_loop`) against the host loop they replace — ``u = command(x)`` on the device
state, ``x = get_rollouts(x, U=u[None])[0, 0] + disturbance[s]`` — bit for bit, and the controller left exactly where
that loop leaves it; the recorded costs against the models' torch twins; an fp64 episode against the oracle; and the
C2 pendulum swinging up."""
import math

import numpy as np
import pytest
import torch

import pytorch_mppi_b200 as eng
from tests import closed_loop_models as clm

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _host_loop(c, x0, steps, dist=None, plants=None):
    """The Python loop run_closed_loop replaces; `plants`: a controller per environment whose get_rollouts is the plant
    (default: `c` itself)."""
    x = x0.clone()
    xs, us = [x], []
    for s in range(steps):
        u = c.command(x)
        if plants is None:
            xn = c.get_rollouts(x, U=u[None])[0, 0] if x.dim() == 1 else c.get_rollouts(x, num_rollouts=x.shape[0], U=u[:1])[:, 0]
        elif x.dim() == 1:
            xn = plants.get_rollouts(x, U=u[None])[0, 0]
        else:
            xn = torch.stack([p.get_rollouts(x[e], U=u[e][None])[0, 0] for e, p in enumerate(plants)])
        if dist is not None:
            xn = xn + dist[s]
        xs.append(xn.contiguous())
        us.append(u)
        x = xs[-1]
    return torch.stack(xs), torch.stack(us)


def _same_controller(a, b):
    assert torch.equal(a.U, b.U) and torch.equal(a.cost_total, b.cost_total)
    if isinstance(a, eng.SMPPI):
        assert torch.equal(a.action_sequence, b.action_sequence)
    if isinstance(a, eng.KMPPI):
        assert torch.equal(a.theta, b.theta)
    if not isinstance(a, eng.MPPI_Batched):
        assert torch.equal(a.beta, b.beta) and torch.equal(a.eta, b.eta)
        assert torch.equal(a.noise, b.noise) and torch.equal(a.perturbed_action, b.perturbed_action)
        assert a.state.data_ptr() != 0 and torch.equal(a.state, b.state)


def _pair(make):
    """Two controllers that start alike (a nominal drawn at construction comes from the same torch seed)."""
    torch.manual_seed(0)
    a = make()
    torch.manual_seed(0)
    return a, make()


def _check(make, x0, steps, dist=None, plant_params=None, plants=None):
    a, b = _pair(make)
    res = a.run_closed_loop(x0, steps, plant_params=plant_params, disturbance=dist)
    xs, us = _host_loop(b, x0, steps, dist, plants)
    assert torch.equal(res.states, xs) and torch.equal(res.actions, us)
    _same_controller(a, b)
    # the RNG position: a further command of both draws the same noise
    x = res.states[-1].clone()
    assert torch.equal(a.command(x), b.command(x)) and torch.equal(a.U, b.U)
    return res


def _pendulum_c2(model=None, dtype=torch.float32, **kw):
    m = model or eng.Pendulum()
    kw.setdefault("num_samples", 16384)
    kw.setdefault("horizon", 30)
    return eng.MPPI(m.dynamics, m.running_cost, 2, torch.tensor(10.0, dtype=dtype), lambda_=1.0, device=DEV,
                    u_min=torch.tensor(-2.0, dtype=dtype), u_max=torch.tensor(2.0, dtype=dtype), rng_seed=5, **kw)


def test_pendulum_c2_split_cost_route_equals_host_loop():
    make = _pendulum_c2
    x0 = torch.tensor([math.pi, 0.0], device=DEV)
    res = _check(make, x0, 100)
    c = make()
    c.command(x0.clone())
    assert c.launch_info.split_cost == 1
    pend = eng.Pendulum()
    assert torch.allclose(res.costs, pend.running_cost(res.states[1:], res.actions), rtol=1e-5, atol=1e-5)


def test_pendulum_torch_rng_and_disturbance_equal_host_loop():
    make = lambda: _pendulum_c2(num_samples=2048, horizon=20, rng="torch")
    x0 = torch.tensor([1.0, -0.5], device=DEV)
    dist = 0.01 * torch.randn(12, 2, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    a, b = _pair(make)
    gen = torch.cuda.default_generators[0]
    off = gen.get_offset()
    res = a.run_closed_loop(x0, 12, disturbance=dist)
    gen.set_offset(off)
    xs, us = _host_loop(b, x0, 12, dist)
    assert torch.equal(res.states, xs) and torch.equal(res.actions, us)
    _same_controller(a, b)


def test_linear_point_smppi_equals_host_loop():
    m = eng.LinearPoint.unit_test_env()
    make = lambda: eng.SMPPI(m.dynamics, m.running_cost, 2, torch.eye(2, dtype=torch.float64) * 0.5, num_samples=1024,
                             horizon=15, device=DEV, u_max=torch.tensor([1.0, 1.0], dtype=torch.float64), rng_seed=9,
                             w_action_seq_cost=0.1, action_min=torch.tensor([-1.0, -1.0], dtype=torch.float64),
                             action_max=torch.tensor([1.0, 1.0], dtype=torch.float64))
    x0 = torch.tensor([-3.0, 2.0], dtype=torch.float64, device=DEV)
    res = _check(make, x0, 20)
    assert (res.costs - m.running_cost(res.states[1:], res.actions)).abs().max() < 1e-12


def test_kmppi_toy2d_nav_fp64_equals_host_loop():
    m = eng.LinearPoint.toy2d_nav()
    dt = torch.float64
    make = lambda: eng.KMPPI(m.dynamics, m.running_cost, 2, torch.eye(2, dtype=dt), num_samples=2048, horizon=20,
                             device=DEV, terminal_state_cost=m.terminal_cost, u_max=torch.tensor([1.0, 1.0], dtype=dt),
                             num_support_pts=5, kernel=eng.RBFKernel(sigma=2), rng_seed=4)
    x0 = torch.tensor([-3.0, -2.0], dtype=dt, device=DEV)
    res = _check(make, x0, 15)
    assert (res.costs - m.running_cost(res.states[1:], res.actions)).abs().max() < 1e-12


def test_cuda_model_with_costmap_equals_host_loop():
    cmap = clm.make_costmap()
    m = clm.costmap_model(cmap)
    make = lambda: eng.MPPI(m.dynamics, m.running_cost, 2, torch.eye(2) * 0.3, num_samples=4096, horizon=20, device=DEV,
                            u_max=torch.tensor([1.0, 1.0]), rng_seed=2)
    x0 = torch.tensor([-1.0, -1.5], device=DEV)
    res = _check(make, x0, 25)
    assert torch.isfinite(res.costs).all() and (res.costs > 0).all()


def test_cuda_model_copies_plant_is_copy_zero():
    K = 2048
    m = clm.pendulum_ensemble(K)
    dt = torch.float64
    make = lambda: eng.MPPI(m.dynamics, m.running_cost, 2, torch.tensor(5.0, dtype=dt), num_samples=K, horizon=20,
                            device=DEV, terminal_state_cost=m.terminal_cost, rollout_samples=clm.ENSEMBLE_M,
                            u_max=torch.tensor(2.0, dtype=dt), rng_seed=8)
    x0 = torch.tensor([2.5, 0.0], dtype=dt, device=DEV)
    res0 = _check(make, x0, 12)
    # another copy's physics through plant_params: the plant replays copy 0 of a model whose copy 0 is copy 1
    p = list(m.params)
    masses, lengths = p[6:6 + 3], p[9:12]
    rot = p[:6] + masses[1:] + masses[:1] + lengths[1:] + lengths[:1]
    plant = eng.CudaModel(2, 1, m._step_code, m._cost_code, params=rot, terminal_code=m._terminal_code, copies=3,
                          dynamics=m._dyn, running_cost=m._cost, terminal_cost=m._term)
    pc = eng.MPPI(plant.dynamics, plant.running_cost, 2, torch.tensor(5.0, dtype=dt), num_samples=K, horizon=20,
                  device=DEV, terminal_state_cost=plant.terminal_cost, rollout_samples=3, rng_seed=8)
    res = _check(make, x0, 12, plant_params=rot, plants=pc)
    assert not torch.equal(res.states, res0.states)


def test_global_tile_beyond_the_shared_tile_equals_host_loop():
    m = eng.Pendulum()
    dt = torch.float64
    make = lambda: eng.MPPI(m.dynamics, m.running_cost, 2, torch.tensor(10.0, dtype=dt), num_samples=1024, horizon=1500,
                            device=DEV, u_max=torch.tensor(2.0, dtype=dt), rng_seed=6, tile_memory="auto")
    x0 = torch.tensor([math.pi, 0.0], dtype=dt, device=DEV)
    _check(make, x0, 4)
    c = make()
    c.command(x0.clone())
    assert c.launch_info.global_tile == 1


def test_batched_per_environment_plants_equal_host_loop():
    N, K, T = 4, 1024, 20
    masses = [1.0, 1.2, 0.8, 1.5]
    nominal = eng.Pendulum()
    make = lambda: eng.MPPI_Batched(nominal.dynamics, nominal.running_cost, 2, torch.tensor(10.0), N, num_samples=K,
                                    horizon=T, device=DEV, u_max=torch.tensor(2.0), rng_seed=12)
    plants = []
    for mass in masses:
        pm = eng.Pendulum(m=mass)
        plants.append(eng.MPPI(pm.dynamics, pm.running_cost, 2, torch.tensor(10.0), num_samples=64, horizon=T, device=DEV))
    pp = torch.tensor([eng.Pendulum(m=mass).param_blob() for mass in masses], dtype=torch.float64)
    x0 = torch.tensor([[math.pi, 0.0], [1.0, 0.5], [-2.0, 0.0], [0.3, -1.0]], device=DEV)
    dist = 0.01 * torch.randn(10, N, 2, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    a, b = _pair(make)
    res = a.run_closed_loop(x0, 10, plant_params=pp, disturbance=dist)
    xs, us = _host_loop(b, x0, 10, dist, plants)
    assert res.states.shape == (11, N, 2) and res.actions.shape == (10, N, 1) and res.costs.shape == (10, N)
    assert torch.equal(res.states, xs) and torch.equal(res.actions, us)
    _same_controller(a, b)
    for e, mass in enumerate(masses):      # each environment's cost under its own plant
        c = eng.Pendulum(m=mass).running_cost(res.states[1:, e], res.actions[:, e])
        assert torch.allclose(res.costs[:, e], c, rtol=1e-5, atol=1e-5)


def test_oracle_fp64_closed_loop():
    """K=257, T=13, 10 steps: noise from the Philox oracle at the offset of each command, commands from the oracle's
    mppi_command, the plant the model's torch twin."""
    from oracle import mppi_oracle as orc
    from oracle import philox_oracle as ph
    K, T, steps, dt = 257, 13, 10, torch.float64
    pend = eng.Pendulum()
    c = eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0, dtype=dt), num_samples=K, horizon=T,
                 device=DEV, u_min=torch.tensor(-2.0, dtype=dt), u_max=torch.tensor(2.0, dtype=dt), rng_seed=21,
                 U_init=torch.zeros(T, 1, dtype=dt))
    x0 = torch.tensor([math.pi - 0.3, 0.2], dtype=dt)
    res = c.run_closed_loop(x0.to(DEV), steps)
    m = orc.PendulumModel()
    prob = orc.Problem(m.dynamics, m.running_cost, 2, torch.tensor(10.0, dtype=dt), K=K, T=T,
                       u_min=torch.tensor(-2.0, dtype=dt), u_max=torch.tensor(2.0, dtype=dt))
    U, x = torch.zeros(T, 1, dtype=dt), x0
    chunks = (T + 1) // 2
    for s in range(steps):
        z = torch.from_numpy(ph.normals(21, s * chunks, 0, K, T, np.float64)).reshape(K, T, 1)
        r = orc.mppi_command(prob, U, x, z)
        U = r["U"]
        assert abs(float(res.actions[s, 0].cpu()) - float(r["action"][0])) < 1e-9
        x = pend.dynamics(x.view(1, 2), r["action"].view(1, 1)).view(2)
        assert (res.states[s + 1].cpu() - x).abs().max() < 1e-9
        x = res.states[s + 1].cpu()          # continue from the engine's state (the 1e-9 gap does not compound)
    assert (c.U.cpu() - U).abs().max() < 1e-9


def test_pendulum_swings_up_and_heavier_plant_differs():
    make = _pendulum_c2
    x0 = torch.tensor([math.pi, 0.0], device=DEV)
    c, _ = _pair(make)
    res = c.run_closed_loop(x0, 200)
    th = res.states[-20:, 0]
    ang = torch.remainder(th + math.pi, 2 * math.pi) - math.pi
    assert ang.abs().max() < 0.1, ang
    heavy = eng.Pendulum(m=1.3)
    pc = _pendulum_c2(model=heavy, num_samples=64)
    res_h = _check(make, x0, 60, plant_params=heavy.param_blob(), plants=pc)
    assert not torch.equal(res_h.states, res.states[:61])
