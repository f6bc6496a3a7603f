"""GPU: closed loops against a plant named apart from the controller's model (`run_closed_loop(plant=...)`), against the
host loop they replace — ``u = command(x)`` on the device state, ``x = P.get_rollouts(x, U=u[None])[0, 0] +
disturbance[s]`` with P a controller on the plant — bit for bit, with the controller left where that loop leaves it.
Learned controllers (PendulumMLP on the tensor-core and FFMA kernels, the ensemble, MPPI_Batched) on analytic and
user-written plants; a plant reading its own tensors; a learned controller swinging up the true pendulum; and the
autotuner's population path against a structurally different plant."""
import math

import pytest
import torch

import pytorch_mppi_b200 as eng
from pytorch_mppi_b200 import autotune
from tests import closed_loop_models as clm
from tests import closed_loop_plant_models as cpm
from tests.golden import cases
from tests.test_gpu_closed_loop import _host_loop, _pair, _same_controller

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _check(make, x0, steps, plant, plants, dist=None, plant_params=None):
    """run_closed_loop(plant=) of one controller against the host loop of its twin, whose plant steps are `plants`'
    get_rollouts (a controller on the plant model, or one per environment)."""
    a, b = _pair(make)
    res = a.run_closed_loop(x0, steps, plant=plant, plant_params=plant_params, disturbance=dist)
    xs, us = _host_loop(b, x0, steps, dist, plants)
    assert torch.equal(res.states, xs) and torch.equal(res.actions, us)
    _same_controller(a, b)
    # the RNG position: a further command of both draws the same noise
    x = res.states[-1].clone()
    assert torch.equal(a.command(x), b.command(x)) and torch.equal(a.U, b.U)
    return res


def _on(model, dtype=torch.float32, **kw):
    """A small controller on `model` whose get_rollouts is the host loop's plant step."""
    return eng.MPPI(model.dynamics, model.running_cost, model.nx, torch.eye(model.nu, dtype=dtype), num_samples=64,
                    horizon=5, device=DEV, **kw)


def _mlp_controller(net, dtype=torch.float32, K=32768, T=30, sigma=1.0, **kw):
    m = eng.PendulumMLP(net.to(dtype))
    return eng.MPPI(m.dynamics, m.running_cost, 2, torch.tensor(sigma, dtype=dtype), num_samples=K, horizon=T, lambda_=1.0,
                    device=DEV, u_min=torch.tensor(-2.0, dtype=dtype), u_max=torch.tensor(2.0, dtype=dtype), rng_seed=3, **kw)


def test_own_model_as_plant_reproduces_plant_none():
    """plant= the controller's own model class with the same parameters is the old closed loop, bit for bit."""
    pend = eng.Pendulum()
    cm = clm.costmap_model(clm.make_costmap())       # a CudaModel: the plant reads the same tensor through its own refs
    for make, plant, x0 in (
            (lambda: eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), num_samples=16384, horizon=30,
                              device=DEV, u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), rng_seed=5),
             eng.Pendulum(), torch.tensor([math.pi, 0.0], device=DEV)),
            (lambda: eng.MPPI(cm.dynamics, cm.running_cost, 2, torch.eye(2) * 0.3, num_samples=4096, horizon=20, device=DEV,
                              u_max=torch.tensor([1.0, 1.0]), rng_seed=2),
             cm, torch.tensor([-1.0, -1.5], device=DEV))):
        a, b = _pair(make)
        dist = 0.01 * torch.randn(30, 2, device=DEV, generator=torch.Generator(device=DEV).manual_seed(4))
        ra = a.run_closed_loop(x0, 30, disturbance=dist)
        rb = b.run_closed_loop(x0, 30, plant=plant, disturbance=dist)
        assert torch.equal(ra.states, rb.states) and torch.equal(ra.actions, rb.actions) and torch.equal(ra.costs, rb.costs)
        _same_controller(a, b)


def test_mlp_c4_wgmma_controller_on_pendulum_plant():
    """The C4 shape: PendulumMLP fp32 on the wgmma kernel (K=32768, T=30), a Pendulum plant."""
    net = cases.make_mlp_net(25, torch.float32)
    make = lambda: _mlp_controller(net)
    plant = eng.Pendulum()
    x0 = torch.tensor([math.pi, 1.0], device=DEV)
    c = make()
    c.command(x0.clone())
    assert c.launch_info.block_threads == 256 and c.launch_info.threads_per_sample == 2       # the wgmma tiles
    res = _check(make, x0, 40, plant, _on(plant))
    assert torch.allclose(res.costs, plant.running_cost(res.states[1:], res.actions), rtol=1e-5, atol=1e-5)


def test_mlp_fp64_ffma_controller_on_true_pendulum_cuda_plant():
    """PendulumMLP fp64 (FFMA kernel) on the reference's true pendulum as a CudaModel plant, with a disturbance."""
    dt = torch.float64
    net = cases.make_mlp_net(25, dt)
    make = lambda: _mlp_controller(net, dt, K=4096, T=20)
    plant = cpm.true_pendulum()
    x0 = torch.tensor([math.pi - 0.2, 0.5], dtype=dt, device=DEV)
    dist = 0.01 * torch.randn(25, 2, dtype=dt, device=DEV, generator=torch.Generator(device=DEV).manual_seed(6))
    res = _check(make, x0, 25, plant, _on(plant, dt), dist=dist)
    assert (res.costs - cpm.true_cost(res.states[1:], res.actions)).abs().max() < 1e-12
    # the plant's step is the integrate-then-clip of true_dynamics, not Pendulum's clip-then-integrate
    step = cpm.true_dynamics(res.states[:-1], res.actions) + dist
    assert (res.states[1:] - step).abs().max() < 1e-12


def test_mlp_ensemble_controller_on_pendulum_plant():
    nets = [cases.make_mlp_net(30 + i, torch.float32) for i in range(4)]
    ens = eng.PendulumMLPEnsemble(nets)
    make = lambda: eng.MPPI(ens.dynamics, ens.running_cost, 2, torch.tensor(1.0), num_samples=8192, horizon=30, device=DEV,
                            u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), rollout_samples=4, rng_seed=7)
    plant = eng.Pendulum()
    _check(make, torch.tensor([math.pi, 1.0], device=DEV), 20, plant, _on(plant))


def test_batched_mlp_controller_on_per_environment_plants():
    N, masses = 4, [1.0, 1.2, 0.8, 1.5]
    m = eng.PendulumMLP(cases.make_mlp_net(25, torch.float32))
    make = lambda: eng.MPPI_Batched(m.dynamics, m.running_cost, 2, torch.tensor(1.0), N, num_samples=4096, horizon=30,
                                    device=DEV, u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), rng_seed=12)
    pp = torch.tensor([eng.Pendulum(m=mass).param_blob() for mass in masses], dtype=torch.float64)
    x0 = torch.tensor([[math.pi, 0.0], [1.0, 0.5], [-2.0, 0.0], [0.3, -1.0]], device=DEV)
    dist = 0.01 * torch.randn(10, N, 2, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    res = _check(make, x0, 10, eng.Pendulum(), [_on(eng.Pendulum(m=mass)) for mass in masses], dist=dist, plant_params=pp)
    for e, mass in enumerate(masses):      # each environment's cost under its own plant
        c = eng.Pendulum(m=mass).running_cost(res.states[1:, e], res.actions[:, e])
        assert torch.allclose(res.costs[:, e], c, rtol=1e-5, atol=1e-5)


def test_batched_env_model_params_do_not_leak_into_an_explicit_plant():
    N, masses = 3, [1.0, 1.6, 0.7]
    pend = eng.Pendulum()
    env = torch.tensor([eng.Pendulum(m=mass).param_blob() for mass in masses], dtype=torch.float64)

    def make():
        c = eng.MPPI_Batched(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), N, num_samples=2048, horizon=20,
                             device=DEV, u_max=torch.tensor(2.0), rng_seed=4)
        c.set_env_params(model_params=env)
        return c

    x0 = torch.tensor([[math.pi, 0.0], [2.0, 0.0], [-1.0, 1.0]], device=DEV)
    # the explicit plant (default parameters) for every environment, although the controllers plan with their own masses
    res = _check(make, x0, 15, eng.Pendulum(), [_on(eng.Pendulum())] * N)
    torch.manual_seed(0)
    own = make().run_closed_loop(x0, 15)     # plant=None: each environment's plant is its own model
    assert not torch.equal(own.states[:, 1:], res.states[:, 1:])


def test_smppi_linear_point_on_costmap_plant_reads_the_plants_tensor():
    lp = eng.LinearPoint.unit_test_env()
    make = lambda: eng.SMPPI(lp.dynamics, lp.running_cost, 2, torch.eye(2) * 0.5, num_samples=1024, horizon=15, device=DEV,
                             u_max=torch.tensor([1.0, 1.0]), rng_seed=9, w_action_seq_cost=0.1,
                             action_min=torch.tensor([-1.0, -1.0]), action_max=torch.tensor([1.0, 1.0]))
    x0 = torch.tensor([-1.0, -1.5], device=DEV)
    cmap_a, cmap_b = clm.make_costmap(seed=1), clm.make_costmap(seed=2)
    plant_a, plant_b = cpm.costmap_plant(cmap_a), cpm.costmap_plant(cmap_b)
    res_a = _check(make, x0, 20, plant_a, _on(plant_a))
    a, _ = _pair(make)
    res_b = a.run_closed_loop(x0, 20, plant=plant_b)
    # the controller and the plant's step never read a costmap: only the plant's cost does, from its own tensor
    assert torch.equal(res_a.states, res_b.states) and torch.equal(res_a.actions, res_b.actions)
    assert not torch.equal(res_a.costs, res_b.costs)
    p = cpm.COSTMAP_PLANT_PARAMS
    xs = res_a.states[1:]
    i = ((xs[:, 1] - p[1]) * p[2]).to(torch.int64).clamp(0, clm.COSTMAP_HW[0] - 1)
    j = ((xs[:, 0] - p[1]) * p[2]).to(torch.int64).clamp(0, clm.COSTMAP_HW[1] - 1)
    goal = (xs[:, 0] - p[3]) ** 2 + (xs[:, 1] - p[4]) ** 2
    assert torch.allclose(res_a.costs, goal + cmap_a[i, j], rtol=1e-5, atol=1e-5)
    assert torch.allclose(res_b.costs, goal + cmap_b[i, j], rtol=1e-5, atol=1e-5)


def _fit_mlp(adam_steps, n=4096):
    """A PendulumMLP fitted to seeded transitions of the analytic pendulum (residual targets, full-batch Adam, fp64)."""
    g = torch.Generator().manual_seed(0)
    x = torch.cat(((torch.rand(n, 1, generator=g, dtype=torch.float64) * 2 - 1) * math.pi,
                   (torch.rand(n, 1, generator=g, dtype=torch.float64) * 2 - 1) * 8.0), 1)
    u = (torch.rand(n, 1, generator=g, dtype=torch.float64) * 2 - 1) * 2.0
    y = (eng.Pendulum().dynamics(x, u) - x).to(DEV)
    xu = torch.cat((x, u), 1).to(DEV)
    net = cases.make_mlp_net(25, torch.float64).to(DEV)
    for p in net.parameters():
        p.requires_grad_(True)
    opt = torch.optim.Adam(net.parameters(), lr=3e-3)
    for _ in range(adam_steps):
        opt.zero_grad()
        loss = ((net(xu) - y) ** 2).mean()
        loss.backward()
        opt.step()
    for p in net.parameters():
        p.requires_grad_(False)
    return net.cpu().float(), loss.item()


def test_learned_controller_swings_up_the_true_pendulum():
    """The reference's learned-dynamics use case: MPPI planning on a fitted network, the episode on the pendulum."""
    x0 = torch.tensor([math.pi, 0.0], device=DEV)

    def final_angles(net):
        c = _mlp_controller(net, K=16384, T=30, sigma=10.0)
        res = c.run_closed_loop(x0, 200, plant=eng.Pendulum())
        th = res.states[-20:, 0]
        return (torch.remainder(th + math.pi, 2 * math.pi) - math.pi).abs().max().item()

    net, loss = _fit_mlp(1500)
    trained = final_angles(net)
    untrained = final_angles(cases.make_mlp_net(25, torch.float32))
    # measured on an H100: fit loss 7.26e-4; max |angle| over the last 20 steps 0.0359 trained, 3.1408 untrained (the
    # untrained network leaves the pendulum hanging)
    assert loss < 5e-3, loss
    assert trained < 0.1 <= untrained, (trained, untrained)


def test_closed_loop_evaluation_with_a_structurally_different_plant():
    """A candidate's episode cost from ClosedLoopEvaluation(plant=) is the sum of the costs of a direct
    MPPI_Batched.run_closed_loop(plant=) with the same settings."""
    pend = eng.Pendulum()
    ctrl = eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(5.0), num_samples=2048, horizon=20, device=DEV,
                    u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), rng_seed=17)
    plant = cpm.true_pendulum()
    x0 = torch.tensor([[math.pi, 0.0], [1.0, 0.0]], device=DEV)
    lam = torch.tensor([1.0, 3.0], dtype=torch.float64)
    ev = autotune.ClosedLoopEvaluation(ctrl, x0, 30, plant=plant)
    costs, states = ev.evaluate(2, {"lambda_": lam})
    b = autotune.ClosedLoopEvaluation(ctrl, x0, 30, plant=plant).controller(2)        # a fresh controller, same settings
    b.set_env_params(lambda_=lam.repeat_interleave(2))
    b.U = ev.U0.unsqueeze(0).expand(4, -1, -1)
    res = b.run_closed_loop(x0.repeat(2, 1), 30, plant=plant)
    assert torch.equal(costs, res.costs.sum(0).view(2, 2))
    assert torch.equal(states, res.states.view(31, 2, 2, -1))
    # the plant is the true pendulum, not the controller's model
    own = autotune.ClosedLoopEvaluation(ctrl, x0, 30).evaluate(2, {"lambda_": lam})[0]
    assert not torch.equal(own, costs)
