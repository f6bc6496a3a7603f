"""GPU: `MPPI_Batched.set_env_params` — every environment with its own model parameters, temperature and noise on the
fused kernel.  Environment e against the oracle's single-environment command with e's settings on the same draws; neutral
per-environment values bit-identical to the shared controller; closed loops against the host loop; updates between
commands; and a lambda sweep of the C2 pendulum in one closed-loop call."""
import math

import pytest
import torch

import pytorch_mppi_b200 as eng
from oracle import mppi_oracle as orc
from tests import closed_loop_models as clm
from tests import user_models

pytestmark = pytest.mark.gpu
DEV = "cuda"
N, K, T = 5, 300, 9
LAMBDAS = [0.8, 1.5, 0.3, 2.0, 1.0]
GOALS = [[2.0, 2.0], [-1.0, 0.5], [0.0, -2.0], [1.5, -0.5], [-2.0, -2.0]]
MUS = [[0.0, 0.0], [0.1, -0.2], [-0.1, 0.05], [0.2, 0.0], [0.0, 0.3]]


def _sigmas(dtype):
    """A mix of diagonal and full 2x2 covariances."""
    return torch.stack([torch.tensor(s, dtype=dtype) for s in (
        [[0.8, 0.1], [0.1, 0.6]], [[0.5, 0.0], [0.0, 0.9]], [[1.2, -0.3], [-0.3, 0.4]], [[0.3, 0.0], [0.0, 0.3]],
        [[0.7, 0.2], [0.2, 0.5]])])


def _lin(goal):
    return eng.LinearPoint(B=[[1.0, 0.0], [0.0, -1.0]], goal=goal)


@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-10), (torch.float32, 5e-5)])
def test_linear_point_per_environment_settings_match_oracle(dtype, tol):
    umax = torch.tensor([0.9, 0.7], dtype=dtype)
    sig = _sigmas(dtype)
    lin0 = _lin(GOALS[0])
    torch.manual_seed(1)
    ctrl = eng.MPPI_Batched(lin0.dynamics, lin0.running_cost, 2, torch.eye(2, dtype=dtype), num_envs=N, num_samples=K,
                            horizon=T, u_max=umax, u_scale=1.2, device=DEV)
    ctrl.set_env_params(model_params=torch.tensor([_lin(g).param_blob() for g in GOALS], dtype=torch.float64),
                        lambda_=torch.tensor(LAMBDAS, dtype=torch.float64), noise_sigma=sig,
                        noise_mu=torch.tensor(MUS, dtype=dtype))
    probs = []
    for e in range(N):
        ol = orc.LinearPointModel(B=lin0.B, goal=GOALS[e], dtype=dtype)
        probs.append(orc.Problem(ol.dynamics, ol.running_cost, 2, sig[e], K=K, T=T, lambda_=LAMBDAS[e],
                                 noise_mu=torch.tensor(MUS[e], dtype=dtype), u_max=umax, u_scale=1.2))
    g = torch.Generator().manual_seed(9)
    U = ctrl.U.cpu().clone()
    x = torch.randn(N, 2, generator=g, dtype=dtype)
    for _ in range(3):
        z = torch.randn(K, T, 2, generator=g, dtype=dtype)
        ctrl.inject_noise(z)
        a = ctrl.command(x.to(DEV)).cpu()
        Un, xn = [], []
        for e in range(N):
            r = orc.mppi_command(probs[e], U[e], x[e], z)
            assert float((ctrl.U[e].cpu() - r["U"]).abs().max()) < tol
            assert float((a[e] - r["action"]).abs().max()) < tol
            c = ctrl.cost_total[e].cpu()
            assert float(((c - r["cost_total"]).abs() / r["cost_total"].abs().clamp_min(1.0)).max()) < (1e-10 if dtype == torch.float64 else 2e-4)
            Un.append(r["U"])
            xn.append(probs[e].dynamics(x[e].view(1, 2), 1.2 * r["action"].view(1, 2)).view(2))
        om = ctrl.omega.cpu()
        assert float((om.sum(dim=1) - 1).abs().max()) < 1e-5
        U = torch.stack(Un)
        ctrl.U = U
        x = torch.stack(xn)


def _single(model, sigma, lam, mu, umax, dtype):
    return eng.MPPI(model.dynamics, model.running_cost, 2, sigma, num_samples=K, horizon=T, lambda_=lam, noise_mu=mu,
                    u_max=umax, device=DEV)


@pytest.mark.parametrize("which", ["params", "costmap"])
def test_cuda_model_per_environment_params_match_single_controllers(which):
    """Environment e equals a single-environment MPPI built with e's settings (fp32, on the same draws)."""
    dtype = torch.float32
    if which == "params":
        base = user_models.pendulum_user_model()
        rows = [[10.0, 1.0 + 0.1 * e, 1.0, 0.05, 2.0, 8.0, 0.1] for e in range(N)]
        make = lambda p: eng.CudaModel(2, 1, user_models.PEND_STEP, user_models.PEND_COST, params=p)
        nu = 1
    else:
        cmap = clm.make_costmap()
        base = clm.costmap_model(cmap)
        rows = [[0.1, -2.0, 16.0] + GOALS[e] for e in range(N)]
        make = lambda p: clm.costmap_model(cmap, params=p)
        nu = 2
    sig = _sigmas(dtype)[:, :nu, :nu]
    mus = torch.tensor(MUS, dtype=dtype)[:, :nu]
    umax = torch.full((nu,), 2.0 if nu == 1 else 1.0, dtype=dtype)
    torch.manual_seed(3)
    ctrl = eng.MPPI_Batched(base.dynamics, base.running_cost, 2, torch.eye(nu, dtype=dtype), num_envs=N, num_samples=K,
                            horizon=T, u_max=umax, device=DEV)
    ctrl.set_env_params(model_params=rows, lambda_=LAMBDAS, noise_sigma=sig, noise_mu=mus)
    singles = [_single(make(rows[e]), sig[e], LAMBDAS[e], mus[e], umax, dtype) for e in range(N)]
    for e in range(N):
        singles[e].U = ctrl.U[e]
    g = torch.Generator().manual_seed(4)
    x = torch.randn(N, 2, generator=g, dtype=dtype).to(DEV)
    for _ in range(3):
        z = torch.randn(K, T, nu, generator=g, dtype=dtype)
        ctrl.inject_noise(z)
        a = ctrl.command(x)
        for e in range(N):
            singles[e].inject_noise(z)
            ae = singles[e].command(x[e])
            assert float((ctrl.U[e] - singles[e].U).abs().max()) < 5e-5
            assert float((a[e] - ae).abs().max()) < 5e-5
            assert torch.allclose(ctrl.cost_total[e], singles[e].cost_total, rtol=2e-4, atol=1e-4)
            singles[e].U = ctrl.U[e]


@pytest.mark.parametrize("tile_memory", ["shared", "global"])
@pytest.mark.parametrize("model", ["pendulum", "linear"])
def test_neutral_per_environment_values_are_bit_identical(tile_memory, model):
    m = eng.Pendulum() if model == "pendulum" else eng.LinearPoint.toy2d_nav(terminal_scale=0.0)
    nu = 1 if model == "pendulum" else 2
    sigma = torch.tensor(4.0) if nu == 1 else torch.tensor([[0.5, 0.1], [0.1, 0.4]])
    n_env, lam = 6, 0.7
    make = lambda: eng.MPPI_Batched(m.dynamics, m.running_cost, 2, sigma, num_envs=n_env, num_samples=2048, horizon=20,
                                    lambda_=lam, u_max=torch.full((nu,), 2.0), rng_seed=3, device=DEV,
                                    tile_memory=tile_memory)
    torch.manual_seed(0)
    a = make()
    torch.manual_seed(0)
    b = make()
    blob = m.param_blob() + m.param_blob_ext()
    b.set_env_params(model_params=[blob] * n_env, lambda_=[lam] * n_env,
                     noise_sigma=sigma.reshape(nu, nu).expand(n_env, nu, nu).clone(), noise_mu=torch.zeros(n_env, nu))
    x = torch.randn(n_env, 2, generator=torch.Generator().manual_seed(2)).to(DEV)
    for _ in range(3):
        ua, ub = a.command(x), b.command(x)
        for f in ("block_threads", "threads_per_sample", "grid_blocks", "smem_bytes", "cluster_size", "global_tile"):
            assert getattr(a.launch_info, f) == getattr(b.launch_info, f), f
        assert torch.equal(ua, ub) and torch.equal(a.U, b.U) and torch.equal(a.cost_total, b.cost_total)
    # back to shared settings: still the same controller
    b.set_env_params()
    assert b.env_lambda is None and b.env_model_params is None and b.env_noise_sigma is None and b.env_noise_mu is None
    assert torch.equal(a.command(x), b.command(x)) and torch.equal(a.U, b.U)


def test_closed_loop_with_per_environment_settings_equals_host_loop():
    n_env, Kc, Tc, steps = 4, 1024, 20, 10
    masses, lams = [1.0, 1.2, 0.8, 1.5], [1.0, 0.5, 2.0, 1.0]
    nominal = eng.Pendulum()
    blobs = torch.tensor([eng.Pendulum(m=mm).param_blob() for mm in masses], dtype=torch.float64)
    sig = torch.tensor([10.0, 5.0, 8.0, 12.0]).view(n_env, 1, 1)

    def make():
        c = eng.MPPI_Batched(nominal.dynamics, nominal.running_cost, 2, torch.tensor(10.0), n_env, num_samples=Kc,
                             horizon=Tc, device=DEV, u_max=torch.tensor(2.0), rng_seed=12)
        c.set_env_params(model_params=blobs, lambda_=lams, noise_sigma=sig)
        return c
    plants = []
    for mm in masses:
        pm = eng.Pendulum(m=mm)
        plants.append(eng.MPPI(pm.dynamics, pm.running_cost, 2, torch.tensor(10.0), num_samples=64, horizon=Tc, device=DEV))
    x0 = torch.tensor([[math.pi, 0.0], [1.0, 0.5], [-2.0, 0.0], [0.3, -1.0]], device=DEV)
    torch.manual_seed(0)
    a = make()
    torch.manual_seed(0)
    b = make()
    res = a.run_closed_loop(x0, steps)
    x, xs, us = x0.clone(), [x0.clone()], []
    for _ in range(steps):
        u = b.command(x)
        x = torch.stack([p.get_rollouts(x[e], U=u[e][None])[0, 0] for e, p in enumerate(plants)]).contiguous()
        xs.append(x)
        us.append(u)
    assert torch.equal(res.states, torch.stack(xs)) and torch.equal(res.actions, torch.stack(us))
    assert torch.equal(a.U, b.U) and torch.equal(a.cost_total, b.cost_total)
    for e, mm in enumerate(masses):      # each plant's own running cost
        c = eng.Pendulum(m=mm).running_cost(res.states[1:, e], res.actions[:, e])
        assert torch.allclose(res.costs[:, e], c, rtol=1e-5, atol=1e-5)
    xl = res.states[-1].clone()            # the RNG position
    assert torch.equal(a.command(xl), b.command(xl)) and torch.equal(a.U, b.U)


def test_update_between_commands_changes_the_second_only():
    lin = eng.LinearPoint.unit_test_env()
    make = lambda: eng.MPPI_Batched(lin.dynamics, lin.running_cost, 2, torch.eye(2) * 0.5, 3, num_samples=1024,
                                    horizon=12, rng_seed=5, device=DEV)
    torch.manual_seed(0)
    a = make()
    torch.manual_seed(0)
    b = make()
    x = torch.tensor([[0.0, 0.0], [1.0, -1.0], [-1.0, 2.0]], device=DEV)
    lams = torch.tensor([0.2, 1.0, 3.0], dtype=torch.float64)
    # a: the update is enqueued between its two commands; b: before its first
    u1a = a.command(x).clone()
    a.set_env_params(lambda_=lams)
    u2a = a.command(x)
    b.set_env_params(lambda_=lams)
    u1b = b.command(x).clone()
    torch.manual_seed(0)
    c = make()
    u1c = c.command(x).clone()
    assert torch.equal(u1a, u1c) and not torch.equal(u1a, u1b)
    om = a.omega
    assert float((om.sum(dim=1) - 1).abs().max()) < 1e-5
    beta = a._stats[:, 0:1].float()
    eta = a._stats[:, 1:2].float()
    ref = torch.exp(-(a.cost_total - beta) / lams.to(DEV, torch.float32).view(3, 1)) / eta
    assert torch.allclose(om, ref, rtol=1e-5, atol=1e-7)
    assert u2a.shape == (3, 2)


def test_lambda_sweep_closed_loop_swings_up():
    """16 C2-shaped pendulums (K = 16384, T = 30, noise variance 10), one closed-loop call over a lambda sweep that
    includes the C2 temperature, 1.0: those environments swing up from hanging down, as the C2 controller does."""
    lams = [0.1, 0.3, 1.0, 3.0, 10.0, 1.0, 30.0, 100.0, 0.5, 2.0, 5.0, 10.0, 20.0, 50.0, 200.0, 1000.0]
    n_env = len(lams)
    pend = eng.Pendulum()
    c = eng.MPPI_Batched(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), n_env, num_samples=16384, horizon=30,
                         device=DEV, u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), rng_seed=5)
    c.set_env_params(lambda_=lams)
    x0 = torch.tensor([[math.pi, 0.0]] * n_env, device=DEV)
    res = c.run_closed_loop(x0, 200)
    ang = torch.remainder(res.states[-20:, :, 0] + math.pi, 2 * math.pi) - math.pi
    for e, lam in enumerate(lams):
        if lam == 1.0:
            assert float(ang[:, e].abs().max()) < 0.1, (e, ang[:, e])
    ep_cost = res.costs.sum(dim=0)
    assert torch.isfinite(ep_cost).all() and len(set(ep_cost.tolist())) > 1
