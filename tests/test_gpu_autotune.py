"""GPU: per-environment horizons on the fused batched kernels (`MPPI_Batched.set_env_horizon`) and the tuner's population
path (`autotune.ClosedLoopEvaluation` / `BatchedAutotune`).  Environment e against the oracle's command with T = h_e on
the first h_e rows of the same draws; horizons all equal to T bit-identical to none; changes between commands; closed
loops against the host loop; a population's candidate against the same settings run alone; and a tuning run that turns
a pendulum controller that does not swing up into one that does."""
import math

import pytest
import torch

import pytorch_mppi_b200 as eng
from pytorch_mppi_b200 import autotune
from oracle import mppi_oracle as orc
from tests import user_models

pytestmark = pytest.mark.gpu
DEV = "cuda"
N, K, T = 5, 300, 9
H = [9, 1, 4, 7, 2]
LAMBDAS = [0.8, 1.5, 0.3, 2.0, 1.0]
GOALS = [[2.0, 2.0], [-1.0, 0.5], [0.0, -2.0], [1.5, -0.5], [-2.0, -2.0]]
MUS = [[0.0, 0.0], [0.1, -0.2], [-0.1, 0.05], [0.2, 0.0], [0.0, 0.3]]


def _sigmas(dtype):
    return torch.stack([torch.tensor(s, dtype=dtype) for s in (
        [[0.8, 0.1], [0.1, 0.6]], [[0.5, 0.0], [0.0, 0.9]], [[1.2, -0.3], [-0.3, 0.4]], [[0.3, 0.0], [0.0, 0.3]],
        [[0.7, 0.2], [0.2, 0.5]])])


def _lin(goal):
    return eng.LinearPoint(B=[[1.0, 0.0], [0.0, -1.0]], goal=goal)


def _assert_tail_is_u_init(ctrl, horizons):
    for e, h in enumerate(horizons):
        assert torch.equal(ctrl.U[e, h:], ctrl.u_init.to(ctrl.dtype).expand(ctrl.T - h, ctrl.nu)), e


@pytest.mark.parametrize("env_kernel", [False, True])
@pytest.mark.parametrize("tile_memory", ["shared", "global"])
@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-10), (torch.float32, 5e-5)])
def test_linear_point_per_environment_horizons_match_oracle(dtype, tol, tile_memory, env_kernel):
    """env_kernel: per-environment goals too (the kernel that reads one parameter block per environment)."""
    umax = torch.tensor([0.9, 0.7], dtype=dtype)
    sig = _sigmas(dtype)
    lin0 = _lin(GOALS[0])
    goals = GOALS if env_kernel else [GOALS[0]] * N
    torch.manual_seed(1)
    ctrl = eng.MPPI_Batched(lin0.dynamics, lin0.running_cost, 2, torch.eye(2, dtype=dtype), num_envs=N, num_samples=K,
                            horizon=T, u_max=umax, u_scale=1.2, device=DEV, tile_memory=tile_memory)
    ctrl.set_env_params(model_params=torch.tensor([_lin(g).param_blob() for g in goals], dtype=torch.float64)
                        if env_kernel else None,
                        lambda_=torch.tensor(LAMBDAS, dtype=torch.float64), noise_sigma=sig,
                        noise_mu=torch.tensor(MUS, dtype=dtype))
    ctrl.set_env_horizon(H)
    assert ctrl.env_horizon.tolist() == H
    _assert_tail_is_u_init(ctrl, H)
    probs = []
    for e in range(N):
        ol = orc.LinearPointModel(B=lin0.B, goal=goals[e], dtype=dtype)
        probs.append(orc.Problem(ol.dynamics, ol.running_cost, 2, sig[e], K=K, T=H[e], lambda_=LAMBDAS[e],
                                 noise_mu=torch.tensor(MUS[e], dtype=dtype), u_max=umax, u_scale=1.2))
    g = torch.Generator().manual_seed(9)
    U = ctrl.U.cpu().clone()
    x = torch.randn(N, 2, generator=g, dtype=dtype)
    for _ in range(3):
        z = torch.randn(K, T, 2, generator=g, dtype=dtype)
        ctrl.inject_noise(z)
        a = ctrl.command(x.to(DEV)).cpu()
        xn = []
        for e in range(N):
            h = H[e]
            r = orc.mppi_command(probs[e], U[e, :h], x[e], z[:, :h].contiguous())
            assert float((ctrl.U[e, :h].cpu() - r["U"]).abs().max()) < tol, e
            assert float((a[e] - r["action"]).abs().max()) < tol, e
            c = ctrl.cost_total[e].cpu()
            assert float(((c - r["cost_total"]).abs() / r["cost_total"].abs().clamp_min(1.0)).max()) < \
                (1e-10 if dtype == torch.float64 else 2e-4), e
            xn.append(probs[e].dynamics(x[e].view(1, 2), 1.2 * r["action"].view(1, 2)).view(2))
        _assert_tail_is_u_init(ctrl, H)
        U = ctrl.U.cpu().clone()
        x = torch.stack(xn)


def test_cuda_model_per_environment_horizons_match_single_controllers():
    """A CudaModel (the batched kernel its NVRTC module exports): environment e equals a single MPPI with horizon h_e
    on the first h_e rows of the same draws (fp32)."""
    dtype = torch.float32
    base = user_models.pendulum_user_model()
    sig = torch.tensor([2.0, 1.0, 4.0, 0.5, 3.0], dtype=dtype).view(N, 1, 1)
    umax = torch.tensor([2.0], dtype=dtype)
    torch.manual_seed(3)
    ctrl = eng.MPPI_Batched(base.dynamics, base.running_cost, 2, torch.eye(1, dtype=dtype), num_envs=N, num_samples=K,
                            horizon=T, u_max=umax, device=DEV)
    ctrl.set_env_params(lambda_=LAMBDAS, noise_sigma=sig)
    ctrl.set_env_horizon(H)
    singles = [eng.MPPI(base.dynamics, base.running_cost, 2, sig[e], num_samples=K, horizon=H[e], lambda_=LAMBDAS[e],
                        u_max=umax, device=DEV) for e in range(N)]
    for e in range(N):
        singles[e].U = ctrl.U[e, :H[e]]
    g = torch.Generator().manual_seed(4)
    x = torch.randn(N, 2, generator=g, dtype=dtype).to(DEV)
    for _ in range(3):
        z = torch.randn(K, T, 1, generator=g, dtype=dtype)
        ctrl.inject_noise(z)
        a = ctrl.command(x)
        for e in range(N):
            singles[e].inject_noise(z[:, :H[e]].contiguous())
            ae = singles[e].command(x[e])
            assert float((ctrl.U[e, :H[e]] - singles[e].U).abs().max()) < 5e-5, e
            assert float((a[e] - ae).abs().max()) < 5e-5, e
            assert torch.allclose(ctrl.cost_total[e], singles[e].cost_total, rtol=2e-4, atol=1e-4), e
            singles[e].U = ctrl.U[e, :H[e]]
        _assert_tail_is_u_init(ctrl, H)


@pytest.mark.parametrize("tile_memory", ["shared", "global"])
@pytest.mark.parametrize("model", ["pendulum", "linear"])
def test_horizons_equal_to_T_are_bit_identical(tile_memory, model):
    m = eng.Pendulum() if model == "pendulum" else eng.LinearPoint.toy2d_nav(terminal_scale=0.0)
    nu = 1 if model == "pendulum" else 2
    sigma = torch.tensor(4.0) if nu == 1 else torch.tensor([[0.5, 0.1], [0.1, 0.4]])
    n_env, Th = 6, 20
    make = lambda: eng.MPPI_Batched(m.dynamics, m.running_cost, 2, sigma, num_envs=n_env, num_samples=2048, horizon=Th,
                                    lambda_=0.7, u_max=torch.full((nu,), 2.0), rng_seed=3, device=DEV,
                                    tile_memory=tile_memory)
    torch.manual_seed(0)
    a = make()
    torch.manual_seed(0)
    b = make()
    b.set_env_horizon([Th] * n_env)
    x = torch.randn(n_env, 2, generator=torch.Generator().manual_seed(2)).to(DEV)
    for _ in range(3):
        ua, ub = a.command(x), b.command(x)
        for f in ("block_threads", "threads_per_sample", "grid_blocks", "smem_bytes", "cluster_size", "global_tile"):
            assert getattr(a.launch_info, f) == getattr(b.launch_info, f), f
        assert torch.equal(ua, ub) and torch.equal(a.U, b.U) and torch.equal(a.cost_total, b.cost_total)
    b.set_env_horizon(None)
    assert b.env_horizon is None
    assert torch.equal(a.command(x), b.command(x)) and torch.equal(a.U, b.U)


def test_changing_one_horizon_between_commands_changes_that_environment_only():
    pend = eng.Pendulum()
    n_env, Th = 4, 15
    make = lambda: eng.MPPI_Batched(pend.dynamics, pend.running_cost, 2, torch.tensor(4.0), n_env, num_samples=2048,
                                    horizon=Th, u_max=torch.tensor(2.0), rng_seed=8, device=DEV)
    torch.manual_seed(0)
    a = make()
    torch.manual_seed(0)
    b = make()
    hs = [15, 10, 12, 6]
    a.set_env_horizon(hs)
    b.set_env_horizon(hs)
    x = torch.tensor([[math.pi, 0.0], [1.0, 0.5], [-2.0, 0.0], [0.3, -1.0]], device=DEV)
    assert torch.equal(a.command(x), b.command(x)) and torch.equal(a.U, b.U)
    # shrink environment 1's horizon, grow environment 3's: change_horizon's rows
    U_before = b.U.clone()
    hs2 = [15, 5, 12, 11]
    b.set_env_horizon(hs2)
    assert torch.equal(b.U[1, :5], U_before[1, :5]) and torch.equal(b.U[1, 5:], torch.zeros(10, 1, device=DEV))
    assert torch.equal(b.U[3], U_before[3])                    # rows 6..10 already held u_init
    ua, ub = a.command(x), b.command(x)
    for e in (0, 2):
        assert torch.equal(ua[e], ub[e]) and torch.equal(a.U[e], b.U[e]) and torch.equal(a.cost_total[e], b.cost_total[e])
    for e in (1, 3):
        assert not torch.equal(a.cost_total[e], b.cost_total[e])
    _assert_tail_is_u_init(b, hs2)
    _assert_tail_is_u_init(a, hs)


def test_closed_loop_with_per_environment_horizons_equals_host_loop():
    n_env, Kc, Tc, steps = 4, 1024, 20, 10
    pend = eng.Pendulum()
    hs = [20, 7, 13, 3]

    def make():
        c = eng.MPPI_Batched(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), n_env, num_samples=Kc, horizon=Tc,
                             device=DEV, u_max=torch.tensor(2.0), rng_seed=12)
        c.set_env_params(lambda_=[1.0, 0.5, 2.0, 1.0])
        c.set_env_horizon(hs)
        return c
    plant = eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), num_samples=64, horizon=Tc, device=DEV)
    x0 = torch.tensor([[math.pi, 0.0], [1.0, 0.5], [-2.0, 0.0], [0.3, -1.0]], device=DEV)
    torch.manual_seed(0)
    a = make()
    torch.manual_seed(0)
    b = make()
    res = a.run_closed_loop(x0, steps)
    x, xs, us = x0.clone(), [x0.clone()], []
    for _ in range(steps):
        u = b.command(x)
        x = torch.stack([plant.get_rollouts(x[e], U=u[e][None])[0, 0] for e in range(n_env)]).contiguous()
        xs.append(x)
        us.append(u)
    assert torch.equal(res.states, torch.stack(xs)) and torch.equal(res.actions, torch.stack(us))
    assert torch.equal(a.U, b.U) and torch.equal(a.cost_total, b.cost_total)
    _assert_tail_is_u_init(a, hs)
    xl = res.states[-1].clone()            # the RNG position
    assert torch.equal(a.command(xl), b.command(xl)) and torch.equal(a.U, b.U)


def _pendulum_ctrl(sigma, lam, T, K=4096):
    pend = eng.Pendulum()
    return eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(sigma), num_samples=K, horizon=T, lambda_=lam,
                    u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device=DEV, rng_seed=21)


START = [[math.pi, 0.0], [math.pi - 0.4, 0.0], [math.pi + 0.3, 0.5], [2.5, -0.5]]


def test_population_candidate_equals_its_settings_alone():
    torch.manual_seed(0)
    ctrl = _pendulum_ctrl(1.0, 1.0, 20, K=2048)
    x0 = torch.tensor(START, device=DEV)
    ev = autotune.ClosedLoopEvaluation(ctrl, x0, 40, max_horizon=24)
    lams = torch.tensor([0.5, 2.0, 1.0], dtype=torch.float64)
    sigs = torch.tensor([2.0, 6.0, 1.0]).view(3, 1, 1)
    hs = torch.tensor([24, 9, 20], dtype=torch.int32)
    costs, states = ev.evaluate(3, {"lambda_": lams, "noise_sigma": sigs, "horizon": hs})
    assert costs.shape == (3, 4) and states.shape == (41, 3, 4, 2)
    assert torch.equal(states[0], x0.view(1, 4, 2).expand(3, 4, 2))
    pend = eng.Pendulum()
    for c in range(3):
        lone = eng.MPPI_Batched(pend.dynamics, pend.running_cost, 2, torch.tensor(1.0), 4, num_samples=2048, horizon=24,
                                lambda_=1.0, u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device=DEV,
                                rng_seed=ev.seed)
        lone.set_env_params(lambda_=lams[c].repeat(4), noise_sigma=sigs[c].expand(4, 1, 1).clone())
        lone.U = ev.U0.unsqueeze(0).expand(4, -1, -1)
        lone.set_env_horizon(hs[c].repeat(4))
        res = lone.run_closed_loop(x0.clone(), 40)
        assert torch.equal(res.costs.sum(0), costs[c]), c
        assert torch.equal(res.states, states[:, c])


def test_batched_autotune_swings_up_a_pendulum():
    """From settings that do not swing up (noise variance 0.05, horizon 8), BatchedAutotune over sigma, lambda and
    horizon finds settings whose own closed loop swings up from hanging down (K = 4096, max horizon 30, fp32).

    Measured on an H100 80GB HBM3 at 700 W: first-generation incumbent 1274.1, best-ever 271.8 after 6 generations
    (sigma 2.73, lambda at its eps, horizon 16); the tuned controller's last 20 angles within 0.017 rad of upright.
    The thresholds below (best-ever under half the first incumbent, angles within 0.1 rad) leave room for that."""
    torch.manual_seed(0)
    ctrl = _pendulum_ctrl(0.05, 1.0, 8)
    x0 = torch.tensor(START, device=DEV)
    down = torch.tensor([math.pi, 0.0], device=DEV)

    def settled(c):
        res = c.run_closed_loop(down.clone(), 200)
        ang = torch.remainder(res.states[-20:, 0] + math.pi, 2 * math.pi) - math.pi
        return float(ang.abs().max())
    assert settled(ctrl) > 1.0                       # the start settings do not swing up
    ev = autotune.ClosedLoopEvaluation(ctrl, x0, 150, max_horizon=30)
    tuner = autotune.BatchedAutotune([autotune.SigmaParameter(ctrl), autotune.LambdaParameter(ctrl),
                                      autotune.HorizonParameter(ctrl)], ev, optimizer=autotune.CMAESOpt(12, 2.0, seed=0))
    res = tuner.optimize_all(6)
    best_f = tuner.optim.optim.best_f
    print(f"incumbent costs per generation {[round(c, 1) for c in tuner.incumbent_costs]}, best-ever {best_f:.1f}, "
          f"params {res.params}")
    assert best_f < 0.5 * tuner.incumbent_costs[0]
    ang = settled(ctrl)
    print(f"tuned ctrl: sigma {ctrl.noise_sigma.item():.3f} lambda {ctrl.lambda_:.3f} T {ctrl.T}: max |angle| {ang:.3f}")
    assert ang < 0.1
