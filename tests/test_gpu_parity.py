"""GPU parity: the CUDA engine (through the Python API -> C-ABI -> sm_90a kernels) against the oracle and restatements of
the reference on injected draws, and its own properties (determinism, launch geometries, routes, the RNG streams).  The
golden fixtures are replayed in tests/test_gpu_golden_replay.py; the tolerances on U are tests/golden/cases.py U_TOL."""
import numpy as np
import pytest
import torch

from tests.golden.cases import BASE
from tests.golden.replay import OracleRunner, load

pytestmark = pytest.mark.gpu


def test_closed_loop_free_running_c2():
    """10 closed-loop commands WITHOUT resynchronising U: error vs the fp32 reference stays at the
    fp32 noise floor (SURVEY.md §8d parity check)."""
    case, gold = load("pendulum_c2_f32")
    run = OracleRunner(case)
    ctrl = BASE.engine(case, gold, run.stream.U0, "fused")
    x = torch.tensor(case["x0"], dtype=torch.float32)
    model = ctrl._model
    errs = []
    for step in range(case["steps"]):
        ctrl.inject_noise(run.stream.next_z())
        a = ctrl.command(x)
        errs.append(float(np.abs(ctrl.U.cpu().numpy() - gold[f"U_{step}"]).max()))
        x = model.dynamics(x.view(1, -1), a.cpu().view(1, -1)).view(-1)
    assert errs[0] <= 1e-5, errs
    assert max(errs) <= 1e-4, errs      # free-running drift over 10 steps (reference fp32 vs fp64: 1.2e-5 after 10)


def test_philox_stream_matches_oracle_and_parity_holds():
    """Speed mode: in-kernel Philox.  (a) the normals the kernel used equal the numpy statement of the
    stream; (b) feeding exactly those normals to the oracle reproduces the engine's update."""
    from oracle import philox_oracle as po
    for name, np_dt in (("pendulum_small_f32", np.float32), ("linear_mppi_f64", np.float64), ("nav2d_kmppi_f64", np.float64)):
        case, gold = load(name)
        run = OracleRunner(case)
        ctrl = BASE.engine(case, gold, run.stream.U0, "fused", rng_seed=0xC0FFEE1234)
        ctrl.record_noise(True)
        x = torch.tensor(case["x0"], dtype=run.prob.dtype)
        rows = ctrl._noise_rows()
        per = 4 if np_dt == np.float32 else 2
        offset = 0
        for step in range(2):
            ctrl.command(x)
            z_used = ctrl.z_used.cpu().numpy().reshape(case["K"], rows)
            z_orc = po.normals(0xC0FFEE1234, offset, 0, case["K"], rows, np_dt)
            offset += (rows + per - 1) // per
            # fp32 device normals come from the SFU (MUFU.LG2/SIN/COS): a few 1e-6 from the spec
            np.testing.assert_allclose(z_used, z_orc, atol=2e-5 if np_dt == np.float32 else 1e-12, rtol=0)
            r = run.step(x, torch.from_numpy(z_used).reshape(case["K"], -1, run.prob.nu))
            tol = 1e-9 if case["dtype"] == "f64" else 1e-5
            np.testing.assert_allclose(ctrl.U.cpu().numpy(), r["U"].numpy(), atol=tol, rtol=0)
        assert abs(float(z_used.mean())) < 0.1 and abs(float(z_used.std()) - 1.0) < 0.1


def test_same_seed_determinism_and_torch_generator():
    """reference tests/test_mppi.py:103-115, 898-914: same seed -> identical actions."""
    import pytorch_mppi_b200 as eng
    pend = eng.Pendulum()

    def make():
        torch.manual_seed(42)
        return eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), num_samples=1000, horizon=20,
                        u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda")
    c1 = make()
    a1 = [c1.command([3.0, 0.5]).clone() for _ in range(3)]
    c2 = make()
    a2 = [c2.command([3.0, 0.5]).clone() for _ in range(3)]
    for p, q in zip(a1, a2):
        assert torch.equal(p, q)
    assert not torch.equal(a1[0], a1[1])
    assert a1[0].shape == (1,) and a1[0].dtype == torch.float32


def test_large_k_grid_stride_and_block_sizes():
    """K far above SMs x resident CTAs (grid-stride tiles, online rescaling across tiles) and every
    block size give the same update as the small-grid launch."""
    import pytorch_mppi_b200 as eng
    pend = eng.Pendulum()
    K, T = 300_000 + 37, 20
    g = torch.Generator().manual_seed(5)
    z = torch.randn(K, T, 1, generator=g)
    U0 = torch.randn(T, 1, generator=g)
    outs = []
    for bt, tps in ((64, 1), (128, 1), (256, 1), (512, 1), (128, 2), (128, 4), (64, 4)):
        c = eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(4.0), num_samples=K, horizon=T, U_init=U0.clone(),
                     u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda", block_threads=bt, threads_per_sample=tps)
        c.inject_noise(z)
        c.command([2.0, -1.0])
        outs.append(c.U.cpu().clone())
    for o in outs[1:]:
        assert (o - outs[0]).abs().max() < 2e-6
    # yardstick: the oracle in fp64 on the same draws; the engine (fp32) must be no further from it
    # than the fp32 oracle itself is (x2 + 1e-5)
    from oracle import mppi_oracle as orc
    m = orc.PendulumModel(numpy_sin=False)
    res = {}
    for dt in (torch.float32, torch.float64):
        prob = orc.Problem(m.dynamics, m.running_cost, 2, torch.tensor(4.0, dtype=dt), K=K, T=T, u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0))
        res[dt] = orc.mppi_command(prob, U0.to(dt), torch.tensor([2.0, -1.0], dtype=dt), z.to(dt))["U"].double()
    floor = (res[torch.float32] - res[torch.float64]).abs().max().item()
    err = (outs[1].double() - res[torch.float64]).abs().max().item()
    assert err <= 2 * floor + 1e-5, (err, floor)


def test_command_host_zero_copy_equals_command():
    """The pinned-mailbox delivery returns exactly the action `command()` leaves on the device."""
    import pytorch_mppi_b200 as eng
    nav = eng.LinearPoint.toy2d_nav()
    for cls, kw in ((eng.MPPI, {}), (eng.SMPPI, dict(w_action_seq_cost=10.0, action_max=torch.tensor([1.0, 1.0]))),
                    (eng.KMPPI, dict(num_support_pts=5, kernel=eng.RBFKernel(sigma=2)))):
        outs = []
        for host in (False, True):
            torch.manual_seed(3)          # the initial nominal sequence is drawn from the global generator (mppi.py:145)
            c = cls(nav.dynamics, nav.running_cost, 2, torch.eye(2), num_samples=1024, horizon=20, device="cuda",
                    terminal_state_cost=nav.terminal_cost, u_max=torch.tensor([1.0, 1.0]), rng_seed=7, u_per_command=2, **kw)
            acts = []
            x = [-3.0, -2.0]
            for _ in range(3):
                a = c.command_host(x) if host else c.command(x).cpu()
                assert a.shape == (2, 2) and a.device.type == "cpu"
                acts.append(a.clone())
            outs.append(torch.stack(acts))
        assert torch.equal(outs[0], outs[1])


def _mlp_dynamics(dtype, device, seed=25):
    """BASELINE config 4 workload (reference tests/pendulum_approximate.py:47-67): residual MLP
    Linear(3,32)-tanh-Linear(32,32)-tanh-Linear(32,2) on [state, clamp(u)], then angle-normalise theta."""
    import math
    torch.manual_seed(seed)
    net = torch.nn.Sequential(torch.nn.Linear(3, 32), torch.nn.Tanh(), torch.nn.Linear(32, 32), torch.nn.Tanh(),
                              torch.nn.Linear(32, 2)).to(dtype)
    net_d = torch.nn.Sequential(torch.nn.Linear(3, 32), torch.nn.Tanh(), torch.nn.Linear(32, 32), torch.nn.Tanh(),
                                torch.nn.Linear(32, 2)).to(dtype).to(device)
    net_d.load_state_dict(net.state_dict())

    def make(n):
        def dynamics(state, action):
            with torch.no_grad():
                u = torch.clamp(action, -2.0, 2.0)
                xu = torch.cat((state, u), dim=1)
                nxt = state + n(xu)
                th = ((nxt[:, 0] + math.pi) % (2 * math.pi)) - math.pi
                return torch.stack((th, nxt[:, 1]), dim=1)
        return dynamics

    def cost(state, action):
        th = ((state[:, 0] + math.pi) % (2 * math.pi)) - math.pi
        return th ** 2 + 0.1 * state[:, 1] ** 2
    return make(net), make(net_d), cost


@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-9), (torch.float32, 5e-5)])
def test_mlp_dynamics_stepped_route_matches_oracle(dtype, tol):
    """Config 4 shape (K reduced): a torch MLP is an arbitrary callable -> stepped route; injected noise;
    compared with the oracle running the same weights on the CPU."""
    import pytorch_mppi_b200 as eng
    from oracle import mppi_oracle as orc
    dyn_cpu, dyn_gpu, cost = _mlp_dynamics(dtype, "cuda")
    K, T = 4096, 30
    g = torch.Generator().manual_seed(1)
    U0 = torch.randn(T, 1, generator=g, dtype=dtype)
    prob = orc.Problem(dyn_cpu, cost, 2, torch.tensor(1.0, dtype=dtype), K=K, T=T, u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0))
    ctrl = eng.MPPI(dyn_gpu, cost, 2, torch.tensor(1.0, dtype=dtype), num_samples=K, horizon=T, U_init=U0.clone(),
                    u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda")
    assert ctrl._model is None
    U = U0.clone()
    x = torch.tensor([3.0, 0.5], dtype=dtype)
    for step in range(3):
        z = torch.randn(K, T, 1, generator=g, dtype=dtype)
        ctrl.inject_noise(z)
        a = ctrl.command(x)
        r = orc.mppi_command(prob, U, x, z)
        U = r["U"]
        err = float((ctrl.U.cpu() - U).abs().max())
        assert err < tol, (step, err)
        assert float((a.cpu() - r["action"]).abs().max()) < tol
        ctrl.U = U
        x = dyn_cpu(x.view(1, -1), r["action"].view(1, -1)).view(-1)


def test_stepped_route_M_gt_1_and_action_sampler_match_oracle_semantics():
    """rollout_samples M>1 with a variance cost (mppi.py:334-373) and a SpecificActionSampler
    (mppi.py:387-400) against a direct torch restatement on the same injected noise."""
    import pytorch_mppi_b200 as eng
    from oracle import mppi_oracle as orc
    dt = torch.float64
    lin = eng.LinearPoint.unit_test_env()
    g = torch.Generator().manual_seed(3)
    K, T, M = 256, 8, 3
    U0 = torch.randn(T, 2, generator=g, dtype=dt) * 0.2

    class Sampler(eng.SpecificActionSampler):
        def sample_trajectories(self, state, info):
            return torch.full((2, T, 2), 0.25, dtype=dt, device=state.device)

    samp = Sampler()
    dyn = lambda s, a: lin.dynamics(s, a)
    cost = lambda s, a: lin.running_cost(s, a)
    ctrl = eng.MPPI(dyn, cost, 2, torch.eye(2, dtype=dt), num_samples=K, horizon=T, U_init=U0.clone(), device="cuda",
                    rollout_samples=M, rollout_var_cost=0.5, rollout_var_discount=0.9, sample_null_action=True,
                    specific_action_sampler=samp, u_max=torch.tensor([1.0, 1.0], dtype=dt))
    z = torch.randn(K, T, 2, generator=g, dtype=dt)
    ctrl.inject_noise(z)
    x = torch.tensor([-1.0, 0.5], dtype=dt)
    ctrl.command(x)
    assert (samp.start_idx, samp.end_idx) == (1, 3)
    # restatement (deterministic dynamics: the M copies are identical, the variance term is 0)
    olin = orc.LinearPointModel(B=lin.B, goal=lin.goal, dtype=dt)
    prob = orc.Problem(olin.dynamics, olin.running_cost, 2, torch.eye(2, dtype=dt), K=K, T=T, u_max=torch.tensor([1.0, 1.0], dtype=dt))
    Us = orc.shift_rows(U0.clone(), prob.u_init)
    pa = Us + prob.colour(z)
    pa[0] = 0
    pa[1:3] = 0.25
    pa = prob.clamp_u(pa)
    noise = pa - Us
    roll, _, _ = orc.rollout_costs(prob, x, pa)
    total = roll + torch.sum(Us * prob.action_cost(noise), dim=(1, 2))
    _, _, _, omega = orc.softmin_weights(total, 1.0)
    U_want = Us + torch.einsum("k,ktn->tn", omega, noise)
    assert float((ctrl.U.cpu() - U_want).abs().max()) < 1e-10
    assert float((ctrl.cost_total.cpu() - total).abs().max()) < 1e-9
    np.testing.assert_allclose(ctrl.perturbed_action.cpu().numpy(), pa.numpy(), atol=1e-12)


@pytest.mark.parametrize("route", ["fused", "stepped"])
def test_autotune_parameter_flows_refresh_kernel_constants(route):
    """The reference's tuner mutates a LIVE controller (autotune.py:158-162 sigma, :184-187 mu, :213-215
    lambda, :235-237 horizon).  Every such write must reach the kernel's constants: after each one the
    next command equals the oracle built with the new value (same injected noise)."""
    import pytorch_mppi_b200 as eng
    from oracle import mppi_oracle as orc
    dt = torch.float64
    lin = eng.LinearPoint.unit_test_env()
    olin = orc.LinearPointModel(B=lin.B, goal=lin.goal, dtype=dt)
    g = torch.Generator().manual_seed(12)
    K, T = 512, 8
    U0 = torch.randn(T, 2, generator=g, dtype=dt) * 0.3
    if route == "fused":
        dyn, cost = lin.dynamics, lin.running_cost
    else:
        dyn, cost = (lambda s, a: lin.dynamics(s, a)), (lambda s, a: lin.running_cost(s, a))
    ctrl = eng.MPPI(dyn, cost, 2, torch.eye(2, dtype=dt), num_samples=K, horizon=T, U_init=U0.clone(), device="cuda",
                    u_max=torch.tensor([1.5, 1.5], dtype=dt))
    assert (ctrl._model is not None) == (route == "fused")
    x = torch.tensor([-1.0, 0.5], dtype=dt)
    spec = dict(noise_sigma=torch.eye(2, dtype=dt), lambda_=1.0, T=T)

    def check(tag):
        Tn = spec["T"]
        prob = orc.Problem(olin.dynamics, olin.running_cost, 2, spec["noise_sigma"].clone(), K=K, T=Tn, lambda_=spec["lambda_"],
                           u_max=torch.tensor([1.5, 1.5], dtype=dt))
        U_in = ctrl.U.cpu().clone()
        z = torch.randn(K, Tn, 2, generator=g, dtype=dt)
        ctrl.inject_noise(z)
        a = ctrl.command(x)
        r = orc.mppi_command(prob, U_in, x, z)
        assert float((ctrl.U.cpu() - r["U"]).abs().max()) < 1e-10, tag
        assert float((a.cpu() - r["action"]).abs().max()) < 1e-10, tag
        assert float((ctrl.cost_total.cpu() - r["cost_total"]).abs().max()) < 1e-8, tag

    check("initial")
    # SigmaParameter.apply_parameter_value (autotune.py:158-162)
    sigma = torch.tensor([0.4, 2.5], dtype=dt, device=ctrl.d)
    ctrl.noise_sigma = torch.diag(sigma)
    ctrl.noise_dist = torch.distributions.MultivariateNormal(ctrl.noise_mu, covariance_matrix=ctrl.noise_sigma)
    ctrl.noise_sigma_inv = torch.inverse(ctrl.noise_sigma.detach())
    spec["noise_sigma"] = torch.diag(sigma).cpu()
    check("sigma")
    # a full (non-diagonal) covariance takes the Cholesky path
    full = torch.tensor([[1.0, 0.3], [0.3, 0.5]], dtype=dt)
    ctrl.noise_sigma = full.to(ctrl.d)
    spec["noise_sigma"] = full
    check("full sigma")
    # LambdaParameter.apply_parameter_value (autotune.py:213-215)
    ctrl.lambda_ = 0.2
    spec["lambda_"] = 0.2
    check("lambda")
    # HorizonParameter.apply_parameter_value (autotune.py:235-237): longer, then shorter
    for Tn in (13, 5):
        ctrl.change_horizon(Tn)
        spec["T"] = Tn
        assert ctrl.U.shape == (Tn, 2)
        check(f"horizon {Tn}")


@pytest.mark.parametrize("route", ["fused", "stepped"])
@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-10), (torch.float32, 5e-5)])
def test_mppi_batched_matches_oracle(route, dtype, tol):
    """MPPI_Batched (mppi.py:691-873): N environments share the K noise samples; per-environment softmin.
    Both routes against the oracle's restatement on injected noise, two closed-loop commands."""
    import pytorch_mppi_b200 as eng
    from oracle import mppi_oracle as orc
    N, K, T = 5, 300, 9
    lin = eng.LinearPoint.unit_test_env()
    olin = orc.LinearPointModel(B=lin.B, goal=lin.goal, dtype=dtype)
    g = torch.Generator().manual_seed(9)
    sigma = torch.tensor([[0.8, 0.1], [0.1, 0.6]], dtype=dtype)
    umax = torch.tensor([0.9, 0.7], dtype=dtype)
    prob = orc.Problem(olin.dynamics, olin.running_cost, 2, sigma, K=K, T=T, lambda_=0.8, u_max=umax, u_scale=1.2)
    dyn, cost = (lin.dynamics, lin.running_cost) if route == "fused" else ((lambda s, a: lin.dynamics(s, a)), (lambda s, a: lin.running_cost(s, a)))
    torch.manual_seed(1)
    ctrl = eng.MPPI_Batched(dyn, cost, 2, sigma, num_envs=N, num_samples=K, horizon=T, lambda_=0.8, u_max=umax, u_scale=1.2, device="cuda")
    assert (ctrl._model is not None) == (route == "fused")
    U = ctrl.U.cpu().clone()
    assert U.shape == (N, T, 2)
    x = torch.randn(N, 2, generator=g, dtype=dtype)
    for step in range(2):
        z = torch.randn(K, T, 2, generator=g, dtype=dtype)
        ctrl.inject_noise(z)
        a = ctrl.command(x.cuda())
        r = orc.mppi_batched_command(prob, U, x, z)
        assert a.shape == (N, 2)
        assert float((ctrl.U.cpu() - r["U"]).abs().max()) < tol
        assert float((a.cpu() - r["action"]).abs().max()) < tol
        np.testing.assert_allclose(ctrl.cost_total.cpu().numpy(), r["cost_total"].numpy(), rtol=1e-9 if dtype == torch.float64 else 2e-4, atol=0 if dtype == torch.float64 else 1e-4)
        om = ctrl.omega.cpu()
        assert float((om.sum(dim=1) - 1).abs().max()) < 1e-5
        U = r["U"]
        ctrl.U = U
        x = olin.dynamics(x, 1.2 * r["action"])


def test_mppi_batched_envs_are_independent_and_bounded():
    """reference tests/test_mppi.py:743-771: bounds hold; identical start states with identical nominal
    sequences give identical actions, different states give different ones; reset resamples U."""
    import pytorch_mppi_b200 as eng
    pend = eng.Pendulum()
    N = 64
    c = eng.MPPI_Batched(pend.dynamics, pend.running_cost, 2, torch.tensor(4.0), num_envs=N, num_samples=2048, horizon=20,
                         u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda", rng_seed=5)
    c.U = torch.zeros(N, 20, 1)
    x = torch.zeros(N, 2)
    x[:, 0] = 3.0
    x[N // 2:, 0] = 1.0
    a = c.command(x.cuda()).cpu()
    assert a.shape == (N, 1) and (a.abs() <= 2.0 + 1e-6).all()
    assert torch.equal(a[0], a[1]) and torch.equal(a[N // 2], a[N - 1]) and not torch.equal(a[0], a[N - 1])
    before = c.U.clone()
    c.reset()
    assert not torch.allclose(c.U, before)
    # the batched launch equals N single-environment controllers fed the same draws
    single = eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(4.0), num_samples=2048, horizon=20,
                      u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda", rng_seed=5, U_init=torch.zeros(20, 1))
    a1 = single.command([3.0, 0.0]).cpu()
    assert float((a1 - a[0]).abs().max()) < 2e-6


def test_full_size_c5_properties():
    """BASELINE config 5 size on one GPU (K=2^20, T=50, fp32), checked through size-independent
    properties: weights sum to one, beta is the minimum cost, bounds hold, the update is a convex
    combination of the clamped samples (so it stays inside the bounds), same seed -> same result, and a
    different launch geometry gives the same nominal sequence to fp32 accuracy."""
    import pytorch_mppi_b200 as eng
    pend = eng.Pendulum()
    K, T = 1 << 20, 50
    outs = []
    for bt in (0, 256):
        c = eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), num_samples=K, horizon=T,
                     u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), U_init=torch.zeros(T, 1), device="cuda", rng_seed=77,
                     block_threads=bt)
        for _ in range(2):
            a = c.command([3.14159, 1.0])
        cost = c.cost_total
        assert cost.shape == (K,) and torch.isfinite(cost).all()
        assert abs(c.omega.double().sum().item() - 1.0) < 1e-4
        assert abs(cost.min().item() - c.beta.item()) < 1e-6 * max(1.0, abs(c.beta.item()))
        assert (c.U.abs() <= 2.0 + 1e-5).all() and (a.abs() <= 2.0 + 1e-5).all()
        outs.append(c.U.cpu().clone())
    assert float((outs[0] - outs[1]).abs().max()) < 5e-5


@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-9), (torch.float32, 5e-5)])
def test_fused_mlp_dynamics_matches_oracle(dtype, tol):
    """BASELINE config 4 workload on the FUSED route: the registered PendulumMLP model evaluates the
    3-32-32-2 tanh network inside the rollout kernel; compared with the oracle running the same torch
    module on the CPU (injected noise, 3 closed-loop commands), and with the stepped route."""
    import pytorch_mppi_b200 as eng
    from oracle import mppi_oracle as orc
    torch.manual_seed(25)                                             # pendulum_approximate.py:31
    net = torch.nn.Sequential(torch.nn.Linear(3, 32), torch.nn.Tanh(), torch.nn.Linear(32, 32), torch.nn.Tanh(),
                              torch.nn.Linear(32, 2)).to(dtype)
    import copy
    cpu_model = eng.PendulumMLP(copy.deepcopy(net))
    gpu_model = eng.PendulumMLP(copy.deepcopy(net).cuda(), tensor_cores=False)      # the FFMA kernel (fp64 has no other)
    K, T = 4096, 30
    g = torch.Generator().manual_seed(2)
    U0 = torch.randn(T, 1, generator=g, dtype=dtype)
    prob = orc.Problem(cpu_model.dynamics, cpu_model.running_cost, 2, torch.tensor(1.0, dtype=dtype), K=K, T=T,
                       u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0))
    mk = lambda dyn, cost: eng.MPPI(dyn, cost, 2, torch.tensor(1.0, dtype=dtype), num_samples=K, horizon=T, U_init=U0.clone(),
                                    u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda")
    fused = mk(gpu_model.dynamics, gpu_model.running_cost)
    stepped = mk(lambda s, a: gpu_model.dynamics(s, a), lambda s, a: gpu_model.running_cost(s, a))
    assert fused._model is gpu_model and stepped._model is None
    U = U0.clone()
    x = torch.tensor([3.0, 0.5], dtype=dtype)
    for step in range(3):
        z = torch.randn(K, T, 1, generator=g, dtype=dtype)
        fused.inject_noise(z)
        stepped.inject_noise(z)
        a = fused.command(x)
        stepped.command(x)
        r = orc.mppi_command(prob, U, x, z)
        U = r["U"]
        err = float((fused.U.cpu() - U).abs().max())
        assert err < tol, (step, err)
        assert float((a.cpu() - r["action"]).abs().max()) < tol
        assert float((fused.U - stepped.U).abs().max()) < tol
        np.testing.assert_allclose(fused.cost_total.cpu().numpy(), r["cost_total"].numpy(), rtol=1e-9 if dtype == torch.float64 else 2e-4, atol=1e-4)
        fused.U = U
        stepped.U = U
        x = cpu_model.dynamics(x.view(1, -1), r["action"].view(1, -1)).view(-1)


def test_mlp_default_route_is_the_tensor_core_kernel_in_fp32():
    """PendulumMLP() without a route argument ("auto"): fp32 controllers run the wgmma kernel with split operands (the
    parity route), fp64 controllers and MPPI_Batched the FFMA kernel."""
    import copy
    import pytorch_mppi_b200 as eng
    torch.manual_seed(25)
    net = torch.nn.Sequential(torch.nn.Linear(3, 32), torch.nn.Tanh(), torch.nn.Linear(32, 32), torch.nn.Tanh(), torch.nn.Linear(32, 2))
    geo = {}
    for dt in (torch.float32, torch.float64):
        m = eng.PendulumMLP(copy.deepcopy(net).to(dt).cuda())
        c = eng.MPPI(m.dynamics, m.running_cost, 2, torch.tensor(1.0, dtype=dt), num_samples=2048, horizon=10, device="cuda",
                     u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0))
        a = c.command(torch.tensor([3.0, 0.5], dtype=dt))
        assert torch.isfinite(a).all()
        geo[dt] = (c.launch_info.block_threads, c.launch_info.threads_per_sample)
    assert geo[torch.float32] == (256, 2)          # the tensor-core kernel: two threads per sample, 128 samples per CTA
    assert geo[torch.float64] != (256, 2)


@pytest.mark.parametrize("variant", ["mppi", "smppi", "kmppi", "mppi_multipass"])
def test_fused_mlp_tensor_core_route_matches_fp32_kernel(variant, monkeypatch):
    """PendulumMLP(tensor_cores=True): the hidden and output layers run as wgmma MMAs (hi/lo-split bf16 operands,
    fp32 register accumulators).  Same injected noise as the FFMA kernel: costs agree to ~1e-4 relative and
    the updated plan to 2e-4 (operand split error ~2^-16 per layer, 30 steps of a chaotic rollout), for a
    ragged K (partial last tile) and over closed-loop commands; MPPI is also checked against the oracle.
    "mppi_multipass": K large enough that every CTA runs more than two 128-sample tiles (grid-stride loop)."""
    import copy
    import pytorch_mppi_b200 as eng
    from oracle import mppi_oracle as orc
    torch.manual_seed(25)
    net = torch.nn.Sequential(torch.nn.Linear(3, 32), torch.nn.Tanh(), torch.nn.Linear(32, 32), torch.nn.Tanh(),
                              torch.nn.Linear(32, 2))
    cpu_model = eng.PendulumMLP(copy.deepcopy(net))
    ffma = eng.PendulumMLP(copy.deepcopy(net).cuda(), tensor_cores=False)
    tcm = eng.PendulumMLP(copy.deepcopy(net).cuda(), tensor_cores=True)
    K, T = 4096 + 37, 30
    if variant == "mppi_multipass":
        variant = "mppi"
        K = torch.cuda.get_device_properties(0).multi_processor_count * 128 * 5 + 37
    cls = {"mppi": eng.MPPI, "smppi": eng.SMPPI, "kmppi": eng.KMPPI}[variant]
    kw = {"smppi": dict(w_action_seq_cost=2.0, action_max=torch.tensor(2.0)), "kmppi": dict(num_support_pts=6)}.get(variant, {})
    g = torch.Generator().manual_seed(4)
    U0 = torch.randn(T, 1, generator=g) if variant == "mppi" else None
    mk = lambda m: cls(m.dynamics, m.running_cost, 2, torch.tensor(1.0), num_samples=K, horizon=T, U_init=None if U0 is None else U0.clone(),
                       u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda", **kw)
    torch.manual_seed(8)
    a_ref = mk(ffma)
    torch.manual_seed(8)
    a_tc = mk(tcm)                      # same random initial plan (KMPPI draws its control points)
    assert a_tc._model is tcm
    prob = orc.Problem(cpu_model.dynamics, cpu_model.running_cost, 2, torch.tensor(1.0), K=K, T=T, u_min=torch.tensor(-2.0),
                       u_max=torch.tensor(2.0))
    x = torch.tensor([3.0, 0.5])
    for step in range(3):
        if variant == "kmppi":
            z = torch.randn(K, 6, 1, generator=g)
        else:
            z = torch.randn(K, T, 1, generator=g)
        a_ref.inject_noise(z)
        a_tc.inject_noise(z)
        U_before = a_ref.U.cpu().clone()
        u1 = a_ref.command(x)
        u2 = a_tc.command(x)
        c1, c2 = a_ref.cost_total.cpu().numpy(), a_tc.cost_total.cpu().numpy()
        assert np.isfinite(c2).all()
        assert a_tc.launch_info.block_threads == 256 and a_tc.launch_info.threads_per_sample == 2     # two threads per sample
        n_tiles = (K + 127) // 128
        if K > 4096 + 37:
            assert n_tiles > 2 * a_tc.launch_info.grid_blocks, (n_tiles, a_tc.launch_info.grid_blocks)
        assert a_ref.launch_info.block_threads != 128
        np.testing.assert_allclose(c2, c1, rtol=2e-3, atol=2e-3)
        assert float(np.median(np.abs(c2 - c1) / np.maximum(1.0, np.abs(c1)))) < 2e-5
        assert float((a_tc.U - a_ref.U).abs().max()) < 2e-4, step
        assert float((u1 - u2).abs().max()) < 2e-4
        if variant == "mppi":
            r = orc.mppi_command(prob, U_before, x, z)
            assert float((a_tc.U.cpu() - r["U"]).abs().max()) < 2e-4
        a_tc.U = a_ref.U.clone()
        x = cpu_model.dynamics(x.view(1, -1), u1.cpu().view(1, -1)).view(-1)


def test_fused_mlp_tensor_core_bf16_mode_is_close_and_controls():
    """tensor_cores="bf16": plain bf16 operands in the hidden layers, with the MUFU.TANH and the exp-based tanh.
    Not a parity route (2^-8 operand rounding): the costs must track the fp32 kernel's to a few percent, the softmin
    weights must correlate, and the controller must still drive the learned pendulum's cost down."""
    import copy
    import pytorch_mppi_b200 as eng
    torch.manual_seed(25)
    net = torch.nn.Sequential(torch.nn.Linear(3, 32), torch.nn.Tanh(), torch.nn.Linear(32, 32), torch.nn.Tanh(),
                              torch.nn.Linear(32, 2))
    ffma = eng.PendulumMLP(copy.deepcopy(net).cuda(), tensor_cores=False)
    K, T = 8192, 20
    mk = lambda m: eng.MPPI(m.dynamics, m.running_cost, 2, torch.tensor(1.0), num_samples=K, horizon=T, U_init=torch.zeros(T, 1),
                            u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda")
    for fast in (True, False):
        tcm = eng.PendulumMLP(copy.deepcopy(net).cuda(), tensor_cores="bf16", fast_tanh=fast)
        a_ref, a_tc = mk(ffma), mk(tcm)
        g = torch.Generator().manual_seed(9)
        z = torch.randn(K, T, 1, generator=g)
        a_ref.inject_noise(z)
        a_tc.inject_noise(z)
        x = torch.tensor([2.5, 0.3])
        a_ref.command(x)
        a_tc.command(x)
        assert a_tc.launch_info.block_threads == 256 and a_tc.launch_info.threads_per_sample == 2, fast
        c1, c2 = a_ref.cost_total.double().cpu(), a_tc.cost_total.double().cpu()
        assert torch.isfinite(c2).all()
        rel = ((c2 - c1).abs() / c1.abs().clamp_min(1.0))
        assert float(rel.median()) < 2e-2 and float(rel.max()) < 0.5, (fast, float(rel.median()), float(rel.max()))
        assert float(torch.corrcoef(torch.stack((c1, c2)))[0, 1]) > 0.999, fast
        assert float((a_tc.U - a_ref.U).abs().max()) < 0.1, fast


@pytest.mark.parametrize("variant", ["mppi", "smppi", "kmppi"])
def test_compile_cuda_graph_replay_equals_eager_stepped(variant):
    """compile() on the stepped route captures the whole command in a CUDA graph; replays must equal the
    eager stepped commands bit for bit (same seed; the Philox counter advances on the device)."""
    import pytorch_mppi_b200 as eng
    dyn_cpu, dyn_gpu, cost = _mlp_dynamics(torch.float32, "cuda")
    cls = {"mppi": eng.MPPI, "smppi": eng.SMPPI, "kmppi": eng.KMPPI}[variant]
    kw = {"smppi": dict(w_action_seq_cost=2.0, action_max=torch.tensor(2.0)), "kmppi": dict(num_support_pts=6)}.get(variant, {})

    def make():
        return cls(dyn_gpu, cost, 2, torch.tensor(1.0), num_samples=2048, horizon=12, U_init=torch.zeros(12, 1),
                   u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda", rng_seed=11, **kw)
    eager, graphed = make(), make()
    graphed.compile()
    x = torch.tensor([3.0, 0.5])
    for step in range(4):
        a1 = eager.command(x)
        a2 = graphed.command(x)
        assert torch.equal(a1, a2), (variant, step)
        assert torch.equal(eager.U, graphed.U)
        assert torch.equal(eager.cost_total, graphed.cost_total)
        x = dyn_cpu(x.view(1, -1), a1.cpu().view(1, -1)).view(-1)
    assert len(graphed._graphs) == 1
    # refinement without shifting is a second captured graph
    assert torch.equal(eager.command(x, shift_nominal_trajectory=False), graphed.command(x, shift_nominal_trajectory=False))
    assert len(graphed._graphs) == 2


def test_user_cuda_model_equals_builtin_and_oracle():
    """CudaModel (compiled at run time with NVRTC, loaded with cudaLibraryLoadData): the pendulum written as user CUDA
    snippets gives bit-identical commands to the built-in registered model — fused route, resident route and
    get_rollouts; a model that exists nowhere else (double integrator with drag, quadratic + terminal cost) matches
    the oracle running its torch definition."""
    import pytorch_mppi_b200 as eng
    from oracle import mppi_oracle as orc
    from tests import user_models as um_
    ref = eng.Pendulum()
    um = um_.pendulum_user_model()
    outs = []
    for model in (ref, um):
        c = eng.MPPI(model.dynamics, model.running_cost, 2, torch.tensor(10.0), num_samples=4096, horizon=25,
                     U_init=torch.zeros(25, 1), u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda", rng_seed=3)
        assert c._model is model
        acts = [c.command([3.0, 0.4]).clone() for _ in range(3)]
        with c.resident(idle_us=200000):                      # the user model's resident kernel
            acts += [c.command_host([3.0, 0.4]).to("cuda") for _ in range(3)]
        acts.append(c.get_rollouts(torch.tensor([3.0, 0.4]))[0, -1, :1])     # its states kernel
        outs.append(torch.stack(acts))
        assert c.launch_info.split_cost == 1
    assert torch.equal(outs[0], outs[1])

    m = um_.integrator_user_model()
    dyn, rc, tc = um_.int_dyn, um_.int_cost, um_.int_term
    K, T = 1500, 18
    dt = torch.float64
    g = torch.Generator().manual_seed(4)
    U0 = torch.randn(T, 1, generator=g, dtype=dt) * 0.3
    c = eng.MPPI(m.dynamics, m.running_cost, 2, torch.tensor(0.5, dtype=dt), num_samples=K, horizon=T, U_init=U0.clone(),
                 terminal_state_cost=m.terminal_cost, u_max=torch.tensor(1.0, dtype=dt), device="cuda")
    assert c._model is m
    prob = orc.Problem(dyn, rc, 2, torch.tensor(0.5, dtype=dt), K=K, T=T, u_max=torch.tensor(1.0, dtype=dt), terminal_state_cost=tc)
    U = U0.clone()
    x = torch.tensor([0.0, 0.0], dtype=dt)
    for _ in range(3):
        z = torch.randn(K, T, 1, generator=g, dtype=dt)
        c.inject_noise(z)
        a = c.command(x)
        r = orc.mppi_command(prob, U, x, z)
        U = r["U"]
        assert float((c.U.cpu() - U).abs().max()) < 1e-10
        np.testing.assert_allclose(c.states.cpu().numpy(), r["states"].numpy(), atol=1e-10)
        x = dyn(x.view(1, -1), r["action"].view(1, -1)).view(-1)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("shape", [(16384, 30, 1), (1000, 7, 2), (300000, 20, 1), (999, 7, 3)])
def test_torch_compatible_rng_reproduces_torch_randn(dtype, shape):
    """rng="torch": the kernel regenerates, sample by sample, exactly the tensor torch.randn(K,T,nu,
    device="cuda") would have produced from the same generator state — the stream the reference draws on a
    CUDA device (mppi.py:203) — and advances the generator by the same amount.  (999, 7, 3): T*nu = 21 normals per
    sample, an odd count, with the (3,3) model of tests/shape_models.py."""
    import pytorch_mppi_b200 as eng
    from tests import shape_models as shm
    K, T, nu = shape
    model = {1: eng.Pendulum, 2: eng.LinearPoint.unit_test_env, 3: lambda: shm.shape_model(3, 3)}[nu]()
    nx = 3 if nu == 3 else 2
    x0 = [1.0, 0.5, -0.2][:nx]
    sigma = torch.tensor(1.0, dtype=dtype) if nu == 1 else torch.eye(nu, dtype=dtype)
    c = eng.MPPI(model.dynamics, model.running_cost, nx, sigma, num_samples=K, horizon=T, U_init=torch.zeros(T, nu, dtype=dtype),
                 terminal_state_cost=model.terminal_cost if model.has_terminal else None, device="cuda", rng="torch")
    c.record_noise(True)
    gen = torch.cuda.default_generators[0]
    for rep in range(2):
        torch.manual_seed(1234 + rep)
        torch.rand(17, device="cuda")                       # move the generator off zero
        state = gen.get_state()
        want = torch.randn(K, T, nu, device="cuda", dtype=dtype)
        off_after = gen.get_offset()
        gen.set_state(state)
        c.command(x0)
        assert gen.get_offset() == off_after
        got = c.z_used
        if dtype == torch.float32:
            assert torch.equal(got, want), float((got - want).abs().max())
        else:
            assert float((got - want).abs().max()) < 1e-14
    # and the command run on those draws equals the oracle fed torch.randn's tensor
    if K <= 20000:
        from oracle import mppi_oracle as orc
        if nu == 3:
            f, rc, tc = shm.twins(3, 3)
            prob = orc.Problem(f, rc, 3, sigma, K=K, T=T, terminal_state_cost=tc)
        else:
            m = orc.PendulumModel(numpy_sin=False) if nu == 1 else orc.LinearPointModel(B=model.B, goal=model.goal, dtype=dtype)
            prob = orc.Problem(m.dynamics, m.running_cost, 2, sigma, K=K, T=T)
        U0 = torch.zeros(T, nu, dtype=dtype)
        c.U = U0
        gen.set_state(state)
        c.command(x0)
        r = orc.mppi_command(prob, U0, torch.tensor(x0, dtype=dtype), want.cpu())
        assert float((c.U.cpu() - r["U"]).abs().max()) < (2e-5 if dtype == torch.float32 else 1e-9)
