"""tile_memory on one GPU: the global-tile kernels compute what the shared-memory kernels compute (bit for bit at a pinned
geometry), they match the fp64 oracle at horizons past the shared-memory edge on both routes, "auto" keeps today's plan
wherever it fits, and the refusals name their reason before anything launches."""
import json

import numpy as np
import pytest
import torch

import pytorch_mppi_b200 as eng
from oracle import mppi_oracle as orc
from pytorch_mppi_b200._cabi import MppiLibraryError
from tests import ensemble_models as em
from tests import reports
from tests import shape_models as shm
from tests import step_models as sm
from tests import tensor_models as tm
from tests.golden.shape_cases import SIG3

pytestmark = pytest.mark.gpu

CLASSES = {"mppi": eng.MPPI, "smppi": eng.SMPPI, "kmppi": eng.KMPPI}


def _sigma(nu, dtype):
    return torch.tensor(SIG3 if nu == 3 else np.eye(nu) * 0.7 + 0.1, dtype=dtype)


def _kw(variant, T, S=None):
    if variant == "smppi":
        return dict(w_action_seq_cost=2.0, delta_t=0.5)
    if variant == "kmppi":
        return dict(num_support_pts=S or max(2, T // 2), kernel=eng.RBFKernel(sigma=2.0))
    return {}


def _ctrl(variant, nx, nu, dtype, K, T, route, tile_memory, S=None, **extra):
    m = shm.shape_model(nx, nu)
    f, c, t = shm.twins(nx, nu)
    dyn, cost, term = (m.dynamics, m.running_cost, m.terminal_cost) if route == "fused" else (f, c, t)
    U0 = None if variant == "smppi" else torch.randn(T, nu, dtype=dtype, generator=torch.Generator().manual_seed(T)) * 0.3
    return CLASSES[variant](dyn, cost, nx, _sigma(nu, dtype), num_samples=K, horizon=T, U_init=U0, terminal_state_cost=term,
                            u_max=torch.full((nu,), 1.2, dtype=dtype), device="cuda", tile_memory=tile_memory,
                            **_kw(variant, T, S), **extra)


def _z(K, rows, nu, dtype, seed):
    return torch.randn(K, rows, nu, generator=torch.Generator().manual_seed(seed), dtype=dtype)


def _seq(ctrl):
    out = [ctrl.U.clone()]
    if isinstance(ctrl, eng.SMPPI):
        out.append(ctrl.action_sequence.clone())
    if isinstance(ctrl, eng.KMPPI):
        out.append(ctrl.theta.clone())
    return out


# ---- 1. same arithmetic: "global" against "shared" where both plan, at a pinned geometry -------------------------------
@pytest.mark.parametrize("route", ["fused", "stepped"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("shape", shm.SHAPES, ids=lambda s: f"n{s[0]}u{s[1]}")
@pytest.mark.parametrize("variant", sorted(CLASSES))
def test_global_tile_is_bit_identical_to_shared(variant, shape, dtype, route, monkeypatch):
    monkeypatch.setenv("MPPI_B200_CLUSTER", "1")
    nx, nu = shape
    K, T = 2048, 24
    rows = T // 2 if variant == "kmppi" else T
    x = torch.linspace(-0.5, 0.5, nx, dtype=dtype)
    res = {}
    for tm in ("shared", "global"):
        ctrl = _ctrl(variant, nx, nu, dtype, K, T, route, tm, block_threads=64, threads_per_sample=1, rng_seed=11)
        seqs, costs, acts = [], [], []
        for i in range(5):
            if i < 2:
                ctrl.inject_noise(_z(K, rows, nu, dtype, 100 + i))      # injected z, then the Philox stream
            acts.append(ctrl.command(x).clone())
            costs.append(ctrl.cost_total.clone())
            seqs.append(_seq(ctrl))
        info = ctrl.launch_info
        assert info.global_tile == (1 if tm == "global" else 0)
        if route == "fused":
            assert (info.block_threads, info.threads_per_sample, info.cluster_size) == (64, 1, 1)
        res[tm] = (acts, costs, seqs)
    for a, b in zip(res["shared"][1], res["global"][1]):
        assert torch.equal(a, b)
    for a, b in zip(res["shared"][0], res["global"][0]):
        assert torch.equal(a, b)
    for sa, sb in zip(res["shared"][2], res["global"][2]):
        for a, b in zip(sa, sb):
            assert torch.equal(a, b)


@pytest.mark.parametrize("route", ["fused", "stepped"])
def test_global_tile_torch_rng_batched_and_multipass(route, monkeypatch):
    """rng="torch", MPPI_Batched with 3 environments and a multi-pass grid (K = 131072) at equal geometry."""
    monkeypatch.setenv("MPPI_B200_CLUSTER", "1")
    nx, nu, dtype, T = 3, 3, torch.float64, 20
    x = torch.linspace(-0.5, 0.5, nx, dtype=dtype)
    for kw in (dict(rng="torch", K=4096), dict(K=131072, rng_seed=3)):
        K = kw.pop("K")
        out = []
        for tm in ("shared", "global"):
            torch.manual_seed(7)
            ctrl = _ctrl("mppi", nx, nu, dtype, K, T, route, tm, block_threads=64, threads_per_sample=1, **kw)
            ctrl.command(x)
            out.append((ctrl.U.clone(), ctrl.cost_total.clone(), ctrl.launch_info.grid_blocks))
        assert torch.equal(out[0][1], out[1][1])
        # the global-tile grid is capped (its tile slices stay bounded): at K = 131072 the records combine in another
        # order, so the update agrees to fp64 rounding instead of bit for bit
        if K <= 8192:
            assert torch.equal(out[0][0], out[1][0])
        else:
            assert torch.allclose(out[0][0], out[1][0], rtol=1e-12, atol=1e-13)
    m = shm.shape_model(nx, nu)
    f, c, _ = shm.twins(nx, nu)
    dyn, cost = (m.dynamics, m.running_cost) if route == "fused" else (f, c)
    states = torch.linspace(-0.4, 0.4, 3 * nx, dtype=dtype).reshape(3, nx).cuda()
    out = []
    for tm in ("shared", "global"):
        torch.manual_seed(7)            # the random initial nominal sequences
        b = eng.MPPI_Batched(dyn, cost, nx, _sigma(nu, dtype), 3, num_samples=2048, horizon=T, device="cuda",
                             u_max=torch.full((nu,), 1.2, dtype=dtype), rng_seed=5, block_threads=64, tile_memory=tm)
        b.command(states)
        assert b.launch_info.global_tile == (tm == "global")
        out.append((b.U.clone(), b.cost_total.clone()))
    # MPPI_Batched plans its own helper threads (the layouts differ, so may the geometry): the costs are the same
    # operations, the update agrees to fp64 rounding
    assert torch.equal(out[0][1], out[1][1])
    assert torch.allclose(out[0][0], out[1][0], rtol=1e-12, atol=1e-13)


# ---- 2. oracle parity past today's edge ---------------------------------------------------------------------------------
LONG = [(v, nx, nu, dt, T, S)
        for (nx, nu, dt, T) in ((8, 4, torch.float64, 512), (3, 3, torch.float32, 682), (1, 1, torch.float64, 2048))
        for (v, S) in (("mppi", None), ("smppi", None), ("kmppi", T // 2), ("kmppi", 8))]


def _oracle(variant, prob, U, A, theta, x, z, T, S, dtype):
    if variant == "mppi":
        return orc.mppi_command(prob, U, x, z)
    if variant == "smppi":
        return orc.smppi_command(prob, orc.SmoothParams(w_action_seq_cost=2.0, delta_t=0.5), U, A, x, z)
    W, Wshift = orc.kernel_matrices(T, S, lambda a, b: orc.rbf_kernel(a, b, 2.0), dtype)
    return orc.kmppi_command(prob, U, theta, x, z, W, Wshift)


@pytest.mark.parametrize("route", ["fused", "stepped"])
@pytest.mark.parametrize("case", LONG, ids=lambda c: f"{c[0]}_n{c[1]}u{c[2]}_T{c[4]}_S{c[5]}_{str(c[3])[-7:]}")
def test_long_horizon_matches_the_oracle(case, route):
    variant, nx, nu, dtype, T, S = case
    K = 2048
    f, c_, t_ = shm.twins(nx, nu)
    prob = orc.Problem(f, c_, nx, _sigma(nu, dtype), K=K, T=T, u_max=torch.full((nu,), 1.2, dtype=dtype), terminal_state_cost=t_)
    x = torch.linspace(-0.5, 0.5, nx, dtype=dtype)
    ctrl = _ctrl(variant, nx, nu, dtype, K, T, route, "auto", S=S)
    tol = 1e-9 if dtype == torch.float64 else 2e-5
    err = 0.0
    for i in range(3):
        z = _z(K, S or T, nu, dtype, 40 + i)
        U_in = ctrl.U.cpu().clone()
        A_in = ctrl.action_sequence.cpu().clone() if variant == "smppi" else None
        th_in = ctrl.theta.cpu().clone() if variant == "kmppi" else None
        ctrl.inject_noise(z)
        ctrl.command(x)
        assert ctrl.launch_info.global_tile == 1
        r = _oracle(variant, prob, U_in, A_in, th_in, x, z, T, S, dtype)
        err = max(err, float((ctrl.U.cpu() - r["U"]).abs().max()))
    reports.write(f"long_horizon_{variant}_n{nx}u{nu}_T{T}_S{S}_{route}.txt", f"{err}\n")
    assert err <= tol, err


def test_long_horizon_intermediates_rollouts_and_batched():
    """At (8,4) T = 512 fp64: the on-demand noise / perturbed_action / omega / states through the global-tile sampling
    kernel, get_rollouts, and a 3-environment MPPI_Batched against the oracle."""
    nx, nu, dtype, T, K = 8, 4, torch.float64, 512, 2048
    f, c_, t_ = shm.twins(nx, nu)
    prob = orc.Problem(f, c_, nx, _sigma(nu, dtype), K=K, T=T, u_max=torch.full((nu,), 1.2, dtype=dtype), terminal_state_cost=t_)
    x = torch.linspace(-0.5, 0.5, nx, dtype=dtype)
    ctrl = _ctrl("mppi", nx, nu, dtype, K, T, "fused", "global")
    z = _z(K, T, nu, dtype, 9)
    U_in = ctrl.U.cpu().clone()
    ctrl.inject_noise(z)
    ctrl.command(x)
    U_sh = orc.shift_rows(U_in, torch.zeros(nu, dtype=dtype))
    noise = z @ torch.linalg.cholesky(_sigma(nu, dtype)).T
    pa = torch.clamp(U_sh + noise, -1.2, 1.2)
    assert float((ctrl.perturbed_action.cpu() - pa).abs().max()) <= 1e-12
    assert float((ctrl.noise.cpu() - (pa - U_sh)).abs().max()) <= 1e-12
    costs = ctrl.cost_total.cpu()
    w = torch.exp(-(costs - costs.min()) / 1.0)
    assert float((ctrl.omega.cpu() - w / w.sum()).abs().max()) <= 1e-9
    st = ctrl.states
    assert st.shape == (1, K, T, nx)
    # the (8,4) model's states grow to ~1e8 over 512 steps: relative agreement
    _, ref_states, _ = orc.rollout(prob, x, pa[:4])
    assert torch.allclose(st[0, :4].cpu(), ref_states[0], rtol=1e-12, atol=1e-12)
    U_now = ctrl.U.cpu()
    roll = ctrl.get_rollouts(x, num_rollouts=2)
    _, ref_roll, _ = orc.rollout(prob, x, U_now.unsqueeze(0).expand(2, -1, -1))
    assert roll.shape == (2, T, nx)
    assert torch.allclose(roll.cpu(), ref_roll[0], rtol=1e-12, atol=1e-12)

    states = torch.linspace(-0.4, 0.4, 3 * nx, dtype=dtype).reshape(3, nx)
    m = shm.shape_model(nx, nu)
    b = eng.MPPI_Batched(m.dynamics, m.running_cost, nx, _sigma(nu, dtype), 3, num_samples=K, horizon=T, device="cuda",
                         u_max=torch.full((nu,), 1.2, dtype=dtype), tile_memory="auto")
    U3 = b.U.cpu().clone()
    zb = _z(K, T, nu, dtype, 10)
    b.inject_noise(zb)
    b.command(states.cuda())
    assert b.launch_info.global_tile == 1
    prob_b = orc.Problem(f, c_, nx, _sigma(nu, dtype), K=K, T=T, u_max=torch.full((nu,), 1.2, dtype=dtype))
    r = orc.mppi_batched_command(prob_b, U3, states, zb)
    assert float((b.U.cpu() - r["U"]).abs().max()) <= 1e-9


# ---- 3. "auto" ----------------------------------------------------------------------------------------------------------
def _plans(T, tm):
    try:
        c = _ctrl("mppi", 8, 4, torch.float64, 2048, T, "fused", tm)
        c._pack()
        return c.launch_info.global_tile
    except MppiLibraryError as e:
        assert "shared-memory" in str(e) or "global-tile" in str(e), e
        return None


def test_auto_keeps_shared_plans_and_crosses_the_edge():
    lo, hi = 8, 1024
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if _plans(mid, "shared") is not None else (lo, mid)
    t_shared = lo
    assert _plans(t_shared, "auto") == 0 and _plans(t_shared + 1, "auto") == 1
    lo, hi = 512, 4096
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if _plans(mid, "auto") is not None else (lo, mid)
    reports.write("long_horizon_auto.json", json.dumps({"mppi_f64_n8u4_K2048": {"shared_T_max": t_shared, "auto_T_max": lo}}))
    assert lo >= 512
    # bench shapes plan unchanged and compute the same under "auto"
    pend = eng.Pendulum()
    outs = []
    for tm in ("shared", "auto"):
        torch.manual_seed(1)
        c = eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), num_samples=16384, horizon=30,
                     u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda", rng_seed=1, tile_memory=tm)
        c.command([3.14159, 1.0])
        outs.append((c.U.clone(), c.cost_total.clone(), c.launch_info.global_tile, c.launch_info.grid_blocks))
    assert outs[1][2] == 0 and outs[0][3] == outs[1][3]
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    # change_horizon across the edge
    c = _ctrl("smppi", 8, 4, torch.float64, 2048, 30, "fused", "auto")
    c.command(torch.zeros(8, dtype=torch.float64))
    assert c.launch_info.global_tile == 0
    c.change_horizon(512)
    c.command(torch.zeros(8, dtype=torch.float64))
    assert c.launch_info.global_tile == 1 and c.U.shape == (512, 4) and torch.isfinite(c.U).all()


# ---- 4. refusals ---------------------------------------------------------------------------------------------------------
def test_refusals():
    c = _ctrl("mppi", 3, 3, torch.float32, 2048, 24, "fused", "global")
    c.command(torch.zeros(3))
    with pytest.raises(MppiLibraryError, match="resident mode keeps its tiles in shared memory"):
        c.start_resident()
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(3, 32), torch.nn.Tanh(), torch.nn.Linear(32, 32), torch.nn.Tanh(),
                              torch.nn.Linear(32, 2)).double()
    pend = eng.PendulumMLP(net)
    for tm_ in ("global", "auto"):
        with pytest.raises(ValueError, match="PendulumMLP"):
            eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(1.0, dtype=torch.float64), num_samples=256, horizon=20,
                     device="cuda", tile_memory=tm_)
    with pytest.raises(ValueError, match="sharded"):
        eng.MPPI(lambda s, a: s, lambda s, a: s[:, 0], 2, torch.eye(2), num_samples=256, horizon=20, device="cuda",
                 process_group=object(), tile_memory="auto")
    beyond = _ctrl("mppi", 8, 4, torch.float64, 2048, 4096, "fused", "auto")
    U_before = beyond.U.clone()
    with pytest.raises(MppiLibraryError, match="global-tile plan"):
        beyond.command(torch.zeros(8, dtype=torch.float64))
    assert torch.equal(beyond.U, U_before) and beyond.cost_total is None


# ---- 5. the stepped route's "auto", and the other model kinds on the global tile ------------------------------------------
def test_stepped_auto_keeps_shared_plans():
    """A controller of torch callables: "auto" plans the shared-memory sampling / softmin kernels at a short horizon
    (identical results) and the global-tile ones past the edge; change_horizon re-decides."""
    x = torch.linspace(-0.5, 0.5, 8, dtype=torch.float64)
    outs = []
    for tm_ in ("shared", "auto"):
        c = _ctrl("smppi", 8, 4, torch.float64, 2048, 24, "stepped", tm_, rng_seed=4)
        c.command(x)
        outs.append((c.launch_info.global_tile, c.U.clone(), c.cost_total.clone()))
    assert outs[1][0] == 0
    assert torch.equal(outs[0][1], outs[1][1]) and torch.equal(outs[0][2], outs[1][2])
    c.change_horizon(512)
    c.command(x)
    assert c.launch_info.global_tile == 1 and torch.isfinite(c.U).all()
    c.change_horizon(24)
    c.command(x)
    assert c.launch_info.global_tile == 0
    b = eng.MPPI_Batched(lambda s_, a: shm.twins(8, 4)[0](s_, a), lambda s_, a: shm.twins(8, 4)[1](s_, a), 8,
                         _sigma(4, torch.float64), 2, num_samples=1024, horizon=24, device="cuda", tile_memory="auto")
    b.command(torch.zeros(2, 8, dtype=torch.float64, device="cuda"))
    assert b.launch_info.global_tile == 0


def _pair(make, cls, dtype, T, **kw):
    """(shared, global) results of two controllers made by `make()` over 3 shifted commands with injected noise at a pinned
    geometry: every output list."""
    res = []
    for tm_ in ("shared", "global"):
        m, x, nx, nu, extra = make()
        if getattr(m, "has_terminal", False) and "terminal_state_cost" not in extra:
            extra = dict(extra, terminal_state_cost=m.terminal_cost)
        rows = kw.get("num_support_pts", T)
        torch.manual_seed(0)            # the random initial nominal sequence
        c = cls(m.dynamics, m.running_cost, nx, torch.eye(nu, dtype=dtype) * 0.5, num_samples=2048, horizon=T, device="cuda",
                u_max=torch.full((nu,), 2.0, dtype=dtype), block_threads=64, threads_per_sample=1, rng_seed=2,
                tile_memory=tm_, **extra, **kw)
        assert c._model is m
        out = []
        for i in range(3):
            c.inject_noise(_z(2048, rows, nu, dtype, 60 + i))
            out += [c.command(x).clone(), c.cost_total.clone()] + _seq(c)
        assert c.launch_info.global_tile == (tm_ == "global")
        res.append(out)
    for a, b in zip(*res):
        assert torch.equal(a, b)


def test_global_tile_other_models_bit_identical(monkeypatch):
    """copies = 3 (copies_rollout), a step-dependent model, a model reading device tensors, and the registered
    (nvcc-compiled) Pendulum and LinearPoint kernels: "global" against "shared" at a pinned geometry."""
    monkeypatch.setenv("MPPI_B200_CLUSTER", "1")
    T, f64 = 24, torch.float64
    _pair(lambda: (em.pendulum_ensemble(3, 2048), [0.5, 0.1], 2, 1,
                   dict(rollout_samples=3, rollout_var_cost=0.2, rollout_var_discount=0.9)), eng.MPPI, f64, T)
    _pair(lambda: (sm.step_dependent_user_model(), [0.2, -0.1], 2, 1, dict(step_dependent_dynamics=True)), eng.SMPPI, f64, T,
          w_action_seq_cost=0.5, delta_t=0.5)
    _pair(lambda: (tm.nav_model(tm.make_costmap(torch.float32), tm.make_path(T)), [-1.0, -1.0], 2, 2,
                   dict(step_dependent_dynamics=True)), eng.KMPPI, f64, T, num_support_pts=6, kernel=eng.RBFKernel(sigma=2.0))
    pend = eng.Pendulum()
    _pair(lambda: (pend, [3.0, 0.5], 2, 1, {}), eng.MPPI, f64, T)
    nav = eng.LinearPoint.toy2d_nav()
    _pair(lambda: (nav, [-3.0, -2.0], 2, 2, dict(terminal_state_cost=nav.terminal_cost)), eng.KMPPI, torch.float32, T,
          num_support_pts=5, kernel=eng.RBFKernel(sigma=2.0))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_registered_model_long_horizon_bit_identical(dtype, monkeypatch):
    """The registered Pendulum's nvcc-compiled global-tile kernel at T = 600, near the shared-memory edge of its
    32-sample tiles, against the shared-memory kernel at the same geometry: 3 shifted commands, injected noise."""
    monkeypatch.setenv("MPPI_B200_CLUSTER", "1")
    pend = eng.Pendulum()
    T, K = 600, 2048
    outs = []
    for tm_ in ("shared", "global"):
        c = eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(1.0, dtype=dtype), num_samples=K, horizon=T,
                     device="cuda", U_init=torch.zeros(T, 1, dtype=dtype), u_min=torch.tensor(-2.0, dtype=dtype),
                     u_max=torch.tensor(2.0, dtype=dtype), block_threads=32, threads_per_sample=2, tile_memory=tm_)
        assert c._model is pend
        out = []
        for i in range(3):
            c.inject_noise(_z(K, T, 1, dtype, 80 + i))
            out += [c.command([3.0, 0.5]).clone(), c.cost_total.clone(), c.U.clone()]
        info = c.launch_info
        assert info.global_tile == (tm_ == "global") and (info.block_threads, info.threads_per_sample) == (64, 2)
        outs.append(out)
    for a, b in zip(*outs):
        assert torch.equal(a, b)
