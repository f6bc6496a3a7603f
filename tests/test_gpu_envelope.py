"""GPU: the fused command across its model envelope.

  - resident mode, get_rollouts and the in-kernel draws at the (1,1), (3,3) and (8,4) models of tests/shape_models.py
    (their live-reference fixtures, tests/golden/shape_cases.py, and the split-cost rollout against the single loop on
    them are replayed in tests/test_gpu_golden_replay.py);
  - the softmin tail in each of its forms (one CTA; one cluster record; LL and ticket exchange of cluster records; cluster
    sizes 8/4/2/1; one wave, two CTAs per SM, grid-stride multi-pass; 32-sample tiles; ragged K), each run first asserting
    from launch_info that it got the geometry it was written for, then compared with the fp64 oracle at 1e-10;
  - cost edge cases of the softmin: all costs equal, one sample far cheaper than the rest, +inf costs, costs near 1e6;
  - the shared-memory edge of the planner: the largest horizon it accepts, a command there, and the error beyond it.

Measured worst errors go to tests/_reports/envelope_errors.json.
"""
import itertools
import json

import numpy as np
import pytest
import torch

import pytorch_mppi_b200 as eng
from oracle import mppi_oracle as orc
from pytorch_mppi_b200._cabi import MppiLibraryError
from tests import reports
from tests import shape_models as shm
from tests.golden.shape_cases import SIG3

pytestmark = pytest.mark.gpu


def _record(key, err):
    reports.worst("envelope_errors.json", key, err)


# ---- B: resident mode, get_rollouts and the draws at the new shapes ---------------------------------------------------
def _shape_ctrl(nx, nu, K, T, dtype, **kw):
    m = shm.shape_model(nx, nu)
    sigma = torch.tensor(SIG3 if nu == 3 else np.eye(nu) * 0.7 + 0.1, dtype=dtype)
    c = eng.MPPI(m.dynamics, m.running_cost, nx, sigma, num_samples=K, horizon=T, terminal_state_cost=m.terminal_cost,
                 u_max=torch.full((nu,), 1.2, dtype=dtype), device="cuda", **kw)
    assert c._model is m
    return c, m


@pytest.mark.parametrize("nx,nu,dtype", [(3, 3, torch.float32), (8, 4, torch.float64)])
def test_shape_resident_equals_launch_route(nx, nu, dtype):
    """command_host() under resident() is bit-identical to the launch route at nu = 3..4 and nx = 8."""
    K, T = 4096, 13
    res, _ = _shape_ctrl(nx, nu, K, T, dtype, U_init=torch.zeros(T, nu, dtype=dtype), rng_seed=21)
    ref, _ = _shape_ctrl(nx, nu, K, T, dtype, U_init=torch.zeros(T, nu, dtype=dtype), rng_seed=21)
    with res.resident(idle_us=200000):
        for step in range(4):
            x = [0.1 * (i + 1) * (-1) ** (i + step) for i in range(nx)]
            a, b = res.command_host(x), ref.command_host(x)
            assert torch.equal(a, b), step
            assert torch.equal(res.U, ref.U) and torch.equal(res.cost_total, ref.cost_total)
        assert res.resident_launches >= 1
    assert res.launch_info.split_cost == 1


def test_shape_get_rollouts_nx8():
    T = 13
    c, m = _shape_ctrl(8, 4, 512, T, torch.float64, U_init=torch.randn(T, 4, dtype=torch.float64), u_scale=1.3)
    x0 = torch.randn(3, 8, dtype=torch.float64, generator=torch.Generator().manual_seed(6)).cuda()
    got = c.get_rollouts(x0, num_rollouts=3)
    s, out = x0, []
    for t in range(T):
        s = m.dynamics(s, 1.3 * c.U[t].expand(3, -1))
        out.append(s)
    assert got.shape == (3, T, 8)
    assert float((got - torch.stack(out, dim=1)).abs().max()) <= 1e-12


@pytest.mark.parametrize("route", ["fused", "stepped"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_philox_draws_at_odd_rows(dtype, route):
    """nu = 3, T = 7: R = 21 normals per sample, not a multiple of the 4 (fp32) or 2 (fp64) normals of one Philox call,
    so a call straddles two time steps; the normals a command used equal the numpy statement of the stream, and the
    oracle fed them reproduces the command."""
    from oracle import philox_oracle as po
    K, T, nu, seed = 1000, 7, 3, 0xBADC0FFEE
    m = shm.shape_model(3, 3)
    f, cst, term = shm.twins(3, 3)
    sigma = torch.tensor(SIG3, dtype=dtype)
    dyn, rc, tc = (m.dynamics, m.running_cost, m.terminal_cost) if route == "fused" else (
        (lambda s, a: f(s, a)), (lambda s, a: cst(s, a)), (lambda s, a: term(s, a)))
    U0 = torch.randn(T, nu, dtype=dtype, generator=torch.Generator().manual_seed(3)) * 0.3
    c = eng.MPPI(dyn, rc, 3, sigma, num_samples=K, horizon=T, U_init=U0.clone(), terminal_state_cost=tc, device="cuda",
                 rng_seed=seed)
    assert (c._model is not None) == (route == "fused")
    c.record_noise(True)
    prob = orc.Problem(f, cst, 3, sigma, K=K, T=T, terminal_state_cost=term)
    np_dt = np.float32 if dtype == torch.float32 else np.float64
    per = 4 if dtype == torch.float32 else 2
    x = torch.tensor([0.3, -0.2, 0.1], dtype=dtype)
    offset, U = 0, U0.clone()
    for _ in range(2):
        c.command(x)
        z_used = c.z_used.cpu().numpy().reshape(K, T * nu)
        z_orc = po.normals(seed, offset, 0, K, T * nu, np_dt)
        offset += (T * nu + per - 1) // per
        np.testing.assert_allclose(z_used, z_orc, atol=2e-5 if dtype == torch.float32 else 1e-12, rtol=0)
        r = orc.mppi_command(prob, U, x, torch.from_numpy(z_used).reshape(K, T, nu))
        tol = 1e-5 if dtype == torch.float32 else 1e-10
        err = float((c.U.cpu() - r["U"]).abs().max())
        _record(f"philox_odd_rows/{route}/{dtype}", err)
        assert err <= tol
        U = c.U.cpu().clone()


# ---- C: the softmin tail, every geometry --------------------------------------------------------------------------
LL_STAGE_BYTES = 49152          # MPPI_LL_STAGE_BYTES: LL mode stages (clusters x (R+2)) doubles at most


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


# (name, K, samples per tile, threads per sample (0: automatic), [(MPPI_B200_CLUSTER, MPPI_B200_XCHG_DIRECT,
#  MPPI_B200_SPLIT_COST)], what the geometry must be)
def _geometries(sm):
    full = list(itertools.product((8, 4, 2, 1), (1, 0), (1, 0)))
    return [
        ("one_cta_k1", 1, 32, 0, [(8, 1, 1), (1, 0, 0)], dict(grid=1)),
        ("one_cta_k31", 31, 32, 0, [(8, 1, 1), (2, 0, 0)], dict(grid=1)),
        ("one_cluster_k33", 33, 32, 0, [(2, 1, 1), (2, 0, 0)], dict(grid=2, cluster=2)),
        ("two_records_k33", 33, 32, 0, [(1, 1, 1), (1, 0, 1)], dict(grid=2, cluster=1)),
        ("cluster_wave", 16 * 64 - 5, 64, 4, full, dict(grid=16, cluster="env")),
        ("cluster_wave_32", 16 * 64 - 5, 32, 2, [(8, 1, 1), (8, 0, 0), (2, 0, 1)], dict(grid=32, cluster="env")),
        ("two_per_sm", 2 * sm * 64 - 1, 64, 1, [(2, 1, 0), (1, 1, 0), (1, 0, 0)], dict(grid=2 * sm)),
        ("tiles_sm_minus_1", sm * 64 - 1, 64, 1, [(8, 1, 0), (1, 0, 0)], dict(grid=sm)),
        ("tiles_sm_plus_1", sm * 64 + 1, 64, 1, [(8, 1, 0), (1, 0, 0)], dict(single_wave=True)),
        # one thread per sample asked for: 32-sample tiles still run two (a CTA has at least two warps)
        ("multipass_32", 2 * 16 * sm * 32 + 33, 32, 1, [(2, 1, 0), (1, 1, 0), (1, 0, 0)], dict(multipass=True)),
    ]


def _tail_of(info, K, bs, env, R, want):
    """Assert the geometry a run was written for; return (tail mode, cluster size, passes > 1)."""
    cl, direct, split = env
    assert info.block_threads // info.threads_per_sample == bs and info.block_threads >= 64
    n_tiles = -(-K // bs)
    grid, cs, rec = info.grid_blocks, info.cluster_size, info.xchg_records
    assert 1 <= cs <= cl and grid % cs == 0, (cs, cl, grid)
    nc = grid // cs
    if nc == 1:
        mode = "one"
        assert rec == 1
    elif direct and nc * (R + 2) * 8 <= LL_STAGE_BYTES:
        mode = "ll"
        assert rec == nc
    else:
        mode = "ticket"
        assert rec == 1
    assert info.split_cost == (1 if split and info.threads_per_sample > 1 else 0)
    if "grid" in want:
        assert grid == want["grid"], (grid, want)
    if want.get("cluster") == "env":
        assert cs == cl
    elif "cluster" in want:
        assert cs == want["cluster"]
    if want.get("single_wave"):
        assert n_tiles <= grid
    if want.get("multipass"):
        assert n_tiles > grid
    return mode, cs, n_tiles > grid


def _tail_model(kind, dtype, bounded=True):
    """(engine model, nx, nu, sigma, u_max, oracle problem factory) of the tail tests."""
    if not bounded:         # the linear point without action bounds
        m, nx, nu, sigma, _, _ = _tail_model(kind, dtype)
        olin = orc.LinearPointModel(B=m.B, goal=m.goal, dtype=dtype)
        return m, nx, nu, sigma, None, lambda K, T, lam: orc.Problem(olin.dynamics, olin.running_cost, 2, sigma, K=K, T=T,
                                                                    lambda_=lam)
    if kind == "shape":
        m = shm.shape_model(3, 3)
        f, c, t = shm.twins(3, 3)
        sigma, umax = torch.tensor(SIG3, dtype=dtype), torch.tensor([1.0, 0.8, 1.2], dtype=dtype)
        return m, 3, 3, sigma, umax, lambda K, T, lam: orc.Problem(f, c, 3, sigma, K=K, T=T, lambda_=lam, u_max=umax,
                                                                  terminal_state_cost=t)
    m = eng.LinearPoint.unit_test_env()
    olin = orc.LinearPointModel(B=m.B, goal=m.goal, dtype=dtype)
    sigma, umax = torch.tensor([[0.8, 0.1], [0.1, 0.6]], dtype=dtype), torch.tensor([0.9, 0.7], dtype=dtype)
    return m, 2, 2, sigma, umax, lambda K, T, lam: orc.Problem(olin.dynamics, olin.running_cost, 2, sigma, K=K, T=T,
                                                              lambda_=lam, u_max=umax)


def _tail_ctrl(monkeypatch, kind, dtype, K, T, bs, tps, env, U0, lam=1.0, model=None, bounded=True):
    cl, direct, split = env
    monkeypatch.setenv("MPPI_B200_CLUSTER", str(cl))
    monkeypatch.setenv("MPPI_B200_XCHG_DIRECT", str(direct))
    monkeypatch.setenv("MPPI_B200_SPLIT_COST", str(split))
    m, nx, nu, sigma, umax, _ = _tail_model(kind, dtype, bounded)
    m = model or m
    c = eng.MPPI(m.dynamics, m.running_cost, nx, sigma, num_samples=K, horizon=T, lambda_=lam, U_init=U0.clone(), u_max=umax,
                 terminal_state_cost=m.terminal_cost if m.has_terminal else None, device="cuda", block_threads=bs,
                 threads_per_sample=tps)
    assert c._model is m
    return c


@pytest.mark.parametrize("kind", ["linear", "shape"])
def test_tail_geometry_matrix_fp64(kind, monkeypatch):
    """Every geometry x tail mode against the fp64 oracle at 1e-10 (U, action, cost_total, omega); together the runs
    reach one CTA, one cluster record, LL and ticket exchange, cluster sizes 8/4/2/1, both rollout kernels, two CTAs per
    SM and grid-stride multi-pass."""
    dtype, T = torch.float64, 6
    sm = _sm_count()
    *_, problem = _tail_model(kind, dtype)
    nu = 3 if kind == "shape" else 2
    R = T * nu
    seen = set()
    x = torch.tensor([0.4, -0.3, 0.2][:nu], dtype=dtype)
    for name, K, bs, tps, envs, want in _geometries(sm):
        g = torch.Generator().manual_seed(K)
        U0 = torch.randn(T, nu, generator=g, dtype=dtype) * 0.3
        z = torch.randn(K, T, nu, generator=g, dtype=dtype)
        r = orc.mppi_command(problem(K, T, 1.0), U0, x, z)
        for env in envs:
            c = _tail_ctrl(monkeypatch, kind, dtype, K, T, bs, tps, env, U0)
            c.inject_noise(z)
            a = c.command(x)
            seen.add(_tail_of(c.launch_info, K, bs, env, R, want))
            err = float((c.U.cpu() - r["U"]).abs().max())
            _record(f"tail/{kind}/{name}/{env}", err)
            assert err <= 1e-10, (name, env, err)
            assert float((a.cpu() - r["action"]).abs().max()) <= 1e-10
            np.testing.assert_allclose(c.cost_total.cpu().numpy(), r["cost_total"].numpy(), rtol=1e-10, atol=0)
            np.testing.assert_allclose(c.omega.cpu().numpy(), r["omega"].numpy(), atol=1e-10, rtol=0)
            seen.add(("split", c.launch_info.split_cost, None))
    tails = [t for t in seen if t[0] != "split"]
    assert {t[0] for t in tails} == {"one", "ll", "ticket"}, seen
    assert {t[1] for t in tails} >= {8, 4, 2, 1}, seen
    assert any(t[2] for t in tails), seen
    assert {("split", 0, None), ("split", 1, None)} <= seen


@pytest.mark.parametrize("kind", ["linear", "shape"])
def test_tail_geometries_agree_fp32(kind, monkeypatch):
    """fp32: the same draws through every tail of one K (cluster sizes, LL / ticket, split / single loop, 64- and
    32-sample tiles) give the same plan within 5e-7 (the fp64 reduction runs in a geometry-dependent order)."""
    dtype, T, K = torch.float32, 9, 16 * 64 - 5
    nu = 3 if kind == "shape" else 2
    g = torch.Generator().manual_seed(11)
    U0 = torch.randn(T, nu, generator=g, dtype=dtype) * 0.3
    z = torch.randn(K, T, nu, generator=g, dtype=dtype)
    x = torch.tensor([0.4, -0.3, 0.2][:nu], dtype=dtype)
    outs = []
    for name, K_, bs, tps, envs, want in _geometries(_sm_count()):
        if K_ != K:
            continue
        for env in envs:
            c = _tail_ctrl(monkeypatch, kind, dtype, K, T, bs, tps, env, U0)
            c.inject_noise(z)
            a = c.command(x)
            _tail_of(c.launch_info, K, bs, env, T * nu, want)
            outs.append(((name, env), c.U.cpu().clone(), a.cpu().clone()))
    for tag, U, a in outs[1:]:
        err = float((U - outs[0][1]).abs().max())
        _record(f"tail_fp32_spread/{kind}", err)
        assert err <= 5e-7, (tag, err)
        assert float((a - outs[0][2]).abs().max()) <= 5e-7


_EDGE_GEOMETRIES = [("cluster_wave", (8, 1, 0)), ("cluster_wave", (1, 1, 0)), ("cluster_wave", (2, 0, 1)),
                    ("multipass_32", (1, 0, 0))]


def _edge_geometry(name):
    return next(gm for gm in _geometries(_sm_count()) if gm[0] == name)


@pytest.mark.parametrize("geom,env", _EDGE_GEOMETRIES)
@pytest.mark.parametrize("edge", ["equal", "one_cheap", "inf"])
def test_softmin_cost_edges_fp64(edge, geom, env, monkeypatch):
    """equal: every sample has the same cost (z = 0: eta = K, omega = 1/K, the plan only shifts); one_cheap: lambda so
    small that every other weight underflows (eta = 1); inf: whole tiles (so whole warp, CTA and cluster records) and
    scattered samples with cost +inf (a hard constraint: weight 0, mppi.py:256-258)."""
    dtype, T = torch.float64, 6
    _, K, bs, tps, _, want = _edge_geometry(geom)
    g = torch.Generator().manual_seed(31)
    U0 = torch.randn(T, 2, generator=g, dtype=dtype) * 0.3
    z = torch.randn(K, T, 2, generator=g, dtype=dtype)
    lam = 1.0
    if edge == "equal":
        z.zero_()
    elif edge == "one_cheap":
        lam = 1e-7
    else:
        z[: 8 * bs] = 1e200                 # the linear point's quadratic cost overflows to +inf, never to -inf
        z[torch.randperm(K, generator=g)[:K // 10]] = 1e200
    bounded = edge != "inf"                 # unbounded: the overflowing samples keep their huge actions
    *_, problem = _tail_model("linear", dtype, bounded)
    prob = problem(K, T, lam)
    x = torch.tensor([0.4, -0.3], dtype=dtype)
    c = _tail_ctrl(monkeypatch, "linear", dtype, K, T, bs, tps, env, U0, lam=lam, bounded=bounded)
    c.inject_noise(z)
    a = c.command(x)
    _tail_of(c.launch_info, K, bs, env, T * 2, want)
    r = orc.mppi_command(prob, U0, x, z)
    U = c.U.cpu()
    assert torch.isfinite(U).all() and torch.isfinite(c.omega.cpu()).all()
    err = float((U - r["U"]).abs().max())
    _record(f"cost_edge/{edge}/{geom}/{env}", err)
    assert err <= 1e-10, err
    assert float((a.cpu() - r["action"]).abs().max()) <= 1e-10
    np.testing.assert_allclose(c.omega.cpu().numpy(), r["omega"].numpy(), atol=1e-10, rtol=0)
    if edge == "equal":
        assert float(c.eta) == K and float(r["eta"]) == K
        assert torch.equal(U, r["U_before"])
    elif edge == "one_cheap":
        assert float(c.eta) == 1.0 and float(r["eta"]) == 1.0
    else:
        cost = c.cost_total.cpu()
        assert torch.equal(torch.isinf(cost), torch.isinf(r["cost_total"])) and int(torch.isinf(cost).sum()) >= 8 * bs
        assert float(c.omega.cpu()[torch.isinf(cost)].abs().max()) == 0.0


@pytest.mark.parametrize("geom,env", _EDGE_GEOMETRIES)
def test_softmin_costs_near_1e6_fp32(geom, env, monkeypatch):
    """fp32 costs of ~5e6 (a goal 600 away): the kernel subtracts beta before the exponent, so the update equals the
    fp64 softmin of its own costs; the costs themselves are the fp64 oracle's to fp32 rounding."""
    T = 7
    _, K, bs, tps, _, want = _edge_geometry(geom)
    far = eng.LinearPoint(B=[[1.0, 0.0], [0.0, -1.0]], goal=[600.0, -600.0])
    g = torch.Generator().manual_seed(41)
    U0 = torch.randn(T, 2, generator=g) * 0.3
    z = torch.randn(K, T, 2, generator=g)
    lam = 2000.0
    c = _tail_ctrl(monkeypatch, "linear", torch.float32, K, T, bs, tps, env, U0, lam=lam, model=far)
    c.inject_noise(z)
    x = torch.tensor([0.4, -0.3])
    c.command(x)
    _tail_of(c.launch_info, K, bs, env, T * 2, want)
    cost = c.cost_total.cpu().double()
    assert float(cost.min()) > 1e6
    olin = orc.LinearPointModel(B=far.B, goal=far.goal, dtype=torch.float64)
    sig = torch.tensor([[0.8, 0.1], [0.1, 0.6]], dtype=torch.float64)
    r = orc.mppi_command(orc.Problem(olin.dynamics, olin.running_cost, 2, sig, K=K, T=T, lambda_=lam,
                                     u_max=torch.tensor([0.9, 0.7], dtype=torch.float64)), U0.double(), x.double(), z.double())
    np.testing.assert_allclose(cost.numpy(), r["cost_total"].numpy(), rtol=2e-6, atol=0)
    # the softmin of the engine's own fp32 costs and noise, in fp64
    w = torch.exp(-(cost - cost.min()) / lam)
    U_want = c.noise.cpu().double().mul(w.view(-1, 1, 1) / w.sum()).sum(0) + r["U_before"]
    err = float((c.U.cpu().double() - U_want).abs().max())
    _record(f"cost_1e6_fp32/{geom}/{env}", err)
    assert err <= 2e-6, err


# ---- D: the shared-memory edge ----------------------------------------------------------------------------------------
# (controller class, dtype, (nx, nu), kwargs of a horizon T)
_EDGE = {
    "mppi_f64_nu4": (eng.MPPI, torch.float64, (8, 4), lambda T: {}),
    "smppi_f64_nu4": (eng.SMPPI, torch.float64, (8, 4), lambda T: dict(w_action_seq_cost=2.0, delta_t=0.5)),
    "kmppi_f64_nu4": (eng.KMPPI, torch.float64, (8, 4), lambda T: dict(num_support_pts=max(2, T // 2),
                                                                         kernel=eng.RBFKernel(sigma=2.0))),
    "mppi_f32_nu3": (eng.MPPI, torch.float32, (3, 3), lambda T: {}),
}
EDGE_K = 2048


def _edge_ctrl(key, T, route="fused"):
    cls, dtype, (nx, nu), kw = _EDGE[key]
    m = shm.shape_model(nx, nu)
    f, c, t = shm.twins(nx, nu)
    dyn, cost, term = (m.dynamics, m.running_cost, m.terminal_cost) if route == "fused" else (
        (lambda s, a: f(s, a)), (lambda s, a: c(s, a)), (lambda s, a: t(s, a)))
    sigma = torch.tensor(SIG3 if nu == 3 else np.eye(nu) * 0.7 + 0.1, dtype=dtype)
    U0 = None if cls is eng.SMPPI else torch.randn(T, nu, dtype=dtype, generator=torch.Generator().manual_seed(T)) * 0.3
    ctrl = cls(dyn, cost, nx, sigma, num_samples=EDGE_K, horizon=T, U_init=U0, terminal_state_cost=term,
               u_max=torch.full((nu,), 1.2, dtype=dtype), device="cuda", **kw(T))
    assert (ctrl._model is m) == (route == "fused")
    return ctrl


def _plans(key, T):
    """Whether the fused route plans a command of horizon T (mppi_fused_query + mppi_plan_create; nothing launched)."""
    try:
        _edge_ctrl(key, T)._pack()
        return True
    except MppiLibraryError as e:
        assert "shared-memory" in str(e), e
        return False


def _largest_horizon(key):
    lo, hi = 8, 1024
    assert _plans(key, lo) and not _plans(key, hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if _plans(key, mid) else (lo, mid)
    return lo


@pytest.mark.parametrize("key", sorted(_EDGE))
def test_shared_memory_edge(key):
    """The largest horizon the planner accepts at K = 2048 runs on 32-sample tiles (no larger tile fits there) and
    matches the fp64 oracle on both routes; one step beyond, the first command raises MppiLibraryError naming shared
    memory before anything is launched."""
    T = _largest_horizon(key)
    reports_key = f"smem_edge/{key}"
    _record(reports_key + "/T_max", T)
    cls, dtype, (nx, nu), kw = _EDGE[key]
    f, c_, t_ = shm.twins(nx, nu)
    sigma = torch.tensor(SIG3 if nu == 3 else np.eye(nu) * 0.7 + 0.1, dtype=dtype)
    prob = orc.Problem(f, c_, nx, sigma, K=EDGE_K, T=T, u_max=torch.full((nu,), 1.2, dtype=dtype), terminal_state_cost=t_)
    g = torch.Generator().manual_seed(5)
    x = torch.linspace(-0.5, 0.5, nx, dtype=dtype)
    S = kw(T).get("num_support_pts")
    z = torch.randn(EDGE_K, S or T, nu, generator=g, dtype=dtype)
    tol = 1e-9 if dtype == torch.float64 else 2e-5
    for route in ("fused", "stepped"):
        ctrl = _edge_ctrl(key, T, route)
        U_in = ctrl.U.cpu().clone()
        ctrl.inject_noise(z)
        ctrl.command(x)
        if route == "fused":
            info = ctrl.launch_info
            assert info.block_threads // info.threads_per_sample == 32, (T, info.block_threads, info.threads_per_sample)
        if cls is eng.MPPI:
            r = orc.mppi_command(prob, U_in, x, z)
        elif cls is eng.SMPPI:
            sp = orc.SmoothParams(w_action_seq_cost=2.0, delta_t=0.5)
            r = orc.smppi_command(prob, sp, U_in, torch.zeros(T, nu, dtype=dtype), x, z)
        else:
            W, Wshift = orc.kernel_matrices(T, S, lambda a, b: orc.rbf_kernel(a, b, 2.0), dtype)
            r = orc.kmppi_command(prob, U_in, torch.zeros(S, nu, dtype=dtype), x, z, W, Wshift)
        err = float((ctrl.U.cpu() - r["U"]).abs().max())
        _record(f"{reports_key}/{route}", err)
        assert err <= tol, (route, T, err)
    beyond = _edge_ctrl(key, T + 1)
    U_before = beyond.U.clone()
    with pytest.raises(MppiLibraryError, match="shared-memory"):
        beyond.command(x)
    assert torch.equal(beyond.U, U_before) and beyond.cost_total is None


def test_bench_workload_geometries_keep_their_tiles():
    """The 32-sample fallback of the automatic search is taken only where no larger tile fits: the analytic bench.py
    workload shapes still plan tiles of 64 samples or more (the MLP workload's tensor-core kernel fixes its own
    128-sample tile)."""
    import math
    pend = eng.Pendulum()
    nav = eng.LinearPoint.toy2d_nav()
    out = {}
    for name, ctrl in (
            ("pendulum_c2", eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), num_samples=16384, horizon=30,
                                     u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda")),
            ("nav2d_c3", eng.KMPPI(nav.dynamics, nav.running_cost, 2, torch.eye(2), num_samples=8192, horizon=40,
                                   terminal_state_cost=nav.terminal_cost, u_max=torch.tensor([1.0, 1.0]), num_support_pts=5,
                                   kernel=eng.RBFKernel(sigma=2.0), device="cuda")),
            ("pendulum_c5", eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), num_samples=131072, horizon=50,
                                     u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda"))):
        ctrl.command([math.pi, 1.0] if "pend" in name else [-3.0, -2.0])
        i = ctrl.launch_info
        out[name] = dict(block_threads=i.block_threads, threads_per_sample=i.threads_per_sample, grid=i.grid_blocks,
                         cluster=i.cluster_size, records=i.xchg_records, split=i.split_cost, smem=i.smem_bytes)
        assert i.block_threads // i.threads_per_sample >= 64, (name, out[name])
    reports.write("bench_geometries.json", json.dumps(out, indent=1, sort_keys=True))
