"""GPU: every `MPPI_Batched` environment against the fp64 oracle on the batched fused kernels, with per-environment model
parameters, temperatures, noise and horizons (set_env_params / set_env_horizon).

The reference of environment e is the oracle's single-environment command with T = h_e and e's goal, lambda, Sigma and
mu on the first h_e rows of the shared standard normals, chained on its own nominal sequence from command to command:
  - the softmin tail in each of its forms with N > 1 (one CTA, one cluster, cluster sizes 8..1 at N = 2..3, LL and
    ticket exchange, one wave, grid-stride multi-pass, the global tile, and the N = 16, K = 16384, T = 30 shape of
    BASELINE config 2, whose N grids span more than one wave), each run first asserting from launch_info the geometry it
    was written for; the environments' lambdas span 1e-3 .. 1e3, so their beta and eta differ by orders of magnitude;
  - the controller options on the per-environment kernel (u_per_command = 2, noise_abs_cost, u_init, u_scale, asymmetric
    bounds, no shift, N = 2, a terminal cost in one environment's parameter block);
  - noise rows past an environment's horizon (+inf costs there must not reach it);
  - the in-kernel Philox draws at nu = 3 with mixed horizons, against the numpy statement of the stream;
  - a closed loop against a loop built from the oracle alone;
  - N = 1 and N = 64.

Measured worst errors and the launch geometry of each run go to tests/_reports/batched_envelope_errors.json.
"""
import json
import math

import numpy as np
import pytest
import torch

import pytorch_mppi_b200 as eng
from oracle import mppi_oracle as orc
from oracle import philox_oracle as po
from tests import reports
from tests import shape_models as shm
from tests import test_gpu_envelope as envl
from tests.golden.shape_cases import SIG3

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64, F32 = torch.float64, torch.float32

_MEASURED = {}
_LAUNCH = {}


def _record(key, err):
    _MEASURED[key] = max(_MEASURED.get(key, 0.0), float(err))
    reports.write("batched_envelope_errors.json",
                  json.dumps(dict(errors=_MEASURED, launch_info=_LAUNCH), indent=1, sort_keys=True))


def _record_launch(key, c):
    i = c.launch_info
    _LAUNCH[key] = dict(N=c.N, K=c.K, T=c.T, block_threads=i.block_threads, threads_per_sample=i.threads_per_sample,
                        grid=[i.grid_blocks, c.N], cluster_size=i.cluster_size, xchg_records=i.xchg_records,
                        global_tile=i.global_tile, max_blocks_per_sm=i.max_blocks_per_sm, sm_count=i.sm_count)


# ---- per-environment settings ----------------------------------------------------------------------------------------
SIGMAS = ([[0.8, 0.1], [0.1, 0.6]], [[0.5, 0.0], [0.0, 0.9]], [[1.2, -0.3], [-0.3, 0.4]], [[0.3, 0.0], [0.0, 0.3]],
          [[0.7, 0.2], [0.2, 0.5]])
B = [[1.0, 0.0], [0.0, -1.0]]
UMAX = [0.9, 0.7]


def _lin(goal, terminal_scale=0.0):
    return eng.LinearPoint(B=B, goal=goal, terminal_scale=terminal_scale)


def _settings(N, T, dtype, upc=1, lam_exp=(-3.0, 3.0)):
    """Environment e: lambda 10^(lam_exp[0] .. lam_exp[1]) log-spaced, its own goal, a diagonal or full Sigma, a
    non-zero mu, and a horizon from a pattern that includes 1 (u_per_command), T // 2 and T."""
    span = lam_exp[1] - lam_exp[0]
    lam = [10.0 ** (lam_exp[0] + span * e / max(1, N - 1)) for e in range(N)]
    goals = [[2.0 * math.cos(1.3 * e + 0.4), 2.0 * math.sin(1.3 * e + 0.4)] for e in range(N)]
    sig = torch.stack([torch.tensor(SIGMAS[e % len(SIGMAS)], dtype=dtype) for e in range(N)])
    mu = torch.tensor([[0.1 * math.sin(e + 1.0), -0.1 * math.cos(e + 1.0)] for e in range(N)], dtype=dtype)
    pattern = [T, 1, max(1, T // 2), T - 1, 2]
    H = [min(T, max(upc, pattern[e % len(pattern)])) for e in range(N)]
    return dict(lam=lam, goals=goals, sig=sig, mu=mu, H=H)


def _linear_batched(N, K, T, dtype, st, *, block_threads=0, tile_memory="shared", u_min=None, u_max=UMAX, u_init=None,
                    u_scale=1.0, upc=1, abs_cost=False, terminal=None, seed=0, rng_seed=None):
    """The LinearPoint controller with st's per-environment settings and horizons, U0 random inside each horizon and
    u_init past it; and the oracle problem of each environment.  terminal: {e: terminal_scale} of the blocks."""
    terminal = terminal or {}
    base = _lin(st["goals"][0])
    tens = lambda v: None if v is None else torch.tensor(v, dtype=dtype)
    c = eng.MPPI_Batched(base.dynamics, base.running_cost, 2, torch.eye(2, dtype=dtype), N, num_samples=K, horizon=T,
                         u_min=tens(u_min), u_max=tens(u_max), u_init=tens(u_init), u_scale=u_scale, u_per_command=upc,
                         noise_abs_cost=abs_cost, device=DEV, block_threads=block_threads, tile_memory=tile_memory,
                         rng_seed=rng_seed)
    assert c._model is base
    blocks = [_lin(g, terminal.get(e, 0.0)).param_blob() for e, g in enumerate(st["goals"])]
    c.set_env_params(model_params=torch.tensor(blocks, dtype=torch.float64), lambda_=st["lam"], noise_sigma=st["sig"],
                     noise_mu=st["mu"])
    U0 = torch.randn(N, T, 2, generator=torch.Generator().manual_seed(seed), dtype=dtype) * 0.3
    c.U = U0
    c.set_env_horizon(st["H"])
    probs = []
    o64 = lambda v: None if v is None else torch.tensor(v, dtype=F64)
    for e in range(N):
        ol = orc.LinearPointModel(B=B, goal=st["goals"][e], terminal_scale=terminal.get(e, 0.0), dtype=F64)
        probs.append(orc.Problem(ol.dynamics, ol.running_cost, 2, st["sig"][e].double(), K=K, T=st["H"][e],
                                 lambda_=st["lam"][e], noise_mu=st["mu"][e].double(), u_min=o64(u_min), u_max=o64(u_max),
                                 u_init=o64(u_init), u_scale=u_scale, noise_abs_cost=abs_cost,
                                 terminal_state_cost=ol.terminal_cost if e in terminal else None))
    return c, probs, U0


def _oracle_steps(probs, U0, H, x, zs, shift=True):
    """The oracle's commands of every environment over the noise tensors zs, each chained on its own U."""
    out, U = [], [U0[e, :H[e]].double().clone() for e in range(len(probs))]
    for z in zs:
        step = []
        for e, prob in enumerate(probs):
            r = orc.mppi_command(prob, U[e], x[e].double(), z[:, :H[e]].double().contiguous(), shift=shift)
            U[e] = r["U"]
            step.append(r)
        out.append(step)
    return out


def _rel(a, b):
    return float(((a - b).abs() / b.abs().clamp_min(1.0)).max())


def _compare(c, refs, H, x, zs, key, *, tol, ctol, exact_stats, inject=True, shift=True, upc=1):
    """Run len(zs) commands and assert every environment against the oracle's step (U inside the horizon, u_init past
    it exactly, the action(s), cost_total, and in fp64 omega, beta and eta); no environment reports a timeout."""
    N, T, nu = c.N, c.T, c.nu
    ui = c.u_init.to("cpu", F64).view(nu)
    for s, z in enumerate(zs):
        if inject:
            c.inject_noise(z)
        a = c.command(x.to(DEV, c.dtype), shift_nominal_trajectory=shift).cpu().double()
        U, cost, stats = c.U.cpu().double(), c.cost_total.cpu().double(), c._stats.cpu()
        om = c.omega.cpu().double()
        assert torch.equal(stats[:, 3], torch.zeros(N, dtype=F64)), (key, stats[:, 3])
        for e in range(N):
            r, h = refs[s][e], H[e]
            where = (key, s, e)
            assert torch.equal(U[e, h:], ui.expand(T - h, nu)), where
            err = float((U[e, :h] - r["U"]).abs().max())
            _record(f"{key}/U", err)
            assert err <= tol, (where, err)
            want_a = r["U"][:upc] if upc > 1 else r["action"]
            assert float((a[e] - want_a).abs().max()) <= tol, where
            if upc > 1:
                assert torch.equal(a[e], U[e, :upc]), where
            inf = torch.isinf(r["cost_total"])
            assert torch.equal(torch.isinf(cost[e]), inf), where
            fin = ~inf
            cerr = _rel(cost[e][fin], r["cost_total"][fin])
            _record(f"{key}/cost_rel", cerr)
            assert cerr <= ctol, (where, cerr)
            if exact_stats:
                oerr = float((om[e] - r["omega"]).abs().max())
                _record(f"{key}/omega", oerr)
                assert oerr <= 1e-10, (where, oerr)
                if bool(inf.any()):
                    assert float(om[e][inf].abs().max()) == 0.0, where
                berr = abs(float(stats[e, 0]) - float(r["beta"])) / max(1.0, abs(float(r["beta"])))
                eerr = abs(float(stats[e, 1]) - float(r["eta"])) / float(r["eta"])
                _record(f"{key}/beta_rel", berr)
                _record(f"{key}/eta_rel", eerr)
                assert berr <= 1e-10 and eerr <= 1e-10, (where, berr, eerr)
            else:
                berr = abs(float(stats[e, 0]) - float(r["beta"])) / max(1.0, abs(float(r["beta"])))
                _record(f"{key}/beta_rel", berr)
                assert berr <= ctol, (where, berr)


def _draws(K, T, nu, dtype, n, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(K, T, nu, generator=g, dtype=dtype) for _ in range(n)]


def _states(N, nx, dtype, seed=5):
    return torch.randn(N, nx, generator=torch.Generator().manual_seed(seed), dtype=dtype)


# ---- 1: the softmin tail, every geometry, N > 1 -----------------------------------------------------------------------
# name of tests/test_gpu_envelope.py's geometry -> N.  The batched kernels have no split-cost form (choose_fused takes it
# for single environments only), so each (cluster, direct, split) request runs with split = 0.
_TAIL_N = {"one_cta_k31": 4, "one_cluster_k33": 3, "two_records_k33": 3, "cluster_wave": 3, "cluster_wave_32": 2,
           "tiles_sm_plus_1": 3, "multipass_32": 2}
TAIL_T = 6


def _tail_geometries():
    """(name, N, K, samples per tile (0: automatic), T, tile memory, [(cluster, direct, 0)], want)."""
    sm = envl._sm_count()
    out = []
    for name, K, bs, _, envs, want in envl._geometries(sm):
        if name in _TAIL_N:
            reqs = list(dict.fromkeys((cl, d, 0) for cl, d, _ in envs))
            out.append((name, _TAIL_N[name], K, bs, TAIL_T, "shared", reqs, want))
    # the global tile: clusters of one CTA, LL and ticket exchange
    out.append(("global_tile", 3, sm * 64 + 1, 64, TAIL_T, "global", [(8, 1, 0), (1, 0, 0)], dict(cluster=1)))
    # BASELINE config 2's shape with 16 environments: the automatic tile, N grids over more than one wave
    out.append(("c2_n16", 16, 16384, 0, 30, "shared", [(8, 1, 0)], dict(waves=True)))
    return out


def _check_geometry(c, name, K, bs, T, env, want):
    info = c.launch_info
    bs = bs or info.block_threads // info.threads_per_sample
    mode = envl._tail_of(info, K, bs, env, T * 2, {k: v for k, v in want.items() if k != "waves"})
    if want.get("waves"):
        assert info.grid_blocks * c.N > info.sm_count * info.max_blocks_per_sm, _LAUNCH
    if c._tile_memory == "global":
        assert info.global_tile == 1 and info.workspace_bytes % 256 == 0
    return mode


@pytest.mark.parametrize("dtype", [F64, F32])
def test_batched_tail_geometry_matrix(dtype, monkeypatch):
    """Every geometry x tail request, 3 commands per controller (the ticket's self-reset and the LL epochs of every
    environment), each environment against the oracle: fp64 at 1e-10 (U, action, cost_total, omega, beta, eta), fp32 at
    5e-5 on U and 2e-4 relative on cost.  fp32 runs lambda over 0.3 .. 3: at 1e-3 the fp32 rounding of costs of ~10
    would reach the weights' exponents a thousandfold.  Together the runs reach a one-CTA tail, LL and ticket exchange,
    cluster sizes > 1 and 1, and grid-stride multi-pass, all with N > 1."""
    f64 = dtype == F64
    seen = set()
    for name, N, K, bs, T, tile, reqs, want in _tail_geometries():
        st = _settings(N, T, dtype, lam_exp=(-3.0, 3.0) if f64 else (-0.5, 0.5))
        zs = _draws(K, T, 2, dtype, 3, seed=K)
        x = _states(N, 2, dtype)
        refs = None
        for env in reqs:
            for k, v in zip(("MPPI_B200_CLUSTER", "MPPI_B200_XCHG_DIRECT", "MPPI_B200_SPLIT_COST"), env):
                monkeypatch.setenv(k, str(v))
            c, probs, U0 = _linear_batched(N, K, T, dtype, st, block_threads=bs, tile_memory=tile)
            refs = refs or _oracle_steps(probs, U0, st["H"], x, zs)
            key = f"tail/{'f64' if f64 else 'f32'}/{name}/{env}"
            c.inject_noise(zs[0])
            c._pack()
            _record_launch(f"{name}/{env}", c)
            seen.add(_check_geometry(c, name, K, bs, T, env, want))
            _compare(c, refs, st["H"], x, zs, key, tol=1e-10 if f64 else 5e-5, ctol=1e-10 if f64 else 2e-4,
                     exact_stats=f64)
            _record_launch(f"{name}/{env}", c)
    assert {t[0] for t in seen} == {"one", "ll", "ticket"}, seen
    assert any(t[1] > 1 for t in seen) and any(t[1] == 1 for t in seen), seen
    assert any(t[2] for t in seen), seen


def test_batched_tail_geometries_agree_fp32(monkeypatch):
    """fp32: the same draws and settings through every tail of one K (cluster sizes 8..1, LL / ticket, 64- and
    32-sample tiles) give every environment the same plan within 5e-7."""
    N, T = 2, 9
    sm = envl._sm_count()
    K = 16 * 64 - 5
    st = _settings(N, T, F32, lam_exp=(-0.5, 0.5))
    zs = _draws(K, T, 2, F32, 2, seed=11)
    x = _states(N, 2, F32)
    outs = []
    for name, K_, bs, _, envs, want in envl._geometries(sm):
        if K_ != K:
            continue
        for env in dict.fromkeys((cl, d, 0) for cl, d, _ in envs):
            for k, v in zip(("MPPI_B200_CLUSTER", "MPPI_B200_XCHG_DIRECT", "MPPI_B200_SPLIT_COST"), env):
                monkeypatch.setenv(k, str(v))
            c, _, _ = _linear_batched(N, K, T, F32, st, block_threads=bs)
            for z in zs:
                c.inject_noise(z)
                a = c.command(x.to(DEV))
            _check_geometry(c, name, K, bs, T, env, want)
            outs.append(((name, env), c.U.cpu().clone(), a.cpu().clone()))
    assert len(outs) >= 8
    for tag, U, a in outs[1:]:
        err = float((U - outs[0][1]).abs().max())
        _record("tail_fp32_spread", err)
        assert err <= 5e-7, (tag, err)
        assert float((a - outs[0][2]).abs().max()) <= 5e-7, tag


# ---- 2: options on the per-environment kernel --------------------------------------------------------------------------
# (name, K, samples per tile (0: automatic), (cluster, direct, split), want)
_OPT_GEOMETRIES = [("small", 31, 32, (8, 1, 0), dict(grid=1)),
                   ("clusters", 16 * 64 - 5, 64, (8, 1, 0), dict(grid=16, cluster=8))]
_OPTIONS = {
    "upc2": dict(upc=2),
    "abs_cost": dict(abs_cost=True),
    "u_init": dict(u_init=[0.2, -0.3]),
    "u_scale": dict(u_scale=1.3),
    "asym_bounds": dict(u_min=[-0.4, -1.1], u_max=[0.9, 0.3]),
    "no_shift": dict(),
    "n2": dict(),
    "terminal": dict(terminal={2: 2.5}),
}


@pytest.mark.parametrize("option", sorted(_OPTIONS))
@pytest.mark.parametrize("geom", [g[0] for g in _OPT_GEOMETRIES])
def test_batched_options_fp64(geom, option, monkeypatch):
    """fp64 at 1e-10 with per-environment settings and mixed horizons.  upc2: the (N, 2, nu) action is U[e, :2];
    terminal: environment 2 (h = T // 2) has terminal_scale != 0 in its parameter block, the other blocks none, so its
    cost adds the terminal cost of its state after h_e steps; no_shift: command(shift_nominal_trajectory=False)."""
    name, K, bs, env, want = next(g for g in _OPT_GEOMETRIES if g[0] == geom)
    for k, v in zip(("MPPI_B200_CLUSTER", "MPPI_B200_XCHG_DIRECT", "MPPI_B200_SPLIT_COST"), env):
        monkeypatch.setenv(k, str(v))
    N, T = (2 if option == "n2" else 3), 7
    kw = dict(_OPTIONS[option])
    upc = kw.get("upc", 1)
    st = _settings(N, T, F64, upc=upc)
    kw.setdefault("u_max", UMAX)
    c, probs, U0 = _linear_batched(N, K, T, F64, st, block_threads=bs, **kw)
    zs = _draws(K, T, 2, F64, 3, seed=17)
    x = _states(N, 2, F64)
    shift = option != "no_shift"
    refs = _oracle_steps(probs, U0, st["H"], x, zs, shift=shift)
    if option == "terminal":     # the terminal cost changes the result: the oracle without it is not the engine
        p2 = probs[2]
        bare = orc.Problem(p2.dynamics, p2.running_cost, 2, p2.noise_sigma, K=K, T=p2.T, lambda_=p2.lambda_,
                           noise_mu=p2.noise_mu, u_min=p2.u_min, u_max=p2.u_max)
        r0 = orc.mppi_command(bare, U0[2, :st["H"][2]], x[2], zs[0][:, :st["H"][2]].contiguous())
        assert float((r0["cost_total"] - refs[0][2]["cost_total"]).abs().max()) > 1e-2
    _compare(c, refs, st["H"], x, zs, f"options/{geom}/{option}", tol=1e-10, ctol=1e-10, exact_stats=True, shift=shift,
             upc=upc)
    _record_launch(f"options/{geom}", c)
    _check_geometry(c, name, K, bs, T, env, want)


# ---- 3: noise rows past an environment's horizon -----------------------------------------------------------------------
@pytest.mark.parametrize("env", [(8, 1, 0), (1, 0, 0)])
def test_noise_rows_past_the_horizon_do_not_reach_the_environment(env, monkeypatch):
    """LinearPoint without bounds; z = 1e200 at rows t >= h_min of a set S of samples (8 whole tiles, so whole warp,
    CTA and cluster records, and 10 % scattered).  Environments with h_e = h_min never read those rows: they equal their
    finite oracle.  The longer ones get cost +inf on exactly S, weight 0 there, and a finite update equal to the
    oracle's."""
    for k, v in zip(("MPPI_B200_CLUSTER", "MPPI_B200_XCHG_DIRECT", "MPPI_B200_SPLIT_COST"), env):
        monkeypatch.setenv(k, str(v))
    N, T, K, bs = 4, 6, 16 * 64 - 5, 64
    st = _settings(N, T, F64, lam_exp=(-1.0, 1.0))
    st["H"] = [2, 6, 2, 4]
    h_min = 2
    c, probs, U0 = _linear_batched(N, K, T, F64, st, block_threads=bs, u_max=None)
    g = torch.Generator().manual_seed(23)
    S = torch.zeros(K, dtype=torch.bool)
    S[: 8 * bs] = True
    S[torch.randperm(K, generator=g)[: K // 10]] = True
    zs = []
    for _ in range(3):
        z = torch.randn(K, T, 2, generator=g, dtype=F64)
        z[S, h_min:] = 1e200
        zs.append(z)
    x = _states(N, 2, F64)
    refs = _oracle_steps(probs, U0, st["H"], x, zs)
    for e in range(N):           # the oracle itself: finite where h_e = h_min, +inf on exactly S elsewhere
        assert torch.equal(torch.isinf(refs[0][e]["cost_total"]), S if st["H"][e] > h_min else torch.zeros_like(S))
    _compare(c, refs, st["H"], x, zs, f"past_horizon/{env}", tol=1e-10, ctol=1e-10, exact_stats=True)
    assert bool(torch.isfinite(c.U).all())
    _check_geometry(c, "past_horizon", K, bs, T, env, dict(grid=16))


# ---- 4: the in-kernel draws with horizons ------------------------------------------------------------------------------
@pytest.mark.parametrize("tile_memory", ["shared", "global"])
@pytest.mark.parametrize("dtype", [F64, F32])
def test_in_kernel_draws_with_horizons_match_oracle(dtype, tile_memory):
    """nu = 3, T = 7: R = 21 normals per sample, not a multiple of the 4 (fp32) or 2 (fp64) of one Philox call.  No
    injected noise: z of each command is the numpy statement of the stream at the command's counter offset, and each
    environment (its own full Sigma, mu, lambda and horizon) equals the oracle on z[:, :h_e]."""
    N, K, T, nu, seed = 4, 1000, 7, 3, 0x5EED5
    f64 = dtype == F64
    H = [7, 1, 4, 6]
    lam = [0.5, 1.0, 2.0, 0.8]
    base_sig = torch.tensor(SIG3, dtype=F64)
    sig = torch.stack([base_sig * (0.6 + 0.3 * e) + torch.eye(3, dtype=F64) * 0.05 * e for e in range(N)]).to(dtype)
    mu = torch.tensor([[0.05 * (e + 1), -0.03 * e, 0.02] for e in range(N)], dtype=dtype)
    m = shm.shape_model(3, 3, terminal=False)
    f, cst, _ = shm.twins(3, 3)
    umax = torch.full((nu,), 1.2, dtype=dtype)
    c = eng.MPPI_Batched(m.dynamics, m.running_cost, 3, torch.eye(nu, dtype=dtype), N, num_samples=K, horizon=T,
                         u_max=umax, device=DEV, rng_seed=seed, tile_memory=tile_memory)
    assert c._model is m
    c.set_env_params(lambda_=lam, noise_sigma=sig, noise_mu=mu)
    U0 = torch.randn(N, T, nu, generator=torch.Generator().manual_seed(3), dtype=dtype) * 0.3
    c.U = U0
    c.set_env_horizon(H)
    probs = [orc.Problem(f, cst, 3, sig[e].double(), K=K, T=H[e], lambda_=lam[e], noise_mu=mu[e].double(),
                         u_max=umax.double()) for e in range(N)]
    np_dt = np.float64 if f64 else np.float32
    per = 2 if f64 else 4
    chunks = (T * nu + per - 1) // per
    zs = [torch.from_numpy(po.normals(seed, s * chunks, 0, K, T * nu, np_dt)).reshape(K, T, nu).double()
          for s in range(3)]
    x = torch.tensor([[0.3, -0.2, 0.1], [-0.4, 0.1, 0.2], [0.0, 0.5, -0.3], [0.2, 0.2, 0.2]], dtype=dtype)
    refs = _oracle_steps(probs, U0, H, x, zs)
    _compare(c, refs, H, x, zs, f"philox/{'f64' if f64 else 'f32'}/{tile_memory}", tol=1e-10 if f64 else 5e-5,
             ctol=1e-10 if f64 else 2e-4, exact_stats=f64, inject=False)
    assert c.launch_info.global_tile == (1 if tile_memory == "global" else 0)
    # environment e's workspace starts e x workspace_bytes in: fp32 tile slices of R = 21 rows once left it 4-byte
    # aligned, and the kernel's 8-byte ticket, record and mailbox accesses of environments e > 0 faulted
    assert c.launch_info.workspace_bytes % 256 == 0


# ---- 5: a closed loop against the oracle -------------------------------------------------------------------------------
def test_closed_loop_with_per_environment_settings_matches_oracle_loop():
    """fp64, N = 4, 15 steps of run_closed_loop with per-environment goals, lambda, Sigma, mu and horizons, one plant per
    environment (its own B and goal) and a disturbance, against a loop of the oracle alone: Philox-oracle z per step,
    the oracle's command per environment chained on its own U, and the oracle's dynamics of each plant plus the
    disturbance.  Each step continues from the engine's state, so the 1e-10 gap does not compound."""
    N, K, T, steps, seed = 4, 512, 10, 15, 77
    st = _settings(N, T, F64, lam_exp=(-1.0, 1.0))
    st["H"] = [10, 3, 1, 7]
    c, probs, U0 = _linear_batched(N, K, T, F64, st, u_init=[0.1, -0.05], rng_seed=seed)
    plant_B = [[[1.0 + 0.1 * e, 0.05], [0.0, -1.0 + 0.05 * e]] for e in range(N)]
    plant_goal = [[1.0, -1.0 + 0.5 * e] for e in range(N)]
    pp = torch.tensor([eng.LinearPoint(B=plant_B[e], goal=plant_goal[e]).param_blob() for e in range(N)],
                      dtype=torch.float64)
    dist = 0.02 * torch.randn(steps, N, 2, generator=torch.Generator().manual_seed(8), dtype=F64)
    x0 = torch.tensor([[0.5, -0.5], [-1.0, 1.0], [0.0, 0.3], [1.5, 1.5]], dtype=F64)
    res = c.run_closed_loop(x0.to(DEV), steps, plant_params=pp, disturbance=dist.to(DEV))
    states, actions, costs = res.states.cpu(), res.actions.cpu(), res.costs.cpu()
    plants = [orc.LinearPointModel(B=plant_B[e], goal=plant_goal[e], dtype=F64) for e in range(N)]
    chunks = T       # (T * nu + 1) // 2 fp64 Philox calls per sample
    U = [U0[e, :st["H"][e]].clone() for e in range(N)]
    for s in range(steps):
        z = torch.from_numpy(po.normals(seed, s * chunks, 0, K, T * 2, np.float64)).reshape(K, T, 2)
        for e in range(N):
            h = st["H"][e]
            r = orc.mppi_command(probs[e], U[e], states[s, e], z[:, :h].contiguous())
            U[e] = r["U"]
            err = float((actions[s, e] - r["action"]).abs().max())
            _record("closed_loop/action", err)
            assert err <= 1e-10, (s, e, err)
            xn = plants[e].dynamics(states[s, e].view(1, 2), actions[s, e].view(1, 2)).view(2) + dist[s, e]
            serr = float((states[s + 1, e] - xn).abs().max())
            _record("closed_loop/state", serr)
            assert serr <= 1e-12, (s, e, serr)
            cc = plants[e].running_cost(states[s + 1, e].view(1, 2), actions[s, e].view(1, 2))
            assert abs(float(costs[s, e]) - float(cc)) <= 1e-10 * max(1.0, abs(float(cc))), (s, e)
    for e in range(N):
        h = st["H"][e]
        err = float((c.U[e, :h].cpu() - U[e]).abs().max())
        _record("closed_loop/U", err)
        assert err <= 1e-10, (e, err)
        assert torch.equal(c.U[e, h:].cpu(), torch.tensor([0.1, -0.05], dtype=F64).expand(T - h, 2))


# ---- 6: N = 1 and N = 64 ------------------------------------------------------------------------------------------------
def test_one_environment_matches_oracle_and_refuses_per_environment_settings():
    """MPPI_Batched(num_envs=1) with a full Sigma, mu and lambda against the oracle; a per-environment setting or horizon
    on it raises ValueError and leaves the controller as it was."""
    K, T = 300, 9
    sig = torch.tensor(SIGMAS[2], dtype=F64)
    mu = torch.tensor([0.1, -0.2], dtype=F64)
    base = _lin([1.0, -1.5])
    c = eng.MPPI_Batched(base.dynamics, base.running_cost, 2, sig, 1, num_samples=K, horizon=T, lambda_=0.7, noise_mu=mu,
                         u_max=torch.tensor(UMAX, dtype=F64), device=DEV)
    assert c._model is base
    U0 = torch.randn(1, T, 2, generator=torch.Generator().manual_seed(2), dtype=F64) * 0.3
    c.U = U0
    ol = orc.LinearPointModel(B=B, goal=[1.0, -1.5], dtype=F64)
    prob = orc.Problem(ol.dynamics, ol.running_cost, 2, sig, K=K, T=T, lambda_=0.7, noise_mu=mu,
                       u_max=torch.tensor(UMAX, dtype=F64))
    zs = _draws(K, T, 2, F64, 3, seed=4)
    x = torch.tensor([[0.4, 0.2]], dtype=F64)
    refs = _oracle_steps([prob], U0, [T], x, zs)
    for phase in ("before the first command", "after it"):
        U_before = c.U.clone()
        with pytest.raises(ValueError, match="one environment"):
            c.set_env_params(lambda_=[2.0])
        with pytest.raises(ValueError, match="one environment"):
            c.set_env_horizon([4])
        c.set_env_params()
        c.set_env_horizon(None)
        assert c.env_lambda is None and c.env_noise_sigma is None and c.env_horizon is None, phase
        assert torch.equal(c.U, U_before), phase
        if phase == "before the first command":
            _compare(c, refs, [T], x, zs, "n1", tol=1e-10, ctol=1e-10, exact_stats=True)
    _record_launch("n1", c)


def test_sixty_four_environments_match_oracle():
    """N = 64 (gridDim.y = 64) with every environment's own settings and horizon, K = 256."""
    N, K, T = 64, 256, 9
    st = _settings(N, T, F64)
    c, probs, U0 = _linear_batched(N, K, T, F64, st)
    zs = _draws(K, T, 2, F64, 3, seed=64)
    x = _states(N, 2, F64)
    refs = _oracle_steps(probs, U0, st["H"], x, zs)
    _compare(c, refs, st["H"], x, zs, "n64", tol=1e-10, ctol=1e-10, exact_stats=True)
    _record_launch("n64", c)
