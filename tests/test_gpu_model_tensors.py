"""GPU: user models that read device tensors (CudaModel(tensors=...)) on the fused route — a costmap read with bilinear
interpolation and a reference path indexed by t (tests/tensor_models.py).  Parity with the oracle on both rollout shapes,
uint8 / int32 maps, in-place edits and set_tensors between commands, clamped lookups outside the map, resident mode,
get_rollouts / states, copies=M with per-copy maps and MPPI_Batched.  The live-reference fixtures are replayed in
tests/test_gpu_golden_replay.py."""
import functools

import numpy as np
import pytest
import torch

import pytorch_mppi_b200 as eng
from oracle import mppi_oracle as orc
from tests import tensor_models as tm
from tests.golden.step_cases import HorizonClock

pytestmark = pytest.mark.gpu

SIGMA, UMAX = 1.0, 3.0


def _ctrl(cls, m, K, T, dtype, U0=None, **kw):
    c = cls(m.dynamics, m.running_cost, 2, SIGMA * torch.eye(2, dtype=dtype), num_samples=K, horizon=T, U_init=U0,
            u_max=torch.full((2,), UMAX, dtype=dtype), step_dependent_dynamics=True, device="cuda", **kw)
    assert c._model is m, "fused route not selected"
    return c


def _problem(m, K, T, dtype, **kw):
    """The oracle's problem on the CPU copies of the model's tensors."""
    cm = {k: v.cpu() for k, v in m.tensors.items()}
    cost = functools.partial(tm.nav_cost, p=m.params, costmap=cm["costmap"], path=cm["path"])
    if kw.get("rollout_samples", 1) > 1:
        K_ = K

        def cost(s, a, t):
            copy = torch.div(torch.arange(s.shape[0]), K_, rounding_mode="floor")
            return tm.nav_cost(s, a, t, m.params, cm["costmap"], cm["path"], copy)
    clock = HorizonClock(functools.partial(tm.nav_dyn, p=m.params), cost, T)
    return orc.Problem(clock.dynamics, clock.running_cost, 2, SIGMA * torch.eye(2, dtype=dtype), K=K, T=T,
                       u_max=torch.full((2,), UMAX, dtype=dtype), **kw)


def _closed_loop_vs_oracle(m, variant, K, T, dtype, tol, steps=3, x=(-1.2, -0.9), S=6, states_tol=None, **ckw):
    g = torch.Generator().manual_seed(21)
    okw = {k: v for k, v in ckw.items() if k in ("rollout_samples", "rollout_var_cost", "rollout_var_discount")}
    prob = _problem(m, K, T, dtype, **okw)
    U0 = torch.randn(T, 2, generator=g, dtype=dtype)
    x = torch.tensor(x, dtype=dtype)
    if variant == "mppi":
        c = _ctrl(eng.MPPI, m, K, T, dtype, U0.clone(), **ckw)
        U = U0.clone()
    elif variant == "smppi":
        c = _ctrl(eng.SMPPI, m, K, T, dtype, w_action_seq_cost=2.0, delta_t=0.5,
                  action_max=torch.full((2,), UMAX, dtype=dtype), **ckw)
        sp = orc.SmoothParams(w_action_seq_cost=2.0, delta_t=0.5, action_max=torch.full((2,), UMAX, dtype=dtype))
        U, A = torch.zeros(T, 2, dtype=dtype), torch.zeros(T, 2, dtype=dtype)
    else:
        c = _ctrl(eng.KMPPI, m, K, T, dtype, U0.clone(), num_support_pts=S, kernel=eng.RBFKernel(sigma=2.0), **ckw)
        W, Wshift = orc.kernel_matrices(T, S, lambda a, b: orc.rbf_kernel(a, b, 2.0), dtype)
        U, theta = U0.clone(), torch.zeros(S, 2, dtype=dtype)
    for _ in range(steps):
        z = torch.randn(K, S if variant == "kmppi" else T, 2, generator=g, dtype=dtype)
        c.inject_noise(z)
        a = c.command(x)
        if variant == "mppi":
            r = orc.mppi_command(prob, U, x, z)
            U = r["U"]
        elif variant == "smppi":
            r = orc.smppi_command(prob, sp, U, A, x, z)
            U, A = r["U"], r["action_sequence"]
        else:
            r = orc.kmppi_command(prob, U, theta, x, z, W, Wshift)
            U, theta = r["U"], r["theta"]
        err = float((c.U.cpu() - U).abs().max())
        assert err <= tol, f"{variant} K={K}: |U - U_oracle| = {err:.3e}"
        assert float((a.cpu() - r["action"]).abs().max()) <= tol
        assert torch.isfinite(c.cost_total).all()
        if states_tol is not None:
            np.testing.assert_allclose(c.states.cpu().numpy(), r["states"].numpy(), atol=states_tol, rtol=0)
        x = tm.nav_dyn(x.view(1, -1), r["action"].view(1, -1), 0, m.params).view(-1)
    return c


def _nav(T, map_dtype=torch.float32, hw=tm.MAP_HW, seed=0):
    return tm.nav_model(tm.make_costmap(map_dtype, hw, seed=seed), tm.make_path(T))


@pytest.mark.parametrize("variant", ["mppi", "smppi", "kmppi"])
def test_fp64_parity_with_oracle_split_cost(variant):
    c = _closed_loop_vs_oracle(_nav(20), variant, 1024, 20, torch.float64, 1e-10)
    assert c.launch_info.split_cost == 1


@pytest.mark.parametrize("variant,K", [("mppi", 131072), ("kmppi", 131072), ("smppi", 16384)])
def test_fp64_parity_with_oracle_single_loop(variant, K, monkeypatch):
    """K=131072 runs one thread per sample on the single-loop rollout; SMPPI's effective-noise tile at nu=2 does not fit
    that geometry, so its single loop is taken at K=16384 with the split-cost rollout switched off."""
    monkeypatch.setenv("MPPI_B200_SPLIT_COST", "0")
    c = _closed_loop_vs_oracle(_nav(15), variant, K, 15, torch.float64, 1e-10, steps=2)
    assert c.launch_info.split_cost == 0


def test_fp32_c3_shape_parity_with_oracle():
    """The C3 shape: KMPPI S=5, K=8192, T=40, a 256 x 256 fp32 map.  Bound 4e-5 rather than the north-star 1e-5: costs
    are 50..400 at lambda=1 and the effective sample size of these commands is 1.1..2.5 (omega of the oracle), so the
    update follows one or two samples, and a 1-ulp difference in their costs (6e-6 at 100; the interpolated trajectory
    W theta is a matrix product, summed in another order than the oracle's) moves U by ~1e-5 — as for pendulum_small_f32
    (tests/golden/cases.py).  Measured 1.8e-5 on H100."""
    m = _nav(40, hw=(256, 256))
    _closed_loop_vs_oracle(m, "kmppi", 8192, 40, torch.float32, 4e-5, S=5)


@pytest.mark.parametrize("map_dtype", [torch.uint8, torch.int32])
def test_integer_maps_match_oracle(map_dtype):
    m = _nav(20, map_dtype)
    assert m.tensors["costmap"].dtype == map_dtype and m.tensors["costmap"].max() > 100
    _closed_loop_vs_oracle(m, "mppi", 1024, 20, torch.float64, 1e-10)


def _single(m, T):
    U0 = torch.randn(T, 2, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    return _ctrl(eng.MPPI, m, 2048, T, torch.float64, U0, rng_seed=7)


def test_in_place_edit_equals_fresh_controller():
    """costmap.copy_(...) between commands takes effect at the next command with no call: A after the edit computes
    exactly what B, built on the edited map with A's nominal and RNG position, computes."""
    T = 20
    m = _nav(T)
    A = _single(m, T)
    x = [-1.0, -1.0]
    A.command(x)
    plan = A._plan.value
    new_map = tm.make_costmap(seed=5)
    m.tensors["costmap"].copy_(new_map)
    B = _ctrl(eng.MPPI, tm.nav_model(new_map.clone(), tm.make_path(T)), 2048, T, torch.float64, A.U.clone(), rng_seed=7)
    B._rng_counter = A._rng_counter
    a, b = A.command(x), B.command(x)
    assert torch.equal(a, b) and torch.equal(A.U, B.U) and torch.equal(A.cost_total, B.cost_total)
    assert A._plan.value == plan


def test_set_tensors_new_shape_no_replan_equals_fresh_controller():
    T = 20
    m = _nav(T)
    A = _single(m, T)
    x = [-1.0, -1.0]
    A.command(x)
    plan, info = A._plan.value, A.launch_info
    big, path2 = tm.make_costmap(hw=(96, 80), seed=6), tm.make_path(T + 7)
    m.set_tensors(costmap=big, path=path2)
    B = _ctrl(eng.MPPI, tm.nav_model(big, path2), 2048, T, torch.float64, A.U.clone(), rng_seed=7)
    B._rng_counter = A._rng_counter
    a, b = A.command(x), B.command(x)
    assert torch.equal(a, b) and torch.equal(A.U, B.U) and torch.equal(A.cost_total, B.cost_total)
    assert A._plan.value == plan and A.launch_info is info


def test_lookups_far_outside_the_map_are_clamped():
    """Start states far outside the map on both sides: every lookup is clamped to the border, results are finite and
    equal the twin's (oracle) and the rollouts equal the twin's."""
    for x in ((40.0, -35.0), (-60.0, 25.0)):
        m = _nav(15)
        c = _closed_loop_vs_oracle(m, "mppi", 1024, 15, torch.float64, 1e-10, steps=2, x=x)
        x0 = torch.tensor([x], dtype=torch.float64, device="cuda")
        got = c.get_rollouts(x0, num_rollouts=1)
        s, want = x0, []
        for t in range(15):
            s = m.dynamics(s, c.U[t].view(1, -1), t)
            want.append(s)
        assert torch.isfinite(got).all() and float((got - torch.stack(want, dim=1)).abs().max()) <= 1e-12


def test_resident_equals_launch_route_across_set_tensors():
    m = _nav(30)
    res = _ctrl(eng.MPPI, m, 16384, 30, torch.float32, torch.zeros(30, 2), rng_seed=5)
    ref = _ctrl(eng.MPPI, m, 16384, 30, torch.float32, torch.zeros(30, 2), rng_seed=5)
    with res.resident(idle_us=200000):
        for step in range(6):
            if step == 3:
                plan, launches = res._plan.value, res.resident_launches
                m.set_tensors(costmap=tm.make_costmap(hw=(48, 72), seed=9))
            x = [-1.0 + 0.1 * step, -0.05 * step]
            a, b = res.command_host(x), ref.command_host(x)
            assert torch.equal(a, b), step
            assert torch.equal(res.U, ref.U) and torch.equal(res.cost_total, ref.cost_total)
        assert res._plan.value == plan and res.resident_launches > launches
    assert res.launch_info.split_cost == 1


def test_get_rollouts_equals_the_twin():
    T = 20
    m = _nav(T)
    c = _ctrl(eng.MPPI, m, 512, T, torch.float64, torch.randn(T, 2, dtype=torch.float64), u_scale=1.3)
    x0 = torch.tensor([[-1.0, -1.0], [0.5, 1.5], [30.0, -9.0]], dtype=torch.float64, device="cuda")
    s, out = x0, []
    for t in range(T):
        s = m.dynamics(s, 1.3 * c.U[t].expand(3, -1), t)
        out.append(s)
    assert float((c.get_rollouts(x0, num_rollouts=3) - torch.stack(out, dim=1)).abs().max()) <= 1e-12


def test_copies_with_per_copy_maps_match_oracle():
    M, K, T = tm.ENSEMBLE_M, 1024, 20
    maps = torch.stack([tm.make_costmap(seed=20 + i) for i in range(M)]).contiguous()
    m = tm.nav_ensemble(maps, tm.make_path(T), K)
    _closed_loop_vs_oracle(m, "mppi", K, T, torch.float64, 1e-10, rollout_samples=M, rollout_var_cost=0.5,
                           rollout_var_discount=0.9)


def test_mppi_batched_equals_single_controllers():
    N, K, T, dt = 3, 1024, 20, torch.float64
    m = _nav(T)
    g = torch.Generator().manual_seed(8)
    U0 = torch.randn(N, T, 2, generator=g, dtype=dt)
    xs = torch.tensor([[-1.0, -1.0], [0.5, -0.5], [1.2, 1.4]], dtype=dt)
    bat = eng.MPPI_Batched(m.dynamics, m.running_cost, 2, SIGMA * torch.eye(2, dtype=dt), N, num_samples=K, horizon=T,
                           u_max=torch.full((2,), UMAX, dtype=dt), step_dependent_dynamics=True, device="cuda")
    assert bat._model is m
    bat.U = U0.clone()
    singles = [_ctrl(eng.MPPI, m, K, T, dt, U0[n].clone()) for n in range(N)]
    for _ in range(2):
        z = torch.randn(K, T, 2, generator=g, dtype=dt)
        bat.inject_noise(z)
        a = bat.command(xs)
        for n, c in enumerate(singles):
            c.inject_noise(z)
            an = c.command(xs[n])
            assert float((bat.U[n] - c.U).abs().max()) <= 1e-10 and float((a[n] - an).abs().max()) <= 1e-10
            np.testing.assert_allclose(bat.cost_total[n].cpu().numpy(), c.cost_total.cpu().numpy(), rtol=0, atol=1e-10)


def test_tensor_on_another_device_is_refused_at_pack():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    m = tm.nav_model(tm.make_costmap(device="cuda:1"), tm.make_path(20, device="cuda:1"))
    with pytest.raises(ValueError, match="controller on"):
        _ctrl(eng.MPPI, m, 512, 20, torch.float64).command([0.0, 0.0])
