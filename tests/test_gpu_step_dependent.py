"""GPU: step-dependent user models on the fused route (CudaModel(step_dependent=True), step_dependent_dynamics=True) —
parity with the oracle on both rollout shapes, resident mode, get_rollouts, and set_params between commands.  Their
golden fixtures, MPPI_Batched's among them, are replayed in tests/test_gpu_golden_replay.py."""
import functools

import numpy as np
import pytest
import torch

import pytorch_mppi_b200 as eng
from oracle import mppi_oracle as orc
from tests import step_models as um
from tests.golden.step_cases import HorizonClock

pytestmark = pytest.mark.gpu

SIGMA, UMAX = 1.0, 3.0


def _ctrl(cls, m, K, T, dtype, U0=None, **kw):
    c = cls(m.dynamics, m.running_cost, 2, torch.tensor(SIGMA, dtype=dtype), num_samples=K, horizon=T, U_init=U0,
            u_max=torch.tensor(UMAX, dtype=dtype), terminal_state_cost=m.terminal_cost if m.has_terminal else None,
            step_dependent_dynamics=True, device="cuda", **kw)
    assert c._model is m, "fused route not selected"
    return c


def _problem(params, K, T, dtype):
    clock = HorizonClock(functools.partial(um.sd_dyn, p=params), functools.partial(um.sd_cost, p=params), T)
    return orc.Problem(clock.dynamics, clock.running_cost, 2, torch.tensor(SIGMA, dtype=dtype), K=K, T=T,
                       u_max=torch.tensor(UMAX, dtype=dtype), terminal_state_cost=functools.partial(um.sd_term, p=params))


def _plant(x, a, params):
    return um.sd_dyn(x.view(1, -1), a.reshape(1, -1), 0, params).view(-1)


def _closed_loop_vs_oracle(variant, K, T, dtype, tol, steps=3, states_tol=None):
    """`steps` closed-loop commands of the engine and the oracle on the same injected draws; returns the controller."""
    g = torch.Generator().manual_seed(17)
    m = um.step_dependent_user_model()
    prob = _problem(um.SD_PARAMS, K, T, dtype)
    U0 = torch.randn(T, 1, generator=g, dtype=dtype)
    x = torch.tensor([0.2, -0.3], dtype=dtype)
    if variant == "mppi":
        c = _ctrl(eng.MPPI, m, K, T, dtype, U0.clone())
        U = U0.clone()
    elif variant == "smppi":
        c = _ctrl(eng.SMPPI, m, K, T, dtype, w_action_seq_cost=2.0, delta_t=0.5, action_max=torch.tensor(UMAX, dtype=dtype))
        sp = orc.SmoothParams(w_action_seq_cost=2.0, delta_t=0.5, action_max=torch.tensor(UMAX, dtype=dtype))
        U, A = torch.zeros(T, 1, dtype=dtype), torch.zeros(T, 1, dtype=dtype)
    else:
        S = 6
        c = _ctrl(eng.KMPPI, m, K, T, dtype, U0.clone(), num_support_pts=S, kernel=eng.RBFKernel(sigma=2.0))
        W, Wshift = orc.kernel_matrices(T, S, lambda a, b: orc.rbf_kernel(a, b, 2.0), dtype)
        U, theta = U0.clone(), torch.zeros(S, 1, dtype=dtype)
    for _ in range(steps):
        z = torch.randn(K, S if variant == "kmppi" else T, 1, generator=g, dtype=dtype)
        c.inject_noise(z)
        a = c.command(x)
        if variant == "mppi":
            r = orc.mppi_command(prob, U, x, z)
            U = r["U"]
        elif variant == "smppi":
            r = orc.smppi_command(prob, sp, U, A, x, z)
            U, A = r["U"], r["action_sequence"]
            assert float((c.action_sequence.cpu() - A).abs().max()) <= tol
        else:
            r = orc.kmppi_command(prob, U, theta, x, z, W, Wshift)
            U, theta = r["U"], r["theta"]
            assert float((c.theta.cpu() - theta).abs().max()) <= tol
        err = float((c.U.cpu() - U).abs().max())
        assert err <= tol, f"{variant} K={K}: |U - U_oracle| = {err:.3e}"
        assert float((a.cpu() - r["action"]).abs().max()) <= tol
        if states_tol is not None:
            np.testing.assert_allclose(c.states.cpu().numpy(), r["states"].numpy(), atol=states_tol, rtol=0)
        x = _plant(x, r["action"], um.SD_PARAMS)
    return c


@pytest.mark.parametrize("variant", ["mppi", "smppi", "kmppi"])
def test_fp64_parity_with_oracle(variant):
    c = _closed_loop_vs_oracle(variant, 1024, 20, torch.float64, 1e-10, states_tol=1e-10)
    assert c.launch_info.split_cost == 1


def test_fp32_parity_with_oracle_north_star_shape():
    c = _closed_loop_vs_oracle("mppi", 16384, 30, torch.float32, 1e-5, steps=2)
    assert c.launch_info.split_cost == 1


def test_single_loop_rollout_matches_oracle():
    """K=131072: one thread per sample, the single T-loop that evaluates step t's cost in iteration t, after step t's
    dynamics.  An off-by-one in t there would miss by > 2e-4 (tests/test_step_dependent.py)."""
    c = _closed_loop_vs_oracle("mppi", 131072, 15, torch.float64, 1e-9, steps=2)
    assert c.launch_info.split_cost == 0


def test_split_cost_rollout_equals_single_loop_bit_for_bit(monkeypatch):
    """The split-cost rollout (helper thread per t) and the single-loop kernel (step t's cost in iteration t) give the
    same per-sample costs bit for bit, as for the registered models (tests/test_gpu_golden_replay.py); the softmin reduction
    order follows each kernel's cluster size, so U and the action agree to fp32 rounding of that order."""
    m = um.step_dependent_user_model()
    ctrls = {}
    for split in ("1", "0"):
        monkeypatch.setenv("MPPI_B200_SPLIT_COST", split)
        ctrls[split] = _ctrl(eng.MPPI, m, 16384, 30, torch.float32, torch.zeros(30, 1), rng_seed=9)
    for step in range(3):
        x = [0.1 * step, 0.0]
        a1, a0 = ctrls["1"].command(x), ctrls["0"].command(x)
        assert torch.equal(ctrls["1"].cost_total, ctrls["0"].cost_total), step
        assert torch.allclose(ctrls["1"].U, ctrls["0"].U, rtol=0, atol=5e-7) and torch.allclose(a1, a0, rtol=0, atol=5e-7)
        ctrls["0"].U = ctrls["1"].U                  # the next command starts from the same nominal
    assert ctrls["1"].launch_info.split_cost == 1 and ctrls["0"].launch_info.split_cost == 0
    assert ctrls["1"].launch_info.threads_per_sample == ctrls["0"].launch_info.threads_per_sample > 1


def test_resident_equals_launch_route_across_set_params():
    """command_host() under resident() is bit-identical to the launch route, also when set_params moves the target
    between commands: the grid leaves, the plan takes the new values, and the next command brings the grid back."""
    m = um.step_dependent_user_model()
    res = _ctrl(eng.MPPI, m, 16384, 30, torch.float32, torch.zeros(30, 1), rng_seed=5)
    ref = _ctrl(eng.MPPI, m, 16384, 30, torch.float32, torch.zeros(30, 1), rng_seed=5)
    p = list(um.SD_PARAMS)
    with res.resident(idle_us=200000):
        for step in range(6):
            if step == 3:
                plan, launches = res._plan.value, res.resident_launches
                p[3] += 0.25
                m.set_params(p)
            x = [0.1 * step, -0.05 * step]
            a, b = res.command_host(x), ref.command_host(x)
            assert torch.equal(a, b), step
            assert torch.equal(res.U, ref.U) and torch.equal(res.cost_total, ref.cost_total)
        assert res._plan.value == plan and res.resident_launches > launches
    assert launches >= 1
    # the record epochs of both resident sessions stay used: a later session or launch-route command never reuses a tag
    # whose records are still in the workspace (6 commands + the stop record of the session set_params ended)
    assert int(res._lib.mppi_plan_epoch(res._plan)) >= 7


def test_get_rollouts_equals_torch_loop():
    m = um.step_dependent_user_model()
    T = 20
    c = _ctrl(eng.MPPI, m, 512, T, torch.float64, torch.randn(T, 1, dtype=torch.float64), u_scale=1.3)
    x0 = torch.tensor([[0.0, 0.0], [1.0, -0.5], [-0.4, 2.0]], dtype=torch.float64, device="cuda")

    def loop():
        s, out = x0, []
        for t in range(T):
            s = m.dynamics(s, 1.3 * c.U[t].expand(3, -1), t)
            out.append(s)
        return torch.stack(out, dim=1)

    for _ in range(2):
        got = c.get_rollouts(x0, num_rollouts=3)
        assert float((got - loop()).abs().max()) <= 1e-12
        p = list(m.params)
        p[1] = -p[1]
        m.set_params(p)                     # get_rollouts uses the current parameters, before any command took them


def test_set_params_takes_effect_at_the_next_command_without_a_new_plan():
    """Controller A, given set_params(p2) before its second command, computes exactly what a controller B built with p2
    and A's nominal computes; A keeps its plan; A's states of the first command still describe that command."""
    dt, K, T = torch.float64, 2048, 20
    p2 = list(um.SD_PARAMS)
    p2[3], p2[4] = 1.5, -0.2
    U0 = torch.randn(T, 1, generator=torch.Generator().manual_seed(2), dtype=dt)
    mA, mC = um.step_dependent_user_model(), um.step_dependent_user_model()
    A, C = _ctrl(eng.MPPI, mA, K, T, dt, U0.clone()), _ctrl(eng.MPPI, mC, K, T, dt, U0.clone())
    g = torch.Generator().manual_seed(3)
    z1, z2 = torch.randn(K, T, 1, generator=g, dtype=dt), torch.randn(K, T, 1, generator=g, dtype=dt)
    x = [0.3, 0.1]
    for c in (A, C):
        c.inject_noise(z1)
        c.command(x)
    plan, info = A._plan.value, A.launch_info
    mA.set_params(p2)
    assert torch.equal(A.states, C.states)                 # materialised after set_params: still the first command's
    B = _ctrl(eng.MPPI, um.step_dependent_user_model(p2), K, T, dt, A.U.clone())
    A.inject_noise(z2)
    B.inject_noise(z2)
    a, b = A.command(x), B.command(x)
    assert torch.equal(a, b) and torch.equal(A.U, B.U) and torch.equal(A.cost_total, B.cost_total)
    assert torch.equal(A.states, B.states)
    assert A._plan.value == plan and A.launch_info is info
    C.inject_noise(z2)
    C.command(x)
    assert not torch.equal(C.U, A.U)                         # the new target really changed the command
