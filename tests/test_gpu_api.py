"""GPU: API conformance with the reference's class surface.  Each test restates, for the CUDA engine,
a behaviour the reference's own suite pins (reference tests/test_mppi.py — cited per test); both
execution routes are exercised: `fused` (registered LinearPoint model) and `stepped` (plain callables)."""
import numpy as np
import pytest
import torch

import pytorch_mppi_b200 as eng

pytestmark = pytest.mark.gpu
DT = torch.double
DEV = "cuda"
GOAL = torch.tensor([2.0, 2.0], dtype=DT)
B = torch.tensor([[1.0, 0.0], [0.0, -1.0]], dtype=DT)


_DEV_CACHE = {}


def _on(t, like):
    """device/dtype copy of a module-level constant, cached so the plugins never issue a host->device copy
    on the hot path (which would also be illegal inside CUDA-graph capture)"""
    key = (id(t), like.device, like.dtype)
    if key not in _DEV_CACHE:
        _DEV_CACHE[key] = t.to(like.device, like.dtype)
    return _DEV_CACHE[key]


def lin_dyn(s, a):
    return s + a @ _on(B, s).T


def quad_cost(s, a):
    return ((_on(GOAL, s) - s) ** 2).sum(-1)


def term_cost(states, actions):
    return ((_on(GOAL, states) - states[..., -1, :]) ** 2).sum(-1)


def plugins(route, terminal=False):
    if route == "fused":
        m = eng.LinearPoint.unit_test_env(terminal_scale=1.0 if terminal else 0.0)
        return m.dynamics, m.running_cost, (m.terminal_cost if terminal else None)
    return lin_dyn, quad_cost, (term_cost if terminal else None)


def make(cls=None, route="fused", terminal=False, seed=42, **kw):
    torch.manual_seed(seed)
    dyn, cost, term = plugins(route, terminal)
    args = dict(num_samples=100, horizon=10, device=DEV, lambda_=1.0, terminal_state_cost=term)
    args.update(kw)
    c = (cls or eng.MPPI)(dyn, cost, 2, args.pop("noise_sigma", torch.eye(2, dtype=DT)), **args)
    assert (c._model is not None) == (route == "fused")
    return c


def x0(v=(-3.0, -2.0)):
    return torch.tensor(v, dtype=DT, device=DEV)


ROUTES = ["fused", "stepped"]


@pytest.mark.parametrize("route", ROUTES)
def test_command_shape_dtype_and_progress(route):          # test_mppi.py:82-101
    c = make(route=route, num_samples=500)
    s = x0()
    a = c.command(s)
    assert a.shape == (2,) and a.dtype == DT and a.is_cuda
    c0 = quad_cost(s[None], None).item()
    for _ in range(5):
        a = c.command(s)
        s = lin_dyn(s[None], a[None])[0]
    assert quad_cost(s[None], None).item() < c0


@pytest.mark.parametrize("route", ROUTES)
def test_same_seed_same_actions(route):                    # :103-115
    a1 = make(route=route).command(x0((0.0, 0.0)))
    a2 = make(route=route).command(x0((0.0, 0.0)))
    assert torch.equal(a1, a2)


@pytest.mark.parametrize("route", ROUTES)
def test_bounds_and_one_sided_bounds(route):               # :117-140
    um = torch.tensor([0.5, 0.5], dtype=DT)
    c = make(route=route, u_min=-um, u_max=um)
    s = x0()
    for _ in range(10):
        a = c.command(s)
        s = lin_dyn(s[None], a[None])[0]
        assert (a.cpu().abs() <= um + 1e-6).all()
    c = make(route=route, u_max=torch.tensor([1.0, 1.0], dtype=DT))
    assert torch.allclose(c.u_min.cpu().double(), -torch.ones(2, dtype=DT))
    c = make(route=route, u_min=torch.tensor([-1.0, -1.0], dtype=DT))
    assert torch.allclose(c.u_max.cpu().double(), torch.ones(2, dtype=DT))
    assert (c.command(x0()).cpu().abs() <= 1 + 1e-6).all()


@pytest.mark.parametrize("route", ROUTES)
def test_terminal_cost_states_actions(route):              # :142-147, 241-260, 317-322
    c = make(route=route)
    c.command(x0((0.0, 0.0)))
    assert c.states is None and c.actions is None
    c = make(route=route, terminal=True, u_scale=2.0)
    a = c.command(x0((0.0, 0.0)))
    assert a.shape == (2,)
    assert c.states is not None and c.states.shape == (1, 100, 10, 2)
    assert c.actions is not None and c.actions.shape == (1, 100, 10, 2)
    # the stored states are the rollout of u_scale * actions from the start state
    st, ac = c.states[0].cpu(), c.actions[0].cpu()
    s = torch.zeros(100, 2, dtype=DT)
    for t in range(10):
        s = lin_dyn(s, 2.0 * ac[:, t])
        assert torch.allclose(s, st[:, t], atol=1e-9)


def test_step_dependent_plugins():                         # :149-159
    c = eng.MPPI(lambda s, a, t: lin_dyn(s, a), lambda s, a, t: quad_cost(s, a), 2, torch.eye(2, dtype=DT), num_samples=100,
                 horizon=10, device=DEV, step_dependent_dynamics=True)
    assert c.command(x0((-1.0, -1.0))).shape == (2,)


@pytest.mark.parametrize("route", ROUTES)
def test_options_abs_cost_null_action_upc_u_scale(route):  # :161-180
    assert make(route=route, noise_abs_cost=True).command(x0()).shape == (2,)
    assert make(route=route, sample_null_action=True).command(x0()).shape == (2,)
    c = make(route=route, u_per_command=3)
    a = c.command(x0())
    assert a.shape == (3, 2) and torch.equal(a, c.U[:3])


def test_rollout_samples_M():                              # :182-188
    c = make(route="stepped", rollout_samples=3, rollout_var_cost=0.1)
    assert c.command(x0((0.0, 0.0))).shape == (2,)


@pytest.mark.parametrize("route", ROUTES)
def test_get_rollouts(route):                              # :190-206
    c = make(route=route)
    s = x0((0.0, 0.0))
    c.command(s)
    assert c.get_rollouts(s, num_rollouts=5).shape == (5, c.T, 2)
    r = c.get_rollouts(s, num_rollouts=1, U=torch.zeros(c.T, 2, dtype=DT, device=DEV))
    assert torch.allclose(r, torch.zeros_like(r))


@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-12), (torch.float32, 2e-5)])
@pytest.mark.parametrize("model", ["pendulum", "linear"])
def test_get_rollouts_kernel_equals_plugin_replay(model, dtype, tol):   # mppi.py:425-448 on the registered-model route
    """Registered models replay the sequence in ONE kernel launch (mppi_rollout_states); the result must be the
    reference's loop `x <- dynamics(x, u_scale * U[t])` over the same model's torch callables."""
    torch.manual_seed(3)
    if model == "pendulum":
        m = eng.Pendulum()
        sigma, nu, lo, hi = torch.tensor(4.0, dtype=dtype), 1, -1.0, 1.0
    else:
        m = eng.LinearPoint.toy2d_nav()
        sigma, nu, lo, hi = torch.eye(2, dtype=dtype), 2, -3.0, 3.0
    term = m.terminal_cost if m.has_terminal else None
    c = eng.MPPI(m.dynamics, m.running_cost, 2, sigma, num_samples=64, horizon=12, device=DEV, u_scale=1.5,
                 terminal_state_cost=term)
    assert c._model is m

    def replay(x, U):
        out = []
        for t in range(U.shape[0]):
            x = m.dynamics(x, (c.u_scale * U[t]).expand(x.shape[0], -1))
            out.append(x)
        return torch.stack(out, dim=1)

    # (a) the controller's own plan, one start state broadcast to 5 rollouts
    s = torch.tensor([lo, hi], dtype=dtype, device=DEV)
    c.command(s)
    r = c.get_rollouts(s, num_rollouts=5)
    assert r.shape == (5, c.T, 2) and r.dtype == dtype
    assert (r - replay(s.view(1, 2).expand(5, 2), c.U)).abs().max().item() <= tol
    assert torch.equal(r[0], r[4])
    # (b) one start state per rollout, a caller-supplied sequence of a different length (ragged: 130 rollouts, T=7)
    S = torch.rand(130, 2, dtype=dtype, device=DEV) * (hi - lo) + lo
    Useq = torch.randn(7, nu, dtype=dtype, device=DEV)
    r = c.get_rollouts(S, num_rollouts=130, U=Useq)
    assert r.shape == (130, 7, 2)
    assert (r - replay(S, Useq)).abs().max().item() <= tol
    # (c) a single step, a single rollout
    r = c.get_rollouts(S[:1], num_rollouts=1, U=Useq[:1])
    assert (r - replay(S[:1], Useq[:1])).abs().max().item() <= tol
    with pytest.raises(ValueError):
        c.get_rollouts(S[:3], num_rollouts=5)


@pytest.mark.parametrize("route", ROUTES)
def test_change_horizon_reset_shift(route):                # :208-230, 293-315
    c = make(route=route, horizon=10)
    c.change_horizon(5)
    assert c.T == 5 and c.U.shape[0] == 5
    assert c.command(x0()).shape == (2,)
    c = make(route=route, horizon=5)
    c.change_horizon(10)
    assert c.T == 10 and c.U.shape == (10, 2)
    assert torch.allclose(c.U[5:], torch.zeros(5, 2, dtype=DT, device=DEV))
    c.command(x0())
    before = c.U.clone()
    c.reset()
    assert not torch.allclose(c.U, before)
    c.command(x0())
    before = c.U.clone()
    c.shift_nominal_trajectory()
    assert torch.allclose(c.U[-1], c.u_init) and torch.allclose(c.U[0], before[1])
    c.command(x0(), shift_nominal_trajectory=False)
    assert c.U.shape == before.shape


@pytest.mark.parametrize("route", ROUTES)
def test_no_shift_refinement_is_the_unshifted_update(route):
    """command(shift=False) must equal: un-shifted nominal + softmin update (checked against the oracle)."""
    from oracle import mppi_oracle as orc
    c = make(route=route)
    m = orc.LinearPointModel(B=B.tolist(), goal=GOAL.tolist())
    prob = orc.Problem(m.dynamics, m.running_cost, 2, torch.eye(2, dtype=DT), K=100, T=10)
    z = torch.randn(100, 10, 2, dtype=DT)
    U0 = c.U.cpu().clone()
    c.inject_noise(z)
    c.command(x0(), shift_nominal_trajectory=False)
    r = orc.mppi_command(prob, U0, torch.tensor([-3.0, -2.0], dtype=DT), z, shift=False)
    assert float((c.U.cpu() - r["U"]).abs().max()) < 1e-10


@pytest.mark.parametrize("route", ROUTES)
def test_per_sample_start_states(route):                   # :232-239  (K x nx) state
    c = make(route=route, num_samples=100)
    s = torch.randn(100, 2, dtype=DT, device=DEV)
    assert c.command(s).shape == (2,)
    from oracle import mppi_oracle as orc
    m = orc.LinearPointModel(B=B.tolist(), goal=GOAL.tolist())
    prob = orc.Problem(m.dynamics, m.running_cost, 2, torch.eye(2, dtype=DT), K=100, T=10)
    z = torch.randn(100, 10, 2, dtype=DT)
    U0 = c.U.cpu().clone()
    c.inject_noise(z)
    c.command(s)
    r = orc.mppi_command(prob, U0, s.cpu(), z)
    assert float((c.U.cpu() - r["U"]).abs().max()) < 1e-10


@pytest.mark.parametrize("route", ROUTES)
def test_cost_total_and_omega(route):                      # :262-274
    c = make(route=route)
    c.command(x0((0.0, 0.0)))
    assert c.cost_total.shape == (100,)
    assert abs(c.omega.sum().item() - 1.0) < 1e-5
    assert torch.allclose(c.cost_total_non_zero / c.cost_total_non_zero.sum(), c.omega)
    assert c.noise.shape == (100, 10, 2) and c.perturbed_action.shape == (100, 10, 2)
    assert "K=100" in c.get_params() and "T=10" in c.get_params()     # :324-328


def test_scalar_noise_sigma_1d_control():                  # :276-291
    c = eng.MPPI(lambda s, a: s + a, lambda s, a: (s[:, 0] - 1.0) ** 2, nx=1, noise_sigma=torch.tensor(1.0, dtype=DT),
                 num_samples=50, horizon=5, device=DEV)
    assert c.command(torch.tensor([0.0], dtype=DT, device=DEV)).shape == (1,)


# ---- SMPPI (:334-466) ------------------------------------------------------------------------------
@pytest.mark.parametrize("route", ROUTES)
def test_smppi_surface(route):
    c = make(eng.SMPPI, route=route, w_action_seq_cost=1.0, delta_t=1.0)
    assert c.command(x0()).shape == (2,)
    assert torch.equal(c.get_action_sequence(), c.action_sequence) and c.action_sequence.shape == (10, 2)
    assert "w=" in c.get_params() and "t=" in c.get_params()
    am = torch.tensor([0.5, 0.5], dtype=DT)
    c = make(eng.SMPPI, route=route, action_min=-am, action_max=am)
    s = x0()
    for _ in range(10):
        a = c.command(s)
        s = lin_dyn(s[None], a[None])[0]
        assert (a.cpu().abs() <= am + 1e-6).all()
    c.reset()
    assert torch.all(c.U == 0) and torch.all(c.action_sequence == 0)
    c.change_horizon(5)
    assert c.U.shape[0] == 5 and c.action_sequence.shape[0] == 5
    c.change_horizon(12)
    assert c.U.shape[0] == 12 and c.action_sequence.shape[0] == 12
    assert c.command(x0()).shape == (2,)
    assert make(eng.SMPPI, route=route, delta_t=0.1).command(x0()).shape == (2,)


@pytest.mark.parametrize("route", ROUTES)
def test_smppi_plans_are_smoother(route):                  # :379-407 (closed loop: finite) and :916-936 (open-loop plan)
    def run(c):
        s = x0()
        acts = []
        for _ in range(8):
            a = c.command(s)
            acts.append(a.cpu())
            s = lin_dyn(s[None], a[None])[0]
        return torch.stack(acts).diff(dim=0).abs().sum().item()
    assert np.isfinite(run(make(eng.SMPPI, route=route, num_samples=200, w_action_seq_cost=10.0)))
    assert np.isfinite(run(make(route=route, num_samples=200)))
    cm = make(route=route, num_samples=500, horizon=15)
    cm.command(x0())
    cs = make(eng.SMPPI, route=route, num_samples=500, horizon=15, w_action_seq_cost=10.0)
    cs.command(x0())
    assert cs.get_action_sequence().diff(dim=0).abs().sum().item() < cm.U.diff(dim=0).abs().sum().item() * 2.0


# ---- KMPPI (:468-585) ------------------------------------------------------------------------------
@pytest.mark.parametrize("route", ROUTES)
def test_kmppi_surface(route):
    c = make(eng.KMPPI, route=route, num_support_pts=5, kernel=eng.RBFKernel(sigma=1.0))
    assert c.command(x0()).shape == (2,)
    assert c.num_support_pts == 5 and c.theta.shape == (5, 2)
    assert make(eng.KMPPI, route=route).num_support_pts == 5                 # default T // 2
    assert make(eng.KMPPI, route=route, num_support_pts=5, kernel=eng.RBFKernel(sigma=2.0)).interpolation_kernel.sigma == 2.0
    traj, _ = c.deparameterize_to_trajectory_single(c.theta)
    assert traj.shape == (10, 2)
    trajb, _ = c.deparameterize_to_trajectory_batch(torch.randn(100, 5, 2, dtype=DT, device=DEV))
    assert trajb.shape == (100, 10, 2)
    um = torch.tensor([0.5, 0.5], dtype=DT)
    cb = make(eng.KMPPI, route=route, num_support_pts=5, u_min=-um, u_max=um)
    for _ in range(5):
        assert (cb.command(x0()).cpu().abs() <= um + 1e-6).all()
    c.command(x0())
    c.reset()
    assert torch.all(c.theta == 0)
    p = c.get_params()
    assert "num_support_pts=5" in p and "RBFKernel" in p
    s = x0()
    for _ in range(20):                                                     # :572-585
        a = c.command(s)
        s = lin_dyn(s[None], a[None])[0]
        assert torch.isfinite(a).all()


def test_rbf_kernel_closed_form():                         # :560-570
    k = eng.RBFKernel(sigma=1.0)
    t = torch.tensor([[0.0], [1.0]], dtype=DT)
    m = k(t, t)
    assert m.shape == (2, 2) and torch.allclose(m.diag(), torch.ones(2, dtype=DT), atol=1e-6)
    assert abs(m[0, 1].item() - np.exp(-0.5)) < 1e-6


def test_specific_action_sampler_hook():                   # :587-607
    class S(eng.SpecificActionSampler):
        def sample_trajectories(self, state, info):
            return torch.zeros(2, 10, 2, dtype=DT, device=DEV)
    s = S()
    c = eng.MPPI(lin_dyn, quad_cost, 2, torch.eye(2, dtype=DT), num_samples=100, horizon=10, device=DEV, specific_action_sampler=s)
    assert c.command(x0((0.0, 0.0))).shape == (2,)
    assert (s.start_idx, s.end_idx) == (0, 2)
    assert torch.all(c.perturbed_action[:2] == 0)


# ---- edge cases (:610-702) -------------------------------------------------------------------------
@pytest.mark.parametrize("route", ROUTES)
def test_edge_cases(route):
    assert make(route=route, num_samples=50, horizon=5).command(np.array([0.0, 0.0])).shape == (2,)      # numpy state
    assert make(route=route, num_samples=50, horizon=5).command([0.0, 0.0]).shape == (2,)                # list state
    assert make(route=route, num_samples=20, horizon=50).command(x0((0.0, 0.0))).shape == (2,)           # long horizon
    assert make(route=route, num_samples=1, horizon=5).command(x0((0.0, 0.0))).shape == (2,)             # K = 1
    c = make(route=route, num_samples=50, horizon=5, noise_sigma=torch.eye(2, dtype=torch.float32))
    assert c.command(torch.tensor([0.0, 0.0])).dtype == torch.float32                                    # fp32
    c = make(route=route, num_samples=50, horizon=5)
    c.compile()                                                                                           # :673-687
    s = x0((0.0, 0.0))
    for _ in range(5):
        a = c.command(s)
        s = lin_dyn(s[None], a[None])[0]
    assert torch.isfinite(s).all()


def test_high_dimensional_state_stepped():                 # :621-640  nx=10, nu=3
    nx, nu = 10, 3

    def dyn(s, a):
        d = torch.zeros_like(s)
        d[..., :nu] = a
        return s + d
    c = eng.MPPI(dyn, lambda s, a: (s ** 2).sum(-1), nx, torch.eye(nu, dtype=DT), num_samples=50, horizon=5, device=DEV)
    assert c.command(torch.randn(nx, dtype=DT, device=DEV)).shape == (nu,)


# ---- MPPI_Batched (:704-810) -----------------------------------------------------------------------
@pytest.mark.parametrize("route", ROUTES)
def test_mppi_batched_surface(route):
    torch.manual_seed(42)
    dyn, cost, _ = plugins(route)
    N = 4
    c = eng.MPPI_Batched(dyn, cost, 2, torch.eye(2, dtype=DT), num_envs=N, num_samples=100, horizon=10, device=DEV)
    s = torch.tensor([[-3.0, -2.0]] * N, dtype=DT, device=DEV)
    a = c.command(s)
    assert a.shape == (N, 2) and c.U.shape == (N, 10, 2)
    c0 = quad_cost(s, None).sum().item()
    for _ in range(8):
        a = c.command(s)
        s = lin_dyn(s, a)
    assert quad_cost(s, None).sum().item() < c0
    um = torch.tensor([0.3, 0.3], dtype=DT)
    cb = eng.MPPI_Batched(dyn, cost, 2, torch.eye(2, dtype=DT), num_envs=N, num_samples=100, horizon=10, device=DEV, u_max=um)
    assert (cb.command(s).cpu().abs() <= um + 1e-6).all()
    cb.compile()
    cu = eng.MPPI_Batched(dyn, cost, 2, torch.eye(2, dtype=DT), num_envs=N, num_samples=50, horizon=6, device=DEV, u_per_command=2)
    assert cu.command(s).shape == (N, 2, 2)


# ---- solution quality (:813-948): loose bounds, same as the reference's ------------------------------
def _loop(c, steps=20):
    s = x0()
    acc = 0.0
    for _ in range(steps):
        a = c.command(s)
        s = lin_dyn(s[None], a[None])[0]
        acc += quad_cost(s[None], None).item()
    return (GOAL.to(DEV) - s).norm().item(), acc


@pytest.mark.parametrize("route", ROUTES)
def test_quality_bounds(route):
    d, acc = _loop(make(route=route, num_samples=500, horizon=15))
    assert d < 2.0 and acc < 200.0                                                                       # :821-866
    d, acc = _loop(make(eng.KMPPI, route=route, num_samples=500, horizon=15, num_support_pts=5))
    assert d < 3.0
    d, acc = _loop(make(eng.SMPPI, route=route, num_samples=500, horizon=15, w_action_seq_cost=1.0))
    assert np.isfinite(d) and np.isfinite(acc)
    for T in (5, 15):
        d, acc = _loop(make(route=route, num_samples=500, horizon=T))
        assert d < 5.0 and acc < 300.0                                                                   # :884-896


def test_command_host_after_replan_returns_the_new_action():
    """ADVICE r1: a re-plan (any parameter setter) restarts the C plan; the pinned mailbox still holds the tags of the
    previous plan.  The mailbox tag is carried across plans, so command_host() after a re-plan waits for ITS kernel
    and returns the same action command() does."""
    import pytorch_mppi_b200 as eng
    pend = eng.Pendulum()

    def make():
        torch.manual_seed(0)
        U0 = torch.randn(15, 1) * 2
        return eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(4.0), num_samples=2048, horizon=15, U_init=U0,
                        u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda", rng_seed=5)
    a, b = make(), make()
    x = [3.0, 0.4]
    for lam in (1.0, 0.5, 2.0, 0.7):                 # exactly ONE command_host per plan: the stale tag would be 1 again
        a.lambda_ = lam
        b.lambda_ = lam
        ah = a.command_host(x)
        bd = b.command(x)
        assert torch.equal(ah, bd.cpu()), lam
        assert torch.equal(a.U, b.U)
    a.record_noise()                                  # another kind of re-plan
    b.record_noise()
    assert torch.equal(a.command_host(x), b.command(x).cpu())


def test_fused_command_equals_plan_command():
    """mppi_fused_command is a one-shot plan: on a C2-shaped fp32 controller (K=16384, T=30) it returns the same action,
    U and cost_total, bit for bit, as mppi_plan_command on an identically seeded twin."""
    import ctypes as C
    from pytorch_mppi_b200 import _cabi
    pend = eng.Pendulum()

    def make():
        torch.manual_seed(0)
        U0 = torch.randn(30, 1) * 2
        return eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(4.0), num_samples=16384, horizon=30, U_init=U0,
                        u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda", rng_seed=5)
    planned, oneshot = make(), make()
    assert oneshot.dtype == torch.float32
    oneshot._pack()
    p = oneshot._p
    stream = torch._C._cuda_getCurrentRawStream(oneshot.d.index)
    for x in ([3.0, 0.4], [2.5, -1.0], [0.1, 0.2]):
        want = planned.command(x)
        p.flags = oneshot._base_flags | _cabi.FLAG_SHIFT
        p.seed, p.offset = oneshot._next_rng()
        p.z, p.state_dev, p.host_mailbox = None, None, None
        for i, v in enumerate(x):
            p.state[i] = v
        action = torch.empty((1, 1), device="cuda", dtype=oneshot.dtype)
        p.action_out = action.data_ptr()
        _cabi.check(oneshot._lib.mppi_fused_command(C.byref(p), stream), "mppi_fused_command")
        torch.cuda.synchronize()
        assert torch.equal(action[0], want), x
        assert torch.equal(oneshot.U, planned.U) and torch.equal(oneshot._cost_buf, planned._cost_buf), x


def test_plan_rejects_a_batched_workspace_stride_too_small():
    """A plan checks the per-environment workspace stride before any launch: 256 bytes is less than the local record
    mailbox alone."""
    import ctypes as C
    m = eng.LinearPoint.unit_test_env()
    c = eng.MPPI_Batched(m.dynamics, m.running_cost, 2, torch.eye(2, dtype=DT), num_envs=4, num_samples=100, horizon=10,
                         device=DEV)
    c._pack()
    p = c._p
    assert p.env_ws_stride == c.launch_info.workspace_bytes and p.workspace_bytes >= 4 * p.env_ws_stride
    p.env_ws_stride = 256
    plan = C.c_void_p()
    assert c._lib.mppi_plan_create(C.byref(p), C.byref(plan)) == -3          # MPPI_ERR_WORKSPACE
    assert plan.value is None


def test_kmppi_change_horizon_rebuilds_interpolation():
    """ADVICE r1: KMPPI.change_horizon must rebuild W / Wshift / Tk / Hs for the new horizon (growing T used to read
    the old (T_old x S) matrix out of bounds)."""
    import pytorch_mppi_b200 as eng
    from oracle import mppi_oracle as orc
    dt = torch.float64
    lin = eng.LinearPoint.unit_test_env()
    K, S = 256, 4
    ctrl = eng.KMPPI(lin.dynamics, lin.running_cost, 2, torch.eye(2, dtype=dt), num_samples=K, horizon=8, num_support_pts=S,
                     kernel=eng.RBFKernel(sigma=1.5), device="cuda")
    ctrl.command([0.0, 0.0])
    for T in (14, 6):
        theta0 = ctrl.theta.clone()
        ctrl.change_horizon(T)
        assert ctrl.T == T and ctrl.U.shape == (T, 2) and ctrl.Hs.shape == (1, T)
        W, Wsh = orc.kernel_matrices(T, S, lambda a, b: orc.rbf_kernel(a, b, 1.5), dt)
        assert torch.allclose(ctrl._W.cpu(), W, atol=1e-12) and torch.allclose(ctrl._Wshift.cpu(), Wsh, atol=1e-12)
        assert torch.equal(ctrl.theta, theta0)
        assert torch.allclose(ctrl.U.cpu(), W @ theta0.cpu(), atol=1e-12)
        # and a command on the new horizon matches the oracle
        olin = orc.LinearPointModel(B=lin.B, goal=lin.goal, dtype=dt)
        prob = orc.Problem(olin.dynamics, olin.running_cost, 2, torch.eye(2, dtype=dt), K=K, T=T)
        z = torch.randn(K, S, 2, dtype=dt)
        ctrl.inject_noise(z)
        U_before, th_before = ctrl.U.cpu().clone(), ctrl.theta.cpu().clone()
        ctrl.command([0.5, -0.5])
        r = orc.kmppi_command(prob, U_before, th_before, torch.tensor([0.5, -0.5], dtype=dt), z, W, Wsh)
        assert float((ctrl.theta.cpu() - r["theta"]).abs().max()) < 1e-10
        assert float((ctrl.U.cpu() - r["U"]).abs().max()) < 1e-10


def test_compile_fallback_applies_exactly_one_command():
    """ADVICE r1: a plugin that is not capture-safe makes compile() fall back to the eager stepped route; the warm-up
    commands of the failed capture must be undone, so the nominal moves by exactly one command.  Runs in its own process:
    a CUDA-graph capture that dies inside a plugin can leave process-wide torch state (the default generator) unusable,
    and the rest of this suite must not depend on the repair."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = r'''
import sys, torch
sys.path.insert(0, %r)
import pytorch_mppi_b200 as eng
lin = eng.LinearPoint.unit_test_env()
dt = torch.float64
def bad_cost(s, a):
    c = lin.running_cost(s, a)
    float(c[0])                      # host sync: illegal during stream capture
    return c
def make(cost):
    torch.manual_seed(3)
    U0 = torch.randn(7, 2, dtype=dt) * 0.1
    return eng.MPPI(lambda s, a: lin.dynamics(s, a), cost, 2, torch.eye(2, dtype=dt), num_samples=128, horizon=7,
                    U_init=U0, device="cuda", rng_seed=11)
ref_ctrl = make(lambda s, a: lin.running_cost(s, a))
bad = make(bad_cost)
bad.compile()
a0 = ref_ctrl.command([1.0, 1.0])
a1 = bad.command([1.0, 1.0])          # capture fails -> eager; one command applied
assert bad._graph_mode is False
assert torch.allclose(a0, a1, atol=1e-12) and torch.allclose(ref_ctrl.U, bad.U, atol=1e-12), (a0, a1)
assert torch.allclose(ref_ctrl.command([0.9, 1.1]), bad.command([0.9, 1.1]), atol=1e-12)
print("FALLBACK_OK")
try:
    torch.randn(4, device="cuda")
    print("GENERATOR_OK")
except RuntimeError as e:
    print("GENERATOR_BROKEN", e)
''' % root
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert "FALLBACK_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
    assert "GENERATOR_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
