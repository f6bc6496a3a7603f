"""CPU: the tuner (`pytorch_mppi_b200.autotune`).  CMA-ES on test functions, the parameters and the sequential
`Autotune` on a stub controller, and `ClosedLoopEvaluation` / `BatchedAutotune` with `MPPI_Batched` replaced by a stub
that records what it is given: the environment layout c * S + s, the per-environment settings, the incumbent slot and
every refusal."""
import math
import types

import numpy as np
import pytest
import torch

import pytorch_mppi_b200 as eng
from pytorch_mppi_b200 import autotune
from pytorch_mppi_b200.mppi import ClosedLoopResult


# ---- CMA-ES ---------------------------------------------------------------------------------------------------------
def _run(f, x0, sigma, gens, seed=1, popsize=None):
    es = autotune.CMAES(x0, sigma, popsize, np.random.default_rng(seed))
    trace = []
    for _ in range(gens):
        X = es.ask()
        trace.append(X)
        es.tell(X, np.array([f(x) for x in X]))
    return es, trace


def sphere(x):
    return float(np.sum(x ** 2))


_Q = np.linalg.qr(np.random.default_rng(5).standard_normal((8, 8)))[0]


def rotated_ellipsoid(x):
    y = _Q @ x
    return float(np.sum(10.0 ** (6 * np.arange(8) / 7) * y ** 2))


@pytest.mark.parametrize("f,gens", [(sphere, 400), (rotated_ellipsoid, 1500)])
def test_cmaes_converges(f, gens):
    es = autotune.CMAES(np.full(8, 2.0), 1.0, None, np.random.default_rng(3))
    for _ in range(gens):
        X = es.ask()
        es.tell(X, np.array([f(x) for x in X]))
        if es.best_f < 1e-10:
            break
    assert es.best_f < 1e-10, f"{f.__name__}: best {es.best_f:.3e} after {es.gen} generations"
    assert f(es.best_x) == es.best_f


def test_cmaes_same_seed_same_trajectory():
    _, a = _run(sphere, np.ones(5), 0.5, 30, seed=7)
    _, b = _run(sphere, np.ones(5), 0.5, 30, seed=7)
    _, c = _run(sphere, np.ones(5), 0.5, 30, seed=8)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    assert not np.array_equal(a[-1], c[-1])


def test_cmaes_uses_ranks_only():
    ea, a = _run(sphere, np.ones(8), 0.5, 40)
    eb, b = _run(lambda x: math.exp(sphere(x)), np.ones(8), 0.5, 40)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    assert np.array_equal(ea.best_x, eb.best_x)


def test_cmaes_tell_refuses_wrong_shapes():
    es = autotune.CMAES(np.zeros(3), 1.0, 6, np.random.default_rng(0))
    X = es.ask()
    assert X.shape == (6, 3)
    with pytest.raises(ValueError, match="shape"):
        es.tell(X[:5], np.zeros(5))
    with pytest.raises(ValueError, match="shape"):
        es.tell(X, np.zeros(5))
    with pytest.raises(ValueError, match="shape"):
        es.tell(X[:, :2], np.zeros(6))
    with pytest.raises(ValueError, match="NaN"):
        es.tell(X, np.array([0, 1, 2, np.nan, 4, 5.0]))
    assert es.gen == 0


# ---- parameters and the sequential Autotune on a stub controller ----------------------------------------------------
class _Ctrl:
    """What the parameters read and write on a controller."""

    def __init__(self, nu=2, T=10):
        self.d, self.dtype, self.nu, self.T = torch.device("cpu"), torch.float64, nu, T
        self.noise_sigma = torch.diag(torch.arange(1.0, nu + 1, dtype=torch.float64))
        self.noise_mu = torch.zeros(nu, dtype=torch.float64)
        self.lambda_ = 1.5
        self.horizons = []

    def change_horizon(self, h):
        self.horizons.append(h)
        self.T = h


def _params(c):
    return [autotune.SigmaParameter(c), autotune.HorizonParameter(c), autotune.LambdaParameter(c)]


def test_flatten_unflatten_round_trip_in_the_references_order():
    c = _Ctrl()
    tuner = autotune.Autotune(_params(c), evaluate_fn=lambda: None, optimizer=autotune.CMAESOpt(seed=0))
    x = tuner.flatten_params()
    assert x.tolist() == [1.0, 2.0, 10.0, 1.5]                 # sigma0, sigma1, horizon, lambda
    v = tuner.unflatten_params(np.array([0.5, 3.0, 7.4, 0.25]))
    assert torch.equal(v["sigma"], torch.tensor([0.5, 3.0], dtype=torch.float64))
    assert v["horizon"] == 7 and v["lambda"] == 0.25
    assert torch.equal(c.noise_sigma, torch.diag(torch.tensor([0.5, 3.0], dtype=torch.float64)))
    assert c.T == 7 and c.lambda_ == 0.25
    assert tuner.flatten_params().tolist() == [0.5, 3.0, 7.0, 0.25]
    assert tuner.config_to_params({"sigma0": 1.0, "sigma1": 2.0, "horizon": 5, "lambda": 3.0})["horizon"] == 5


def test_eps_clamps_rounding_and_mu():
    c = _Ctrl()
    s, h, lam, mu = (autotune.SigmaParameter(c), autotune.HorizonParameter(c), autotune.LambdaParameter(c),
                     autotune.MuParameter(c))
    assert s.ensure_valid_value(np.array([-1.0, 2.0])).tolist() == [s.eps, 2.0]
    assert lam.ensure_valid_value(np.array([-3.0])) == lam.eps and lam.ensure_valid_value(0.5) == 0.5
    assert h.ensure_valid_value(np.array([-2.0])) == 1 and h.ensure_valid_value(np.array([4.6])) == 5
    h.max_horizon = 8
    assert h.ensure_valid_value(np.array([30.0])) == 8
    mu.apply_parameter_value(np.array([0.5, -0.5]))            # the engine's noise_mu (the reference's does nothing)
    assert c.noise_mu.tolist() == [0.5, -0.5]
    assert s.get_config_from_parameter_value(torch.tensor([1.0, 2.0])) == {"sigma0": 1.0, "sigma1": 2.0}


def _quadratic_evaluate(c):
    """costs = distance of (sigma, lambda) from (0.7, 0.7, 2.0), one 'episode' per start"""
    def evaluate():
        v = torch.cat((torch.diagonal(c.noise_sigma), torch.tensor([c.lambda_], dtype=torch.float64)))
        cost = ((v - torch.tensor([0.7, 0.7, 2.0], dtype=torch.float64)) ** 2).sum()
        return autotune.EvaluationResult(cost.repeat(3), torch.zeros(3, 4, 2))
    return evaluate


def test_optimize_step_applies_the_best_ever_point_and_logs():
    c = _Ctrl()
    calls = []
    ev = _quadratic_evaluate(c)

    def evaluate():
        calls.append((torch.diagonal(c.noise_sigma).tolist(), c.lambda_))
        return ev()
    tuner = autotune.Autotune([autotune.SigmaParameter(c), autotune.LambdaParameter(c)], evaluate,
                              optimizer=autotune.CMAESOpt(population=6, sigma=0.3, seed=0))
    res = tuner.optimize_step()
    assert len(calls) == 7                           # 6 candidates, then the best point again (as the reference)
    assert res.iteration == 0 and set(res.params) == {"sigma", "lambda"}
    best = tuner.optim.optim.best_x
    assert calls[-1] == ([max(best[0], 1e-4), max(best[1], 1e-4)], max(best[2], 1e-4))
    assert res.params["lambda"] == c.lambda_ == max(best[2], 1e-4)
    for _ in range(40):
        tuner.optimize_step()
    assert [r.iteration for r in tuner.results] == list(range(41))
    b = tuner.get_best_result()
    assert b.costs.mean().item() == min(r.costs.mean().item() for r in tuner.results) < 1e-3
    assert abs(c.lambda_ - 2.0) < 0.05


def _gain_parameter():
    class Gain(autotune.TunableParameter):
        def __init__(self):
            self.v = 1.0

        @staticmethod
        def name():
            return "gain"

        def dim(self):
            return 1

        def get_current_parameter_value(self):
            return self.v

        def ensure_valid_value(self, value):
            return float(np.asarray(value).reshape(-1)[0])

        def apply_parameter_value(self, value):
            self.v = self.ensure_valid_value(value)

        def attach_to_state(self, state):
            pass
    return Gain()


def test_sequential_autotune_accepts_a_user_parameter():
    g = _gain_parameter()
    tuner = autotune.Autotune([g], lambda: autotune.EvaluationResult(torch.tensor([(g.v - 3.0) ** 2]), torch.zeros(1)),
                              optimizer=autotune.CMAESOpt(population=8, sigma=1.0, seed=2))
    tuner.optimize_all(30)
    assert abs(g.v - 3.0) < 1e-2


# ---- ClosedLoopEvaluation / BatchedAutotune with MPPI_Batched stubbed -----------------------------------------------
class _Batched:
    """Records the constructor arguments and every call; episode costs depend on each environment's settings."""
    made = []

    def __init__(self, dynamics, running_cost, nx, noise_sigma, num_envs, **kw):
        self.nx, self.N, self.kw, self.calls = nx, num_envs, kw, []
        self.nu = noise_sigma.shape[0]
        self.T = kw["horizon"]
        self.sigma0, self.lam0 = noise_sigma, kw["lambda_"]
        self._U = torch.zeros(num_envs, self.T, self.nu, dtype=torch.float64)
        _Batched.made.append(self)

    @property
    def U(self):
        return self._U

    @U.setter
    def U(self, value):
        self._U = torch.as_tensor(value).reshape(self.N, self.T, self.nu).clone()
        self.calls.append(("U", self._U.clone()))

    def set_env_params(self, **kw):
        self.calls.append(("set_env_params", kw))
        self.env = kw

    def set_env_horizon(self, h):
        self.calls.append(("set_env_horizon", None if h is None else h.clone()))
        self.h = h

    def run_closed_loop(self, x0, steps, plant_params=None):
        self.calls.append(("run_closed_loop", x0.clone(), steps, plant_params))
        lam = self.env.get("lambda_", torch.full((self.N,), float(self.lam0), dtype=torch.float64))
        sig = self.env.get("noise_sigma", self.sigma0.expand(self.N, self.nu, self.nu))
        h = self.h if self.h is not None else torch.full((self.N,), self.T)
        per_env = (lam - 2.0) ** 2 + (torch.diagonal(sig, dim1=1, dim2=2)[:, 0] - 0.5) ** 2 + (h.double() - 6) ** 2
        per_env = per_env + 1e-3 * x0[:, 0].double()                    # the start state matters too
        costs = (per_env / steps).to(torch.float32).expand(steps, self.N).clone()
        states = (x0.unsqueeze(0) + torch.arange(steps + 1).view(-1, 1, 1)).to(torch.float32)
        return ClosedLoopResult(states, torch.zeros(steps, self.N, self.nu), costs)


def _mppi(monkeypatch, model=None, T=10, **over):
    """A plain MPPI as far as ClosedLoopEvaluation and the parameters read it (no device)."""
    monkeypatch.setattr(autotune, "MPPI_Batched", _Batched)
    _Batched.made = []
    c = eng.MPPI.__new__(eng.MPPI)
    model = eng.Pendulum() if model is None else model
    c.d, c.dtype, c.nx, c.nu, c.T, c.K = torch.device("cpu"), torch.float32, model.nx, 1, T, 256
    c._model, c.M, c.terminal_state_cost, c.u_per_command, c._world = model, 1, None, 1, 1
    c.F, c.running_cost, c._rng_seed, c._tile_memory, c.noise_abs_cost = model.dynamics, model.running_cost, 5, "shared", False
    c._lambda, c._u_scale, c._noise_mu = 1.0, 1.0, torch.zeros(1)
    c._u_min, c._u_max, c._u_init = torch.tensor(-2.0), torch.tensor(2.0), torch.tensor([0.25])
    c._set_sigma(torch.eye(1))
    c._Ubuf = torch.arange(1.0, T + 1)
    c._dirty = False
    for k, v in over.items():
        setattr(c, k, v)
    # change_horizon without a device: the nominal buffer only
    c._resize_horizon = types.MethodType(lambda self, h, U: (setattr(self, "T", int(h)), setattr(self, "_Ubuf", U.reshape(-1).clone())), c)
    return c


def test_layout_settings_and_incumbent(monkeypatch):
    c = _mppi(monkeypatch, T=10)
    x0 = torch.tensor([[0.0, 0.0], [1.0, 0.0], [2.0, 0.0]])
    ev = autotune.ClosedLoopEvaluation(c, x0, 7, max_horizon=12)
    tuner = autotune.BatchedAutotune([autotune.SigmaParameter(c), autotune.LambdaParameter(c), autotune.HorizonParameter(c)],
                                     ev, optimizer=autotune.CMAESOpt(4, 0.5, seed=0))
    inc = tuner.optim.incumbent()
    assert inc.tolist() == [1.0, 1.0, 10.0]
    X = tuner.optim.optim.ask()
    tuner.optim.optim.ask = lambda: X                # the step runs on these candidates
    res = tuner.optimize_step()
    (b,) = _Batched.made
    assert b.N == 5 * 3 and b.T == 12 and b.kw["num_samples"] == 256 and b.kw["rng_seed"] == 5
    assert b.kw["u_per_command"] == 1 and b.kw["tile_memory"] == "shared" and b.kw["u_scale"] == 1.0
    names = [k[0] for k in b.calls]
    assert names == ["set_env_params", "U", "set_env_horizon", "run_closed_loop"]
    pts = np.concatenate((X, inc[None]))
    env = b.calls[0][1]
    assert set(env) == {"noise_sigma", "lambda_"}
    for e in range(15):                              # environment c * S + s is candidate c
        cnd = e // 3
        assert env["lambda_"][e].item() == max(pts[cnd, 1], 1e-4)
        assert env["noise_sigma"][e].item() == pytest.approx(max(pts[cnd, 0], 1e-4), rel=1e-6)
        assert b.calls[2][1][e].item() == min(max(round(pts[cnd, 2]), 1), 12)
    assert b.calls[2][1].dtype == torch.int32
    # every environment starts from ctrl's nominal, extended with u_init to max_horizon
    U = b.calls[1][1]
    start = torch.cat((torch.arange(1.0, 11), torch.full((2,), 0.25))).view(12, 1)
    assert all(torch.equal(U[e], start) for e in range(15))
    x_run, steps, plant = b.calls[3][1:]
    assert steps == 7 and plant is None and torch.equal(x_run, x0.repeat(5, 1))
    # the returned result is the best point's, from the same launch; ctrl carries its settings
    costs = (((torch.tensor(pts[:, 1]).clamp(min=1e-4) - 2) ** 2 + (torch.tensor(pts[:, 0]).clamp(min=1e-4) - 0.5) ** 2
             + (torch.tensor([min(max(round(v), 1), 12) for v in pts[:, 2]]).double() - 6) ** 2))
    best = int(torch.argmin(costs[:4]))
    assert res.costs.shape == (3,) and res.rollouts.shape == (3, 8, 2)
    assert torch.allclose(res.costs.double(), costs[best] + 1e-3 * x0[:, 0].double(), rtol=1e-5)
    assert torch.equal(res.rollouts[:, 0], x0)
    assert c.lambda_ == max(pts[best, 1], 1e-4) and c.T == min(max(round(pts[best, 2]), 1), 12)
    assert tuner.optim.incumbent().tolist() == X[best].tolist()
    assert res.iteration == 0 and res.params["horizon"] == c.T


def test_incumbent_result_when_no_candidate_improves(monkeypatch):
    c = _mppi(monkeypatch)
    ev = autotune.ClosedLoopEvaluation(c, torch.zeros(2, 2), 3)
    tuner = autotune.BatchedAutotune([autotune.LambdaParameter(c)], ev, optimizer=autotune.CMAESOpt(4, 0.5, seed=0))
    tuner.optimize_step()
    es = tuner.optim.optim
    es.best_f = -1.0                                 # nothing told from now on can beat it
    inc = es.best_x.copy()
    res = tuner.optimize_step()
    b = _Batched.made[0]
    lam = b.env["lambda_"]
    assert lam[-1].item() == lam[-2].item() == max(inc[0], 1e-4)     # the last candidate slot (both starts) is the incumbent
    assert c.lambda_ == max(inc[0], 1e-4)
    assert b.calls[-1][0] == "run_closed_loop"
    assert torch.allclose(res.costs.double(), (lam[-2:] - 2) ** 2 + 0.25 + 16, rtol=1e-5)
    # a horizon that is not tuned stays the controller's: with T == max_horizon, no horizons are set
    assert b.calls[-2] == ("set_env_horizon", None)


def test_plant_params_follow_the_start_states(monkeypatch):
    c = _mppi(monkeypatch)
    n = len(c._model.param_blob())
    rows = torch.arange(2.0 * n).view(2, n)
    ev = autotune.ClosedLoopEvaluation(c, torch.zeros(2, 2), 3, plant_params=rows, max_horizon=14)
    tuner = autotune.BatchedAutotune([autotune.LambdaParameter(c)], ev, optimizer=autotune.CMAESOpt(3, 0.5, seed=0))
    tuner.optimize_step()
    b = _Batched.made[0]
    plant = b.calls[-1][3]
    assert torch.equal(plant, rows.double().repeat(4, 1))
    # horizon not tuned, max_horizon > T: every environment rolls out the controller's T
    assert b.calls[-2][1].tolist() == [10] * 8


@pytest.mark.parametrize("change,why", [
    (dict(_model=None), "stepped route"),
    (dict(M=2), "rollout_samples"),
    (dict(terminal_state_cost=lambda s, a: s), "terminal cost"),
    (dict(u_per_command=2), "u_per_command"),
    (dict(_world=2), "sharded"),
])
def test_evaluation_refusals(monkeypatch, change, why):
    c = _mppi(monkeypatch, **change)
    with pytest.raises(ValueError, match=why):
        autotune.ClosedLoopEvaluation(c, torch.zeros(2, 2), 3)


def test_evaluation_refuses_other_controllers_and_models(monkeypatch):
    c = _mppi(monkeypatch)
    with pytest.raises(ValueError, match="plain MPPI"):
        autotune.ClosedLoopEvaluation(types.SimpleNamespace(**vars(c)), torch.zeros(2, 2), 3)
    s = eng.SMPPI.__new__(eng.SMPPI)
    s.__dict__.update(vars(c))
    with pytest.raises(ValueError, match="SMPPI"):
        autotune.ClosedLoopEvaluation(s, torch.zeros(2, 2), 3)
    net = torch.nn.Sequential(torch.nn.Linear(3, 32), torch.nn.Tanh(), torch.nn.Linear(32, 32), torch.nn.Tanh(),
                              torch.nn.Linear(32, 2))
    with pytest.raises(ValueError, match="PendulumMLP"):
        autotune.ClosedLoopEvaluation(_mppi(monkeypatch, model=eng.PendulumMLP(net)), torch.zeros(2, 2), 3)
    with pytest.raises(ValueError, match="start_states"):
        autotune.ClosedLoopEvaluation(c, torch.zeros(2, 3), 3)
    with pytest.raises(ValueError, match="steps"):
        autotune.ClosedLoopEvaluation(c, torch.zeros(2, 2), 0)
    with pytest.raises(ValueError, match="max_horizon"):
        autotune.ClosedLoopEvaluation(c, torch.zeros(2, 2), 3, max_horizon=5)
    with pytest.raises(ValueError, match="plant_params"):
        autotune.ClosedLoopEvaluation(c, torch.zeros(2, 2), 3, plant_params=torch.zeros(3, 2))
    assert _Batched.made == []


def test_batched_autotune_refuses_a_user_parameter(monkeypatch):
    c = _mppi(monkeypatch)
    ev = autotune.ClosedLoopEvaluation(c, torch.zeros(2, 2), 3)
    g = _gain_parameter()
    with pytest.raises(ValueError, match="Gain"):
        autotune.BatchedAutotune([autotune.LambdaParameter(c), g], ev, optimizer=autotune.CMAESOpt(4, 0.5, seed=0))
    assert _Batched.made == []
