"""Tuning of controller parameters, with the API of the reference's `pytorch_mppi.autotune`.

`Autotune(params_to_tune, evaluate_fn, optimizer=CMAESOpt())` evaluates candidates one at a time through the user's
`evaluate_fn`, as the reference does, and works with every controller.  `BatchedAutotune` evaluates a whole CMA-ES
generation as ONE `MPPI_Batched.run_closed_loop` call on the GPU (`ClosedLoopEvaluation`): every candidate, and the
best point found before the generation, from every start state, on the same noise.

CMA-ES is implemented here in numpy (Hansen, "The CMA Evolution Strategy: A Tutorial", arXiv:1604.00772), so the `cma`
package is not needed; it runs on the host and is a few small matrix operations per generation.

Differences from the reference:
- `MuParameter` sets the controller's `noise_mu`.  The reference only rebuilds `noise_dist`, which its sampler does not
  read, so tuning mu there changes nothing.
- `BatchedAutotune.optimize_step` returns the result of the best point from the generation's own launch; the reference
  evaluates that point a second time after `tell`.
- Horizons are rounded and clamped to [1, max_horizon] (`ClosedLoopEvaluation`'s `max_horizon`, the longest horizon its
  batched controller can roll out).
"""
from __future__ import annotations

import abc
import logging
import math
import typing

import numpy as np
import torch

from .mppi import MPPI, MPPI_Batched
from . import _cabi

logger = logging.getLogger(__name__)


class EvaluationResult(typing.NamedTuple):
    costs: torch.Tensor          # (S) cost of each evaluated episode / trajectory
    rollouts: torch.Tensor       # (S, H, nx) their states
    params: dict = None          # parameter values, filled in by the tuner
    iteration: int = None        # filled in by the tuner


# ---- CMA-ES ---------------------------------------------------------------------------------------------------------
class CMAES:
    """(mu/mu_w, lambda)-CMA-ES with the tutorial's default weights and learning rates (arXiv:1604.00772, table 1):
    rank-one and rank-mu covariance updates, cumulative step-size adaptation with the h_sigma stall, and one
    eigendecomposition of C per generation.  Only the ranks of the costs are used.  `best_x` / `best_f` track the best
    point ever told; before the first `tell`, `best_x` is the start point."""

    def __init__(self, x0, sigma0, popsize=None, rng: typing.Optional[np.random.Generator] = None):
        self.mean = np.asarray(x0, dtype=np.float64).reshape(-1).copy()
        n = self.n = self.mean.size
        if n < 1 or not sigma0 > 0:
            raise ValueError("CMAES needs at least one dimension and sigma0 > 0")
        self.lam = int(popsize) if popsize else 4 + int(3 * math.log(n))
        if self.lam < 2:
            raise ValueError(f"CMAES needs a population of at least 2, got {self.lam}")
        self.mu = self.lam // 2
        w = math.log((self.lam + 1) / 2) - np.log(np.arange(1, self.mu + 1))
        self.w = w / w.sum()
        self.mueff = 1.0 / float(np.sum(self.w ** 2))
        me = self.mueff
        self.cc = (4 + me / n) / (n + 4 + 2 * me / n)
        self.cs = (me + 2) / (n + me + 5)
        self.c1 = 2 / ((n + 1.3) ** 2 + me)
        self.cmu = min(1 - self.c1, 2 * (me - 2 + 1 / me) / ((n + 2) ** 2 + me))
        self.ds = 1 + 2 * max(0.0, math.sqrt((me - 1) / (n + 1)) - 1) + self.cs
        self.chin = math.sqrt(n) * (1 - 1 / (4 * n) + 1 / (21 * n * n))
        self.sigma = float(sigma0)
        self.C = np.eye(n)
        self.B = np.eye(n)
        self.D = np.ones(n)
        self.pc = np.zeros(n)
        self.ps = np.zeros(n)
        self.gen = 0
        self.rng = rng if rng is not None else np.random.default_rng()
        self.best_x, self.best_f = self.mean.copy(), math.inf
        self.best_index = None           # row of the last tell's X that became best_x (None: it stayed)

    def ask(self) -> np.ndarray:
        """(lambda, n) candidates x = m + sigma * B D z, z ~ N(0, I)."""
        z = self.rng.standard_normal((self.lam, self.n))
        return self.mean + self.sigma * (z * self.D) @ self.B.T

    def tell(self, X, f) -> None:
        X = np.asarray(X, dtype=np.float64)
        f = np.asarray(f, dtype=np.float64)
        if X.shape != (self.lam, self.n) or f.shape != (self.lam,):
            raise ValueError(f"tell expects X of shape {(self.lam, self.n)} and f of shape {(self.lam,)}, "
                             f"got {X.shape} and {f.shape}")
        if np.isnan(f).any():
            raise ValueError("tell: a cost is NaN")
        order = np.argsort(f, kind="stable")
        self.best_index = None
        if f[order[0]] < self.best_f:
            self.best_f, self.best_x, self.best_index = float(f[order[0]]), X[order[0]].copy(), int(order[0])
        n, cs, cc, c1, cmu = self.n, self.cs, self.cc, self.c1, self.cmu
        y = (X[order[: self.mu]] - self.mean) / self.sigma          # selected steps, (mu, n)
        yw = self.w @ y
        self.mean = self.mean + self.sigma * yw
        c_inv_sqrt_yw = self.B @ ((self.B.T @ yw) / self.D)
        self.ps = (1 - cs) * self.ps + math.sqrt(cs * (2 - cs) * self.mueff) * c_inv_sqrt_yw
        ps_norm = float(np.linalg.norm(self.ps))
        hsig = ps_norm / math.sqrt(1 - (1 - cs) ** (2 * (self.gen + 1))) < (1.4 + 2 / (n + 1)) * self.chin
        self.pc = (1 - cc) * self.pc + (math.sqrt(cc * (2 - cc) * self.mueff) * yw if hsig else 0.0)
        dh = 0.0 if hsig else cc * (2 - cc)
        rank_mu = (y.T * self.w) @ y
        self.C = (1 + c1 * dh - c1 - cmu * self.w.sum()) * self.C + c1 * np.outer(self.pc, self.pc) + cmu * rank_mu
        self.sigma *= math.exp((cs / self.ds) * (ps_norm / self.chin - 1))
        self.C = (self.C + self.C.T) / 2
        d2, self.B = np.linalg.eigh(self.C)
        self.D = np.sqrt(np.maximum(d2, 1e-300))
        self.gen += 1


# ---- optimizers -----------------------------------------------------------------------------------------------------
class Optimizer:
    def __init__(self):
        self.tuner: typing.Optional[Autotune] = None
        self.optim = None

    @abc.abstractmethod
    def setup_optimization(self) -> None:
        """Create the search state from the tuner's current parameters."""

    @abc.abstractmethod
    def optimize_step(self) -> EvaluationResult:
        """One step of the search; returns the evaluation of the parameters it leaves applied."""

    def optimize_all(self, iterations) -> EvaluationResult:
        res = None
        for _ in range(iterations):
            res = self.optimize_step()
        return res


class CMAESOpt(Optimizer):
    """CMA-ES (`CMAES`) from the tuner's current parameters with step size `sigma`; `seed` seeds its numpy Generator.
    Each step asks `population` candidates, has the tuner evaluate them (`evaluate_candidates`), tells their mean costs
    and applies the best point found so far to the controller."""

    def __init__(self, population=10, sigma=0.1, seed=None):
        self.population = population
        self.sigma = sigma
        self.seed = seed
        super().__init__()

    def setup_optimization(self):
        self.optim = CMAES(self.tuner.flatten_params(), self.sigma, self.population, np.random.default_rng(self.seed))

    def incumbent(self) -> np.ndarray:
        """The best point before the next generation (the start point until a generation was told)."""
        return self.optim.best_x.copy()

    def optimize_step(self):
        X = self.optim.ask()
        costs, results = self.tuner.evaluate_candidates(X)
        self.optim.tell(X, costs)
        self.tuner.unflatten_params(self.optim.best_x)
        return self.tuner.result_of_best(results, self.optim.best_index)


# ---- parameters -----------------------------------------------------------------------------------------------------
class TunableParameter(abc.ABC):
    """A tunable value, with a reference to the object that holds it.  `env_keyword` names the per-environment setting
    of a batched evaluation that carries it (`MPPI_Batched.set_env_params` keyword, or "horizon" for
    `set_env_horizon`); None: the parameter can only be tuned with the sequential `Autotune`."""
    env_keyword = None

    @staticmethod
    @abc.abstractmethod
    def name():
        """The parameter's name"""

    @abc.abstractmethod
    def dim(self):
        """Number of values"""

    @abc.abstractmethod
    def get_current_parameter_value(self):
        """The value the object holds now"""

    @abc.abstractmethod
    def ensure_valid_value(self, value):
        """The valid value closest in intent to `value`"""

    @abc.abstractmethod
    def apply_parameter_value(self, value):
        """Give the object this value"""

    @abc.abstractmethod
    def attach_to_state(self, state: dict):
        """Attach to a new object (as __init__ would)"""

    def env_values(self, values):
        """The (P, ...) tensor of per-environment values for the P given valid values (see `env_keyword`)."""
        raise NotImplementedError(f"{type(self).__name__} has no per-environment setting")

    def get_parameter_value_from_config(self, config):
        return config[self.name()]

    def get_config_from_parameter_value(self, value):
        return {self.name(): value}


class MPPIParameter(TunableParameter, abc.ABC):
    def __init__(self, mppi: MPPI, dim=None):
        self.mppi = mppi
        self._dim = dim
        if mppi is not None:
            self.d, self.dtype = mppi.d, mppi.dtype
            if dim is None:
                self._dim = mppi.nu

    def attach_to_state(self, state: dict):
        self.mppi = state["mppi"]
        self.d, self.dtype = self.mppi.d, self.mppi.dtype


def _tensor(value, device, dtype):
    if torch.is_tensor(value):
        return value.detach().to(device, dtype).clone().reshape(-1)
    return torch.as_tensor(np.asarray(value, dtype=np.float64), dtype=dtype, device=device).reshape(-1)


def _scalar(value):
    if torch.is_tensor(value) or isinstance(value, np.ndarray):
        value = value.reshape(-1)[0]
    return float(value)


class _VectorConfig:
    """Config entries name0, name1, ... for a vector parameter."""

    def get_parameter_value_from_config(self, config):
        return torch.tensor([config[f"{self.name()}{i}"] for i in range(self.dim())], dtype=self.dtype, device=self.d)

    def get_config_from_parameter_value(self, value):
        return {f"{self.name()}{i}": value[i].item() for i in range(self.dim())}


class SigmaParameter(_VectorConfig, MPPIParameter):
    """The diagonal of the noise covariance; values below `eps` are raised to it."""
    eps = 0.0001
    env_keyword = "noise_sigma"

    @staticmethod
    def name():
        return "sigma"

    def dim(self):
        return self._dim

    def get_current_parameter_value(self):
        return torch.diagonal(self.mppi.noise_sigma).clone()

    def ensure_valid_value(self, value):
        sigma = _tensor(value, self.d, self.dtype)
        return torch.clamp(sigma, min=self.eps)

    def apply_parameter_value(self, value):
        self.mppi.noise_sigma = torch.diag(self.ensure_valid_value(value))

    def env_values(self, values):
        return torch.stack([torch.diag(v) for v in values])


class MuParameter(_VectorConfig, MPPIParameter):
    """The noise mean (sets `noise_mu`; see the module docstring)."""
    env_keyword = "noise_mu"

    @staticmethod
    def name():
        return "mu"

    def dim(self):
        return self._dim

    def get_current_parameter_value(self):
        return self.mppi.noise_mu.detach().clone().reshape(-1)

    def ensure_valid_value(self, value):
        return _tensor(value, self.d, self.dtype)

    def apply_parameter_value(self, value):
        self.mppi.noise_mu = self.ensure_valid_value(value)

    def env_values(self, values):
        return torch.stack(list(values))


class LambdaParameter(MPPIParameter):
    """The temperature; values below `eps` are raised to it."""
    eps = 0.0001
    env_keyword = "lambda_"

    @staticmethod
    def name():
        return "lambda"

    def dim(self):
        return 1

    def get_current_parameter_value(self):
        return self.mppi.lambda_

    def ensure_valid_value(self, value):
        return max(_scalar(value), self.eps)

    def apply_parameter_value(self, value):
        self.mppi.lambda_ = self.ensure_valid_value(value)

    def env_values(self, values):
        return torch.tensor(list(values), dtype=torch.float64)


class HorizonParameter(MPPIParameter):
    """The horizon, rounded to an integer >= 1 (and <= `max_horizon` when set: `BatchedAutotune` sets it to its
    evaluation's longest horizon)."""
    env_keyword = "horizon"
    max_horizon = None

    @staticmethod
    def name():
        return "horizon"

    def dim(self):
        return 1

    def get_current_parameter_value(self):
        return self.mppi.T

    def ensure_valid_value(self, value):
        v = max(round(_scalar(value)), 1)
        return v if self.max_horizon is None else min(v, self.max_horizon)

    def apply_parameter_value(self, value):
        self.mppi.change_horizon(self.ensure_valid_value(value))

    def env_values(self, values):
        return torch.tensor(list(values), dtype=torch.int32)


# ---- tuners ---------------------------------------------------------------------------------------------------------
class Autotune:
    """Tune `params_to_tune` to minimise the mean of `evaluate_fn().costs`.  Each candidate is applied to the controller
    and evaluated by one `evaluate_fn()` call; after each step the best point so far is applied and evaluated again.
    `reload_state_fn` returns a dict (e.g. {"mppi": controller}) the parameters are re-attached to."""
    eps = 0.0001

    def __init__(self, params_to_tune: typing.Sequence[TunableParameter],
                 evaluate_fn: typing.Optional[typing.Callable[[], EvaluationResult]],
                 reload_state_fn: typing.Optional[typing.Callable[[], dict]] = None,
                 optimizer: typing.Optional[Optimizer] = None):
        self.evaluate_fn = evaluate_fn
        self.reload_state_fn = reload_state_fn
        self.params = list(params_to_tune)
        self.optim = optimizer if optimizer is not None else CMAESOpt()
        self.optim.tuner = self
        self.results = []
        self.attach_parameters()
        self.optim.setup_optimization()

    def optimize_step(self) -> EvaluationResult:
        return self.log_current_result(self.optim.optimize_step())

    def optimize_all(self, iterations) -> EvaluationResult:
        return self.log_current_result(self.optim.optimize_all(iterations))

    def get_best_result(self) -> EvaluationResult:
        return min(self.results, key=lambda res: res.costs.mean().item())

    def log_current_result(self, res: EvaluationResult):
        with torch.no_grad():
            iteration = len(self.results)
            kv = self.get_parameter_values(self.params)
            res = res._replace(iteration=iteration,
                               params={k: v.detach().clone() if torch.is_tensor(v) else v for k, v in kv.items()})
            logger.info("i:%d cost: %s params:%s", iteration, res.costs.mean().item(), kv)
            self.results.append(res)
        return res

    def get_parameter_values(self, params_to_tune: typing.Sequence[TunableParameter]):
        return {p.name(): p.get_current_parameter_value() for p in params_to_tune}

    def flatten_params(self) -> np.ndarray:
        x = []
        for v in self.get_parameter_values(self.params).values():
            x.append(v.detach().cpu().double().numpy().reshape(-1) if torch.is_tensor(v) else np.array([v], dtype=np.float64))
        return np.concatenate(x)

    def unflatten_params(self, x, apply=True):
        values, i = {}, 0
        for p in self.params:
            values[p.name()] = p.ensure_valid_value(x[i:i + p.dim()])
            i += p.dim()
        if apply:
            self.apply_parameters(values)
        return values

    def apply_parameters(self, param_values):
        for p in self.params:
            p.apply_parameter_value(param_values[p.name()])

    def attach_parameters(self):
        if self.reload_state_fn is not None:
            state = self.reload_state_fn()
            for p in self.params:
                p.attach_to_state(state)

    def config_to_params(self, config):
        return {p.name(): p.get_parameter_value_from_config(config) for p in self.params}

    # the optimizer's hooks
    def evaluate_candidates(self, X):
        """(costs (P,), results): each candidate applied in turn and evaluated with `evaluate_fn`."""
        costs, results = [], []
        for x in X:
            self.unflatten_params(x)
            res = self.evaluate_fn()
            costs.append(float(res.costs.mean()))
            results.append(res)
        return np.array(costs), results

    def result_of_best(self, results, index):
        """The result to report after a step, with the best point applied: evaluated again."""
        return self.evaluate_fn()


# ---- the GPU population path ----------------------------------------------------------------------------------------
class ClosedLoopEvaluation:
    """Closed-loop episodes of a population of settings of `ctrl`, all in one `MPPI_Batched.run_closed_loop` call.

    ctrl          a plain `MPPI` on the fused route (a registered model or a CudaModel; not a PendulumMLP model, not
                  step-dependent), rollout_samples = 1, no terminal cost, u_per_command = 1, one GPU
    start_states  (S, nx) start states; every candidate runs one episode from each
    steps         control steps per episode
    plant         None (the plant is the controller's model), or the system the episodes run on, as
                  `run_closed_loop`'s plant (e.g. a nonlinear plant for a controller that plans with a linear model)
    plant_params  None (the plant's current parameters), (n_params,) or (S, n_params) in the plant's layout: the plant
                  of each start
    max_horizon   the longest horizon a candidate may have (default ctrl.T, at least ctrl.T)

    The batched controller takes K, dtype, bounds, u_init, u_scale, noise_abs_cost and tile_memory from `ctrl` and has
    T = max_horizon and N = P * S environments for a population of P: environment c * S + s is candidate c from start s.
    Every episode of a call starts from ctrl's nominal sequence as it was when this object was made (cut or extended
    with u_init to each candidate's horizon), and all candidates share the K draws of every command."""

    def __init__(self, ctrl, start_states, steps, plant=None, plant_params=None, max_horizon=None):
        why = self._refusal(ctrl)
        if why is not None:
            raise ValueError(f"ClosedLoopEvaluation: {why}")
        if plant is not None:
            try:
                ctrl._check_plant(plant)
            except ValueError as e:
                raise ValueError(f"ClosedLoopEvaluation: {e}") from None
        self.plant = plant
        if isinstance(steps, bool) or not isinstance(steps, int) or steps < 1:
            raise ValueError(f"ClosedLoopEvaluation: steps must be an integer >= 1, got {steps!r}")
        x0 = torch.as_tensor(start_states).to(ctrl.d, ctrl.dtype)
        if x0.dim() != 2 or x0.shape[1] != ctrl.nx or x0.shape[0] < 1:
            raise ValueError(f"ClosedLoopEvaluation: start_states must be (S, nx={ctrl.nx}), got {tuple(x0.shape)}")
        self.max_horizon = ctrl.T if max_horizon is None else int(max_horizon)
        if self.max_horizon < ctrl.T:
            raise ValueError(f"ClosedLoopEvaluation: max_horizon={self.max_horizon} is below the controller's T={ctrl.T}")
        self.ctrl, self.steps, self.start_states = ctrl, steps, x0.contiguous()
        self.S = x0.shape[0]
        m = ctrl._model if plant is None else plant
        n_params = len(m.param_blob()) + len(m.param_blob_ext())
        self.plant_params = None
        if plant_params is not None:
            pp = torch.as_tensor(plant_params, dtype=torch.float64).detach().cpu()
            if tuple(pp.shape) not in ((n_params,), (self.S, n_params)):
                raise ValueError(f"ClosedLoopEvaluation: plant_params must be ({n_params},) or ({self.S}, {n_params}), "
                                 f"got {tuple(pp.shape)}")
            self.plant_params = pp
        # the start sequence of every episode: ctrl's nominal now, extended with u_init to max_horizon
        U0 = ctrl.U.detach().clone()
        pad = ctrl.u_init.to(ctrl.d, ctrl.dtype).reshape(1, -1).expand(self.max_horizon - U0.shape[0], ctrl.nu)
        self.U0 = torch.cat((U0, pad))
        self.seed = ctrl._rng_seed if ctrl._rng_seed is not None else int(torch.randint(0, 2 ** 62, ()).item())
        self.batched = None

    @staticmethod
    def _refusal(ctrl):
        if type(ctrl) is not MPPI:
            return (f"the controller must be a plain MPPI, got {type(ctrl).__name__} (SMPPI, KMPPI and other controllers "
                    "tune with the sequential Autotune)")
        m = ctrl._model
        if m is None:
            return ("the controller is on the stepped route (dynamics / cost callables); tune it with the sequential "
                    "Autotune")
        if m.model_id in (_cabi.MODEL_PENDULUM_MLP, _cabi.MODEL_PENDULUM_MLP_ENSEMBLE):
            return "the PendulumMLP models have no per-environment batched kernel"
        if m.step_dependent:
            return "step-dependent models have no per-step schedule in a closed loop"
        if ctrl.M != 1:
            return "rollout_samples must be 1"
        if ctrl.terminal_state_cost is not None:
            return "the controller has a terminal cost"
        if ctrl.u_per_command != 1:
            return "u_per_command must be 1"
        if ctrl._world > 1:
            return "sharded controllers are not supported (one GPU)"
        return None

    def controller(self, P) -> MPPI_Batched:
        """The batched controller for a population of P (made on first use)."""
        N = P * self.S
        if self.batched is None or self.batched.N != N:
            c = self.ctrl
            self.batched = MPPI_Batched(c.F, c.running_cost, c.nx, c.noise_sigma.detach().clone(), N, num_samples=c.K,
                                        horizon=self.max_horizon, device=c.d, lambda_=c.lambda_,
                                        noise_mu=c.noise_mu.detach().clone(), u_min=c.u_min, u_max=c.u_max,
                                        u_init=c.u_init, u_scale=c.u_scale, u_per_command=1,
                                        noise_abs_cost=c.noise_abs_cost, rng_seed=self.seed, tile_memory=c._tile_memory)
        return self.batched

    def evaluate(self, P, env_settings: dict):
        """One closed-loop call for P candidates.  `env_settings`: set_env_params keywords and "horizon", each a (P, ...)
        tensor of per-candidate values (missing: the shared value).  Returns the (P, S) episode costs (device) and the
        (steps+1, P, S, nx) states."""
        b = self.controller(P)
        S = self.S
        per_env = {k: v.repeat_interleave(S, dim=0) for k, v in env_settings.items()}
        horizon = per_env.pop("horizon", None)
        if horizon is None and self.ctrl.T != self.max_horizon:
            horizon = torch.full((P * S,), self.ctrl.T, dtype=torch.int32)
        b.set_env_params(**per_env)
        b.U = self.U0.unsqueeze(0).expand(P * S, -1, -1)
        b.set_env_horizon(horizon)
        x0 = self.start_states.repeat(P, 1)
        plant = None
        if self.plant_params is not None:
            plant = self.plant_params if self.plant_params.dim() == 1 else self.plant_params.repeat(P, 1)
        kw = {} if self.plant is None else {"plant": self.plant}
        res = b.run_closed_loop(x0, self.steps, plant_params=plant, **kw)
        costs = res.costs.sum(0).view(P, S)
        return costs, res.states.view(self.steps + 1, P, S, -1)


class BatchedAutotune(Autotune):
    """`Autotune` whose CMA-ES generations run on the GPU: the lambda candidates and the incumbent (the best point
    before the generation) are the environments of one `ClosedLoopEvaluation` call, on the same noise.  A candidate's
    cost is the mean of its S episode costs.  After each step the best point so far is applied to the controller, and
    its result (costs (S,), rollouts (S, steps+1, nx)) comes from the same launch.

    Every parameter must have a per-environment setting: the four parameter classes of this module do.  Parameters not
    tuned stay shared (the controller's values)."""

    def __init__(self, params_to_tune, evaluation: ClosedLoopEvaluation, reload_state_fn=None,
                 optimizer: typing.Optional[CMAESOpt] = None):
        for p in params_to_tune:
            if p.env_keyword is None:
                raise ValueError(f"BatchedAutotune: {type(p).__name__} has no per-environment setting; tune it with the "
                                 "sequential Autotune")
            if isinstance(p, HorizonParameter):
                p.max_horizon = evaluation.max_horizon
        optimizer = optimizer if optimizer is not None else CMAESOpt()
        if not hasattr(optimizer, "incumbent"):
            raise ValueError(f"BatchedAutotune: the optimizer must report its incumbent (CMAESOpt), got "
                             f"{type(optimizer).__name__}")
        self.evaluation = evaluation
        self.incumbent_costs = []        # per generation: the mean cost of the point that was best before it
        super().__init__(params_to_tune, None, reload_state_fn=reload_state_fn, optimizer=optimizer)

    def population_settings(self, points):
        """The per-environment settings of candidate points (P, n): one (P, ...) tensor per parameter."""
        values = [self.unflatten_params(x, apply=False) for x in points]
        return {p.env_keyword: p.env_values([v[p.name()] for v in values]) for p in self.params}

    def evaluate_candidates(self, X):
        points = np.concatenate((np.asarray(X, dtype=np.float64), self.optim.incumbent()[None]))
        P = points.shape[0]
        costs, states = self.evaluation.evaluate(P, self.population_settings(points))
        rollouts = states.permute(1, 2, 0, 3)                       # (P, S, steps+1, nx)
        results = [EvaluationResult(costs[c], rollouts[c]) for c in range(P)]
        f = costs.mean(1).double().cpu().numpy()
        self.incumbent_costs.append(float(f[-1]))
        # an episode that diverged ranks last
        return np.nan_to_num(f[: P - 1], nan=np.inf), results

    def result_of_best(self, results, index):
        """The best point's result from this generation's launch: the candidate that became best, or the incumbent."""
        return results[-1] if index is None else results[index]
