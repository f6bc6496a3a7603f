"""Golden fixture families, and the base family's case tables.

A family is a table of cases plus the .npz fixtures tests/golden/make_golden.py makes from them by running the live
reference; the tests replay those fixtures against the oracle (tests/golden/replay.py) and the CUDA engine
(tests/golden/engine.py, tests/test_gpu_golden_replay.py).  `Family` holds what differs between families, on the oracle's
side and on the engine's; everything else is shared.

Each case is plain JSON-able data; a case with "N" is an MPPI_Batched case.  `draw_z` defines the injected
standard-normal stream.
"""
import math
from dataclasses import dataclass
from typing import Callable

import numpy as np
import torch

import pytorch_mppi_b200 as eng
from oracle import mppi_oracle as orc
from tests import ensemble_models as em
from tests import shape_models as shm

_DT = {"f32": torch.float32, "f64": torch.float64}

# The engine's tolerance on U and the action against a fixture, per dtype:
#   fp64: 1e-9   the engine reduces in a different order and accumulates the final sums in fp64
#   fp32: 1e-5   the north-star target for the pendulum (BASELINE.json); the reference's OWN fp32-vs-fp64 gap on these
#                draws is 1.2e-5..3.7e-5 (SURVEY.md App. C), so this is at the fp32 noise floor
U_TOL = {"f64": 1e-9, "f32": 1e-5}

PENDULUM = {"kind": "pendulum"}
# test-suite fixture environment (reference tests/test_mppi.py:24-51)
LINEAR2D = {"kind": "linear_point", "B": [[1.0, 0.0], [0.0, -1.0]], "goal": [2.0, 2.0]}
LINEAR2D_TERM = dict(LINEAR2D, terminal_scale=1.0)
# Toy2D navigation (reference tests/smooth_mppi.py:79-142, main() :539-560)
NAV2D = {"kind": "linear_point", "B": [[0.5, 0.0], [0.0, -0.5]], "goal": [2.0, 2.0],
         "R": [[0.01, 0.0], [0.0, 0.01]],
         "hills": [[[[0.25, 0.125], [0.125, 0.25]], [-0.5, -1.0], 200.0]],
         "terminal_scale": 10.0}

# learned pendulum dynamics of BASELINE config 4 (reference tests/pendulum_approximate.py:31, 47-67):
# the 3-32-32-2 tanh network as torch initialises it right after torch.manual_seed(25) (the reference then trains it
# against gym, which is not available here; the fixture stores the weights it was generated with)
MLP_C4 = {"kind": "pendulum_mlp", "seed": 25}

CASES = {
    # BASELINE config 1: pendulum K=100 T=15 fp64, fp32 0-dim bounds (tests/pendulum.py:16-27,72-77)
    "pendulum_c1_f64": dict(variant="mppi", model=PENDULUM, dtype="f64", K=100, T=15, lambda_=1.0,
                            noise_sigma=10.0, u_min=-2.0, u_max=2.0, bounds_fp32=True, x0=[math.pi, 1.0],
                            U_init_scale=math.sqrt(10.0), steps=5, seed=101),
    # BASELINE config 2 (north star): pendulum K=16384 T=30 fp32
    "pendulum_c2_f32": dict(variant="mppi", model=PENDULUM, dtype="f32", K=16384, T=30, lambda_=1.0,
                            noise_sigma=10.0, u_min=-2.0, u_max=2.0, x0=[math.pi, 1.0],
                            U_init_scale=math.sqrt(10.0), steps=10, seed=102),
    # same draws (z is generated in fp32 then widened), fp64 arithmetic: the fp32 noise-floor yardstick
    "pendulum_c2_f64": dict(variant="mppi", model=PENDULUM, dtype="f64", z_dtype="f32", K=16384, T=30, lambda_=1.0,
                            noise_sigma=10.0, u_min=-2.0, u_max=2.0, x0=[math.pi, 1.0],
                            U_init_scale=math.sqrt(10.0), steps=10, seed=102),
    "pendulum_small_f32": dict(variant="mppi", model=PENDULUM, dtype="f32", K=257, T=12, lambda_=0.5,
                               noise_sigma=4.0, u_min=-2.0, u_max=2.0, x0=[2.5, -0.5], steps=4, seed=103),
    # unit-test environment, plain
    "linear_mppi_f64": dict(variant="mppi", model=LINEAR2D, dtype="f64", K=100, T=10, lambda_=1.0,
                            noise_sigma=[[1.0, 0.0], [0.0, 1.0]], x0=[-3.0, -2.0], steps=4, seed=201),
    # bounds + terminal cost + u_scale + null action + noise_mu + u_init
    "linear_mppi_opts_f64": dict(variant="mppi", model=LINEAR2D_TERM, dtype="f64", K=96, T=9, lambda_=2.0,
                                 noise_sigma=[[0.5, 0.0], [0.0, 1.5]], noise_mu=[0.1, -0.2], u_init=[0.05, 0.0],
                                 u_min=[-0.8, -0.6], u_max=[0.7, 0.9], u_scale=1.5, sample_null_action=True,
                                 x0=[-3.0, -2.0], steps=4, seed=202),
    # full (non-diagonal) covariance + |noise| action cost
    "linear_mppi_fullsigma_f64": dict(variant="mppi", model=LINEAR2D, dtype="f64", K=130, T=8, lambda_=0.7,
                                      noise_sigma=[[1.0, 0.3], [0.3, 0.5]], noise_abs_cost=True,
                                      u_max=[1.0, 1.0], x0=[1.0, -1.0], steps=3, seed=203),
    "linear_mppi_f32": dict(variant="mppi", model=LINEAR2D, dtype="f32", K=512, T=15, lambda_=1.0,
                            noise_sigma=[[1.0, 0.0], [0.0, 1.0]], u_max=[0.5, 0.5], x0=[-3.0, -2.0], steps=4, seed=204),
    "linear_smppi_f64": dict(variant="smppi", model=LINEAR2D, dtype="f64", K=100, T=10, lambda_=1.0,
                             noise_sigma=[[1.0, 0.0], [0.0, 1.0]], x0=[-3.0, -2.0],
                             smooth=dict(w=10.0, delta_t=1.0, action_max=[1.0, 1.0]), steps=4, seed=301),
    "linear_smppi_dt_f64": dict(variant="smppi", model=LINEAR2D_TERM, dtype="f64", K=64, T=12, lambda_=1.5,
                                noise_sigma=[[0.6, 0.2], [0.2, 0.9]], u_max=[2.0, 2.0], u_scale=0.8, sample_null_action=True,
                                x0=[0.5, 0.5], smooth=dict(w=2.5, delta_t=0.5, action_min=[-0.9, -0.7], action_max=[0.8, 1.1]),
                                steps=4, seed=302),
    "linear_kmppi_f64": dict(variant="kmppi", model=LINEAR2D, dtype="f64", K=100, T=10, lambda_=1.0,
                             noise_sigma=[[1.0, 0.0], [0.0, 1.0]], x0=[-3.0, -2.0],
                             kernel=dict(S=5, sigma=1.0), steps=4, seed=401),
    # BASELINE config 3 shape, reduced K/T: 2-D navigation, KMPPI RBF(sigma=2) S=5
    "nav2d_kmppi_f64": dict(variant="kmppi", model=NAV2D, dtype="f64", K=256, T=20, lambda_=1.0,
                            noise_sigma=[[1.0, 0.0], [0.0, 1.0]], u_max=[1.0, 1.0], x0=[-3.0, -2.0],
                            kernel=dict(S=5, sigma=2.0), steps=4, seed=402),
    "nav2d_kmppi_c3_f32": dict(variant="kmppi", model=NAV2D, dtype="f32", K=8192, T=40, lambda_=1.0,
                               noise_sigma=[[1.0, 0.0], [0.0, 1.0]], u_max=[1.0, 1.0], x0=[-3.0, -2.0],
                               kernel=dict(S=5, sigma=2.0), steps=3, seed=403),
    "nav2d_mppi_f64": dict(variant="mppi", model=NAV2D, dtype="f64", K=200, T=20, lambda_=1.0,
                           noise_sigma=[[1.0, 0.0], [0.0, 1.0]], u_max=[1.0, 1.0], x0=[-3.0, -2.0], steps=3, seed=404),
    "nav2d_smppi_f64": dict(variant="smppi", model=NAV2D, dtype="f64", K=200, T=20, lambda_=1.0,
                            noise_sigma=[[1.0, 0.0], [0.0, 1.0]], u_max=[1.0, 1.0], x0=[-3.0, -2.0],
                            smooth=dict(w=10.0, delta_t=1.0, action_max=[1.0, 1.0]), steps=3, seed=405),
    # ---- rollout_samples M>1 (mppi.py:334-373): dynamics that differ between the M copies of a sample (copy m is
    # displaced by m*copy_offset per step), so the discounted variance cost is non-zero; with and without a terminal cost
    "linear_mppi_multi_f64": dict(variant="mppi", model=dict(LINEAR2D_TERM, copy_offset=[0.05, -0.03]), dtype="f64", K=96, T=8,
                                  lambda_=1.2, noise_sigma=[[0.7, 0.0], [0.0, 0.9]], u_max=[1.0, 1.0], x0=[-1.0, 0.5],
                                  rollout_samples=3, rollout_var_cost=0.7, rollout_var_discount=0.9, routes=["stepped"],
                                  steps=3, seed=501),
    "linear_mppi_multi_f32": dict(variant="mppi", model=dict(LINEAR2D, copy_offset=[0.04, 0.02]), dtype="f32", K=160, T=10,
                                  lambda_=1.0, noise_sigma=[[1.0, 0.0], [0.0, 1.0]], u_max=[0.8, 0.8], x0=[-2.0, -1.0],
                                  rollout_samples=4, rollout_var_cost=1.5, rollout_var_discount=0.95, routes=["stepped"],
                                  steps=3, seed=502),
    # ---- SpecificActionSampler rows behind the null action (mppi.py:387-400)
    "linear_mppi_sampler_f64": dict(variant="mppi", model=LINEAR2D, dtype="f64", K=128, T=9, lambda_=0.9,
                                    noise_sigma=[[1.0, 0.0], [0.0, 1.0]], u_max=[0.9, 0.9], x0=[-3.0, -2.0],
                                    sample_null_action=True, sampler=dict(n=3, scale=0.4), routes=["stepped"], steps=3, seed=503),
    "linear_mppi_sampler_multi_f64": dict(variant="mppi", model=dict(LINEAR2D, copy_offset=[0.03, 0.03]), dtype="f64", K=64, T=7,
                                          lambda_=1.0, noise_sigma=[[1.0, 0.0], [0.0, 1.0]], x0=[1.0, 1.5],
                                          sampler=dict(n=2, scale=-0.3), rollout_samples=2, rollout_var_cost=0.3,
                                          rollout_var_discount=0.8, routes=["stepped"], steps=2, seed=504),
    # ---- BASELINE config 4: MLP dynamics, sigma^2 = 1 (pendulum_approximate.py:25), K reduced to 4096
    "mlp_c4_f32": dict(variant="mppi", model=MLP_C4, dtype="f32", K=4096, T=30, lambda_=1.0, noise_sigma=1.0,
                       u_min=-2.0, u_max=2.0, x0=[math.pi, 1.0], steps=3, seed=601),
    "mlp_c4_f64": dict(variant="mppi", model=MLP_C4, dtype="f64", z_dtype="f32", K=4096, T=30, lambda_=1.0, noise_sigma=1.0,
                       u_min=-2.0, u_max=2.0, x0=[math.pi, 1.0], steps=3, seed=601),
}

# MPPI_Batched (mppi.py:691-873): N environments share the K noise samples; one fixture per case
BATCHED_CASES = {
    "linear_batched_f64": dict(model=LINEAR2D, dtype="f64", N=5, K=300, T=9, lambda_=0.8, noise_sigma=[[0.8, 0.1], [0.1, 0.6]],
                               u_max=[0.9, 0.7], u_scale=1.2, x0=[[-3.0, -2.0], [1.0, 0.5], [0.0, 0.0], [2.5, -1.0], [-1.0, 3.0]],
                               steps=3, seed=701),
    "linear_batched_abs_f64": dict(model=LINEAR2D, dtype="f64", N=3, K=128, T=6, lambda_=1.5, noise_sigma=[[1.0, 0.0], [0.0, 0.5]],
                                   noise_mu=[0.05, -0.05], u_init=[0.1, 0.0], noise_abs_cost=True, u_per_command=2,
                                   x0=[[-1.0, -1.0], [0.5, 2.0], [3.0, 3.0]], steps=3, seed=702),
    "pendulum_batched_f32": dict(model=PENDULUM, dtype="f32", N=4, K=512, T=12, lambda_=1.0, noise_sigma=4.0, u_min=-2.0, u_max=2.0,
                                 x0=[[math.pi, 1.0], [0.3, -0.2], [-2.0, 3.0], [1.5, 0.0]], steps=3, seed=703),
}


@dataclass(frozen=True)
class Family:
    """What one fixture family supplies; cases with "N" run MPPI_Batched, the others MPPI / SMPPI / KMPPI."""
    name: str
    cases: dict
    # (case, fixture) -> (the oracle's Problem, plant): plant(x, u) steps the closed loop's simulated system on rows of
    # states and scaled actions.  `fixture` maps the names of the extra arrays (below) to their values.
    model: Callable
    # (case, oracle Problem, fixture) -> (dynamics, running_cost, controller keywords) the live reference is given; the
    # keyword `specific_actions` (state -> (n,T,nu)) becomes a SpecificActionSampler
    reference: Callable
    # case -> the extra arrays the fixture stores and `model` reads (networks, maps)
    fixture: Callable = lambda case: {}
    smooth_key: str = "A"           # the fixture key of SMPPI's action sequence
    scalars: bool = True            # whether the fixture stores cost_sum, beta and eta per step
    # ---- the engine's side
    # (case, fixture, U0, route, copy_rows=None, **controller keywords) -> the engine's controller of a case on `route`,
    # asserted to have taken it.  `copy_rows`: the samples per rollout copy that per-copy dynamics see (default K; a
    # shard of a sharded controller sees its K_local).
    engine: Callable = None
    # (name, case) -> the routes the fixture is replayed on
    routes: Callable = lambda name, case: ["fused"]
    # (name, case, route) -> the tolerance on U, the action and theta / the action sequence
    u_tol: Callable = lambda name, case, route: U_TOL[case["dtype"]]
    # (name, case, route, got, want, tol): asserts the engine's per-sample costs against the fixture's
    check_costs: Callable = lambda name, case, route, got, want, tol: None
    # route -> whether a single controller's replay resets the nominal to the fixture's after each command (a sharded
    # replay always does)
    reset_nominal: Callable = lambda route: False
    # case -> whether the oracle can step alongside a replay that resets the nominal
    lockable: Callable = lambda case: False


def make_mlp_net(seed, dtype):
    """pendulum_approximate.py:35, 47-53: seed, then build the network (no draws in between)."""
    torch.manual_seed(seed)
    net = torch.nn.Sequential(torch.nn.Linear(3, 32), torch.nn.Tanh(), torch.nn.Linear(32, 32), torch.nn.Tanh(),
                              torch.nn.Linear(32, 2))
    for p_ in net.parameters():
        p_.requires_grad_(False)
    return net.to(dtype)


def mlp_state_arrays(net):
    return {f"mlp_{k.replace('.', '_')}": v.detach().cpu().numpy() for k, v in net.state_dict().items()}


def load_mlp_net(fixture, dtype):
    """The network a fixture was generated with (weights stored in the .npz)."""
    net = make_mlp_net(0, dtype)
    sd = {k: torch.from_numpy(np.asarray(fixture[f"mlp_{k.replace('.', '_')}"])).to(dtype) for k in net.state_dict()}
    net.load_state_dict(sd)
    return net


MlpPendulumModel = orc.MlpPendulumModel


def copy_offset_dynamics(base_dynamics, K, offset):
    """Dynamics that differ between the M rollout copies of a sample: the reference flattens (M,K) copy-major
    (mppi.py:348-351), so row r belongs to copy r // K, and copy m is pushed by m * offset every step.  Works on any
    device (the engine calls it with CUDA tensors on the stepped route)."""
    def dynamics(state, action):
        nxt = base_dynamics(state, action)
        m = torch.div(torch.arange(state.shape[0], device=state.device), K, rounding_mode="floor").to(state.dtype)
        off = torch.as_tensor(offset, dtype=state.dtype, device=state.device)
        return nxt + m.unsqueeze(1) * off
    return dynamics


def sampler_actions(case, state):
    """SpecificActionSampler.sample_trajectories of the sampler cases: n fixed-shape trajectories scaled by the first
    state component (so they change along the closed loop)."""
    sp, T = case["sampler"], case["T"]
    nu = 1 if not isinstance(case["noise_sigma"], list) else len(case["noise_sigma"])
    ramp = torch.linspace(-1.0, 1.0, sp["n"] * T * nu, dtype=state.dtype, device=state.device).reshape(sp["n"], T, nu)
    return sp["scale"] * state.reshape(-1)[0] * ramp


def draw_z(gen: np.random.Generator, shape, dtype: torch.dtype, z_dtype=None):
    """Standard normals for one command.  fp32 cases draw fp32; fp64 cases draw fp64 unless the
    case says z_dtype='f32' (same numbers as the fp32 case, widened)."""
    np_dt = np.float32 if (dtype == torch.float32 or z_dtype == "f32") else np.float64
    return torch.from_numpy(gen.standard_normal(shape, dtype=np_dt)).to(dtype)


def build_problem(case, fixture):
    dt = _DT[case["dtype"]]
    m = case["model"]
    if m["kind"] == "pendulum":
        model = orc.PendulumModel()
        model.has_terminal = False
        model.terminal_cost = None
    elif m["kind"] == "pendulum_mlp":
        model = MlpPendulumModel(load_mlp_net(fixture, dt))
    elif m["kind"] == "shape":
        from tests.golden.shape_cases import ShapeTwin
        model = ShapeTwin(m)
    else:
        model = orc.LinearPointModel(B=m["B"], goal=m["goal"], Q=m.get("Q"), R=m.get("R"),
                                     hills=[tuple(h) for h in m.get("hills", [])],
                                     terminal_scale=m.get("terminal_scale", 0.0), dtype=dt)
    bd = torch.float32 if case.get("bounds_fp32") else dt
    dynamics = model.dynamics
    if m.get("copy_offset") is not None:
        dynamics = copy_offset_dynamics(model.dynamics, case["K"], m["copy_offset"])
    prob = orc.Problem(
        dynamics=dynamics, running_cost=model.running_cost, nx=model.nx,
        noise_sigma=torch.tensor(case["noise_sigma"], dtype=dt), K=case["K"], T=case["T"],
        lambda_=case["lambda_"],
        noise_mu=None if case.get("noise_mu") is None else torch.tensor(case["noise_mu"], dtype=dt),
        u_min=None if case.get("u_min") is None else torch.tensor(case["u_min"], dtype=bd),
        u_max=None if case.get("u_max") is None else torch.tensor(case["u_max"], dtype=bd),
        u_init=None if case.get("u_init") is None else torch.tensor(case["u_init"], dtype=dt),
        u_scale=case.get("u_scale", 1),
        terminal_state_cost=model.terminal_cost if getattr(model, "has_terminal", False) else None,
        sample_null_action=case.get("sample_null_action", False),
        noise_abs_cost=case.get("noise_abs_cost", False),
        rollout_samples=case.get("rollout_samples", 1), rollout_var_cost=case.get("rollout_var_cost", 0),
        rollout_var_discount=case.get("rollout_var_discount", 0.95),
        specific_actions=(lambda state: sampler_actions(case, state)) if case.get("sampler") is not None else None)
    return prob, model


def _base_fixture(case):
    m = case["model"]
    return mlp_state_arrays(make_mlp_net(m["seed"], _DT[case["dtype"]])) if m["kind"] == "pendulum_mlp" else {}


def _base_model(case, fixture):
    prob, _ = build_problem(case, fixture)
    return prob, prob.dynamics


def _pendulum_plugins():
    """The pendulum written with the same np.sin / np.clip-on-tensor calls as reference tests/pendulum.py:30-60, so the
    fixtures also pin that those equal the oracle's torch.sin / torch.clamp."""
    def dynamics(state, perturbed_action):
        th = state[:, 0].view(-1, 1)
        thdot = state[:, 1].view(-1, 1)
        g, m, l, dt = 10, 1, 1, 0.05
        u = torch.clamp(perturbed_action, -2, 2)
        newthdot = thdot + (3 * g / (2 * l) * np.sin(th) + 3.0 / (m * l ** 2) * u) * dt
        newthdot = np.clip(newthdot, -8, 8)
        newth = th + newthdot * dt
        return torch.cat((newth, newthdot), dim=1)

    def angle_normalize(x):
        return ((x + math.pi) % (2 * math.pi)) - math.pi

    def running_cost(state, action):
        return angle_normalize(state[:, 0]) ** 2 + 0.1 * state[:, 1] ** 2

    return dynamics, running_cost


def _base_reference(case, prob, fixture):
    """Every model but the pendulum hands the reference the callables of the oracle's problem (the MLP network and the
    per-copy offset dynamics are torch callables)."""
    dt = prob.dtype
    bd = torch.float32 if case.get("bounds_fp32") else dt
    kw = {k: case[k] for k in ("u_scale", "sample_null_action", "noise_abs_cost", "rollout_samples", "rollout_var_cost",
                               "rollout_var_discount", "u_per_command") if k in case}
    kw.update({k: torch.tensor(case[k], dtype=bd if k in ("u_min", "u_max") else dt)
               for k in ("noise_mu", "u_init", "u_min", "u_max") if case.get(k) is not None})
    kw["noise_sigma"] = torch.tensor(case["noise_sigma"], dtype=dt)
    if prob.terminal_state_cost is not None:
        kw["terminal_state_cost"] = prob.terminal_state_cost
    if case.get("sampler") is not None:
        kw["specific_actions"] = lambda state: sampler_actions(case, state)
    if case["model"]["kind"] == "pendulum":
        return (*_pendulum_plugins(), kw)
    return prob.dynamics, prob.running_cost, kw


# ---- the engine's side ------------------------------------------------------------------------------------------------
# Overrides of the fp32 north-star bound, each <= 2x the error measured on H100 (DESIGN.md §2):
#  pendulum_small_f32: K=257, lambda=0.5 (ESS ~ 3): a 2e-7 relative (1-2 ulp) difference in a sample cost -- which
#    sinf-vs-numpy-sin alone produces -- already moves U by 1e-5 (measured 1.04e-5).
#  mlp_c4_f32: the network's three contractions run as FMA chains in the kernel and as BLAS calls in the reference
#    (different summation order through two tanh layers and 30 steps).
U_TOL_OVERRIDE = {"pendulum_small_f32": 2.1e-5, "mlp_c4_f32": 5e-5}
# BASELINE config 4 (mlp_c4_f32) on the wgmma kernel: (PendulumMLP keywords, tolerance on U).  Hi/lo-split bf16 operands
# keep the layer outputs at ~2^-16 relative; over 30-step rollouts of the (chaotic) learned pendulum the plan agrees with
# the fp32 reference to 2.1e-4 (measured on H100, DESIGN.md §2) -- bound 5e-4; MUFU.TANH's 1e-3 absolute error per
# activation shows at 2e-3.  The MLP's other routes run the FFMA kernel, whose tolerance the golden bound is.
TENSOR_CORE_ROUTES = {"wgmma": (dict(tensor_cores="bf16x3", fast_tanh=False), 5e-4),
                      "wgmma_mufu": (dict(tensor_cores="bf16x3", fast_tanh=True), 2e-3)}


def plain(f):
    """A plain function calling `f`: a controller given one takes the stepped route even where `f` is a model's method."""
    return None if f is None else (lambda *args: f(*args))


def controller(case, dynamics, running_cost, nx, sigma, U0=None, **kw):
    """The MPPI / SMPPI / KMPPI controller of a single-controller case; SMPPI starts from its own (zero) nominal, the
    others from `U0`."""
    dt = _DT[case["dtype"]]
    kw = dict(dict(num_samples=case["K"], horizon=case["T"], lambda_=case["lambda_"], device="cuda"), **kw)
    if case["variant"] == "smppi":
        sm = case["smooth"]
        kw.update({k: torch.tensor(sm[k], dtype=dt) for k in ("action_min", "action_max") if sm.get(k) is not None})
        return eng.SMPPI(dynamics, running_cost, nx, sigma, w_action_seq_cost=sm["w"], delta_t=sm["delta_t"], **kw)
    if U0 is not None:
        kw["U_init"] = U0.clone()
    if case["variant"] == "kmppi":
        km = case["kernel"]
        return eng.KMPPI(dynamics, running_cost, nx, sigma, num_support_pts=km["S"], kernel=eng.RBFKernel(sigma=km["sigma"]),
                         **kw)
    return eng.MPPI(dynamics, running_cost, nx, sigma, **kw)


def took_route(ctrl, model, route):
    assert ctrl._model is (None if route == "stepped" else model), f"route {route} not taken"
    return ctrl


def _base_engine_model(case, gold, route):
    m = case["model"]
    if route == "copies":       # the per-copy dynamics as a CudaModel(copies=M) with the oracle's terminal cost
        return em.copy_offset_linear(case["rollout_samples"], m["B"], m["goal"], m["copy_offset"],
                                     m.get("terminal_scale", 0.0), terminal_cost=build_problem(case, gold)[0].terminal_state_cost)
    if m["kind"] == "pendulum":
        return eng.Pendulum()
    if m["kind"] == "pendulum_mlp":
        net = load_mlp_net(gold, _DT[case["dtype"]]).to("cuda")
        return eng.PendulumMLP(net, **TENSOR_CORE_ROUTES.get(route, (dict(tensor_cores=False),))[0])
    if m["kind"] == "shape":
        return shm.shape_model(m["nx"], m["nu"], terminal=m["terminal"])
    return eng.LinearPoint(B=m["B"], goal=m["goal"], Q=m.get("Q"), R=m.get("R"),
                           hills=[tuple(h) for h in m.get("hills", [])], terminal_scale=m.get("terminal_scale", 0.0))


def _base_engine(case, gold, U0, route, copy_rows=None, **controller_kw):
    """route "fused" (or a tensor-core route) passes the registered model's bound methods; "stepped" hides them behind
    plain functions so the controller takes the per-step (arbitrary-callable) path, which alone serves per-copy torch
    dynamics and SpecificActionSamplers; "copies" runs the per-copy dynamics fused, as a CudaModel(copies=M)."""
    dt = _DT[case["dtype"]]
    model = _base_engine_model(case, gold, route)
    wrap = plain if route == "stepped" else (lambda f: f)
    dyn, cost = wrap(model.dynamics), wrap(model.running_cost)
    sigma = torch.tensor(case["noise_sigma"], dtype=dt)
    if "N" in case:
        kw = dict(num_envs=case["N"], num_samples=case["K"], horizon=case["T"], lambda_=case["lambda_"], device="cuda",
                  u_scale=case.get("u_scale", 1), u_per_command=case.get("u_per_command", 1),
                  noise_abs_cost=case.get("noise_abs_cost", False))
        kw.update({k: torch.tensor(case[k], dtype=dt) for k in ("noise_mu", "u_init", "u_min", "u_max") if case.get(k) is not None})
        ctrl = eng.MPPI_Batched(dyn, cost, model.nx, sigma, **kw, **controller_kw)
        ctrl.U = U0.clone()
        return took_route(ctrl, model, route)
    if case["model"].get("copy_offset") is not None and route != "copies":
        assert route == "stepped"
        dyn = copy_offset_dynamics(model.dynamics, copy_rows or case["K"], case["model"]["copy_offset"])
    bd = torch.float32 if case.get("bounds_fp32") else dt
    kw = dict(u_scale=case.get("u_scale", 1), sample_null_action=case.get("sample_null_action", False),
              noise_abs_cost=case.get("noise_abs_cost", False),
              terminal_state_cost=wrap(model.terminal_cost) if model.has_terminal else None,
              rollout_samples=case.get("rollout_samples", 1), rollout_var_cost=case.get("rollout_var_cost", 0),
              rollout_var_discount=case.get("rollout_var_discount", 0.95), u_per_command=case.get("u_per_command", 1))
    kw.update({k: torch.tensor(case[k], dtype=bd if k in ("u_min", "u_max") else dt)
               for k in ("noise_mu", "u_init", "u_min", "u_max") if case.get(k) is not None})
    if case.get("sampler") is not None:
        class Sampler(eng.SpecificActionSampler):
            def sample_trajectories(self, state, info):
                return sampler_actions(case, state)
        kw["specific_action_sampler"] = Sampler()
    return took_route(controller(case, dyn, cost, model.nx, sigma, U0, **kw, **controller_kw), model, route)


def _is_mlp(case):
    return case["model"]["kind"] == "pendulum_mlp"


def _base_routes(name, case):
    """Batched cases: fused and stepped.  Single controllers: the case's routes (default fused and stepped), the stepped
    route only at K <= 2048 or for the MLP; the copy-offset cases also fused as a CudaModel(copies=M), and the config-4
    MLP also on its tensor-core kernels."""
    if "N" in case:
        return ["fused", "stepped"]
    routes = [r for r in case.get("routes", ["fused", "stepped"]) if r == "fused" or case["K"] <= 2048 or _is_mlp(case)]
    if case["model"].get("copy_offset") is not None and case.get("sampler") is None:
        routes.append("copies")
    if name == "mlp_c4_f32":
        routes += list(TENSOR_CORE_ROUTES)
    return routes


def _base_u_tol(name, case, route):
    if route in TENSOR_CORE_ROUTES:
        return TENSOR_CORE_ROUTES[route][1]
    return U_TOL_OVERRIDE.get(name, U_TOL[case["dtype"]])


def base_check_costs(name, case, route, got, want, tol, atol=None):
    """rtol = atol: 1e-10 in fp64; in fp32 5e-6, or 2e-3 for the MLP's network (FFMA or wgmma).  The copy-offset
    CudaModel's replay checks the plan only."""
    if route == "copies":
        return
    rtol = 1e-10 if case["dtype"] == "f64" else (2e-3 if _is_mlp(case) or route in TENSOR_CORE_ROUTES else 5e-6)
    np.testing.assert_allclose(got, want, rtol=rtol, atol=rtol if atol is None else atol)


def base_lockable(case):
    """Single controllers at K <= 2048 whose oracle is not the MLP (whose fp32 rollouts are chaotic)."""
    return "N" not in case and case["K"] <= 2048 and not _is_mlp(case)


BASE = Family("base", dict(CASES, **BATCHED_CASES), _base_model, _base_reference, _base_fixture,
              engine=_base_engine, routes=_base_routes, u_tol=_base_u_tol, check_costs=base_check_costs,
              reset_nominal=lambda route: route != "copies", lockable=base_lockable)
