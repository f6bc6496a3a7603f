"""Golden cases of an ensemble of learned pendulum networks (PendulumMLPEnsemble, rollout_samples = M networks, one per
copy; reference mppi.py:334-373) under MPPI, SMPPI and KMPPI.  Fixtures tests/golden/mlpens_*.npz, produced by the live
reference with the ensemble's torch twin (tests/golden/make_golden.py); they store the networks' weights, so replaying
them needs neither the reference nor the seeds' torch initialisation."""
import numpy as np
import torch

from oracle import mppi_oracle as orc
from pytorch_mppi_b200.models import PendulumMLP, PendulumMLPEnsemble
from tests.golden.cases import _DT, Family, controller, make_mlp_net, plain, took_route

_BASE = dict(lambda_=1.0, noise_sigma=1.0, u_max=2.0, steps=3)
MLP_ENSEMBLE_CASES = {
    "mlpens_mppi_f64": dict(_BASE, variant="mppi", dtype="f64", M=4, K=512, T=30, x0=[2.5, 0.5], var_cost=0.5,
                            var_discount=0.9, seed=921, net_seed=60),
    "mlpens_kmppi_f64": dict(_BASE, variant="kmppi", dtype="f64", M=5, K=256, T=30, x0=[2.8, 0.0], var_cost=0.3,
                             var_discount=0.85, kernel=dict(S=5, sigma=2.0), seed=922, net_seed=70),
    "mlpens_smppi_f32": dict(_BASE, variant="smppi", dtype="f32", M=3, K=1024, T=30, noise_sigma=0.5, x0=[2.0, -0.3],
                             var_cost=0.8, var_discount=0.95, smooth=dict(w=0.5, delta_t=0.5, action_max=2.0), seed=923,
                             net_seed=80),
    "mlpens_mppi_f32": dict(_BASE, variant="mppi", dtype="f32", M=8, K=1024, T=30, x0=[-2.0, 1.0], var_cost=1.0,
                            var_discount=0.9, seed=924, net_seed=90),
}


def make_nets(case):
    """The case's M networks: pendulum_approximate.py's network, seeded net_seed + m (different weights per copy)."""
    return [make_mlp_net(case["net_seed"] + m, _DT[case["dtype"]]) for m in range(case["M"])]


def net_arrays(nets):
    """The networks' weights as fixture arrays: net{m}_{parameter}."""
    return {f"net{m}_{k.replace('.', '_')}": v.detach().cpu().numpy()
            for m, net in enumerate(nets) for k, v in net.state_dict().items()}


def load_nets(case, gold, dtype=None):
    """The networks a fixture was generated with (weights stored in the .npz), in `dtype` (default: the case's)."""
    dtype = dtype or _DT[case["dtype"]]
    nets = []
    for m in range(case["M"]):
        net = make_mlp_net(0, dtype)
        net.load_state_dict({k: torch.from_numpy(np.asarray(gold[f"net{m}_{k.replace('.', '_')}"])).to(dtype)
                             for k in net.state_dict()})
        nets.append(net)
    return nets


def twin(case, nets):
    return PendulumMLPEnsemble(nets, max_torque=case["u_max"])


def _model(case, fixture):
    """The oracle's problem runs the twin (M*K rows, block m through network m); the closed loop's simulated system is
    network 0."""
    nets = load_nets(case, fixture)
    ens, dt = twin(case, nets), _DT[case["dtype"]]
    prob = orc.Problem(ens.dynamics, ens.running_cost, 2, torch.tensor(case["noise_sigma"], dtype=dt), K=case["K"],
                       T=case["T"], lambda_=case["lambda_"], u_max=torch.tensor(case["u_max"], dtype=dt),
                       rollout_samples=case["M"], rollout_var_cost=case["var_cost"],
                       rollout_var_discount=case["var_discount"])
    return prob, lambda x, u: PendulumMLP.net_step(nets[0], x, u, case["u_max"])


def _reference(case, prob, fixture):
    dt = _DT[case["dtype"]]
    return prob.dynamics, prob.running_cost, dict(
        noise_sigma=torch.tensor(case["noise_sigma"], dtype=dt), u_max=torch.tensor(case["u_max"], dtype=dt),
        rollout_samples=case["M"], rollout_var_cost=case["var_cost"], rollout_var_discount=case["var_discount"])


# ---- the engine's side
# DESIGN §2, C4 (the learned pendulum), on U and the action: fp64 FFMA, fp32 FFMA, fp32 wgmma with hi/lo-split bf16
# operands
TOL = {("f64", False): 1e-9, ("f32", False): 5e-5, ("f32", "bf16x3"): 5e-4}
# ... except mlpens_smppi_f32 on the wgmma kernel: 1.35e-3 measured at step 2 (steps 0-1 within 5e-4), held to 2e-3, the
# C4 wgmma tolerance with MUFU.TANH.  That command's U is more sensitive to the network's rounding than C4's: the oracle
# on the fixture, with every step's output perturbed by 1.5e-5 relative noise (bf16x3's layer accuracy), moves U by
# 0.6-1.2e-3, while the FFMA kernel (fp32 operands) stays within 5e-5.
FIXTURE_TOL = {("mlpens_smppi_f32", "bf16x3"): 2e-3}
TENSOR_CORES = {"fused": False, "wgmma": "bf16x3"}      # route -> PendulumMLPEnsemble(tensor_cores=)


def assert_costs_close(got, want, tol, dtype):
    """Per-sample costs.  fp64: within tol (relative to the largest cost).  fp32: C4's cost tolerance of the base family
    (rtol = atol = 2e-3), except for at most one sample in 500, which may be off by up to 1 %.  Those are rollouts that
    reach the angle wrap (x0 -> +-pi) within a rounding error: on the other branch the next network input differs, so
    the sample's cost is not determined to fp32 accuracy by its inputs.  The fixtures show it without the engine:
    re-evaluating mlpens_mppi_f32 in fp64 moves sample 431's cost at step 1 by 0.36 (of ~300), and moving x by -1e-6
    moves sample 969's at step 0 by 0.28, while U stays within 4e-5."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    d, scale = np.abs(got - want), max(1.0, float(np.abs(want).max()))
    if dtype == torch.float64:
        assert float(d.max()) <= tol * scale, float(d.max())
        return
    out = d > 2e-3 + 2e-3 * np.abs(want)
    assert int(out.sum()) <= max(1, want.size // 500), (int(out.sum()), np.flatnonzero(out)[:8], d[out][:8])
    assert float(d.max()) <= 1e-2 * scale, float(d.max())


def ensemble_controller(case, ens, route="fused", U0=None, **kw):
    """The controller of a case around the ensemble `ens`: on the fused route, or on the stepped route with its torch
    twin."""
    dt = _DT[case["dtype"]]
    c = controller(case, plain(ens.dynamics) if route == "stepped" else ens.dynamics, ens.running_cost, 2,
                   torch.tensor(case["noise_sigma"], dtype=dt), U0, **dict(dict(
                       u_max=torch.tensor(case["u_max"], dtype=dt), rollout_samples=case["M"],
                       rollout_var_cost=case["var_cost"], rollout_var_discount=case["var_discount"]), **kw))
    return took_route(c, ens, route)


def _engine(case, gold, U0, route, copy_rows=None, **controller_kw):
    """The fixture's networks on the FFMA kernel ("fused") or the bf16x3 tensor-core kernel ("wgmma")."""
    ens = PendulumMLPEnsemble([n.cuda() for n in load_nets(case, gold)], max_torque=case["u_max"],
                              tensor_cores=TENSOR_CORES[route])
    return ensemble_controller(case, ens, "fused", U0, **controller_kw)


def _u_tol(name, case, route):
    tc = TENSOR_CORES[route]
    return FIXTURE_TOL.get((name, tc), TOL[(case["dtype"], tc)])


MLP_ENSEMBLE = Family("mlp_ensemble", MLP_ENSEMBLE_CASES, _model, _reference, lambda case: net_arrays(make_nets(case)),
                      smooth_key="action_sequence", scalars=False, engine=_engine,
                      routes=lambda name, case: ["fused", "wgmma"] if case["dtype"] == "f32" else ["fused"], u_tol=_u_tol,
                      check_costs=lambda name, case, route, got, want, tol: assert_costs_close(got, want, tol,
                                                                                              _DT[case["dtype"]]),
                      reset_nominal=lambda route: True)
