"""Golden cases of an ensemble of learned pendulum networks (PendulumMLPEnsemble, rollout_samples = M networks, one per
copy; reference mppi.py:334-373) under MPPI, SMPPI and KMPPI.  Fixtures tests/golden/mlpens_*.npz, produced by the live
reference with the ensemble's torch twin (tests/golden/make_golden.py); they store the networks' weights, so replaying
them needs neither the reference nor the seeds' torch initialisation."""
import numpy as np
import torch

from oracle import mppi_oracle as orc
from pytorch_mppi_b200.models import PendulumMLP, PendulumMLPEnsemble
from tests.golden.cases import _DT, Family, make_mlp_net

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


MLP_ENSEMBLE = Family("mlp_ensemble", MLP_ENSEMBLE_CASES, _model, _reference, lambda case: net_arrays(make_nets(case)),
                      smooth_key="action_sequence", scalars=False)
