"""Generate tests/golden/mlpens_*.npz (tests/golden/mlp_ensemble_cases.py) by running the LIVE reference with
rollout_samples=M and the torch twin of an ensemble of M learned pendulum networks (PendulumMLPEnsemble: block m of the
M*K copy-major rows through network m, mppi.py:334-373) on injected standard-normal draws, and pin the oracle bit for bit
against it, as make_golden_ensemble.py does.  The fixtures store the networks' weights.

Run only where the reference sources are available:

    python tests/golden/make_golden_mlp_ensemble.py
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(HERE, "_shim"))
sys.path.insert(0, "/root/reference/src")
sys.path.insert(0, ROOT)

from pytorch_mppi import mppi as ref  # noqa: E402  (the untouched reference)
from tests.golden.cases import _DT  # noqa: E402
from tests.golden.mlp_ensemble_cases import (MLP_ENSEMBLE_CASES, MLPEnsembleOracleRunner, make_nets,  # noqa: E402
                                             net_arrays, twin)


def run_case(name, case):
    nets = make_nets(case)
    run = MLPEnsembleOracleRunner(case, nets)
    prob, dt = run.prob, _DT[case["dtype"]]
    ens = twin(case, nets)
    kw = dict(num_samples=case["K"], horizon=case["T"], lambda_=case["lambda_"], device="cpu",
              u_max=torch.tensor(case["u_max"], dtype=dt), rollout_samples=case["M"], rollout_var_cost=case["var_cost"],
              rollout_var_discount=case["var_discount"])
    sigma = torch.tensor(case["noise_sigma"], dtype=dt)
    variant = case["variant"]
    if variant == "kmppi":
        km = case["kernel"]
        ctrl = ref.KMPPI(ens.dynamics, ens.running_cost, 2, sigma, U_init=run.stream.U0.clone(), num_support_pts=km["S"],
                         kernel=ref.RBFKernel(sigma=km["sigma"]), **kw)
    elif variant == "smppi":
        sm = case["smooth"]
        ctrl = ref.SMPPI(ens.dynamics, ens.running_cost, 2, sigma, w_action_seq_cost=sm["w"], delta_t=sm["delta_t"],
                         action_max=torch.tensor(sm["action_max"], dtype=dt), **kw)
    else:
        ctrl = ref.MPPI(ens.dynamics, ens.running_cost, 2, sigma, U_init=run.stream.U0.clone(), **kw)
    zbox = {}
    ctrl._sample_noise = lambda shape: prob.colour(zbox["z"])   # injection point (mppi.py:201-206)
    x = torch.tensor(case["x0"], dtype=dt)
    out, zsums = {"U0": run.stream.U0.numpy()}, []
    out.update(net_arrays(nets))
    for step in range(case["steps"]):
        z = run.stream.next_z()
        zsums.append(float(z.double().sum()))
        zbox["z"] = z
        a_ref = ctrl.command(x.clone())
        r = run.step(x, z)
        # ---- the pin: oracle == live reference, bit for bit
        for key, got in (("U", ctrl.U), ("cost_total", ctrl.cost_total), ("action", a_ref), ("noise", ctrl.noise),
                         ("perturbed_action", ctrl.perturbed_action)):
            assert torch.equal(r[key], got), f"{name} step {step}: {key} mismatch"
        if variant == "kmppi":
            assert torch.equal(r["theta"], ctrl.theta), f"{name} step {step}: theta mismatch"
            out[f"theta_{step}"] = r["theta"].numpy()
        if variant == "smppi":
            assert torch.equal(r["action_sequence"], ctrl.action_sequence), f"{name} step {step}: action_sequence mismatch"
            out[f"action_sequence_{step}"] = r["action_sequence"].numpy()
        out[f"U_{step}"] = r["U"].numpy()
        out[f"action_{step}"] = r["action"].numpy()
        out[f"cost_total_{step}"] = r["cost_total"].numpy()
        out[f"x_{step}"] = x.numpy().copy()
        x = run.advance(x, r["action"])
    out["z_sums"] = np.asarray(zsums)
    out["case_json"] = np.asarray(json.dumps(case))
    return out


def main():
    torch.set_num_threads(1)   # fixed reduction order inside ATen sums
    only = set(sys.argv[1:])
    for name, case in MLP_ENSEMBLE_CASES.items():
        if only and name not in only:
            continue
        path = os.path.join(HERE, f"{name}.npz")
        np.savez_compressed(path, **run_case(name, case))
        print(f"{name}: oracle == reference over {case['steps']} step(s); wrote {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
