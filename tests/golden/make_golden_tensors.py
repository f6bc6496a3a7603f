"""Generate tests/golden/tens_*.npz (tests/golden/tensor_cases.py) by running the LIVE reference with the torch twins of
the tensor-reading navigation model (step_dependent_dynamics=True) on injected standard-normal draws, and pin the oracle
bit for bit against it, as make_golden_step.py does for the step-dependent cases.  The costmap and the path go into the
fixture.

Run only where the reference sources are available:

    python tests/golden/make_golden_tensors.py
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
from tests.golden.tensor_cases import TENSOR_CASES, TensorOracleRunner, callables, case_tensors  # noqa: E402


def run_case(name, case):
    costmap, path = case_tensors(case)
    run = TensorOracleRunner(case, costmap, path)
    prob, dt = run.prob, _DT[case["dtype"]]
    dyn, cost = callables(costmap, path)
    kw = dict(num_samples=case["K"], horizon=case["T"], lambda_=case["lambda_"], device="cpu",
              u_max=torch.full((2,), case["u_max"], dtype=dt), U_init=run.stream.U0.clone(), step_dependent_dynamics=True)
    sigma = case["noise_sigma"] * torch.eye(2, dtype=dt)
    if case["variant"] == "kmppi":
        km = case["kernel"]
        ctrl = ref.KMPPI(dyn, cost, 2, sigma, num_support_pts=km["S"], kernel=ref.RBFKernel(sigma=km["sigma"]), **kw)
    else:
        ctrl = ref.MPPI(dyn, cost, 2, sigma, **kw)
    zbox = {}
    ctrl._sample_noise = lambda shape: prob.colour(zbox["z"])   # injection point (mppi.py:201-206)
    x = torch.tensor(case["x0"], dtype=dt)
    out, zsums = {"U0": run.stream.U0.numpy(), "costmap": costmap.numpy(), "path": path.numpy()}, []
    for step in range(case["steps"]):
        z = run.stream.next_z()
        zsums.append(float(z.double().sum()))
        zbox["z"] = z
        a_ref = ctrl.command(x.clone())
        r = run.step(x, z)
        # ---- the pin: oracle == live reference, bit for bit
        for key, got in (("U", ctrl.U), ("cost_total", ctrl.cost_total), ("omega", ctrl.omega), ("action", a_ref),
                         ("noise", ctrl.noise), ("perturbed_action", ctrl.perturbed_action)):
            assert torch.equal(r[key], got), f"{name} step {step}: {key} mismatch"
        if case["variant"] == "kmppi":
            assert torch.equal(r["theta"], ctrl.theta), f"{name} step {step}: theta mismatch"
            out[f"theta_{step}"] = r["theta"].numpy()
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
    for name, case in TENSOR_CASES.items():
        if only and name not in only:
            continue
        path = os.path.join(HERE, f"{name}.npz")
        np.savez_compressed(path, **run_case(name, case))
        print(f"{name}: oracle == reference over {case['steps']} step(s); wrote {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
