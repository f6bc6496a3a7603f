"""Generate tests/golden/stepint_*.npz (tests/golden/step_cases.py) by running the LIVE reference with step-dependent
plugins (`step_dependent_dynamics=True`, mppi.py:147-157) on injected standard-normal draws, and pin the oracle
(through step_cases.HorizonClock) bit for bit against it, as make_golden.py does for the other cases.

Run only where the reference sources are available:

    python tests/golden/make_golden_step.py
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
from tests.golden.step_cases import (STEP_BATCHED_CASES, STEP_CASES, StepBatchedOracleRunner,  # noqa: E402
                                     StepOracleRunner, callables)


def run_case(name, case):
    run = StepOracleRunner(case)
    prob, dt = run.prob, _DT[case["dtype"]]
    dyn, cost, term = callables(case)
    kw = dict(num_samples=case["K"], horizon=case["T"], lambda_=case["lambda_"], device="cpu", terminal_state_cost=term,
              u_max=torch.tensor(case["u_max"], dtype=dt), U_init=run.stream.U0.clone(), step_dependent_dynamics=True)
    sigma = torch.tensor(case["noise_sigma"], dtype=dt)
    if case["variant"] == "kmppi":
        km = case["kernel"]
        ctrl = ref.KMPPI(dyn, cost, 2, sigma, num_support_pts=km["S"], kernel=ref.RBFKernel(sigma=km["sigma"]), **kw)
    else:
        ctrl = ref.MPPI(dyn, cost, 2, sigma, **kw)
    zbox = {}
    ctrl._sample_noise = lambda shape: prob.colour(zbox["z"])   # injection point (mppi.py:201-206)
    x = torch.tensor(case["x0"], dtype=dt)
    out, zsums = {"U0": run.stream.U0.numpy()}, []
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
        if case["K"] <= 2048 or step == 0:
            out[f"cost_total_{step}"] = r["cost_total"].numpy()
        out[f"cost_sum_{step}"] = np.asarray(r["cost_total"].double().sum().item())
        out[f"beta_{step}"] = np.asarray(r["beta"].item())
        out[f"eta_{step}"] = np.asarray(r["eta"].item())
        out[f"x_{step}"] = x.numpy().copy()
        x = run.advance(x, r["action"])
    out["z_sums"] = np.asarray(zsums)
    out["case_json"] = np.asarray(json.dumps(case))
    return out


def run_batched_case(name, case):
    run = StepBatchedOracleRunner(case)
    dt = _DT[case["dtype"]]
    dyn, cost, _ = callables(case)
    ctrl = ref.MPPI_Batched(dyn, cost, 2, torch.tensor(case["noise_sigma"], dtype=dt), num_envs=case["N"],
                            num_samples=case["K"], horizon=case["T"], lambda_=case["lambda_"], device="cpu",
                            u_max=torch.tensor(case["u_max"], dtype=dt), step_dependent_dynamics=True)
    ctrl.U = run.U0.clone()
    zbox = {}
    ctrl._sample_noise = lambda shape: run.prob.colour(zbox["z"])     # mppi.py:807-811 (shared (K,T,nu) draw)
    x = torch.tensor(case["x0"], dtype=dt)
    out, zsums = {"U0": run.U0.numpy()}, []
    for step in range(case["steps"]):
        z = run.next_z()
        zsums.append(float(z.double().sum()))
        zbox["z"] = z
        a_ref = ctrl.command(x.clone())
        r = run.step(x, z)
        assert torch.equal(r["U"], ctrl.U), f"{name} step {step}: U mismatch {(r['U'] - ctrl.U).abs().max()}"
        assert torch.equal(r["action"], a_ref), f"{name} step {step}: action mismatch"
        out[f"U_{step}"] = r["U"].numpy()
        out[f"action_{step}"] = r["action"].numpy()
        out[f"cost_total_{step}"] = r["cost_total"].numpy()
        out[f"omega_{step}"] = r["omega"].numpy()
        out[f"x_{step}"] = x.numpy().copy()
        x = run.advance(x, r["action"])
    out["z_sums"] = np.asarray(zsums)
    out["case_json"] = np.asarray(json.dumps(case))
    return out


def main():
    torch.set_num_threads(1)   # fixed reduction order inside ATen sums
    only = set(sys.argv[1:])
    for table, runner in ((STEP_CASES, run_case), (STEP_BATCHED_CASES, run_batched_case)):
        for name, case in table.items():
            if only and name not in only:
                continue
            path = os.path.join(HERE, f"{name}.npz")
            np.savez_compressed(path, **runner(name, case))
            print(f"{name}: oracle == reference over {case['steps']} step(s); wrote {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
