"""Generate tests/golden/*.npz by running the LIVE reference (read-only at /root/reference) with
injected standard-normal draws, and pin the oracle (oracle/mppi_oracle.py) bit-for-bit against it.

Run only where the reference sources are available:

    python tests/golden/make_golden.py [family | case ...]

With no argument every fixture of every family (tests/golden/replay.py FAMILIES) is written; otherwise those of the
named families (base, shapes, step, tensors, ensemble, mlp_ensemble) and the named cases.

The reference's tests hold no known-answer vectors for `command()` (SURVEY.md §8c), so these
fixtures are the pin: every command asserts `torch.equal(oracle, reference)` on U, the action, cost_total and the
other intermediates before the fixture is written.  Noise is injected by replacing `ctrl._sample_noise` (mppi.py:201-206)
with a function returning `colour(z)` where z comes from numpy's Philox bit generator (seeded per case, so
the fixture stores only the seed + a checksum of z, not z itself).
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
from tests.golden.replay import FAMILIES, runner, stored  # noqa: E402


def reference_controller(family, case, run, fixture):
    """The live reference's controller of a case, on the callables and keywords its family hands it."""
    dyn, cost, kw = family.reference(case, run.prob, fixture)
    kw = dict(kw, num_samples=case["K"], horizon=case["T"], lambda_=case["lambda_"], device="cpu")
    if "specific_actions" in kw:
        actions = kw.pop("specific_actions")

        class Sampler(ref.SpecificActionSampler):                       # mppi.py:16-32
            def sample_trajectories(self, state, info):
                return actions(state)
        kw["specific_action_sampler"] = Sampler()
    nx, dt = run.prob.nx, run.prob.dtype
    if "N" in case:
        ctrl = ref.MPPI_Batched(dyn, cost, nx, num_envs=case["N"], **kw)
        ctrl.U = run.stream.U0.clone()
    elif case["variant"] == "smppi":
        # SMPPI zeroes U and (with U_init=None) the action sequence (mppi.py:480-484)
        sm = case["smooth"]
        bounds = {k: torch.tensor(sm[k], dtype=dt) for k in ("action_min", "action_max") if sm.get(k) is not None}
        ctrl = ref.SMPPI(dyn, cost, nx, w_action_seq_cost=sm["w"], delta_t=sm["delta_t"], **bounds, **kw)
    elif case["variant"] == "kmppi":
        km = case["kernel"]
        ctrl = ref.KMPPI(dyn, cost, nx, U_init=run.stream.U0.clone(), num_support_pts=km["S"],
                         kernel=ref.RBFKernel(sigma=km["sigma"]), **kw)
    else:
        ctrl = ref.MPPI(dyn, cost, nx, U_init=run.stream.U0.clone(), **kw)
    return ctrl


def pin(name, step, case, r, ctrl, action):
    """The oracle's result equals the live reference's state after the same command, bit for bit."""
    got = {"U": ctrl.U, "action": action}
    if "N" not in case:
        got.update(cost_total=ctrl.cost_total, omega=ctrl.omega, noise=ctrl.noise, perturbed_action=ctrl.perturbed_action)
        if case["variant"] == "smppi":
            got["action_sequence"] = ctrl.action_sequence
        if case["variant"] == "kmppi":
            got["theta"] = ctrl.theta
        if ctrl.M > 1:
            got.update(states=ctrl.states, actions=ctrl.actions)
            # the case must exercise the variance term: the M copies of a sample really differ
            assert float(ctrl.states.var(dim=0).max()) > 1e-4, f"{name}: rollout copies are identical"
        if case.get("sampler") is not None:
            i0 = 1 if case.get("sample_null_action") else 0
            smp = ctrl.specific_action_sampler
            assert (smp.start_idx, smp.end_idx) == (i0, i0 + case["sampler"]["n"])
    for key, value in got.items():
        assert torch.equal(r[key], value), f"{name} step {step}: {key} mismatch"


def run_case(family, name, case):
    fixture = family.fixture(case)
    run = runner(case, fixture, family)
    ctrl = reference_controller(family, case, run, fixture)
    zbox = {}
    ctrl._sample_noise = lambda shape: run.prob.colour(zbox["z"])   # injection point (mppi.py:201-206, 807-811)
    x = torch.tensor(case["x0"], dtype=run.prob.dtype)
    out = dict(fixture, U0=run.stream.U0.numpy())
    zsums = []
    for step in range(case["steps"]):
        z = run.stream.next_z()
        zsums.append(float(z.double().sum()))
        zbox["z"] = z
        a_ref = ctrl.command(x.clone())
        r = run.step(x, z)
        pin(name, step, case, r, ctrl, a_ref)
        out.update({f"{k}_{step}": v for k, v in stored(family, case, step, x, r).items()})
        x = run.advance(x, r["action"])      # closed loop on the same model (SURVEY §8d)
    out["z_sums"] = np.asarray(zsums)
    out["case_json"] = np.asarray(json.dumps(case))
    return out


def main():
    torch.set_num_threads(1)   # fixed reduction order inside ATen sums
    only = set(sys.argv[1:])
    known = {f.name for f in FAMILIES} | {n for f in FAMILIES for n in f.cases}
    if only - known:
        sys.exit(f"unknown family or case: {' '.join(sorted(only - known))}")
    for family in FAMILIES:
        for name, case in family.cases.items():
            if only and family.name not in only and name not in only:
                continue
            path = os.path.join(HERE, f"{name}.npz")
            np.savez_compressed(path, **run_case(family, name, case))
            print(f"{name}: oracle == reference over {case['steps']} step(s); wrote {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
