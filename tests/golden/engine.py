"""Replay a golden fixture on a pytorch_mppi_b200 controller (the family's `engine` builds it: tests/golden/cases.py)."""
import numpy as np
import torch


ORACLE_TOL = {"f64": 1e-9, "f32": 2e-5}      # omega, noise and perturbed_action of the engine against the oracle


def replay(ctrl, run, gold, tol, cost=None, reset_nominal=False, lock_step=False, record=None):
    """Replays a fixture on the engine controller `ctrl` with the draws of `run` (an oracle runner of the same case), at
    the fixture's states, so per-step errors do not compound through x.  Compares U, the action, theta / the action
    sequence and the omega of MPPI_Batched fixtures with the fixture within `tol`, and the costs through
    `cost(got, want)`.  `reset_nominal`: after each command the engine's nominal is the fixture's, so neither do errors
    compound through it.  `lock_step` (single controllers): the oracle commands alongside, from the fixture's nominal,
    and omega, noise, perturbed_action and the states are checked against it.  `record(err)` sees each U error.  Returns
    the largest U error."""
    case, smooth = run.case, run.family.smooth_key
    worst = 0.0
    for step in range(case["steps"]):
        z = run.stream.next_z()
        ctrl.inject_noise(z)
        x = torch.from_numpy(gold[f"x_{step}"])
        a = ctrl.command(x)
        err = float(np.abs(ctrl.U.detach().cpu().numpy() - gold[f"U_{step}"]).max())
        worst = max(worst, err)
        if record is not None:
            record(err)
        assert err <= tol, f"step {step}: |U - U_ref| = {err:.3e} > {tol}"
        assert a.shape == gold[f"action_{step}"].shape
        aerr = float(np.abs(a.detach().cpu().numpy() - gold[f"action_{step}"]).max())
        assert aerr <= tol, f"step {step}: action error {aerr:.3e}"
        for key, attr in (("theta", "theta"), (smooth, "action_sequence")):
            if f"{key}_{step}" in gold:
                assert np.abs(getattr(ctrl, attr).detach().cpu().numpy() - gold[f"{key}_{step}"]).max() <= tol, key
        if f"omega_{step}" in gold:
            np.testing.assert_allclose(ctrl.omega.cpu().numpy(), gold[f"omega_{step}"], atol=ORACLE_TOL[case["dtype"]], rtol=0)
        if cost is not None and f"cost_total_{step}" in gold:
            cost(ctrl.cost_total.detach().cpu().numpy(), gold[f"cost_total_{step}"])
        if lock_step:
            _check_lock_step(ctrl, run, gold, step, x, z)
        if reset_nominal:
            ctrl.U = torch.from_numpy(gold[f"U_{step}"])
            for key, attr in (("theta", "theta"), (smooth, "action_sequence")):
                if f"{key}_{step}" in gold:
                    setattr(ctrl, attr, torch.from_numpy(gold[f"{key}_{step}"]))
    return worst


def _check_lock_step(ctrl, run, gold, step, x, z):
    case = run.case
    otol = ORACLE_TOL[case["dtype"]]
    r = run.step(x, z)
    om = ctrl.omega.detach().cpu().numpy()
    np.testing.assert_allclose(om, r["omega"].numpy(), atol=otol, rtol=0)
    assert abs(om.sum() - 1.0) < 1e-5                                    # test_mppi.py:269-274
    np.testing.assert_allclose(ctrl.noise.cpu().numpy(), r["noise"].numpy(), atol=otol, rtol=0)
    np.testing.assert_allclose(ctrl.perturbed_action.cpu().numpy(), r["perturbed_action"].numpy(), atol=otol, rtol=0)
    if f"pa_head_{step}" in gold:                     # null action + SpecificActionSampler rows (mppi.py:387-400)
        n = gold[f"pa_head_{step}"].shape[0]
        np.testing.assert_allclose(ctrl.perturbed_action[:n].cpu().numpy(), gold[f"pa_head_{step}"], atol=otol, rtol=0)
        i0 = 1 if case.get("sample_null_action") else 0
        smp = ctrl.specific_action_sampler
        assert (smp.start_idx, smp.end_idx) == (i0, i0 + case["sampler"]["n"])
    if r["states"] is not None and ctrl.states is not None:
        assert ctrl.states.shape == r["states"].shape
        np.testing.assert_allclose(ctrl.states.cpu().numpy(), r["states"].numpy(),
                                   atol=max(otol, 1e-5 if case["dtype"] == "f32" else 0), rtol=0)
    # the oracle's next command starts from the fixture's nominal, as the engine's
    run.U = torch.from_numpy(gold[f"U_{step}"]).clone()
    if case["variant"] == "smppi":
        run.A = torch.from_numpy(gold[f"{run.family.smooth_key}_{step}"]).clone()
    if case["variant"] == "kmppi":
        run.theta = torch.from_numpy(gold[f"theta_{step}"]).clone()
