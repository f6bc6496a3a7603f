"""Build a pytorch_mppi_b200 controller for a golden case (GPU tests / bench / smoke), and replay a fixture on it."""
import numpy as np
import torch

import pytorch_mppi_b200 as eng
from tests.golden.cases import _DT


def make_model(case, gold=None, **model_kw):
    m = case["model"]
    if m["kind"] == "pendulum":
        return eng.Pendulum()
    if m["kind"] == "pendulum_mlp":
        from tests.golden.cases import load_mlp_net, make_mlp_net
        dt = _DT[case["dtype"]]
        net = (load_mlp_net(gold, dt) if gold is not None else make_mlp_net(m["seed"], dt)).to("cuda")
        model_kw.setdefault("tensor_cores", False)     # the golden tolerance of the fused route is the FFMA kernel's; the
        return eng.PendulumMLP(net, **model_kw)          # tensor-core route is tested with its own (explicit model_kw)
    if m["kind"] == "shape":
        from tests.golden.shape_cases import engine_model
        return engine_model(m)
    return eng.LinearPoint(B=m["B"], goal=m["goal"], Q=m.get("Q"), R=m.get("R"),
                           hills=[tuple(h) for h in m.get("hills", [])], terminal_scale=m.get("terminal_scale", 0.0))


def make_engine(case, U0, device="cuda", route="fused", gold=None, model_kw=None, copy_rows=None, **extra):
    """route='fused' passes the registered model's bound methods; route='stepped' hides them behind
    plain functions so the controller takes the per-step (arbitrary-callable) path.  Cases with M>1 rollouts,
    per-copy dynamics or a SpecificActionSampler exist on the stepped route only (case["routes"]).  `copy_rows`: the
    samples per rollout copy the per-copy dynamics see (default K; a shard of a sharded controller sees its K_local)."""
    dt = _DT[case["dtype"]]
    model = make_model(case, gold, **(model_kw or {}))
    dyn, cost = model.dynamics, model.running_cost
    term = model.terminal_cost if model.has_terminal else None
    if route == "stepped":
        dyn = (lambda f: (lambda s, a: f(s, a)))(model.dynamics)
        cost = (lambda f: (lambda s, a: f(s, a)))(model.running_cost)
        if term is not None:
            term = (lambda f: (lambda s, a: f(s, a)))(model.terminal_cost)
    if case["model"].get("copy_offset") is not None:
        from tests.golden.cases import copy_offset_dynamics
        assert route == "stepped"
        dyn = copy_offset_dynamics(model.dynamics, copy_rows or case["K"], case["model"]["copy_offset"])
    kw = dict(num_samples=case["K"], horizon=case["T"], lambda_=case["lambda_"], device=device,
              u_scale=case.get("u_scale", 1), sample_null_action=case.get("sample_null_action", False),
              noise_abs_cost=case.get("noise_abs_cost", False), terminal_state_cost=term,
              rollout_samples=case.get("rollout_samples", 1), rollout_var_cost=case.get("rollout_var_cost", 0),
              rollout_var_discount=case.get("rollout_var_discount", 0.95), u_per_command=case.get("u_per_command", 1))
    if case.get("sampler") is not None:
        from tests.golden.cases import sampler_actions

        class Sampler(eng.SpecificActionSampler):
            def sample_trajectories(self, state, info):
                return sampler_actions(case, state)
        kw["specific_action_sampler"] = Sampler()
    if case.get("noise_mu") is not None:
        kw["noise_mu"] = torch.tensor(case["noise_mu"], dtype=dt)
    if case.get("u_init") is not None:
        kw["u_init"] = torch.tensor(case["u_init"], dtype=dt)
    bd = torch.float32 if case.get("bounds_fp32") else dt
    if case.get("u_min") is not None:
        kw["u_min"] = torch.tensor(case["u_min"], dtype=bd)
    if case.get("u_max") is not None:
        kw["u_max"] = torch.tensor(case["u_max"], dtype=bd)
    kw.update(extra)
    sigma = torch.tensor(case["noise_sigma"], dtype=dt)
    v = case["variant"]
    if v == "mppi":
        return eng.MPPI(dyn, cost, model.nx, sigma, U_init=U0.clone(), **kw)
    if v == "smppi":
        sm = case["smooth"]
        ex = {}
        if sm.get("action_max") is not None:
            ex["action_max"] = torch.tensor(sm["action_max"], dtype=dt)
        if sm.get("action_min") is not None:
            ex["action_min"] = torch.tensor(sm["action_min"], dtype=dt)
        return eng.SMPPI(dyn, cost, model.nx, sigma, w_action_seq_cost=sm["w"], delta_t=sm["delta_t"], **ex, **kw)
    km = case["kernel"]
    return eng.KMPPI(dyn, cost, model.nx, sigma, U_init=U0.clone(), num_support_pts=km["S"],
                     kernel=eng.RBFKernel(sigma=km["sigma"]), **kw)


def make_batched_engine(case, U0, device="cuda", route="fused"):
    """MPPI_Batched controller for a BATCHED_CASES entry."""
    dt = _DT[case["dtype"]]
    model = make_model(case)
    dyn, cost = model.dynamics, model.running_cost
    if route == "stepped":
        dyn = (lambda f: (lambda s, a: f(s, a)))(model.dynamics)
        cost = (lambda f: (lambda s, a: f(s, a)))(model.running_cost)
    kw = dict(num_envs=case["N"], num_samples=case["K"], horizon=case["T"], lambda_=case["lambda_"], device=device,
              u_scale=case.get("u_scale", 1), u_per_command=case.get("u_per_command", 1),
              noise_abs_cost=case.get("noise_abs_cost", False))
    for key in ("noise_mu", "u_init", "u_min", "u_max"):
        if case.get(key) is not None:
            kw[key] = torch.tensor(case[key], dtype=dt)
    ctrl = eng.MPPI_Batched(dyn, cost, model.nx, torch.tensor(case["noise_sigma"], dtype=dt), **kw)
    ctrl.U = U0.clone()
    return ctrl


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
