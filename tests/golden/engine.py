"""Build a pytorch_mppi_b200 controller for a golden case (GPU tests / bench / smoke)."""
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


def make_engine(case, U0, device="cuda", route="fused", gold=None, model_kw=None, **extra):
    """route='fused' passes the registered model's bound methods; route='stepped' hides them behind
    plain functions so the controller takes the per-step (arbitrary-callable) path.  Cases with M>1 rollouts,
    per-copy dynamics or a SpecificActionSampler exist on the stepped route only (case["routes"])."""
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
        dyn = copy_offset_dynamics(model.dynamics, case["K"], case["model"]["copy_offset"])
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
