"""Generate tests/golden/*.npz by running the LIVE reference (read-only at /root/reference) with
injected standard-normal draws, and pin the oracle (oracle/mppi_oracle.py) bit-for-bit against it.

Run only where the reference sources are available:

    python tests/golden/make_golden.py

The reference's tests hold no known-answer vectors for `command()` (SURVEY.md §8c), so these
fixtures are the pin: every case asserts `torch.equal(oracle, reference)` on U, cost_total and omega
before it is written.  Noise is injected by replacing `ctrl._sample_noise` (mppi.py:201-206) with a
function returning `colour(z)` where z comes from numpy's Philox bit generator (seeded per case, so
the fixture stores only the seed + a checksum of z, not z itself).
"""
import json
import math
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
from oracle import mppi_oracle as orc  # noqa: E402
from tests.golden.cases import (BATCHED_CASES, CASES, build_problem, draw_z, mlp_state_arrays,  # noqa: E402
                                sampler_actions)


def ref_plugins(case, prob, model):
    """Plugins handed to the reference controller.  The pendulum is written with the same
    np.sin / np.clip-on-tensor calls as reference tests/pendulum.py:30-60 so the fixture
    also pins that those equal the oracle's torch.sin / torch.clamp.  Every other model hands the reference the
    callables of the oracle's problem (the MLP network and the per-copy offset dynamics are torch callables)."""
    if case["model"]["kind"] == "pendulum":
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

        return dynamics, running_cost, None
    return prob.dynamics, prob.running_cost, prob.terminal_state_cost


def make_ref_controller(case, prob, model, U_init):
    dyn, cost, term = ref_plugins(case, prob, model)
    kw = dict(num_samples=case["K"], horizon=case["T"], lambda_=case["lambda_"], device="cpu",
              u_scale=case.get("u_scale", 1), sample_null_action=case.get("sample_null_action", False),
              noise_abs_cost=case.get("noise_abs_cost", False), terminal_state_cost=term,
              rollout_samples=case.get("rollout_samples", 1), rollout_var_cost=case.get("rollout_var_cost", 0),
              rollout_var_discount=case.get("rollout_var_discount", 0.95), u_per_command=case.get("u_per_command", 1))
    if case.get("sampler") is not None:
        class Sampler(ref.SpecificActionSampler):                       # mppi.py:16-32
            def sample_trajectories(self, state, info):
                return sampler_actions(case, state)
        kw["specific_action_sampler"] = Sampler()
    dt = prob.dtype
    if case.get("noise_mu") is not None:
        kw["noise_mu"] = torch.tensor(case["noise_mu"], dtype=dt)
    if case.get("u_init") is not None:
        kw["u_init"] = torch.tensor(case["u_init"], dtype=dt)
    bd = torch.float32 if case.get("bounds_fp32") else dt
    if case.get("u_min") is not None:
        kw["u_min"] = torch.tensor(case["u_min"], dtype=bd)
    if case.get("u_max") is not None:
        kw["u_max"] = torch.tensor(case["u_max"], dtype=bd)
    sigma = torch.tensor(case["noise_sigma"], dtype=dt)
    variant = case["variant"]
    if variant == "mppi":
        ctrl = ref.MPPI(dyn, cost, prob.nx, sigma, U_init=U_init.clone(), **kw)
    elif variant == "smppi":
        sm = case["smooth"]
        extra = {}
        if sm.get("action_max") is not None:
            extra["action_max"] = torch.tensor(sm["action_max"], dtype=dt)
        if sm.get("action_min") is not None:
            extra["action_min"] = torch.tensor(sm["action_min"], dtype=dt)
        ctrl = ref.SMPPI(dyn, cost, prob.nx, sigma, w_action_seq_cost=sm["w"], delta_t=sm["delta_t"], **extra, **kw)
        # SMPPI zeroes U and (with U_init=None) the action sequence (mppi.py:480-484)
    elif variant == "kmppi":
        km = case["kernel"]
        ctrl = ref.KMPPI(dyn, cost, prob.nx, sigma, U_init=U_init.clone(), num_support_pts=km["S"],
                         kernel=ref.RBFKernel(sigma=km["sigma"]), **kw)
    else:
        raise ValueError(variant)
    return ctrl


def run_case(name, case):
    prob, model = build_problem(case)
    dt = prob.dtype
    K, T, nu = case["K"], case["T"], prob.nu
    variant = case["variant"]
    S = case["kernel"]["S"] if variant == "kmppi" else None
    g = np.random.Generator(np.random.Philox(key=case["seed"]))
    U0 = (torch.from_numpy(g.standard_normal((T, nu), dtype=np.float32)) * np.float32(case.get("U_init_scale", 1.0))).to(dt)
    ctrl = make_ref_controller(case, prob, model, U0)
    zbox = {}
    ctrl._sample_noise = lambda shape: prob.colour(zbox["z"])   # injection point (mppi.py:201-206)

    # oracle state
    if variant == "smppi":
        U = torch.zeros(T, nu, dtype=dt)
        A = torch.zeros(T, nu, dtype=dt)
        sp = orc.SmoothParams(w_action_seq_cost=case["smooth"]["w"], delta_t=case["smooth"]["delta_t"],
                              action_min=None if case["smooth"].get("action_min") is None else torch.tensor(case["smooth"]["action_min"], dtype=dt),
                              action_max=None if case["smooth"].get("action_max") is None else torch.tensor(case["smooth"]["action_max"], dtype=dt))
    else:
        U = U0.clone()
    if variant == "kmppi":
        theta = torch.zeros(S, nu, dtype=dt)
        W, Wshift = orc.kernel_matrices(T, S, lambda a, b: orc.rbf_kernel(a, b, case["kernel"]["sigma"]), dt)

    x = torch.tensor(case["x0"], dtype=dt)
    out = {"U0": U0.numpy()}
    if case["model"]["kind"] == "pendulum_mlp":
        out.update(mlp_state_arrays(model.net))
    zsums = []
    for step in range(case["steps"]):
        zshape = (K, S, nu) if variant == "kmppi" else (K, T, nu)
        z = draw_z(g, zshape, dt, case.get("z_dtype"))
        zsums.append(float(z.double().sum()))
        zbox["z"] = z
        a_ref = ctrl.command(x.clone())
        if variant == "mppi":
            r = orc.mppi_command(prob, U, x, z)
            U = r["U"]
        elif variant == "smppi":
            r = orc.smppi_command(prob, sp, U, A, x, z)
            U, A = r["U"], r["action_sequence"]
            assert torch.equal(A, ctrl.action_sequence), f"{name} step {step}: action_sequence mismatch"
        else:
            r = orc.kmppi_command(prob, U, theta, x, z, W, Wshift)
            U, theta = r["U"], r["theta"]
            assert torch.equal(theta, ctrl.theta), f"{name} step {step}: theta mismatch"
        upc = case.get("u_per_command", 1)
        if upc > 1:                                    # mppi.py:271-274: the first u_per_command rows
            r["action"] = r["action_sequence" if variant == "smppi" else "U"][:upc]
        # ---- the pin: oracle == live reference, bit for bit -------------------------------
        assert torch.equal(r["U"], ctrl.U), f"{name} step {step}: U mismatch {(r['U'] - ctrl.U).abs().max()}"
        assert torch.equal(r["cost_total"], ctrl.cost_total), f"{name} step {step}: cost_total mismatch"
        assert torch.equal(r["omega"], ctrl.omega), f"{name} step {step}: omega mismatch"
        assert torch.equal(r["action"], a_ref), f"{name} step {step}: action mismatch"
        assert torch.equal(r["noise"], ctrl.noise)
        assert torch.equal(r["perturbed_action"], ctrl.perturbed_action)
        if case.get("rollout_samples", 1) > 1:
            assert torch.equal(r["states"], ctrl.states) and torch.equal(r["actions"], ctrl.actions)
            # the case must exercise the variance term: the M copies of a sample really differ
            assert float(ctrl.states.var(dim=0).max()) > 1e-4, f"{name}: rollout copies are identical"
        if case.get("sampler") is not None:
            i0 = 1 if case.get("sample_null_action") else 0
            smp = ctrl.specific_action_sampler
            assert (smp.start_idx, smp.end_idx) == (i0, i0 + case["sampler"]["n"])
            out[f"pa_head_{step}"] = r["perturbed_action"][: i0 + case["sampler"]["n"] + 1].numpy()
        out[f"U_{step}"] = r["U"].numpy()
        out[f"action_{step}"] = r["action"].numpy()
        if K <= 2048 or step == 0:      # keep the big cases' fixtures small: full cost vector for step 0 only
            out[f"cost_total_{step}"] = r["cost_total"].numpy()
        out[f"cost_sum_{step}"] = np.asarray(r["cost_total"].double().sum().item())
        out[f"beta_{step}"] = np.asarray(r["beta"].item())
        out[f"eta_{step}"] = np.asarray(r["eta"].item())
        out[f"x_{step}"] = x.numpy().copy()
        if variant == "smppi":
            out[f"A_{step}"] = r["action_sequence"].numpy()
        if variant == "kmppi":
            out[f"theta_{step}"] = r["theta"].numpy()
        # closed loop on the same model (SURVEY §8d)
        a0 = r["action"] if upc == 1 else r["action"][0]
        x = prob.dynamics(x.view(1, -1), (prob.u_scale * a0).view(1, -1)).view(-1)[: prob.nx]
    out["z_sums"] = np.asarray(zsums)
    out["case_json"] = np.asarray(json.dumps(case))
    return out


def run_batched_case(name, case):
    """MPPI_Batched (mppi.py:691-873): the live class against oracle.mppi_batched_command on injected shared noise."""
    prob, model = build_problem(dict(case, variant="mppi"))
    dt = prob.dtype
    N, K, T, nu = case["N"], case["K"], case["T"], prob.nu
    upc = case.get("u_per_command", 1)
    g = np.random.Generator(np.random.Philox(key=case["seed"]))
    U0 = torch.from_numpy(g.standard_normal((N, T, nu), dtype=np.float32)).to(dt)
    dyn, cost, _ = ref_plugins(dict(case, variant="mppi"), prob, model)
    kw = dict(num_envs=N, num_samples=K, horizon=T, lambda_=case["lambda_"], device="cpu", u_scale=case.get("u_scale", 1),
              u_per_command=upc, noise_abs_cost=case.get("noise_abs_cost", False))
    for key in ("noise_mu", "u_init", "u_min", "u_max"):
        if case.get(key) is not None:
            kw[key] = torch.tensor(case[key], dtype=dt)
    ctrl = ref.MPPI_Batched(dyn, cost, prob.nx, torch.tensor(case["noise_sigma"], dtype=dt), **kw)
    ctrl.U = U0.clone()
    zbox = {}
    ctrl._sample_noise = lambda shape: prob.colour(zbox["z"])            # mppi.py:807-811 (shared (K,T,nu) draw)
    U = U0.clone()
    x = torch.tensor(case["x0"], dtype=dt)
    out = {"U0": U0.numpy()}
    zsums = []
    for step in range(case["steps"]):
        z = draw_z(g, (K, T, nu), dt, case.get("z_dtype"))
        zsums.append(float(z.double().sum()))
        zbox["z"] = z
        a_ref = ctrl.command(x.clone())
        r = orc.mppi_batched_command(prob, U, x, z, u_per_command=upc)
        assert torch.equal(r["U"], ctrl.U), f"{name} step {step}: U mismatch {(r['U'] - ctrl.U).abs().max()}"
        assert torch.equal(r["action"], a_ref), f"{name} step {step}: action mismatch"
        U = r["U"]
        out[f"U_{step}"] = r["U"].numpy()
        out[f"action_{step}"] = r["action"].numpy()
        out[f"cost_total_{step}"] = r["cost_total"].numpy()
        out[f"omega_{step}"] = r["omega"].numpy()
        out[f"x_{step}"] = x.numpy().copy()
        a0 = r["action"] if upc == 1 else r["action"][:, 0]
        x = prob.dynamics(x, prob.u_scale * a0)[:, : prob.nx]
    out["z_sums"] = np.asarray(zsums)
    out["case_json"] = np.asarray(json.dumps(case))
    return out


def main():
    torch.set_num_threads(1)   # fixed reduction order inside ATen sums
    only = set(sys.argv[1:])
    for name, case in CASES.items():
        if only and name not in only:
            continue
        res = run_case(name, case)
        path = os.path.join(HERE, f"{name}.npz")
        np.savez_compressed(path, **res)
        print(f"{name}: oracle == reference over {case['steps']} step(s); wrote {os.path.getsize(path)} bytes")
    for name, case in BATCHED_CASES.items():
        if only and name not in only:
            continue
        res = run_batched_case(name, case)
        path = os.path.join(HERE, f"{name}.npz")
        np.savez_compressed(path, **res)
        print(f"{name}: oracle == reference (MPPI_Batched) over {case['steps']} step(s); wrote {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
