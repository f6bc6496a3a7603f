"""Replay helpers: regenerate a golden case's injected draws and step the oracle through it."""
import contextlib
import json
import os

import numpy as np
import torch

from oracle import mppi_oracle as orc
from tests.golden.cases import BASE, draw_z
from tests.golden.ensemble_cases import ENSEMBLE
from tests.golden.mlp_ensemble_cases import MLP_ENSEMBLE
from tests.golden.shape_cases import SHAPES
from tests.golden.step_cases import STEP
from tests.golden.tensor_cases import TENSORS

HERE = os.path.dirname(os.path.abspath(__file__))


def load(name):
    data = np.load(os.path.join(HERE, f"{name}.npz"))
    case = json.loads(str(data["case_json"]))
    return case, data


FAMILIES = [BASE, SHAPES, STEP, TENSORS, ENSEMBLE, MLP_ENSEMBLE]
FAMILY = {name: family for family in FAMILIES for name in family.cases}


class Stream:
    """The injected-noise stream of a golden case: U0 first ((T,nu), or (N,T,nu) for MPPI_Batched), then one z per
    command."""

    def __init__(self, case, prob):
        self.case, self.prob = case, prob
        self.gen = np.random.Generator(np.random.Philox(key=case["seed"]))
        shape = (case["N"], case["T"], prob.nu) if "N" in case else (case["T"], prob.nu)
        self.U0 = (torch.from_numpy(self.gen.standard_normal(shape, dtype=np.float32))
                   * np.float32(case.get("U_init_scale", 1.0))).to(prob.dtype)

    def next_z(self):
        c = self.case
        S = c["kernel"]["S"] if c.get("variant") == "kmppi" else c["T"]
        return draw_z(self.gen, (c["K"], S, self.prob.nu), self.prob.dtype, c.get("z_dtype"))


@contextlib.contextmanager
def multi_copy_rollouts():
    """Inside: the oracle's `rollout_costs` is `rollout_costs_multi`.  The oracle's `mppi_command` rolls out through
    `rollout`, which dispatches on M (mppi.py:292-295), but its `smppi_command` and `kmppi_command` call the one-copy
    `rollout_costs` by name, while the reference's SMPPI and KMPPI dispatch on M too (mppi.py:564, inherited
    `_compute_rollout_costs`); the oracle itself is unchanged."""
    one_copy = orc.rollout_costs
    orc.rollout_costs = orc.rollout_costs_multi
    try:
        yield
    finally:
        orc.rollout_costs = one_copy


class OracleRunner:
    """Steps the oracle through a single-controller case of `family`; `.step(x, z)` returns the oracle's result dict.
    `fixture` holds the family's extra arrays (default: made from the case); `prob` replaces the family's problem."""

    def __init__(self, case, fixture=None, family=BASE, prob=None):
        self.case, self.family, self.variant = case, family, case["variant"]
        model_prob, self.plant = family.model(case, family.fixture(case) if fixture is None else fixture)
        self.prob = p = prob or model_prob
        dt = p.dtype
        self.stream = Stream(case, p)
        T, nu = case["T"], p.nu
        if self.variant == "smppi":
            sm = case["smooth"]
            self.U = torch.zeros(T, nu, dtype=dt)
            self.A = torch.zeros(T, nu, dtype=dt)
            self.sp = orc.SmoothParams(
                w_action_seq_cost=sm["w"], delta_t=sm["delta_t"],
                action_min=None if sm.get("action_min") is None else torch.tensor(sm["action_min"], dtype=dt),
                action_max=None if sm.get("action_max") is None else torch.tensor(sm["action_max"], dtype=dt))
        else:
            self.U = self.stream.U0.clone()
        if self.variant == "kmppi":
            S, sig = case["kernel"]["S"], case["kernel"]["sigma"]
            self.theta = torch.zeros(S, nu, dtype=dt)
            self.W, self.Wshift = orc.kernel_matrices(T, S, lambda a, b: orc.rbf_kernel(a, b, sig), dt)

    def step(self, x, z):
        p = self.prob
        multi = p.rollout_samples > 1 and self.variant != "mppi"
        with multi_copy_rollouts() if multi else contextlib.nullcontext():
            if self.variant == "mppi":
                r = orc.mppi_command(p, self.U, x, z)
            elif self.variant == "smppi":
                r = orc.smppi_command(p, self.sp, self.U, self.A, x, z)
                self.A = r["action_sequence"]
            else:
                r = orc.kmppi_command(p, self.U, self.theta, x, z, self.W, self.Wshift)
                self.theta = r["theta"]
        self.U = r["U"]
        upc = self.case.get("u_per_command", 1)
        if upc > 1:                                     # mppi.py:271-274: the first u_per_command rows
            r["action"] = r["action_sequence" if self.variant == "smppi" else "U"][:upc]
        return r

    def advance(self, x, action):
        p = self.prob
        a0 = action if self.case.get("u_per_command", 1) == 1 else action[0]
        return self.plant(x.view(1, -1), (p.u_scale * a0).view(1, -1)).view(-1)[: p.nx]


class BatchedOracleRunner:
    """MPPI_Batched cases of `family`: shared (K,T,nu) draws, (N,T,nu) nominal, (N,nx) states."""

    def __init__(self, case, fixture=None, family=BASE):
        self.case, self.family = case, family
        self.prob, self.plant = family.model(case, family.fixture(case) if fixture is None else fixture)
        self.stream = Stream(case, self.prob)
        self.U = self.stream.U0.clone()
        self.upc = case.get("u_per_command", 1)

    def step(self, x, z):
        r = orc.mppi_batched_command(self.prob, self.U, x, z, u_per_command=self.upc)
        self.U = r["U"]
        return r

    def advance(self, x, action):
        a0 = action if self.upc == 1 else action[:, 0]
        return self.plant(x, self.prob.u_scale * a0)[:, : self.prob.nx]


def runner(case, fixture=None, family=BASE):
    return (BatchedOracleRunner if "N" in case else OracleRunner)(case, fixture, family)


def stored(family, case, step, x, r):
    """The arrays a fixture of `family` stores for command `step` (fixture key f"{name}_{step}"), from the state it was
    given and the oracle's result."""
    out = {"U": r["U"].numpy(), "action": r["action"].numpy()}
    if "N" in case:
        return dict(out, cost_total=r["cost_total"].numpy(), omega=r["omega"].numpy(), x=x.numpy().copy())
    if case["variant"] == "kmppi":
        out["theta"] = r["theta"].numpy()
    if case["variant"] == "smppi":
        out[family.smooth_key] = r["action_sequence"].numpy()
    if case.get("sampler") is not None:            # the null action and the SpecificActionSampler rows
        out["pa_head"] = r["perturbed_action"][: int(case.get("sample_null_action", False)) + case["sampler"]["n"] + 1].numpy()
    if case["K"] <= 2048 or step == 0:      # keep the big cases' fixtures small: full cost vector for step 0 only
        out["cost_total"] = r["cost_total"].numpy()
    if family.scalars:
        out["cost_sum"] = np.asarray(r["cost_total"].double().sum().item())
        out["beta"] = np.asarray(r["beta"].item())
        out["eta"] = np.asarray(r["eta"].item())
    out["x"] = x.numpy().copy()
    return out
