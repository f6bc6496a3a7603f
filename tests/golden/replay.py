"""Replay helpers: regenerate a golden case's injected draws and step the oracle through it."""
import json
import os

import numpy as np
import torch

from oracle import mppi_oracle as orc
from tests.golden.cases import BATCHED_CASES, CASES, draw_z, build_problem  # noqa: F401

HERE = os.path.dirname(os.path.abspath(__file__))


def load(name):
    data = np.load(os.path.join(HERE, f"{name}.npz"))
    case = json.loads(str(data["case_json"]))
    return case, data


class Stream:
    """The injected-noise stream of a golden case: U0 first, then one z per command."""

    def __init__(self, case, prob):
        self.case, self.prob = case, prob
        self.gen = np.random.Generator(np.random.Philox(key=case["seed"]))
        self.U0 = (torch.from_numpy(self.gen.standard_normal((case["T"], prob.nu), dtype=np.float32))
                   * np.float32(case.get("U_init_scale", 1.0))).to(prob.dtype)

    def next_z(self):
        c = self.case
        S = c["kernel"]["S"] if c["variant"] == "kmppi" else c["T"]
        return draw_z(self.gen, (c["K"], S, self.prob.nu), self.prob.dtype, c.get("z_dtype"))


class OracleRunner:
    """Steps the oracle through a case; `.step(x, z)` returns the oracle's result dict."""

    def __init__(self, case, gold=None):
        self.case = case
        self.prob, self.model = build_problem(case, gold)      # gold: the MLP cases read their weights from the fixture
        p, dt = self.prob, self.prob.dtype
        self.variant = case["variant"]
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
        if self.variant == "mppi":
            r = orc.mppi_command(p, self.U, x, z)
            self.U = r["U"]
        elif self.variant == "smppi":
            r = orc.smppi_command(p, self.sp, self.U, self.A, x, z)
            self.U, self.A = r["U"], r["action_sequence"]
        else:
            r = orc.kmppi_command(p, self.U, self.theta, x, z, self.W, self.Wshift)
            self.U, self.theta = r["U"], r["theta"]
        upc = self.case.get("u_per_command", 1)
        if upc > 1:                                     # mppi.py:271-274: the first u_per_command rows
            r["action"] = r["action_sequence" if self.variant == "smppi" else "U"][:upc]
        return r

    def advance(self, x, action):
        p = self.prob
        a0 = action if self.case.get("u_per_command", 1) == 1 else action[0]
        return p.dynamics(x.view(1, -1), (p.u_scale * a0).view(1, -1)).view(-1)[: p.nx]


class BatchedOracleRunner:
    """MPPI_Batched golden cases: shared (K,T,nu) draws, (N,T,nu) nominal, (N,nx) states."""

    def __init__(self, case):
        self.case = case
        self.prob, self.model = build_problem(dict(case, variant="mppi"))
        p = self.prob
        self.gen = np.random.Generator(np.random.Philox(key=case["seed"]))
        self.U0 = torch.from_numpy(self.gen.standard_normal((case["N"], case["T"], p.nu), dtype=np.float32)).to(p.dtype)
        self.U = self.U0.clone()
        self.upc = case.get("u_per_command", 1)

    def next_z(self):
        c = self.case
        return draw_z(self.gen, (c["K"], c["T"], self.prob.nu), self.prob.dtype, c.get("z_dtype"))

    def step(self, x, z):
        r = orc.mppi_batched_command(self.prob, self.U, x, z, u_per_command=self.upc)
        self.U = r["U"]
        return r

    def advance(self, x, action):
        a0 = action if self.upc == 1 else action[:, 0]
        return self.prob.dynamics(x, self.prob.u_scale * a0)[:, : self.prob.nx]
