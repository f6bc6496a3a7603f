"""GPU: every golden fixture of every family (tests/golden/replay.py FAMILIES), produced by the LIVE reference, replayed on
the CUDA engine through the Python API -> C-ABI -> sm_90a kernels, on each of the family's routes, single controllers and
MPPI_Batched.  U, the action, theta / the action sequence and the costs are compared with the fixture; where the family
resets the nominal after each command and the oracle can step alongside, omega, noise, perturbed_action and the states
are compared with the oracle (tests/golden/engine.py `replay`).  Each family states its controller, routes, tolerances
and resets once, in its tests/golden/*_cases.py.

Measured worst errors of the base and shape fixtures go to tests/_reports/parity_errors.json, and those of the
single-controller shape fixtures to tests/_reports/envelope_errors.json too.
"""
import numpy as np
import pytest
import torch

from tests import reports
from tests.golden.cases import TENSOR_CORE_ROUTES
from tests.golden.engine import replay
from tests.golden.replay import FAMILIES, FAMILY, OracleRunner, load, runner

pytestmark = pytest.mark.gpu


def _replays():
    return [(name, route) for fam in FAMILIES for name, case in sorted(fam.cases.items())
            for route in fam.routes(name, case)]


@pytest.mark.parametrize("name,route", _replays())
def test_engine_matches_reference_golden(name, route):
    torch.set_num_threads(1)
    fam = FAMILY[name]
    case, gold = load(name)
    run = runner(case, gold, fam)
    ctrl = fam.engine(case, gold, run.stream.U0, route)
    tol = fam.u_tol(name, case, route)
    single = "N" not in case
    # the report keys of the base and shape fixtures: the tensor-core routes are the fused route with model keywords
    reported = fam.name in ("base", "shapes") and route != "copies"
    model_kw, engine_route = (TENSOR_CORE_ROUTES[route][0], "fused") if route in TENSOR_CORE_ROUTES else (None, route)

    def record(err):
        if reported:
            reports.worst("parity_errors.json", f"{name}/{engine_route}" + (f"/{model_kw}" if model_kw else ""), err)

    def cost(got, want):
        if reported and single:
            reports.worst("parity_errors.json", f"{name}/{engine_route}/cost_abs", np.abs(got - want).max())
        fam.check_costs(name, case, route, got, want, tol)

    reset = fam.reset_nominal(route)
    worst = replay(ctrl, run, gold, tol, cost, reset_nominal=reset, lock_step=reset and fam.lockable(case), record=record)
    if fam.name == "shapes" and single:
        reports.worst("envelope_errors.json", f"{name}/{route}", worst)
    if case.get("M", 1) > 1:                # the ensembles' M-copy kernels have no split-cost rollout
        assert ctrl.launch_info.split_cost == 0


def _split_cost_cases():
    return sorted(name for fam in FAMILIES if fam.name in ("base", "shapes") for name, case in fam.cases.items()
                  if "N" not in case and "fused" in fam.routes(name, case) and case["K"] > 1
                  and case["model"]["kind"] != "pendulum_mlp")


@pytest.mark.parametrize("name", _split_cost_cases())
def test_split_cost_rollout_is_bit_identical_to_the_single_loop(name, monkeypatch):
    """MPPI_FLAG_SPLIT_COST (the default for single-GPU problems small enough to run with helper threads;
    MPPI_B200_SPLIT_COST=0 turns it off): the rollout thread runs the bare recurrence, the sample's
    helper threads evaluate the running costs in parallel, the sum is taken in the reference's order.  Same
    operations, same rounding, same order -> cost_total, U (A, theta) and the action must be BIT-identical to the
    single-loop kernel on the same draws, for every golden case (all three variants, both dtypes, ragged K)."""
    fam = FAMILY[name]
    case, gold = load(name)
    run = OracleRunner(case)
    monkeypatch.setenv("MPPI_B200_SPLIT_COST", "0")
    plain = fam.engine(case, gold, run.stream.U0, "fused")
    monkeypatch.setenv("MPPI_B200_SPLIT_COST", "1")
    split = fam.engine(case, gold, run.stream.U0, "fused")
    for step in range(min(case["steps"], 3)):
        x = torch.from_numpy(gold[f"x_{step}"]).to(run.prob.dtype).numpy()
        z = run.stream.next_z()
        plain.inject_noise(z)
        split.inject_noise(z)
        a0 = plain.command(x)
        a1 = split.command(x)
        # the flag is honoured exactly when the problem is small enough to run with helper threads
        assert plain.launch_info.split_cost == 0
        assert split.launch_info.split_cost == (1 if split.launch_info.threads_per_sample > 1 else 0)
        assert split.launch_info.threads_per_sample == plain.launch_info.threads_per_sample
        # the rollout itself: same operations in the same order (fp32: bit for bit; fp64: the two kernels inline libdevice's
        # double-precision sin / fmod in different surroundings, 1-ulp differences are possible)
        if case["dtype"] == "f64":
            rel = float(((plain.cost_total - split.cost_total).abs() / plain.cost_total.abs().clamp_min(1e-300)).max())
            reports.worst("parity_errors.json", f"{name}/split_vs_loop_cost_rel", rel)
            assert rel <= 1e-13, (name, rel)
        else:
            assert torch.equal(plain.cost_total, split.cost_total), name
        # the softmin reduction is fp64 in a fixed order per launch geometry; the two kernels may get different cluster
        # sizes (different shared-memory footprints), i.e. a different — equally valid — summation order
        close = dict(rtol=0, atol=1e-12 if case["dtype"] == "f64" else 5e-7)
        assert torch.allclose(plain.U, split.U, **close), name
        assert torch.allclose(a0, a1, **close), name
        if case["variant"] == "smppi":
            assert torch.allclose(plain.action_sequence, split.action_sequence, **close)
        if case["variant"] == "kmppi":
            assert torch.allclose(plain.theta, split.theta, **close)
    # every golden case is small enough to keep its helper threads (no more tiles than SMs)
    assert split.launch_info.split_cost == 1, (name, split.launch_info.threads_per_sample)
    # and the split kernel meets the reference tolerance on its own (first command, golden U)
    tol = fam.u_tol(name, case, "fused")
    run2 = OracleRunner(case)
    monkeypatch.setenv("MPPI_B200_SPLIT_COST", "1")
    again = fam.engine(case, gold, run2.stream.U0, "fused")
    again.inject_noise(run2.stream.next_z())
    again.command(torch.from_numpy(gold["x_0"]).to(run2.prob.dtype).numpy())
    assert float(np.abs(again.U.cpu().numpy() - gold["U_0"]).max()) <= tol
