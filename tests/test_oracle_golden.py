"""CPU: the oracle replays every committed golden vector (which were produced by the LIVE
reference, tests/golden/make_golden.py).  On the image that generated them the match is bit-exact;
tolerances below only absorb libm/SIMD-dispatch differences between host CPUs."""
import numpy as np
import pytest
import torch

from tests.golden.cases import BATCHED_CASES, CASES
from tests.golden.replay import BatchedOracleRunner, OracleRunner, load

TOL = {"f64": 1e-11, "f32": 2e-5}


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_reference_golden(name):
    torch.set_num_threads(1)
    case, gold = load(name)
    assert case == CASES[name], "fixture is stale: re-run tests/golden/make_golden.py"
    run = OracleRunner(case, gold)
    tol = TOL[case["dtype"]]
    np.testing.assert_array_equal(run.stream.U0.numpy(), gold["U0"])
    if case["model"]["kind"] == "pendulum_mlp":
        # the fixture's network is what torch builds right after manual_seed(25) (pendulum_approximate.py:31, 47-53)
        from tests.golden.cases import make_mlp_net
        fresh = make_mlp_net(case["model"]["seed"], run.prob.dtype).state_dict()
        for k, v in run.model.net.state_dict().items():
            np.testing.assert_allclose(v.numpy(), fresh[k].numpy(), atol=1e-7, rtol=0)
    x = torch.tensor(case["x0"], dtype=run.prob.dtype)
    for step in range(case["steps"]):
        z = run.stream.next_z()
        assert abs(float(z.double().sum()) - float(gold["z_sums"][step])) < 1e-6, "injected-noise stream drifted"
        np.testing.assert_allclose(x.numpy(), gold[f"x_{step}"], atol=tol, rtol=0)
        r = run.step(x, z)
        np.testing.assert_allclose(r["U"].numpy(), gold[f"U_{step}"], atol=tol, rtol=0)
        np.testing.assert_allclose(r["action"].numpy(), gold[f"action_{step}"], atol=tol, rtol=0)
        if f"cost_total_{step}" in gold:
            np.testing.assert_allclose(r["cost_total"].numpy(), gold[f"cost_total_{step}"], rtol=50 * tol, atol=0)
        np.testing.assert_allclose(r["beta"].item(), gold[f"beta_{step}"], rtol=50 * tol)
        assert abs(r["omega"].sum().item() - 1.0) < 1e-5
        if case["variant"] == "smppi":
            np.testing.assert_allclose(r["action_sequence"].numpy(), gold[f"A_{step}"], atol=tol, rtol=0)
        if case["variant"] == "kmppi":
            np.testing.assert_allclose(r["theta"].numpy(), gold[f"theta_{step}"], atol=tol, rtol=0)
        if f"pa_head_{step}" in gold:       # null action + SpecificActionSampler rows (mppi.py:387-400)
            n = gold[f"pa_head_{step}"].shape[0]
            np.testing.assert_allclose(r["perturbed_action"][:n].numpy(), gold[f"pa_head_{step}"], atol=tol, rtol=0)
        x = run.advance(x, r["action"])


@pytest.mark.parametrize("name", sorted(BATCHED_CASES))
def test_oracle_matches_reference_golden_batched(name):
    """MPPI_Batched (mppi.py:691-873): fixtures produced by the live `ref.MPPI_Batched`."""
    torch.set_num_threads(1)
    case, gold = load(name)
    assert case == BATCHED_CASES[name], "fixture is stale: re-run tests/golden/make_golden.py"
    run = BatchedOracleRunner(case)
    tol = TOL[case["dtype"]]
    np.testing.assert_array_equal(run.U0.numpy(), gold["U0"])
    x = torch.tensor(case["x0"], dtype=run.prob.dtype)
    for step in range(case["steps"]):
        z = run.next_z()
        assert abs(float(z.double().sum()) - float(gold["z_sums"][step])) < 1e-6
        np.testing.assert_allclose(x.numpy(), gold[f"x_{step}"], atol=tol, rtol=0)
        r = run.step(x, z)
        np.testing.assert_allclose(r["U"].numpy(), gold[f"U_{step}"], atol=tol, rtol=0)
        np.testing.assert_allclose(r["action"].numpy(), gold[f"action_{step}"], atol=tol, rtol=0)
        np.testing.assert_allclose(r["cost_total"].numpy(), gold[f"cost_total_{step}"], rtol=50 * tol, atol=0)
        np.testing.assert_allclose(r["omega"].numpy(), gold[f"omega_{step}"], atol=10 * tol, rtol=0)
        assert float((r["omega"].sum(dim=1) - 1).abs().max()) < 1e-5          # test_mppi.py:269-274 per environment
        x = run.advance(x, r["action"])


def test_fp32_noise_floor_documented():
    """The reference's own fp32-vs-fp64 gap on identical draws at the north-star config — the
    yardstick the 1e-5 target is read against (SURVEY.md §7 'hard parts')."""
    _, g32 = load("pendulum_c2_f32")
    _, g64 = load("pendulum_c2_f64")
    gap = np.abs(g32["U_0"].astype(np.float64) - g64["U_0"]).max()
    assert 1e-7 < gap < 2e-4, gap


def test_rbf_closed_form():
    # reference tests/test_mppi.py:560-570 pins exp(-0.5) for unit-distance points at sigma=1
    from oracle.mppi_oracle import rbf_kernel
    t = torch.tensor([[0.0], [1.0]], dtype=torch.double)
    k = rbf_kernel(t, t, 1.0)
    assert abs(k[0, 1].item() - np.exp(-0.5)) < 1e-6 and abs(k[0, 0].item() - 1.0) < 1e-12
