"""CPU: the oracle replays every committed golden fixture of every family (produced by the LIVE reference,
tests/golden/make_golden.py).  On the image that generated them the match is bit-exact; tolerances below only absorb
libm/SIMD-dispatch differences between host CPUs."""
import numpy as np
import pytest
import torch

from tests.golden.replay import FAMILY, load, runner, stored

TOL = {"f64": 1e-11, "f32": 2e-5}


def _assert_close(key, got, want, tol):
    if key in ("cost_total", "cost_sum", "beta", "eta"):
        np.testing.assert_allclose(got, want, rtol=50 * tol, atol=0, err_msg=key)
    else:
        np.testing.assert_allclose(got, want, atol=10 * tol if key == "omega" else tol, rtol=0, err_msg=key)


@pytest.mark.parametrize("name", sorted(FAMILY))
def test_oracle_matches_reference_golden(name):
    torch.set_num_threads(1)
    family = FAMILY[name]
    case, gold = load(name)
    assert case == family.cases[name], f"fixture is stale: re-run tests/golden/make_golden.py {name}"
    for key, value in family.fixture(case).items():         # the networks / maps the case makes
        np.testing.assert_array_equal(gold[key], value, err_msg=key)
    run = runner(case, gold, family)
    tol = TOL[case["dtype"]]
    np.testing.assert_array_equal(run.stream.U0.numpy(), gold["U0"])
    x = torch.tensor(case["x0"], dtype=run.prob.dtype)
    for step in range(case["steps"]):
        z = run.stream.next_z()
        assert abs(float(z.double().sum()) - float(gold["z_sums"][step])) < 1e-6, "injected-noise stream drifted"
        r = run.step(x, z)
        want = stored(family, case, step, x, r)
        assert sorted(want) == sorted(k[: -len(f"_{step}")] for k in gold.files if k.endswith(f"_{step}")), step
        for key, got in want.items():
            _assert_close(key, got, gold[f"{key}_{step}"], tol)
        omega_sums = r["omega"].sum(dim=-1)                # test_mppi.py:269-274, per environment when batched
        assert float((omega_sums - 1).abs().max()) < 1e-5
        x = run.advance(x, r["action"])
