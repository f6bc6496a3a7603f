"""CPU: user models whose rollout copies differ (CudaModel(copies=M), rollout_samples=M) — generated header, NVRTC
compilation, the route rule, the controller setters, what the live-reference fixtures detect, and the C entry points'
argument checks.  No GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

import pytorch_mppi_b200 as eng
from pytorch_mppi_b200 import _cabi, build
from pytorch_mppi_b200.mppi import SpecificActionSampler, fused_route_model
from tests import ensemble_models as em
from tests import user_models
from tests.golden.ensemble_cases import ENSEMBLE, ENSEMBLE_CASES, ensemble_problem, shifted_params
from tests.golden.replay import OracleRunner, load


def test_copies_header():
    h = em.pendulum_ensemble(4, 64).header_text()
    assert "static const int COPIES = 4;" in h and "STEP_DEPENDENT" not in h
    assert h.count("const real* u, const int m)") == 2 and "const real* x, const int m)" in h     # step, cost | terminal
    h = em.scenario_integrator(3, 10, 64).header_text()
    assert "static const bool STEP_DEPENDENT = true;\n    static const int COPIES = 3;" in h
    assert h.count("const real* u, const int t, const int m)") == 2 and "const real* x, const int m)" in h
    assert "COPIES" not in user_models.integrator_user_model().header_text()


@pytest.mark.parametrize("copies", [0, 9, 1.5, True, "2"])
def test_copies_out_of_range_is_refused(copies):
    with pytest.raises(ValueError, match="copies"):
        eng.CudaModel(2, 1, em.PEND_STEP, em.PEND_COST, params=em.pendulum_params(2), copies=copies)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("variant", [0, 1, 2])
@pytest.mark.parametrize("copies", [2, 4, 8])
def test_copies_header_compiles_with_nvrtc(copies, variant, dtype):
    m = em.pendulum_ensemble(copies, 128) if copies != 4 else em.scenario_integrator(copies, 12, 128)
    cubin, names = m.compile_rtc(dtype, variant)
    assert cubin[:4] == b"\x7fELF"
    # the single-loop fused kernel and the states kernel; no split-cost, batched or resident kernel
    assert len(names) == 5 and names[0] and names[4] and names[1:4] == [None, None, None]


def test_route_rule():
    ens, sci, plain = em.pendulum_ensemble(4, 64), em.scenario_integrator(3, 10, 64), user_models.integrator_user_model()

    def route(m, M, term, sdd=False, sampler=None):
        return fused_route_model(m.dynamics, m.running_cost, term, 2, 1, M, sampler, sdd)

    # a model with copies=M runs fused with rollout_samples=M and no sampler
    assert route(ens, 4, ens.terminal_cost) is ens
    assert route(ens, 4, None) is None                               # its terminal cost would be dropped
    assert route(ens, 4, ens.terminal_cost, sampler=SpecificActionSampler()) is None
    assert route(sci, 3, sci.terminal_cost, sdd=True) is sci
    with pytest.raises(ValueError, match="step_dependent_dynamics=True"):
        route(sci, 3, sci.terminal_cost)
    # ... and is refused with any other rollout_samples, sampler or not
    for M in (1, 2, 5):
        for sampler in (None, SpecificActionSampler()):
            with pytest.raises(ValueError, match="copies=4"):
                route(ens, M, ens.terminal_cost, sampler=sampler)
    # models without copies keep their routes: M > 1 is the stepped route
    assert route(plain, 1, plain.terminal_cost) is plain
    assert route(plain, 3, plain.terminal_cost) is None
    assert route(eng.Pendulum(), 2, None) is None


def test_torch_twins_tell_the_copies_apart_by_row():
    M, K = 3, 5
    m = em.pendulum_ensemble(M, K)
    s = torch.tensor([[2.0, 0.5]], dtype=torch.float64).repeat(M * K, 1)
    a = torch.full((M * K, 1), 0.7, dtype=torch.float64)
    nxt = m.dynamics(s, a).view(M, K, 2)
    assert all(torch.equal(nxt[c], nxt[c, :1].expand(K, 2)) for c in range(M))   # rows of one copy agree
    assert not torch.equal(nxt[0], nxt[1]) and not torch.equal(nxt[1], nxt[2])  # the copies do not
    term = m.terminal_cost(nxt.unsqueeze(2), None)
    assert term.shape == (M, K) and not torch.equal(term[0], term[1])


def test_rollout_var_setters_mark_the_constants_dirty():
    c = eng.MPPI.__new__(eng.MPPI)               # the setters only, without a device
    for name, value in (("rollout_var_cost", 2.5), ("rollout_var_discount", 0.8)):
        c._dirty = False
        setattr(c, name, value)
        assert c._dirty and getattr(c, name) == value


@pytest.mark.parametrize("name", sorted(ENSEMBLE_CASES))
def test_fixture_detects_a_copy_index_off_by_one(name):
    """Every fixture's copies differ enough that dynamics reading copy m+1's parameters for copy m miss it by orders of
    magnitude more than any tolerance the engine or the oracle is held to (<= 2e-5)."""
    torch.set_num_threads(1)
    case, gold = load(name)
    run = OracleRunner(case, family=ENSEMBLE, prob=ensemble_problem(case, shifted_params(case, 1)))
    r = run.step(torch.tensor(case["x0"], dtype=run.prob.dtype), run.stream.next_z())
    assert float(np.abs(r["cost_total"].numpy() - gold["cost_total_0"]).max()) > 1e-3
    assert float(np.abs(r["U"].numpy() - gold["U_0"]).max()) > 2e-4


def test_copies_arguments_are_checked_before_any_cuda_call():
    build.build()
    lib = _cabi.load()
    assert lib.mppi_user_model_set_copies(None, 2) == -1
    p = _cabi.MppiFusedParams(struct_size=C.sizeof(_cabi.MppiFusedParams), model=_cabi.MODEL_PENDULUM, K=64, T=8, nx=2,
                              nu=1, u_per_command=1, lambda_=1.0, rollout_samples=2, rollout_var_cost=1.0)
    info = _cabi.MppiLaunchInfo()
    # a registered model's copies are identical: unsupported on the fused route (the stepped route serves it)
    assert lib.mppi_plan_create(C.byref(p), C.byref(C.c_void_p())) == -2
    assert lib.mppi_fused_query(C.byref(p), C.byref(info)) == -2
    assert b"copies" in lib.mppi_last_cuda_error()
    p.rollout_samples = -1
    assert lib.mppi_plan_create(C.byref(p), C.byref(C.c_void_p())) == -1
