"""CPU: step-dependent user models (CudaModel(step_dependent=True), step_dependent_dynamics=True) — generated header,
NVRTC compilation, the route rule, set_params, what the live-reference fixtures detect, and the C entry point's argument
checks.  No GPU."""
import ctypes as C
import hashlib

import numpy as np
import pytest
import torch

import pytorch_mppi_b200 as eng
from pytorch_mppi_b200 import _cabi, build
from pytorch_mppi_b200.mppi import SpecificActionSampler, fused_route_model
from tests import step_models as um
from tests import user_models
from tests.golden.replay import OracleRunner, load
from tests.golden.step_cases import STEP, HorizonClock, step_problem


def test_header_without_t_is_unchanged():
    """The header of a model without t is byte for byte what it was before models could take t: same NVRTC cache keys,
    same kernels.  (sha1 of the text the previous generator produced for these two models.)"""
    sha = lambda m: hashlib.sha1(m.header_text().encode()).hexdigest()
    assert sha(user_models.pendulum_user_model()) == "0f25d3de524f9fb4f81348896838ac5122b65e4f"
    assert sha(user_models.integrator_user_model()) == "03349ca88aff26350bd9177d852bde94f5c36d6d"
    assert "STEP_DEPENDENT" not in user_models.integrator_user_model().header_text()


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("variant", [0, 1, 2])
def test_step_dependent_header_compiles_with_nvrtc(dtype, variant):
    m = um.step_dependent_user_model()
    h = m.header_text()
    assert "static const bool STEP_DEPENDENT = true;" in h
    assert h.count("const real* u, const int t)") == 2          # step and cost; the terminal cost takes no t
    cubin, names = m.compile_rtc(dtype, variant)
    assert cubin[:4] == b"\x7fELF"
    assert len(names) == 5 and all(names[i] for i in (0, 1, 3, 4))
    assert (names[2] is not None) == (variant == 0)                # the batched kernel exists for MPPI only


def test_route_rule():
    sd, plain_cm, pend = um.step_dependent_user_model(), user_models.integrator_user_model(), eng.Pendulum()

    def route(m, sdd, term=None, M=1, sampler=None, nx=2, nu=1):
        return fused_route_model(m.dynamics, m.running_cost, term, nx, nu, M, sampler, sdd)

    # a step-dependent CudaModel runs fused with step_dependent_dynamics=True, one rollout per sample, no sampler
    assert route(sd, True, sd.terminal_cost) is sd
    assert route(um.step_dependent_user_model(terminal=False), True) is not None
    assert route(sd, True) is None                                   # its terminal cost would be dropped
    assert route(sd, True, sd.terminal_cost, M=2) is None
    assert route(sd, True, sd.terminal_cost, sampler=SpecificActionSampler()) is None
    # ... and is refused without it: the reference would call its callables without t
    for kw in ({}, {"M": 2}, {"sampler": SpecificActionSampler()}):
        with pytest.raises(ValueError, match="step_dependent_dynamics=True"):
            route(sd, False, sd.terminal_cost, **kw)
    # models without t: unchanged
    assert route(plain_cm, False, plain_cm.terminal_cost) is plain_cm
    assert route(plain_cm, True, plain_cm.terminal_cost) is None
    assert route(pend, False) is pend and route(pend, True) is None
    lam = lambda s, a, t: s
    assert fused_route_model(lam, lam, None, 2, 1, 1, None, True) is None


def test_torch_callables_take_t():
    sd, plain_cm = um.step_dependent_user_model(), user_models.integrator_user_model()
    s, a = torch.randn(5, 2, dtype=torch.float64), torch.randn(5, 1, dtype=torch.float64)
    assert torch.equal(sd.dynamics(s, a, 3), um.sd_dyn(s, a, 3))
    assert not torch.equal(sd.running_cost(s, a, 3), sd.running_cost(s, a, 4))
    with pytest.raises(TypeError, match="step-dependent"):
        sd.dynamics(s, a)
    # a model without t ignores it (a step_dependent_dynamics=True controller passes it)
    assert torch.equal(plain_cm.dynamics(s, a, 7), plain_cm.dynamics(s, a))


def test_set_params():
    m = um.step_dependent_user_model()
    v0 = m._param_version
    with pytest.raises(ValueError, match="compiled with 8 parameters"):
        m.set_params(um.SD_PARAMS[:-1])
    with pytest.raises(ValueError):
        m.set_params(um.SD_PARAMS + [1.0])
    assert m._param_version == v0 and m.params == um.SD_PARAMS
    p2 = list(um.SD_PARAMS)
    p2[3] = 2.0
    header = m.header_text()
    m.set_params(p2)
    assert m._param_version == v0 + 1 and m.param_blob() == p2
    assert m.header_text() == header                                # the same kernels serve the new values
    s, a = torch.zeros(3, 2, dtype=torch.float64), torch.zeros(3, 1, dtype=torch.float64)
    assert torch.equal(m.running_cost(s, a, 0), um.sd_cost(s, a, 0, p2))    # the torch twins follow


@pytest.mark.parametrize("shift", [-1, 1])
def test_fixture_detects_an_off_by_one_in_t(shift):
    """The golden model's t weight is large enough that evaluating it at t -+ 1 misses the fixture by orders of magnitude
    more than any tolerance the engine or the oracle is held to (<= 2e-5)."""
    case, gold = load("stepint_mppi_f64")
    p = case["model"]["params"]
    x0 = torch.tensor(case["x0"], dtype=torch.float64)
    for kw in (dict(running_cost=lambda s, a, t: um.sd_cost(s, a, t + shift, p)),
               dict(dynamics=lambda s, a, t: um.sd_dyn(s, a, t + shift, p))):
        run = OracleRunner(case, family=STEP, prob=step_problem(case, **kw))
        r = run.step(x0, run.stream.next_z())
        assert float(np.abs(r["U"].numpy() - gold["U_0"]).max()) > 2e-4


def test_horizon_clock_hands_out_t_in_rollout_order():
    """The oracle adapter of the step cases: t = 0..T-1 per rollout, dynamics before cost, any other order refused."""
    seen = []
    clock = HorizonClock(lambda s, u, t: seen.append(("f", t)) or s, lambda s, u, t: seen.append(("c", t)) or t, 3)
    for _ in range(2):
        for _ in range(3):
            clock.dynamics(None, None)
            clock.running_cost(None, None)
    assert seen == [(k, t) for _ in range(2) for t in range(3) for k in ("f", "c")]
    clock.dynamics(None, None)
    with pytest.raises(AssertionError):
        clock.dynamics(None, None)


def test_set_model_params_checks_arguments_before_any_cuda_call():
    build.build()
    lib = _cabi.load()
    blob = (C.c_double * _cabi.MPPI_MODEL_PARAM_DOUBLES)()
    assert lib.mppi_plan_set_model_params(None, blob, None, 0) == -1
    assert lib.mppi_plan_set_model_params(None, None, None, 0) == -1
