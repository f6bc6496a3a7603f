"""CPU: closed loops against a plant named apart from the controller's model (`run_closed_loop(plant=...)`,
`mppi_plan_closed_loop_plant`).  The library's layout probes and its refusals of null or malformed descriptors, before
any CUDA call; the Python side with the C entry points replaced by a stub (as tests/test_closed_loop.py does): the call
it makes with and without a plant, and every refusal, raised before anything is launched."""
import contextlib
import ctypes as C

import pytest
import torch

import pytorch_mppi_b200 as eng
from pytorch_mppi_b200 import _cabi, autotune, build
from tests import closed_loop_plant_models as cpm
from tests.golden import cases


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _cabi.load()


def test_plant_layout_matches_the_library(lib):
    S = _cabi.MppiPlantModel
    assert lib.mppi_abi_layout(17) == C.sizeof(S) == 32
    assert lib.mppi_abi_layout(18) == S.model_tensors.offset == 16
    assert S.n_model_tensors.offset == 24 and S.reserved.offset == 28


def _plant(**kw):
    return _cabi.MppiPlantModel(struct_size=C.sizeof(_cabi.MppiPlantModel), model=_cabi.MODEL_PENDULUM, **kw)


def test_entry_points_refuse_bad_descriptors_before_any_cuda_call(lib):
    cl = _cabi.MppiClosedLoop(struct_size=C.sizeof(_cabi.MppiClosedLoop), steps=1)
    run = lambda pm, plan=None: lib.mppi_plan_closed_loop_plant(plan, C.byref(cl), None if pm is None else C.byref(pm), None)
    size = lambda pm, plan=None: lib.mppi_plant_block_bytes(plan, None if pm is None else C.byref(pm))
    # a null plan: the plan's model (no descriptor) or a well-formed descriptor
    assert run(None) == -1 and size(None) == 0
    assert run(_plant()) == -1 and size(_plant()) == 0
    # the descriptor itself is checked first
    bad = _plant()
    bad.struct_size = 0
    assert run(bad) == -5 and size(bad) == 0
    assert run(_plant(reserved=1)) == -1
    assert run(_plant(n_model_tensors=-1)) == -1
    for model in (_cabi.MODEL_PENDULUM_MLP, _cabi.MODEL_PENDULUM_MLP_ENSEMBLE):
        pm = _plant()
        pm.model = model
        assert run(pm) == -2 and size(pm) == 0                   # a learned model has no plant step
    for model in (0, 5, 99):
        pm = _plant()
        pm.model = model
        assert run(pm) == -1
    pm = _plant()
    pm.model = _cabi.MODEL_USER                                   # a user plant without its handle
    assert run(pm) == -1 and size(pm) == 0
    fake = (C.c_uint32 * 64)()                                    # not a handle: wrong magic
    pm.user_model = C.cast(fake, C.c_void_p)
    assert run(pm) == -1
    # the closed-loop struct is still checked when no plant is named
    assert lib.mppi_plan_closed_loop(None, C.byref(cl), None) == -1


# ---- the Python side, with a stub library ----------------------------------------------------------------------------
class _Gen:
    def __init__(self, seed=11, offset=40):
        self.seed, self.offset = seed, offset

    def initial_seed(self):
        return self.seed

    def get_offset(self):
        return self.offset

    def set_offset(self, v):
        self.offset = v


class _Lib:
    BLOCK, PLANT_BLOCK = 48, 64

    def __init__(self):
        self.calls = []

    def mppi_plan_model_block_bytes(self, plan):
        return self.BLOCK

    def mppi_plant_block_bytes(self, plan, pm_ref):
        return self.PLANT_BLOCK

    def _record(self, entry, cl, pm):
        rows = None
        if cl.plant_params:
            rows = list((C.c_double * (cl.n_plant * cl.n_plant_params)).from_address(cl.plant_params))
        call = dict(entry=entry, steps=cl.steps, n_plant=cl.n_plant, n_plant_params=cl.n_plant_params, rows=rows,
                    blocks=bool(cl.plant_blocks))
        if pm is not None:
            call.update(model=pm.model, user_model=pm.user_model, n_tensors=pm.n_model_tensors, reserved=pm.reserved,
                        struct_size=pm.struct_size)
        self.calls.append(call)
        return 0

    def mppi_plan_closed_loop(self, plan, cl_ref, stream):
        return self._record("plan", cl_ref._obj, None)

    def mppi_plan_closed_loop_plant(self, plan, cl_ref, pm_ref, stream):
        return self._record("plant", cl_ref._obj, pm_ref._obj)


def _controller(monkeypatch, cls=eng.MPPI, model=None, dtype=torch.float32, T=30, N=None):
    """What MPPI.__init__ + _pack leave behind, as far as run_closed_loop reads it."""
    monkeypatch.setattr(torch._C, "_cuda_getCurrentRawStream", lambda index: 0, raising=False)
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    gen = _Gen()
    monkeypatch.setattr(torch.cuda, "default_generators", {None: gen})
    c = cls.__new__(cls)
    model = eng.Pendulum() if model is None else model
    c.d, c.dtype, c.nx, c.nu, c.T, c.K = torch.device("cpu"), dtype, model.nx, model.nu, T, 1024
    if N is not None:
        c.N = N
    c._model, c._model_version, c._dirty, c._resident = model, 0, False, False
    c.u_per_command, c._world, c._z_inject, c._z_out = 1, 1, None, None
    c._rng_mode, c._rng_seed, c._rng_counter, c._torch_counter_offset = "philox", 7, 100, 24
    c._plan, c._lib, c._cmd_count, c._cost_buf = C.c_void_p(1), _Lib(), 3, torch.zeros(4)
    c._base_flags = _cabi.FLAG_DIAG_SIGMA
    c._gen = gen
    return c


def _mlp():
    return eng.PendulumMLP(cases.make_mlp_net(25, torch.float32))


def test_plant_call_carries_the_plants_model_and_rows(monkeypatch):
    c = _controller(monkeypatch, model=_mlp())
    x0 = torch.tensor([3.0, 0.5])
    res = c.run_closed_loop(x0, 4, plant=eng.Pendulum(m=1.3))
    call = c._lib.calls[-1]
    assert call["entry"] == "plant" and call["model"] == _cabi.MODEL_PENDULUM and call["struct_size"] == 32
    assert not call["user_model"] and call["n_tensors"] == 0 and call["reserved"] == 0
    # default plant_params: the plant's current parameters, in its own layout (not the network's 1,254 doubles)
    assert call["n_plant"] == 1 and call["n_plant_params"] == 7 and call["rows"] == eng.Pendulum(m=1.3).param_blob()
    assert res.states.shape == (5, 2) and res.actions.shape == (4, 1) and res.costs.shape == (4,)
    assert c._cmd_count == 7 and c.state.data_ptr() == res.states[3].data_ptr()
    # explicit rows in the plant's layout
    lp = eng.LinearPoint.toy2d_nav()
    d = _controller(monkeypatch, model=eng.LinearPoint.unit_test_env())
    d.run_closed_loop(x0, 2, plant=lp, plant_params=torch.tensor(lp.param_blob(), dtype=torch.float64))
    call = d._lib.calls[-1]
    assert call["model"] == _cabi.MODEL_LINEAR_POINT and call["rows"] == lp.param_blob()
    assert call["n_plant_params"] == len(lp.param_blob())


def test_batched_plants_ignore_the_controllers_per_environment_parameters(monkeypatch):
    b = _controller(monkeypatch, cls=eng.MPPI_Batched, model=_mlp(), N=3)
    rows = [eng.Pendulum(m=1.0 + 0.1 * e).param_blob() for e in range(3)]
    b.run_closed_loop(torch.zeros(3, 2), 2, plant=eng.Pendulum(), plant_params=torch.tensor(rows, dtype=torch.float64))
    call = b._lib.calls[-1]
    assert call["entry"] == "plant" and call["n_plant"] == 3 and call["rows"] == [v for r in rows for v in r]
    b = _controller(monkeypatch, cls=eng.MPPI_Batched, N=3)
    b.run_closed_loop(torch.zeros(3, 2), 2, plant=eng.Pendulum(m=2.0))
    call = b._lib.calls[-1]          # one plant for every environment, with the plant's own parameters
    assert call["n_plant"] == 1 and call["rows"] == eng.Pendulum(m=2.0).param_blob()


def test_cuda_model_plant_passes_its_handle(monkeypatch):
    plant = cpm.true_pendulum()
    seen = []
    monkeypatch.setattr(plant, "rtc_handle", lambda lib, dtype, variant: seen.append((dtype, variant)) or C.c_void_p(0x1230))
    c = _controller(monkeypatch, model=_mlp(), dtype=torch.float64)
    c.run_closed_loop(torch.tensor([3.0, 0.5], dtype=torch.float64), 3, plant=plant)
    call = c._lib.calls[-1]
    assert call["model"] == _cabi.MODEL_USER and call["user_model"] == 0x1230 and call["n_tensors"] == 0
    assert call["rows"] == cpm.TRUE_PARAMS and seen == [(torch.float64, eng.MPPI._VARIANT)]
    s = _controller(monkeypatch, cls=eng.SMPPI, model=eng.LinearPoint.unit_test_env())
    cm = cpm.costmap_plant(torch.empty(4, 4, device="meta"))
    monkeypatch.setattr(cm, "rtc_handle", lambda lib, dtype, variant: C.c_void_p(0x1230))
    # the plant's tensors are checked against the controller's device before anything runs
    _refused(s, torch.zeros(2), 2, plant=cm, match="tensor 'costmap'")


def test_without_a_plant_the_old_call_is_made(monkeypatch):
    c = _controller(monkeypatch)
    c.run_closed_loop(torch.tensor([3.0, 0.5]), 2)
    c.run_closed_loop(torch.tensor([3.0, 0.5]), 2, plant_params=eng.Pendulum(m=1.3).param_blob())
    assert [k["entry"] for k in c._lib.calls] == ["plan", "plan"]
    assert c._lib.calls[0]["rows"] is None and c._lib.calls[1]["n_plant_params"] == 7


def _refused(c, *args, match, **kw):
    n = len(c._lib.calls)
    counter = (c._rng_counter, c._cmd_count)
    with pytest.raises(ValueError, match=match):
        c.run_closed_loop(*args, **kw)
    assert len(c._lib.calls) == n and (c._rng_counter, c._cmd_count) == counter      # nothing launched, nothing consumed


def test_refusals(monkeypatch):
    x0 = torch.tensor([3.0, 0.5])
    mlp = _mlp()
    c = _controller(monkeypatch, model=mlp)
    # a learned controller without a plant: still refused, and told to name one
    _refused(c, x0, 2, match="PendulumMLP.*plant=")
    ens = eng.PendulumMLPEnsemble([cases.make_mlp_net(s, torch.float32) for s in (1, 2)])
    _refused(_controller(monkeypatch, model=ens), x0, 2, match="PendulumMLP")
    # plants that are not plants
    _refused(c, x0, 2, plant=mlp, match="plant: a learned PendulumMLP")
    _refused(c, x0, 2, plant=ens, match="plant: a learned PendulumMLP")
    _refused(c, x0, 2, plant=eng.Pendulum().dynamics, match="plant must be an AnalyticModel")
    _refused(c, x0, 2, plant="Pendulum", match="plant must be an AnalyticModel")
    sd = eng.CudaModel(2, 1, "x[0] = O::add(x[0], u[0]);", "return x[0];", params=[1.0], step_dependent=True)
    _refused(c, x0, 2, plant=sd, match="plant: a step-dependent")
    _refused(c, x0, 2, plant=eng.LinearPoint.unit_test_env(), match="plant: nx=2, nu=2")
    _refused(c, x0, 2, plant=eng.CudaModel(3, 1, "", "return (real)0;"), match="plant: nx=3")
    # plant_params in the plant's layout: shape and dtype
    _refused(c, x0, 2, plant=eng.Pendulum(), plant_params=[1.0] * 6, match="plant_params.*plant's")
    _refused(c, x0, 2, plant=eng.Pendulum(), plant_params=mlp.param_blob() + mlp.param_blob_ext(), match="plant_params")
    _refused(c, x0, 2, plant=eng.Pendulum(), plant_params=torch.zeros(7, dtype=torch.int64), match="plant_params")
    _refused(c, x0, 2, plant=eng.Pendulum(), plant_params=torch.zeros(2, 7), match="plant_params")
    b = _controller(monkeypatch, cls=eng.MPPI_Batched, model=mlp, N=3)
    _refused(b, torch.zeros(3, 2), 2, plant=eng.Pendulum(), plant_params=torch.zeros(2, 7), match="plant_params")
    # step-dependent controllers stay refused with a plant
    _refused(_controller(monkeypatch, model=sd), x0, 2, plant=eng.Pendulum(), match="step-dependent")
    # after all of that, a valid call still goes through
    c.run_closed_loop(x0, 2, plant=eng.Pendulum())
    assert len(c._lib.calls) == 1


def test_closed_loop_evaluation_passes_the_plant(monkeypatch):
    calls = []

    class _Batched:
        def __init__(self, *a, **kw):
            self.N = a[4]

        U = property(lambda self: None, lambda self, v: None)

        def set_env_params(self, **kw):
            pass

        def set_env_horizon(self, h):
            pass

        def run_closed_loop(self, x0, steps, plant_params=None, plant=None):
            calls.append((plant, plant_params))
            return eng.ClosedLoopResult(torch.zeros(steps + 1, self.N, 2), torch.zeros(steps, self.N, 1),
                                        torch.ones(steps, self.N))

    monkeypatch.setattr(autotune, "MPPI_Batched", _Batched)
    c = eng.MPPI.__new__(eng.MPPI)
    lin = eng.CudaModel(2, 1, "x[0] = O::add(x[0], u[0]);", "return x[0];", params=[1.0])
    c.d, c.dtype, c.nx, c.nu, c.T, c.K = torch.device("cpu"), torch.float32, 2, 1, 10, 256
    c._model, c.M, c.terminal_state_cost, c.u_per_command, c._world = lin, 1, None, 1, 1
    c.F, c.running_cost, c._rng_seed, c._tile_memory, c.noise_abs_cost = lin.dynamics, lin.running_cost, 5, "shared", False
    c._lambda, c._u_scale, c._noise_mu = 1.0, 1.0, torch.zeros(1)
    c._u_min, c._u_max, c._u_init = torch.tensor(-2.0), torch.tensor(2.0), torch.tensor([0.0])
    c._set_sigma(torch.eye(1))
    c._Ubuf = torch.zeros(10)
    c._dirty = False
    plant = eng.Pendulum()
    # plant_params in the plant's layout (7 doubles), not the controller model's (1)
    rows = torch.tensor([eng.Pendulum(m=1.0).param_blob(), eng.Pendulum(m=1.2).param_blob()], dtype=torch.float64)
    ev = autotune.ClosedLoopEvaluation(c, torch.zeros(2, 2), 3, plant=plant, plant_params=rows)
    costs, _ = ev.evaluate(2, {})
    assert calls[-1][0] is plant and torch.equal(calls[-1][1], rows.repeat(2, 1)) and costs.shape == (2, 2)
    with pytest.raises(ValueError, match="ClosedLoopEvaluation: plant_params"):
        autotune.ClosedLoopEvaluation(c, torch.zeros(2, 2), 3, plant=plant, plant_params=torch.zeros(1))
    with pytest.raises(ValueError, match="ClosedLoopEvaluation: plant: a learned PendulumMLP"):
        autotune.ClosedLoopEvaluation(c, torch.zeros(2, 2), 3, plant=_mlp())
    # a PendulumMLP controller stays refused, plant or not (its kernels have no per-environment horizons)
    c._model = _mlp()
    with pytest.raises(ValueError, match="PendulumMLP"):
        autotune.ClosedLoopEvaluation(c, torch.zeros(2, 2), 3, plant=plant)
