"""CPU: the Python side of `run_closed_loop()` with the C entry point replaced by a stub (a controller cannot be built
without a CUDA device, so the object is assembled by hand with the attributes that path reads, on the CPU "device").
Pins what the GPU tests cannot see from outside: the MppiClosedLoop layout, the arguments Python hands the library —
the Philox stride of one command in every RNG mode, the stream advanced by `steps` commands — result shapes and dtypes,
and every refusal, raised before anything is launched."""
import ctypes as C

import pytest
import torch

import pytorch_mppi_b200 as eng
from pytorch_mppi_b200 import _cabi, build


def test_closed_loop_layout_matches_the_library():
    build.build()
    lib = _cabi.load()
    S = _cabi.MppiClosedLoop
    assert lib.mppi_abi_layout(9) == C.sizeof(S) == 88
    assert lib.mppi_abi_layout(10) == S.states.offset
    assert lib.mppi_abi_layout(11) == S.plant_params.offset
    assert lib.mppi_abi_layout(12) == S.plant_blocks.offset
    # argument checks come before any CUDA call
    cl = S(struct_size=C.sizeof(S), steps=1)
    assert lib.mppi_plan_closed_loop(None, C.byref(cl), None) == -1
    assert lib.mppi_plan_model_block_bytes(None) == 0


class _Gen:
    """The torch CUDA generator protocol _next_rng consumes (seed, offset)."""

    def __init__(self, seed=11, offset=40):
        self.seed, self.offset = seed, offset

    def initial_seed(self):
        return self.seed

    def get_offset(self):
        return self.offset

    def set_offset(self, v):
        self.offset = v


class _Lib:
    BLOCK = 48

    def __init__(self):
        self.calls = []

    def mppi_plan_model_block_bytes(self, plan):
        return self.BLOCK

    def mppi_plan_closed_loop(self, plan, cl_ref, stream):
        cl = cl_ref._obj
        plant = None
        if cl.plant_params:
            n = cl.n_plant * cl.n_plant_params
            plant = list((C.c_double * n).from_address(cl.plant_params))
        self.calls.append(dict(steps=cl.steps, seed=cl.seed, offset=cl.offset, stride=cl.offset_stride,
                               n_plant=cl.n_plant, n_plant_params=cl.n_plant_params, plant=plant,
                               costs=bool(cl.costs), disturbance=bool(cl.disturbance), blocks=bool(cl.plant_blocks)))
        return 0


def _controller(monkeypatch, cls=eng.MPPI, model=None, dtype=torch.float32, T=30, nu=1, N=None, rng="seed"):
    """What MPPI.__init__ + _pack leave behind, as far as run_closed_loop reads it."""
    monkeypatch.setattr(torch._C, "_cuda_getCurrentRawStream", lambda index: 0, raising=False)
    gen = _Gen()
    monkeypatch.setattr(torch.cuda, "default_generators", {None: gen})     # indexed by the (CPU) device's index
    c = cls.__new__(cls)
    model = eng.Pendulum() if model is None else model
    c.d, c.dtype, c.nx, c.nu, c.T, c.K = torch.device("cpu"), dtype, model.nx, nu, T, 1024
    if N is not None:
        c.N = N
    c._model, c._model_version, c._dirty, c._resident = model, 0, False, False
    c.u_per_command, c._world, c._z_inject, c._z_out = 1, 1, None, None
    c._rng_mode = "torch" if rng == "torch" else "philox"
    c._rng_seed, c._rng_counter = (7 if rng == "seed" else None), 100
    c._torch_counter_offset = 24
    c._plan, c._lib, c._cmd_count, c._cost_buf = C.c_void_p(1), _Lib(), 3, torch.zeros(4)
    c._base_flags = _cabi.FLAG_DIAG_SIGMA
    c._gen = gen
    return c


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("rng", ["seed", "generator", "torch"])
def test_offset_stride_and_rng_advance(monkeypatch, dtype, rng):
    c = _controller(monkeypatch, dtype=dtype, rng=rng)
    x0 = torch.tensor([3.0, 0.5], dtype=dtype)
    per = 4 if dtype == torch.float32 else 2
    chunks = (30 + per - 1) // per
    res = c.run_closed_loop(x0, 5)
    call = c._lib.calls[-1]
    assert call["steps"] == 5 and call["n_plant"] == 1 and call["plant"] is None and call["costs"] and call["blocks"]
    assert not call["disturbance"]
    if rng == "seed":          # the controller's own counter: one command = `chunks` Philox calls per sample
        assert (call["seed"], call["offset"], call["stride"]) == (7, 100, chunks)
        assert c._rng_counter == 100 + 5 * chunks
    elif rng == "generator":   # the torch CUDA generator's (seed, offset), 4 offsets per Philox call
        assert (call["seed"], call["offset"], call["stride"]) == (11, 10, chunks)
        assert c._gen.offset == 40 + 5 * 4 * chunks
    else:                      # rng="torch": torch.randn's counter increment per command
        assert (call["seed"], call["offset"], call["stride"]) == (11, 10, 6)
        assert c._gen.offset == 40 + 5 * 24
    # a command after the loop continues where `steps` commands leave the stream
    seed, off = c._next_rng()
    assert off == call["offset"] + 5 * call["stride"]
    # the last command's bookkeeping: counter, state, the flags / noise position lazy materialisation reads
    assert c._cmd_count == 8 and c.state.data_ptr() == res.states[4].data_ptr()
    flags, seed_l, off_l, z, sdev = c._last
    assert flags == _cabi.FLAG_DIAG_SIGMA | _cabi.FLAG_STATE_DEVICE | _cabi.FLAG_SHIFT
    assert (seed_l, off_l, z, sdev) == (call["seed"], call["offset"] + 4 * call["stride"], None, res.states[4].data_ptr())


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_result_shapes_and_dtypes(monkeypatch, dtype):
    c = _controller(monkeypatch, dtype=dtype)
    x0 = torch.tensor([3.0, 0.5], dtype=dtype)
    res = c.run_closed_loop(x0, 7, disturbance=torch.zeros(7, 2, dtype=dtype))
    assert isinstance(res, eng.ClosedLoopResult) and res._fields == ("states", "actions", "costs")
    assert res.states.shape == (8, 2) and res.actions.shape == (7, 1) and res.costs.shape == (7,)
    assert all(t.dtype == dtype for t in res) and torch.equal(res.states[0], x0)
    assert c._lib.calls[-1]["disturbance"]
    b = _controller(monkeypatch, cls=eng.MPPI_Batched, dtype=dtype, N=4)
    xs = torch.zeros(4, 2, dtype=dtype)
    res = b.run_closed_loop(xs, 3)
    assert res.states.shape == (4, 4, 2) and res.actions.shape == (3, 4, 1) and res.costs.shape == (3, 4)


def test_plant_params_rows(monkeypatch):
    c = _controller(monkeypatch)
    x0 = torch.tensor([3.0, 0.5])
    heavy = eng.Pendulum(m=1.3).param_blob()
    c.run_closed_loop(x0, 2, plant_params=heavy)
    call = c._lib.calls[-1]
    assert call["n_plant"] == 1 and call["n_plant_params"] == 7 and call["plant"] == heavy
    b = _controller(monkeypatch, cls=eng.MPPI_Batched, N=3)
    rows = [eng.Pendulum(m=1.0 + 0.1 * e).param_blob() for e in range(3)]
    b.run_closed_loop(torch.zeros(3, 2), 2, plant_params=torch.tensor(rows, dtype=torch.float64))
    call = b._lib.calls[-1]
    assert call["n_plant"] == 3 and call["plant"] == [v for r in rows for v in r]
    b.run_closed_loop(torch.zeros(3, 2), 2, plant_params=heavy)     # one plant for every environment
    assert b._lib.calls[-1]["n_plant"] == 1


def _refused(c, *args, match, **kw):
    n = len(c._lib.calls)
    counter = (c._rng_counter, c._cmd_count)
    with pytest.raises(ValueError, match=match):
        c.run_closed_loop(*args, **kw)
    assert len(c._lib.calls) == n and (c._rng_counter, c._cmd_count) == counter      # nothing launched, nothing consumed


def test_refusals(monkeypatch):
    x0 = torch.tensor([3.0, 0.5])
    c = _controller(monkeypatch)
    for steps in (0, -1, 2.0, True, "3"):
        _refused(c, x0, steps, match="steps")
    # state: shape, dtype, device, not a tensor
    _refused(c, torch.zeros(3), 2, match="state")
    _refused(c, torch.zeros(1, 2), 2, match="state")
    _refused(c, x0.double(), 2, match="state")
    _refused(c, torch.zeros(2, device="meta"), 2, match="state")
    _refused(c, [3.0, 0.5], 2, match="state")
    # disturbance
    _refused(c, x0, 2, disturbance=torch.zeros(3, 2), match="disturbance")
    _refused(c, x0, 2, disturbance=torch.zeros(2, 2, dtype=torch.float64), match="disturbance")
    _refused(c, x0, 2, disturbance=torch.zeros(2, 2, device="meta"), match="disturbance")
    _refused(c, x0, 2, disturbance=[[0.0, 0.0]] * 2, match="disturbance")
    # plant parameters
    _refused(c, x0, 2, plant_params=[1.0] * 6, match="plant_params")
    _refused(c, x0, 2, plant_params=torch.zeros(2, 7, dtype=torch.float64), match="plant_params")
    _refused(c, x0, 2, plant_params=torch.zeros(7, dtype=torch.int64), match="plant_params")
    _refused(c, x0, 2, plant_params=torch.zeros(7, device="meta"), match="plant_params")
    b = _controller(monkeypatch, cls=eng.MPPI_Batched, N=3)
    _refused(b, torch.zeros(3, 2), 2, plant_params=torch.zeros(2, 7), match="plant_params")
    _refused(b, torch.zeros(2), 2, match="state")
    _refused(b, torch.zeros(3, 2), 2, disturbance=torch.zeros(2, 2), match="disturbance")
    # controller configurations
    c.u_per_command = 2
    _refused(c, x0, 2, match="u_per_command")
    c.u_per_command = 1
    c._world = 2
    _refused(c, x0, 2, match="sharded")
    c._world = 1
    c._z_inject = torch.zeros(1)
    _refused(c, x0, 2, match="inject_noise")
    c._z_inject = None
    c._z_out = torch.zeros(1)
    _refused(c, x0, 2, match="record_noise")
    c._z_out = None
    c._offset_dev = torch.zeros(1)
    _refused(c, x0, 2, match="compile")
    del c._offset_dev
    c._model = None
    _refused(c, x0, 2, match="stepped route")
    # models
    mlp = eng.PendulumMLP.__new__(eng.PendulumMLP)
    _refused(_controller(monkeypatch, model=mlp), x0, 2, match="PendulumMLP")
    ens = eng.PendulumMLPEnsemble.__new__(eng.PendulumMLPEnsemble)
    _refused(_controller(monkeypatch, model=ens), x0, 2, match="PendulumMLP")
    sd = eng.CudaModel(2, 1, "x[0] = O::add(x[0], u[0]);", "return x[0];", params=[1.0], step_dependent=True)
    _refused(_controller(monkeypatch, model=sd), x0, 2, match="step-dependent")
    # after all of that, a valid call still goes through
    c = _controller(monkeypatch)
    c.run_closed_loop(x0, 2)
    assert len(c._lib.calls) == 1
