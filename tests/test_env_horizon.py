"""CPU: the Python side of `MPPI_Batched.set_env_horizon()` with the C entry points replaced by a stub (a controller
cannot be built without a CUDA device, so the object is assembled by hand on the CPU "device").  Pins the int32 array
handed to the library, that no plan is created, that rows past each horizon hold u_init after set_env_horizon and after
reset(), every refusal (raised before anything is handed over), and the ABI's argument checks."""
import ctypes as C

import pytest
import torch

import pytorch_mppi_b200 as eng
from pytorch_mppi_b200 import _cabi, build


def test_abi_checks_come_before_any_cuda_call():
    build.build()
    lib = _cabi.load()
    h = (C.c_int32 * 3)(3, 4, 5)
    assert lib.mppi_plan_set_env_horizon(None, h, None, None) == -1          # MPPI_ERR_BAD_ARG
    assert lib.mppi_plan_set_env_horizon(None, None, None, None) == -1
    assert lib.mppi_plan_env_horizon_bytes(None) == 0


class _Lib:
    def __init__(self):
        self.calls, self.creates, self.refuse = [], 0, False

    def mppi_plan_create(self, p, out):
        self.creates += 1
        return 0

    def mppi_plan_env_horizon_bytes(self, plan):
        return 16

    def mppi_plan_set_env_horizon(self, plan, h, scratch, stream):
        n = 3
        self.calls.append(dict(h=None if not h else list((C.c_int32 * n).from_address(h)), scratch=bool(scratch)))
        return -2 if self.refuse else 0          # MPPI_ERR_UNSUPPORTED


def _controller(monkeypatch, model=None, N=3, nu=2, T=6, upc=1, dtype=torch.float64):
    monkeypatch.setattr(torch._C, "_cuda_getCurrentRawStream", lambda index: 0, raising=False)
    c = eng.MPPI_Batched.__new__(eng.MPPI_Batched)
    model = eng.LinearPoint.unit_test_env() if model is None else model
    c.d, c.dtype, c.nx, c.nu, c.T, c.K, c.N = torch.device("cpu"), dtype, 2, nu, T, 64, N
    c.u_per_command = upc
    c._model, c._plan, c._lib = model, C.c_void_p(1), _Lib()
    c._env_model_params = c._env_lambda = c._env_sigma = c._env_mu = c._env_factors = None
    c._env_scratch = c._env_horizon = c._env_horizon_scratch = None
    c._lambda = 1.0
    c._noise_mu = torch.zeros(nu, dtype=dtype)
    c._set_sigma(torch.eye(nu, dtype=dtype))
    c._u_init = torch.tensor([0.25, -0.5][:nu], dtype=dtype)
    c._Ubuf = torch.zeros(N, 16, dtype=dtype)
    c.U = torch.arange(N * T * nu, dtype=dtype).view(N, T, nu) + 1.0
    return c


def test_int32_array_and_rows_past_the_horizon(monkeypatch):
    c = _controller(monkeypatch)
    U_before = c.U.clone()
    c.set_env_horizon([6, 2, 4])
    assert c._lib.calls[-1] == dict(h=[6, 2, 4], scratch=True) and c._lib.creates == 0
    assert c.env_horizon.dtype == torch.int32 and c.env_horizon.tolist() == [6, 2, 4]
    for e, h in enumerate([6, 2, 4]):
        assert torch.equal(c.U[e, :h], U_before[e, :h])                  # kept: change_horizon truncates
        assert torch.equal(c.U[e, h:], c._u_init.expand(6 - h, 2))        # ... and extends with u_init
    # growing a horizon extends with u_init (the rows it held past the old horizon)
    c.set_env_horizon(torch.tensor([6, 5, 4]))
    assert torch.equal(c.U[1, 2:], c._u_init.expand(4, 2))
    assert c._lib.calls[-1]["h"] == [6, 5, 4]
    # reset(): fresh random rows inside each horizon, u_init past it
    torch.manual_seed(0)
    c.reset()
    for e, h in enumerate([6, 5, 4]):
        assert torch.equal(c.U[e, h:], c._u_init.expand(6 - h, 2))
        assert not torch.equal(c.U[e, :h], c._u_init.expand(h, 2))
    # None: every environment back to T, nothing changed in U
    U_now = c.U.clone()
    c.set_env_horizon(None)
    assert c._lib.calls[-1] == dict(h=None, scratch=False) and c.env_horizon is None
    assert torch.equal(c.U, U_now) and c._lib.creates == 0
    # without a plan yet, the horizons wait for it
    c._plan = None
    n = len(c._lib.calls)
    c.set_env_horizon([3, 3, 3])
    assert len(c._lib.calls) == n and c.env_horizon.tolist() == [3, 3, 3]


@pytest.mark.parametrize("h,why", [
    ([6, 0, 4], r"\[1, T=6\]"),
    ([6, 7, 4], r"\[1, T=6\]"),
    ([6, -1, 4], r"\[1, T=6\]"),
    ([6, 4], "shape"),
    ([[6, 4, 4]], "shape"),
    ([6.0, 4.0, 4.0], "integers"),
    (torch.tensor([True, True, True]), "integers"),
])
def test_refusals_before_anything_is_handed_over(monkeypatch, h, why):
    c = _controller(monkeypatch)
    U_before = c.U.clone()
    with pytest.raises(ValueError, match=why):
        c.set_env_horizon(h)
    assert c._lib.calls == [] and c.env_horizon is None and torch.equal(c.U, U_before)


def test_a_library_refusal_keeps_the_horizons_and_U(monkeypatch):
    """The library refuses the new horizons (or the return to T): the controller keeps the horizons the plan has, and
    U is not filled with u_init past horizons that never took effect."""
    build.build()
    c = _controller(monkeypatch)
    c.set_env_horizon([6, 2, 4])
    h_before, U_before = c.env_horizon, c.U.clone()
    c._lib.refuse = True
    for h in ([3, 3, 3], None):
        with pytest.raises(_cabi.MppiLibraryError, match="mppi_plan_set_env_horizon"):
            c.set_env_horizon(h)
        assert c.env_horizon is h_before and c.env_horizon.tolist() == [6, 2, 4], h
        assert torch.equal(c.U, U_before), h


def test_one_environment_refuses_per_environment_horizons(monkeypatch):
    """MPPI_Batched(num_envs=1): ValueError before anything changes; None is a no-op."""
    c = _controller(monkeypatch, N=1)
    U_before = c.U.clone()
    with pytest.raises(ValueError, match="one environment"):
        c.set_env_horizon([3])
    c.set_env_horizon(None)
    assert c.env_horizon is None and torch.equal(c.U, U_before) and c._lib.calls == []


def test_refusal_below_u_per_command(monkeypatch):
    c = _controller(monkeypatch, upc=3)
    with pytest.raises(ValueError, match=r"\[3, T=6\]"):
        c.set_env_horizon([6, 2, 4])
    c.set_env_horizon([6, 3, 4])
    assert c._lib.calls[-1]["h"] == [6, 3, 4]


def test_refusal_of_the_stepped_route_and_the_mlp_models(monkeypatch):
    c = _controller(monkeypatch)
    c._model = None
    with pytest.raises(ValueError, match="fused route"):
        c.set_env_horizon([6, 6, 6])
    net = torch.nn.Sequential(torch.nn.Linear(3, 32), torch.nn.Tanh(), torch.nn.Linear(32, 32), torch.nn.Tanh(),
                              torch.nn.Linear(32, 2))
    c2 = _controller(monkeypatch, model=eng.PendulumMLP(net), nu=1, dtype=torch.float32)
    with pytest.raises(ValueError, match="PendulumMLP"):
        c2.set_env_horizon([6, 6, 6])
    assert c._lib.calls == [] and c2._lib.calls == []
