"""CPU: the Python side of `MPPI_Batched.set_env_params()` with the C entry points replaced by a stub (a controller
cannot be built without a CUDA device, so the object is assembled by hand on the CPU "device").  Pins the MppiEnvParams
layout, the factors Python hands the library (the reference's formulas for diagonal and full covariances), that no plan
is created, that clearing restores the shared values, and every refusal, raised before anything launches."""
import ctypes as C

import pytest
import torch

import pytorch_mppi_b200 as eng
from pytorch_mppi_b200 import _cabi, build
from pytorch_mppi_b200.mppi import _factor_sigma


def test_env_params_layout_matches_the_library():
    build.build()
    lib = _cabi.load()
    S = _cabi.MppiEnvParams
    assert lib.mppi_abi_layout(13) == C.sizeof(S) == 72
    assert lib.mppi_abi_layout(14) == S.chol.offset
    assert lib.mppi_abi_layout(15) == S.model_params.offset
    assert lib.mppi_abi_layout(16) == S.scratch.offset
    # argument checks come before any CUDA call
    ep = S(struct_size=C.sizeof(S), n_env=2)
    assert lib.mppi_plan_set_env_params(None, C.byref(ep), None) == -1
    assert lib.mppi_plan_env_scratch_bytes(None) == 0


class _Lib:
    SCRATCH = 512

    def __init__(self):
        self.calls, self.creates, self.refuse = [], 0, False

    def mppi_plan_create(self, p, out):
        self.creates += 1
        return 0

    def mppi_plan_env_scratch_bytes(self, plan):
        return self.SCRATCH

    def mppi_plan_set_env_params(self, plan, ep_ref, stream):
        ep = ep_ref._obj
        n, MU = ep.n_env, _cabi.MPPI_MAX_NU
        rd = lambda ptr, k: None if not ptr else list((C.c_double * k).from_address(ptr))
        self.calls.append(dict(n_env=n, lam=rd(ep.lambda_, n), chol=rd(ep.chol, n * MU * MU),
                               sinv=rd(ep.sigma_inv, n * MU * MU), mu=rd(ep.noise_mu, n * MU),
                               mp=rd(ep.model_params, n * ep.n_model_params), n_mp=ep.n_model_params,
                               scratch=bool(ep.scratch), size=ep.struct_size))
        return -2 if self.refuse else 0          # MPPI_ERR_UNSUPPORTED


def _controller(monkeypatch, model=None, N=3, nu=2, dtype=torch.float64):
    monkeypatch.setattr(torch._C, "_cuda_getCurrentRawStream", lambda index: 0, raising=False)
    c = eng.MPPI_Batched.__new__(eng.MPPI_Batched)
    model = eng.LinearPoint.unit_test_env() if model is None else model
    c.d, c.dtype, c.nx, c.nu, c.T, c.K, c.N = torch.device("cpu"), dtype, 2, nu, 10, 64, N
    c._model, c._plan, c._lib = model, C.c_void_p(1), _Lib()
    c._env_model_params = c._env_lambda = c._env_sigma = c._env_mu = c._env_factors = None
    c._env_scratch = None
    c._lambda = 1.0
    c._noise_mu = torch.zeros(nu, dtype=dtype)
    c._set_sigma(torch.eye(nu, dtype=dtype))
    return c


def test_factors_are_the_reference_formulas(monkeypatch):
    c = _controller(monkeypatch)
    diag = torch.tensor([[0.5, 0.0], [0.0, 2.0]], dtype=torch.float64)
    full = torch.tensor([[1.2, -0.3], [-0.3, 0.4]], dtype=torch.float64)
    sig = torch.stack([diag, full, diag * 3])
    c.set_env_params(noise_sigma=sig)
    call = c._lib.calls[-1]
    L = torch.tensor(call["chol"], dtype=torch.float64).view(3, 4, 4)[:, :2, :2]
    Si = torch.tensor(call["sinv"], dtype=torch.float64).view(3, 4, 4)[:, :2, :2]
    for e, s in enumerate(sig):
        if e != 1:      # diagonal: sqrt / 1/diag (mppi.py:131-136)
            assert torch.equal(L[e], torch.diag(torch.sqrt(torch.diag(s))))
            assert torch.equal(Si[e], torch.diag(1.0 / torch.diag(s)))
        else:           # full: cholesky / inv (mppi.py:138-139)
            assert torch.equal(L[e], torch.linalg.cholesky(s))
            assert torch.equal(Si[e], torch.linalg.inv(s))
        assert torch.equal(L[e], _factor_sigma(s)[1])
    assert call["lam"] is None and call["mu"] is None and call["mp"] is None and call["scratch"]
    assert call["size"] == C.sizeof(_cabi.MppiEnvParams)


def test_no_plan_is_created_and_clearing_restores_shared(monkeypatch):
    c = _controller(monkeypatch)
    lin = eng.LinearPoint.unit_test_env()
    rows = [lin.param_blob()] * 3
    c.set_env_params(model_params=rows, lambda_=[0.5, 1.0, 2.0], noise_mu=[[0.1, 0.0], [0.0, 0.2], [0.0, 0.0]])
    assert c._lib.creates == 0
    call = c._lib.calls[-1]
    assert call["lam"] == [0.5, 1.0, 2.0] and call["n_mp"] == len(lin.param_blob()) and call["mp"] == sum(rows, [])
    assert call["mu"][:2] == [0.1, 0.0] and call["mu"][4:6] == [0.0, 0.2]
    assert c.env_lambda.tolist() == [0.5, 1.0, 2.0] and c.env_model_params.shape == (3, len(lin.param_blob()))
    assert c.env_noise_mu.shape == (3, 2) and c.env_noise_sigma is None
    c.set_env_params()
    call = c._lib.calls[-1]
    assert all(call[k] is None for k in ("lam", "chol", "sinv", "mu", "mp")) and not call["scratch"]
    assert c.env_lambda is None and c.env_model_params is None and c.env_noise_mu is None and c.env_noise_sigma is None
    assert c._lib.creates == 0
    # without a plan yet, the settings wait for it: nothing is handed over
    c._plan = None
    n = len(c._lib.calls)
    c.set_env_params(lambda_=[1.0, 1.0, 1.0])
    assert len(c._lib.calls) == n and c.env_lambda is not None


@pytest.mark.parametrize("kw,why", [
    (dict(lambda_=[1.0, 0.0, 1.0]), "> 0"),
    (dict(lambda_=[1.0, -2.0, 1.0]), "> 0"),
    (dict(lambda_=[1.0, 1.0]), "shape"),
    (dict(lambda_=torch.tensor([1, 1, 1])), "float32 or float64"),
    (dict(noise_sigma=torch.eye(2).expand(2, 2, 2)), "shape"),
    (dict(noise_sigma=torch.tensor([[[1.0, 2.0], [2.0, 1.0]]] * 3)), "positive definite"),
    (dict(noise_sigma=torch.tensor([[[1.0, 0.0], [0.0, -1.0]]] * 3)), "positive definite"),
    (dict(noise_sigma=torch.tensor([[[1.0, 0.1], [0.2, 1.0]]] * 3)), "symmetric"),
    (dict(noise_mu=torch.zeros(3, 3)), "shape"),
    (dict(model_params=torch.zeros(3, 4)), "shape"),
    (dict(lambda_=[1.0, float("nan"), 1.0]), "non-finite"),
])
def test_refusals_before_anything_launches(monkeypatch, kw, why):
    c = _controller(monkeypatch)
    with pytest.raises(ValueError, match=why):
        c.set_env_params(**kw)
    assert c._lib.calls == [] and c.env_lambda is None and c.env_noise_sigma is None


def test_a_library_refusal_keeps_the_settings_the_plan_has(monkeypatch):
    """The library refuses the new settings: every per-environment attribute (omega's lambda, _sample_noise's factors
    and mu, the model blocks) is still the one the plan was given before."""
    build.build()
    c = _controller(monkeypatch)
    lin = eng.LinearPoint.unit_test_env()
    sig = torch.tensor([[[0.5, 0.0], [0.0, 2.0]]] * 3, dtype=torch.float64)
    c.set_env_params(model_params=[lin.param_blob()] * 3, lambda_=[0.5, 1.0, 2.0], noise_sigma=sig)
    before = (c._env_model_params, c._env_lambda, c._env_sigma, c._env_mu, c._env_factors)
    c._lib.refuse = True
    for kw in (dict(lambda_=[3.0, 3.0, 3.0], noise_mu=[[0.1, 0.0]] * 3), dict()):
        with pytest.raises(_cabi.MppiLibraryError, match="mppi_plan_set_env_params"):
            c.set_env_params(**kw)
        after = (c._env_model_params, c._env_lambda, c._env_sigma, c._env_mu, c._env_factors)
        assert all(a is b for a, b in zip(after, before)), kw
    assert c.env_lambda.tolist() == [0.5, 1.0, 2.0] and c.env_noise_mu is None


def test_one_environment_refuses_per_environment_settings(monkeypatch):
    """MPPI_Batched(num_envs=1): the library has no per-environment settings for one environment, so a setting raises
    ValueError before any attribute changes; clearing is a no-op."""
    c = _controller(monkeypatch, N=1)
    for kw in (dict(lambda_=[2.0]), dict(noise_mu=[[0.1, 0.0]]), dict(model_params=[eng.LinearPoint.unit_test_env().param_blob()])):
        with pytest.raises(ValueError, match="one environment"):
            c.set_env_params(**kw)
        assert c.env_lambda is None and c.env_noise_mu is None and c.env_model_params is None and c._env_factors is None
    c.set_env_params()
    assert c._lib.calls == [] and c.env_lambda is None


def test_refusal_on_a_device_other_than_the_controllers(monkeypatch):
    c = _controller(monkeypatch)
    with pytest.raises(ValueError, match="on the CPU"):
        c.set_env_params(lambda_=torch.ones(3, device="meta"))
    assert c._lib.calls == []


def test_refusal_of_mlp_model_params_and_of_the_stepped_route(monkeypatch):
    net = torch.nn.Sequential(torch.nn.Linear(3, 32), torch.nn.Tanh(), torch.nn.Linear(32, 32), torch.nn.Tanh(),
                              torch.nn.Linear(32, 2))
    mlp = eng.PendulumMLP(net)
    c = _controller(monkeypatch, model=mlp, nu=1, dtype=torch.float32)
    n = len(mlp.param_blob()) + len(mlp.param_blob_ext())
    with pytest.raises(ValueError, match="PendulumMLP"):
        c.set_env_params(model_params=torch.zeros(3, n))
    c.set_env_params(lambda_=[1.0, 2.0, 3.0])       # the noise side is per environment on the MLP's batched kernel too
    c2 = _controller(monkeypatch)
    c2._model = None
    with pytest.raises(ValueError, match="fused route"):
        c2.set_env_params(lambda_=[1.0, 2.0, 3.0])
    assert c2._lib.calls == []
