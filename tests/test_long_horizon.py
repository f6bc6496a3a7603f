"""tile_memory (global-tile kernels) without a GPU: the keyword's validation, the C ABI of MPPI_FLAG_GLOBAL_TILE and
MppiLaunchInfo.global_tile, and the refusals the library makes before any CUDA call."""
import ctypes as C

import pytest
import torch

import pytorch_mppi_b200 as eng
from pytorch_mppi_b200 import _cabi


@pytest.fixture(scope="module")
def lib():
    return _cabi.load()


def _dyn(s, a):
    return s


def _cost(s, a):
    return s[:, 0]


@pytest.mark.parametrize("cls", [eng.MPPI, eng.SMPPI, eng.KMPPI])
@pytest.mark.parametrize("bad", ["SHARED", "l2", "", None, 1])
def test_tile_memory_is_validated_before_anything_else(cls, bad):
    with pytest.raises(ValueError, match="tile_memory"):
        cls(_dyn, _cost, 2, torch.eye(2, dtype=torch.float64), num_samples=64, horizon=8, tile_memory=bad)


def test_batched_tile_memory_is_validated():
    with pytest.raises(ValueError, match="tile_memory"):
        eng.MPPI_Batched(_dyn, _cost, 2, torch.eye(2, dtype=torch.float64), 2, num_samples=64, horizon=8, tile_memory="x")


def test_flag_and_launch_info_layout(lib):
    assert _cabi.FLAG_GLOBAL_TILE == 1 << 11
    flags = [v for k, v in vars(_cabi).items() if k.startswith("FLAG_") and k != "FLAG_GLOBAL_TILE"]
    assert all(f & _cabi.FLAG_GLOBAL_TILE == 0 for f in flags)
    assert _cabi.MppiLaunchInfo.global_tile.offset == 60
    assert C.sizeof(_cabi.MppiLaunchInfo) == 64 == lib.mppi_abi_layout(6)


def _params(**kw):
    p = _cabi.MppiFusedParams(struct_size=C.sizeof(_cabi.MppiFusedParams), K=256, T=600, nx=2, nu=4, u_per_command=1,
                              lambda_=1.0, dtype=_cabi.F64, flags=_cabi.FLAG_GLOBAL_TILE)
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _refusal(lib, rc):
    assert rc == -2, rc
    return lib.mppi_last_cuda_error().decode()


def test_sharded_global_tile_is_refused_before_any_cuda_call(lib):
    p = _params(world=2)
    info = _cabi.MppiLaunchInfo()
    assert "sharded" in _refusal(lib, lib.mppi_fused_query(C.byref(p), C.byref(info)))
    buf = C.create_string_buffer(64)
    assert "sharded" in _refusal(lib, lib.mppi_sample_perturb(C.byref(_params(world=2, U=16, nominal_used=16)), buf, buf, None,
                                                               None, None, 0, 0, None))
    p = _params(world=1, flags=_cabi.FLAG_GLOBAL_TILE | _cabi.FLAG_EXPORT_PARTIAL)
    assert "sharded" in _refusal(lib, lib.mppi_fused_query(C.byref(p), C.byref(info)))


def test_pendulum_mlp_global_tile_is_refused_before_any_cuda_call(lib):
    ext = (C.c_double * 4096)()
    p = _params(model=_cabi.MODEL_PENDULUM_MLP, nx=2, nu=1, T=40, model_params_ext=C.cast(ext, C.c_void_p),
                n_model_params_ext=4096)
    info = _cabi.MppiLaunchInfo()
    assert "PendulumMLP" in _refusal(lib, lib.mppi_fused_query(C.byref(p), C.byref(info)))
