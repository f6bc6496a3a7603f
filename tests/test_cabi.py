"""CPU: the C-ABI library loads, exports every symbol include/mppi_b200.h declares, and the ctypes
mirror of MppiFusedParams has the library's layout.  No compute calls (no GPU here)."""
import ctypes as C
import os
import re

import pytest

from pytorch_mppi_b200 import _cabi, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _cabi.load()


def test_header_symbols_all_exported(lib):
    hdr = open(os.path.join(ROOT, "include", "mppi_b200.h")).read()
    declared = set(re.findall(r"^(?:int|uint64_t|const char\*)\s+(mppi_\w+)\s*\(", hdr, flags=re.M))
    assert len(declared) >= 17
    bound = {name for name, _, _ in _cabi.SYMBOLS}
    assert declared == bound, declared ^ bound
    for name in declared:
        assert hasattr(lib, name)


def test_struct_layout_matches_library(lib):
    P = _cabi.MppiFusedParams
    assert lib.mppi_abi_layout(0) == C.sizeof(P)
    for which, field in ((1, "seed"), (2, "state"), (3, "U"), (4, "rank"), (5, "partial_out")):
        assert lib.mppi_abi_layout(which) == getattr(P, field).offset, field
    assert lib.mppi_abi_layout(6) == C.sizeof(_cabi.MppiLaunchInfo)
    assert lib.mppi_b200_abi_version() == _cabi.ABI_VERSION


def test_bad_arguments_return_status_not_crash(lib):
    p = _cabi.MppiFusedParams()
    assert lib.mppi_fused_command(C.byref(p), None) == -5          # struct_size unset -> ABI error
    p.struct_size = C.sizeof(p)
    assert lib.mppi_fused_command(C.byref(p), None) == -1          # K == 0 -> bad argument
    assert lib.mppi_status_string(-3) == b"workspace too small"
    assert lib.mppi_cost_accumulate(None, None, None, 1, 1, 1.0, 0, None) == -1
    # every pointer-taking entry point answers a null / empty request with a status, before any CUDA call
    assert lib.mppi_rollout_states(C.byref(p), None, None, 0, 1, 1, None, None) == -1
    assert lib.mppi_rollout_states(C.byref(p), 16, 16, 0, 0, 1, 16, None) == -1      # n_rollouts < 1
    assert lib.mppi_rollout_states(C.byref(p), 16, 16, -1, 1, 1, 16, None) == -1     # negative stride
    assert lib.mppi_plan_create(C.byref(p), None) == -1
    assert lib.mppi_plan_destroy(None) == -1
    assert lib.mppi_plan_command(None, None, None, 0, 0, 0, None, None, None) == -1
    assert lib.mppi_omega(None, None, None, 1.0, 1, 0, None) == -1
    assert lib.mppi_softmin_update(C.byref(p), None, None, None) == -1
    assert lib.mppi_xchg_open(None, None) == -1
    # resident mode: a null plan / unarmed plan is an argument error, never a launch
    assert lib.mppi_resident_start(None, None, None, None, 1000, None) == -1
    assert lib.mppi_resident_command(None, None, 0, 0, 0, None) == -1
    assert lib.mppi_resident_sync(None) == -1
    assert lib.mppi_resident_stop(None) == -1
    assert lib.mppi_resident_launches(None) == 0
    # a run-time user model without its handle
    u = _cabi.MppiFusedParams(struct_size=C.sizeof(p), model=_cabi.MODEL_USER, K=1, T=1, nx=1, nu=1, u_per_command=1, lambda_=1.0)
    assert lib.mppi_plan_create(C.byref(u), C.byref(C.c_void_p())) == -1


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    monkeypatch.setattr(_cabi, "_lib", None)
    monkeypatch.setattr(_cabi, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_cabi.MppiLibraryError):
        _cabi.load()


def test_cpu_device_is_rejected():
    import torch
    import pytorch_mppi_b200 as eng
    pend = eng.Pendulum()
    with pytest.raises(ValueError, match="CUDA"):
        eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(1.0), device="cpu")
