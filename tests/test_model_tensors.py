"""CPU: user models that read device tensors (CudaModel(tensors=...)) — the generated header and its NVRTC compilation,
the agreement between the views the library packs and the struct the header declares, every ValueError of the Python
API, the ABI of the new fields and the C entry points' argument checks.  No GPU."""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np
import pytest
import torch

import pytorch_mppi_b200 as eng
from pytorch_mppi_b200 import _cabi, build
from tests import tensor_models as tm
from tests import user_models

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pytorch_mppi_b200", "csrc")


def _meta(*shape, dtype=torch.float32):
    return torch.empty(*shape, dtype=dtype, device="meta")


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _cabi.load()


def test_header_without_tensors_is_unchanged():
    sha = lambda m: hashlib.sha1(m.header_text().encode()).hexdigest()
    assert sha(user_models.pendulum_user_model()) == "0f25d3de524f9fb4f81348896838ac5122b65e4f"
    assert "TensorView" not in user_models.integrator_user_model().header_text()


def test_header_depends_on_names_dtypes_and_ndims_only():
    a = tm.nav_model(_meta(64, 64), _meta(20, 2, dtype=torch.float64)).header_text()
    assert a == tm.nav_model(_meta(7, 300), _meta(3, 2, dtype=torch.float64)).header_text()
    assert "TensorView<float, 2> t0; TensorView<double, 2> t1;" in a
    assert a.count("const auto& costmap = P_.t0;") == 3               # step, cost and terminal bodies
    assert a != tm.nav_model(_meta(64, 64, dtype=torch.uint8), _meta(20, 2, dtype=torch.float64)).header_text()


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("variant", [0, 1, 2])
def test_tensor_model_compiles_with_nvrtc(dtype, variant):
    cubin, names = tm.meta_model().compile_rtc(dtype, variant)
    assert cubin[:4] == b"\x7fELF" and all(names[i] for i in (0, 1, 3, 4))


def test_tensor_model_with_copies_and_a_terminal_body_compiles_with_nvrtc():
    m = eng.CudaModel(2, 2, tm.NAV_STEP, tm.nav_cost_code(per_copy=True), params=tm.NAV_PARAMS, step_dependent=True,
                      copies=tm.ENSEMBLE_M, tensors={"costmap": _meta(3, 8, 8), "path": _meta(4, 2, dtype=torch.float64)},
                      terminal_code="return (real)costmap(m, costmap.size(1) - 1, 0) + (real)path.size(0);")
    cubin, names = m.compile_rtc(torch.float64, 2)
    assert cubin[:4] == b"\x7fELF" and names[0] and names[4] and names[1] is None


_LAYOUT_SRC = r"""
#include <stddef.h>
#include <stdio.h>
#define MPPI_HD inline
namespace mppi { template <typename T> struct Ops {}; }
#include "HEADER"
#include "mppi_model_tensors.h"
using namespace mppi;
template <typename real> int check() {
    typedef UserModel::P<real> P;
    static_assert(sizeof(P) % 8 == 0, "");
    if ((int)sizeof(P) != mppi_tensors::block_bytes(UserModel::NP, sizeof(real), 3)) return 1;
    if ((int)offsetof(P, t0) != mppi_tensors::views_offset(UserModel::NP, sizeof(real))) return 2;
    static float a[2 * 3 * 5];
    static unsigned char b[7];
    static int c[2 * 2 * 2 * 3];
    for (int i = 0; i < 30; ++i) a[i] = (float)i;
    for (int i = 0; i < 7; ++i) b[i] = (unsigned char)(10 * i);
    for (int i = 0; i < 24; ++i) c[i] = -i;
    MppiTensorRef refs[3] = {{a, MPPI_F32, 3, {2, 3, 5, 0}}, {b, MPPI_U8, 1, {7, 0, 0, 0}}, {c, MPPI_I32, 4, {2, 2, 2, 3}}};
    P blk;
    memset(&blk, 0xff, sizeof(blk));
    mppi_tensors::pack_views(&blk, UserModel::NP, sizeof(real), refs, 3);
    if (blk.t0.size(0) != 2 || blk.t0.size(1) != 3 || blk.t0.size(2) != 5 || blk.t1.size(0) != 7 || blk.t2.size(3) != 3) return 3;
    if (blk.t0(1, 2, 4) != 29.0f || blk.t0(0, 1, 0) != 5.0f || blk.t1(3) != 30 || blk.t2(1, 0, 1, 2) != -17) return 4;
    // clamped: border replication on every side
    if (blk.t0(-4, 9, 100) != 14.0f || blk.t0(7, -1, -1) != 15.0f || blk.t1(-3) != 0 || blk.t1(99) != 60) return 5;
    if (blk.t2(5, 5, 5, 5) != -23 || blk.t2(-1, -1, -1, -1) != 0) return 6;
    return 0;
}
int main() { int rc = check<float>(); if (!rc) rc = 10 * check<double>(); printf("%d\n", rc); return rc; }
"""


@pytest.mark.parametrize("np_", [1, 3, 7])
def test_packed_views_match_the_generated_struct(tmp_path, np_):
    """The library's packer (csrc/mppi_model_tensors.h) and the struct the generated header declares, compiled together
    on the host: sizeof / offsetof agree, and reads through the header's accessor return the packed tensors' elements,
    clamped, for an odd and an even parameter count in both dtypes."""
    m = eng.CudaModel(2, 1, "", "return (real)0;", params=[1.0] * np_,
                      tensors={"a": _meta(2, 3, 5), "b": _meta(7, dtype=torch.uint8), "c": _meta(2, 2, 2, 3, dtype=torch.int32)})
    (tmp_path / "model.h").write_text(m.header_text())
    (tmp_path / "main.cpp").write_text(_LAYOUT_SRC.replace("HEADER", str(tmp_path / "model.h")))
    exe = tmp_path / "layout"
    subprocess.run(["g++", "-std=c++17", "-O1", f"-I{CSRC}", "-o", str(exe), str(tmp_path / "main.cpp")], check=True)
    assert subprocess.run([str(exe)], capture_output=True, text=True).stdout.strip() == "0"


@pytest.mark.parametrize("name", ["1x", "has space", "x", "m", "p", "real", "O", "P_", "NX", "NU", "NP", "COPIES",
                                  "STEP_DEPENDENT", "int", "return", "__x", ""])
def test_bad_names_are_refused(name):
    with pytest.raises(ValueError, match="C identifier"):
        eng.CudaModel(2, 1, "", "return (real)0;", tensors={name: _meta(4)})


@pytest.mark.parametrize("t,match", [
    (torch.zeros(4), "CUDA"),
    (torch.zeros(4, dtype=torch.int64, device="meta"), "dtype"),
    (torch.zeros(4, dtype=torch.float16, device="meta"), "dtype"),
    (torch.zeros((), device="meta"), "dimensions"),
    (torch.zeros(1, 1, 1, 1, 2, device="meta"), "dimensions"),
    (torch.zeros(4, 6, device="meta").t(), "contiguous"),
    (torch.empty(2 ** 31, dtype=torch.uint8, device="meta"), "elements"),
    ([1.0, 2.0], "torch tensor"),
])
def test_bad_tensors_are_refused(t, match):
    with pytest.raises(ValueError, match=match):
        eng.CudaModel(2, 1, "", "return (real)0;", tensors={"map": t})
    m = eng.CudaModel(2, 1, "", "return (real)0;", tensors={"map": _meta(4)})
    with pytest.raises(ValueError, match=match):
        m.set_tensors(map=t)


def test_too_many_tensors_are_refused():
    with pytest.raises(ValueError, match="at most 8"):
        eng.CudaModel(2, 1, "", "return (real)0;", tensors={f"t{i}": _meta(2) for i in range(9)})


def test_set_tensors():
    m = tm.nav_model(_meta(64, 64), _meta(20, 2, dtype=torch.float64))
    v0, header = m._param_version, m.header_text()
    with pytest.raises(ValueError, match="no tensor 'cost'"):
        m.set_tensors(cost=_meta(64, 64))
    with pytest.raises(ValueError, match="compiled as torch.float32 with 2"):
        m.set_tensors(costmap=_meta(64, 64, dtype=torch.float64))
    with pytest.raises(ValueError, match="compiled as torch.float32 with 2"):
        m.set_tensors(costmap=_meta(64, 64, 2))
    assert m._param_version == v0
    new = _meta(10, 300)
    m.set_tensors(costmap=new)
    assert m._param_version == v0 + 1 and m.tensors["costmap"] is new and m.header_text() == header


def test_tensor_refs_refuse_another_device():
    m = tm.nav_model(_meta(64, 64), _meta(20, 2, dtype=torch.float64))
    with pytest.raises(ValueError, match="controller on cuda:0"):
        m.tensor_refs(torch.device("cuda", 0))
    assert eng.CudaModel(2, 1, "", "return (real)0;").tensor_refs("cuda:0") is None


def test_abi_layout_of_the_new_fields(lib):
    P = _cabi.MppiFusedParams
    assert lib.mppi_b200_abi_version() == _cabi.ABI_VERSION == 3
    assert lib.mppi_abi_layout(0) == C.sizeof(P)
    assert lib.mppi_abi_layout(7) == P.model_weights.offset
    assert lib.mppi_abi_layout(8) == P.model_tensors.offset
    # the tensor fields sit in front of model_weights, which stays the last field
    assert P.model_tensors.offset == P.var_discount.offset + 8
    assert P.n_model_tensors.offset == P.model_tensors.offset + 8
    assert P.model_weights.offset == P.n_model_tensors.offset + 8 == C.sizeof(P) - 8
    assert C.sizeof(_cabi.MppiTensorRef) == 48 and _cabi.MppiTensorRef.shape.offset == 16


def test_entry_points_refuse_bad_arguments_before_any_cuda_call(lib):
    dt = (C.c_int32 * 2)(_cabi.F32, _cabi.F64)
    nd = (C.c_int32 * 2)(2, 2)
    assert lib.mppi_user_model_set_tensors(None, 2, dt, nd) == -1
    fake = (C.c_uint32 * 64)()                               # not a handle: wrong magic
    assert lib.mppi_user_model_set_tensors(fake, 2, dt, nd) == -1
    refs = (_cabi.MppiTensorRef * 1)()
    assert lib.mppi_plan_set_model_tensors(None, refs, 1) == -1
    assert lib.mppi_plan_set_model_tensors(None, None, 0) == -1
    # a registered model takes no tensors: the count differs from the model's (0)
    p = _cabi.MppiFusedParams(struct_size=C.sizeof(_cabi.MppiFusedParams), model=_cabi.MODEL_PENDULUM, K=64, T=4, nx=2,
                              nu=1, u_per_command=1, lambda_=1.0)
    p.model_tensors = C.cast(refs, C.c_void_p)
    p.n_model_tensors = 1
    assert lib.mppi_plan_create(C.byref(p), C.byref(C.c_void_p())) == -1
    assert lib.mppi_rollout_states(C.byref(p), 16, 16, 0, 1, 1, 16, None) == -1


def test_twin_clamps_lookups_to_the_border():
    """The twin's bilinear lookup outside the map equals the border values (what the kernel's clamped accessor reads)."""
    cm = torch.arange(12, dtype=torch.float32).view(3, 4)
    p = [0.1, 0.0, 0.0, 1.0, 1.0, 0.0, 0.0]
    s = torch.tensor([[-5.0, -7.0], [100.0, 0.0], [0.0, 100.0], [100.0, 100.0]])
    np.testing.assert_array_equal(tm.bilinear(cm, s, p).numpy(), [0.0, 3.0, 8.0, 11.0])
