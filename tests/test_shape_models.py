"""CPU: the models at the edges of the (nx, nu) envelope (tests/shape_models.py) — NVRTC compilation of every variant
and dtype, the prebuilt cubins the GPU tests load, and that the live-reference fixtures (tests/golden/shape_cases.py)
notice the kernel errors they are meant to catch.  No GPU."""
import numpy as np
import pytest
import torch

from pytorch_mppi_b200 import rtc
from tests import shape_models as shm
from tests.golden.replay import OracleRunner, load
from tests.golden.shape_cases import SHAPE_CASES, sigma_is_full


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("variant", [0, 1, 2])
@pytest.mark.parametrize("nx,nu", shm.SHAPES)
def test_shape_model_compiles_with_nvrtc(nx, nu, variant, dtype):
    m = shm.shape_model(nx, nu)
    assert f"NX = {nx}, NU = {nu}," in m.header_text()
    cubin, names = m.compile_rtc(dtype, variant)
    assert cubin[:4] == b"\x7fELF"
    assert all(names[i] for i in (0, 1, 3, 4)) and (names[2] is not None) == (variant == 0)


def test_build_prebuilt_every_shape_model_kernel(monkeypatch):
    """`__graft_entry__.build()` leaves the cubins of every kernel the GPU tests load in the tree: served from the cache
    with NVRTC out of reach."""
    def no_nvrtc():
        raise rtc.RtcError("NVRTC must not be needed")
    monkeypatch.setattr(rtc, "_load_nvrtc", no_nvrtc)
    for model, dtype, variant in shm.prebuilt():
        cubin, _ = model.compile_rtc(dtype, variant)
        assert len(cubin) > 0


@pytest.mark.parametrize("nx,nu", shm.SHAPES)
def test_every_component_has_its_own_coefficient(nx, nu):
    """Swapping two state components or two action components changes the step and the cost: a kernel that mixes up
    indices cannot agree with the twins by accident."""
    g = torch.Generator().manual_seed(nx * 10 + nu)
    x = torch.randn(64, nx, generator=g, dtype=torch.float64)
    u = torch.randn(64, nu, generator=g, dtype=torch.float64)
    f, c, term = shm.twins(nx, nu)
    for n, swap in ((nx, lambda i, j: (x[:, _perm(nx, i, j)], u)), (nu, lambda i, j: (x, u[:, _perm(nu, i, j)]))):
        for i in range(n):
            for j in range(i + 1, n):
                xs, us = swap(i, j)
                assert not torch.allclose(c(xs, us), c(x, u)), (i, j)
                assert not torch.allclose(f(xs, us), f(x, u)), (i, j)
    states = f(x, u).view(1, 64, 1, nx)
    for i in range(nx):
        for j in range(i + 1, nx):
            assert not torch.allclose(term(states[..., _perm(nx, i, j)], None), term(states, None))


def _perm(n, i, j):
    p = list(range(n))
    p[i], p[j] = p[j], p[i]
    return p


def test_cases_reach_the_envelope():
    assert {(c["model"]["nx"], c["model"]["nu"]) for c in SHAPE_CASES.values()} == set(shm.SHAPES)
    big = SHAPE_CASES["shape_mppi_n8u4_f64"]
    assert sigma_is_full(big) and big["T"] * 4 % 2 == 0 and big["K"] % 32 != 0
    # R = T*nu not a multiple of the normals per Philox call (4 in fp32, 2 in fp64): one call straddles two time steps
    assert SHAPE_CASES["shape_smppi_n3u3_f64"]["T"] * 3 % 2 == 1
    assert SHAPE_CASES["shape_mppi_n3u3_f32"]["T"] * 3 % 4 != 0


@pytest.mark.parametrize("keep", [1, 2, 3])
def test_fixture_detects_a_truncated_colouring(keep):
    """A colouring eps = L z that stops after `keep` of the four components (or an action cost that does the same with
    Sigma^-1) misses the nu=4 fixture by far more than the 1e-9 the engine is held to."""
    case, gold = load("shape_mppi_n8u4_f64")
    run = OracleRunner(case)
    run.prob.sigma_chol = run.prob.sigma_chol.clone()
    run.prob.sigma_chol[:, keep:] = 0
    r = run.step(torch.tensor(case["x0"], dtype=torch.float64), run.stream.next_z())
    assert float(np.abs(r["U"].numpy() - gold["U_0"]).max()) > 1e-4
