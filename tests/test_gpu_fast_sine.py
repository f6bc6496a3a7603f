"""GPU: the pendulum's branch-free sine and its range guard.

`Ops<float>::sin_fast_` (csrc/mppi_math.cuh) must return exactly what the library's `sinf` returns for every float with
|x| < 105615 and for NaN: it is checked here on all of them.  The built-in pendulum rolls out on it only when its range
guard holds; starts outside the guard (far out, NaN, infinite) run the exact step, so the built-in pendulum must agree
to the bit with the user-written one (tests/user_models.py, which calls `sinf`) everywhere, on every route that steps
the model: the split-cost and single-loop command kernels, the resident kernel and `get_rollouts`' states kernel."""
import ctypes
import math
import os
import subprocess

import pytest
import torch

import pytorch_mppi_b200 as eng
from tests import user_models

pytestmark = pytest.mark.gpu

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pytorch_mppi_b200", "csrc")

SCAN_SRC = r"""
#include "mppi_math.cuh"
// one thread per float bit pattern: count the inputs in the fast range (or NaN) and those where sin_fast_ != sinf
__global__ void scan(unsigned long long base, unsigned long long* out) {
    const unsigned long long i = base + blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
    const unsigned bits = (unsigned)i;
    const float x = __uint_as_float(bits);
    const bool in = fabsf(x) < mppi::Ops<float>::SIN_FAST_RANGE || x != x;
    const float a = sinf(x), b = mppi::Ops<float>::sin_fast_(x);
    const bool same = __float_as_uint(a) == __float_as_uint(b) || (a != a && b != b);
    const unsigned n_in = __popc(__ballot_sync(0xffffffffu, in));
    if ((threadIdx.x & 31) == 0 && n_in) atomicAdd(out, (unsigned long long)n_in);
    if (in && !same && atomicAdd(out + 1, 1ull) == 0) {
        out[2] = bits;
        out[3] = __float_as_uint(a);
        out[4] = __float_as_uint(b);
    }
}
extern "C" int scan_all(unsigned long long* out) {      // out: device, 5 words, zeroed
    const unsigned long long chunk = 1ull << 30;
    for (unsigned long long base = 0; base < (1ull << 32); base += chunk) scan<<<(unsigned)(chunk / 256), 256>>>(base, out);
    return (int)cudaDeviceSynchronize();
}
"""


@pytest.fixture(scope="module")
def scan_lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("fast_sine")
    src, lib = d / "scan.cu", d / "libscan.so"
    src.write_text(SCAN_SRC)
    nvcc = os.environ.get("NVCC", "nvcc")
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-shared", "-Xcompiler", "-fPIC",
                    "-I", CSRC, str(src), "-o", str(lib)], check=True, capture_output=True, text=True)
    return ctypes.CDLL(str(lib))


def test_fast_sine_is_sinf_bit_for_bit_over_its_whole_range(scan_lib):
    out = torch.zeros(5, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    assert scan_lib.scan_all(ctypes.c_void_p(out.data_ptr())) == 0
    tested, bad, x, want, got = (int(v) & 0xFFFFFFFFFFFFFFFF for v in out.cpu())
    n_range = 2 * 0x47CE4780                          # |x| < 105615 = 0x47ce4780: bit patterns 0 .. 0x47ce477f, both signs
    n_nan = 2 * (0x7FFFFFFF - 0x7F800000)             # exponent all ones, mantissa non-zero, both signs
    assert tested == n_range + n_nan
    assert bad == 0, f"{bad} mismatches, first at x = {x:#010x}: sinf {want:#010x}, sin_fast_ {got:#010x}"


def _controller(model, K, T, seed):
    return eng.MPPI(model.dynamics, model.running_cost, 2, torch.tensor(10.0), num_samples=K, horizon=T,
                    U_init=torch.zeros(T, 1), u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda", rng_seed=seed)


def _run(model, state, split, monkeypatch):
    monkeypatch.setenv("MPPI_B200_SPLIT_COST", "1" if split else "0")
    c = _controller(model, 4096, 25, 7)
    assert c._model is model
    outs = [c.command(state).clone() for _ in range(2)]
    assert c.launch_info.split_cost == (1 if split else 0)
    outs.append(c.U.clone())
    outs.append(c.cost_total.clone())
    outs.append(c.get_rollouts(torch.tensor(state)).reshape(-1))
    if split:
        with c.resident(idle_us=200000):
            outs.append(c.command_host(state).to("cuda"))
    return outs


# inside the guard (including a start close to its edge: 105000 + 25 (0.4 + 1) < 105615), and outside it
STATES = [(3.0, 0.4), (-2.5, 7.9), (105000.0, 8.0), (-105000.0, -8.0), (2.0e5, 1.0), (-3.0e7, 0.0), (1.0e38, 0.5),
          (math.inf, 0.0), (-math.inf, 1.0), (math.nan, 0.0), (0.5, math.nan), (0.5, math.inf)]


@pytest.mark.parametrize("split", [True, False], ids=["split", "single_loop"])
@pytest.mark.parametrize("state", STATES, ids=[f"{s[0]:g},{s[1]:g}" for s in STATES])
def test_builtin_pendulum_matches_the_sinf_pendulum_inside_and_outside_the_guard(state, split, monkeypatch):
    builtin = eng.Pendulum()
    user = user_models.pendulum_user_model()
    a = _run(builtin, list(state), split, monkeypatch)
    b = _run(user, list(state), split, monkeypatch)
    for x, y in zip(a, b):
        assert torch.equal(torch.nan_to_num(x, nan=12345.0), torch.nan_to_num(y, nan=12345.0)), (state, split)
        assert torch.equal(torch.isnan(x), torch.isnan(y))

