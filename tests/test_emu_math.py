"""CPU: the per-sample math header the kernels are built from (csrc/mppi_math.cuh), compiled for the host
with g++ (tests/emu/emu_math.cpp — test infrastructure, never part of the product path), against the oracle:
Philox known answers, the normal-stream definition, model rollouts (states and accumulated cost), noise
colouring and the action-cost term, torch.remainder semantics.

g++ takes the header's host branch.  For the float primitives with a separate device body (fmod_, fmod_small_ and
remainder, tanh_ and tanh4_, Normals<float>::pair) that branch is plain libm, so this file checks the host bodies only;
tests/test_gpu_device_math.py checks the device bodies on the GPU."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import mppi_oracle as orc
from oracle import philox_oracle as po
import pytorch_mppi_b200 as eng

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "emu_math.cpp")
OUT = os.path.join(HERE, "emu", "_emu_math.so")


@pytest.fixture(scope="module")
def emu():
    deps = [SRC, os.path.join(os.path.dirname(HERE), "pytorch_mppi_b200", "csrc", "mppi_math.cuh")]
    if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in deps):
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-o", OUT, SRC], check=True)
    lib = C.CDLL(OUT)
    lib.emu_remainder.restype = C.c_double
    lib.emu_remainder.argtypes = [C.c_double, C.c_double]
    lib.emu_remainderf.restype = C.c_float
    lib.emu_remainderf.argtypes = [C.c_float, C.c_float]
    lib.emu_colour_and_action_cost.restype = C.c_double
    return lib


def _arr(x):
    a = np.ascontiguousarray(np.asarray(x, dtype=np.float64))
    return a, a.ctypes.data_as(C.c_void_p)


def test_philox_and_normals_match_the_stream_definition(emu):
    out = (C.c_uint32 * 4)()
    emu.emu_philox(C.c_uint64(0), C.c_uint64(0), C.c_uint64(0), out)
    assert list(out) == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]
    seed, k, off = 0xDEADBEEF12345, 77, 5
    ctr = np.array([[off & 0xFFFFFFFF, off >> 32, k & 0xFFFFFFFF, k >> 32]], dtype=np.uint32)
    want = po.philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32))[0]
    emu.emu_philox(C.c_uint64(seed), C.c_uint64(k), C.c_uint64(off), out)
    assert list(out) == [int(v) for v in want]
    f4 = (C.c_float * 4)()
    emu.emu_normals_f32(C.c_uint64(seed), C.c_uint64(k), C.c_uint64(off), f4)
    np.testing.assert_allclose(np.array(list(f4)), po.normals(seed, off, k, 1, 4, np.float32)[0], atol=2e-6)
    d2 = (C.c_double * 2)()
    emu.emu_normals_f64(C.c_uint64(seed), C.c_uint64(k), C.c_uint64(off), d2)
    np.testing.assert_allclose(np.array(list(d2)), po.normals(seed, off, k, 1, 2, np.float64)[0], atol=1e-13)


def _rollout(emu, model_id, dtype_id, blob, ext, T, x0, v, u_scale, nx):
    blob_a, blob_p = _arr(list(blob) + [0.0] * (48 - len(blob)))
    ext_a, ext_p = _arr(ext if len(ext) else [0.0])
    x0_a, x0_p = _arr(x0)
    v_a, v_p = _arr(v)
    states = np.zeros((T, nx))
    cost = C.c_double()
    rc = emu.emu_rollout(model_id, dtype_id, blob_p, ext_p if len(ext) else None, len(ext), T, x0_p, v_p, C.c_double(u_scale),
                         states.ctypes.data_as(C.c_void_p), C.byref(cost))
    assert rc == 0
    return states, cost.value


@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-13), (torch.float32, 3e-6)])
def test_pendulum_rollout_matches_oracle(emu, dtype, tol):
    g = torch.Generator().manual_seed(0)
    T = 40
    model = orc.PendulumModel(numpy_sin=False)
    for trial in range(5):
        x0 = (torch.randn(2, generator=g) * torch.tensor([3.0, 2.0])).to(dtype)
        v = (torch.randn(T, 1, generator=g) * 3).to(dtype)
        s = x0.view(1, 2)
        cost = torch.zeros(1, dtype=dtype)
        want = []
        for t in range(T):
            s = model.dynamics(s, v[t].view(1, 1))
            cost = cost + model.running_cost(s, v[t].view(1, 1))
            want.append(s[0].clone())
        got, c = _rollout(emu, 1, 0 if dtype == torch.float32 else 1, eng.Pendulum().param_blob(), [], T, x0.double().tolist(),
                          v.double().reshape(-1).tolist(), 1.0, 2)
        np.testing.assert_allclose(got, torch.stack(want).double().numpy(), atol=tol * 10, rtol=0)
        assert abs(c - cost.item()) <= tol * max(1.0, abs(cost.item())) * 20


def test_linear_point_rollout_with_hills_and_terminal_matches_oracle(emu):
    nav = eng.LinearPoint.toy2d_nav()
    onav = orc.LinearPointModel(B=nav.B, goal=nav.goal, R=nav.R, hills=nav.hills, terminal_scale=10.0)
    g = torch.Generator().manual_seed(1)
    T = 25
    x0 = torch.tensor([-3.0, -2.0], dtype=torch.float64)
    v = torch.randn(T, 2, generator=g, dtype=torch.float64)
    s = x0.view(1, 2)
    cost = torch.zeros(1, dtype=torch.float64)
    sts = []
    for t in range(T):
        u = 1.3 * v[t].view(1, 2)
        s = onav.dynamics(s, u)
        cost = cost + onav.running_cost(s, u)
        sts.append(s[0].clone())
    cost = cost + onav.terminal_cost(torch.stack(sts).view(1, 1, T, 2), None).view(1)
    got, c = _rollout(emu, 2, 1, nav.param_blob(), [], T, x0.tolist(), v.reshape(-1).tolist(), 1.3, 2)
    np.testing.assert_allclose(got, torch.stack(sts).numpy(), atol=1e-13)
    assert abs(c - cost.item()) < 1e-10


def test_mlp_rollout_matches_torch_module(emu):
    torch.manual_seed(25)
    net = torch.nn.Sequential(torch.nn.Linear(3, 32), torch.nn.Tanh(), torch.nn.Linear(32, 32), torch.nn.Tanh(),
                              torch.nn.Linear(32, 2)).double()
    m = eng.PendulumMLP(net)
    T = 20
    g = torch.Generator().manual_seed(2)
    x0 = torch.tensor([2.5, -0.7], dtype=torch.float64)
    v = torch.randn(T, 1, generator=g, dtype=torch.float64) * 2
    s = x0.view(1, 2)
    cost = 0.0
    sts = []
    for t in range(T):
        s = m.dynamics(s, v[t].view(1, 1))
        cost += m.running_cost(s, None).item()
        sts.append(s[0].clone())
    got, c = _rollout(emu, 3, 1, m.param_blob(), m.param_blob_ext(), T, x0.tolist(), v.reshape(-1).tolist(), 1.0, 2)
    np.testing.assert_allclose(got, torch.stack(sts).numpy(), atol=1e-12)
    assert abs(c - cost) < 1e-10


def test_colour_and_action_cost_match_oracle(emu):
    g = torch.Generator().manual_seed(3)
    for diag, abs_cost in ((True, False), (False, False), (False, True), (True, True)):
        sigma = torch.tensor([[0.9, 0.0], [0.0, 1.7]], dtype=torch.float64) if diag else torch.tensor([[1.0, 0.3], [0.3, 0.5]], dtype=torch.float64)
        prob = orc.Problem(lambda s, a: s, lambda s, a: s[:, 0], 2, sigma, K=1, T=1, lambda_=0.7,
                           noise_mu=torch.tensor([0.1, -0.2], dtype=torch.float64), noise_abs_cost=abs_cost)
        z = torch.randn(1, 1, 2, generator=g, dtype=torch.float64)
        eps = torch.randn(1, 1, 2, generator=g, dtype=torch.float64)
        U = torch.randn(1, 2, generator=g, dtype=torch.float64)
        want_raw = prob.colour(z)[0, 0]
        want_ac = torch.sum(U * prob.action_cost(eps), dim=(1, 2)).item()
        L = torch.zeros(4, 4, dtype=torch.float64)
        Si = torch.zeros(4, 4, dtype=torch.float64)
        L[:2, :2] = torch.diag(prob.sigma_sqrt_diag) if diag else prob.sigma_chol
        Si[:2, :2] = prob.sigma_inv
        mu_a, mu_p = _arr([0.1, -0.2, 0, 0])
        L_a, L_p = _arr(L.reshape(-1).tolist())
        S_a, S_p = _arr(Si.reshape(-1).tolist())
        z_a, z_p = _arr(z.reshape(-1).tolist() + [0, 0])
        e_a, e_p = _arr(eps.reshape(-1).tolist() + [0, 0])
        U_a, U_p = _arr(U.reshape(-1).tolist() + [0, 0])
        raw = np.zeros(4)
        ac = emu.emu_colour_and_action_cost(2, int(diag), int(abs_cost), C.c_double(0.7), mu_p, L_p, S_p, z_p, e_p, U_p,
                                            raw.ctypes.data_as(C.c_void_p))
        np.testing.assert_allclose(raw[:2], want_raw.numpy(), atol=1e-14)
        assert abs(ac - want_ac) < 1e-13


def test_remainder_is_torch_remainder(emu):
    g = torch.Generator().manual_seed(4)
    a = torch.cat([torch.randn(2000, generator=g, dtype=torch.float64) * 50, torch.tensor([0.0, -0.0, 2 * math.pi, -2 * math.pi, 1e6, -1e6])])
    b = 2 * math.pi
    want = torch.remainder(a, b)
    got = torch.tensor([emu.emu_remainder(float(v), b) for v in a], dtype=torch.float64)
    assert torch.equal(got, want)
    a32 = a.float()
    want32 = torch.remainder(a32, torch.tensor(b, dtype=torch.float32))
    got32 = torch.tensor([emu.emu_remainderf(float(v), float(np.float32(b))) for v in a32], dtype=torch.float32)
    assert torch.equal(got32, want32)
