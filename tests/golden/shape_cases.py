"""Golden cases at the edges of the model envelope: the (nx, nu) = (1,1), (3,3) and (8,4) models of
tests/shape_models.py under MPPI, SMPPI, KMPPI and MPPI_Batched.  Fixtures tests/golden/shape_*.npz, produced by the live
reference (tests/golden/make_golden.py); kept apart from cases.CASES so that the tests parametrised over those do not see
them.  `cases.build_problem` and the base family's engine know the model kind "shape", so the family runs on the base
family's hooks, on both routes at every K.

What the cases reach that no other fixture does: a 4x4 covariance whose off-diagonal entries are all non-zero (the
colouring and the Sigma^-1 action cost with a full Cholesky factor), R = T*nu not a multiple of the normals per Philox
call (13*4, 7*3, 11*3), per-dimension bounds at nu > 2, an 8-component state, and the single-sample and single-step
edges."""
import torch

from tests import shape_models as shm
from tests.golden import cases

SIG3 = [[1.0, 0.3, -0.2], [0.3, 0.8, 0.25], [-0.2, 0.25, 0.9]]
SIG4 = [[1.0, 0.3, -0.2, 0.1], [0.3, 0.8, 0.25, -0.15], [-0.2, 0.25, 0.9, 0.2], [0.1, -0.15, 0.2, 0.7]]


def shape(nx, nu, terminal=True):
    return {"kind": "shape", "nx": nx, "nu": nu, "terminal": terminal}


SHAPE_CASES = {
    "shape_mppi_n8u4_f64": dict(variant="mppi", model=shape(8, 4), dtype="f64", K=333, T=13, lambda_=0.9, noise_sigma=SIG4,
                                noise_mu=[0.05, -0.1, 0.02, 0.08], u_init=[0.1, -0.05, 0.0, 0.2],
                                u_min=[-0.9, -1.3, -0.5, -1.1], u_max=[1.2, 0.7, 0.95, 0.6], u_scale=1.3,
                                sample_null_action=True, u_per_command=2,
                                x0=[0.3, -0.2, 0.5, 0.1, -0.4, 0.25, -0.1, 0.6], steps=3, seed=901),
    "shape_smppi_n3u3_f64": dict(variant="smppi", model=shape(3, 3), dtype="f64", K=256, T=7, lambda_=1.1, noise_sigma=SIG3,
                                 noise_abs_cost=True, x0=[0.5, -0.3, 0.2],
                                 smooth=dict(w=3.0, delta_t=0.4, action_min=[-0.8, -1.2, -0.6], action_max=[0.9, 0.5, 1.1]),
                                 steps=3, seed=902),
    "shape_kmppi_n3u3_f64": dict(variant="kmppi", model=shape(3, 3), dtype="f64", K=300, T=11, lambda_=0.8, noise_sigma=SIG3,
                                 u_max=[1.0, 0.8, 1.2], x0=[-0.4, 0.3, 0.1], kernel=dict(S=4, sigma=1.5), steps=3, seed=903),
    "shape_mppi_n3u3_f32": dict(variant="mppi", model=shape(3, 3), dtype="f32", K=4096, T=15, lambda_=1.0, noise_sigma=SIG3,
                                u_max=[1.0, 0.8, 1.2], x0=[0.6, -0.2, 0.3], steps=3, seed=904),
    "shape_mppi_n1u1_k1_f64": dict(variant="mppi", model=shape(1, 1), dtype="f64", K=1, T=9, lambda_=1.0, noise_sigma=0.8,
                                   u_max=1.5, x0=[0.7], steps=3, seed=905),
    "shape_mppi_n1u1_t1_f64": dict(variant="mppi", model=shape(1, 1), dtype="f64", K=64, T=1, lambda_=0.7, noise_sigma=0.6,
                                   u_min=-1.0, u_max=1.4, x0=[-0.5], steps=3, seed=906),
}
SHAPE_BATCHED_CASES = {
    "shape_batched_n3u3_f64": dict(model=shape(3, 3, terminal=False), dtype="f64", N=3, K=200, T=8, lambda_=0.9,
                                   noise_sigma=SIG3, u_max=[1.0, 0.8, 1.2], u_scale=1.1,
                                   x0=[[0.5, -0.3, 0.2], [-0.6, 0.1, 0.4], [0.0, 0.7, -0.5]], steps=3, seed=908),
}


class ShapeTwin:
    """The oracle's model object of a "shape" case: the torch twins of tests/shape_models.py."""

    def __init__(self, m):
        self.nx, self.nu = m["nx"], m["nu"]
        self.has_terminal = m["terminal"]
        f, c, t = shm.twins(self.nx, self.nu)
        self.dynamics, self.running_cost = f, c
        self.terminal_cost = t if self.has_terminal else None


def sigma_is_full(case):
    s = torch.tensor(case["noise_sigma"])
    return s.dim() == 2 and bool((s - torch.diag(torch.diag(s)) != 0).sum() == s.numel() - s.shape[0])


# shape_mppi_n3u3_f32: the reference colours (z @ L^T) and weighs the noise (noise @ Sigma^-1) with fp32 matrix products,
# the kernels with individually rounded products and sums over the 3 components: costs (down to 3.6e-3) differ by up to
# 1.9e-5 absolute, on both routes (measured on H100; restating the kernels' order on the CPU gives the same 1.9e-5)
COST_ATOL = {"shape_mppi_n3u3_f32": 3.8e-5}


def _check_costs(name, case, route, got, want, tol):
    cases.base_check_costs(name, case, route, got, want, tol, atol=COST_ATOL.get(name))


SHAPES = cases.Family("shapes", dict(SHAPE_CASES, **SHAPE_BATCHED_CASES), cases.BASE.model, cases.BASE.reference,
                      engine=cases.BASE.engine, routes=lambda name, case: ["fused", "stepped"], u_tol=cases.BASE.u_tol,
                      check_costs=_check_costs, reset_nominal=lambda route: True, lockable=cases.base_lockable)
