"""User-written CUDA models the closed-loop tests and scripts/time_closed_loop.py run; their cubins are compiled by
`__graft_entry__.build()`, so the GPU tests load them without compiling.

* A 2-D point with velocity inputs whose running cost reads a costmap tensor (nearest cell, clamped at the border) plus
  the squared distance to a goal: p = [dt, origin, cells per unit, goal x, goal y].
* The three-copy pendulum ensemble of tests/ensemble_models.py (copy m: its own mass and length), whose plant is copy 0.
"""
import torch

import pytorch_mppi_b200 as eng
from tests import ensemble_models

COSTMAP_PARAMS = [0.1, -2.0, 16.0, 1.5, 1.0]
COSTMAP_HW = (64, 64)
COSTMAP_STEP = "x[0] = O::add(x[0], O::mul(p[0], u[0])); x[1] = O::add(x[1], O::mul(p[0], u[1]));"
COSTMAP_COST = """
    const int i = (int)O::mul(O::sub(x[1], p[1]), p[2]), j = (int)O::mul(O::sub(x[0], p[1]), p[2]);
    const real dx = O::sub(x[0], p[3]), dy = O::sub(x[1], p[4]);
    return O::add(O::add(O::mul(dx, dx), O::mul(dy, dy)), (real)costmap(i, j));
"""


def make_costmap(device="cuda", seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(COSTMAP_HW, generator=g) * 4.0).to(device)


def costmap_model(costmap, params=COSTMAP_PARAMS):
    return eng.CudaModel(2, 2, COSTMAP_STEP, COSTMAP_COST, params=params, tensors={"costmap": costmap})


ENSEMBLE_M = 3


def pendulum_ensemble(K):
    return ensemble_models.pendulum_ensemble(ENSEMBLE_M, K)


def prebuilt():
    """(model, dtype, variant) of every closed-loop kernel the GPU tests load."""
    meta = torch.empty(COSTMAP_HW, device="meta")
    return [(costmap_model(meta), torch.float32, 0), (pendulum_ensemble(1), torch.float64, 0)]
