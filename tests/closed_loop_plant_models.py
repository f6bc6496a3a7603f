"""Plants named apart from the controller's model (`run_closed_loop(plant=...)`), for tests/test_gpu_closed_loop_plant.py;
their cubins are compiled by `__graft_entry__.build()`, so the GPU tests load them without compiling.

* The true pendulum of the reference's learned-dynamics example (tests/pendulum_approximate.py, `true_dynamics`): the
  velocity is integrated, the angle advanced with the unclipped velocity, and only then the velocity clipped; gravity
  enters as -3g/(2l) sin(theta + pi).  p = [-3g/(2l), 3/(m l^2), dt, max_torque, max_speed, w_thdot].
* The costmap point of tests/closed_loop_models.py with other parameters, as the plant of an SMPPI controller on
  `LinearPoint` (compiled for the SMPPI variant, whose module the plant step is taken from).
"""
import math

import torch

import pytorch_mppi_b200 as eng
from tests import closed_loop_models as clm

TRUE_PARAMS = [-3 * 10.0 / (2 * 1.0), 3.0 / (1.0 * 1.0 ** 2), 0.05, 2.0, 8.0, 0.1]
TRUE_STEP = """
    const real pi = (real)3.141592653589793;
    real uc = clamp<real>(u[0], -p[3], p[3]);
    real acc = O::add(O::mul(p[0], O::sin_(O::add(x[0], pi))), O::mul(p[1], uc));
    real thd = O::add(x[1], O::mul(acc, p[2]));
    x[0] = O::add(x[0], O::mul(thd, p[2]));
    x[1] = clamp<real>(thd, -p[4], p[4]);
"""
TRUE_COST = """
    const real pi = (real)3.141592653589793, two_pi = (real)(2 * 3.141592653589793);
    real an = O::sub(remainder<real>(O::add(x[0], pi), two_pi), pi);
    return O::add(O::mul(an, an), O::mul(p[5], O::mul(x[1], x[1])));
"""


def true_dynamics(state, action, p=TRUE_PARAMS):
    """The torch twin (pendulum_approximate.py `true_dynamics`)."""
    th, thdot = state[:, 0:1], state[:, 1:2]
    u = torch.clamp(action[:, 0:1], -p[3], p[3])
    newthdot = thdot + (p[0] * torch.sin(th + math.pi) + p[1] * u) * p[2]
    newth = th + newthdot * p[2]
    return torch.cat((newth, torch.clamp(newthdot, -p[4], p[4])), dim=1)


def true_cost(state, action, p=TRUE_PARAMS):
    return eng.Pendulum.angle_normalize(state[:, 0]) ** 2 + p[5] * state[:, 1] ** 2


def true_pendulum(params=TRUE_PARAMS):
    return eng.CudaModel(2, 1, TRUE_STEP, TRUE_COST, params=params, dynamics=lambda s, a: true_dynamics(s, a, params),
                         running_cost=lambda s, a: true_cost(s, a, params))


COSTMAP_PLANT_PARAMS = [0.05, -2.0, 16.0, 0.5, -0.5]


def costmap_plant(costmap):
    return clm.costmap_model(costmap, params=COSTMAP_PLANT_PARAMS)


def prebuilt():
    """(model, dtype, variant) of every plant the GPU tests load."""
    meta = torch.empty(clm.COSTMAP_HW, device="meta")
    return [(true_pendulum(), torch.float64, 0), (true_pendulum(), torch.float32, 0), (costmap_plant(meta), torch.float32, 1)]
