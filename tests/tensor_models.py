"""User-written CUDA models that read device tensors (CudaModel(tensors=...)), used by the tests and by
scripts/time_model_tensors.py; their cubins are compiled by `__graft_entry__.build()` (from meta tensors that stand in for
the real ones), so the GPU tests load them without compiling.

2-D navigation: x' = x + dt u.  The running cost at horizon step t is
    w_map * bilinear(costmap, (x - origin) / resolution) + w_path * |x - path[t]|^2 + w_u * |u|^2
The costmap is indexed costmap(row = y cell, column = x cell) through the clamped accessor (border replication outside
the map), interpolated with floor and individually rounded ops; the reference path has one row per horizon step (rows
past its end repeat the last one, by the same clamping).  With copies=M the map is (M, H, W) and copy m reads map m.

The torch twins do the same individually rounded ops in the same order, so the fused kernel's per-sample costs match
them and the oracle bit for bit; they read the model's current tensors (`model.tensors`), so they follow in-place edits
and `set_tensors` as the kernels do.  With copies=M they are called with M*K rows, copy-major, and have to know K."""
import numpy as np
import torch

import pytorch_mppi_b200 as eng

# dt, origin x, origin y, 1 / resolution, w_map, w_path, w_u
NAV_PARAMS = [0.1, -2.0, -2.0, 16.0, 5.0, 0.5, 0.01]
MAP_HW = (64, 64)          # 4 x 4 world units at 16 cells per unit

NAV_STEP = """
    x[0] = O::add(x[0], O::mul(p[0], u[0]));
    x[1] = O::add(x[1], O::mul(p[0], u[1]));
"""


def nav_cost_code(per_copy=False):
    """The cost body; `per_copy`: the costmap is (M, H, W) and copy m reads map m."""
    mi = "m, " if per_copy else ""
    return f"""
    const real gx = O::mul(O::sub(x[0], p[1]), p[3]);
    const real gy = O::mul(O::sub(x[1], p[2]), p[3]);
    const real fx = floor(gx), fy = floor(gy);
    const int i = (int)fx, j = (int)fy;
    const real ax = O::sub(gx, fx), ay = O::sub(gy, fy);
    const real c00 = (real)costmap({mi}j, i), c01 = (real)costmap({mi}j, i + 1);
    const real c10 = (real)costmap({mi}j + 1, i), c11 = (real)costmap({mi}j + 1, i + 1);
    const real top = O::add(c00, O::mul(ax, O::sub(c01, c00)));
    const real bot = O::add(c10, O::mul(ax, O::sub(c11, c10)));
    const real val = O::add(top, O::mul(ay, O::sub(bot, top)));
    const real dx = O::sub(x[0], (real)path(t, 0)), dy = O::sub(x[1], (real)path(t, 1));
    const real c = O::add(O::mul(p[4], val), O::mul(p[5], O::add(O::mul(dx, dx), O::mul(dy, dy))));
    return O::add(c, O::mul(p[6], O::add(O::mul(u[0], u[0]), O::mul(u[1], u[1]))));
"""


def _scalars(p, like):
    """The parameters rounded to `like`'s dtype, as the kernel holds them (P<real>)."""
    r = np.float32 if like.dtype == torch.float32 else np.float64
    return [float(r(v)) for v in p]


def nav_dyn(s, a, t, p):
    P = _scalars(p, s)
    return torch.stack((s[:, 0] + P[0] * a[:, 0], s[:, 1] + P[0] * a[:, 1]), dim=1)


def bilinear(costmap, s, p, copy=None):
    """The map term of the cost at the rows of s: costmap (H, W), or (M, H, W) with `copy` the map index of each row."""
    P = _scalars(p, s)
    gx, gy = (s[:, 0] - P[1]) * P[3], (s[:, 1] - P[2]) * P[3]
    fx, fy = torch.floor(gx), torch.floor(gy)
    i, j = fx.long(), fy.long()
    ax, ay = gx - fx, gy - fy
    cm = costmap.to(s.device)
    H, W = cm.shape[-2], cm.shape[-1]

    def at(jj, ii):
        jj, ii = jj.clamp(0, H - 1), ii.clamp(0, W - 1)
        v = cm[jj, ii] if copy is None else cm[copy, jj, ii]
        return v.to(s.dtype)

    c00, c01, c10, c11 = at(j, i), at(j, i + 1), at(j + 1, i), at(j + 1, i + 1)
    top = c00 + ax * (c01 - c00)
    bot = c10 + ax * (c11 - c10)
    return top + ay * (bot - top)


def nav_cost(s, a, t, p, costmap, path, copy=None):
    P = _scalars(p, s)
    val = bilinear(costmap, s, p, copy)
    row = path.to(s.device)[min(t, path.shape[0] - 1)].to(s.dtype)
    dx, dy = s[:, 0] - float(row[0]), s[:, 1] - float(row[1])
    c = P[4] * val + P[5] * (dx * dx + dy * dy)
    return c + P[6] * (a[:, 0] * a[:, 0] + a[:, 1] * a[:, 1])


def make_costmap(dtype=torch.float32, hw=MAP_HW, device="cuda", seed=0):
    """A smooth random field with obstacles: values in [0, 1] for floats, [0, 250] for integer maps."""
    g = torch.Generator().manual_seed(seed)
    H, W = hw
    base = torch.nn.functional.interpolate(torch.rand(1, 1, H // 8, W // 8, generator=g), size=(H, W), mode="bilinear",
                                           align_corners=False)[0, 0]
    if dtype in (torch.uint8, torch.int32):
        base = (base * 250).round()
    return base.to(dtype).to(device).contiguous()


def make_path(T, dtype=torch.float64, device="cuda"):
    """A (T, 2) reference path: a quarter circle from (-1, -1) towards (1, 1)."""
    s = torch.linspace(0.0, 1.0, T, dtype=torch.float64)
    path = torch.stack((-1.0 + 2.0 * torch.sin(s * np.pi / 2), 1.0 - 2.0 * torch.cos(s * np.pi / 2)), dim=1)
    return path.to(dtype).to(device).contiguous()


def nav_model(costmap, path, params=NAV_PARAMS):
    """The navigation model on these tensors.  The twins read `m.tensors` and `m.params`."""
    m = eng.CudaModel(2, 2, NAV_STEP, nav_cost_code(), params=params, step_dependent=True,
                      tensors={"costmap": costmap, "path": path},
                      dynamics=lambda s, a, t: nav_dyn(s, a, t, m.params),
                      running_cost=lambda s, a, t: nav_cost(s, a, t, m.params, m.tensors["costmap"], m.tensors["path"]))
    return m


def nav_ensemble(costmaps, path, K, params=NAV_PARAMS):
    """copies=M: copy m reads costmaps[m] of an (M, H, W) map.  The twins take M*K rows, copy-major."""
    M = costmaps.shape[0]

    def cost(s, a, t):
        copy = torch.div(torch.arange(s.shape[0], device=s.device), K, rounding_mode="floor")
        return nav_cost(s, a, t, m.params, m.tensors["costmap"], m.tensors["path"], copy)

    m = eng.CudaModel(2, 2, NAV_STEP, nav_cost_code(per_copy=True), params=params, step_dependent=True, copies=M,
                      tensors={"costmap": costmaps, "path": path},
                      dynamics=lambda s, a, t: nav_dyn(s, a, t, m.params), running_cost=cost)
    return m


def meta_model(map_dtype=torch.float32, path_dtype=torch.float64, copies=1):
    """The model of these tensor dtypes with meta tensors in place of device ones: what build() compiles."""
    path = torch.empty(1, 2, dtype=path_dtype, device="meta")
    if copies > 1:
        return nav_ensemble(torch.empty(copies, 1, 1, dtype=map_dtype, device="meta"), path, K=1)
    return nav_model(torch.empty(1, 1, dtype=map_dtype, device="meta"), path)


ENSEMBLE_M = 3


def prebuilt():
    """(model, dtype, variant) of every tensor model the GPU tests and scripts/time_model_tensors.py run."""
    out = [(meta_model(), dt, v) for dt in (torch.float32, torch.float64) for v in (0, 1, 2)]
    out += [(meta_model(md), torch.float64, 0) for md in (torch.uint8, torch.int32)]
    out += [(meta_model(copies=ENSEMBLE_M), torch.float64, 0)]
    return out
