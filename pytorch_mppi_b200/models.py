"""Registry of analytic models whose dynamics + running cost are compiled into the fused kernel.

The reference's plugin surface is a pair of Python callables ``dynamics(state, action)`` /
``running_cost(state, action)`` (mppi.py:63-64, README.md:53-58).  Arbitrary callables cannot be
inlined into CUDA, so the fused path recognises callables that are *bound methods of a registered
model object*: pass ``model.dynamics`` / ``model.running_cost`` (and optionally
``model.terminal_cost``) to the controller exactly as you would pass your own functions, and the
controller launches the fused sm_90a kernel.  The same bound methods are ordinary torch functions
(any device, any dtype), so they also serve as the simulator you step your real system with and as
the callables of the per-step path.

Anything else (a torch MLP, a lambda, a plain step-dependent function) takes the per-step path:
the T-loop stays in Python with sampling / accumulation / softmin in CUDA kernels.  A `CudaModel` declared
``step_dependent=True`` is the compiled form of a step-dependent pair (``step_dependent_dynamics=True``).
"""
from __future__ import annotations

import math
from typing import Optional, Sequence

import torch

from . import _cabi


class AnalyticModel:
    """Base class: a model known to the CUDA registry (include/mppi_b200.h `MppiModel`)."""
    model_id: int = 0
    nx: int = 0
    nu: int = 0
    step_dependent: bool = False     # dynamics / running_cost take the horizon index t (CudaModel(step_dependent=True))
    copies: int = 1                  # compiled rollout copies per sample (CudaModel(copies=M)): runs with rollout_samples=M
    _param_version: int = 0          # bumped by CudaModel.set_params; controllers compare it at command time

    def param_blob(self) -> list:
        """The `model_params` doubles of MppiFusedParams for this instance."""
        raise NotImplementedError

    def param_blob_ext(self) -> list:
        """Extra parameters too large for `model_params` (e.g. network weights); [] if none."""
        return []

    @property
    def has_terminal(self) -> bool:
        return False

    # -- recognition of bound methods --------------------------------------------------------
    @staticmethod
    def owner_of(fn) -> Optional["AnalyticModel"]:
        owner = getattr(fn, "__self__", None)
        return owner if isinstance(owner, AnalyticModel) else None


class Pendulum(AnalyticModel):
    """Gym pendulum swing-up, the model of BASELINE configs 1/2/5
    (reference tests/pendulum.py:30-60): state (theta, theta_dot), one torque input.

        u      <- clamp(u, +-max_torque)
        thdot' =  clip(thdot + (3g/(2l) sin(theta) + 3/(m l^2) u) dt, +-max_speed)
        theta' =  theta + thdot' dt
        cost   =  angle_normalize(theta')^2 + w_thdot thdot'^2
    """
    model_id = _cabi.MODEL_PENDULUM
    nx, nu = 2, 1

    def __init__(self, g=10.0, m=1.0, l=1.0, dt=0.05, max_torque=2.0, max_speed=8.0, w_thdot=0.1):
        self.g, self.m, self.l, self.dt = float(g), float(m), float(l), float(dt)
        self.max_torque, self.max_speed, self.w_thdot = float(max_torque), float(max_speed), float(w_thdot)

    def param_blob(self):
        return [self.g, self.m, self.l, self.dt, self.max_torque, self.max_speed, self.w_thdot]

    def dynamics(self, state, action):
        th = state[:, 0:1]
        thdot = state[:, 1:2]
        u = torch.clamp(action[:, 0:1], -self.max_torque, self.max_torque)
        acc = (3 * self.g / (2 * self.l)) * torch.sin(th) + (3.0 / (self.m * self.l ** 2)) * u
        new_thdot = torch.clamp(thdot + acc * self.dt, -self.max_speed, self.max_speed)
        new_th = th + new_thdot * self.dt
        return torch.cat((new_th, new_thdot), dim=1)

    @staticmethod
    def angle_normalize(x):
        return ((x + math.pi) % (2 * math.pi)) - math.pi

    def running_cost(self, state, action):
        return self.angle_normalize(state[:, 0]) ** 2 + self.w_thdot * state[:, 1] ** 2


class LinearPoint(AnalyticModel):
    """2-D point mass with linear-delta dynamics ``x + u @ B.T``, a quadratic goal cost
    ``(g-x)^T Q (g-x)``, optional action cost ``u^T R u``, up to three Gaussian hill costs
    ``h exp(-(c-x)^T Q_h (c-x))`` and an optional terminal cost ``terminal_scale * state_cost(x_T)``.

    `LinearPoint.unit_test_env()` is the fixture of the reference's test-suite
    (reference tests/test_mppi.py:24-51); `LinearPoint.toy2d_nav()` is the Toy2D navigation
    environment of reference tests/smooth_mppi.py:79-142 (BASELINE config 3).
    """
    model_id = _cabi.MODEL_LINEAR_POINT
    nx, nu = 2, 2
    MAX_HILLS = 3

    def __init__(self, B, goal, Q=None, R=None, hills: Sequence = (), terminal_scale: float = 0.0):
        self.B = [[float(v) for v in row] for row in B]
        self.goal = [float(v) for v in goal]
        self.Q = [[1.0, 0.0], [0.0, 1.0]] if Q is None else [[float(v) for v in row] for row in Q]
        self.R = None if R is None else [[float(v) for v in row] for row in R]
        self.hills = [([[float(v) for v in row] for row in q], [float(v) for v in c], float(h)) for q, c, h in hills]
        if len(self.hills) > self.MAX_HILLS:
            raise ValueError(f"at most {self.MAX_HILLS} hills are compiled into the fused kernel")
        self.terminal_scale = float(terminal_scale)
        self._cache = {}

    @classmethod
    def unit_test_env(cls, terminal_scale=0.0):
        return cls(B=[[1.0, 0.0], [0.0, -1.0]], goal=[2.0, 2.0], terminal_scale=terminal_scale)

    @classmethod
    def toy2d_nav(cls, terminal_scale=10.0, r=0.01):
        return cls(B=[[0.5, 0.0], [0.0, -0.5]], goal=[2.0, 2.0], R=[[r, 0.0], [0.0, r]],
                   hills=[([[0.25, 0.125], [0.125, 0.25]], [-0.5, -1.0], 200.0)], terminal_scale=terminal_scale)

    @property
    def has_terminal(self):
        return self.terminal_scale != 0.0

    def param_blob(self):
        flat = lambda m: [m[0][0], m[0][1], m[1][0], m[1][1]]
        b = flat(self.B) + self.goal + flat(self.Q)
        b += [1.0 if self.R is not None else 0.0] + (flat(self.R) if self.R is not None else [0.0] * 4)
        b += [self.terminal_scale, float(len(self.hills))]
        for q, c, h in self.hills:
            b += flat(q) + c + [h]
        b += [0.0] * (7 * (self.MAX_HILLS - len(self.hills)))
        return b

    # ---- torch implementations (any device/dtype) ---------------------------------------------
    def _t(self, name, like):
        key = (name, like.device, like.dtype)
        if key not in self._cache:
            src = {"B": self.B, "goal": self.goal, "Q": self.Q, "R": self.R}.get(name)
            if src is None and name.startswith("hq"):
                src = self.hills[int(name[2:])][0]
            if src is None and name.startswith("hc"):
                src = self.hills[int(name[2:])][1]
            self._cache[key] = torch.tensor(src, device=like.device, dtype=like.dtype)
        return self._cache[key]

    @staticmethod
    def _quad(d, Q):
        return (d * (d @ Q.transpose(0, 1))).sum(dim=-1)

    def dynamics(self, state, action):
        return state + action @ self._t("B", state).transpose(0, 1)

    def state_cost(self, state):
        c = self._quad(self._t("goal", state) - state, self._t("Q", state))
        for i, (_, _, h) in enumerate(self.hills):
            c = c + h * torch.exp(-self._quad(self._t(f"hc{i}", state) - state, self._t(f"hq{i}", state)))
        return c

    def running_cost(self, state, action):
        c = self.state_cost(state)
        if self.R is not None:
            c = c + self._quad(action, self._t("R", state))
        return c

    def terminal_cost(self, states, actions):
        return self.terminal_scale * self.state_cost(states[..., -1, :])


class PendulumMLP(AnalyticModel):
    """Learned pendulum dynamics of BASELINE config 4 (reference tests/pendulum_approximate.py:47-67):
    ``x' = x + net([x, clamp(u)])`` with ``net = Linear(3,32)-Tanh-Linear(32,32)-Tanh-Linear(32,2)``, then the
    angle is wrapped to [-pi, pi); running cost as the analytic pendulum.

    Pass ``model.dynamics`` / ``model.running_cost`` to the controller: the fused kernel then evaluates the
    network inside the rollout (weights in the kernel's constant parameter block).  The torch callables
    below evaluate the same ``net`` module, so they are the stepped-route / simulator definition too.
    Call ``refresh()`` after retraining ``net`` (the controller re-reads the weights when repacked).
    """
    model_id = _cabi.MODEL_PENDULUM_MLP
    nx, nu = 2, 1
    H = 32

    def __init__(self, net: torch.nn.Sequential, max_torque=2.0, w_thdot=0.1, fast_tanh=False, tensor_cores="auto"):
        self.check_net(net)
        self.net = net
        self.max_torque, self.w_thdot, self.fast_tanh = float(max_torque), float(w_thdot), bool(fast_tanh)
        self.tensor_cores = self.tensor_core_mode(tensor_cores)

    @classmethod
    def check_net(cls, net):
        """Raise ValueError unless `net` is the network the kernels compile: Linear(3,32)-Tanh-Linear(32,32)-Tanh-Linear(32,2)."""
        lin = [m for m in net if isinstance(m, torch.nn.Linear)]
        act = [m for m in net if not isinstance(m, torch.nn.Linear)]
        shapes = [tuple(l.weight.shape) for l in lin]
        if shapes != [(cls.H, 3), (cls.H, cls.H), (2, cls.H)] or not all(isinstance(a, torch.nn.Tanh) for a in act):
            raise ValueError("PendulumMLP expects Linear(3,32)-Tanh-Linear(32,32)-Tanh-Linear(32,2); got " + str(shapes))

    @staticmethod
    def tensor_core_mode(tensor_cores):
        """model_params[3] of a `tensor_cores` argument.
        tensor_cores (fp32 controllers only): the hidden and output layers run as wgmma MMAs with fp32 accumulators
        (csrc/mppi_mlp_tc.cuh); layer 1 runs in exact fp32 in both modes, so the states and the action never pass
        through bf16.  True / "bf16x3": layers 2 and 3 take hi/lo-split bf16 operands; on an H100 one step's cost stays
        within 0.37 of the error bound of tests/mlp_bounds.py, whose median is 9e-5 of the cost on the default network.
        "bf16": plain bf16 operands for layers 2 and 3 (~2^-8 relative per product), the fastest route; its one-step
        costs leave the bf16x3 bound on 87 % of the probe samples, by up to 21 times.
        "auto" (default): "bf16x3" wherever the tensor-core kernel exists (fp32 controllers, one environment), the FFMA
        kernel elsewhere (fp64, MPPI_Batched); False pins the FFMA kernel."""
        if not any(tensor_cores is v or tensor_cores == v for v in (False, True, None, "auto", "bf16x3", "bf16")):
            raise ValueError("tensor_cores must be 'auto', False, True, 'bf16x3' or 'bf16'")
        if tensor_cores is True:
            tensor_cores = "bf16x3"
        return {False: 0, None: 0, "bf16x3": 1, "bf16": 2, "auto": 3}[tensor_cores]

    def param_blob(self):
        return [self.max_torque, self.w_thdot, 1.0 if self.fast_tanh else 0.0, float(self.tensor_cores)]

    def param_blob_ext(self):
        out = []
        with torch.no_grad():
            for m in self.net:
                if isinstance(m, torch.nn.Linear):
                    out += m.weight.detach().double().cpu().reshape(-1).tolist()
                    out += m.bias.detach().double().cpu().reshape(-1).tolist()
        return out

    @staticmethod
    def net_step(net, state, action, max_torque):
        """x' = x + net([x, clamp(u)]), angle wrapped (pendulum_approximate.py:60-67)."""
        with torch.no_grad():
            u = torch.clamp(action[:, 0:1], -max_torque, max_torque)
            nxt = state + net(torch.cat((state, u), dim=1))
            th = Pendulum.angle_normalize(nxt[:, 0])
            return torch.stack((th, nxt[:, 1]), dim=1)

    def dynamics(self, state, action):
        return self.net_step(self.net, state, action, self.max_torque)

    def running_cost(self, state, action):
        return Pendulum.angle_normalize(state[:, 0]) ** 2 + self.w_thdot * state[:, 1] ** 2


class PendulumMLPEnsemble(AnalyticModel):
    """A bootstrapped ensemble of learned pendulum dynamics (PETS-style model uncertainty): M = len(nets) networks of
    `PendulumMLP`'s shape (2 <= M <= MPPI_MAX_COPIES), one per rollout copy.  Build the controller with
    ``rollout_samples=M``: every sample's action sequence is rolled out through each network, and its cost is the mean
    over the networks plus ``rollout_var_cost * sum_t rollout_var_discount**t * var_m(c_{m,t})`` (mppi.py:334-373).
    MPPI / SMPPI / KMPPI (also sharded) without a SpecificActionSampler then run the fused kernel; resident mode and
    MPPI_Batched are not available.  `fast_tanh` and `tensor_cores` mean what they mean for `PendulumMLP`.

    The torch callables are called as the reference calls an M-copy rollout: `dynamics` gets M*K rows, copy-major, and
    sends block m of M equal blocks through ``nets[m]`` (a row count that is not a multiple of M raises ValueError);
    `running_cost` is PendulumMLP's; there is no terminal cost.  `get_rollouts` on the fused route runs ``nets[0]``.
    The controller copies the weights to a device table when it packs its constants: call ``refresh()`` on it after
    retraining the networks.
    """
    model_id = _cabi.MODEL_PENDULUM_MLP_ENSEMBLE
    nx, nu = 2, 1

    def __init__(self, nets, max_torque=2.0, w_thdot=0.1, fast_tanh=False, tensor_cores="auto"):
        nets = list(nets)
        if not 2 <= len(nets) <= _cabi.MPPI_MAX_COPIES:
            raise ValueError(f"an ensemble takes 2..{_cabi.MPPI_MAX_COPIES} networks, got {len(nets)}")
        for net in nets:
            PendulumMLP.check_net(net)
        self.nets = nets
        self.copies = len(nets)
        self.max_torque, self.w_thdot, self.fast_tanh = float(max_torque), float(w_thdot), bool(fast_tanh)
        self.tensor_cores = PendulumMLP.tensor_core_mode(tensor_cores)

    param_blob = PendulumMLP.param_blob

    def weight_table(self, device, dtype):
        """(M, 1250) tensor of the networks' weights on `device` in `dtype`, row m in PyTorch Linear order
        (W1, b1, W2, b2, W3, b3): MppiFusedParams.model_weights."""
        with torch.no_grad():
            return torch.stack([torch.cat([p.detach().to(device=device, dtype=dtype).reshape(-1)
                                           for m in net if isinstance(m, torch.nn.Linear) for p in (m.weight, m.bias)])
                                for net in self.nets]).contiguous()

    def dynamics(self, state, action):
        n, M = state.shape[0], self.copies
        if n % M:
            raise ValueError(f"an ensemble of {M} networks steps M*K rows (copy-major); got {n} rows")
        K = n // M
        return torch.cat([PendulumMLP.net_step(net, state[m * K:(m + 1) * K], action[m * K:(m + 1) * K], self.max_torque)
                          for m, net in enumerate(self.nets)])

    running_cost = PendulumMLP.running_cost


class CudaModel(AnalyticModel):
    """A user-written analytic model compiled INTO the fused kernel.

    The reference takes arbitrary Python callables (mppi.py:63-64); those cannot be inlined into CUDA, so for
    analytic dynamics/costs you give the two function bodies as CUDA C++ and the engine compiles the fused / split-cost /
    resident / states kernels for your model at run time with NVRTC (in process, cached on disk: pytorch_mppi_b200.rtc)
    and loads them into the stock library (`mppi_user_model_register`).  Inside the bodies:

        x[NX]      state (read/write in `step_code`, read-only in `cost_code` / `terminal_code`)
        u[NU]      action, already multiplied by u_scale
        p[...]     your `params` (cast to the controller dtype)
        t          step_dependent=True only: the horizon index 0..T-1 of this step (`const int`), in `step_code` and
                   `cost_code` (not in `terminal_code`, as the reference's terminal cost)
        m          copies=M > 1 only: the copy index 0..M-1 (`const int`), in `step_code`, `cost_code` and
                   `terminal_code`; `COPIES` is M
        real       the controller dtype; O::add/sub/mul/div are individually rounded ops (use them if you want
                   bit-level agreement with an eager fp32 torch implementation), sinf/exp/... via O::sin_, O::exp_

    `cost_code` and `terminal_code` must `return` a `real`.  `dynamics` / `running_cost` / `terminal_cost`
    are the torch callables of the same model (used by the stepped route and as your simulator;
    `get_rollouts` runs the compiled `step_code`); pass ``model.dynamics`` / ``model.running_cost`` to the
    controller as usual.

    Step-dependent models (time-varying problems: a moving target, a reference trajectory to track, a forcing
    schedule): with ``step_dependent=True`` the torch callables are called as ``dynamics(state, action, t)`` and
    ``running_cost(state, action, t)``, and the controller must be built with ``step_dependent_dynamics=True``, exactly as
    the reference calls such plugins (mppi.py:147-157).  MPPI / SMPPI / KMPPI / MPPI_Batched with
    ``rollout_samples=1`` and no SpecificActionSampler then run the fused kernel.

    `set_params(values)` replaces the parameter values (same count as at construction).  Every controller using the
    model takes them at its next command, without re-planning; a resident grid leaves and the next `command_host()`
    brings it back.  Intermediates of earlier commands (`states`, `noise`, ...) keep the values they were computed
    with, `get_rollouts` uses the current ones.  Your torch callables see the change only if they read `model.params`.
    A sharded (multi-GPU) controller needs the same values on every rank before the same command.

    Ensembles (robust control under model uncertainty: domain randomisation over masses and lengths, disturbance
    scenarios): with ``copies=M`` (2 <= M <= MPPI_MAX_COPIES) every sample's action sequence is rolled out through M
    copies of the model, and the bodies tell the copies apart by `m` (e.g. ``p[2 + m]`` a per-copy mass, or a scenario
    table ``p[m * T + t]`` with ``step_dependent=True``; long tables go in `params`, past the first
    MPPI_MODEL_PARAM_DOUBLES values).  The controller must be built with ``rollout_samples=M``: the cost of a sample is
    the mean over its copies plus ``rollout_var_cost * sum_t rollout_var_discount**t * var_m(c_{m,t})``, as the
    reference computes it (mppi.py:334-373).  MPPI / SMPPI / KMPPI (also sharded) without a SpecificActionSampler then
    run the fused kernel, which keeps the M states in registers; resident mode and MPPI_Batched are not available.
    The torch callables are called exactly as the reference calls an M-copy rollout: with M*K rows, copy-major, so row r
    belongs to copy ``r // K``.  Your twins therefore have to know K (the controller's num_samples; on a sharded
    controller, its shard's sample count).  `get_rollouts` runs copy 0, which is what such a twin computes for
    ``num_rollouts <= K`` rows.

    Device tensors (costmaps, lookup tables, reference paths: data too large for `params`, or indexed by the state):
    ``tensors={"costmap": cm, "path": path}`` makes each tensor a read-only view with its own name in `step_code`,
    `cost_code` and `terminal_code`.  ``costmap(i, j)`` takes one integer index per dimension and returns the element
    (``float``, ``double``, ``unsigned char`` or ``int`` for float32 / float64 / uint8 / int32 tensors); each index is
    clamped to ``[0, costmap.size(d) - 1]``, so a lookup never leaves the tensor and acts as border replication outside a
    map.  Tensors are contiguous, 1- to 4-dimensional, with at most 2**31 - 1 elements, on the controller's device
    (at most MPPI_MAX_MODEL_TENSORS of them).  Only their names, dtypes and ndims are compiled into the kernels; a meta
    tensor can stand in for one to compile ahead of time without a GPU (swap the real one in with `set_tensors`).
    Contents edited in place on the controller's stream (``cm.copy_(new)``) take effect at the next `command()`, as
    edits of `U` do.  `set_tensors(costmap=other)` swaps a tensor (same dtype and ndim, any shape) for the following
    commands of every controller using the model, without recompiling or re-planning; each controller keeps the tensors
    its plan points at alive.  Resident mode: the grid keeps running between `command_host()` calls, so it would race
    with an in-place edit — while resident, change tensor contents only through `set_tensors`, which makes the grid
    leave (as `set_params` does); the next `command_host()` brings it back.  Your torch callables close over the same
    tensors (read them through `model.tensors` to follow `set_tensors`).
    """
    model_id = _cabi.MODEL_USER

    def __init__(self, nx, nu, step_code, cost_code, params=(), terminal_code=None, dynamics=None, running_cost=None,
                 terminal_cost=None, step_dependent=False, copies=1, tensors=None):
        if not (1 <= nx <= _cabi.MPPI_MAX_NX and 1 <= nu <= _cabi.MPPI_MAX_NU):
            raise ValueError(f"nx <= {_cabi.MPPI_MAX_NX} and nu <= {_cabi.MPPI_MAX_NU} required")
        if isinstance(copies, bool) or not isinstance(copies, int) or not 1 <= copies <= _cabi.MPPI_MAX_COPIES:
            raise ValueError(f"copies must be an integer 1..{_cabi.MPPI_MAX_COPIES}, got {copies!r}")
        self.copies = copies
        self.nx, self.nu = int(nx), int(nu)
        self.params = [float(v) for v in params]
        self.step_dependent = bool(step_dependent)
        self._step_code, self._cost_code, self._terminal_code = step_code, cost_code, terminal_code
        self._dyn, self._cost, self._term = dynamics, running_cost, terminal_cost
        self._rtc_handles = {}
        tensors = dict(tensors or {})
        if len(tensors) > _cabi.MPPI_MAX_MODEL_TENSORS:
            raise ValueError(f"at most {_cabi.MPPI_MAX_MODEL_TENSORS} tensors, got {len(tensors)}")
        for name, t in tensors.items():
            _check_tensor(name, t)
        self.tensors = tensors

    @property
    def has_terminal(self):
        return self._terminal_code is not None

    def param_blob(self):
        return self.params[: _cabi.MPPI_MODEL_PARAM_DOUBLES]

    def param_blob_ext(self):
        return self.params[_cabi.MPPI_MODEL_PARAM_DOUBLES:]

    def set_params(self, values):
        """New values of `params` for the following commands of every controller using this model (see the class
        docstring).  The number of parameters is compiled into the kernels: it must not change."""
        values = [float(v) for v in values]
        if len(values) != len(self.params):
            raise ValueError(f"this model was compiled with {len(self.params)} parameters, got {len(values)}")
        self.params = values
        self._param_version += 1

    def set_tensors(self, **tensors):
        """Replace device tensors by name, for the following commands of every controller using this model (see the
        class docstring).  Each replacement keeps its tensor's dtype and ndim (they are compiled into the kernels); its
        shape may change, without recompiling or re-planning."""
        for name, t in tensors.items():
            if name not in self.tensors:
                raise ValueError(f"this model has no tensor {name!r} (it has {sorted(self.tensors)})")
            _check_tensor(name, t)
            old = self.tensors[name]
            if t.dtype != old.dtype or t.dim() != old.dim():
                raise ValueError(f"tensor {name!r} was compiled as {old.dtype} with {old.dim()} dimension(s); "
                                 f"got {t.dtype} with {t.dim()}")
        self.tensors = dict(self.tensors, **tensors)
        self._param_version += 1

    def tensor_refs(self, device):
        """(MppiTensorRef array, tensors) of MppiFusedParams.model_tensors for a controller on `device`; None if the
        model has no tensors.  The caller keeps both alive while the library may read them."""
        if not self.tensors:
            return None
        ts = list(self.tensors.values())
        arr = (_cabi.MppiTensorRef * len(ts))()
        for r, (name, t) in zip(arr, self.tensors.items()):
            if t.device != torch.device(device):
                raise ValueError(f"tensor {name!r} is on {t.device}, the controller on {device}")
            r.data, r.dtype, r.ndim = t.data_ptr(), _TENSOR_DTYPES[t.dtype][0], t.dim()
            for d in range(t.dim()):
                r.shape[d] = t.shape[d]
        return arr, ts

    def header_text(self):
        n = max(len(self.params), 1)
        term = self._terminal_code if self._terminal_code is not None else "return (real)0;"
        sd = self.step_dependent
        decl = "\n    static const bool STEP_DEPENDENT = true;" if sd else ""
        targ = ", const int t" if sd else ""
        tvoid = " (void)t;" if sd else ""
        cp = self.copies > 1
        decl += f"\n    static const int COPIES = {self.copies};" if cp else ""
        marg = ", const int m" if cp else ""
        mvoid = " (void)m;" if cp else ""
        # device tensors: views behind the parameters (csrc/mppi_model_tensors.h packs them), bound to their names in
        # every body; nothing of this is emitted for a model without tensors, whose header stays what it always was
        views = "".join(f" TensorView<{_TENSOR_DTYPES[t.dtype][1]}, {t.dim()}> t{i};" for i, t in enumerate(self.tensors.values()))
        tbind = "".join(f" const auto& {name} = P_.t{i}; (void){name};" for i, name in enumerate(self.tensors))
        tview = _TENSOR_VIEW if self.tensors else ""
        return f"""// generated by pytorch_mppi_b200.models.CudaModel
namespace mppi {{{tview}
struct UserModel {{
    static const int NX = {self.nx}, NU = {self.nu}, NP = {n};{decl}
    template <typename real> struct P {{ real v[NP];{views} }};
    template <typename real> static void load(P<real>& P_, const double* b, const double* ext = nullptr, int n_ext = 0) {{
        for (int i = 0; i < NP; ++i)
            P_.v[i] = (real)(i < {_cabi.MPPI_MODEL_PARAM_DOUBLES} ? b[i] : (ext != nullptr && i - {_cabi.MPPI_MODEL_PARAM_DOUBLES} < n_ext ? ext[i - {_cabi.MPPI_MODEL_PARAM_DOUBLES}] : 0.0));
    }}
    template <typename real> static MPPI_HD void step(const P<real>& P_, real* x, const real* u{targ}{marg}) {{
        typedef Ops<real> O;
        const real* p = P_.v;
        (void)p;{tvoid}{mvoid}{tbind}
        {self._step_code}
    }}
    template <typename real> static MPPI_HD real cost(const P<real>& P_, const real* x, const real* u{targ}{marg}) {{
        typedef Ops<real> O;
        const real* p = P_.v;
        (void)p; (void)u;{tvoid}{mvoid}{tbind}
        {self._cost_code}
    }}
    template <typename real> static MPPI_HD bool has_terminal(const P<real>&) {{ return {"true" if self.has_terminal else "false"}; }}
    template <typename real> static MPPI_HD real terminal(const P<real>& P_, const real* x{marg}) {{
        typedef Ops<real> O;
        const real* p = P_.v;
        (void)p; (void)x;{mvoid}{tbind}
        {term}
    }}
}};
}}  // namespace mppi
"""

    def compile_rtc(self, dtype, variant):
        """(cubin bytes, lowered kernel names) of this model's kernels for one dtype and controller variant
        (0 MPPI / 1 SMPPI / 2 KMPPI): NVRTC, cached on disk.  Needs no GPU."""
        from . import rtc
        return rtc.compile_user_model(self.header_text(), "float" if dtype == torch.float32 else "double", int(variant),
                                      self.copies, plant=not self.step_dependent)

    def rtc_handle(self, lib, dtype, variant):
        """The handle `MppiFusedParams.user_model` takes: the compiled kernels registered with the C library on the
        CURRENT CUDA device (once per (library, dtype, variant, device))."""
        import ctypes as C
        key = (id(lib), dtype, int(variant), torch.cuda.current_device())
        if key not in self._rtc_handles:
            cubin, names = self.compile_rtc(dtype, variant)
            arr = (C.c_char_p * len(names))(*[None if n is None else n.encode() for n in names])
            handle = C.c_void_p()
            buf = C.create_string_buffer(cubin, len(cubin))
            rc = lib.mppi_user_model_register(buf, len(cubin), self.nx, self.nu, max(len(self.params), 1),
                                              _cabi.F32 if dtype == torch.float32 else _cabi.F64, int(variant), arr, C.byref(handle))
            _cabi.check(rc, "mppi_user_model_register")
            if self.copies > 1:
                _cabi.check(lib.mppi_user_model_set_copies(handle, self.copies), "mppi_user_model_set_copies")
            if self.tensors:
                n = len(self.tensors)
                dtypes = (C.c_int32 * n)(*[_TENSOR_DTYPES[t.dtype][0] for t in self.tensors.values()])
                ndims = (C.c_int32 * n)(*[t.dim() for t in self.tensors.values()])
                _cabi.check(lib.mppi_user_model_set_tensors(handle, n, dtypes, ndims), "mppi_user_model_set_tensors")
            self._rtc_handles[key] = handle
        return self._rtc_handles[key]

    def _with_t(self, fn, what, args, t):
        if fn is None:
            raise NotImplementedError(f"this CudaModel was created without a torch `{what}` callable")
        if not self.step_dependent:
            return fn(*args)
        if t is None:
            raise TypeError(f"this CudaModel is step-dependent: call {what}(state, action, t)")
        return fn(*args, t)

    def dynamics(self, state, action, t=None):
        return self._with_t(self._dyn, "dynamics", (state, action), t)

    def running_cost(self, state, action, t=None):
        return self._with_t(self._cost, "running_cost", (state, action), t)

    def terminal_cost(self, states, actions):
        if self._term is None:
            raise NotImplementedError("this CudaModel was created without a torch `terminal_cost` callable")
        return self._term(states, actions)


# element types a model tensor may have: torch dtype -> (MppiDType, C++ element type in the bodies)
_TENSOR_DTYPES = {torch.float32: (_cabi.F32, "float"), torch.float64: (_cabi.F64, "double"),
                  torch.uint8: (_cabi.U8, "unsigned char"), torch.int32: (_cabi.I32, "int")}
# names a tensor cannot take: what the generated struct and bodies already use, and C++ keywords
_RESERVED = set("x u p t m real O P_ NX NU NP COPIES STEP_DEPENDENT".split()) | set("""
    alignas alignof and and_eq asm auto bitand bitor bool break case catch char char16_t char32_t char8_t class compl
    concept const consteval constexpr constinit const_cast continue co_await co_return co_yield decltype default delete
    do double dynamic_cast else enum explicit export extern false float for friend goto if inline int long mutable
    namespace new noexcept not not_eq nullptr operator or or_eq private protected public register reinterpret_cast
    requires return short signed sizeof static static_assert static_cast struct switch template this thread_local
    throw true try typedef typeid typename union unsigned using virtual void volatile wchar_t while xor xor_eq""".split())
_INT31 = 2 ** 31 - 1
# the read-only view a body reads a tensor through: one index per dimension, each clamped to [0, size(d) - 1] (border
# replication outside a map), loads through the read-only data path; no pointer is exposed
_TENSOR_VIEW = """
template <typename T, int N> struct TensorView {
    MPPI_HD int size(int d) const { return shape_[d]; }
    template <typename... I> MPPI_HD T operator()(I... idx) const {
        static_assert(sizeof...(I) == N, "a tensor takes one index per dimension");
        const int ix[N] = {(int)idx...};
        int off = 0;
        for (int d = 0; d < N; ++d) off = off * shape_[d] + (ix[d] < 0 ? 0 : (ix[d] < shape_[d] ? ix[d] : shape_[d] - 1));
#if defined(__CUDA_ARCH__)
        return __ldg(data_ + off);
#else
        return data_[off];
#endif
    }
  private:
    const T* data_;
    int shape_[4];
};"""


def _check_tensor(name, t):
    """ValueError unless `t` can be a model tensor called `name`."""
    if not isinstance(name, str) or not name.isidentifier() or not name.isascii() or name in _RESERVED or name.startswith("__"):
        raise ValueError(f"tensor name {name!r} must be a C identifier that the generated model does not already use")
    if not torch.is_tensor(t):
        raise ValueError(f"tensor {name!r} must be a torch tensor")
    if t.dtype not in _TENSOR_DTYPES:
        raise ValueError(f"tensor {name!r} has dtype {t.dtype}; model tensors are float32, float64, uint8 or int32")
    if not 1 <= t.dim() <= 4:
        raise ValueError(f"tensor {name!r} has {t.dim()} dimensions; model tensors have 1 to 4")
    if not t.is_contiguous():
        raise ValueError(f"tensor {name!r} must be contiguous")
    if t.numel() == 0 or t.numel() > _INT31:
        raise ValueError(f"tensor {name!r} has {t.numel()} elements; model tensors have 1 to 2**31 - 1")
    if t.device.type not in ("cuda", "meta"):
        raise ValueError(f"tensor {name!r} must be a CUDA tensor (or a meta tensor standing in for one), got {t.device}")


def resolve_fused_model(dynamics, running_cost, terminal_state_cost) -> Optional[AnalyticModel]:
    """The registered model these plugins belong to, or None if they are not (all) bound methods of
    one registered model — in which case the controller uses the per-step path."""
    m = AnalyticModel.owner_of(dynamics)
    if m is None or AnalyticModel.owner_of(running_cost) is not m:
        return None
    # the class that REGISTERED the model (declares model_id): a user subclass that overrides dynamics / running_cost /
    # terminal_cost in Python is no longer the compiled model and must take the stepped route
    reg = next((c for c in type(m).__mro__ if "model_id" in c.__dict__ and c is not AnalyticModel), None)
    if reg is None:
        return None
    if getattr(dynamics, "__func__", None) is not reg.__dict__.get("dynamics"):
        return None
    if getattr(running_cost, "__func__", None) is not reg.__dict__.get("running_cost"):
        return None
    if terminal_state_cost is None:
        # the kernel adds the model's terminal cost iff terminal_scale != 0; without the plugin the
        # reference adds none, so only models whose terminal term is off qualify
        return m if not m.has_terminal else None
    if AnalyticModel.owner_of(terminal_state_cost) is not m or not m.has_terminal:
        return None
    if getattr(terminal_state_cost, "__func__", None) is not reg.__dict__.get("terminal_cost"):
        return None
    return m
