"""CPU oracle for the MPPI / SMPPI / KMPPI ``command()`` hot path.

TEST INFRASTRUCTURE ONLY.  This module is the checker the CUDA engine in
``pytorch_mppi_b200`` is compared against.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline legs may import it;
the product package never does (it fails loudly when its CUDA library is
missing instead of falling back to this).

It is a functional restatement (torch-CPU tensor ops, explicit state in / state
out, no classes with hidden RNG) of the algorithm in the reference
``reference src/pytorch_mppi/mppi.py``.  Torch CPU ops are used (rather
than numpy) because every flop of the reference runs in torch: using the same
ATen kernels makes the oracle *bit-identical* to the reference in fp32 and fp64
when both consume the same standard-normal draws ``z`` — see
``tests/golden/make_golden.py`` which pins exactly that against the live
reference, and ``tests/test_oracle_golden.py`` which replays the committed
vectors.  Parity status: PINNED against the live reference (the reference's own
tests contain no golden vectors for ``command()``; SURVEY.md §8c).

Every function cites the reference lines it restates.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, Optional

import numpy as np
import torch


# --------------------------------------------------------------------------------------
# Workload definitions (the analytic models BASELINE.json's configs are quoted on)
# --------------------------------------------------------------------------------------
class PendulumModel:
    """Gym pendulum, restating reference tests/pendulum.py:30-60.

    dynamics : u <- clamp(u, +-max_torque); thdot' = clip(thdot + (3g/(2l) sin th + 3/(m l^2) u) dt, +-max_speed)
               th' = th + thdot' dt                         (velocity clipped BEFORE integrating th)
    cost     : angle_normalize(th)^2 + 0.1 thdot^2          (action ignored; evaluated on the post-step state)
    """

    nx, nu = 2, 1

    def __init__(self, g=10.0, m=1.0, l=1.0, dt=0.05, max_torque=2.0, max_speed=8.0, numpy_sin=True):
        self.numpy_sin = numpy_sin
        self.g, self.m, self.l, self.dt = g, m, l, dt
        self.max_torque, self.max_speed = max_torque, max_speed
        # python-float coefficients, multiplied into tensors exactly as the reference's
        # literals are (pendulum.py:43): 3*g/(2*l) and 3.0/(m*l**2)
        self.c_sin = 3 * g / (2 * l)
        self.c_u = 3.0 / (m * l ** 2)

    def dynamics(self, state, action):
        th = state[:, 0:1]
        thdot = state[:, 1:2]
        u = torch.clamp(action, -self.max_torque, self.max_torque)
        # pendulum.py:43 calls np.sin on the tensor: for fp32 that is NUMPY's sinf, which differs from
        # torch.sin in the last bit on ~some inputs; follow the reference (CPU-only oracle anyway).
        sin_th = torch.from_numpy(np.sin(th.numpy())) if self.numpy_sin else torch.sin(th)
        acc = self.c_sin * sin_th + self.c_u * u
        new_thdot = torch.clamp(thdot + acc * self.dt, -self.max_speed, self.max_speed)
        new_th = th + new_thdot * self.dt
        return torch.cat((new_th, new_thdot), dim=1)

    @staticmethod
    def angle_normalize(x):
        # pendulum.py:51-52; `%` on tensors is torch.remainder (sign of the divisor)
        return ((x + math.pi) % (2 * math.pi)) - math.pi

    def running_cost(self, state, action):
        th = state[:, 0]
        thdot = state[:, 1]
        return self.angle_normalize(th) ** 2 + 0.1 * thdot ** 2


class LinearPointModel:
    """2-D point with linear-delta dynamics, quadratic goal cost, optional action cost,
    optional Gaussian 'hill' costs and an optional terminal cost.

    With B=diag(1,-1), Q=I, R=0, no hills it is the fixture environment of the reference's
    unit tests (reference tests/test_mppi.py:24-51).  With B=diag(.5,-.5), R=0.01 I,
    one hill (Q_h=2.5*[[.1,.05],[.05,.1]], centre (-.5,-1), height 200), goal (2,2) and
    terminal_scale=10 it is the Toy2D navigation environment of
    reference tests/smooth_mppi.py:29-36,50-76,102-111,131-142 (BASELINE config 3).
    Quadratic forms are evaluated as sum_i sum_j d_i Q_ij d_j per row (the reference delegates
    to arm_pytorch_utilities.linalg.batch_quadratic_product, which is not vendored).
    """

    nx, nu = 2, 2

    def __init__(self, B, goal, Q=None, R=None, hills=(), terminal_scale=0.0, dtype=torch.double):
        self.dtype = dtype
        self.B = torch.as_tensor(B, dtype=dtype)
        self.goal = torch.as_tensor(goal, dtype=dtype)
        self.Q = torch.eye(2, dtype=dtype) if Q is None else torch.as_tensor(Q, dtype=dtype)
        self.R = None if R is None else torch.as_tensor(R, dtype=dtype)
        # hills: sequence of (Q_h (2x2), centre (2,), height)
        self.hills = [(torch.as_tensor(q, dtype=dtype), torch.as_tensor(c, dtype=dtype), float(h)) for q, c, h in hills]
        self.terminal_scale = float(terminal_scale)

    @staticmethod
    def _quad(d, Q):
        # d: (..., 2), Q: (2,2) -> (...,)   sum_i d_i * (sum_j Q_ij d_j)
        return (d * (d @ Q.transpose(0, 1))).sum(dim=-1)

    def dynamics(self, state, action):
        return state + action @ self.B.transpose(0, 1)

    def _state_cost(self, state):
        c = self._quad(self.goal - state, self.Q)
        for q, centre, h in self.hills:
            c = c + h * torch.exp(-self._quad(centre - state, q))
        return c

    def running_cost(self, state, action):
        c = self._state_cost(state)
        if self.R is not None:
            c = c + self._quad(action, self.R)
        return c

    def terminal_cost(self, states, actions):
        # states: (M,K,T,nx) -> (M,K); smooth_mppi.py:102-103 / test_mppi.py:49-51
        return self.terminal_scale * self._state_cost(states[..., -1, :])

    @property
    def has_terminal(self):
        return self.terminal_scale != 0.0


class MlpPendulumModel:
    """Learned pendulum dynamics of BASELINE config 4, restating the plugins of
    reference tests/pendulum_approximate.py:54-66, 100-110 around a given 3-32-32-2 tanh network:
    x' = x + net([x, clamp(u, +-2)]), theta' wrapped to [-pi, pi); cost as the analytic pendulum."""
    nx, nu = 2, 1
    has_terminal = False
    terminal_cost = None

    def __init__(self, net):
        self.net = net

    @staticmethod
    def angle_normalize(x):
        return (((x + math.pi) % (2 * math.pi)) - math.pi)

    def dynamics(self, state, perturbed_action):
        u = torch.clamp(perturbed_action, -2.0, 2.0)
        if state.dim() == 1 or u.dim() == 1:
            state = state.view(1, -1)
            u = u.view(1, -1)
        if u.shape[1] > 1:
            u = u[:, 0].view(-1, 1)
        xu = torch.cat((state, u), dim=1)
        with torch.no_grad():
            state_residual = self.net(xu)
        next_state = state + state_residual
        next_state[:, 0] = self.angle_normalize(next_state[:, 0])
        return next_state

    def running_cost(self, state, action):
        theta = state[:, 0]
        theta_dt = state[:, 1]
        return self.angle_normalize(theta) ** 2 + 0.1 * theta_dt ** 2


# --------------------------------------------------------------------------------------
# Problem description
# --------------------------------------------------------------------------------------
@dataclass
class Problem:
    """Everything `MPPI.__init__` (mppi.py:45-184) resolves, as plain data."""
    dynamics: Callable
    running_cost: Callable
    nx: int
    noise_sigma: torch.Tensor            # 0-dim, or (nu,nu)
    K: int = 100
    T: int = 15
    lambda_: float = 1.0
    noise_mu: Optional[torch.Tensor] = None
    u_min: Optional[torch.Tensor] = None
    u_max: Optional[torch.Tensor] = None
    u_init: Optional[torch.Tensor] = None
    u_scale: float = 1
    terminal_state_cost: Optional[Callable] = None
    sample_null_action: bool = False
    noise_abs_cost: bool = False
    # M > 1 rollouts of stochastic dynamics (mppi.py:54-58, 166-177)
    rollout_samples: int = 1
    rollout_var_cost: float = 0
    rollout_var_discount: float = 0.95
    # SpecificActionSampler.sample_trajectories as a plain function state -> (n,T,nu) (mppi.py:16-32, 393-399)
    specific_actions: Optional[Callable] = None
    # derived
    dtype: torch.dtype = field(init=False)
    nu: int = field(init=False)

    def __post_init__(self):
        self.dtype = self.noise_sigma.dtype                       # mppi.py:88
        self.nu = 1 if self.noise_sigma.dim() == 0 else self.noise_sigma.shape[0]   # mppi.py:94
        if self.noise_mu is None:
            self.noise_mu = torch.zeros(self.nu, dtype=self.dtype)  # mppi.py:97-98
        if self.u_init is None:
            self.u_init = torch.zeros_like(self.noise_mu)           # mppi.py:100-101
        if self.nu == 1:                                            # mppi.py:104-106
            self.noise_mu = self.noise_mu.view(-1)
            self.noise_sigma = self.noise_sigma.view(-1, 1)
        # one-sided bounds become symmetric; none -> +-inf (mppi.py:112-126)
        if self.u_max is not None and self.u_min is None:
            self.u_max = torch.as_tensor(self.u_max)
            self.u_min = -self.u_max
        if self.u_min is not None and self.u_max is None:
            self.u_min = torch.as_tensor(self.u_min)
            self.u_max = -self.u_min
        if self.u_min is None:
            self.u_min = torch.tensor(float("-inf"))
            self.u_max = torch.tensor(float("inf"))
        # covariance factorisation (mppi.py:131-139)
        sig = self.noise_sigma
        self.diagonal = bool(torch.equal(sig, torch.diag(torch.diag(sig))))
        if self.diagonal:
            d = torch.diag(sig)
            self.sigma_inv_diag = 1.0 / d
            self.sigma_sqrt_diag = torch.sqrt(d)
            self.sigma_inv = torch.diag(self.sigma_inv_diag)
        else:
            self.sigma_inv = torch.linalg.inv(sig)
            self.sigma_chol = torch.linalg.cholesky(sig)

    # mppi.py:201-206 with the randn factored out: z are the standard normals
    def colour(self, z):
        if self.diagonal:
            return z * self.sigma_sqrt_diag + self.noise_mu
        return z @ self.sigma_chol.T + self.noise_mu

    # mppi.py:186-199
    def action_cost(self, noise):
        g = torch.abs(noise) if self.noise_abs_cost else noise
        if self.diagonal:
            return self.lambda_ * g * self.sigma_inv_diag
        return self.lambda_ * g @ self.sigma_inv

    def clamp_u(self, a):                                           # mppi.py:419-420
        return torch.clamp(a, self.u_min, self.u_max)


# --------------------------------------------------------------------------------------
# Shared pieces
# --------------------------------------------------------------------------------------
def shift_rows(U, fill):
    """mppi.py:232-238: drop the first row, append `fill`."""
    U = torch.roll(U, -1, dims=0)
    U[-1] = fill
    return U


def rollout_costs(prob: Problem, x0, perturbed_action):
    """mppi.py:297-332 (M=1): returns (cost (K,), states|None, actions|None).

    The running cost is evaluated on the POST-step state, never on x0; actions fed to the
    model are u_scale * perturbed_action.
    """
    K, T, nu = perturbed_action.shape
    cost = torch.zeros(K, dtype=prob.dtype)
    if x0.shape == (K, prob.nx):
        state = x0.clone()
    else:
        state = x0.view(1, -1).expand(K, -1)
    keep = prob.terminal_state_cost is not None
    if keep:
        states = torch.empty(1, K, T, prob.nx, dtype=prob.dtype)
        actions = torch.empty(1, K, T, nu, dtype=prob.dtype)
    for t in range(T):
        u = prob.u_scale * perturbed_action[:, t]
        state = prob.dynamics(state, u)
        cost = cost + prob.running_cost(state, u).reshape(K)
        if keep:
            states[0, :, t] = state[:, :prob.nx]
            actions[0, :, t] = u
    if keep:
        c = prob.terminal_state_cost(states, actions)
        if torch.is_tensor(c) and c.dim() > 1:
            c = c.squeeze(0)
        cost = cost + c
        return cost, states, actions
    return cost, None, None


def rollout_costs_multi(prob: Problem, x0, perturbed_action):
    """mppi.py:334-373 (M>1): the K action sequences are rolled out M times through (stochastic)
    dynamics — rows are copy-major, row m*K+k is copy m of sample k (`state.repeat(M,1,1)` :351) —;
    cost = mean over copies + rollout_var_cost * sum_t discount^t * var_m(c_t)  (unbiased variance,
    torch.var's default).  Returns (cost (K,), states (M,K,T,nx), actions (M,K,T,nu))."""
    K, T, nu = perturbed_action.shape
    M = prob.rollout_samples
    cost_total = torch.zeros(K, dtype=prob.dtype)
    cost_samples = cost_total.repeat(M, 1)                                     # :340
    cost_var = torch.zeros_like(cost_total)                                    # :341
    if x0.shape == (K, prob.nx):
        state = x0
    else:
        state = x0.view(1, -1).expand(K, -1)
    state = state.repeat(M, 1, 1)                                              # :348
    states = torch.empty(M, K, T, prob.nx, dtype=prob.dtype)
    actions = torch.empty(M, K, T, nu, dtype=prob.dtype)
    discount = prob.rollout_var_discount ** torch.arange(T, dtype=prob.dtype)  # :174-175
    MK = M * K
    state_flat = state.reshape(MK, prob.nx)
    for t in range(T):
        u = prob.u_scale * perturbed_action[:, t].expand(M, -1, -1)            # :355
        u_flat = u.reshape(MK, nu)
        state_flat = prob.dynamics(state_flat, u_flat)                         # :357
        c = prob.running_cost(state_flat, u_flat)                              # :362
        cost_samples = cost_samples + c.reshape(M, K)                          # :363
        cost_var += c.reshape(M, K).var(dim=0) * discount[t]                   # :364
        states[:, :, t] = state_flat.reshape(M, K, -1)[:, :, :prob.nx]
        actions[:, :, t] = u
    c = prob.terminal_state_cost(states, actions) if prob.terminal_state_cost is not None else 0   # :161, :369
    cost_samples = cost_samples + c
    cost_total = cost_total + cost_samples.mean(dim=0)                         # :371
    cost_total = cost_total + cost_var * prob.rollout_var_cost                 # :372
    return cost_total, states, actions


def rollout(prob: Problem, x0, perturbed_action):
    """mppi.py:292-295"""
    if prob.rollout_samples == 1:
        return rollout_costs(prob, x0, perturbed_action)
    return rollout_costs_multi(prob, x0, perturbed_action)


def softmin_weights(cost_total, lambda_):
    """mppi.py:254-259 + 12-13: beta=min c; w=exp(-(1/lambda)(c-beta)); eta=sum w; omega=w/eta."""
    beta = torch.min(cost_total)
    w = torch.exp(-(1 / lambda_) * (cost_total - beta))
    eta = torch.sum(w)
    omega = (1.0 / eta) * w
    return beta, w, eta, omega


def _apply_null_action(prob, perturbed_action, x0=None):
    """mppi.py:387-400 (`_sample_specific_actions`): sample 0 is overwritten with zeros, then the rows after it with
    the SpecificActionSampler's trajectories — all BEFORE the clamp."""
    i = 0
    if prob.sample_null_action:
        perturbed_action[i] = 0                                    # :390-392
        i += 1
    if prob.specific_actions is not None:
        acts = prob.specific_actions(x0).reshape(-1, perturbed_action.shape[1], perturbed_action.shape[2])   # :394-396
        perturbed_action[i:i + acts.shape[0]] = acts               # :397
    return perturbed_action


# --------------------------------------------------------------------------------------
# MPPI
# --------------------------------------------------------------------------------------
def mppi_command(prob: Problem, U, x0, z, shift=True):
    """One `MPPI.command(state)` (mppi.py:240-275) with injected standard normals z (K,T,nu).

    Returns a dict with the new U, the action (U[0]) and all API-visible intermediates.
    """
    U = U.clone()
    if shift:
        U = shift_rows(U, prob.u_init)
    x0 = torch.as_tensor(x0).to(prob.dtype)
    eps_raw = prob.colour(z)                                   # mppi.py:378
    pa = U + eps_raw                                           # :380
    pa = _apply_null_action(prob, pa, x0)                      # :381
    pa = prob.clamp_u(pa)                                      # :383
    noise = pa - U                                             # :385
    ac = prob.action_cost(noise)                               # :409
    roll, states, actions = rollout(prob, x0, pa)              # :411
    pert = torch.sum(U * ac, dim=(1, 2))                       # :415
    cost_total = roll + pert                                   # :416
    beta, w, eta, omega = softmin_weights(cost_total, prob.lambda_)
    dU = torch.einsum("k,ktn->tn", omega, noise)               # :268
    U_new = U + dU                                             # :270
    return dict(U=U_new, U_before=U, action=U_new[0], cost_total=cost_total, omega=omega, w=w, beta=beta,
                eta=eta, noise=noise, perturbed_action=pa, states=states,
                actions=None if actions is None else actions / prob.u_scale)


# --------------------------------------------------------------------------------------
# SMPPI
# --------------------------------------------------------------------------------------
@dataclass
class SmoothParams:
    """SMPPI extras (mppi.py:456-484)."""
    w_action_seq_cost: float = 1.0
    delta_t: float = 1.0
    action_min: Optional[torch.Tensor] = None
    action_max: Optional[torch.Tensor] = None

    def __post_init__(self):
        if self.action_min is not None and self.action_max is None:
            self.action_min = torch.as_tensor(self.action_min)
            self.action_max = -self.action_min
        if self.action_max is not None and self.action_min is None:
            self.action_max = torch.as_tensor(self.action_max)
            self.action_min = -self.action_max
        if self.action_min is None:
            self.action_min = torch.tensor(float("-inf"))
            self.action_max = torch.tensor(float("inf"))


def smppi_command(prob: Problem, sp: SmoothParams, U, A, x0, z, shift=True):
    """One `SMPPI.command` (mppi.py:489-493, 520-570).  U is the control-derivative sequence,
    A the integrated action sequence.  Note (mppi.py:546 vs :548) the u_min/u_max clamp result is
    not used: the *unclamped* perturbed control is integrated."""
    U = U.clone()
    A = A.clone()
    if shift:
        U = shift_rows(U, prob.u_init)
        A = torch.roll(A, -1, dims=0)
        A[-1] = A[-2]                                           # :493
    x0 = torch.as_tensor(x0).to(prob.dtype)
    eps_raw = prob.colour(z)                                    # :542
    pc = U + eps_raw                                            # :544
    pa = A + pc * sp.delta_t                                    # :548
    pa = _apply_null_action(prob, pa)                           # :549
    pa = torch.clamp(pa, sp.action_min, sp.action_max)          # :550
    noise = (pa - A) / sp.delta_t - U                           # :552
    ac = prob.action_cost(noise)                                # :556
    diff = prob.u_scale * torch.diff(pa, dim=-2)                # :559
    smooth = torch.sum(torch.square(diff), dim=(1, 2))          # :560
    smooth = smooth * sp.w_action_seq_cost                      # :562
    roll, states, actions = rollout_costs(prob, x0, pa)         # :564
    pert = torch.sum(U * ac, dim=(1, 2))                        # :568
    cost_total = roll + pert + smooth                           # :569
    beta, w, eta, omega = softmin_weights(cost_total, prob.lambda_)
    dU = torch.einsum("k,ktn->tn", omega, noise)                # :527
    U_new = U + dU                                              # :529
    A_new = A + U_new * sp.delta_t                              # :531
    return dict(U=U_new, action_sequence=A_new, action=A_new[0], cost_total=cost_total, omega=omega,
                beta=beta, eta=eta, noise=noise, perturbed_action=pa, states=states,
                actions=None if actions is None else actions / prob.u_scale)


# --------------------------------------------------------------------------------------
# KMPPI
# --------------------------------------------------------------------------------------
def rbf_kernel(t, tk, sigma):
    """RBFKernel.__call__ (mppi.py:587-590) on (n,1),(m,1) time columns -> (n,m)."""
    d = torch.sum((t[:, None] - tk) ** 2, dim=-1)
    return torch.exp(-d / (1e-8 + 2 * sigma ** 2))


def kernel_matrices(T, S, kernel, dtype):
    """The two sample-independent interpolation operators KMPPI uses
    (mppi.py:621-627, 636-640, 617-619):  W = k(Hs,Tk) k(Tk,Tk)^-1 (T x S) and
    Wshift = k(Tk+1,Tk) k(Tk,Tk)^-1 (S x S), Tk=linspace(0,T-1,S), Hs=0..T-1."""
    Tk = torch.linspace(0, T - 1, int(S), dtype=dtype)
    Hs = torch.linspace(0, T - 1, int(T), dtype=dtype)
    G = kernel(Tk.unsqueeze(-1), Tk.unsqueeze(-1))
    W = torch.linalg.solve(G, kernel(Hs.unsqueeze(-1), Tk.unsqueeze(-1)), left=False)
    Wshift = torch.linalg.solve(G, kernel((Tk + 1).unsqueeze(-1), Tk.unsqueeze(-1)), left=False)
    return W, Wshift


def kmppi_command(prob: Problem, U, theta, x0, z, W, Wshift, shift=True):
    """One `KMPPI.command` (mppi.py:617-619, 657-688) with injected normals z (K,S,nu)."""
    U = U.clone()
    theta = theta.clone()
    if shift:
        U = shift_rows(U, prob.u_init)
        theta = torch.matmul(Wshift, theta)                     # :619
    x0 = torch.as_tensor(x0).to(prob.dtype)
    eps_raw = prob.colour(z)                                    # :660
    pts = prob.clamp_u(theta + eps_raw)                         # :661-663
    noise_theta = pts - theta                                   # :664
    pa = torch.matmul(W, pts)                                   # :665 (K,T,nu) = (T,S) @ (K,S,nu)
    pa = _apply_null_action(prob, pa)                           # :666
    pa = prob.clamp_u(pa)                                       # :668
    noise = pa - U                                              # :670
    ac = prob.action_cost(noise)
    roll, states, actions = rollout_costs(prob, x0, pa)
    pert = torch.sum(U * ac, dim=(1, 2))
    cost_total = roll + pert
    beta, w, eta, omega = softmin_weights(cost_total, prob.lambda_)
    dtheta = torch.einsum("k,ktn->tn", omega, noise_theta)      # :679
    theta_new = theta + dtheta                                  # :681
    U_new = torch.matmul(W, theta_new)                          # :682
    return dict(U=U_new, theta=theta_new, action=U_new[0], cost_total=cost_total, omega=omega, beta=beta,
                eta=eta, noise=noise, noise_theta=noise_theta, perturbed_action=pa, states=states,
                actions=None if actions is None else actions / prob.u_scale)


# --------------------------------------------------------------------------------------
# MPPI_Batched (SURVEY §8f.1)
# --------------------------------------------------------------------------------------
def mppi_batched_command(prob: Problem, U, states0, z, shift=True, u_per_command=1):
    """`MPPI_Batched.command` (mppi.py:822-873): N environments, noise z (K,T,nu) shared across
    environments, independent softmin per environment.  U: (N,T,nu), states0: (N,nx)."""
    U = U.clone()
    N = U.shape[0]
    K, T, nu = z.shape
    if shift:
        U = torch.roll(U, -1, dims=1)
        U[:, -1] = prob.u_init
    noise_s = prob.colour(z)
    pa = torch.clamp(U.unsqueeze(1) + noise_s.unsqueeze(0), prob.u_min, prob.u_max)
    noise = pa - U.unsqueeze(1)
    NK = N * K
    state = states0.to(prob.dtype).unsqueeze(1).expand(N, K, prob.nx).reshape(NK, prob.nx)
    cost = torch.zeros(N, K, dtype=prob.dtype)
    for t in range(T):
        u = prob.u_scale * pa[:, :, t].reshape(NK, nu)
        state = prob.dynamics(state, u)
        cost = cost + prob.running_cost(state, u).reshape(N, K)
    ac = prob.action_cost(noise)
    total = cost + torch.sum(U.unsqueeze(1) * ac, dim=(2, 3))
    beta = total.min(dim=1, keepdim=True).values
    w = torch.exp(-(1.0 / prob.lambda_) * (total - beta))
    eta = w.sum(dim=1, keepdim=True)
    omega = w / eta
    U_new = U + torch.einsum("nk,nktd->ntd", omega, noise)
    action = U_new[:, :u_per_command]                                # :870-873
    if u_per_command == 1:
        action = action[:, 0]
    return dict(U=U_new, action=action, cost_total=total, omega=omega)
