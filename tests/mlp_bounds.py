"""Per-sample error bounds of the learned pendulum kernels against an fp64 network forward pass (test-only, CPU).

The kernels (csrc/mppi_mlp_tc.cuh: wgmma, operands bf16x3 or bf16; csrc/mppi_math.cuh: FFMA in fp32 or fp64) compute
the costs of `PendulumMLP` / `PendulumMLPEnsemble` rollouts.  This module gives, for each sample, the fp64 reference cost
(`PendulumMLP.net_step` on an fp64 copy of the network) and a rigorous bound on how far a kernel of a given arithmetic
can be from it.  The bound is propagated layer by layer in absolute values, `delta_out <= |W| delta_in + local error`,
then through the state update and the cost, and step by step along the fp64 trajectory.  Every constant is derived
below from the arithmetic the kernel performs; none is fitted to measured errors, and there is no safety factor.  A
kernel that drops a product term, misplaces a bias, clamps wrongly or counts the wrong step's cost leaves the bound on
many samples: `emulate` is the kernel arithmetic on the CPU, with `mutation=` faults of that kind, to show it.

u = 2^-24 (fp32) or 2^-53 (fp64) is the unit roundoff; gamma(n) = n u / (1 - n u) bounds n successive roundings.
"""
import copy
import math
from dataclasses import dataclass

import torch

from pytorch_mppi_b200.models import PendulumMLP

U32, U64 = 2.0 ** -24, 2.0 ** -53
BF16_HI = 2.0 ** -8          # x in [2^E, 2^(E+1)): |x - bf16_rn(x)| <= 2^(E-8) (8 significant bits)
BF16_RES = 2.0 ** -17        # and |x - hi - lo| <= 2^(E-17) for the hi / lo split: x - hi lies below 2^(E-8) unless it
                             # is that power of two (then lo is exact), so lo has 8 bits below 2^(E-9) (the device-math
                             # suite asserts the relative form, 2^-17 |x|, over every float)
BF16_TINY = 2.0 ** -126      # below the bf16 normals the split residuals are absolute, at most this much
TANH4_ABS = 1e-6             # tanh4_, exp form, absolute (tests/test_gpu_device_math.py: TANH4_ABS)
TANH_MUFU_REL = 2.0 ** -10.987   # tanh.approx.f32, relative (PTX bound; tests/test_gpu_device_math.py: TANH_APPROX_REL)
TANH_F64_REL = 2.0 ** -52    # libm tanh in fp64: within one ulp
# The wgmma fp32 accumulator.  H100 does not document how an MMA rounds when it adds its 16 exact bf16 products to the
# fp32 accumulator, and it has not been measured here.  Assumed: each MMA issued adds an error of at most 4 * 2^-23 of
# (|accumulator| + sum |products|): the addends aligned to the largest exponent and truncated, losing up to two bits
# more than one round-to-nearest of the sum.  The accumulator starts at the fp32 bias, so per layer the error is at most
# n_mma * ACC_MMA * (|b| + 1.02 sum |a| |w|) (1.02 covers the hi / lo parts' magnitudes against |a| |w|).
ACC_MMA = 4 * 2.0 ** -23
ACT_MAX = 1.0 + 1e-3         # |tanh output| in any form (MUFU's relative error on top of 1)


def gamma(n, u):
    return n * u / (1 - n * u)


@dataclass(frozen=True)
class Mode:
    """One kernel arithmetic.  arith: "bf16x3" / "bf16" (wgmma kernels), "ffma32" / "ffma64" (FFMA kernels); tanh:
    "exp" (tanh4_'s exp form) or "mufu" (MUFU.TANH).  fp64 kernels use libm tanh whatever the flag says."""
    arith: str
    tanh: str = "exp"

    @property
    def f64(self):
        return self.arith == "ffma64"

    @property
    def u(self):
        return U64 if self.f64 else U32

    @property
    def dtype(self):
        return torch.float64 if self.f64 else torch.float32

    def __str__(self):
        return self.arith if self.f64 else f"{self.arith}/{self.tanh}"


# the fp64 reference's own error: fp64 dot products and tanh, bounded as the fp64 kernel's; added to every bound
REF = Mode("ffma64")


def _in(dtype, v):
    """v as the kernel's constant of that dtype, in fp64."""
    return float(torch.tensor(v, dtype=torch.float64).to(dtype).double())


# ------------------------------------------------------------------------------------------------ fp64 reference
def reference_model(net, w_thdot, max_torque):
    """`PendulumMLP` on an fp64 copy of `net`: its `net_step` is the reference forward pass, its `running_cost` the cost."""
    return PendulumMLP(copy.deepcopy(net).double().cpu(), max_torque=max_torque, w_thdot=w_thdot)


def reference_step(model, x, u):
    """One fp64 `PendulumMLP.net_step`: (next state, pre-wrap angle x0 + net_0, tanh outputs h1, h2)."""
    seen = []
    hooks = [m.register_forward_hook(lambda _m, _i, o: seen.append(o)) for m in model.net if isinstance(m, torch.nn.Tanh)]
    outs = []
    last = [m for m in model.net if isinstance(m, torch.nn.Linear)][-1]
    hooks.append(last.register_forward_hook(lambda _m, _i, o: outs.append(o)))
    try:
        nxt = model.dynamics(x, u.view(-1, 1))
    finally:
        for h in hooks:
            h.remove()
    return nxt, x[:, 0] + outs[0][:, 0], seen[0], seen[1]


# ------------------------------------------------------------------------------------------------ the bound
def params(net):
    """fp64 [W1, b1, W2, b2, W3, b3] of a network (W in PyTorch's (out, in) layout)."""
    return [p.detach().double().cpu() for m in net if isinstance(m, torch.nn.Linear) for p in (m.weight, m.bias)]


def split_bf16(w):
    """hi = bf16_rn(w), lo = bf16_rn(w - hi) (w fp32-valued; fp64 out): the kernels' `tc::split_bf16`."""
    hi = w.float().bfloat16().double()
    return hi, (w.float() - hi.float()).bfloat16().double()


def _product_error(W, arith, a_abs):
    """Bound on sum_k |a_k w_k - computed_k| per output unit, for operands |a| <= a_abs, on the tensor cores.  bf16x3
    computes a_hi w_hi + a_lo w_hi + a_hi w_lo; with a = a_hi + a_lo + r_a and w = w_hi + w_lo + r_w it misses
    a_lo w_lo + r_a (w_hi + w_lo) + (a_hi + a_lo) r_w.  For a in the binade [2^E, 2^(E+1)), |a - a_hi| <= 2^(E-8) and
    |r_a| <= 2^(E-17) (|a_lo| <= 2^(E-8) too); w's parts are known exactly.  bf16 computes a_hi w_hi and misses
    (a - a_hi) w + a_hi (w - w_hi).  Below the bf16 normals the residuals are absolute, at most 2^-126."""
    hi, lo = split_bf16(W)
    p2 = torch.exp2(torch.floor(torch.log2(a_abs.clamp(min=BF16_TINY)))) + BF16_TINY     # 2^E >= ... of any |a| <= a_abs
    if arith == "bf16x3":
        return p2 @ (BF16_HI * lo.abs() + BF16_RES * (hi + lo).abs()).T + (a_abs * (1 + BF16_RES)) @ (W - hi - lo).abs().T
    return p2 @ (BF16_HI * W.abs()).T + (a_abs * (1 + BF16_HI)) @ (W - hi).abs().T


def _layer(W, b, a_abs, d_in, mode, n_chain):
    """Bound on the error of z = W a + b: |W| d_in plus the layer's own error given |a| <= a_abs.  Tensor cores (layers
    2 and 3 of the wgmma kernels): the products' split error and the accumulator's; FFMA: a chain of n_chain roundings
    per term (layer 2: 32 FMAs from the bias; layer 3: four 8-FMA chains, then two adds)."""
    Wa = W.abs()
    dot = b.abs() + a_abs @ Wa.T
    if mode.arith in ("bf16x3", "bf16"):
        n_mma = 6 if mode.arith == "bf16x3" else 2
        local = _product_error(W, mode.arith, a_abs) + n_mma * ACC_MMA * (b.abs() + 1.02 * (a_abs @ Wa.T))
    else:
        local = gamma(n_chain, mode.u) * dot
    return d_in @ Wa.T + local


def _tanh(h_ref, dz, mode):
    """Error of the kernel's tanh: 1-Lipschitz propagation of dz (at most 2) plus the form's own error."""
    d = torch.clamp(dz, max=2.0)
    mag = torch.clamp(h_ref.abs() + d, max=1.0)
    if mode.f64:
        return d + TANH_F64_REL * mag
    if mode.tanh == "mufu":
        return d + TANH_MUFU_REL * mag
    return d + TANH4_ABS


def _pis(mode):
    return _in(mode.dtype, math.pi), _in(mode.dtype, 2 * math.pi)


def _wrap_error(th_abs, mode):
    """|W_kernel(th) - W(th)| on the same branch, W(th) = rem(th + pi, 2 pi) - pi exact.  The kernel rounds th + pi,
    rem + 2 pi (negative remainders) and the final - pi once each (fmod is exact) with the dtype's pi and 2 pi, so the
    pi_f cancel and n wraps leave n |2pi_f - 2 pi|."""
    pi, two_pi = _pis(mode)
    n = torch.floor((th_abs + pi) / (2 * math.pi)) + 1
    return mode.u * (th_abs + pi + two_pi + pi) + n * abs(two_pi - 2 * math.pi)


def _branch_margin(th_abs, dth, mode):
    """How far from an odd multiple of pi the exact pre-wrap angle must lie for the kernel to take the same branch:
    the angle's error, the rounding of th + pi, and the kernel's branch points j 2pi_f - pi_f against j 2 pi - pi."""
    pi, two_pi = _pis(mode)
    n = torch.floor((th_abs + dth + pi) / (2 * math.pi)) + 1
    return dth + mode.u * (th_abs + dth + pi) + n * abs(two_pi - 2 * math.pi) + abs(pi - math.pi)


def copy_rollout(model, x0, u, mode):
    """Roll the fp64 reference model out from x0 (N, 2) under the actions u (N, T) (the model clamps them).  Returns
    the reference running costs c (N, T) (step t: the cost of x_{t+1}), per-step error bounds dc (N, T) for a kernel
    of `mode` (the reference's own error included), and the undetermined mask (N,): samples whose pre-wrap angle came
    within its bound of the wrap before the last step.  On the other branch the next network input differs by 2 pi,
    so such a sample's kernel cost is not determined by its inputs to this accuracy."""
    W1, b1, W2, b2, W3, b3 = params(model.net)
    N, T = u.shape
    x = x0.double().clone()
    dx = torch.zeros_like(x)
    und = torch.zeros(N, dtype=torch.bool)
    pi, two_pi = _pis(mode)
    w_k = _in(mode.dtype, model.w_thdot)
    ua = mode.u + U64                       # each rounding of the update and the cost: the kernel's and the reference's
    cs, dcs = [], []
    for t in range(T):
        ut = torch.clamp(u[:, t].double(), -model.max_torque, model.max_torque)
        nxt, th, h1, h2 = reference_step(model, x, ut)
        dd = torch.zeros(N, 2, dtype=torch.float64)
        for m, din in ((mode, dx), (REF, torch.zeros_like(dx))):   # the kernel's error and the reference's own
            # layer 1 in both kernels: an FMA chain of three terms from the bias; the state's error, u exact
            a0 = torch.stack((x[:, 0].abs() + dx[:, 0], x[:, 1].abs() + dx[:, 1], ut.abs()), dim=1)
            d0 = torch.stack((din[:, 0], din[:, 1], torch.zeros_like(ut)), dim=1)
            dz1 = d0 @ W1.abs().T + gamma(3, m.u) * (b1.abs() + a0 @ W1.abs().T)
            dh1 = _tanh(h1, dz1, m)
            dh2 = _tanh(h2, _layer(W2, b2, torch.clamp(h1.abs() + dh1, max=ACT_MAX), dh1, m, 32), m)
            dd = dd + _layer(W3, b3, torch.clamp(h2.abs() + dh2, max=ACT_MAX), dh2, m, 10)
        # the state update: th = x0 + d0 rounded, then the wrap; x1 + d1 rounded
        dth = dx[:, 0] + dd[:, 0] + ua * (th.abs() + dx[:, 0] + dd[:, 0])
        if t < T - 1:
            dist = (torch.remainder(th, 2 * math.pi) - math.pi).abs()      # to the nearest odd multiple of pi
            und |= dist <= _branch_margin(th.abs(), dth, mode)
        ex0 = dth + _wrap_error(th.abs() + dth, mode) + _wrap_error(th.abs(), REF)
        ex1 = dx[:, 1] + dd[:, 1] + ua * (nxt[:, 1].abs() + dx[:, 1] + dd[:, 1])
        # the cost of x_{t+1}, an^2 + w x1^2.  |an| = dist(th, 2 pi Z) is 1-Lipschitz in th and the same on either
        # branch; the kernel's |an| (two wraps: the state's and the cost's) is within dth + E(th) + 3 (E(pi) + |pi_f -
        # pi| + |2pi_f - 2 pi|) of it, the 3 covering a branch flip of the cost's wrap at |an| ~ pi
        an, x1 = nxt[:, 0].abs(), nxt[:, 1].abs()
        da = ex0 + 3 * (_wrap_error(torch.full_like(an, pi), mode) + abs(pi - math.pi) + abs(two_pi - 2 * math.pi))
        sa, sq = (an + da) ** 2, (x1 + ex1) ** 2
        e_an2 = 2 * an * da + da * da + ua * sa
        e_wq = w_k * (2 * x1 * ex1 + ex1 * ex1 + ua * sq) + abs(w_k - model.w_thdot) * x1 * x1 + ua * w_k * (1 + ua) * sq
        c = model.running_cost(nxt, None)
        dc = e_an2 + e_wq
        dcs.append(dc + ua * (c + dc))
        cs.append(c)
        x, dx = nxt, torch.stack((ex0, ex1), dim=1)
    return torch.stack(cs, 1), torch.stack(dcs, 1), und


def _sum(c, dc, n, u):
    """Sequential sums of n terms along the last axis (the kernels' running-cost sums): sum and its error bound."""
    return c.sum(-1), dc.sum(-1) + gamma(max(n - 1, 0), u) * (c + dc).sum(-1)


@dataclass
class Bound:
    cost: torch.Tensor           # (N,) fp64 reference cost_total
    bound: torch.Tensor          # (N,) bound on |kernel - reference|
    undetermined: torch.Tensor   # (N,) bool


def cost_bound(nets, x0, u, mode, *, max_torque, w_thdot, var_cost=0.0, var_disc=None):
    """The reference `cost_total` of a zero-nominal command (sum of the running costs; an ensemble's mean over the
    copies plus var_cost * sum_t var_disc[t] var_m(c_{m,t})) and its bound for a kernel of `mode`.  nets: one network,
    or the ensemble's list; x0 (N, 2); u (N, T) the actions the model receives (u_scale applied, not clamped);
    var_disc: the controller's discount table (its dtype's values)."""
    single = isinstance(nets, torch.nn.Module)
    nets = [nets] if single else list(nets)
    T, M = u.shape[1], len(nets)
    ua = mode.u + U64                       # each rounding below: the kernel's and the reference's
    runs = [copy_rollout(reference_model(n, w_thdot, max_torque), x0, u, mode) for n in nets]
    c = torch.stack([r[0] for r in runs])   # (M, N, T)
    dc = torch.stack([r[1] for r in runs])
    und = torch.stack([r[2] for r in runs]).any(0)
    C, dC = _sum(c, dc, T, ua)              # per copy, (M, N)
    if single:
        return Bound(C[0], dC[0], und)
    mean = C.mean(0)
    dmean = dC.mean(0) + gamma(M, ua) * (C + dC).mean(0)            # M - 1 adds and a division
    disc = torch.as_tensor(var_disc, dtype=torch.float64).view(1, T)
    # the per-step variance over the copies (two-pass, unbiased): first-order sensitivity plus the squared bounds,
    # then the two-pass rounding with the computed mean's error e
    d = c - c.mean(0)
    dd = dc + dc.mean(0)
    var = (d * d).sum(0) / (M - 1)                                     # (N, T)
    e = gamma(M, ua) * (c + dc).mean(0)
    dh = d.abs() + dd
    dvar = ((2 * d.abs() * dd + dd * dd) + 2 * dh * e + e * e + gamma(M + 4, ua) * (dh + e) ** 2).sum(0) / (M - 1)
    V, dV = _sum(disc * var, disc * dvar, T, ua)
    vc = _in(mode.dtype, var_cost)
    total = mean + var_cost * V
    dtot = dmean + vc * dV + abs(vc - var_cost) * V + ua * vc * (1 + ua) * (V + dV)
    return Bound(total, dtot + ua * (total + dtot), und)


# ------------------------------------------------------------------------------------------------ CPU emulation
MUTATIONS = ("l2_drop_lo_hi", "l2_drop_hi_lo", "l3_drop_lo_hi", "l3_drop_hi_lo", "swap_b2", "swap_w2_cols",
             "no_b3_0", "no_b3_1", "no_clamp", "clamp_half", "cost_of_x0", "last_cost_missing",
             "ens_b3_of_copy0", "ens_w1_of_copy0")


def _round_bits(y, bits):
    m, e = torch.frexp(y)
    return torch.ldexp(torch.round(m * 2.0 ** bits) / 2.0 ** bits, e)


def _emu_tanh(z, mode):
    y = torch.tanh(z.double())
    if mode.f64:
        return y
    if mode.tanh == "mufu":            # a tanh good to 11 bits: within MUFU.TANH's 2^-10.987, far outside 1e-6
        y = _round_bits(y, 11)
    return y.float()


def _fma(a, b, c):
    return (a.double() * b.double() + c.double()).to(c.dtype)


def _emu_mma(a, W, b, mode, layer, mutation):
    """z = W a + b on the tensor cores: bf16 parts, exact products summed in fp64, the fp32 accumulator."""
    ah, al = split_bf16(a.double())
    wh, wl = split_bf16(W)
    acc = b.double().expand(a.shape[0], -1).clone()
    for s in range(2):
        k = slice(16 * s, 16 * s + 16)
        acc = acc + ah[:, k] @ wh[:, k].T
        if mode.arith == "bf16x3":
            if mutation != f"l{layer}_drop_lo_hi" or s != 1:
                acc = acc + al[:, k] @ wh[:, k].T
            if mutation != f"l{layer}_drop_hi_lo" or s != 1:
                acc = acc + ah[:, k] @ wl[:, k].T
    return acc.float()


def _emu_step(P, x, u, mode, mutation, max_torque):
    W1, b1, W2, b2, W3, b3 = [p.to(mode.dtype) for p in P]
    if mutation == "swap_b2":
        b2 = b2[[1, 0] + list(range(2, 32))]
    if mutation == "swap_w2_cols":
        W2 = W2[:, [0, 6, 2, 3, 4, 5, 1, 7] + list(range(8, 32))]
    if mutation in ("no_b3_0", "no_b3_1"):
        b3 = b3.clone()
        b3[int(mutation[-1])] = 0
    mt = {"no_clamp": math.inf, "clamp_half": max_torque / 2}.get(mutation, max_torque)
    uc = torch.clamp(u, -mt, mt)
    inp = (x[:, 0:1], x[:, 1:2], uc.view(-1, 1))
    h = b1.expand(x.shape[0], -1)
    for c in range(3):
        h = _fma(W1[:, c], inp[c], h)
    h = _emu_tanh(h, mode)
    if mode.arith in ("bf16x3", "bf16"):
        h = _emu_tanh(_emu_mma(h, W2, b2, mode, 2, mutation), mode)
        d = _emu_mma(h, W3, b3, mode, 3, mutation)
    else:
        acc = b2.expand(x.shape[0], -1)
        for j in range(32):
            acc = _fma(W2[:, j], h[:, j:j + 1], acc)
        h = _emu_tanh(acc, mode)
        o = [b3.expand(x.shape[0], -1)] + [torch.zeros(x.shape[0], 2, dtype=mode.dtype)] * 3
        for j in range(32):
            o[j % 4] = _fma(W3[:, j], h[:, j:j + 1], o[j % 4])
        d = (o[0] + o[1]) + (o[2] + o[3])
    return torch.stack((_emu_wrap(x[:, 0] + d[:, 0], mode), x[:, 1] + d[:, 1]), dim=1)


def _emu_wrap(th, mode):
    pi, two_pi = (torch.tensor(v, dtype=mode.dtype) for v in _pis(mode))
    m = torch.fmod(th + pi, two_pi)
    m = torch.where((m != 0) & (m < 0), m + two_pi, m)
    return m - pi


def _emu_cost(x, mode, w_thdot):
    an = _emu_wrap(x[:, 0], mode)
    return an * an + torch.tensor(w_thdot, dtype=mode.dtype) * (x[:, 1] * x[:, 1])


def emulate(nets, x0, u, mode, *, max_torque, w_thdot, var_cost=0.0, var_disc=None, mutation=None):
    """The kernel arithmetic of `mode` on the CPU: cost_total (N,) of a zero-nominal command, with an optional fault
    (one of MUTATIONS).  Products are exact in fp64, the outputs rounded to the kernel's dtype; bf16 parts come from
    torch's casts, which the device-math suite ties to cvt.rn.bf16x2."""
    single = isinstance(nets, torch.nn.Module)
    nets = [nets] if single else list(nets)
    Ps = [[p.float() if not mode.f64 else p for p in params(n)] for n in nets]
    if mutation in ("ens_b3_of_copy0", "ens_w1_of_copy0"):
        i = 5 if mutation == "ens_b3_of_copy0" else 0
        for P in Ps[1:]:
            P[i] = Ps[0][i]
    N, T = u.shape
    u = u.to(mode.dtype)
    costs = []                                             # (M, N, T): copy m's cost of x_{t+1}
    for P in Ps:
        x = x0.to(mode.dtype)
        c = []
        for t in range(T):
            if mutation == "cost_of_x0":
                c.append(_emu_cost(x, mode, w_thdot))
            x = _emu_step(P, x, u[:, t], mode, mutation, max_torque)
            if mutation != "cost_of_x0" and not (mutation == "last_cost_missing" and t == T - 1):
                c.append(_emu_cost(x, mode, w_thdot))
        costs.append(c)
    zero = torch.zeros(N, dtype=mode.dtype)
    if single:
        roll = zero
        for ct in costs[0]:
            roll = roll + ct
        return roll.double()
    M = len(Ps)
    cs, var = [zero] * M, zero
    disc = torch.as_tensor(var_disc).to(mode.dtype)
    for t in range(len(costs[0])):
        ct = [costs[m][t] for m in range(M)]
        mean = ct[0]
        for m in range(1, M):
            mean = mean + ct[m]
        mean = mean / M
        ss = zero
        for m in range(M):
            dm = ct[m] - mean
            ss = ss + dm * dm
        var = var + (ss / (M - 1)) * disc[t]
        cs = [cs[m] + ct[m] for m in range(M)]
    mean = cs[0]
    for m in range(1, M):
        mean = mean + cs[m]
    mean = mean / M
    return (mean + var * torch.tensor(var_cost, dtype=mode.dtype)).double()


# ------------------------------------------------------------------------------------------------ probes
def probe_inputs(K, T, max_torque, seed):
    """Start states (K, 2) and actions (K, T) (fp32) over the ranges where the kernels go wrong: angles across
    [-pi, pi], unwrapped ones (+-5, +-7) and +-pi exactly (the float nearest pi); velocities across +-8 with +-20 and
    larger ones that push the pre-activations past 10, where tanh4_ clamps; actions up to 3 max_torque with exactly
    +-max_torque and 0.  A rollout that starts at +-pi sits on the wrap after a small first step, so for T > 1 only a
    few samples start there (the rest would be undetermined)."""
    g = torch.Generator().manual_seed(seed)
    pi = float(torch.tensor(math.pi, dtype=torch.float32))
    th = (torch.rand(K, generator=g, dtype=torch.float64) * 2 - 1) * math.pi
    om = (torch.rand(K, generator=g, dtype=torch.float64) * 2 - 1) * 8
    special_th = torch.tensor([5.0, -5.0, 7.0, -7.0, 0.0], dtype=torch.float64)
    special_om = torch.tensor([20.0, -20.0, 60.0, -60.0, 150.0, 8.0, -8.0], dtype=torch.float64)
    th = torch.where(torch.rand(K, generator=g) < 0.2, special_th[torch.randint(0, 5, (K,), generator=g)], th)
    on_pi = torch.rand(K, generator=g) < (0.1 if T == 1 else 0.002)
    th = torch.where(on_pi, torch.where(torch.rand(K, generator=g) < 0.5, pi, -pi).double(), th)
    om = torch.where(torch.rand(K, generator=g) < 0.2, special_om[torch.randint(0, 7, (K,), generator=g)], om)
    u = (torch.rand(K, T, generator=g, dtype=torch.float64) * 2 - 1) * 3 * max_torque
    special_u = torch.tensor([max_torque, -max_torque, 0.0], dtype=torch.float64)
    u = torch.where(torch.rand(K, T, generator=g) < 0.2, special_u[torch.randint(0, 3, (K, T), generator=g)], u)
    if K >= 2:                         # both exact wrap points in every probe
        th[0], th[1] = pi, -pi
    return torch.stack((th, om), 1).float(), u.float()


def _linear_net():
    return torch.nn.Sequential(torch.nn.Linear(3, 32), torch.nn.Tanh(), torch.nn.Linear(32, 32), torch.nn.Tanh(),
                               torch.nn.Linear(32, 2))


def probe_net(kind, seed=0):
    """The probe networks (fp32): "default" (the reference's initialisation, tests/golden/cases.make_mlp_net);
    "binades" (weights spread over 2^-14 .. 2^1, a third of them bf16-exact, lo = 0); "saturating" (large weights:
    most hidden units sit at +-1); "tame" (default with W2 and W3 scaled down: a bound that stays useful over 30 steps);
    "zero" (every weight 0: the increment is exactly 0, the state only wraps)."""
    from tests.golden.cases import make_mlp_net
    net = make_mlp_net(seed, torch.float32)
    lin = [m for m in net if isinstance(m, torch.nn.Linear)]
    g = torch.Generator().manual_seed(1000 + seed)
    with torch.no_grad():
        if kind == "binades":
            for i, m in enumerate(lin):
                for p in (m.weight, m.bias):
                    mag = 2.0 ** (torch.rand(p.shape, generator=g) * 15 - 14 + (0 if i < 2 else -2))
                    v = torch.where(torch.rand(p.shape, generator=g) < 0.5, -mag, mag)
                    exact = torch.rand(p.shape, generator=g) < 1 / 3
                    p.copy_(torch.where(exact, v.bfloat16().float(), v))
        elif kind == "saturating":
            lin[0].weight.mul_(8)
            lin[1].weight.mul_(6)
        elif kind == "tame":
            lin[1].weight.mul_(0.5)
            lin[2].weight.mul_(0.05)
            lin[2].bias.mul_(0.05)
        elif kind == "zero":
            for p in net.parameters():
                p.zero_()
        else:
            assert kind == "default", kind
    return net


MODES = [Mode(a, t) for a in ("bf16x3", "bf16", "ffma32") for t in ("exp", "mufu")] + [Mode("ffma64")]


def probe_sets():
    """(network kind, T, modes) of the probe matrix.  Each probe keeps its undetermined samples under 1 %: bf16 operands
    and MUFU.TANH make bounds that widen fast with T, so they run past T = 1 on the tame network only (bf16 past T = 2),
    and T = 30 runs the exp-tanh modes with split or fp32 operands."""
    narrow = [m for m in MODES if m.arith != "bf16" and (m.tanh == "exp" or m.f64)]
    return [("default", 1, MODES), ("binades", 1, MODES), ("saturating", 1, MODES),
            ("default", 2, [m for m in MODES if m.arith != "bf16"]), ("tame", 2, MODES),
            ("default", 3, narrow), ("tame", 3, MODES), ("tame", 30, narrow)]
