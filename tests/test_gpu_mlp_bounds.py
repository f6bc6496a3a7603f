"""GPU: every learned-dynamics kernel against the fp64 network forward pass, per sample, within the error bound of its
own arithmetic (tests/mlp_bounds.py), outside the chaotic 30-step rollout.

Observable: the first command from a zero nominal (MPPI / KMPPI: U_init = 0; SMPPI: zero action sequence and
w_action_seq_cost = 0; no noise offset).  The action cost lambda U Sigma^-1 eps is then exactly 0, so cost_total[k] is
the sum of sample k's running costs.  Injected z chooses the actions (sigma = 1), a (K, 2) start-state tensor the states
(FLAG_STATE_PER_SAMPLE).  The network input is read back from `perturbed_action`: the sampling kernel that materialises
it runs the command kernels' own transform_column / action_at on the same z, so it is the action the command used (for
MPPI and SMPPI it is z itself, which the tests assert).  Every (kernel, variant, mode, tanh, M, T) writes its worst
error / bound ratio and its undetermined samples to tests/_reports/mlp_bounds.json."""
import json

import pytest
import torch

import pytorch_mppi_b200 as eng
from tests import mlp_bounds as mb
from tests import reports

pytestmark = pytest.mark.gpu

MT, W_THDOT, DISC = 2.0, 0.1, 0.5
K_PROBE = 4096 + 37
REPORT = {}
_LAST = {}
VARIANTS = ("mppi", "smppi", "kmppi")
WGMMA = [(v, a, t) for v in VARIANTS for a in ("bf16x3", "bf16") for t in ("exp", "mufu")]


def _record(key, value):
    REPORT[key] = value
    reports.write("mlp_bounds.json", json.dumps(REPORT, indent=1, sort_keys=True))


def _controller(variant, model, K, T, dtype, M=1, var_cost=0.0):
    kw = dict(num_samples=K, horizon=T, lambda_=1.0, device="cuda")
    if M > 1:
        kw.update(rollout_samples=M, rollout_var_cost=var_cost, rollout_var_discount=DISC)
    sigma = torch.tensor(1.0, dtype=dtype)
    zero = torch.zeros(T, 1, dtype=dtype)
    if variant == "smppi":
        c = eng.SMPPI(model.dynamics, model.running_cost, 2, sigma, w_action_seq_cost=0.0, delta_t=1.0, **kw)
    elif variant == "kmppi":
        c = eng.KMPPI(model.dynamics, model.running_cost, 2, sigma, num_support_pts=T, kernel=eng.RBFKernel(sigma=1.0),
                      U_init=zero, **kw)
    else:
        c = eng.MPPI(model.dynamics, model.running_cost, 2, sigma, U_init=zero, **kw)
    assert c._model is model, "fused route not selected"
    return c


def _check(tag, variant, mode, nets, K, T, *, var_cost=0.0, seed=0, tensor_cores=None, wgmma=True, bound_mode=None):
    """One command on the fused kernel; every determined sample within the bound.  Returns the share of the
    determined samples outside `bound_mode`'s bound instead when that is given (discrimination runs)."""
    dtype = mode.dtype
    ens = not isinstance(nets, torch.nn.Module)
    tc = tensor_cores if tensor_cores is not None else (mode.arith if wgmma else False)
    cuda_nets = [n.to("cuda", dtype) for n in nets] if ens else nets.to("cuda", dtype)
    Model = eng.PendulumMLPEnsemble if ens else eng.PendulumMLP
    model = Model(cuda_nets, max_torque=MT, w_thdot=W_THDOT, fast_tanh=mode.tanh == "mufu", tensor_cores=tc)
    M = len(nets) if ens else 1
    c = _controller(variant, model, K, T, dtype, M, var_cost)
    x0, u = mb.probe_inputs(K, T, MT, seed)
    c.inject_noise(u.to(dtype).view(K, T, 1))
    c.command(x0.to("cuda", dtype) if K > 1 else x0[0].to("cuda", dtype))
    if wgmma:
        assert c.launch_info.block_threads == 256 and c.launch_info.threads_per_sample == 2     # the wgmma tiles
    pa = c.perturbed_action.view(K, T).cpu()
    if variant != "kmppi":
        assert torch.equal(pa, u.to(dtype)), "the materialised action is not z"
    x0 = x0 if K > 1 else x0[:1]
    disc = DISC ** torch.arange(T, dtype=dtype)          # the controller's discount table, in its dtype
    b = mb.cost_bound(nets, x0, pa, bound_mode or mode, max_torque=MT, w_thdot=W_THDOT, var_cost=var_cost, var_disc=disc)
    got = c.cost_total.cpu().double().view(-1)[:K]
    _LAST["cost"] = got
    ok = ~b.undetermined
    ratio = (got - b.cost).abs() / b.bound
    worst = float(ratio[ok].max()) if bool(ok.any()) else 0.0
    und = torch.nonzero(b.undetermined).view(-1).tolist()
    if bound_mode is not None:
        share = float((ratio[ok] > 1).double().mean())
        _record(f"{tag}|discrimination under {bound_mode}", dict(share_outside=share, worst=worst))
        return share
    _record(tag, dict(worst_ratio=worst, undetermined=len(und), undetermined_samples=und, K=K))
    assert len(und) <= 0.01 * K, (tag, und)
    bad = torch.nonzero(ok & (ratio > 1)).view(-1)
    assert len(bad) == 0, (tag, worst, bad[:8].tolist(), got[bad[:4]].tolist(), b.cost[bad[:4]].tolist())
    return worst


def _smppi(variant, mode, runs):
    """SMPPI needs T >= 2 (the library refuses T = 1, as the reference does: its shift reads action_sequence[-2]), so
    its T = 1 probes run at T = 2, on a network of the T = 2 probe set that keeps the mode's bound useful."""
    if variant != "smppi":
        return runs
    ok2 = {k for k, T, modes in mb.probe_sets() if T == 2 and mode in modes}
    return [(kind if kind in ok2 else "tame", K, 2) if T == 1 else (kind, K, T) for kind, K, T in runs]


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("variant,arith,tanh", WGMMA)
def test_wgmma_single_network_within_its_bound(variant, arith, tanh):
    """mlp_tc_command_kernel<V, SPLIT, FAST>: every K geometry (one sample with a shared state, a part tile, one tile,
    one tile and a sample, many tiles, several passes of the grid) at T = 1, T = 2 and 3, and T = 30 on the tame
    network, each probe against its own mode's bound."""
    mode = mb.Mode(arith, tanh)
    big = _sms() * 128 * 5 + 37
    runs = [("default", 1, 1), ("binades", 37, 1), ("saturating", 128, 1), ("default", 129, 1),
            ("default", K_PROBE, 1), ("binades", K_PROBE, 1), ("saturating", K_PROBE, 1), ("default", big, 1)]
    for kind, T, modes in mb.probe_sets():
        if T > 1 and mode in modes:
            runs.append((kind, 1024 if T > 3 else K_PROBE, T))
    for i, (kind, K, T) in enumerate(_smppi(variant, mode, runs)):
        _check(f"wgmma|{variant}|{mode}|M1|T{T}|K{K}|{kind}", variant, mode, mb.probe_net(kind), K, T, seed=i)


@pytest.mark.parametrize("variant,arith,tanh", WGMMA)
def test_wgmma_ensemble_within_its_bound(variant, arith, tanh):
    """mlp_ens_tc_command_kernel<V, SPLIT, FAST>: one real network among all-zero ones, at every copy position (a zero
    copy's increment is exactly 0: it only wraps its state), and all-distinct copies with rollout_var_cost 0 and > 0."""
    mode = mb.Mode(arith, tanh)
    T = 2
    for M in (2, 3, 8):
        for pos in range(M):
            nets = [mb.probe_net("tame" if i == pos else "zero") for i in range(M)]
            _check(f"wgmma|{variant}|{mode}|M{M}|T{T}|real@{pos}", variant, mode, nets, 1000, T, seed=pos)
        for vc in (0.0, 0.25):
            nets = [mb.probe_net("tame", 10 * M + i) for i in range(M)]
            _check(f"wgmma|{variant}|{mode}|M{M}|T{T}|distinct|var{vc}", variant, mode, nets, 1000, T, var_cost=vc, seed=M)


FFMA = [mb.Mode("ffma32", "exp"), mb.Mode("ffma32", "mufu"), mb.Mode("ffma64")]


@pytest.mark.parametrize("mode", FFMA, ids=str)
@pytest.mark.parametrize("variant", VARIANTS)
def test_ffma_kernels_within_their_bound(variant, mode):
    """fused_command_kernel<PendulumMLPModel> (fp32 with tensor_cores=False, both tanh forms; fp64) and
    fused_command_kernel<PendulumMLPEnsembleModel>, each against its own, tighter bound."""
    runs = [("default", 37, 1), ("binades", K_PROBE, 1), ("saturating", K_PROBE, 1)]
    for kind, T, modes in mb.probe_sets():
        if T > 1 and mode in modes:
            runs.append((kind, 1024 if T > 3 else K_PROBE, T))
    for i, (kind, K, T) in enumerate(_smppi(variant, mode, runs)):
        _check(f"ffma|{variant}|{mode}|M1|T{T}|K{K}|{kind}", variant, mode, mb.probe_net(kind), K, T, seed=i, wgmma=False)
    for pos in range(3):
        nets = [mb.probe_net("tame" if i == pos else "zero") for i in range(3)]
        _check(f"ffma|{variant}|{mode}|M3|T2|real@{pos}", variant, mode, nets, 1000, 2, seed=pos, wgmma=False)
    for vc in (0.0, 0.25):
        nets = [mb.probe_net("tame", 30 + i) for i in range(3)]
        _check(f"ffma|{variant}|{mode}|M3|T2|distinct|var{vc}", variant, mode, nets, 1000, 2, var_cost=vc, seed=3, wgmma=False)


def test_the_mode_flags_reach_the_kernel():
    """bf16-mode costs leave the bf16x3 bound on a large share of samples: the operand flag reaches the kernel and the
    probe tells the instantiations apart.  MUFU-mode costs differ from exp-mode costs on the same inputs, on the wgmma
    and the FFMA kernel, so the tanh flag reaches both.  They do not leave the exp-tanh bound: on an H100, MUFU.TANH is
    within 1.1e-5 relative of tanh over every float (tests/test_gpu_device_math.py measures it), far inside its PTX
    bound of 2^-10.987, and a worst-case bound built on 1e-6 absolute per unit does not separate that from the exp
    form.  The share outside the exp-tanh bound is reported."""
    net = mb.probe_net("default")
    share = _check("wgmma|mppi|bf16/exp|M1|T1", "mppi", mb.Mode("bf16"), net, K_PROBE, 1, bound_mode=mb.Mode("bf16x3"))
    assert share >= 0.25, share
    for wgmma, arith in ((True, "bf16x3"), (False, "ffma32")):
        costs = []
        for tanh in ("exp", "mufu"):
            m = mb.Mode(arith, tanh)
            _check(f"{'wgmma' if wgmma else 'ffma'}|mppi|{m}|M1|T1|binades", "mppi", m, mb.probe_net("binades"), K_PROBE, 1,
                   wgmma=wgmma, bound_mode=mb.Mode(arith))
            costs.append(_LAST["cost"])
        d = (costs[0] - costs[1]).abs()
        _record(f"{'wgmma' if wgmma else 'ffma'}|mppi|{arith}|mufu-exp", dict(max_abs=float(d.max()), differ=int((d > 0).sum()),
                                                                         max_rel=float((d / costs[0].abs()).max())))
        assert int((d > 0).sum()) > 0, "MUFU.TANH and the exp form gave identical costs"
