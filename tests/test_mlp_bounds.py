"""CPU: the per-sample error bounds of tests/mlp_bounds.py hold for the kernels' arithmetic and fail for faulty
arithmetic.  `emulate` (the kernel arithmetic on the CPU) stays within the bound of its own mode on every probe of
tests/test_gpu_mlp_bounds.py, and each fault a kernel change could introduce (a dropped hi / lo product term, a swapped
bias or weight column, a missing output bias, a wrong clamp, plain bf16 or MUFU.TANH under a tighter mode's bound, a
running cost lagged one step wrong, an ensemble copy reading copy 0's weights) leaves the bound on a clear share of the
probe samples.  That is the evidence, without a GPU, that the GPU test can fail."""
import pytest
import torch

from tests import mlp_bounds as mb

MT, W_THDOT = 2.0, 0.1
K_SHORT, K_LONG = 4096 + 37, 1024
SHARE = 0.10          # a fault must leave the bound on at least this share of the determined probe samples


def _probe(kind, T, seed=0):
    return mb.probe_net(kind, seed), *mb.probe_inputs(K_SHORT if T <= 3 else K_LONG, T, MT, seed=100 * T + seed)


def _ratio(b, got):
    """error / bound of the determined samples"""
    ok = ~b.undetermined
    return (got[ok] - b.cost[ok]).abs() / b.bound[ok]


@pytest.mark.parametrize("kind,T,modes", mb.probe_sets(), ids=[f"{k}-T{t}" for k, t, _ in mb.probe_sets()])
def test_emulation_stays_within_its_bound(kind, T, modes):
    net, x0, u = _probe(kind, T)
    worst = {}
    for mode in modes:
        b = mb.cost_bound(net, x0, u, mode, max_torque=MT, w_thdot=W_THDOT)
        r = _ratio(b, mb.emulate(net, x0, u, mode, max_torque=MT, w_thdot=W_THDOT))
        worst[str(mode)] = float(r.max())
        assert int(b.undetermined.sum()) <= 0.01 * len(u), (str(mode), int(b.undetermined.sum()))
        assert bool(torch.isfinite(b.bound).all())
    assert max(worst.values()) <= 1.0, worst


@pytest.mark.parametrize("mode", [mb.Mode("bf16x3"), mb.Mode("bf16", "mufu"), mb.Mode("ffma32"), mb.Mode("ffma64")], ids=str)
@pytest.mark.parametrize("var_cost", [0.0, 0.25])
def test_ensemble_emulation_stays_within_its_bound(mode, var_cost):
    T = 2
    nets = [mb.probe_net("tame", m) for m in range(3)] + [mb.probe_net("zero")]
    x0, u = mb.probe_inputs(K_SHORT, T, MT, seed=7)
    disc = 0.5 ** torch.arange(T, dtype=mode.dtype)
    kw = dict(max_torque=MT, w_thdot=W_THDOT, var_cost=var_cost, var_disc=disc)
    b = mb.cost_bound(nets, x0, u, mode, **kw)
    r = _ratio(b, mb.emulate(nets, x0, u, mode, **kw))
    assert int(b.undetermined.sum()) <= 0.01 * len(u)
    assert float(r.max()) <= 1.0, float(r.max())


def _share(nets, T, emu_mode, bound_mode, mutation=None, **kw):
    """share of the determined samples outside `bound_mode`'s bound, over the default and the binades probes"""
    out, n = 0, 0
    for kind in ("default", "binades"):
        net = [mb.probe_net(kind, m) for m in range(nets)] if nets > 1 else mb.probe_net(kind)
        x0, u = mb.probe_inputs(K_SHORT, T, MT, seed=100 * T)
        args = dict(max_torque=MT, w_thdot=W_THDOT, **kw)
        b = mb.cost_bound(net, x0, u, bound_mode, **args)
        r = _ratio(b, mb.emulate(net, x0, u, emu_mode, mutation=mutation, **args))
        out, n = out + int((r > 1).sum()), n + len(r)
    return out / n


X3 = mb.Mode("bf16x3")
FAULTS = {m: (1, 2 if m.startswith(("cost_of", "last_cost")) else 1, X3, X3, m) for m in mb.MUTATIONS}
FAULTS.update({"ens_b3_of_copy0": (3, 1, X3, X3, "ens_b3_of_copy0"), "ens_w1_of_copy0": (3, 1, X3, X3, "ens_w1_of_copy0"),
               "bf16_under_bf16x3": (1, 1, mb.Mode("bf16"), X3, None),
               "mufu_under_exp_wgmma": (1, 1, mb.Mode("bf16x3", "mufu"), X3, None),
               "mufu_under_exp_ffma": (1, 1, mb.Mode("ffma32", "mufu"), mb.Mode("ffma32"), None)})


@pytest.mark.parametrize("fault", sorted(FAULTS))
def test_each_fault_breaks_the_bound(fault):
    nets, T, emu_mode, bound_mode, mutation = FAULTS[fault]
    kw = dict(var_cost=0.25, var_disc=0.5 ** torch.arange(T, dtype=torch.float32)) if nets > 1 else {}
    share = _share(nets, T, emu_mode, bound_mode, mutation, **kw)
    assert share >= SHARE, (fault, share)


def test_the_bound_is_not_vacuous():
    """At T = 1 on the default network the bf16x3 bound's median is below 1e-4 of the cost."""
    net, x0, u = _probe("default", 1)
    b = mb.cost_bound(net, x0, u, X3, max_torque=MT, w_thdot=W_THDOT)
    assert float((b.bound / b.cost).median()) < 1e-4
