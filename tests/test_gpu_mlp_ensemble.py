"""GPU: ensembles of learned pendulum networks (PendulumMLPEnsemble, rollout_samples = M networks) on the fused route —
parity with the live-reference fixtures on the wgmma and FFMA kernels, agreement with the stepped route on the same
twins, every M on the wgmma kernel, M identical networks against one PendulumMLP, refresh() after retraining, resident
mode (refused) and a two-GPU sharded ensemble."""
import os

import numpy as np
import pytest
import torch

import pytorch_mppi_b200 as eng
from pytorch_mppi_b200 import _cabi
from tests.golden.cases import make_mlp_net
from tests.golden.engine import replay
from tests.golden.mlp_ensemble_cases import MLP_ENSEMBLE, MLP_ENSEMBLE_CASES, load_nets
from tests.golden.replay import OracleRunner, load

pytestmark = pytest.mark.gpu

# DESIGN §2, C4 (the learned pendulum), on U and the action: fp64 FFMA, fp32 FFMA, fp32 wgmma with hi/lo-split bf16
# operands
TOL = {("f64", False): 1e-9, ("f32", False): 5e-5, ("f32", "bf16x3"): 5e-4}
# ... except mlpens_smppi_f32 on the wgmma kernel: 1.35e-3 measured at step 2 (steps 0-1 within 5e-4), held to 2e-3, the
# C4 wgmma tolerance with MUFU.TANH.  That command's U is more sensitive to the network's rounding than C4's: the oracle
# on the fixture, with every step's output perturbed by 1.5e-5 relative noise (bf16x3's layer accuracy), moves U by
# 0.6-1.2e-3, while the FFMA kernel (fp32 operands) stays within 5e-5.
FIXTURE_TOL = {("mlpens_smppi_f32", "bf16x3"): 2e-3}


def _assert_costs_close(got, want, tol, dtype):
    """Per-sample costs.  fp64: within tol (relative to the largest cost).  fp32: C4's cost tolerance of
    tests/test_gpu_parity.py (rtol = atol = 2e-3), except for at most one sample in 500, which may be off by up to 1 %.
    Those are rollouts that reach the angle wrap (x0 -> +-pi) within a rounding error: on the other branch the next
    network input differs, so the sample's cost is not determined to fp32 accuracy by its inputs.  The fixtures show it
    without the engine: re-evaluating mlpens_mppi_f32 in fp64 moves sample 431's cost at step 1 by 0.36 (of ~300), and
    moving x by -1e-6 moves sample 969's at step 0 by 0.28, while U stays within 4e-5."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    d, scale = np.abs(got - want), max(1.0, float(np.abs(want).max()))
    if dtype == torch.float64:
        assert float(d.max()) <= tol * scale, float(d.max())
        return
    out = d > 2e-3 + 2e-3 * np.abs(want)
    assert int(out.sum()) <= max(1, want.size // 500), (int(out.sum()), np.flatnonzero(out)[:8], d[out][:8])
    assert float(d.max()) <= 1e-2 * scale, float(d.max())


def _ctrl(case, ens, stepped=False, device="cuda", **kw):
    """The controller of a case on the fused route, or (stepped=True) on the stepped route with the same torch twin."""
    dt = torch.float64 if case["dtype"] == "f64" else torch.float32
    dyn = (lambda s, a: ens.dynamics(s, a)) if stepped else ens.dynamics
    args = dict(num_samples=case["K"], horizon=case["T"], lambda_=case["lambda_"], device=device,
                u_max=torch.tensor(case["u_max"], dtype=dt), rollout_samples=case["M"], rollout_var_cost=case["var_cost"],
                rollout_var_discount=case["var_discount"])
    args.update(kw)
    sigma = torch.tensor(case["noise_sigma"], dtype=dt)
    if case["variant"] == "kmppi":
        c = eng.KMPPI(dyn, ens.running_cost, 2, sigma, num_support_pts=case["kernel"]["S"],
                      kernel=eng.RBFKernel(sigma=case["kernel"]["sigma"]), **args)
    elif case["variant"] == "smppi":
        sm = case["smooth"]
        c = eng.SMPPI(dyn, ens.running_cost, 2, sigma, w_action_seq_cost=sm["w"], delta_t=sm["delta_t"],
                      action_max=torch.tensor(sm["action_max"], dtype=dt), **args)
    else:
        c = eng.MPPI(dyn, ens.running_cost, 2, sigma, **args)
    assert (c._model is None) if stepped else (c._model is ens), "route not selected"
    return c


def _routes():
    return [(n, tc) for n in sorted(MLP_ENSEMBLE_CASES)
            for tc in ((False, "bf16x3") if MLP_ENSEMBLE_CASES[n]["dtype"] == "f32" else (False,))]


@pytest.mark.parametrize("name,tc", _routes())
def test_fused_matches_reference_golden(name, tc):
    case, gold = load(name)
    run = OracleRunner(case, gold, MLP_ENSEMBLE)
    nets = [n.cuda() for n in load_nets(case, gold)]
    ens = eng.PendulumMLPEnsemble(nets, max_torque=case["u_max"], tensor_cores=tc)
    c = _ctrl(case, ens, **({} if case["variant"] == "smppi" else dict(U_init=run.stream.U0.clone())))
    tol = FIXTURE_TOL.get((name, tc), TOL[(case["dtype"], tc)])
    # the nominal in lock-step with the reference's, as tests/test_gpu_parity.py: per-step errors do not compound
    replay(c, run, gold, tol, lambda got, want: _assert_costs_close(got, want, tol, run.prob.dtype), reset_nominal=True)
    assert c.launch_info.split_cost == 0


@pytest.mark.parametrize("name,tc", [("mlpens_mppi_f64", False), ("mlpens_kmppi_f64", False),
                                     ("mlpens_smppi_f32", False), ("mlpens_smppi_f32", "bf16x3"),
                                     ("mlpens_mppi_f32", "bf16x3")])
def test_fused_equals_stepped_route(name, tc):
    """Same twin, same injected noise: the fused kernel and the reference's M-copy T-loop (stepped route) agree on the
    costs, the update, and the (M,K,T,.) states and actions of the command (which the public properties expose only
    with a terminal cost); get_rollouts runs network 0."""
    case = MLP_ENSEMBLE_CASES[name]
    dt = torch.float64 if case["dtype"] == "f64" else torch.float32
    tol = TOL[(case["dtype"], tc)]
    g = torch.Generator().manual_seed(5)
    nets = [make_mlp_net(case["net_seed"] + m, dt).cuda() for m in range(case["M"])]
    ens = eng.PendulumMLPEnsemble(nets, max_torque=case["u_max"], tensor_cores=tc)
    U0 = torch.randn(case["T"], 1, generator=g, dtype=dt)
    kw = {} if case["variant"] == "smppi" else dict(U_init=U0)
    fused, stepped = _ctrl(case, ens, **kw), _ctrl(case, ens, stepped=True, **kw)
    rows = case["kernel"]["S"] if case["variant"] == "kmppi" else case["T"]
    x = torch.tensor(case["x0"], dtype=dt)
    M, K, T = case["M"], case["K"], case["T"]
    for _ in range(2):
        z = torch.randn(K, rows, 1, generator=g, dtype=dt)
        fused.inject_noise(z)
        stepped.inject_noise(z)
        a, b = fused.command(x), stepped.command(x)
        _assert_costs_close(fused.cost_total.cpu(), stepped.cost_total.cpu(), tol, dt)
        assert float((fused.U - stepped.U).abs().max()) <= tol and float((a - b).abs().max()) <= tol
        assert fused.states is None and stepped.states is None          # no terminal cost (mppi.py:307-310)
        fused._materialize(want_states=True)
        assert fused._states_buf.shape == stepped._states.shape == (M, K, T, 2)
        # per rollout; in fp32 a rollout that reaches the angle wrap within a rounding error may take the other branch
        dev = (fused._states_buf - stepped._states).abs().amax(dim=(2, 3)).flatten()
        assert int((dev > tol * 100).sum()) <= (0 if dt == torch.float64 else max(1, M * K // 500)), float(dev.max())
        assert stepped._actions.shape == (M, K, T, 1)
        assert float((fused._pa_buf.unsqueeze(0) - stepped._actions).abs().max()) <= tol
        stepped.U = fused.U
        if case["variant"] == "smppi":
            stepped.action_sequence = fused.action_sequence
        if case["variant"] == "kmppi":
            stepped.theta = fused.theta
    x0 = torch.tensor([[0.5, 0.1], [2.0, -1.0]], dtype=dt, device="cuda")
    got = fused.get_rollouts(x0, num_rollouts=2)
    want, seq = eng.PendulumMLP(nets[0], max_torque=case["u_max"]), fused.get_action_sequence()
    ref = x0
    for t in range(T):
        ref = want.dynamics(ref, seq[t].expand(2, -1))
        assert float((got[:, t] - ref).abs().max()) <= tol * 100, t


@pytest.mark.parametrize("M", range(2, _cabi.MPPI_MAX_COPIES + 1))
def test_every_copy_count_on_the_wgmma_kernel(M):
    """Each M from 2 to MPPI_MAX_COPIES on the tensor-core kernel at small K, against the stepped route."""
    case = dict(MLP_ENSEMBLE_CASES["mlpens_mppi_f32"], M=M, K=300, T=12, net_seed=100 + 10 * M)
    nets = [make_mlp_net(case["net_seed"] + m, torch.float32).cuda() for m in range(M)]
    ens = eng.PendulumMLPEnsemble(nets, max_torque=case["u_max"])
    g = torch.Generator().manual_seed(M)
    U0 = torch.randn(case["T"], 1, generator=g)
    fused, stepped = _ctrl(case, ens, U_init=U0), _ctrl(case, ens, stepped=True, U_init=U0)
    z = torch.randn(case["K"], case["T"], 1, generator=g)
    fused.inject_noise(z)
    stepped.inject_noise(z)
    a, b = fused.command(case["x0"]), stepped.command(case["x0"])
    tol = TOL[("f32", "bf16x3")]
    _assert_costs_close(fused.cost_total.cpu(), stepped.cost_total.cpu(), tol, torch.float32)
    assert float((fused.U - stepped.U).abs().max()) <= tol and float((a - b).abs().max()) <= tol
    assert fused.launch_info.block_threads == 256 and fused.launch_info.threads_per_sample == 2   # the wgmma tiles


def test_identical_networks_match_a_single_network_controller():
    """M copies of one network with rollout_var_cost = 0: the ensemble's cost is that network's (fp64, FFMA kernel)."""
    case = MLP_ENSEMBLE_CASES["mlpens_mppi_f64"]
    net = make_mlp_net(7, torch.float64).cuda()
    ens = eng.PendulumMLPEnsemble([net] * 4, max_torque=2.0)
    one = eng.PendulumMLP(net, max_torque=2.0)
    g = torch.Generator().manual_seed(2)
    U0 = torch.randn(case["T"], 1, generator=g, dtype=torch.float64)
    sigma = torch.tensor(1.0, dtype=torch.float64)
    kw = dict(num_samples=case["K"], horizon=case["T"], lambda_=1.0, device="cuda", U_init=U0,
              u_max=torch.tensor(2.0, dtype=torch.float64))
    A = eng.MPPI(ens.dynamics, ens.running_cost, 2, sigma, rollout_samples=4, rollout_var_cost=0.0, **kw)
    B = eng.MPPI(one.dynamics, one.running_cost, 2, sigma, **kw)
    assert A._model is ens and B._model is one
    for _ in range(2):
        z = torch.randn(case["K"], case["T"], 1, generator=g, dtype=torch.float64)
        A.inject_noise(z)
        B.inject_noise(z)
        a, b = A.command([2.5, 0.5]), B.command([2.5, 0.5])
        assert float((A.cost_total - B.cost_total).abs().max()) <= 1e-12 * float(B.cost_total.abs().max())
        assert float((A.U - B.U).abs().max()) <= 1e-12 and float((a - b).abs().max()) <= 1e-12


@pytest.mark.parametrize("tc", [False, "bf16x3"])
def test_refresh_rereads_the_weights(tc):
    case = MLP_ENSEMBLE_CASES["mlpens_smppi_f32"]
    nets = [make_mlp_net(case["net_seed"] + m, torch.float32).cuda() for m in range(case["M"])]
    ens = eng.PendulumMLPEnsemble(nets, max_torque=2.0, tensor_cores=tc)
    A = _ctrl(case, ens)
    g = torch.Generator().manual_seed(6)
    z1, z2 = (torch.randn(case["K"], case["T"], 1, generator=g) for _ in range(2))
    A.inject_noise(z1)
    A.command(case["x0"])
    with torch.no_grad():                           # "retraining"
        for net in nets:
            for p in net.parameters():
                p.mul_(1.1).add_(0.01)
    A.refresh()
    fresh = [make_mlp_net(0, torch.float32).cuda() for _ in nets]
    for f, net in zip(fresh, nets):
        f.load_state_dict(net.state_dict())
    B = _ctrl(case, eng.PendulumMLPEnsemble(fresh, max_torque=2.0, tensor_cores=tc))
    B.U, B.action_sequence = A.U.clone(), A.action_sequence.clone()
    A.inject_noise(z2)
    B.inject_noise(z2)
    a, b = A.command(case["x0"]), B.command(case["x0"])
    assert torch.equal(a, b) and torch.equal(A.U, B.U) and torch.equal(A.cost_total, B.cost_total)


def test_resident_mode_is_refused():
    case = MLP_ENSEMBLE_CASES["mlpens_mppi_f32"]
    nets = [make_mlp_net(case["net_seed"] + m, torch.float32).cuda() for m in range(case["M"])]
    c = _ctrl(case, eng.PendulumMLPEnsemble(nets, max_torque=2.0))
    c.command(case["x0"])
    with pytest.raises(_cabi.MppiLibraryError, match="split-cost"):
        c.start_resident()


def _shard_worker(rank, world, port, out):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        res = {}
        for name in ("mlpens_mppi_f64", "mlpens_mppi_f32"):
            case = dict(MLP_ENSEMBLE_CASES[name], K=4097)
            dt = torch.float64 if case["dtype"] == "f64" else torch.float32
            nets = [make_mlp_net(case["net_seed"] + m, dt).to(dev) for m in range(case["M"])]
            g = torch.Generator().manual_seed(3)
            z = torch.randn(case["K"], case["T"], 1, generator=g, dtype=dt)
            U0 = torch.randn(case["T"], 1, generator=g, dtype=dt)
            for exchange in ("p2p", "nccl"):
                one = _ctrl(case, eng.PendulumMLPEnsemble(nets), U_init=U0.clone(), device=dev)
                many = _ctrl(case, eng.PendulumMLPEnsemble(nets), U_init=U0.clone(), device=dev,
                             process_group=dist.group.WORLD, exchange=exchange)
                for _ in range(2):
                    one.inject_noise(z)
                    many.inject_noise(z)
                    a1, a2 = one.command(case["x0"]), many.command(case["x0"])
                res[(name, exchange)] = (float((one.U - many.U).abs().max()), float((a1 - a2).abs().max()))
        out[rank] = res
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_sharded_ensemble_equals_unsharded():
    """Copies never cross a shard: each rank rolls out all M networks for its samples."""
    import torch.multiprocessing as mp
    out = mp.Manager().dict()
    mp.spawn(_shard_worker, args=(2, 29700 + os.getpid() % 1000, out), nprocs=2, join=True)
    for rank in range(2):
        for key, (err, aerr) in out[rank].items():
            tol = 1e-9 if "f64" in key[0] else 1e-5
            assert err < tol and aerr < tol, (rank, key, err, aerr)
