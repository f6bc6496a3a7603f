"""GPU: ensembles of learned pendulum networks (PendulumMLPEnsemble, rollout_samples = M networks) on the fused route —
agreement with the stepped route on the same twins, every M on the wgmma kernel, M identical networks against one
PendulumMLP, refresh() after retraining, resident mode (refused) and a two-GPU sharded ensemble.  The live-reference
fixtures are replayed on the wgmma and FFMA kernels in tests/test_gpu_golden_replay.py."""
import os

import pytest
import torch

import pytorch_mppi_b200 as eng
from pytorch_mppi_b200 import _cabi
from tests.golden.cases import make_mlp_net
from tests.golden.mlp_ensemble_cases import MLP_ENSEMBLE_CASES, TOL, assert_costs_close, ensemble_controller

pytestmark = pytest.mark.gpu

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
    fused, stepped = ensemble_controller(case, ens, **kw), ensemble_controller(case, ens, "stepped", **kw)
    rows = case["kernel"]["S"] if case["variant"] == "kmppi" else case["T"]
    x = torch.tensor(case["x0"], dtype=dt)
    M, K, T = case["M"], case["K"], case["T"]
    for _ in range(2):
        z = torch.randn(K, rows, 1, generator=g, dtype=dt)
        fused.inject_noise(z)
        stepped.inject_noise(z)
        a, b = fused.command(x), stepped.command(x)
        assert_costs_close(fused.cost_total.cpu(), stepped.cost_total.cpu(), tol, dt)
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
    fused, stepped = ensemble_controller(case, ens, U_init=U0), ensemble_controller(case, ens, "stepped", U_init=U0)
    z = torch.randn(case["K"], case["T"], 1, generator=g)
    fused.inject_noise(z)
    stepped.inject_noise(z)
    a, b = fused.command(case["x0"]), stepped.command(case["x0"])
    tol = TOL[("f32", "bf16x3")]
    assert_costs_close(fused.cost_total.cpu(), stepped.cost_total.cpu(), tol, torch.float32)
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
    A = ensemble_controller(case, ens)
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
    B = ensemble_controller(case, eng.PendulumMLPEnsemble(fresh, max_torque=2.0, tensor_cores=tc))
    B.U, B.action_sequence = A.U.clone(), A.action_sequence.clone()
    A.inject_noise(z2)
    B.inject_noise(z2)
    a, b = A.command(case["x0"]), B.command(case["x0"])
    assert torch.equal(a, b) and torch.equal(A.U, B.U) and torch.equal(A.cost_total, B.cost_total)


def test_resident_mode_is_refused():
    case = MLP_ENSEMBLE_CASES["mlpens_mppi_f32"]
    nets = [make_mlp_net(case["net_seed"] + m, torch.float32).cuda() for m in range(case["M"])]
    c = ensemble_controller(case, eng.PendulumMLPEnsemble(nets, max_torque=2.0))
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
                one = ensemble_controller(case, eng.PendulumMLPEnsemble(nets), U_init=U0.clone(), device=dev)
                many = ensemble_controller(case, eng.PendulumMLPEnsemble(nets), U_init=U0.clone(), device=dev,
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
