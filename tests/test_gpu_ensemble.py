"""GPU: user models whose rollout copies differ (CudaModel(copies=M), rollout_samples=M) on the fused route — agreement
with the stepped route on the same twins, states / actions / get_rollouts, set_params, the argument checks that need a
registered model handle, resident mode (refused), and a two-GPU sharded ensemble.  The live-reference fixtures, and the
base family's M > 1 fixtures through a compiled restatement of their copy-offset dynamics, are replayed in
tests/test_gpu_golden_replay.py."""
import ctypes as C
import os

import pytest
import torch

import pytorch_mppi_b200 as eng
from pytorch_mppi_b200 import _cabi
from tests.golden.ensemble_cases import ENSEMBLE_CASES, case_params, engine_model, ensemble_controller

pytestmark = pytest.mark.gpu

TOL = {torch.float64: 1e-9, torch.float32: 1e-5}     # the fixtures' tolerances (tests/golden/cases.py U_TOL)


@pytest.mark.parametrize("name", ["ens_pend_mppi_f64", "ens_pend_smppi_f32", "ens_pend_kmppi_f64", "ens_stepint_mppi_f64"])
def test_fused_equals_stepped_route(name):
    """Same twins, same injected noise: the fused kernel and the reference's M-copy T-loop (stepped route) agree on the
    costs, the update, states, actions and get_rollouts."""
    case = ENSEMBLE_CASES[name]
    dt = torch.float64 if case["dtype"] == "f64" else torch.float32
    tol = TOL[dt]
    g = torch.Generator().manual_seed(5)
    m = engine_model(case)
    U0 = torch.randn(case["T"], 1, generator=g, dtype=dt)
    kw = {} if case["variant"] == "smppi" else dict(U_init=U0)
    fused, stepped = ensemble_controller(case, m, **kw), ensemble_controller(case, m, "stepped", **kw)
    rows = case["kernel"]["S"] if case["variant"] == "kmppi" else case["T"]
    x = torch.tensor(case["x0"], dtype=dt)
    for _ in range(2):
        z = torch.randn(case["K"], rows, 1, generator=g, dtype=dt)
        fused.inject_noise(z)
        stepped.inject_noise(z)
        a, b = fused.command(x), stepped.command(x)
        ct = stepped.cost_total
        assert float((fused.cost_total - ct).abs().max()) <= tol * max(1.0, float(ct.abs().max()))
        assert float((fused.U - stepped.U).abs().max()) <= tol and float((a - b).abs().max()) <= tol
        assert fused.states.shape == stepped.states.shape == (case["M"], case["K"], case["T"], 2)
        assert float((fused.states - stepped.states).abs().max()) <= tol * 10
        assert fused.actions.shape == stepped.actions.shape == (case["M"], case["K"], case["T"], 1)
        assert float((fused.actions - stepped.actions).abs().max()) <= tol
        stepped.U = fused.U
        if case["variant"] == "smppi":
            stepped.action_sequence = fused.action_sequence
        if case["variant"] == "kmppi":
            stepped.theta = fused.theta
    # get_rollouts: copy 0, which is what the K-based twin computes for num_rollouts <= K rows
    x0 = torch.tensor([[0.5, 0.1], [2.0, -1.0]], dtype=dt, device="cuda")
    got, want = fused.get_rollouts(x0, num_rollouts=2), stepped.get_rollouts(x0, num_rollouts=2)
    assert got.shape == want.shape and float((got - want).abs().max()) <= tol


def test_set_params_between_commands_matches_a_controller_built_with_them():
    case = ENSEMBLE_CASES["ens_pend_mppi_f64"]
    p2 = case_params(case)
    p2[6:10] = [1.5, 0.6, 1.0, 2.0]                   # other masses
    U0 = torch.randn(case["T"], 1, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    mA = engine_model(case)
    A = ensemble_controller(case, mA, U_init=U0.clone())
    g = torch.Generator().manual_seed(8)
    z1, z2 = (torch.randn(case["K"], case["T"], 1, generator=g, dtype=torch.float64) for _ in range(2))
    x = [2.5, 0.5]
    A.inject_noise(z1)
    A.command(x)
    plan = A._plan.value
    mA.set_params(p2)
    B = ensemble_controller(case, engine_model(case, params=p2), U_init=A.U.clone())
    A.inject_noise(z2)
    B.inject_noise(z2)
    a, b = A.command(x), B.command(x)
    assert torch.equal(a, b) and torch.equal(A.U, B.U) and torch.equal(A.cost_total, B.cost_total)
    assert torch.equal(A.states, B.states)
    assert A._plan.value == plan


def test_resident_mode_is_refused_and_plans_check_the_copy_count():
    case = ENSEMBLE_CASES["ens_pend_mppi_f64"]
    c = ensemble_controller(case, engine_model(case))
    c.command([2.5, 0.5])
    with pytest.raises(_cabi.MppiLibraryError, match="split-cost"):
        c.start_resident()
    lib, p, plan = c._lib, _cabi.MppiFusedParams.from_buffer_copy(c._p), C.c_void_p()
    for M in (1, 0, 3, 5):                                     # the model was compiled with 4 copies
        p.rollout_samples = M
        assert lib.mppi_plan_create(C.byref(p), C.byref(plan)) == -1, M
    p.rollout_samples = 4
    p.var_discount = None
    assert lib.mppi_plan_create(C.byref(p), C.byref(plan)) == -1
    assert lib.mppi_user_model_set_copies(p.user_model, 9) == -1 and lib.mppi_user_model_set_copies(p.user_model, 0) == -1
    # a model compiled with one copy has split-cost / resident kernels: it cannot be declared an ensemble
    plain = eng.CudaModel(2, 1, "x[0] = O::add(x[0], u[0]);", "return x[0];", params=[1.0])
    h1 = plain.rtc_handle(lib, torch.float64, 0)
    assert lib.mppi_user_model_set_copies(h1, 2) == -1 and lib.mppi_user_model_set_copies(h1, 1) == 0


def _shard_worker(rank, world, port, out):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        case = dict(ENSEMBLE_CASES["ens_pend_mppi_f64"], K=4097)
        g = torch.Generator().manual_seed(3)
        z = torch.randn(case["K"], case["T"], 1, generator=g, dtype=torch.float64)
        U0 = torch.randn(case["T"], 1, generator=g, dtype=torch.float64)
        res = {}
        for exchange in ("p2p", "nccl"):
            one = ensemble_controller(case, engine_model(case), U_init=U0.clone(), device=dev)
            many = ensemble_controller(case, engine_model(case), U_init=U0.clone(), device=dev, process_group=dist.group.WORLD,
                         exchange=exchange)
            for _ in range(2):
                one.inject_noise(z)
                many.inject_noise(z)
                a1, a2 = one.command([2.5, 0.5]), many.command([2.5, 0.5])
            res[exchange] = (float((one.U - many.U).abs().max()), float((a1 - a2).abs().max()))
        out[rank] = res
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_sharded_ensemble_equals_unsharded():
    """Copies never cross a shard: each rank rolls out all M copies of its samples."""
    import torch.multiprocessing as mp
    out = mp.Manager().dict()
    mp.spawn(_shard_worker, args=(2, 29600 + os.getpid() % 1000, out), nprocs=2, join=True)
    for rank in range(2):
        for key, (err, aerr) in out[rank].items():
            assert err < 1e-9 and aerr < 1e-9, (rank, key, err, aerr)
