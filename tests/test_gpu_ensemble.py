"""GPU: user models whose rollout copies differ (CudaModel(copies=M), rollout_samples=M) on the fused route — parity with
the live-reference fixtures, agreement with the stepped route on the same twins, the existing M > 1 fixtures through a
compiled restatement of their copy-offset dynamics, states / actions / get_rollouts, set_params, the argument checks
that need a registered model handle, resident mode (refused), and a two-GPU sharded ensemble."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import pytorch_mppi_b200 as eng
from pytorch_mppi_b200 import _cabi
from tests import ensemble_models as em
from tests.golden.engine import replay
from tests.golden.ensemble_cases import ENSEMBLE, ENSEMBLE_CASES, case_params
from tests.golden.replay import OracleRunner, load

pytestmark = pytest.mark.gpu

TOL = {torch.float64: 1e-9, torch.float32: 1e-5}     # the parity table's tolerances


def _model(case, K=None, params=None):
    K = K or case["K"]
    p = params or case_params(case)
    if case["model"] == "pendulum":
        return em.pendulum_ensemble(case["M"], K, p)
    return em.scenario_integrator(case["M"], case["T"], K, p)


def _ctrl(case, m, stepped=False, **kw):
    """The controller of a case on the fused route, or (stepped=True) on the stepped route with the same torch twins."""
    dt = torch.float64 if case["dtype"] == "f64" else torch.float32
    sd = case["model"] == "scenario_integrator"
    dyn, cost = m.dynamics, m.running_cost
    if stepped:                       # not bound methods of the model: the reference's M-copy T-loop
        dyn = (lambda s, a, t: m.dynamics(s, a, t)) if sd else (lambda s, a: m.dynamics(s, a))
    args = dict(num_samples=case["K"], horizon=case["T"], lambda_=case["lambda_"], device="cuda",
                u_max=torch.tensor(case["u_max"], dtype=dt), terminal_state_cost=m.terminal_cost,
                rollout_samples=case["M"], rollout_var_cost=case["var_cost"], rollout_var_discount=case["var_discount"],
                step_dependent_dynamics=sd)
    args.update(kw)
    sigma = torch.tensor(case["noise_sigma"], dtype=dt)
    if case["variant"] == "kmppi":
        c = eng.KMPPI(dyn, cost, 2, sigma, num_support_pts=case["kernel"]["S"],
                      kernel=eng.RBFKernel(sigma=case["kernel"]["sigma"]), **args)
    elif case["variant"] == "smppi":
        sm = case["smooth"]
        c = eng.SMPPI(dyn, cost, 2, sigma, w_action_seq_cost=sm["w"], delta_t=sm["delta_t"],
                      action_max=torch.tensor(sm["action_max"], dtype=dt), **args)
    else:
        c = eng.MPPI(dyn, cost, 2, sigma, **args)
    assert (c._model is None) if stepped else (c._model is m), "route not selected"
    return c


@pytest.mark.parametrize("name", sorted(ENSEMBLE_CASES))
def test_fused_matches_reference_golden(name):
    case, gold = load(name)
    run = OracleRunner(case, family=ENSEMBLE)
    m = _model(case)
    kw = {} if case["variant"] == "smppi" else dict(U_init=run.stream.U0.clone())
    c = _ctrl(case, m, **kw)
    tol = TOL[run.prob.dtype]
    replay(c, run, gold, tol, lambda got, want: np.testing.assert_allclose(got, want, rtol=0,
                                                                          atol=tol * max(1.0, float(np.abs(want).max()))))
    assert c.launch_info.split_cost == 0


@pytest.mark.parametrize("name", ["ens_pend_mppi_f64", "ens_pend_smppi_f32", "ens_pend_kmppi_f64", "ens_stepint_mppi_f64"])
def test_fused_equals_stepped_route(name):
    """Same twins, same injected noise: the fused kernel and the reference's M-copy T-loop (stepped route) agree on the
    costs, the update, states, actions and get_rollouts."""
    case = ENSEMBLE_CASES[name]
    dt = torch.float64 if case["dtype"] == "f64" else torch.float32
    tol = TOL[dt]
    g = torch.Generator().manual_seed(5)
    m = _model(case)
    U0 = torch.randn(case["T"], 1, generator=g, dtype=dt)
    kw = {} if case["variant"] == "smppi" else dict(U_init=U0)
    fused, stepped = _ctrl(case, m, **kw), _ctrl(case, m, stepped=True, **kw)
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


@pytest.mark.parametrize("name", ["linear_mppi_multi_f64", "linear_mppi_multi_f32"])
def test_copy_offset_fixtures_replay_on_the_fused_route(name):
    """The reference's M > 1 fixtures (tests/golden/cases.py: copy m of a sample is pushed by m * copy_offset every step)
    through a CudaModel(copies=M) restatement of their linear dynamics."""
    case, gold = load(name)
    run = OracleRunner(case)
    dt = run.prob.dtype
    mdl = case["model"]
    ts = mdl.get("terminal_scale", 0.0)
    m = em.copy_offset_linear(case["rollout_samples"], mdl["B"], mdl["goal"], mdl["copy_offset"], ts,
                              terminal_cost=run.prob.terminal_state_cost)
    c = eng.MPPI(m.dynamics, m.running_cost, 2, torch.tensor(case["noise_sigma"], dtype=dt), num_samples=case["K"],
                 horizon=case["T"], lambda_=case["lambda_"], u_max=torch.tensor(case["u_max"], dtype=dt),
                 U_init=run.stream.U0.clone(), terminal_state_cost=m.terminal_cost if ts else None, device="cuda",
                 rollout_samples=case["rollout_samples"], rollout_var_cost=case["rollout_var_cost"],
                 rollout_var_discount=case["rollout_var_discount"])
    assert c._model is m
    replay(c, run, gold, TOL[dt])


def test_set_params_between_commands_matches_a_controller_built_with_them():
    case = ENSEMBLE_CASES["ens_pend_mppi_f64"]
    p2 = case_params(case)
    p2[6:10] = [1.5, 0.6, 1.0, 2.0]                   # other masses
    U0 = torch.randn(case["T"], 1, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    mA = _model(case)
    A = _ctrl(case, mA, U_init=U0.clone())
    g = torch.Generator().manual_seed(8)
    z1, z2 = (torch.randn(case["K"], case["T"], 1, generator=g, dtype=torch.float64) for _ in range(2))
    x = [2.5, 0.5]
    A.inject_noise(z1)
    A.command(x)
    plan = A._plan.value
    mA.set_params(p2)
    B = _ctrl(case, _model(case, params=p2), U_init=A.U.clone())
    A.inject_noise(z2)
    B.inject_noise(z2)
    a, b = A.command(x), B.command(x)
    assert torch.equal(a, b) and torch.equal(A.U, B.U) and torch.equal(A.cost_total, B.cost_total)
    assert torch.equal(A.states, B.states)
    assert A._plan.value == plan


def test_resident_mode_is_refused_and_plans_check_the_copy_count():
    case = ENSEMBLE_CASES["ens_pend_mppi_f64"]
    c = _ctrl(case, _model(case))
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
            one = _ctrl(case, _model(case), U_init=U0.clone(), device=dev)
            many = _ctrl(case, _model(case), U_init=U0.clone(), device=dev, process_group=dist.group.WORLD,
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
