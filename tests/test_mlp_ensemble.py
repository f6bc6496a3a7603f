"""CPU: ensembles of learned pendulum networks (PendulumMLPEnsemble, rollout_samples = M networks, one per copy) —
constructor checks, the torch twin's block split, the route rule, the C ABI field and the plans' argument checks, and what
the live-reference fixtures detect.  No GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

import pytorch_mppi_b200 as eng
from pytorch_mppi_b200 import _cabi, build
from pytorch_mppi_b200.mppi import SpecificActionSampler, fused_route_model
from tests.golden.cases import make_mlp_net
from tests.golden.mlp_ensemble_cases import MLP_ENSEMBLE, MLP_ENSEMBLE_CASES, load_nets, net_arrays
from tests.golden.replay import OracleRunner, load


def _nets(M, dtype=torch.float64, seed=10):
    return [make_mlp_net(seed + m, dtype) for m in range(M)]


def test_constructor_checks_every_network_and_the_count():
    ens = eng.PendulumMLPEnsemble(_nets(3), max_torque=1.5, w_thdot=0.2, fast_tanh=True, tensor_cores="bf16")
    assert ens.copies == 3 and ens.model_id == _cabi.MODEL_PENDULUM_MLP_ENSEMBLE == 4
    assert ens.param_blob() == eng.PendulumMLP(_nets(1)[0], 1.5, 0.2, True, "bf16").param_blob() == [1.5, 0.2, 1.0, 2.0]
    assert not ens.has_terminal and ens.param_blob_ext() == []
    for n in (0, 1, _cabi.MPPI_MAX_COPIES + 1):
        with pytest.raises(ValueError, match="networks"):
            eng.PendulumMLPEnsemble(_nets(n))
    wide = torch.nn.Sequential(torch.nn.Linear(3, 64), torch.nn.Tanh(), torch.nn.Linear(64, 64), torch.nn.Tanh(),
                               torch.nn.Linear(64, 2))
    relu = torch.nn.Sequential(torch.nn.Linear(3, 32), torch.nn.ReLU(), torch.nn.Linear(32, 32), torch.nn.Tanh(),
                               torch.nn.Linear(32, 2))
    for bad in (wide, relu):
        with pytest.raises(ValueError, match="Linear\\(3,32\\)"):
            eng.PendulumMLPEnsemble(_nets(2) + [bad])
    with pytest.raises(ValueError, match="tensor_cores"):
        eng.PendulumMLPEnsemble(_nets(2), tensor_cores="fp8")


def test_weight_table_is_param_blob_ext_per_network():
    nets = _nets(3)
    tab = eng.PendulumMLPEnsemble(nets).weight_table("cpu", torch.float64)
    assert tab.shape == (3, 1250) and tab.is_contiguous()
    for m, net in enumerate(nets):
        assert tab[m].tolist() == eng.PendulumMLP(net).param_blob_ext()
    assert eng.PendulumMLPEnsemble(nets).weight_table("cpu", torch.float32).dtype == torch.float32


def test_twin_sends_block_m_through_network_m():
    M, K = 4, 6
    nets = _nets(M)
    ens = eng.PendulumMLPEnsemble(nets, max_torque=2.0)
    g = torch.Generator().manual_seed(1)
    s = torch.randn(M * K, 2, generator=g, dtype=torch.float64)
    a = 3 * torch.randn(M * K, 1, generator=g, dtype=torch.float64)
    got = ens.dynamics(s, a)
    for m in range(M):
        want = eng.PendulumMLP(nets[m], max_torque=2.0).dynamics(s[m * K:(m + 1) * K], a[m * K:(m + 1) * K])
        assert torch.equal(got[m * K:(m + 1) * K], want)
    assert not torch.equal(got[:K], eng.PendulumMLP(nets[1]).dynamics(s[:K], a[:K]))
    assert torch.equal(ens.running_cost(s, a), eng.PendulumMLP(nets[0]).running_cost(s, a))
    with pytest.raises(ValueError, match="M\\*K rows"):
        ens.dynamics(s[:-1], a[:-1])


def test_route_rule():
    ens = eng.PendulumMLPEnsemble(_nets(4))

    def route(M, term=None, sampler=None, dyn=ens.dynamics):
        return fused_route_model(dyn, ens.running_cost, term, 2, 1, M, sampler, False)

    assert route(4) is ens
    assert route(4, sampler=SpecificActionSampler()) is None
    assert route(4, dyn=lambda s, a: ens.dynamics(s, a)) is None          # not the bound method: the stepped route
    for M in (1, 2, 3, 5, 8):
        with pytest.raises(ValueError, match="rollout_samples=4"):
            route(M)
    with pytest.raises(ValueError, match="rollout_samples=4"):
        route(2, sampler=SpecificActionSampler())


def _lib():
    build.build()
    return _cabi.load()


def test_abi_offset_of_model_weights():
    lib = _lib()
    assert lib.mppi_abi_layout(7) == _cabi.MppiFusedParams.model_weights.offset
    assert lib.mppi_abi_layout(0) == C.sizeof(_cabi.MppiFusedParams)
    assert _cabi.MppiFusedParams.model_weights.offset == C.sizeof(_cabi.MppiFusedParams) - 8    # the last field


def test_plans_check_the_ensemble_arguments_before_any_cuda_call():
    lib = _lib()
    tab = torch.zeros(8, 1250, dtype=torch.float64)
    disc = torch.ones(8, dtype=torch.float64)
    p = _cabi.MppiFusedParams(struct_size=C.sizeof(_cabi.MppiFusedParams), model=_cabi.MODEL_PENDULUM_MLP_ENSEMBLE,
                              dtype=_cabi.F64, K=64, T=8, nx=2, nu=1, u_per_command=1, lambda_=1.0, rollout_var_cost=1.0,
                              var_discount=disc.data_ptr(), model_weights=tab.data_ptr())
    info = _cabi.MppiLaunchInfo()
    for M in (0, 1, _cabi.MPPI_MAX_COPIES + 1, -1):
        p.rollout_samples = M
        assert lib.mppi_plan_create(C.byref(p), C.byref(C.c_void_p())) == -1, M
        assert lib.mppi_fused_query(C.byref(p), C.byref(info)) == -1, M
    p.rollout_samples = 4
    p.model_weights = None
    assert lib.mppi_plan_create(C.byref(p), C.byref(C.c_void_p())) == -1
    assert lib.mppi_fused_query(C.byref(p), C.byref(info)) == -1
    assert lib.mppi_rollout_states(C.byref(p), tab.data_ptr(), tab.data_ptr(), 0, 1, 8, tab.data_ptr(), None) == -1
    p.model_weights, p.var_discount = tab.data_ptr(), None
    assert lib.mppi_plan_create(C.byref(p), C.byref(C.c_void_p())) == -1
    # every other registered model keeps refusing rollout_samples > 1 as unsupported
    for model in (_cabi.MODEL_PENDULUM, _cabi.MODEL_PENDULUM_MLP):
        p.model, p.var_discount = model, disc.data_ptr()
        assert lib.mppi_plan_create(C.byref(p), C.byref(C.c_void_p())) == (-2 if model == _cabi.MODEL_PENDULUM else -1)


def _replay(case, nets):
    return OracleRunner(case, net_arrays(nets), MLP_ENSEMBLE)


def _replay_error(case, gold, nets):
    """Largest deviation of U and cost_total from a fixture over its closed loop, replayed with these networks."""
    run = _replay(case, nets)
    x, du, dc = torch.tensor(case["x0"], dtype=run.prob.dtype), 0.0, 0.0
    for step in range(case["steps"]):
        r = run.step(x, run.stream.next_z())
        du = max(du, float(np.abs(r["U"].numpy() - gold[f"U_{step}"]).max()))
        dc = max(dc, float(np.abs(r["cost_total"].numpy() - gold[f"cost_total_{step}"]).max()))
        x = run.advance(x, r["action"])
    return du, dc


@pytest.mark.parametrize("name", sorted(MLP_ENSEMBLE_CASES))
def test_fixture_detects_permuted_networks(name):
    """The networks differ enough that a twin with its networks in another order misses every fixture by orders of
    magnitude more than any tolerance (<= 5e-4).  A command's costs are symmetric in the copies (mean and variance over
    them), so a relabelling shows in the closed loop, whose simulated system is network 0; a twin that steps every copy
    through one network already misses the first command."""
    torch.set_num_threads(1)
    case, gold = load(name)
    nets = load_nets(case, gold)
    du, dc = _replay_error(case, gold, nets[1:] + nets[:1])
    assert du > 5e-3 and dc > 1e-2, (du, dc)
    run = _replay(case, [nets[0]] * case["M"])
    r = run.step(torch.tensor(case["x0"], dtype=run.prob.dtype), run.stream.next_z())
    assert float(np.abs(r["cost_total"].numpy() - gold["cost_total_0"]).max()) > 1e-2
    assert float(np.abs(r["U"].numpy() - gold["U_0"]).max()) > 5e-3
