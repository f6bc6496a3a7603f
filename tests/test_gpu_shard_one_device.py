"""GPU: sharded controllers (process_group=, K split over ranks) with every rank a process on ONE device.

With exchange="nccl" each rank's kernel runs the single-GPU tail, exports one (beta, eta, V) record, Python all-gathers
the records (here over a gloo group on loopback) and `mppi_apply_partials` finishes the command.  No kernel waits on
another rank, so two, three or eight processes sharing one GPU run that route end to end: the global sample index
(k_offset + k) in sampling and rollout, the grid planned for the largest shard (K_geom, idle lanes on the last shard),
the record export and `apply_partials_kernel` per variant, and the host code that slices injected noise, per-sample
start states and the SpecificActionSampler rows per shard.  Only the in-kernel NVLink exchange (exchange="p2p") needs
one GPU per rank: it is refused here, and tests/test_gpu_multi.py covers it on two GPUs.

The ranks are spawned once per (world, environment mode); each runs its list of jobs and hands back plain numpy
results, and the tests below compare them, per job, with the golden fixtures, the fp64/fp32 oracle or the unsharded
controller, which the parent process builds itself."""
import os
import socket
import traceback
from datetime import timedelta

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# (MPPI_B200_SPLIT_COST, MPPI_B200_CLUSTER): the default first.  The engine reads both when a controller is built / its
# plan is made, so the rank sets them before it builds anything.
MODES = [("1", "8"), ("0", "8"), ("1", "1"), ("0", "1")]
DEFAULT = MODES[0]
WORLDS = (2, 3)
GLOO_TIMEOUT_S = 120


# ----------------------------------------------------------------------------------------------------------------------
# jobs: each builds its controller with process_group=pg (None: the unsharded controller) and returns numpy results
# ----------------------------------------------------------------------------------------------------------------------
def _np(t):
    return None if t is None else t.detach().cpu().numpy().copy()


def _snap(c, a, **extra):
    """One command's results on this rank."""
    out = dict(U=_np(c.U), action=_np(a), cost=_np(c.cost_total), span=(c._k_offset, c._K_local))
    if hasattr(c, "theta"):
        out["theta"] = _np(c.theta)
    if hasattr(c, "action_sequence"):
        out["A"] = _np(c.action_sequence)
    out.update({k: _np(v) if torch.is_tensor(v) else v for k, v in extra.items()})
    return out


def _resync(c, step):
    """The next command starts from a nominal the sharded and the unsharded controller share: their fp64 record
    combines run in different orders, so the nominals they update may differ in the last bit (bounded in the test), and
    the next costs would differ with them."""
    g = torch.Generator().manual_seed(1000 + step)

    def draw(*shape):
        return (torch.randn(*shape, generator=g, dtype=torch.float64) * 0.3).to(c.dtype)
    c.U = draw(c.T, c.nu)
    if hasattr(c, "theta"):
        c.theta = draw(c.num_support_pts, c.nu)
    if hasattr(c, "action_sequence"):
        c.action_sequence = draw(c.T, c.nu)


def _kw(pg):
    return dict(process_group=pg, exchange="nccl")


def _pendulum(pg, K, T, dtype, U0=None, seed=7, **kw):
    import pytorch_mppi_b200 as eng
    pend = eng.Pendulum()
    args = dict(_kw(pg), **kw)
    return eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0, dtype=dtype), num_samples=K, horizon=T,
                    device="cuda", u_min=torch.tensor(-2.0, dtype=dtype), u_max=torch.tensor(2.0, dtype=dtype),
                    U_init=U0, rng_seed=seed, **args)


def _nav(pg, variant, K, T, dtype, stepped=False, **kw):
    """Toy2D navigation (LinearPoint with a hill and a terminal cost) under MPPI / SMPPI / KMPPI."""
    import pytorch_mppi_b200 as eng
    nav = eng.LinearPoint.toy2d_nav()
    dyn, cost, term = nav.dynamics, nav.running_cost, nav.terminal_cost
    if stepped:
        dyn, cost, term = (lambda s, a: nav.dynamics(s, a)), (lambda s, a: nav.running_cost(s, a)), \
            (lambda s, a: nav.terminal_cost(s, a))
    g = torch.Generator().manual_seed(K + T)
    args = dict(num_samples=K, horizon=T, device="cuda", terminal_state_cost=term,
                u_max=torch.tensor([1.0, 1.0], dtype=dtype), **_kw(pg))
    args.update(kw)
    sigma = torch.eye(2, dtype=dtype)
    if variant == "smppi":
        return eng.SMPPI(dyn, cost, 2, sigma, w_action_seq_cost=5.0, action_max=torch.tensor([1.0, 1.0], dtype=dtype),
                         **args)
    args.setdefault("U_init", (torch.randn(T, 2, generator=g) * 0.3).to(dtype))
    if variant == "kmppi":
        return eng.KMPPI(dyn, cost, 2, sigma, num_support_pts=5, kernel=eng.RBFKernel(sigma=2), **args)
    return eng.MPPI(dyn, cost, 2, sigma, **args)


def job_philox(pg, variant, dtype):
    """Philox noise keyed by the global sample index, two commands; the normals each command used are recorded."""
    dt = getattr(torch, dtype)
    c = _nav(pg, variant, 333, 12, dt, rng_seed=3)
    c.record_noise(True)
    steps = []
    for x in ([-3.0, -2.0], [-2.5, -1.5]):
        a = c.command(x)
        steps.append(_snap(c, a, z=c.z_used))
        _resync(c, len(steps))
    return steps


def job_torch_rng(pg):
    """rng="torch": the normals of torch.randn(K, T, nu, device="cuda") after torch.manual_seed(5)."""
    c = _pendulum(pg, 333, 12, torch.float32, U0=torch.zeros(12, 1), rng="torch")
    c.record_noise(True)
    torch.manual_seed(5)
    a = c.command([3.0, 0.5])
    return [_snap(c, a, z=c.z_used)]


def job_start_states(pg, route):
    """A (K, nx) batch of start states, one per sample: each rank rolls out from its own rows."""
    import pytorch_mppi_b200 as eng
    K, T, dt = 333, 12, torch.float64
    if route == "fused":
        c = _pendulum(pg, K, T, dt, U0=torch.linspace(-1, 1, T, dtype=dt).view(T, 1))
    else:
        pend = eng.Pendulum()
        c = eng.MPPI(lambda s, a: pend.dynamics(s, a), lambda s, a: pend.running_cost(s, a), 2,
                     torch.tensor(10.0, dtype=dt), num_samples=K, horizon=T, device="cuda",
                     u_max=torch.tensor(2.0, dtype=dt), U_init=torch.linspace(-1, 1, T, dtype=dt).view(T, 1),
                     rng_seed=7, **_kw(pg))
    g = torch.Generator().manual_seed(9)
    steps = []
    for _ in range(2):
        x = (torch.rand(K, 2, generator=g, dtype=dt) * 4 - 2).cuda()
        a = c.command(x)
        steps.append(_snap(c, a))
        _resync(c, len(steps))
    return steps


def job_upc_noshift(pg):
    """u_per_command = 2, a command without the shift, then one with it."""
    c = _nav(pg, "mppi", 200, 10, torch.float64, rng_seed=4, u_per_command=2)
    steps = []
    for shift in (False, True):
        a = c.command([-3.0, -2.0], shift_nominal_trajectory=shift)
        steps.append(_snap(c, a))
        _resync(c, len(steps))
    return steps


def job_change_horizon(pg, variant):
    """change_horizon up and down between commands: the nominal and the exported record change size."""
    c = _nav(pg, variant, 200, 10, torch.float64, rng_seed=5)
    steps = []
    for T in (10, 14, 6):
        if T != c.T:
            c.change_horizon(T)
        a = c.command([-3.0, -2.0])
        steps.append(_snap(c, a))
        _resync(c, len(steps))
    return steps


def job_random_nominal(pg):
    """U_init=None and reset(): one draw for the whole controller (rank 0's), whatever the ranks' torch seeds."""
    import torch.distributed as dist
    rank = dist.get_rank(pg) if pg is not None else 0
    torch.manual_seed(100 + rank)
    c = _pendulum(pg, 1000, 12, torch.float32, U0=None)
    U0 = _np(c.U)
    a = c.command([3.0, 0.5])
    s = _snap(c, a, U0=U0)
    torch.manual_seed(200 + rank)
    c.reset()
    s["U_reset"] = _np(c.U)
    return [s]


def job_rollouts_host(pg):
    """get_rollouts after a command, and command_host (which takes command() on this route)."""
    c = _pendulum(pg, 1000, 15, torch.float64, U0=torch.zeros(15, 1))
    a = c.command([3.0, 0.5])
    s0 = _snap(c, a, rollouts=c.get_rollouts(torch.tensor([3.0, 0.5], dtype=torch.float64), num_rollouts=3))
    _resync(c, 1)
    h = c.command_host([2.9, 0.4])
    s1 = _snap(c, h, host_is_cpu=not h.is_cuda)
    return [s0, s1]


def job_step_dependent(pg):
    """A step-dependent CudaModel whose parameters change between commands (set_params)."""
    import pytorch_mppi_b200 as eng
    from tests import step_models as um
    m = um.step_dependent_user_model()
    dt, T = torch.float64, 20
    c = eng.MPPI(m.dynamics, m.running_cost, 2, torch.tensor(1.0, dtype=dt), num_samples=333, horizon=T,
                 U_init=torch.zeros(T, 1, dtype=dt), u_max=torch.tensor(3.0, dtype=dt), terminal_state_cost=m.terminal_cost,
                 step_dependent_dynamics=True, device="cuda", rng_seed=6, **_kw(pg))
    assert c._model is m
    steps = []
    p = list(um.SD_PARAMS)
    for step in range(3):
        if step == 2:
            p[3] += 0.25
            m.set_params(p)
        a = c.command([0.1 * step, -0.05 * step])
        steps.append(_snap(c, a))
        _resync(c, len(steps))
    return steps


def job_copies(pg):
    """CudaModel(copies=3) with rollout_samples=3: every rank rolls out all copies of its samples."""
    import pytorch_mppi_b200 as eng
    from tests import ensemble_models as em
    dt, K, T = torch.float64, 333, 16
    m = em.pendulum_ensemble(3, K)
    c = eng.MPPI(m.dynamics, m.running_cost, 2, torch.tensor(1.0, dtype=dt), num_samples=K, horizon=T, device="cuda",
                 U_init=torch.zeros(T, 1, dtype=dt), u_max=torch.tensor(2.0, dtype=dt), terminal_state_cost=m.terminal_cost,
                 rollout_samples=3, rollout_var_cost=0.5, rollout_var_discount=0.9, rng_seed=8, **_kw(pg))
    assert c._model is m
    steps = []
    for x in ([2.5, 0.5], [2.4, 0.3]):
        a = c.command(x)
        steps.append(_snap(c, a))
        _resync(c, len(steps))
    return steps


def job_costmap(pg):
    """A CudaModel reading device tensors (costmap lookup, reference path)."""
    import pytorch_mppi_b200 as eng
    from tests import tensor_models as tm
    dt, K, T = torch.float64, 333, 20
    m = tm.nav_model(tm.make_costmap(), tm.make_path(T))
    c = eng.MPPI(m.dynamics, m.running_cost, 2, torch.eye(2, dtype=dt), num_samples=K, horizon=T, device="cuda",
                 U_init=torch.zeros(T, 2, dtype=dt), u_max=torch.full((2,), 3.0, dtype=dt), step_dependent_dynamics=True,
                 rng_seed=9, **_kw(pg))
    assert c._model is m
    steps = []
    for x in ([-1.2, -0.9], [-1.1, -0.8]):
        a = c.command(x)
        steps.append(_snap(c, a))
        _resync(c, len(steps))
    return steps


def job_sampler(pg, K):
    """SpecificActionSampler rows behind the null action, across shard boundaries, with a specific_dynamics that
    overwrites its rows' next state through `self.slice` (the hook's contract)."""
    import pytorch_mppi_b200 as eng
    dt, T = torch.float64, 6
    nav = eng.LinearPoint.unit_test_env()
    seen = []

    class Sampler(eng.SpecificActionSampler):
        def sample_trajectories(self, state, info):
            return 0.3 * torch.linspace(-1, 1, 3 * T * 2, dtype=dt, device=state.device).reshape(3, T, 2)

        def specific_dynamics(self, next_state, state, action, t):
            seen.append((self.start_idx, self.end_idx))
            out = next_state.clone()
            out[:, self.slice] = 0.5 * next_state[:, self.slice] + 1.0
            return out

    c = eng.MPPI(lambda s, a: nav.dynamics(s, a), lambda s, a: nav.running_cost(s, a), 2, torch.eye(2, dtype=dt),
                 num_samples=K, horizon=T, device="cuda", U_init=torch.zeros(T, 2, dtype=dt), sample_null_action=True,
                 specific_action_sampler=Sampler(), rng_seed=10, **_kw(pg))
    assert c._model is None
    steps = []
    for x in ([-3.0, -2.0], [-2.0, -1.0]):
        a = c.command(x)
        steps.append(_snap(c, a, registered=seen[-1]))
        _resync(c, len(steps))
    return steps


def job_small(pg):
    """The smallest useful shard: K = 64 over up to MPPI_MAX_RANKS ranks."""
    c = _pendulum(pg, 64, 10, torch.float64, U0=torch.zeros(10, 1), seed=12)
    steps = []
    for x in ([3.0, 0.5], [2.9, 0.6]):
        a = c.command(x)
        steps.append(_snap(c, a))
        _resync(c, len(steps))
    return steps


COMPARE_JOBS = {
    **{f"philox_{v}_{d}": (job_philox, dict(variant=v, dtype=d))
       for v in ("mppi", "smppi", "kmppi") for d in ("float32", "float64")},
    "torch_rng": (job_torch_rng, {}),
    "start_states_fused": (job_start_states, dict(route="fused")),
    "start_states_stepped": (job_start_states, dict(route="stepped")),
    "upc2_noshift": (job_upc_noshift, {}),
    "change_horizon_mppi": (job_change_horizon, dict(variant="mppi")),
    "change_horizon_smppi": (job_change_horizon, dict(variant="smppi")),
    "change_horizon_kmppi": (job_change_horizon, dict(variant="kmppi")),
    "random_nominal": (job_random_nominal, {}),
    "rollouts_host": (job_rollouts_host, {}),
    "step_dependent": (job_step_dependent, {}),
    "copies3": (job_copies, {}),
    "costmap": (job_costmap, {}),
    "sampler_k7": (job_sampler, dict(K=7)),
    "sampler_k128": (job_sampler, dict(K=128)),
}
# the per-sample arithmetic of these runs in kernels the grid does not change (DESIGN §4.1): the concatenated costs are
# the unsharded controller's bit for bit.  The stepped route's rollouts are torch ops on (K_local, nx) batches.
STEPPED_JOBS = {"start_states_stepped", "sampler_k7", "sampler_k128"}


def job_tail(pg, K, T, commands):
    """A C2- / C5-sized problem per shard, fp32, noise recorded for the oracle."""
    g = torch.Generator().manual_seed(K)
    U0 = torch.randn(T, 1, generator=g) * 2
    c = _pendulum(pg, K, T, torch.float32, U0=U0.clone())
    c.record_noise(True)
    steps = []
    x = [3.0, 0.5]
    for _ in range(commands):
        U_before = _np(c.U)
        a = c.command(x)
        i = c.launch_info
        steps.append(_snap(c, a, z=c.z_used, U_before=U_before, x=np.array(x),
                           info=dict(ll_tail=i.ll_tail, cluster_size=i.cluster_size, split_cost=i.split_cost,
                                     threads_per_sample=i.threads_per_sample, grid_blocks=i.grid_blocks,
                                     xchg_records=i.xchg_records)))
        x = [x[0] + 0.05 * x[1], x[1] + 0.1 * float(a.reshape(-1)[0])]
    return steps


def _tail_jobs(world):
    jobs = {}
    for base, T, commands, tag in ((16384, 30, 2, "c2"), (131072, 50, 1, "c5")):
        for extra in (0, 1):
            K = base * world + extra
            jobs[f"{tag}_K{K}"] = (job_tail, dict(K=K, T=T, commands=commands))
    return jobs


# ---- golden fixtures, sharded ----------------------------------------------------------------------------------------
def _sharded_route(fam, case, route):
    """The single-controller replay's routes a fixture also runs sharded on: fused, the stepped route at K <= 2048 (or
    for the MLP), and the config-4 MLP's bf16x3 kernel with the exact tanh.  Not the copy-offset CudaModel, the MUFU
    tanh or the ensembles' tensor-core kernel."""
    if route == "stepped":
        return case["K"] <= 2048 or case["model"]["kind"] == "pendulum_mlp"
    return route == "fused" or (route == "wgmma" and fam.name == "base")


def _fixture_ids():
    """(world, name, route) of every single-controller fixture a sharded controller accepts (K >= world)."""
    from tests.golden.replay import FAMILIES
    return [(w, name, route) for w in WORLDS for fam in FAMILIES for name, case in sorted(fam.cases.items())
            if "N" not in case and case["K"] >= w for route in fam.routes(name, case) if _sharded_route(fam, case, route)]


def job_fixture(pg, name, route):
    """Replays a fixture at its states with its draws; after each command the nominal is the fixture's (replay.py)."""
    import torch.distributed as dist
    from pytorch_mppi_b200.distributed import shard_bounds
    from tests.golden.replay import FAMILY, OracleRunner, load
    case, gold = load(name)
    fam = FAMILY[name]
    run = OracleRunner(case, gold, fam)
    k0, n = shard_bounds(case["K"], dist.get_rank(pg), dist.get_world_size(pg))
    c = fam.engine(case, gold, run.stream.U0, route, copy_rows=n, **_kw(pg))
    lock = fam.lockable(case)
    steps = []
    for step in range(case["steps"]):
        c.inject_noise(run.stream.next_z())
        a = c.command(torch.from_numpy(gold[f"x_{step}"]))
        extra = dict(omega=c.omega, noise=c.noise, pa=c.perturbed_action) if lock else {}
        steps.append(_snap(c, a, **extra))
        c.U = torch.from_numpy(gold[f"U_{step}"])
        for key, attr in (("theta", "theta"), (fam.smooth_key, "action_sequence")):
            if f"{key}_{step}" in gold:
                setattr(c, attr, torch.from_numpy(gold[f"{key}_{step}"]))
    return steps


def _fixture_jobs(world):
    return {f"fixture_{name}_{route}": (job_fixture, dict(name=name, route=route))
            for w, name, route in _fixture_ids() if w == world}


# ---- refusals --------------------------------------------------------------------------------------------------------
def job_refusals(pg):
    """Every refusal of a sharded controller, before anything launches: {name: (exception type, U unchanged)}."""
    import pytorch_mppi_b200 as eng
    out = {}

    def attempt(name, build, act=None):
        c = None
        try:
            c = build()
            if act is None:
                out[name] = ("none", True, "")
                return
            U = c.U.clone()
            act(c)
            out[name] = ("none", bool(torch.equal(c.U, U)), "")
        except Exception as e:      # noqa: BLE001 - the type is what the test checks
            torch.cuda.synchronize()
            out[name] = (type(e).__name__, c is None or bool(torch.equal(c.U, U)), str(e)[:300])

    pend = eng.Pendulum()
    nav = eng.LinearPoint.toy2d_nav()
    attempt("k_below_world", lambda: _pendulum(pg, 1, 10, torch.float32))
    attempt("batched", lambda: eng.MPPI_Batched(pend.dynamics, pend.running_cost, 2, torch.tensor(1.0), num_envs=2,
                                                  num_samples=64, horizon=10, device="cuda", process_group=pg))
    attempt("tile_global", lambda: _pendulum(pg, 64, 10, torch.float32, tile_memory="global"))
    attempt("tile_auto", lambda: _pendulum(pg, 64, 10, torch.float32, tile_memory="auto"))
    attempt("exchange_name", lambda: _pendulum(pg, 64, 10, torch.float32, U0=torch.zeros(10, 1), exchange="nccI"))
    attempt("T_nu_fused", lambda: _pendulum(pg, 64, 1025, torch.float32, U0=torch.zeros(1025, 1)),
            lambda c: c.command([3.0, 0.5]))
    attempt("T_nu_stepped", lambda: eng.MPPI(lambda s, a: nav.dynamics(s, a), lambda s, a: nav.running_cost(s, a), 2,
                                              torch.eye(2), num_samples=64, horizon=513, device="cuda",
                                              U_init=torch.zeros(513, 2), rng_seed=1, **_kw(pg)),
            lambda c: c.command([-3.0, -2.0]))
    attempt("closed_loop", lambda: _pendulum(pg, 64, 10, torch.float32, U0=torch.ones(10, 1)),
            lambda c: c.run_closed_loop(torch.tensor([3.0, 0.5], device="cuda"), 3))
    attempt("resident", lambda: _pendulum(pg, 64, 10, torch.float32, U0=torch.ones(10, 1)),
            lambda c: c.start_resident())
    # the in-kernel exchange with two ranks on one device: refused before a mailbox exists or a kernel runs
    attempt("p2p_same_device", lambda: eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), num_samples=64,
                                                 horizon=10, device="cuda", U_init=torch.ones(10, 1), rng_seed=1,
                                                 process_group=pg, exchange="p2p"),
            lambda c: c.command([3.0, 0.5]))
    return [out]


REFUSALS = {"k_below_world": "ValueError", "batched": "TypeError", "tile_global": "ValueError", "tile_auto": "ValueError",
            "exchange_name": "ValueError", "T_nu_fused": "ValueError", "T_nu_stepped": "ValueError",
            "closed_loop": "ValueError", "resident": "MppiLibraryError", "p2p_same_device": "ValueError"}


# ----------------------------------------------------------------------------------------------------------------------
# the ranks
# ----------------------------------------------------------------------------------------------------------------------
def _rank_main(rank, world, port, mode, jobs, out):
    os.environ["MPPI_B200_SPLIT_COST"], os.environ["MPPI_B200_CLUSTER"] = mode
    os.environ["MPPI_B200_XCHG_TIMEOUT_S"] = "0.3"      # a p2p exchange that slipped through the refusal ends fast
    import torch.distributed as dist
    torch.cuda.set_device(0)
    torch.set_num_threads(1)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world,
                            timeout=timedelta(seconds=GLOO_TIMEOUT_S))
    try:
        for job_id, (fn, kw) in jobs.items():
            try:
                res = fn(dist.group.WORLD, **kw)
            except Exception:       # noqa: BLE001 - reported by the job's test
                res = {"error": traceback.format_exc()}
            torch.cuda.synchronize()
            out[f"{job_id}/{rank}"] = res
    finally:
        dist.destroy_process_group()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _jobs(world, mode):
    jobs = dict(_tail_jobs(world))
    if mode == DEFAULT:
        jobs.update(_fixture_jobs(world))
        jobs.update(COMPARE_JOBS)
        if world == 2:
            jobs["refusals"] = (job_refusals, {})
    return jobs


class _Runs:
    """Results per (world, mode), spawned on first use; unsharded results of the compare jobs, made in this process."""

    def __init__(self):
        self.runs, self.single = {}, {}

    def unsharded(self, job_id):
        if job_id not in self.single:
            fn, kw = COMPARE_JOBS[job_id] if job_id in COMPARE_JOBS else (job_small, {})
            self.single[job_id] = fn(None, **kw)
            torch.cuda.synchronize()
        return self.single[job_id]

    def get(self, world, mode, jobs=None):
        key = (world, mode)
        if key not in self.runs:
            import torch.multiprocessing as mp
            jobs = jobs or _jobs(world, mode)
            for job_id in jobs:          # the parent's own controllers first: NVRTC cubins cached before the ranks start
                if job_id in COMPARE_JOBS or job_id == "small":
                    self.unsharded(job_id)
            with mp.Manager() as mgr:
                out = mgr.dict()
                try:
                    mp.spawn(_rank_main, args=(world, _free_port(), mode, jobs, out), nprocs=world, join=True)
                    self.runs[key] = dict(out)
                except Exception as e:   # noqa: BLE001 - a rank that died: every test of this run reports it, none reruns it
                    self.runs[key] = e
        if isinstance(self.runs[key], Exception):
            raise RuntimeError(f"the ranks of world {world}, mode {key[1]} failed") from self.runs[key]
        return self.runs[key]

    def ranks(self, world, mode, job_id, jobs=None):
        res = self.get(world, mode, jobs)
        got = [res.get(f"{job_id}/{r}") for r in range(world)]
        for r, g in enumerate(got):
            assert g is not None, f"rank {r} returned nothing for {job_id}"
            assert not (isinstance(g, dict) and "error" in g), f"rank {r}, {job_id}:\n{g['error']}"
        return got


@pytest.fixture(scope="module")
def runs():
    return _Runs()


def _record(key, err):
    """Worst errors per family and dtype, in tests/_reports/shard_one_device_errors.json."""
    from tests import reports
    reports.worst("shard_one_device_errors.json", key, err)


def _cat(ranks, step, key):
    return np.concatenate([r[step][key] for r in ranks])


def _spans_partition(ranks, K):
    spans = [r[0]["span"] for r in ranks]
    assert spans[0][0] == 0 and all(a[0] + a[1] == b[0] for a, b in zip(spans, spans[1:]))
    assert spans[-1][0] + spans[-1][1] == K


def _same_on_every_rank(ranks, step, keys=("U", "action", "theta", "A")):
    for key in keys:
        if key in ranks[0][step]:
            for r in ranks[1:]:
                assert np.array_equal(r[step][key], ranks[0][step][key]), (key, step)


# ----------------------------------------------------------------------------------------------------------------------
# (a) every fixture of every family, sharded, against the fixture and the oracle in lock step
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world,name,route", _fixture_ids())
def test_sharded_fixture_replay(runs, world, name, route):
    from tests.golden.engine import ORACLE_TOL
    from tests.golden.replay import FAMILY, OracleRunner, load
    ranks = runs.ranks(world, DEFAULT, f"fixture_{name}_{route}")
    case, gold = load(name)
    fam = FAMILY[name]
    run = OracleRunner(case, gold, fam)
    tol = fam.u_tol(name, case, route)
    _spans_partition(ranks, case["K"])
    otol = ORACLE_TOL[case["dtype"]]
    worst = 0.0
    for step in range(case["steps"]):
        z = run.stream.next_z()
        x = torch.from_numpy(gold[f"x_{step}"])
        _same_on_every_rank(ranks, step)
        got = ranks[0][step]
        err = float(np.abs(got["U"] - gold[f"U_{step}"]).max())
        worst = max(worst, err)
        assert err <= tol, f"step {step}: |U - U_ref| = {err:.3e} > {tol}"
        assert got["action"].shape == gold[f"action_{step}"].shape
        assert float(np.abs(got["action"] - gold[f"action_{step}"]).max()) <= tol
        for key, attr in (("theta", "theta"), (fam.smooth_key, "A")):
            if f"{key}_{step}" in gold:
                assert float(np.abs(got[attr] - gold[f"{key}_{step}"]).max()) <= tol, key
        if f"cost_total_{step}" in gold:
            fam.check_costs(name, case, route, _cat(ranks, step, "cost"), gold[f"cost_total_{step}"], tol)
        if "omega" in got:
            r = run.step(x, z)
            om = _cat(ranks, step, "omega")
            assert abs(om.sum() - 1.0) < 1e-5
            np.testing.assert_allclose(om, r["omega"].numpy(), atol=otol, rtol=0)
            np.testing.assert_allclose(_cat(ranks, step, "noise"), r["noise"].numpy(), atol=otol, rtol=0)
            pa = _cat(ranks, step, "pa")
            np.testing.assert_allclose(pa, r["perturbed_action"].numpy(), atol=otol, rtol=0)
            if f"pa_head_{step}" in gold:
                n = gold[f"pa_head_{step}"].shape[0]
                np.testing.assert_allclose(pa[:n], gold[f"pa_head_{step}"], atol=otol, rtol=0)
            run.U = torch.from_numpy(gold[f"U_{step}"]).clone()
            if case["variant"] == "smppi":
                run.A = torch.from_numpy(gold[f"{fam.smooth_key}_{step}"]).clone()
            if case["variant"] == "kmppi":
                run.theta = torch.from_numpy(gold[f"theta_{step}"]).clone()
    _record(f"fixture/{fam.name}/{case['dtype']}" + ("/wgmma" if route == "wgmma" else ""), worst)


# ----------------------------------------------------------------------------------------------------------------------
# (b, d) sharded against unsharded
# ----------------------------------------------------------------------------------------------------------------------
def _u_tol(U):
    """fp64: 1e-12; fp32: 4 ulp of max|U| — only the order of the fp64 record combines differs."""
    if U.dtype == np.float64:
        return 1e-12
    return 4 * float(np.spacing(np.float32(max(float(np.abs(U).max()), 1e-30))))


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("job_id", sorted(COMPARE_JOBS))
def test_sharded_equals_unsharded(runs, world, job_id):
    ranks = runs.ranks(world, DEFAULT, job_id)
    one = runs.unsharded(job_id)
    for step, ref in enumerate(one):
        K = ref["cost"].shape[-1]
        _spans_partition(ranks, K)
        _same_on_every_rank(ranks, step)
        got = ranks[0][step]
        cost = _cat(ranks, step, "cost")
        if job_id in STEPPED_JOBS:
            np.testing.assert_allclose(cost, ref["cost"], rtol=1e-13, atol=0)
        else:
            assert np.array_equal(cost, ref["cost"]), (step, float(np.abs(cost - ref["cost"]).max()))
        if "z" in ref:
            assert np.array_equal(_cat(ranks, step, "z"), ref["z"]), step
        for key in ("U", "action", "theta", "A"):
            if key in ref:
                err = float(np.abs(got[key] - ref[key]).max())
                _record(f"unsharded/{job_id}/{key}", err)
                assert err <= _u_tol(ref[key]), (step, key, err)
        if "rollouts" in ref:
            np.testing.assert_allclose(got["rollouts"], ref["rollouts"], rtol=0, atol=1e-12)
    if job_id == "torch_rng":
        torch.manual_seed(5)
        want = torch.randn(one[0]["cost"].shape[0], 12, 1, device="cuda").cpu().numpy()
        assert np.array_equal(_cat(ranks, 0, "z"), want)
    if job_id == "random_nominal":
        for key in ("U0", "U_reset"):
            for r in ranks:
                assert np.array_equal(r[0][key], one[0][key]), key        # rank 0's draw, on every rank
    if job_id == "rollouts_host":
        assert all(r[1]["host_is_cpu"] for r in ranks)
    if job_id.startswith("sampler"):
        # global rows [1, 4) (behind the null action) in each rank's local indices
        for r in ranks:
            k0, n = r[0]["span"]
            lo = min(max(1 - k0, 0), n)
            assert r[0]["registered"] == (lo, max(lo, min(4 - k0, n))), (r[0]["span"], r[0]["registered"])


def test_world_of_eight_ranks(runs):
    """MPPI_MAX_RANKS processes on one device: K = 64 in shards of 8."""
    world = 8
    ranks = runs.ranks(world, DEFAULT, "small", jobs={"small": (job_small, {})})
    one = runs.unsharded("small")
    for step, ref in enumerate(one):
        _spans_partition(ranks, 64)
        _same_on_every_rank(ranks, step)
        assert np.array_equal(_cat(ranks, step, "cost"), ref["cost"])
        assert float(np.abs(ranks[0][step]["U"] - ref["U"]).max()) <= 1e-12


# ----------------------------------------------------------------------------------------------------------------------
# (c) tails and geometry on shards, against the oracle fed the recorded noise
# ----------------------------------------------------------------------------------------------------------------------
def _tail_ids():
    return [pytest.param(w, m, j, id=f"world{w}-split{m[0]}-cluster{m[1]}-{j}")
            for w in WORLDS for m in MODES for j in sorted(_tail_jobs(w))]


@pytest.mark.parametrize("world,mode,job_id", _tail_ids())
def test_sharded_tail_against_oracle(runs, world, mode, job_id):
    from oracle import mppi_oracle as orc
    ranks = runs.ranks(world, mode, job_id)
    fn, kw = _tail_jobs(world)[job_id]
    K, T = kw["K"], kw["T"]
    _spans_partition(ranks, K)
    prob = orc.Problem(dynamics=orc.PendulumModel(numpy_sin=False).dynamics,
                       running_cost=orc.PendulumModel(numpy_sin=False).running_cost, nx=2,
                       noise_sigma=torch.tensor(10.0), K=K, T=T, lambda_=1.0, u_min=torch.tensor(-2.0),
                       u_max=torch.tensor(2.0))
    split, cluster = mode
    for step in range(kw["commands"]):
        _same_on_every_rank(ranks, step)
        for r in ranks:
            info = r[step]["info"]
            assert info["ll_tail"] == 0, info                  # the export route's tail, not the single-GPU LL tail
            assert 1 <= info["cluster_size"] <= int(cluster), info
            if split == "0":
                assert info["split_cost"] == 0, info
            elif job_id.startswith("c2"):
                assert info["split_cost"] == 1, info
        got = ranks[0][step]
        z = torch.from_numpy(_cat(ranks, step, "z")).view(K, T, 1)
        r = orc.mppi_command(prob, torch.from_numpy(got["U_before"]), torch.from_numpy(got["x"]).float(), z)
        cost = _cat(ranks, step, "cost")
        np.testing.assert_allclose(cost, r["cost_total"].numpy(), rtol=5e-6, atol=5e-6)
        # The update is checked against fp64 arithmetic, not against the fp32 oracle's own update: that one sums 1e5
        # weighted samples in fp32 in an order set by the CPU's thread count, and moves by ~1e-5 with it.  The
        # reference is the softmin of the engine's costs (checked just above) applied to the oracle's noise, in fp64:
        # it leaves only the engine's tail — per-warp sums in fp32, records combined in fp64 across warps, CTAs and
        # ranks, the result rounded to fp32 — and any sample the records count that the shards do not hold.
        U64 = _fp64_update(r["U_before"], cost, r["noise"])
        err = float((torch.from_numpy(got["U"]).double() - U64).abs().max())
        _record(f"tail/{job_id[:2]}/f32", err)
        _record(f"tail/{job_id[:2]}/f32_oracle_costs",
                float((torch.from_numpy(got["U"]).double() - _fp64_update(r["U_before"], r["cost_total"].numpy(), r["noise"])).abs().max()))
        # 4 ulp of max|U|, as against the unsharded controller (measured on H100: 2.2e-7, about one ulp; the same
        # update from the oracle's costs, whose sines may differ in the last bit, lies ~1e-5 away and is only reported)
        assert err <= _u_tol(got["U"]), err


def _fp64_update(U_before, cost, noise, lambda_=1.0):
    """U_before + sum_k omega_k noise_k with omega the softmin of `cost`, all in fp64 (mppi.py:254-270)."""
    c = torch.as_tensor(cost).double()
    w = torch.exp(-(c - c.min()) / lambda_)
    return U_before.double() + torch.einsum("k,ktn->tn", w / w.sum(), noise.double())


# ----------------------------------------------------------------------------------------------------------------------
# (e) refusals
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(REFUSALS))
def test_sharded_refusals(runs, name):
    ranks = runs.ranks(2, DEFAULT, "refusals")
    for r in ranks:
        kind, unchanged, msg = r[0][name]
        assert kind == REFUSALS[name], (name, kind, msg)
        assert unchanged, name
