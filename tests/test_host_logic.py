"""CPU: host-side logic — model registry resolution, torch model definitions vs the oracle,
K-sharding arithmetic, cross-rank combination (incl. a world_size-2 gloo run), Philox oracle KATs."""
import os

import numpy as np
import pytest
import torch

import pytorch_mppi_b200 as eng
from oracle import mppi_oracle as orc
from oracle import philox_oracle as po
from pytorch_mppi_b200.distributed import combine_partials, shard_bounds
from pytorch_mppi_b200.models import resolve_fused_model


def test_registry_resolution():
    pend = eng.Pendulum()
    assert resolve_fused_model(pend.dynamics, pend.running_cost, None) is pend
    assert resolve_fused_model(lambda s, a: pend.dynamics(s, a), pend.running_cost, None) is None
    other = eng.Pendulum()
    assert resolve_fused_model(pend.dynamics, other.running_cost, None) is None
    nav = eng.LinearPoint.toy2d_nav()
    assert resolve_fused_model(nav.dynamics, nav.running_cost, nav.terminal_cost) is nav
    assert resolve_fused_model(nav.dynamics, nav.running_cost, None) is None          # terminal term would differ
    lin = eng.LinearPoint.unit_test_env()
    assert resolve_fused_model(lin.dynamics, lin.running_cost, None) is lin
    assert resolve_fused_model(lin.dynamics, lin.running_cost, lambda s, a: 0) is None
    assert len(nav.param_blob()) <= 48 and len(pend.param_blob()) == 7


def test_subclass_overriding_a_plugin_takes_the_stepped_route():
    """A user subclass of a registered model that overrides dynamics / running_cost in Python is not the compiled
    model any more: its bound methods must NOT resolve to the fused route (the override would be silently ignored)."""
    class MyPendulum(eng.Pendulum):
        def dynamics(self, state, action):
            return super().dynamics(state, action) * 0.5

    class MyCost(eng.Pendulum):
        def running_cost(self, state, action):
            return super().running_cost(state, action) + 1.0

    class Plain(eng.Pendulum):          # no override: still the compiled model
        pass

    for cls, fused in ((MyPendulum, False), (MyCost, False), (Plain, True)):
        m = cls()
        assert (resolve_fused_model(m.dynamics, m.running_cost, None) is m) == fused, cls.__name__

    class MyNav(eng.LinearPoint):
        def terminal_cost(self, states, actions):
            return 2 * super().terminal_cost(states, actions)
    nav = MyNav(B=[[0.5, 0.0], [0.0, -0.5]], goal=[2.0, 2.0], terminal_scale=10.0)
    assert resolve_fused_model(nav.dynamics, nav.running_cost, nav.terminal_cost) is None


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_torch_models_equal_oracle_models(dtype):
    g = torch.Generator().manual_seed(0)
    s = torch.randn(64, 2, generator=g, dtype=dtype) * 2
    a1 = torch.randn(64, 1, generator=g, dtype=dtype) * 3
    a2 = torch.randn(64, 2, generator=g, dtype=dtype)
    pe, po_ = eng.Pendulum(), orc.PendulumModel(numpy_sin=False)
    assert torch.equal(pe.dynamics(s, a1), po_.dynamics(s, a1))
    assert torch.equal(pe.running_cost(s, a1), po_.running_cost(s, a1))
    ne = eng.LinearPoint.toy2d_nav()
    no = orc.LinearPointModel(B=ne.B, goal=ne.goal, R=ne.R, hills=ne.hills, terminal_scale=10.0, dtype=dtype)
    assert torch.equal(ne.dynamics(s, a2), no.dynamics(s, a2))
    assert torch.allclose(ne.running_cost(s, a2), no.running_cost(s, a2), rtol=1e-6)
    st = s.view(1, 8, 8, 2)
    assert torch.allclose(ne.terminal_cost(st, None), no.terminal_cost(st, None), rtol=1e-6)


def test_shard_bounds_partition_exactly():
    for K in (8, 100, 16384, 2 ** 20, 1000003):
        for world in (1, 2, 3, 4, 8):
            spans = [shard_bounds(K, r, world) for r in range(world)]
            assert spans[0][0] == 0 and sum(n for _, n in spans) == K
            for (o0, n0), (o1, _) in zip(spans, spans[1:]):
                assert o0 + n0 == o1
    with pytest.raises(ValueError):
        shard_bounds(2, 3, 4)


def test_combine_partials_equals_unsharded_softmin():
    g = torch.Generator().manual_seed(1)
    K, R, lam = 1000, 12, 0.7
    cost = torch.rand(K, generator=g, dtype=torch.float64) * 50
    eps = torch.randn(K, R, generator=g, dtype=torch.float64)
    beta, w, eta, omega = orc.softmin_weights(cost, lam)
    want = (omega[:, None] * eps).sum(0)
    recs = []
    for r in range(4):
        o, n = shard_bounds(K, r, 4)
        c, e = cost[o:o + n], eps[o:o + n]
        b = c.min()
        ww = torch.exp(-(c - b) / lam)
        recs.append(torch.cat([b.view(1), ww.sum().view(1), (ww[:, None] * e).sum(0)]))
    b2, eta2, delta = combine_partials(torch.stack(recs), lam)
    assert torch.allclose(delta, want, atol=1e-12) and abs(b2 - beta) < 1e-15 and abs(eta2 - eta) < 1e-9


def _gloo_worker(rank, world, port, K, R, lam, out):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    g = torch.Generator().manual_seed(7)
    cost = torch.rand(K, generator=g, dtype=torch.float64) * 30
    eps = torch.randn(K, R, generator=g, dtype=torch.float64)
    o, n = shard_bounds(K, rank, world)
    c, e = cost[o:o + n], eps[o:o + n]
    b = c.min()
    w = torch.exp(-(c - b) / lam)
    rec = torch.cat([b.view(1), w.sum().view(1), (w[:, None] * e).sum(0)])
    gathered = torch.zeros(world * (R + 2), dtype=torch.float64)
    dist.all_gather_into_tensor(gathered, rec)                # the collective the nccl route issues
    _, _, delta = combine_partials(gathered.view(world, R + 2), lam)
    _, _, _, omega = orc.softmin_weights(cost, lam)
    want = (omega[:, None] * eps).sum(0)
    out[rank] = float((delta - want).abs().max())
    dist.destroy_process_group()


def test_world2_gloo_exchange_matches_single_process():
    import torch.multiprocessing as mp
    mgr = mp.Manager()
    out = mgr.dict()
    port = 29500 + (os.getpid() % 2000)
    mp.spawn(_gloo_worker, args=(2, port, 999, 10, 1.3, out), nprocs=2, join=True)
    assert len(out) == 2 and max(out.values()) < 1e-12


@pytest.mark.parametrize("exchange", ["NCCL", "nvlink", "", None])
def test_unknown_exchange_is_refused(exchange):
    """Only "p2p" and "nccl" name an exchange; anything else used to select the NCCL route silently."""
    pend = eng.Pendulum()
    with pytest.raises(ValueError, match="exchange"):
        eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(1.0), num_samples=64, horizon=10, exchange=exchange)


def _nominal_worker(rank, world, port, out):
    import types
    import torch.distributed as dist
    from pytorch_mppi_b200.mppi import MPPI
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.manual_seed(100 + rank)                              # every process draws differently ...
    fake = types.SimpleNamespace(_world=world, _pg=dist.group.WORLD, d=torch.device("cpu"), dtype=torch.float64)
    t = MPPI._one_draw_for_all_ranks(fake, torch.randn(7, 2, dtype=torch.float64))
    lst = [torch.zeros_like(t) for _ in range(world)]
    dist.all_gather(lst, t)
    torch.manual_seed(100)
    out[rank] = bool(all(torch.equal(lst[0], u) for u in lst)) and bool(torch.equal(t, torch.randn(7, 2, dtype=torch.float64)))
    dist.destroy_process_group()


def test_world2_random_nominal_is_rank0s_draw():
    """Sharded controllers add the same update to every rank's copy of U: a nominal drawn at random (U_init=None, reset())
    must therefore be ONE draw — rank 0's, broadcast (the host logic; the controllers themselves: tests/test_gpu_multi.py)."""
    import torch.multiprocessing as mp
    mgr = mp.Manager()
    out = mgr.dict()
    port = 31500 + (os.getpid() % 2000)
    mp.spawn(_nominal_worker, args=(2, port, out), nprocs=2, join=True)
    assert len(out) == 2 and all(out.values())


def test_philox_known_answers():
    # Random123 kat_vectors: philox4x32_10
    v = po.philox4x32_10(np.zeros((1, 4), dtype=np.uint32), (0, 0))[0]
    assert [int(x) for x in v] == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]
    v = po.philox4x32_10(np.full((1, 4), 0xFFFFFFFF, dtype=np.uint32), (0xFFFFFFFF, 0xFFFFFFFF))[0]
    assert [int(x) for x in v] == [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]
    v = po.philox4x32_10(np.array([[0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344]], dtype=np.uint32), (0xa4093822, 0x299f31d0))[0]
    assert [int(x) for x in v] == [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]


def test_philox_normals_shard_invariant_and_gaussian():
    full = po.normals(99, 5, 0, 4096, 30, np.float32)
    part = po.normals(99, 5, 1024, 512, 30, np.float32)
    assert np.array_equal(full[1024:1536], part)             # keyed by the global sample index
    assert abs(full.mean()) < 0.01 and abs(full.std() - 1) < 0.01
    d = po.normals(99, 5, 0, 4096, 7, np.float64)
    assert d.shape == (4096, 7) and abs(d.std() - 1) < 0.02


def test_kernel_matrices_identities():
    # W theta interpolates: at support times the interpolation reproduces theta (SURVEY.md App. A probe)
    T, S = 20, 5
    W, Wsh = orc.kernel_matrices(T, S, lambda a, b: orc.rbf_kernel(a, b, 2.0), torch.float64)
    assert W.shape == (T, S) and Wsh.shape == (S, S)
    Tk = torch.linspace(0, T - 1, S)
    idx = [int(round(float(t))) for t in Tk if abs(float(t) - round(float(t))) < 1e-9]
    theta = torch.randn(S, 2, dtype=torch.float64)
    full = W @ theta
    for s, t in enumerate(Tk):
        if abs(float(t) - round(float(t))) < 1e-9:
            assert torch.allclose(full[int(round(float(t)))], theta[s], atol=1e-9)
    assert len(idx) >= 2


def test_cuda_model_compiles_with_nvrtc_in_process():
    """User models: NVRTC compiles the fused / split-cost / batched / resident / states kernels of the model from the
    engine's own kernel headers — no nvcc, no GPU — and returns a cubin plus the lowered names the C library resolves
    (`mppi_user_model_register`); the result is cached on disk.  The controller-side resolution treats the model's bound
    methods like any registered model's."""
    from tests.user_models import pendulum_user_model
    ref = eng.Pendulum()
    m = pendulum_user_model()
    assert "struct UserModel" in m.header_text() and "NX = 2, NU = 1" in m.header_text()
    assert resolve_fused_model(m.dynamics, m.running_cost, None) is m
    s = torch.randn(8, 2)
    assert torch.equal(m.dynamics(s, torch.zeros(8, 1)), ref.dynamics(s, torch.zeros(8, 1)))
    cubin, names = m.compile_rtc(torch.float32, 0)
    assert cubin[:4] == b"\x7fELF" and len(cubin) > 100000
    assert len(names) == 5 and all(n is not None for n in names)
    assert "fused_command_kernel" in names[0] and "UserModel" in names[0] and "states_kernel" in names[4]
    assert "resident_command_kernel" in names[3]
    again, names2 = m.compile_rtc(torch.float32, 0)                  # disk cache
    assert again == cubin and names2 == names
    _, names_k = m.compile_rtc(torch.float64, 2)                     # KMPPI, fp64: no batched kernel
    assert names_k[2] is None and "Li2E" in names_k[0] and "dLi2" in names_k[0].replace("UserModelE", "")


def test_tanh4_shared_reciprocal_formula():
    """csrc/mppi_math.cuh `tanh4_`: four tanh with ONE reciprocal — 1 - 2/a_i, a_i = 1 + e^{2 x_i}, 1/a_0 = r (a_2 a_3) a_1
    with r = 1/(a_0 a_1 a_2 a_3), inputs clamped at 10 from above.  The same operations in numpy float32 (exact exp2 and
    reciprocal standing in for MUFU.EX2 / MUFU.RCP, which add ~2 ulp each): the product never overflows and the result
    stays within 1e-6 of tanh over the whole range, groups mixing saturated and small arguments included."""
    import numpy as np
    f = np.float32
    rng = np.random.default_rng(3)
    x = np.concatenate([rng.uniform(-20, 20, (20000, 4)), rng.normal(0, 1.5, (20000, 4)), rng.normal(0, 1e-3, (2000, 4)),
                        np.array([[50.0, -50.0, 0.0, 9.99], [10.0, 10.0, 10.0, 10.0], [-87.0, 88.0, 1e-8, -1e-8],
                                  [np.inf, -np.inf, 3.0, -3.0]])]).astype(f)
    with np.errstate(over="raise", invalid="raise"):
        t = np.exp2((np.minimum(x, f(10.0)) * f(2.8853900817779268)).astype(f)).astype(f)
        a = (f(1.0) + t).astype(f)
        p01, p23 = (a[:, 0] * a[:, 1]).astype(f), (a[:, 2] * a[:, 3]).astype(f)
        r = (f(1.0) / (p01 * p23).astype(f)).astype(f)
        r = (r * f(-2.0)).astype(f)
        r01, r23 = (r * p23).astype(f), (r * p01).astype(f)
        y = np.stack([r01 * a[:, 1] + f(1.0), r01 * a[:, 0] + f(1.0), r23 * a[:, 3] + f(1.0), r23 * a[:, 2] + f(1.0)], 1).astype(f)
    assert np.isfinite(y).all() and float((p01 * p23).max()) < 1e35            # e^80 at most: no overflow
    want = np.tanh(x.astype(np.float64))
    assert float(np.abs(y - want).max()) < 1e-6
    assert (np.abs(y) <= 1.0 + 2.4e-7).all()            # the shared reciprocal can land one ulp outside [-1, 1]; nothing relies on the bound


def test_bf16_split_contraction_precision_model():
    """The arithmetic contract of the tensor-core MLP route (csrc/mppi_mlp_tc.cuh), restated with torch's
    round-to-nearest bf16 casts:  v = hi + lo (both bf16), layer = a_hi*w_hi + a_lo*w_hi + a_hi*w_lo + b_hi + b_lo
    accumulated in fp32.  The dropped a_lo*w_lo term and the lo roundings leave ~2^-16 relative error per
    layer; plain bf16 operands leave ~2^-8.  This pins the tolerances the GPU tests use for the two modes."""
    torch.manual_seed(25)
    net = torch.nn.Sequential(torch.nn.Linear(3, 32), torch.nn.Tanh(), torch.nn.Linear(32, 32), torch.nn.Tanh(),
                              torch.nn.Linear(32, 2))
    g = torch.Generator().manual_seed(0)
    x = torch.cat((torch.rand(4096, 1, generator=g) * 6.28 - 3.14, torch.randn(4096, 1, generator=g) * 3,
                   torch.rand(4096, 1, generator=g) * 4 - 2), dim=1)

    def split(v):
        hi = v.to(torch.bfloat16).to(torch.float32)
        lo = (v - hi).to(torch.bfloat16).to(torch.float32)
        return hi, lo

    def layer(a, lin, mode):
        w, b = lin.weight.detach(), lin.bias.detach()
        wh, wl = split(w)
        bh, bl = split(b)
        ah, al = split(a)
        if mode == "bf16x3":
            return ah @ wh.T + al @ wh.T + ah @ wl.T + bh + bl
        return ah @ wh.T + bh + bl

    def forward(mode_hidden):
        h = torch.tanh(layer(x, net[0], "bf16x3"))               # the state inputs are always split
        h = torch.tanh(layer(h, net[2], mode_hidden))
        return layer(h, net[4], mode_hidden)

    with torch.no_grad():
        want = net.double()(x.double())
        net.float()
        e3 = (forward("bf16x3").double() - want).abs().max().item()
        e1 = (forward("bf16").double() - want).abs().max().item()
    scale = want.abs().max().item()
    assert e3 < 2e-5 * max(1.0, scale), e3
    assert 1e-4 < e1 < 2e-2, e1                                   # plain bf16 really is ~2^-8: not a parity route


def test_build_is_keyed_by_source_hash_not_file_times(tmp_path, monkeypatch):
    """The in-tree library is rebuilt when (and only when) the sources it was compiled from change: the stamp next to
    the .so holds their hash, so a snapshot copy that scrambles file times does not trigger a rebuild on the GPU machine."""
    from pytorch_mppi_b200 import build
    build.build()
    assert not build.needs_build()
    h = build.source_hash()
    assert open(build.STAMP).read().strip() == h and len(h) == 40
    # older/newer file times alone change nothing
    os.utime(os.path.join(build.CSRC, "mppi_b200.cu"), None)
    assert not build.needs_build()
    # a different source does (here: one more header in the C-ABI unit's dependency list)
    fake = tmp_path / "extra.cuh"
    fake.write_text("// edited\n")
    src, defs, hdrs = build.UNITS["cabi"]
    monkeypatch.setitem(build.UNITS, "cabi", (src, defs, [*hdrs, str(fake)]))
    assert build.source_hash() != h and build.needs_build()
    monkeypatch.setitem(build.UNITS, "cabi", (src, defs, hdrs))
    assert not build.needs_build()
    # and so does a missing stamp
    monkeypatch.setattr(build, "STAMP", str(tmp_path / "nope.stamp"))
    assert build.needs_build()
