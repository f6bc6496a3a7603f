"""GPU: the device-only float primitives over their whole input range, against exact or fp64 references.

The fp32 rollouts run on a few primitives whose device bodies differ from their host bodies (csrc/mppi_math.cuh,
csrc/mppi_mlp_tc.cuh): the remainder without the long-division loop (`Ops<float>::fmod_`, `fmod_small_`, `remainder`),
the exp/reciprocal and MUFU.TANH forms of tanh (`tanh_`, `tanh4_`, whose four lanes share one reciprocal), the SFU
Box-Muller pair (`Normals<float>::pair`) and the bf16 hi/lo split of the tensor-core route (`tc::split_bf16`,
`tc::to_operand`).  The probe (tests/device_math_probe.py) runs them on the device for every float bit pattern where a
scan of 2^32 inputs is meaningful and reduces the mismatches and the largest errors there.  The references: the
library's exact `fmodf` and torch's floating remainder rule; `tanh`, `log`, `sin`, `cos` in fp64; the noise stream's
definition in oracle/philox_oracle.py; round-to-nearest-even bf16 (torch's casts on a subset).  The measured maxima go to
tests/_reports/device_math.json."""
import ctypes
import json
import math
import struct

import numpy as np
import pytest
import torch

from oracle import philox_oracle as po
from tests import device_math_probe as probe
from tests import reports

pytestmark = pytest.mark.gpu

U64 = ctypes.c_ulonglong
PTR = ctypes.c_void_p
N_ALL = 1 << 32
N_NAN = 2 * (0x7FFFFFFF - 0x7F800000)            # exponent all ones, mantissa non-zero, both signs
N_FINITE = N_ALL - N_NAN - 2

REPORT = {}


def _record(section, key, value):
    REPORT.setdefault(section, {})[key] = value
    reports.write("device_math.json", json.dumps(REPORT, indent=1, sort_keys=True))


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = ctypes.CDLL(probe.build(tmp_path_factory.mktemp("device_math")))
    for name, args in {"scan_fmod": [ctypes.c_float, PTR], "scan_fmod_random": [PTR], "scan_tanh": [PTR],
                       "scan_normals_a": [ctypes.c_uint, PTR], "scan_normals_b": [ctypes.c_uint, PTR],
                       "scan_normals_double": [U64, PTR], "scan_bf16": [PTR],
                       "set_companions": [PTR, PTR, PTR, PTR], "scan_tanh4": [ctypes.c_int, ctypes.c_int, PTR],
                       "remainder_array": [PTR, PTR, PTR, ctypes.c_int, ctypes.c_int],
                       "tanh4_groups": [PTR, PTR, ctypes.c_int, ctypes.c_int],
                       "split_array": [PTR, PTR, PTR, ctypes.c_int], "to_operand_markers": [PTR, PTR],
                       "normals_double": [PTR, PTR, PTR, ctypes.c_int],
                       "philox_array": [PTR, PTR, PTR, PTR, ctypes.c_int]}.items():
        getattr(so, name).argtypes = args
        getattr(so, name).restype = ctypes.c_int
    return so


def _p(t):
    return PTR(t.data_ptr())


class Check:
    """One check of a scan: inputs tested, inputs failing, the smallest failing key, the largest error and its input."""

    def __init__(self, words):
        t, b, f, m = (int(w) & 0xFFFFFFFFFFFFFFFF for w in words)
        self.tested, self.bad, self.first = t, b, f
        eb = m >> 32
        self.max = math.nan if eb == 0xFFFFFFFF else struct.unpack("<f", struct.pack("<I", eb))[0]
        self.argmax = m & 0xFFFFFFFF

    def where(self):
        return f"{self.bad} of {self.tested} fail, first at key {self.first:#x}"

    def summary(self):
        return {"tested": self.tested, "failing": self.bad, "max": self.max, "argmax": f"{self.argmax:#010x}"}


def _scan(fn, n_checks, *args):
    out = torch.zeros(n_checks, 4, dtype=torch.int64, device="cuda")
    out[:, 2] = -1
    torch.cuda.synchronize()
    assert fn(*args, _p(out)) == 0
    return [Check(row) for row in out.cpu().tolist()]


def _f(bits):
    return struct.unpack("<f", struct.pack("<I", bits))[0]


def _bits(x):
    return struct.unpack("<I", struct.pack("<f", x))[0]


# ------------------------------------------------------------------------------------------------ remainder
TWO_PI = float(np.float32(2 * math.pi))
FLT_MIN = 2.0 ** -126
DIVISORS = {"two_pi": TWO_PI, "pi": float(np.float32(math.pi)), "1": 1.0, "3": 3.0, "0.1f": float(np.float32(0.1)),
            "0x3fffffff": _f(0x3FFFFFFF), "0x3f800001": _f(0x3F800001), "FLT_MIN": _f(0x00800000),
            "min_subnormal": _f(0x00000001), "max_subnormal": _f(0x007FFFFF), "2^126": 2.0 ** 126, "2^127": 2.0 ** 127,
            "FLT_MAX": _f(0x7F7FFFFF), "+inf": math.inf, "+0": 0.0, "-0": -0.0, "-two_pi": -TWO_PI, "nan": math.nan}


def _small_domain_count(b):
    """Floats a with |a| < 2^21 b (fmod_small_'s domain, b a positive normal float): both signs of the bit patterns below
    the edge."""
    if not (FLT_MIN <= b < math.inf):
        return 0
    edge = 2.0 ** 21 * b                             # exact in double
    k = 0x7F800000 if edge > _f(0x7F7FFFFF) else _bits(float(np.float32(edge)))
    while k > 0 and _f(k - 1) >= edge:
        k -= 1
    while k < 0x7F800000 and _f(k) < edge:
        k += 1
    return 2 * k


@pytest.mark.parametrize("name", list(DIVISORS))
def test_fmod_and_remainder_are_exact_for_every_a(lib, name):
    """fmod_ is fmodf bit for bit for all 2^32 a (every NaN counts as equal), fmod_small_ on its whole domain (b a
    positive normal float; the scan runs through both sides of |a| = 2^21 b), and remainder<float> / remainder<float, true> follow torch's floating
    remainder rule on the exact fmodf."""
    b = DIVISORS[name]
    c = _scan(lib.scan_fmod, 4, ctypes.c_float(b))
    _record("remainder", name, {"fmod_": c[0].bad, "fmod_small_": c[1].bad, "remainder": c[2].bad,
                                "remainder_small": c[3].bad, "small_domain": c[1].tested})
    assert c[0].tested == N_ALL and c[2].tested == N_ALL
    assert c[1].tested == c[3].tested == _small_domain_count(b)
    assert c[0].bad == 0, f"fmod_(a, {b!r}): {c[0].where()} (a's bits)"
    assert c[1].bad == 0, f"fmod_small_(a, {b!r}): {c[1].where()}"
    assert c[2].bad == 0, f"remainder<float>(a, {b!r}): {c[2].where()}"
    assert c[3].bad == 0, f"remainder<float, true>(a, {b!r}): {c[3].where()}"


def test_fmod_and_remainder_are_exact_on_random_pairs(lib):
    """2^32 random pairs: b a positive normal float, |a| / b log-uniform over [2^-4, 2^23] (through the fast path's
    2^21 edge), either sign."""
    c = _scan(lib.scan_fmod_random, 4)
    _record("remainder", "random_pairs", {"fmod_": c[0].bad, "fmod_small_": c[1].bad, "remainder": c[2].bad,
                                          "remainder_small": c[3].bad, "small_domain": c[1].tested})
    assert c[0].tested == N_ALL and c[1].tested > N_ALL // 2
    for i, name in enumerate(["fmod_", "fmod_small_", "remainder<float>", "remainder<float, true>"]):
        assert c[i].bad == 0, f"{name}: {c[i].where()} (a's bits << 32 | b's bits)"


def test_remainder_matches_torch_remainder_on_the_device(lib):
    g = torch.Generator(device="cuda").manual_seed(3)
    n = 1 << 22
    mag = torch.exp2(torch.empty(n, device="cuda").uniform_(-30.0, 30.0, generator=g))
    sign = torch.where(torch.rand(n, device="cuda", generator=g) < 0.5, -1.0, 1.0)
    a = mag * sign
    a[:8] = torch.tensor([0.0, -0.0, math.inf, -math.inf, math.nan, 1e38, -1e-40, 2.0 ** 21 * TWO_PI])
    divs = torch.tensor([TWO_PI, math.pi, 1.0, 3.0, 0.1, 1e-3, 1e3, -TWO_PI, -1.0, 2.0 ** -140], device="cuda")
    b = divs[torch.randint(0, len(divs), (n,), device="cuda", generator=g)]
    want = torch.remainder(a, b)
    for small in (0, 1):
        got = torch.empty_like(a)
        assert lib.remainder_array(_p(a), _p(b), _p(got), n, small) == 0
        keep = torch.ones_like(a, dtype=torch.bool)
        if small:                                     # fmod_small_'s domain
            keep = (b >= FLT_MIN) & (a.double().abs() < 2.0 ** 21 * b.double())
        same = (got.view(torch.int32) == want.view(torch.int32)) | (got.isnan() & want.isnan())
        bad = (~same & keep).nonzero()
        assert bad.numel() == 0, f"small={small}: {bad.numel()} differ, first a={a[bad[0]].item()!r} b={b[bad[0]].item()!r}"


# ------------------------------------------------------------------------------------------------ tanh
COMPANIONS = [0.0, 1e-4, -1e-4, 0.5, -3.0, 10.0, 1e4, -1e4, math.inf, -math.inf, math.nan, 0.0]   # the last: x itself
TANH_ABS, TANH4_ABS, TANH_APPROX_REL = 5e-7, 1e-6, 2.0 ** -10.987


def test_tanh_forms_over_every_float(lib):
    """tanh_(x, 0) within 5e-7 of fp64 tanh for every float x; tanh_(x, 1) and tanh4_ mode 1 (MUFU.TANH, x in each
    lane) within the PTX bound for tanh.approx.f32, relative 2^-10.987; every result finite for a non-NaN x, and
    |y| <= 1 + 2^-22."""
    c = _scan(lib.scan_tanh, 5)
    names = ["tanh_mode0_abs", "tanh_mode1_rel", "tanh_mode1_abs", "tanh_abs_y_minus_1", "tanh4_mode1_rel"]
    for name, ch in zip(names, c):
        _record("tanh", name, ch.summary())
    assert c[0].tested == N_ALL - N_NAN and c[4].tested == 4 * c[0].tested
    for i in (0, 1, 3, 4):
        assert c[i].bad == 0, f"{names[i]}: {c[i].where()} (x's bits); max {c[i].max:.3g} at {c[i].argmax:#010x}"
    assert c[0].max <= TANH_ABS and c[1].max <= TANH_APPROX_REL and c[4].max <= TANH_APPROX_REL
    assert c[3].max <= 2.0 ** -22


@pytest.mark.parametrize("lane,shift", [(0, 0), (1, 8), (2, 8), (3, 8)], ids=["lane0-every_float", "lane1-2^24_floats",
                                                                               "lane2-2^24_floats", "lane3-2^24_floats"])
def test_tanh4_against_every_companion_triple(lib, lane, shift):
    """tanh4_ (mode 0) with x in one lane and the other three lanes taking each of the 12^3 triples of companions
    {0, +-1e-4, 0.5, -3, 10, +-1e4, +-inf, NaN, x}: every float x in lane 0, one float in 2^8 (all exponents, hashed
    mantissas) in lanes 1-3.  Every lane within 1e-6 of fp64 tanh, x's and the other three alike: the shared reciprocal
    of the four lanes' product leaks nothing across them, with three lanes saturated and the fourth anywhere (the clamp
    at 10 keeps the product below e^80).  A NaN lane returns +1; a lane holding x >= 10, +inf or NaN returns exactly 1.
    |y| <= 1 + 2^-20: a lane saturated at -1 can come out below it by the roundings of the shared products (2/a is within
    6 * 2^-24 of its value, so y >= -1 - 12 * 2^-24, then rounded)."""
    t = [1.0 if math.isnan(v) else math.tanh(v) for v in COMPANIONS]
    value = np.array(COMPANIONS, dtype=np.float32)
    hi = np.array(t, dtype=np.float32)
    lo = (np.array(t) - hi.astype(np.float64)).astype(np.float32)
    sat = np.array([0 if v < 10 else 1 for v in COMPANIONS], dtype=np.int32)      # NaN < 10 is False: saturating
    assert lib.set_companions(*(PTR(a.ctypes.data) for a in (value, hi, lo, sat))) == 0
    c = _scan(lib.scan_tanh4, 4, lane, shift)
    names = ["x_lane_abs", "other_lanes_abs", "saturation_exactly_1", "abs_y_minus_1"]
    _record("tanh4_mode0_triples", f"lane{lane}", {n: ch.summary() for n, ch in zip(names, c)})
    for name, ch in zip(names, c):
        assert ch.tested == N_ALL >> shift
        assert ch.bad == 0, f"lane {lane}, {name}: {ch.where()} (x's bits); max {ch.max:.3g} at {ch.argmax:#010x}"
    assert c[0].max <= TANH4_ABS and c[1].max <= TANH4_ABS and c[3].max <= 2.0 ** -20


def test_tanh4_nan_lane_returns_one_and_leaves_its_partners_alone(lib):
    """The header's decision: a NaN lane of tanh4_ (mode 0) returns +1, as a saturated one does, and the other three
    lanes (in the wgmma kernel, two of them belong to another sample) keep their own tanh.  MUFU.TANH (mode 1) returns
    NaN for a NaN lane, per lane."""
    others = [0.5, -3.0, 1e-4]
    groups = []
    for nan in (math.nan, -math.nan, _f(0x7F800001), _f(0xFFFFFFFF)):
        for p in range(4):
            g = list(others)
            g.insert(p, nan)
            groups.append(g)
    x = torch.tensor(groups, dtype=torch.float32, device="cuda")
    seen = {}
    for mode in (0, 1):
        y = torch.empty_like(x)
        assert lib.tanh4_groups(_p(x), _p(y), x.shape[0], mode) == 0
        y = y.cpu()
        isnan = x.cpu().isnan()
        seen[f"mode{mode}"] = sorted({repr(v) for v in y[isnan].tolist()})
        other = torch.tanh(x.cpu()[~isnan].double())
        assert (y[~isnan].double() - other).abs().max().item() <= (TANH4_ABS if mode == 0 else 2e-3)
        if mode == 0:
            assert torch.equal(y[isnan], torch.ones(int(isnan.sum())))
        else:
            assert y[isnan].isnan().all()
    _record("tanh", "nan_lane_returns", seen)


# ------------------------------------------------------------------------------------------------ normal draws
REGIONS = ["u1<0.5", "0.5<=u1<1-2^-20", "u1>=1-2^-20"]
NORMAL_ABS = 2e-5


def _check_normals(c, label):
    _record("normals_float", label, {r: ch.summary() for r, ch in zip(REGIONS, c) if ch.tested})
    assert sum(ch.tested for ch in c) == N_ALL
    for r, ch in zip(REGIONS, c):
        assert ch.bad == 0, f"{label}, {r}: {ch.where()}; max |error| {ch.max:.3g} at {ch.argmax:#010x}"


@pytest.mark.parametrize("b", [0, 1 << 30, 1 << 31, 3 << 30, 0xFFFFFFFF], ids=lambda b: f"b={b:#x}")
def test_normal_pair_over_every_first_word(lib, b):
    """Normals<float>::pair(a, b) for all 2^32 a: finite, and within 2e-5 of the stream definition (u in float32, then
    log, sqrt, sin, cos in fp64) — near u1 -> 1 (r -> 0) as well as elsewhere."""
    _check_normals(_scan(lib.scan_normals_a, 3, ctypes.c_uint(b)), f"a_scan,b={b:#x}")


R_ONE = int(math.exp(-0.5) * 2 ** 32)              # -2 ln u1 ~ 1


@pytest.mark.parametrize("a", [0, R_ONE, 0xFFFFFE00], ids=["r~6.76", "r~1", "r~4.9e-4"])
def test_normal_pair_over_every_second_word(lib, a):
    _check_normals(_scan(lib.scan_normals_b, 3, ctypes.c_uint(a)), f"b_scan,a={a:#x}")


def _numpy_normals_f64(a, b):
    """oracle/philox_oracle.py's fp64 statement on the raw 64-bit words."""
    u1 = (a >> np.uint64(11)).astype(np.float64) * 2.0 ** -53 + 2.0 ** -54
    u2 = (b >> np.uint64(11)).astype(np.float64) * 2.0 ** -53 + 2.0 ** -54
    r = np.sqrt(-2.0 * np.log(u1))
    return np.stack([r * np.sin(2.0 * np.pi * u2), r * np.cos(2.0 * np.pi * u2)], axis=-1)


def test_normal_pair_double_at_edge_words_and_random_words(lib):
    """Normals<double>::pair at the ends of the 53-bit uniform (a >> 11 in {0, 1, 2^52, 2^53 - 1}, low bits set or not)
    and at the quadrant edges of 2 pi u2, and on 2^20 random words, against the numpy statement at 1e-13; 2^28 random
    words against the same statement in fp64 on the device."""
    av = [0, 1, 1 << 52, (1 << 53) - 1]
    aw = [v << 11 for v in av] + [(v << 11) | 0x7FF for v in av]
    bv = sorted({min(max(k * (1 << 51) + d, 0), (1 << 53) - 1) for k in range(5) for d in (-1, 0, 1)})
    bw = [v << 11 for v in bv] + [(v << 11) | 0x7FF for v in bv]
    a = np.array([x for x in aw for _ in bw], dtype=np.uint64)
    b = np.array([y for _ in aw for y in bw], dtype=np.uint64)
    rng = np.random.default_rng(11)
    a = np.concatenate([a, rng.integers(0, 2 ** 64, 1 << 20, dtype=np.uint64)])
    b = np.concatenate([b, rng.integers(0, 2 ** 64, 1 << 20, dtype=np.uint64)])
    ta = torch.from_numpy(a.view(np.int64)).cuda()
    tb = torch.from_numpy(b.view(np.int64)).cuda()
    out = torch.empty(len(a), 2, dtype=torch.float64, device="cuda")
    assert lib.normals_double(_p(ta), _p(tb), _p(out), len(a)) == 0
    err = np.abs(out.cpu().numpy() - _numpy_normals_f64(a, b))
    i = int(err.max(axis=1).argmax())
    _record("normals_double", "edges_and_2^20_random_vs_numpy", {"max": float(err.max()), "argmax": [hex(a[i]), hex(b[i])]})
    assert err.max() <= 1e-13, (hex(a[i]), hex(b[i]), err[i])
    c = _scan(lib.scan_normals_double, 1, U64(1 << 28))[0]
    _record("normals_double", "2^28_random_vs_device_fp64", c.summary())
    assert c.tested == 1 << 28 and c.bad == 0, c.where()


def test_philox_on_the_device_matches_the_oracle(lib):
    """The three Random123 known answers, and 2^24 random counters (offset and subsequence high words non-zero) under
    16 random keys, bit for bit against oracle/philox_oracle.py."""
    kat = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
           ((0xFFFFFFFF,) * 4, (0xFFFFFFFF, 0xFFFFFFFF), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
           ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
            (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    rng = np.random.default_rng(7)
    per_key = 1 << 20
    seeds, ctrs, want = [], [], []
    for ctr, key, ans in kat:
        seeds.append(np.array([key[0] | key[1] << 32], dtype=np.uint64))
        ctrs.append(np.array([ctr], dtype=np.uint64))
        want.append(np.array([ans], dtype=np.uint32))
    for _ in range(16):
        key = rng.integers(0, 2 ** 32, 2, dtype=np.uint64)
        ctr = rng.integers(0, 2 ** 32, (per_key, 4), dtype=np.uint64)
        seeds.append(np.full(per_key, int(key[0]) | int(key[1]) << 32, dtype=np.uint64))
        ctrs.append(ctr)
        want.append(po.philox4x32_10(ctr, (int(key[0]), int(key[1]))))
    seed, ctr, want = np.concatenate(seeds), np.concatenate(ctrs), np.concatenate(want)
    assert (ctr[3:, 1] != 0).mean() > 0.99 and (ctr[3:, 3] != 0).mean() > 0.99
    offset = ctr[:, 0] | (ctr[:, 1] << np.uint64(32))
    subseq = ctr[:, 2] | (ctr[:, 3] << np.uint64(32))
    dev = [torch.from_numpy(v.view(np.int64)).cuda() for v in (seed, subseq, offset)]
    out = torch.empty(len(seed), 4, dtype=torch.int32, device="cuda")
    assert lib.philox_array(*(_p(t) for t in dev), _p(out), len(seed)) == 0
    got = out.cpu().numpy().view(np.uint32)
    assert np.array_equal(got[:3], want[:3]), [[hex(w) for w in row] for row in got[:3]]
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert bad.size == 0, f"{bad.size} counters differ, first {ctr[bad[0]]} under seed {seed[bad[0]]:#x}"


# ------------------------------------------------------------------------------------------------ bf16 split
def test_bf16_split_over_every_finite_float(lib):
    """split_bf16: hi = bf16_rn(x), lo = bf16_rn(x - hi) bit for bit for every finite x, and |x - hi - lo| <= 2^-17 |x|
    unless hi overflows to inf (or, below the bf16 normals, half the smallest bf16 subnormal); to_operand<1> packs the
    same halves for every x."""
    c = _scan(lib.scan_bf16, 3)
    for name, ch in zip(["split_bits", "residual_over_abs_x", "to_operand_bits"], c):
        _record("bf16_split", name, ch.summary())
    assert c[0].tested == N_FINITE and c[2].tested == c[0].tested
    assert c[0].bad == 0, c[0].where()
    assert c[1].bad == 0, c[1].where()
    assert c[1].max <= 2.0 ** -17
    assert c[2].bad == 0, c[2].where()


def test_bf16_split_matches_torch_casts(lib):
    bits = torch.arange(0, N_ALL, 509, dtype=torch.int64, device="cuda")
    x = (bits - (bits >= 1 << 31).long() * N_ALL).to(torch.int32).view(torch.float32)
    x = x[x.isfinite()].contiguous()
    hi = torch.empty(x.shape, dtype=torch.int16, device="cuda")
    lo = torch.empty_like(hi)
    assert lib.split_array(_p(x), _p(hi), _p(lo), x.numel()) == 0
    th = x.to(torch.bfloat16)
    tl = (x - th.float()).to(torch.bfloat16)
    assert torch.equal(hi, th.view(torch.int16))
    assert torch.equal(lo, tl.view(torch.int16))


def test_to_operand_fragment_order(lib):
    """to_operand<1> on 16 distinct markers: each half of hi[s][r] and lo[s][r] holds the split of the h element at the
    fragment position the header names.  h[4j + 0/1] is row g, columns 8j + 2t, +1; h[4j + 2/3] row g + 8, same columns;
    a[s] = {(g, 16s + 2t..), (g + 8, 16s + 2t..), (g, 16s + 8 + 2t..), (g + 8, 16s + 8 + 2t..)}, the lower column in the
    low half."""
    h = torch.tensor([(i + 1) * (1.0 + 2.0 ** -12) for i in range(16)], dtype=torch.float32)
    out = torch.empty(16, dtype=torch.int32, device="cuda")
    assert lib.to_operand_markers(_p(h.cuda()), _p(out)) == 0
    words = [w & 0xFFFFFFFF for w in out.cpu().tolist()]
    hb = h.to(torch.bfloat16)
    lb = (h - hb.float()).to(torch.bfloat16)
    hbits = [v & 0xFFFF for v in hb.view(torch.int16).tolist()]
    lbits = [v & 0xFFFF for v in lb.view(torch.int16).tolist()]
    assert len(set(hbits)) == 16 and len(set(lbits)) == 16
    position = {(("g", "g+8")[(i % 4) // 2], 8 * (i // 4) + i % 2): i for i in range(16)}     # h[i] -> (row, column - 2t)
    for s in range(2):
        for r in range(4):
            for half in range(2):
                i = position[(("g", "g+8")[r % 2], 16 * s + 8 * (r // 2) + half)]
                assert (words[4 * s + r] >> (16 * half)) & 0xFFFF == hbits[i], ("hi", s, r, half)
                assert (words[8 + 4 * s + r] >> (16 * half)) & 0xFFFF == lbits[i], ("lo", s, r, half)
