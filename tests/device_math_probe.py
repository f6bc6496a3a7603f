"""The device-only float primitives of csrc/mppi_math.cuh and csrc/mppi_mlp_tc.cuh, compiled into a small probe library
with nvcc for sm_90a (the library's own flags) and checked against fp64 references on the device.  The remainder, the
tanh forms, the Box-Muller pair and the bf16 split each have a device body (`#if defined(__CUDA_ARCH__)`) that the host
build of the header never runs; tests/test_gpu_device_math.py drives this probe over their whole input range, and
tests/test_device_math_probe.py builds it without a GPU, so a change of the headers' names or signatures fails there.

Every scan reduces on the device into checks of four words: the inputs tested, the inputs that failed, the smallest
failing input key, and the largest error packed as (ordered error bits << 32) | input index (the error is rounded up to
float, so its bits order as unsigned integers; a NaN error ranks above everything)."""
import os
import subprocess

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pytorch_mppi_b200", "csrc")

SRC = r"""
#include <float.h>
#include "mppi_mlp_tc.cuh"

using namespace mppi;
typedef unsigned long long u64;

struct Acc {
    u64 tested = 0, bad = 0, first = ~0ull, maxe = 0;
    __device__ void note(bool t, bool b, u64 key) {
        tested += t;
        bad += b;
        if (b && key < first) first = key;
    }
    __device__ void err(double e, unsigned idx) {
        const unsigned bits = e != e ? 0xFFFFFFFFu : (__float_as_uint(__double2float_ru(e)) & 0x7FFFFFFFu);
        const u64 p = ((u64)bits << 32) | idx;
        if (p > maxe) maxe = p;
    }
    // warp-wide reduction, then one atomic per word and warp; called by all 32 lanes
    __device__ void flush(u64* o) {
        u64 t = tested, b = bad, f = first, m = maxe;
#pragma unroll
        for (int s = 16; s; s >>= 1) {
            t += __shfl_xor_sync(0xffffffffu, t, s);
            b += __shfl_xor_sync(0xffffffffu, b, s);
            f = min(f, __shfl_xor_sync(0xffffffffu, f, s));
            m = max(m, __shfl_xor_sync(0xffffffffu, m, s));
        }
        if ((threadIdx.x & 31) == 0) {
            if (t) atomicAdd(o, t);
            if (b) atomicAdd(o + 1, b);
            if (f != ~0ull) atomicMin(o + 2, f);
            if (m > *(volatile u64*)(o + 3)) atomicMax(o + 3, m);
        }
    }
};

__device__ __forceinline__ bool same_bits(float x, float y) { return __float_as_uint(x) == __float_as_uint(y) || (x != x && y != y); }
__device__ __forceinline__ bool finite(float x) { return fabsf(x) <= FLT_MAX; }
__device__ __forceinline__ u64 splitmix64(u64 z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// one input per (thread, step): inputs [0, n) with n <= 2^32, at most 2^28 threads (16 inputs each) per launch
template <class F> __global__ void __launch_bounds__(256) scan_kernel(F f, u64 n, u64* out) {
    Acc acc[F::NOUT];
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) f((unsigned)i, acc);
#pragma unroll
    for (int k = 0; k < F::NOUT; ++k) acc[k].flush(out + 4 * k);
}
template <class F> static int run(F f, u64 n, u64* out) {
    const u64 threads = n < (1ull << 28) ? n : (1ull << 28);
    scan_kernel<<<(unsigned)((threads + 255) / 256), 256>>>(f, n, out);
    return (int)cudaDeviceSynchronize();
}

// ---- remainder ----------------------------------------------------------------------------------------------------
// torch.remainder for floats: fmod, then + b when the remainder is non-zero and its sign differs from b's
__device__ __forceinline__ float torch_remainder(float a, float b) {
    float m = fmodf(a, b);
    if (m != 0.0f && ((b < 0.0f) != (m < 0.0f))) m = __fadd_rn(m, b);
    return m;
}
// fmod_small_'s domain: b a positive normal float, |a| < 2^21 b (exact in double)
__device__ __forceinline__ bool small_domain(float a, float b) {
    return b >= FLT_MIN && b <= FLT_MAX && fabs((double)a) < 2097152.0 * (double)b;
}
// checks: 0 fmod_, 1 fmod_small_ (its domain), 2 remainder<float>, 3 remainder<float, true> (fmod_small_'s domain)
__device__ __forceinline__ void remainder_checks(float a, float b, u64 key, Acc* acc) {
    const float want = fmodf(a, b);
    acc[0].note(true, !same_bits(Ops<float>::fmod_(a, b), want), key);
    const float rw = torch_remainder(a, b);
    acc[2].note(true, !same_bits(remainder<float>(a, b), rw), key);
    if (small_domain(a, b)) {
        acc[1].note(true, !same_bits(Ops<float>::fmod_small_(a, b), want), key);
        acc[3].note(true, !same_bits(remainder<float, true>(a, b), rw), key);
    }
}
struct FmodScan {       // every float a for one b; key = a's bits
    static constexpr int NOUT = 4;
    float b;
    __device__ void operator()(unsigned i, Acc* acc) const { remainder_checks(__uint_as_float(i), b, i, acc); }
};
// b a positive normal float, |a| / b = 2^e with e uniform on [-4, 23), either sign; key = a's bits << 32 | b's bits
__device__ __forceinline__ void random_pair(unsigned i, float& a, float& b) {
    const u64 w = splitmix64(i);
    b = __uint_as_float(0x00800000u + (unsigned)((w & 0xFFFFFFFFull) % 0x7F000000ull));
    const double e = -4.0 + 27.0 * (double)((w >> 32) & 0x7FFFFFFFull) * 4.656612873077393e-10;     // 2^-31
    a = (float)((double)b * exp2(e));
    if (w >> 63) a = -a;
}
struct FmodRandom {
    static constexpr int NOUT = 4;
    __device__ void operator()(unsigned i, Acc* acc) const {
        float a, b;
        random_pair(i, a, b);
        remainder_checks(a, b, ((u64)__float_as_uint(a) << 32) | __float_as_uint(b), acc);
    }
};

// ---- tanh -----------------------------------------------------------------------------------------------------------
constexpr double TANH_ABS = 5e-7, TANH_APPROX_REL = 4.9604088e-04;                       // 2^-10.987
constexpr float TANH4_ABS = 1e-6f, TANH4_OVER = 9.5367431640625e-07f;                     // 2^-20
// checks over every float x: 0 tanh_(x, 0) abs error; 1 tanh_(x, 1) relative error; 2 tanh_(x, 1) abs error;
// 3 |y| - 1 of tanh_ in both modes, at most 2^-22; 4 tanh4_ mode 1 (MUFU.TANH, per lane) with x in each of the four
// lanes, relative error.  A failure in 0, 1 and 4 is a non-finite result for a non-NaN x or an error over the bound.
struct TanhScan {
    static constexpr int NOUT = 5;
    __device__ static double rel(double y, double t) { return t == 0.0 ? (y == 0.0 ? 0.0 : INFINITY) : fabs(y - t) / fabs(t); }
    __device__ static bool bad_value(float y, float x) { return x == x && !finite(y); }
    __device__ static void over(Acc& a, float y, unsigned i) {
        const double o = fmax(fabs((double)y) - 1.0, 0.0);
        a.note(true, !(o <= 2.384185791015625e-07), i);
        a.err(o, i);
    }
    __device__ void operator()(unsigned i, Acc* acc) const {
        const float x = __uint_as_float(i);
        if (x != x) return;
        const double t = tanh((double)x);
        {
            const float y = PendulumMLPModel::tanh_(x, 0);
            const double e = fabs((double)y - t);
            acc[0].note(true, bad_value(y, x) || e > TANH_ABS, i);
            acc[0].err(e, i);
            over(acc[3], y, i);
        }
        {
            const float y = PendulumMLPModel::tanh_(x, 1);
            const double e = rel(y, t);
            acc[1].note(true, bad_value(y, x) || e > TANH_APPROX_REL, i);
            acc[1].err(e, i);
            acc[2].note(true, false, i);
            acc[2].err(fabs((double)y - t), i);
            over(acc[3], y, i);
        }
        for (int p = 0; p < 4; ++p) {
            float w[4] = {0.5f, -3.0f, __int_as_float(0x7fc00000), 1e-4f};
            w[p] = x;
            PendulumMLPModel::tanh4_(w, 1);
            const double r = rel(w[p], t);
            acc[4].note(true, bad_value(w[p], x) || r > TANH_APPROX_REL, i);
            acc[4].err(r, i);
        }
    }
};

// The companions of tanh4_'s cross product: value, the expected result as a float pair (fp64 tanh = hi + lo to ~2^-48;
// +1 for NaN, the header's choice) and whether the lane saturates (>= 10, +inf, NaN: the result must be exactly 1).  The
// last entry stands for x itself.
__constant__ float COMP[12], COMP_HI[12], COMP_LO[12];
__constant__ int COMP_SAT[12];

// tanh4_ mode 0 with x in lane P and the other three lanes taking every one of the 12^3 companion triples.  x's bits:
// i (shift 0: every float) or i << shift with the low bits from a hash of i.  Checks per x (tested: one x; failing: some
// triple failed): 0 the lane of x, abs error; 1 the other three lanes, abs error (lane isolation through the shared
// reciprocal); 2 a saturating lane is exactly 1; 3 |y| - 1 in every lane, at most 2^-20 (the shared products' roundings
// can put a lane saturated at -1 a few ulps below it).  The error bound is 1e-6; a NaN lane is expected to be +1.
template <int P> struct Tanh4Triples {
    static constexpr int NOUT = 4;
    int shift;
    __device__ void operator()(unsigned i, Acc* acc) const {
        const unsigned bits = shift == 0 ? i : (i << shift) | ((i * 2654435761u) >> (32 - shift));
        const float x = __uint_as_float(bits);
        const bool xn = x != x;
        const double t = xn ? 1.0 : tanh((double)x);
        const float thi = (float)t, tlo = (float)(t - (double)thi);
        const bool xsat = !(x < 10.0f);
        float ex = 0.0f, eo = 0.0f, ov = 0.0f;
        bool bx = false, bo = false, bs = false, bover = false;
#pragma unroll 1
        for (int j = 0; j < 12 * 12 * 12; ++j) {
            const int jj[3] = {j % 12, (j / 12) % 12, j / 144};
            float v[4], hi[4], lo[4];
            bool sat[4];
#pragma unroll
            for (int l = 0, o = 0; l < 4; ++l) {
                if (l == P) {
                    v[l] = x; hi[l] = thi; lo[l] = tlo; sat[l] = xsat;
                } else {
                    const int c = jj[o++];
                    const bool self = c == 11;
                    v[l] = self ? x : COMP[c];
                    hi[l] = self ? thi : COMP_HI[c];
                    lo[l] = self ? tlo : COMP_LO[c];
                    sat[l] = self ? xsat : COMP_SAT[c] != 0;
                }
            }
            PendulumMLPModel::tanh4_(v, 0);
#pragma unroll
            for (int l = 0; l < 4; ++l) {
                const float e = fabsf(__fsub_rn(__fsub_rn(v[l], hi[l]), lo[l]));
                if (l == P) {
                    bx |= !(e <= TANH4_ABS);
                    ex = fmaxf(ex, e);
                } else {
                    bo |= !(e <= TANH4_ABS);
                    eo = fmaxf(eo, e);
                }
                bs |= sat[l] && v[l] != 1.0f;
                const float o = __fsub_rn(fabsf(v[l]), 1.0f);           // exact near 1
                bover |= !(o <= TANH4_OVER);
                ov = fmaxf(ov, o);
            }
        }
        acc[0].note(true, bx, bits);
        acc[0].err(ex, bits);
        acc[1].note(true, bo, bits);
        acc[1].err(eo, bits);
        acc[2].note(true, bs, bits);
        acc[3].note(true, bover, bits);
        acc[3].err(ov, bits);
    }
};

// ---- normal draws ---------------------------------------------------------------------------------------------------
// oracle/philox_oracle.py: u = v 2^-32 + 2^-33 in float32, r = sqrt(-2 ln u1), n0 = r sin(2 pi u2), n1 = r cos(2 pi u2)
// in fp64.  Checks by u1: 0 u1 < 0.5, 1 0.5 <= u1 < 1 - 2^-20, 2 u1 >= 1 - 2^-20; a failure is a non-finite draw or an
// error over NORMAL_ABS.
constexpr double NORMAL_ABS = 2e-5;
__device__ __forceinline__ void normal_check(unsigned a, unsigned b, unsigned idx, Acc* acc) {
    const float u1 = (float)a * 2.3283064365386963e-10f + 1.1641532182693481e-10f;
    const float u2 = (float)b * 2.3283064365386963e-10f + 1.1641532182693481e-10f;
    const double r = sqrt(-2.0 * log((double)u1)), ang = 6.283185307179586 * (double)u2;
    float n0, n1;
    Normals<float>::pair(a, b, n0, n1);
    const double e = fmax(fabs((double)n0 - r * sin(ang)), fabs((double)n1 - r * cos(ang)));
    const int reg = u1 < 0.5f ? 0 : (u1 < 0.99999904632568359f ? 1 : 2);
    acc[reg].note(true, !finite(n0) || !finite(n1) || !(e <= NORMAL_ABS), idx);
    acc[reg].err(e != e ? INFINITY : e, idx);
}
struct NormalsA { static constexpr int NOUT = 3; unsigned b; __device__ void operator()(unsigned i, Acc* acc) const { normal_check(i, b, i, acc); } };
struct NormalsB { static constexpr int NOUT = 3; unsigned a; __device__ void operator()(unsigned i, Acc* acc) const { normal_check(a, i, i, acc); } };

// Normals<double>::pair on random 64-bit words against the same statement in fp64 (key: the input index)
struct NormalsDouble {
    static constexpr int NOUT = 1;
    __device__ void operator()(unsigned i, Acc* acc) const {
        const u64 a = splitmix64(2 * (u64)i), b = splitmix64(2 * (u64)i + 1);
        const double u1 = (double)(a >> 11) * 1.1102230246251565e-16 + 5.551115123125783e-17;
        const double u2 = (double)(b >> 11) * 1.1102230246251565e-16 + 5.551115123125783e-17;
        const double r = sqrt(-2.0 * log(u1)), ang = 6.283185307179586 * u2;
        double n0, n1;
        Normals<double>::pair(a, b, n0, n1);
        const double e = fmax(fabs(n0 - r * sin(ang)), fabs(n1 - r * cos(ang)));
        acc[0].note(true, !(e <= 1e-13), i);
        acc[0].err(e, i);
    }
};

// ---- bf16 split -----------------------------------------------------------------------------------------------------
// round to nearest even of a float's bits to bf16 (the rule for every non-NaN float)
__device__ __forceinline__ unsigned short bf16_rn(float x) {
    const unsigned u = __float_as_uint(x);
    return (unsigned short)((u + 0x7FFFu + ((u >> 16) & 1u)) >> 16);
}
__device__ __forceinline__ float bf16_f(unsigned short h) { return __uint_as_float((unsigned)h << 16); }
__device__ __forceinline__ unsigned short bits16(__nv_bfloat16 h) { return __bfloat16_as_ushort(h); }
// checks over every finite x: 0 split_bf16 gives hi = bf16_rn(x), lo = bf16_rn(x - hi) bit for bit; 1 the residual
// |x - hi - lo| <= max(2^-17 |x|, 2^-134) unless hi is inf (error: the residual over |x|, for |x| >= 2^-110, where lo
// is a normal bf16); 2 to_operand<1> on h[i] = x (even i), -x (odd i): every half of hi and lo is the rule's.
struct Bf16Scan {
    static constexpr int NOUT = 3;
    __device__ void operator()(unsigned i, Acc* acc) const {
        const float x = __uint_as_float(i);
        if (!finite(x)) return;
        __nv_bfloat16 h, l;
        tc::split_bf16(x, h, l);
        const unsigned short wh = bf16_rn(x), wl = bf16_rn(x - bf16_f(wh));
        acc[0].note(true, bits16(h) != wh || bits16(l) != wl, i);
        const float hf = __bfloat162float(h), lf = __bfloat162float(l);
        if (finite(hf)) {
            const double res = fabs((double)x - (double)hf - (double)lf);
            acc[1].note(true, !(res <= fmax(7.62939453125e-06 * fabs((double)x), 4.591774807899561e-41)), i);
            if (fabsf(x) >= 7.703719777548943e-34f) acc[1].err(res / fabs((double)x), i);
        }
        float v[16];
        for (int k = 0; k < 16; ++k) v[k] = (k & 1) ? -x : x;
        uint32_t hi[2][4], lo[2][4];
        tc::to_operand<1>(v, hi, lo);
        const unsigned short nh = bf16_rn(-x), nl = bf16_rn(-x - bf16_f(nh));
        const uint32_t want_hi = ((uint32_t)nh << 16) | wh, want_lo = ((uint32_t)nl << 16) | wl;
        bool ok = true;
        for (int s = 0; s < 2; ++s)
            for (int r = 0; r < 4; ++r) ok = ok && hi[s][r] == want_hi && lo[s][r] == want_lo;
        acc[2].note(true, !ok, i);
    }
};

// ---- entry points (device pointers; out: 4 words per check, zeroed but for the third word of each, all ones) -------
extern "C" {
int set_companions(const float* value, const float* hi, const float* lo, const int* sat) {     // host arrays of 12
    int e = (int)cudaMemcpyToSymbol(COMP, value, sizeof(float) * 12);
    if (!e) e = (int)cudaMemcpyToSymbol(COMP_HI, hi, sizeof(float) * 12);
    if (!e) e = (int)cudaMemcpyToSymbol(COMP_LO, lo, sizeof(float) * 12);
    if (!e) e = (int)cudaMemcpyToSymbol(COMP_SAT, sat, sizeof(int) * 12);
    return e;
}
int scan_fmod(float b, u64* out) { return run(FmodScan{b}, 1ull << 32, out); }
int scan_fmod_random(u64* out) { return run(FmodRandom{}, 1ull << 32, out); }
int scan_tanh(u64* out) { return run(TanhScan{}, 1ull << 32, out); }
// lane 0..3; shift 0 scans every float, shift s > 0 one float in 2^s
int scan_tanh4(int lane, int shift, u64* out) {
    const u64 n = 1ull << (32 - shift);
    switch (lane) {
        case 0: return run(Tanh4Triples<0>{shift}, n, out);
        case 1: return run(Tanh4Triples<1>{shift}, n, out);
        case 2: return run(Tanh4Triples<2>{shift}, n, out);
        default: return run(Tanh4Triples<3>{shift}, n, out);
    }
}
int scan_normals_a(unsigned b, u64* out) { return run(NormalsA{b}, 1ull << 32, out); }
int scan_normals_b(unsigned a, u64* out) { return run(NormalsB{a}, 1ull << 32, out); }
int scan_normals_double(u64 n, u64* out) { return run(NormalsDouble{}, n, out); }
int scan_bf16(u64* out) { return run(Bf16Scan{}, 1ull << 32, out); }
}

__global__ void remainder_kernel(const float* a, const float* b, float* out, int n, int small) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = small ? remainder<float, true>(a[i], b[i]) : remainder<float>(a[i], b[i]);
}
__global__ void tanh4_kernel(const float* in, float* out, int n, int mode) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float v[4] = {in[4 * i], in[4 * i + 1], in[4 * i + 2], in[4 * i + 3]};
    PendulumMLPModel::tanh4_(v, mode);
    for (int l = 0; l < 4; ++l) out[4 * i + l] = v[l];
}
__global__ void split_kernel(const float* x, unsigned short* hi, unsigned short* lo, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    __nv_bfloat16 h, l;
    tc::split_bf16(x[i], h, l);
    hi[i] = bits16(h);
    lo[i] = bits16(l);
}
__global__ void to_operand_kernel(const float* h16, uint32_t* out16) {
    float h[16];
    for (int k = 0; k < 16; ++k) h[k] = h16[k];
    uint32_t hi[2][4], lo[2][4];
    tc::to_operand<1>(h, hi, lo);
    for (int k = 0; k < 8; ++k) {
        out16[k] = hi[k >> 2][k & 3];
        out16[8 + k] = lo[k >> 2][k & 3];
    }
}
__global__ void normals_double_kernel(const u64* a, const u64* b, double* out, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) Normals<double>::pair(a[i], b[i], out[2 * i], out[2 * i + 1]);
}
__global__ void philox_kernel(const u64* seed, const u64* subseq, const u64* offset, unsigned* out, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const U4 v = philox4x32_10(seed[i], subseq[i], offset[i]);
    out[4 * i] = v.x; out[4 * i + 1] = v.y; out[4 * i + 2] = v.z; out[4 * i + 3] = v.w;
}
static unsigned blocks(int n) { return (unsigned)((n + 255) / 256); }
extern "C" {
int remainder_array(const float* a, const float* b, float* out, int n, int small) {
    remainder_kernel<<<blocks(n), 256>>>(a, b, out, n, small);
    return (int)cudaDeviceSynchronize();
}
int tanh4_groups(const float* in, float* out, int n, int mode) {
    tanh4_kernel<<<blocks(n), 256>>>(in, out, n, mode);
    return (int)cudaDeviceSynchronize();
}
int split_array(const float* x, unsigned short* hi, unsigned short* lo, int n) {
    split_kernel<<<blocks(n), 256>>>(x, hi, lo, n);
    return (int)cudaDeviceSynchronize();
}
int to_operand_markers(const float* h16, uint32_t* out16) {
    to_operand_kernel<<<1, 1>>>(h16, out16);
    return (int)cudaDeviceSynchronize();
}
int normals_double(const u64* a, const u64* b, double* out, int n) {
    normals_double_kernel<<<blocks(n), 256>>>(a, b, out, n);
    return (int)cudaDeviceSynchronize();
}
int philox_array(const u64* seed, const u64* subseq, const u64* offset, unsigned* out, int n) {
    philox_kernel<<<blocks(n), 256>>>(seed, subseq, offset, out, n);
    return (int)cudaDeviceSynchronize();
}
}
"""


def build(directory):
    """Compile the probe into `directory`/libdevice_math_probe.so with the library's nvcc flags; returns its path."""
    from pytorch_mppi_b200 import build as libbuild
    src = os.path.join(str(directory), "device_math_probe.cu")
    lib = os.path.join(str(directory), "libdevice_math_probe.so")
    with open(src, "w") as f:
        f.write(SRC)
    nvcc = os.environ.get("NVCC", "nvcc")
    r = subprocess.run([nvcc, *libbuild.NVCC_FLAGS, "-shared", "-I", CSRC, src, "-o", lib], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed on the device-math probe:\n{r.stderr[-4000:]}")
    return lib
