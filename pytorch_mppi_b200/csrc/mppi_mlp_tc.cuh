// mppi_mlp_tc.cuh — tensor-core variant of the fused command kernel for the learned pendulum model
// (BASELINE config 4: 3-32-32-2 tanh residual MLP, tests/pendulum_approximate.py:47-67 of the reference).
//
// The network's hidden and output layers are dense contractions, so per rollout step a CTA of 128 samples (two
// warpgroups of 64 rows) runs them as Hopper warpgroup MMAs (wgmma.mma_async, bf16 operands, fp32 accumulate):
//   layer 1 (3 inputs -> 32 units, 96 FMAs per sample) on the FP32 pipe, in exact fp32, computed straight into the
//     register fragment a wgmma A operand expects (rows g and g + 8 of the warp's 16, columns 2t, 2t + 1, 2t + 8, 2t + 9
//     of every 16-wide K step) -> tanh -> bf16 A registers
//   layer 2: m64n32k16 wgmmas, A from registers, W2 from shared memory (descriptor, K-major, no swizzle), accumulators
//     initialised with the fp32 bias -> tanh.  The f32 accumulator fragment of an m64nN wgmma is, column pair by column
//     pair, the bf16 A fragment of the next one, so layer 3's operand never leaves the registers
//   layer 3: m64n8k16 wgmmas (outputs 0 and 1, W3 rows 2..7 zero) -> the two state increments of rows g and g + 8 in
//     the lane with t = 0 -> shared memory -> the sample's thread, which owns the state, the action and the cost.
// Two CTA barriers per step: the inputs of layer 1 (x, clamped u of every sample) and the outputs of layer 3.  The
// running cost of the state a step produced is evaluated one step LATER, in the shadow of the layer-2 MMAs (same
// values, same summation order).  Everything else (sampling, clamp, cost, the warp-fold softmin tail) is the code of
// mppi_fused.cuh.
//
// Precision: operands are bf16.  In the default (SPLIT) mode activations and weights are split into hi + lo bf16
// parts and each layer is issued as  a_hi*w_hi + a_lo*w_hi + a_hi*w_lo  ("3 x bf16"), which brings the layer outputs to
// ~2^-16 relative accuracy instead of bf16's 2^-8; the biases are added in fp32 (accumulator initial value).
#pragma once

#include <cuda_bf16.h>
#include "mppi_fused.cuh"

namespace mppi {

#if defined(__CUDACC__)

namespace tc {

constexpr int H = 32;             // hidden width
constexpr int CH = 128;           // bytes of one 8-row x 16-byte core matrix

// weight tiles in shared memory: canonical K-major / no-swizzle layout of N rows x 32 K; core matrix (row group g, k-chunk
// c) at g * SBO + c * LBO, rows 16 B apart inside a core, LBO = 128 B (adjacent k-chunks), SBO = 4 * 128 B (row groups)
__device__ __forceinline__ int tile_off(int row, int k) { return (row >> 3) * (4 * CH) + (k >> 3) * CH + (row & 7) * 16 + (k & 7) * 2; }

// GmmaDescriptor (sm_90): start >> 4 [0,14) | LBO >> 4 [16,30) | SBO >> 4 [32,46) | base offset 0 | layout 0 (no swizzle)
__device__ __forceinline__ uint64_t smem_desc(const void* base) {
    const uint64_t addr = (uint64_t)(smem_u32(base) >> 4) & 0x3FFF;
    return addr | ((uint64_t)(CH >> 4) << 16) | ((uint64_t)((4 * CH) >> 4) << 32);
}
constexpr uint64_t KSTEP = (2 * CH) >> 4;        // one K = 16 step = two 8-element k-chunks, in 16-byte units

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accesses of an accumulator register across the asynchronous MMA window
template <int N> __device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// d(64 x 32) += a(64 x 16, registers) * B(16 x 32, shared memory)
__device__ __forceinline__ void wgmma_n32(float (&d)[16], const uint32_t (&a)[4], uint64_t b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
}
// d(64 x 8) += a(64 x 16, registers) * B(16 x 8, shared memory)
__device__ __forceinline__ void wgmma_n8(float (&d)[4], const uint32_t (&a)[4], uint64_t b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n8k16.f32.bf16.bf16 {%0, %1, %2, %3}, {%4, %5, %6, %7}, %8, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
}

__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
    hi = __float2bfloat16_rn(x);
    lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}
// two floats -> packed bf16 pair (a in the low half): one cvt.rn.bf16x2.f32
__device__ __forceinline__ uint32_t cvt2(float a, float b) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
    return r;
}

// 32 activations in accumulator order (h[4j + 0/1]: row g, columns 8j + 2t, +1; h[4j + 2/3]: row g + 8, same columns)
// -> the A fragments of the two K = 16 steps: a[s] = {(g, 16s + 2t..), (g + 8, 16s + 2t..), (g, 16s + 8 + 2t..),
// (g + 8, 16s + 8 + 2t..)} — the same registers in the same order.  SPLIT: lo = bf16(h - hi).
template <int SPLIT> __device__ __forceinline__ void to_operand(const float (&h)[16], uint32_t (&hi)[2][4], uint32_t (&lo)[2][4]) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const uint32_t v = cvt2(h[2 * i], h[2 * i + 1]);
        hi[i >> 2][i & 3] = v;
        if (SPLIT) lo[i >> 2][i & 3] = cvt2(h[2 * i] - __uint_as_float(v << 16), h[2 * i + 1] - __uint_as_float(v & 0xFFFF0000u));
    }
}

}  // namespace tc

// =================================================================================================
template <int VARIANT, int SPLIT, int FAST>
__global__ void __launch_bounds__(256, 2) mlp_tc_command_kernel(const __grid_constant__ KArgs<float> a,
                                                             const __grid_constant__ PendulumMLPModel::P<float> mp) {
    typedef float real;
    typedef Ops<real> O;
    typedef PendulumMLPModel Model;
    constexpr int NX = 2, NU = 1, H = tc::H;
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ __align__(128) unsigned char sW2[32 * H * 2];                    // B of layer 2: N = 32 x K = 32
    __shared__ __align__(128) unsigned char sW3[8 * H * 2];                     // B of layer 3: N = 8 (rows 2..7 zero)
    __shared__ __align__(128) unsigned char sW2lo[SPLIT ? 32 * H * 2 : 128];    // w_lo tiles, SPLIT only
    __shared__ __align__(128) unsigned char sW3lo[SPLIT ? 8 * H * 2 : 128];
    __shared__ __align__(16) float sX[128 * 4];                                 // (x0, x1, clamped u) of every sample: layer 1's input
    __shared__ __align__(16) float sO[128 * 2];                                 // layer 3's output of every sample
    const int tid = threadIdx.x, BD = blockDim.x;      // BD == 256: thread = (sample row tid % 128, half tid / 128)
    const int row = tid & 127, half = tid >> 7;
    // wgmma fragment of this thread: rows r0 = 64 * warpgroup + 16 * (warp % 4) + g and r0 + 8, column pairs 2t (+ 8j)
    const int lane = tid & 31, g = lane >> 2, t4 = lane & 3;
    const int r0 = 64 * half + 16 * ((tid >> 5) & 3) + g, r1 = r0 + 8;
    const int BS = BD / a.tps;
    const int xst = fused_xstage_doubles(a.world > 1 && !a.export_partial, a.world, a.xchg_npub, a.R);
    const int cs_ = (int)cluster_nctarank();
    const SmemLayout L = make_layout<real>(VARIANT, a.T, NU, a.S, a.R, BD, BS, fused_layout_nb((int)gridDim.x / cs_, a.xchg_npub),
                                           layout_extra(0, 0, cs_, xst));
    Smem<real> sm(smem, L);
    warp_records_init<real>(a, sm);      // published by the first barrier of the setup
    if (cs_ > 1) cluster_arrive_relaxed();   // phase 0 of the cluster barrier, as in fused_command_kernel
    const NoiseModel<real>& nm = a.nm;
    const int T = a.T;

    // ---- one-time setup: bf16 weight tiles (hi/lo split) --------------------------------------------------------------
    // The weights are kernel parameters (constant bank), cold in this SM's constant cache at every launch: every thread
    // requests its words first (all lines in flight while the tiles are zeroed) and parks them in shared memory, which
    // the tile build and the per-step layer-1 loads read.
    constexpr int NPW = (int)(sizeof(PendulumMLPModel::P<float>) / 4);
    __shared__ __align__(16) float sP[NPW];
    float pw_reg[(NPW + 255) / 256];
    {
        const float* pw = reinterpret_cast<const float*>(&mp);
#pragma unroll
        for (int i = 0; i < (NPW + 255) / 256; ++i) pw_reg[i] = tid + i * 256 < NPW ? pw[tid + i * 256] : 0.0f;
    }
    for (int i = tid; i < 8 * H * 2 / 4; i += BD) {
        reinterpret_cast<uint32_t*>(sW3)[i] = 0u;
        if (SPLIT) reinterpret_cast<uint32_t*>(sW3lo)[i] = 0u;
    }
#pragma unroll
    for (int i = 0; i < (NPW + 255) / 256; ++i)
        if (tid + i * 256 < NPW) sP[tid + i * 256] = pw_reg[i];
    __syncthreads();
    const PendulumMLPModel::P<float>& ms = *reinterpret_cast<const PendulumMLPModel::P<float>*>(sP);
    for (int e = tid; e < H * H; e += BD) {
        const int n = e / H, k = e - n * H;
        __nv_bfloat16 wh, wl;
        tc::split_bf16(ms.W2[k * H + n], wh, wl);                 // W2t[k][n] = W2[n][k]
        reinterpret_cast<__nv_bfloat16*>(sW2)[tc::tile_off(n, k) / 2] = wh;
        if (SPLIT) reinterpret_cast<__nv_bfloat16*>(sW2lo)[tc::tile_off(n, k) / 2] = wl;
    }
    for (int e = tid; e < 2 * H; e += BD) {
        const int n = e / H, k = e - n * H;
        __nv_bfloat16 wh, wl;
        tc::split_bf16(ms.W3[n * H + k], wh, wl);
        reinterpret_cast<__nv_bfloat16*>(sW3)[tc::tile_off(n, k) / 2] = wh;
        if (SPLIT) reinterpret_cast<__nv_bfloat16*>(sW3lo)[tc::tile_off(n, k) / 2] = wl;
    }
    // the tiles are read by the async proxy (wgmma)
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    const uint64_t dW2 = tc::smem_desc(sW2), dW3 = tc::smem_desc(sW3), dW2lo = tc::smem_desc(sW2lo), dW3lo = tc::smem_desc(sW3lo);
    // fp32 biases in accumulator order
    float b2f[8], b3f[2];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        b2f[2 * j] = ms.b2[8 * j + 2 * t4];
        b2f[2 * j + 1] = ms.b2[8 * j + 2 * t4 + 1];
    }
    b3f[0] = t4 == 0 ? ms.b3[0] : 0.0f;
    b3f[1] = t4 == 0 ? ms.b3[1] : 0.0f;

    stage_issue<real, VARIANT, NU>(a, sm);
    bool staged = false;

    // Tile = 128 samples; the two threads of a sample share its draws and its colour/clamp pass (a.tps == 2), thread 0
    // of the pair (half 0, warps 0-3) carries the state and the cost.
    const bool roller = half == 0;                     // warp-uniform
    for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
        const int k = tile * BS + (tid % BS);
        const bool in_range = k < a.K;
        const bool active = in_range && roller;
        const int nvalid = min(BS, a.K - tile * BS);
        const unsigned long long kg = (unsigned long long)(a.k_offset + k);
        fill_normals<real>(a, sm, tile, in_range, kg, nvalid);
        if (!staged) {
            stage_finish<real, VARIANT, NU>(a, sm);
            staged = true;
        } else {
            __syncthreads();
        }
        if (in_range) transform_column<real, VARIANT, NU>(a, sm, kg);
        __syncthreads();

        // ---- rollout: the MMAs are warpgroup-wide, so every thread keeps the step's two barriers ---------------------
        real x[NX] = {(real)0, (real)0};
        if (active) initial_state<real, NX>(a, k, x);
        real roll = (real)0, pert = (real)0, smooth = (real)0, vprev = (real)0, u_prev = (real)0;
        for (int t = 0; t < T; ++t) {
            real v[NU] = {(real)0}, eps[NU] = {(real)0};
            real u = (real)0;
            if (roller) {
                if (active) {
                    action_at<real, VARIANT, NU>(a, sm, kg, t, v);
                    noise_at<real, VARIANT, NU>(a, sm, t, v, eps);
                }
                u = O::mul(nm.u_scale, v[0]);
                const real uc = clamp<real>(u, -mp.max_torque, mp.max_torque);
                *reinterpret_cast<float4*>(sX + 4 * row) = make_float4(x[0], x[1], uc, 0.0f);
            }
            __syncthreads();
            uint32_t ahi[2][4], alo[2][4];
            float h[16];
            {   // layer 1 on the FP32 pipe (exact fp32): rows r0, r1 x columns 8j + 2t, +1 -> tanh -> layer 2's A fragments
                const float4 xa = *reinterpret_cast<const float4*>(sX + 4 * r0);
                const float4 xb = *reinterpret_cast<const float4*>(sX + 4 * r1);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int c = 8 * j + 2 * t4;
                    const float2 w0 = *reinterpret_cast<const float2*>(ms.W1 + 0 * H + c);
                    const float2 w1 = *reinterpret_cast<const float2*>(ms.W1 + 1 * H + c);
                    const float2 w2 = *reinterpret_cast<const float2*>(ms.W1 + 2 * H + c);
                    const float2 bb = *reinterpret_cast<const float2*>(ms.b1 + c);
                    h[4 * j + 0] = fmaf(w2.x, xa.z, fmaf(w1.x, xa.y, fmaf(w0.x, xa.x, bb.x)));
                    h[4 * j + 1] = fmaf(w2.y, xa.z, fmaf(w1.y, xa.y, fmaf(w0.y, xa.x, bb.y)));
                    h[4 * j + 2] = fmaf(w2.x, xb.z, fmaf(w1.x, xb.y, fmaf(w0.x, xb.x, bb.x)));
                    h[4 * j + 3] = fmaf(w2.y, xb.z, fmaf(w1.y, xb.y, fmaf(w0.y, xb.x, bb.y)));
                }
#pragma unroll
                for (int i = 0; i < 16; i += 4) Model::tanh4_(h + i, FAST);
                tc::to_operand<SPLIT>(h, ahi, alo);
            }
            // layer 2: accumulators start at the bias
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                h[4 * j + 0] = h[4 * j + 2] = b2f[2 * j];
                h[4 * j + 1] = h[4 * j + 3] = b2f[2 * j + 1];
            }
            tc::fence_regs(h);
            tc::wgmma_fence();
#pragma unroll
            for (int s = 0; s < 2; ++s) {
                tc::wgmma_n32(h, ahi[s], dW2 + s * tc::KSTEP);
                if (SPLIT) {
                    tc::wgmma_n32(h, alo[s], dW2 + s * tc::KSTEP);
                    tc::wgmma_n32(h, ahi[s], dW2lo + s * tc::KSTEP);
                }
            }
            tc::wgmma_commit();
            // in the shadow of the layer-2 MMAs: the running cost of the state the PREVIOUS step produced (x is x_t, the
            // state step t-1 led to) and this step's action cost — same values and summation order as the plain loop
            if (active) {
                if (t > 0) roll = O::add(roll, Model::template cost<real>(mp, x, &u_prev));   // mppi.py:318-319 (step t-1)
                pert = O::add(pert, action_cost_term<real, NU>(nm, eps, sm.Us + t * NU));
                if (VARIANT == V_SMPPI) {
                    if (t > 0) {
                        const real d = O::mul(nm.u_scale, O::sub(v[0], vprev));
                        smooth = O::add(smooth, O::mul(d, d));
                    }
                    vprev = v[0];
                }
            }
            u_prev = u;
            tc::wgmma_wait();
            tc::fence_regs(h);
            // layer 2 -> tanh -> layer 3's A fragments (the accumulator fragment, repacked in place)
#pragma unroll
            for (int i = 0; i < 16; i += 4) Model::tanh4_(h + i, FAST);
            tc::to_operand<SPLIT>(h, ahi, alo);
            float o[4] = {b3f[0], b3f[1], b3f[0], b3f[1]};
            tc::fence_regs(o);
            tc::wgmma_fence();
#pragma unroll
            for (int s = 0; s < 2; ++s) {
                tc::wgmma_n8(o, ahi[s], dW3 + s * tc::KSTEP);
                if (SPLIT) {
                    tc::wgmma_n8(o, alo[s], dW3 + s * tc::KSTEP);
                    tc::wgmma_n8(o, ahi[s], dW3lo + s * tc::KSTEP);
                }
            }
            tc::wgmma_commit();
            tc::wgmma_wait();
            tc::fence_regs(o);
            if (t4 == 0) {
                *reinterpret_cast<float2*>(sO + 2 * r0) = make_float2(o[0], o[1]);
                *reinterpret_cast<float2*>(sO + 2 * r1) = make_float2(o[2], o[3]);
            }
            __syncthreads();
            if (roller) {
                const float2 d = *reinterpret_cast<const float2*>(sO + 2 * row);
                const real th = O::add(x[0], d.x);
                x[0] = O::sub(remainder<real>(O::add(th, mp.pi), mp.two_pi), mp.pi);    // pendulum_approximate.py:65
                x[1] = O::add(x[1], d.y);
            }
        }
        if (active) roll = O::add(roll, Model::template cost<real>(mp, x, &u_prev));              // step T-1
        real c_tot = O::inf();
        if (active) {
            c_tot = O::add(roll, pert);
            if (VARIANT == V_SMPPI) c_tot = O::add(c_tot, O::mul(smooth, nm.w_smooth));
            a.cost_total[k] = c_tot;
        }
        if (roller) warp_fold<real, VARIANT, false>(a, sm, c_tot, active, nvalid);
        if (tile + (int)gridDim.x < a.n_tiles) __syncthreads();      // the tile is refilled by the next pass
    }
    if (!staged) stage_finish<real, VARIANT, NU>(a, sm);
    warp_tail<real, VARIANT, NU>(a, sm);
}

// =================================================================================================
// The ensemble (PendulumMLPEnsembleModel, rollout_samples = M networks, one per copy) on the same tiles.  Setup: every
// copy's network is staged once per CTA from the device table into dynamic shared memory (PendulumMLPEnsembleModel::TC_*:
// bf16 hi / lo tiles of W2 and W3, fp32 W1, b1, b2, b3).  Per step: the roller thread of a sample writes its clamped
// action (its M states already sit in the copies' layer-1 input rows), one barrier, then for each copy m the warpgroups
// run the network of mlp_tc_command_kernel on copy m's tiles into copy m's outputs, one barrier, and the roller updates
// its M states in place.  Two barriers per step whatever M is.  The roller evaluates the M running costs of the states a
// step produced one step later (as copies_rollout does) and folds them with copies_fold; after the loop,
// (mean + var * rollout_var_cost) + perturbation (+ SMPPI smoothness).
// M is a run-time value: the loop over the copies' networks stays rolled (nothing in it is indexed by m in registers),
// and the roller's cost sums are unrolled to MPPI_MAX_COPIES with guards, so they stay in registers — one kernel per
// (variant, operand mode, tanh) serves every M.  (With the M states in registers too, 4 of the 12 instantiations spilled
// 4 B at this launch bound's 128-register cap; now none spills.)
template <int VARIANT, int SPLIT, int FAST>
__global__ void __launch_bounds__(256, 2) mlp_ens_tc_command_kernel(const __grid_constant__ KArgs<float> a,
                                                                 const __grid_constant__ PendulumMLPEnsembleModel::P<float> mp) {
    typedef float real;
    typedef Ops<real> O;
    typedef PendulumMLPEnsembleModel Model;
    constexpr int NX = 2, NU = 1, H = tc::H, MC = Model::COPIES;
    extern __shared__ __align__(16) unsigned char smem[];
    const int tid = threadIdx.x, BD = blockDim.x;      // BD == 256: thread = (sample row tid % 128, half tid / 128)
    const int row = tid & 127, half = tid >> 7;
    const int lane = tid & 31, g = lane >> 2, t4 = lane & 3;
    const int r0 = 64 * half + 16 * ((tid >> 5) & 3) + g, r1 = r0 + 8;
    const int BS = BD / a.tps;
    const int xst = fused_xstage_doubles(a.world > 1 && !a.export_partial, a.world, a.xchg_npub, a.R);
    const int cs_ = (int)cluster_nctarank();
    const SmemLayout L = make_layout<real>(VARIANT, a.T, NU, a.S, a.R, BD, BS, fused_layout_nb((int)gridDim.x / cs_, a.xchg_npub),
                                           layout_extra(0, 0, cs_, xst));
    Smem<real> sm(smem, L);
    warp_records_init<real>(a, sm);      // published by the first barrier of the setup
    if (cs_ > 1) cluster_arrive_relaxed();   // phase 0 of the cluster barrier, as in fused_command_kernel
    const NoiseModel<real>& nm = a.nm;
    const int T = a.T, M = mp.M;
    // per-copy blocks behind the layout (the host adds Model::tc_smem_bytes(M) to the launch's dynamic shared memory)
    unsigned char* const ens = smem + align_up(L.total, 128);
    float* const sU = reinterpret_cast<float*>(ens + M * Model::TC_COPY);       // clamped action of every sample

    // ---- one-time setup: every copy's network from the table -----------------------------------------------------------
    for (int i = tid; i < M * (8 * H * 2 / 4); i += BD) {                      // W3 tiles: rows 2..7 stay zero
        unsigned char* cp = ens + (i / (8 * H * 2 / 4)) * Model::TC_COPY;
        const int j = i % (8 * H * 2 / 4);
        reinterpret_cast<uint32_t*>(cp + Model::TC_W3)[j] = 0u;
        reinterpret_cast<uint32_t*>(cp + Model::TC_W3LO)[j] = 0u;
    }
    __syncthreads();
    for (int e = tid; e < M * H * H; e += BD) {
        const int m = e / (H * H), nk = e - m * H * H, n = nk / H, k = nk - n * H;
        unsigned char* cp = ens + m * Model::TC_COPY;
        __nv_bfloat16 wh, wl;
        tc::split_bf16(__ldg(mp.w + (size_t)m * Model::N_W + Model::OFF_W2 + nk), wh, wl);     // W2[n][k]
        reinterpret_cast<__nv_bfloat16*>(cp + Model::TC_W2)[tc::tile_off(n, k) / 2] = wh;
        reinterpret_cast<__nv_bfloat16*>(cp + Model::TC_W2LO)[tc::tile_off(n, k) / 2] = wl;
    }
    for (int e = tid; e < M * 2 * H; e += BD) {
        const int m = e / (2 * H), nk = e - m * 2 * H, n = nk / H, k = nk - n * H;
        unsigned char* cp = ens + m * Model::TC_COPY;
        __nv_bfloat16 wh, wl;
        tc::split_bf16(__ldg(mp.w + (size_t)m * Model::N_W + Model::OFF_W3 + nk), wh, wl);     // W3[n][k]
        reinterpret_cast<__nv_bfloat16*>(cp + Model::TC_W3)[tc::tile_off(n, k) / 2] = wh;
        reinterpret_cast<__nv_bfloat16*>(cp + Model::TC_W3LO)[tc::tile_off(n, k) / 2] = wl;
    }
    for (int e = tid; e < M * H; e += BD) {
        const int m = e / H, i = e - m * H;
        const float* w = mp.w + (size_t)m * Model::N_W;
        unsigned char* cp = ens + m * Model::TC_COPY;
        float* w1 = reinterpret_cast<float*>(cp + Model::TC_W1);
#pragma unroll
        for (int c = 0; c < 3; ++c) w1[c * H + i] = __ldg(w + 3 * i + c);                         // W1t[c][i] = W1[i][c]
        reinterpret_cast<float*>(cp + Model::TC_B1)[i] = __ldg(w + Model::OFF_B1 + i);
        reinterpret_cast<float*>(cp + Model::TC_B2)[i] = __ldg(w + Model::OFF_B2 + i);
        if (i < 2) reinterpret_cast<float*>(cp + Model::TC_B3)[i] = __ldg(w + Model::OFF_B3 + i);
    }
    // the tiles are read by the async proxy (wgmma)
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();

    stage_issue<real, VARIANT, NU>(a, sm);
    bool staged = false;

    const bool roller = half == 0;                     // warp-uniform
    for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
        const int k = tile * BS + (tid % BS);
        const bool in_range = k < a.K;
        const bool active = in_range && roller;
        const int nvalid = min(BS, a.K - tile * BS);
        const unsigned long long kg = (unsigned long long)(a.k_offset + k);
        fill_normals<real>(a, sm, tile, in_range, kg, nvalid);
        if (!staged) {
            stage_finish<real, VARIANT, NU>(a, sm);
            staged = true;
        } else {
            __syncthreads();
        }
        if (in_range) transform_column<real, VARIANT, NU>(a, sm, kg);
        __syncthreads();

        // ---- rollout of the M copies: the MMAs are warpgroup-wide, so every thread keeps the step's two barriers -------
        // The M states live in the copies' layer-1 input rows (TC_X), which only the sample's roller writes: x(m) is its
        // copy-m state, read and updated there after the step's second barrier.
        auto xrow = [&](int m) -> float2& { return reinterpret_cast<float2*>(ens + m * Model::TC_COPY + Model::TC_X)[row]; };
        if (roller) {
            real x[NX] = {(real)0, (real)0};
            if (active) initial_state<real, NX>(a, k, x);
#pragma unroll
            for (int m = 0; m < MC; ++m)
                if (m < M) xrow(m) = make_float2(x[0], x[1]);
        }
        real cs[MC];
#pragma unroll
        for (int m = 0; m < MC; ++m) cs[m] = (real)0;
        real var = (real)0, pert = (real)0, smooth = (real)0, vprev = (real)0, u_prev = (real)0;
        for (int t = 0; t < T; ++t) {
            real v[NU] = {(real)0}, eps[NU] = {(real)0};
            real u = (real)0;
            if (roller) {
                if (active) {
                    action_at<real, VARIANT, NU>(a, sm, kg, t, v);
                    noise_at<real, VARIANT, NU>(a, sm, t, v, eps);
                }
                u = O::mul(nm.u_scale, v[0]);
                sU[row] = clamp<real>(u, -mp.max_torque, mp.max_torque);
            }
            __syncthreads();
            // the running costs of the states the PREVIOUS step produced (x_t)
            if (active) {
                if (t > 0) {
                    real c[MC];
#pragma unroll
                    for (int m = 0; m < MC; ++m) {
                        const float2 xm = xrow(m < M ? m : 0);
                        const real xv[NX] = {xm.x, xm.y};
                        c[m] = m < M ? Model::template cost<real>(mp, xv, &u_prev, m) : (real)0;
                    }
                    copies_fold<real, MC>(cs, var, c, __ldg(a.var_disc + t - 1), M);      // mppi.py:362-364 (step t-1)
                }
                pert = O::add(pert, action_cost_term<real, NU>(nm, eps, sm.Us + t * NU));
                if (VARIANT == V_SMPPI) {
                    if (t > 0) {
                        const real d = O::mul(nm.u_scale, O::sub(v[0], vprev));
                        smooth = O::add(smooth, O::mul(d, d));
                    }
                    vprev = v[0];
                }
            }
            u_prev = u;
            const float ua = sU[r0], ub = sU[r1];
#pragma unroll 1
            for (int m = 0; m < M; ++m) {
                unsigned char* cp = ens + m * Model::TC_COPY;
                const float* w1 = reinterpret_cast<const float*>(cp + Model::TC_W1);
                const float* b1 = reinterpret_cast<const float*>(cp + Model::TC_B1);
                const float* b2 = reinterpret_cast<const float*>(cp + Model::TC_B2);
                const float* b3 = reinterpret_cast<const float*>(cp + Model::TC_B3);
                uint32_t ahi[2][4], alo[2][4];
                float h[16];
                {   // layer 1 on the FP32 pipe (exact fp32): rows r0, r1 x columns 8j + 2t, +1 -> tanh -> layer 2's A fragments
                    const float2 xa = reinterpret_cast<const float2*>(cp + Model::TC_X)[r0];
                    const float2 xb = reinterpret_cast<const float2*>(cp + Model::TC_X)[r1];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const int c = 8 * j + 2 * t4;
                        const float2 w0 = *reinterpret_cast<const float2*>(w1 + 0 * H + c);
                        const float2 w1v = *reinterpret_cast<const float2*>(w1 + 1 * H + c);
                        const float2 w2 = *reinterpret_cast<const float2*>(w1 + 2 * H + c);
                        const float2 bb = *reinterpret_cast<const float2*>(b1 + c);
                        h[4 * j + 0] = fmaf(w2.x, ua, fmaf(w1v.x, xa.y, fmaf(w0.x, xa.x, bb.x)));
                        h[4 * j + 1] = fmaf(w2.y, ua, fmaf(w1v.y, xa.y, fmaf(w0.y, xa.x, bb.y)));
                        h[4 * j + 2] = fmaf(w2.x, ub, fmaf(w1v.x, xb.y, fmaf(w0.x, xb.x, bb.x)));
                        h[4 * j + 3] = fmaf(w2.y, ub, fmaf(w1v.y, xb.y, fmaf(w0.y, xb.x, bb.y)));
                    }
#pragma unroll
                    for (int i = 0; i < 16; i += 4) PendulumMLPModel::tanh4_(h + i, FAST);
                    tc::to_operand<SPLIT>(h, ahi, alo);
                }
                // layer 2: accumulators start at the bias
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 bb = *reinterpret_cast<const float2*>(b2 + 8 * j + 2 * t4);
                    h[4 * j + 0] = h[4 * j + 2] = bb.x;
                    h[4 * j + 1] = h[4 * j + 3] = bb.y;
                }
                const uint64_t dW2 = tc::smem_desc(cp + Model::TC_W2), dW2lo = tc::smem_desc(cp + Model::TC_W2LO);
                tc::fence_regs(h);
                tc::wgmma_fence();
#pragma unroll
                for (int s = 0; s < 2; ++s) {
                    tc::wgmma_n32(h, ahi[s], dW2 + s * tc::KSTEP);
                    if (SPLIT) {
                        tc::wgmma_n32(h, alo[s], dW2 + s * tc::KSTEP);
                        tc::wgmma_n32(h, ahi[s], dW2lo + s * tc::KSTEP);
                    }
                }
                tc::wgmma_commit();
                tc::wgmma_wait();
                tc::fence_regs(h);
                // layer 2 -> tanh -> layer 3's A fragments (the accumulator fragment, repacked in place)
#pragma unroll
                for (int i = 0; i < 16; i += 4) PendulumMLPModel::tanh4_(h + i, FAST);
                tc::to_operand<SPLIT>(h, ahi, alo);
                const float b30 = t4 == 0 ? b3[0] : 0.0f, b31 = t4 == 0 ? b3[1] : 0.0f;
                float o[4] = {b30, b31, b30, b31};
                const uint64_t dW3 = tc::smem_desc(cp + Model::TC_W3), dW3lo = tc::smem_desc(cp + Model::TC_W3LO);
                tc::fence_regs(o);
                tc::wgmma_fence();
#pragma unroll
                for (int s = 0; s < 2; ++s) {
                    tc::wgmma_n8(o, ahi[s], dW3 + s * tc::KSTEP);
                    if (SPLIT) {
                        tc::wgmma_n8(o, alo[s], dW3 + s * tc::KSTEP);
                        tc::wgmma_n8(o, ahi[s], dW3lo + s * tc::KSTEP);
                    }
                }
                tc::wgmma_commit();
                tc::wgmma_wait();
                tc::fence_regs(o);
                if (t4 == 0) {
                    float2* so = reinterpret_cast<float2*>(cp + Model::TC_O);
                    so[r0] = make_float2(o[0], o[1]);
                    so[r1] = make_float2(o[2], o[3]);
                }
            }
            __syncthreads();
            if (roller) {
#pragma unroll
                for (int m = 0; m < MC; ++m) {
                    if (m < M) {
                        const float2 d = reinterpret_cast<const float2*>(ens + m * Model::TC_COPY + Model::TC_O)[row];
                        float2& xm = xrow(m);
                        const real th = O::add(xm.x, d.x);
                        xm = make_float2(O::sub(remainder<real>(O::add(th, mp.pi), mp.two_pi), mp.pi),   // pendulum_approximate.py:65
                                         O::add(xm.y, d.y));
                    }
                }
            }
        }
        real c_tot = O::inf();
        if (active) {
            real c[MC];
#pragma unroll
            for (int m = 0; m < MC; ++m) {
                const float2 xm = xrow(m < M ? m : 0);
                const real xv[NX] = {xm.x, xm.y};
                c[m] = m < M ? Model::template cost<real>(mp, xv, &u_prev, m) : (real)0;
            }
            copies_fold<real, MC>(cs, var, c, __ldg(a.var_disc + T - 1), M);              // step T-1
            real mean = cs[0];
#pragma unroll
            for (int m = 1; m < MC; ++m)
                if (m < M) mean = O::add(mean, cs[m]);
            mean = O::div(mean, (real)M);                                                  // mppi.py:371
            c_tot = O::add(O::add(mean, O::mul(var, a.var_cost)), pert);                   // mppi.py:372, 416
            if (VARIANT == V_SMPPI) c_tot = O::add(c_tot, O::mul(smooth, nm.w_smooth));   // mppi.py:562,569
            a.cost_total[k] = c_tot;
        }
        if (roller) warp_fold<real, VARIANT, false>(a, sm, c_tot, active, nvalid);
        if (tile + (int)gridDim.x < a.n_tiles) __syncthreads();      // the tile is refilled by the next pass
    }
    if (!staged) stage_finish<real, VARIANT, NU>(a, sm);
    warp_tail<real, VARIANT, NU>(a, sm);
}

#endif  // __CUDACC__

}  // namespace mppi
