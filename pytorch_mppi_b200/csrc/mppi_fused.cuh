// mppi_fused.cuh — device side of the MPPI engine.
//
// fused_command_kernel: one kernel per MPPI/SMPPI/KMPPI command() for registered analytic models.
// One thread rolls out one sample; a CTA owns tiles of `blockDim.x` samples (grid-stride over tiles,
// so grid <= SMs x resident CTAs for any K).  Per tile:
//   A. standard normals -> shared-memory tile rows[R][BD+1]  (in-kernel Philox4x32-10 keyed by the
//      GLOBAL sample index, or an injected z tensor loaded coalesced)
//   B. colour with the Cholesky factor, add the nominal sequence (staged in shared memory by a TMA
//      bulk copy), clamp -> the tile now holds the perturbed actions (KMPPI: the control points)
//   C. T-step rollout with the state in registers, cost accumulated in the reference's op order
//   D. online-softmin fold of the tile into each rollout warp's running record (beta_w, eta_w, V_w[R])
// The softmin tail (warp_tail) combines the records of the grid, optionally exchanges them with peer
// GPUs through NVLink mailboxes, and writes the updated nominal sequence: `U += sum_k w_k eps_k / eta`
// lands without a second launch.
//
// sample_kernel / softmin_update_kernel: the same stages split at the Python T-loop, for arbitrary
// dynamics/cost callables (A+B with coalesced write-out; D + finish from materialised tensors).
//
// Reference lines replaced: mppi.py:232-238, 375-385, 297-332, 407-417, 254-259, 268-270
// (SMPPI :489-493, 520-570; KMPPI :617-619, 657-688).
#pragma once

#ifndef __CUDACC_RTC__
#include <cuda_runtime.h>
#endif
#include "mppi_math.cuh"

#ifndef MPPI_ROLLOUT_UNROLL
#define MPPI_ROLLOUT_UNROLL 2
#endif
// minimum resident CTAs per SM promised to ptxas for the fused kernel: 2 keeps 512-thread CTAs at 64 registers, two per
// SM — what large K wants (left unspecified, ptxas sizes the kernel for its out-of-line tail functions: 128 registers,
// one CTA per SM, and BASELINE config 5 loses 25 %); the split-cost variant (small K, one CTA per SM) lifts the cap
#ifndef MPPI_FUSED_MIN_BLOCKS
#define MPPI_FUSED_MIN_BLOCKS 2
#endif
#define MPPI_PRAGMA_(x) _Pragma(#x)
#define MPPI_UNROLL_N(n) MPPI_PRAGMA_(unroll n)

namespace mppi {

enum { V_MPPI = 0, V_SMPPI = 1, V_KMPPI = 2 };

template <typename real> struct KArgs {
    NoiseModel<real> nm;
    real u_init[MPPI_MAX_NU];
    real x0[MPPI_MAX_NX];
    const real* state_dev;
    real* U;
    real* A;
    real* theta;
    const real* W;
    const real* Wshift;
    real* cost_total;
    real* action_out;
    real* nominal_used;
    double* stats;
    const real* z;
    real* z_out;
    // workspace carve
    unsigned int* ticket;
    double* crec;                 // cluster records (n_clusters, R+2) doubles: (beta, eta, V[R])
    // multi-GPU
    unsigned long long* peers[8];
    double* partial_out;
    unsigned long long epoch;
    int rank, world, export_partial;
    int xchg_npub;                // records each rank publishes per command: its cluster records (LL mode) or 1
    unsigned int xchg_parity_words;   // 8-byte words between the two epoch parities of a record mailbox
    unsigned long long xchg_timeout_ns;
    long long* xchg_status_host;  // optional pinned host word: set to MPPI_ERR_TIMEOUT when a peer exchange timed out
    // sizes
    int K, T, S, R, TN, upc, n_tiles;
    long long k_offset;
    unsigned long long seed, offset;
    int shift, null_action, tma_ok, state_per_sample;
    int tps;   // threads cooperating on one sample's sampling/transform phases (1, 2 or 4)
    int pdl;   // launched with programmatic stream serialization
    unsigned long long torch_total;   // > 0: reproduce torch.randn's CUDA stream (256 * grid of the ATen kernel)
    unsigned long long* offset_dev;   // optional device-resident Philox counter base (CUDA-graph replays)
    unsigned long long offset_inc;
    // batched environments (MPPI_Batched, mppi.py:691-873): gridDim.y = n_env independent problems that
    // share the noise stream; per-environment buffers are strided
    int n_env;
    long long env_u_stride;      // elements between consecutive environments' U
    long long env_ws_stride;     // BYTES between consecutive environments' workspace
    unsigned long long* dbg;   // optional (grid,16) globaltimer stamps
    unsigned long long* host_mailbox;   // optional pinned host memory: [0]=epoch flag, [2..]=action values
    unsigned long long host_epoch;
    // generic-path extras (sample_kernel / softmin_update_kernel)
    // The batched fused kernels read no generic-path extras: their per-environment horizons (n_env of them, or nullptr:
    // every environment rolls out T) share the space of sample_kernel's perturbed-action output, so KArgs keeps its size.
    union {
        real* out_pa;                     // sample_kernel
        const int* env_horizon;           // batched fused kernels (mppi_plan_set_env_horizon)
    };
    real* out_noise;
    // The batched fused kernels read no generic-path extras: their per-environment noise models (n_env of them, or
    // nullptr: every environment takes `nm`) share the space of sample_kernel's KMPPI output, so KArgs keeps its size.
    union {
        real* out_noise_theta;            // sample_kernel (KMPPI)
        const NoiseModel<real>* env_nm;   // batched fused kernels (mppi_plan_set_env_params)
    };
    real* out_cost_init;
    const real* override_rows;
    int n_override, override_start;
    const real* in_cost;
    // The fused kernel of a model with COPIES > 1 (rollout_samples, mppi.py:334-373) reads none of the generic-path
    // extras: its two constants share their space, so that KArgs keeps its size and every other kernel its code.
    union {
        const real* in_eps;       // softmin_update_kernel
        real var_cost;            // COPIES > 1: rollout_var_cost (mppi.py:372)
    };
    const real* var_disc;         // COPIES > 1: (T) rollout_var_discount^t (mppi.py:174-175, 364)
};

// ---- shared-memory carve, computed identically on host and device -------------------------------
struct SmemLayout {
    int off_uraw, off_araw, off_thraw, off_us, off_as, off_ths, off_w, off_wsh, off_rows, off_rows2, off_part2, off_numd,
        off_xs, off_wrec, off_xstage, off_sqd, total;
    int LD;
};

// `extra` word of make_layout: bit 0 = rows2 tile; bits 8..15 = nx of the split-cost state buffer; bits 16..19 = cluster
// size of the warp-record area (0 = the kernel does not use the warp-fold tail); bits 20..30 = record staging of the
// finisher in units of 16 doubles (at most 8208 doubles: 8 ranks x 1026, or the 48 KB LL budget)
__host__ __device__ inline int layout_extra(int rows2, int nx_split, int cluster, int xstage_doubles) {
    return (rows2 & 1) | (nx_split << 8) | (cluster << 16) | (((xstage_doubles + 15) / 16) << 20);
}

__host__ __device__ inline int align_up(int x, int a) { return (x + a - 1) / a * a; }

// rows2 (a second TN-row tile) is only used by sample_kernel for KMPPI
// BD = threads per CTA, BS = samples per tile (BD / threads-per-sample)
// `extra`: bit 0 = rows2 needed; bits 8.. = nx of the split-cost rollout's per-step state buffer xs[T*nx][BS]
// (0 = none; see fused_command_kernel<..., SPLIT>)
// gtile: the global-tile kernels (fused_command_kernel_gtile, sample_kernel_gtile, softmin_update_kernel_gtile) keep
// the K-proportional buffers — rows, rows2 and KMPPI's W / Wshift — out of shared memory (gtile_bind)
template <typename real>
__host__ __device__ inline SmemLayout make_layout(int variant, int T, int nu, int S, int R, int BD, int BS, int nb, int extra,
                                                  bool gtile = false) {
    SmemLayout L;
    const int need_rows2 = extra & 1, nx_split = (extra >> 8) & 0xff, cluster = (extra >> 16) & 0xf, xstage = (extra >> 20) * 16;
    const int es = (int)sizeof(real);
    const int TN = T * nu, SN = S * nu, nw = BD / 32;
    int o = 16;  // [0,8): mbarrier
    L.off_uraw = o; o = align_up(o + TN * es, 16);
    L.off_araw = o; o = align_up(o + (variant == V_SMPPI ? TN : 0) * es, 16);
    L.off_thraw = o; o = align_up(o + (variant == V_KMPPI ? SN : 0) * es, 16);
    L.off_us = o; o = align_up(o + TN * es, 16);
    L.off_as = o; o = align_up(o + (variant == V_SMPPI ? TN : 0) * es, 16);
    L.off_ths = o; o = align_up(o + (variant == V_KMPPI ? SN : 0) * es, 16);
    L.off_w = o; o = align_up(o + (variant == V_KMPPI && !gtile ? T * S : 0) * es, 16);
    L.off_wsh = o; o = align_up(o + (variant == V_KMPPI && !gtile ? S * S : 0) * es, 16);
    L.LD = gtile ? BS : BS + 1;      // (the +1 column staggers shared-memory banks; in global memory rows stay aligned)
    L.off_rows = o; o = align_up(o + (gtile ? 0 : R * L.LD) * es, 16);
    L.off_rows2 = o; o = align_up(o + (need_rows2 && !gtile ? TN * L.LD : 0) * es, 16);
    L.off_part2 = o; o = align_up(o + nw * R * 8, 16);
    L.off_numd = o; o = align_up(o + (R + 2) * 8, 16);
    L.off_xs = o; o = align_up(o + T * nx_split * BS * es, 16);
    // warp-fold tail: (cluster x rollout warps) records of (R+2) doubles — slots [0, BS/32) are this CTA's own running
    // records, the cluster leader also receives its peers' through distributed shared memory
    L.off_wrec = o; o = align_up(o + cluster * (BS / 32) * (R + 2) * 8, 16);
    L.off_xstage = o; o = align_up(o + xstage * 8, 16);
    // rescale factors of combine_records and combine_narrow (every combine<> in warp_tail): one per record — the cluster's
    // warp records, the staged records, or (ticket mode: the caller passes nb = number of cluster records of the grid) the
    // records in the L2 workspace.  A new caller of combine<> must pass at most nsq records.
    {
        int nsq = cluster * (BS / 32);
        if (xstage / (R + 2) > nsq) nsq = xstage / (R + 2);
        if (nb > nsq) nsq = nb;
        L.off_sqd = o; o = align_up(o + (cluster > 0 ? nsq : 0) * 8, 16);
    }
    L.total = o;
    return L;
}

#define MPPI_XCHG_MAX_R 1024
#define MPPI_LL_STAGE_BYTES 49152                          // finisher staging budget: LL mode needs xw x clusters x (R+2) x 8 <= this
#define MPPI_LL_LOCAL_WORDS (2 * MPPI_LL_STAGE_BYTES / 8)  // words per parity of this GPU's own record mailbox (2 words per double)

// ---- global-tile kernels: every CTA's tiles in the workspace ------------------------------------------------------------
// The workspace is [ticket | cluster records | this GPU's record mailbox (two parities) | tile slices].  CTA b owns slice
// b — rows (R x BS elements), then rows2 (TN x BS) where the kernel has one — and reuses it across its grid-stride tiles.
__host__ __device__ inline long long gtile_slice_bytes(int R, int TN, int rows2, int BS, int es) {
    return ((long long)(R + (rows2 ? TN : 0)) * BS * es + 255) / 256 * 256;
}

#if defined(__CUDACC__)

// ---- mbarrier + TMA bulk copy (cp.async.bulk; SASS: UBLKCP) --------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(void* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(void* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, void* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(void* bar, uint32_t phase) {
    uint32_t done = 0;
    while (!done) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(phase)
            : "memory");
    }
}

__device__ __forceinline__ void stamp(unsigned long long* dbg, int slot) {
    if (dbg != nullptr && threadIdx.x == 0) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        dbg[(size_t)blockIdx.x * 16 + slot] = t;
    }
}

// ---- warp reductions (deterministic: fixed shuffle tree) -------------------------------------------
template <typename T> __device__ __forceinline__ T warp_min(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        T other = __shfl_xor_sync(0xffffffffu, v, o);
        v = other < v ? other : v;
    }
    return v;
}
template <typename T> __device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ---- shared-memory view ---------------------------------------------------------------------
template <typename real> struct Smem {
    unsigned long long* bar;
    real *Uraw, *Araw, *thraw, *Us, *As, *ths, *Ws, *Wsh, *rows, *rows2, *xs;
    double *part2, *numd, *wrec, *xstage, *sqd;
    int LD;
    Smem() = default;
    __device__ Smem(unsigned char* smem, const SmemLayout& L) {
        bar = reinterpret_cast<unsigned long long*>(smem);
        Uraw = reinterpret_cast<real*>(smem + L.off_uraw);
        Araw = reinterpret_cast<real*>(smem + L.off_araw);
        thraw = reinterpret_cast<real*>(smem + L.off_thraw);
        Us = reinterpret_cast<real*>(smem + L.off_us);
        As = reinterpret_cast<real*>(smem + L.off_as);
        ths = reinterpret_cast<real*>(smem + L.off_ths);
        Ws = reinterpret_cast<real*>(smem + L.off_w);
        Wsh = reinterpret_cast<real*>(smem + L.off_wsh);
        rows = reinterpret_cast<real*>(smem + L.off_rows);
        rows2 = reinterpret_cast<real*>(smem + L.off_rows2);
        part2 = reinterpret_cast<double*>(smem + L.off_part2);
        numd = reinterpret_cast<double*>(smem + L.off_numd);
        xs = reinterpret_cast<real*>(smem + L.off_xs);
        wrec = reinterpret_cast<double*>(smem + L.off_wrec);
        xstage = reinterpret_cast<double*>(smem + L.off_xstage);
        sqd = reinterpret_cast<double*>(smem + L.off_sqd);
        LD = L.LD;
    }
};

// global-tile kernels: point the tiles at this CTA's workspace slice (behind the record mailbox a.peers[0], which fill_kargs
// and make_env_args place in this environment's workspace) and KMPPI's matrices at their global copies, read in place.
// Only plain loads and stores reach the slice: it is written and read within the kernel, so never through ld.global.nc.
template <typename real>
__device__ __forceinline__ void gtile_bind(const KArgs<real>& a, Smem<real>& sm, int rows2) {
    const int BS = blockDim.x / a.tps;
    unsigned char* region = reinterpret_cast<unsigned char*>(a.peers[0]) + 2ull * MPPI_LL_LOCAL_WORDS * 8;
    real* base = reinterpret_cast<real*>(region + (size_t)blockIdx.x * gtile_slice_bytes(a.R, a.TN, rows2, BS, (int)sizeof(real)));
    sm.rows = base;
    sm.rows2 = base + (size_t)a.R * BS;
    sm.Ws = const_cast<real*>(a.W);
    sm.Wsh = const_cast<real*>(a.Wshift);
}

// ---- stage 0: nominal sequence(s) into shared memory, shift folded in ----------------------------
// stage_issue starts the (asynchronous) TMA bulk copy; stage_finish waits for it and builds the
// shifted nominal.  The first tile's Philox draws run in between, hiding the global-memory latency.
template <typename real, int VARIANT, int NU>
__device__ void stage_issue(const KArgs<real>& a, Smem<real>& sm) {
    const int tid = threadIdx.x, BD = blockDim.x;
    const int T = a.T, S = a.S, R = a.R, TN = a.TN;
    if (tid == 0) mbar_init(sm.bar, 1);
    __syncthreads();
    if (a.tma_ok) {
        if (tid == 0) {
            const uint32_t bytes = (uint32_t)align_up(TN * (int)sizeof(real), 16);
            mbar_expect_tx(sm.bar, VARIANT == V_SMPPI ? 2 * bytes : bytes);
            tma_bulk_g2s(sm.Uraw, a.U, bytes, sm.bar);
            if (VARIANT == V_SMPPI) tma_bulk_g2s(sm.Araw, a.A, bytes, sm.bar);
        }
    } else {
        for (int j = tid; j < TN; j += BD) {
            sm.Uraw[j] = a.U[j];
            if (VARIANT == V_SMPPI) sm.Araw[j] = a.A[j];
        }
    }
    if (VARIANT == V_KMPPI) {
        for (int j = tid; j < R; j += BD) sm.thraw[j] = a.theta[j];
        for (int j = tid; j < T * S; j += BD) sm.Ws[j] = a.W[j];
        if (a.shift)
            for (int j = tid; j < S * S; j += BD) sm.Wsh[j] = a.Wshift[j];
    }
}

// stage_issue of the global-tile kernels: KMPPI's W / Wshift are read in place (gtile_bind), not staged
template <typename real, int VARIANT, int NU>
__device__ void stage_issue_gtile(const KArgs<real>& a, Smem<real>& sm) {
    const int tid = threadIdx.x, BD = blockDim.x;
    const int R = a.R, TN = a.TN;
    if (tid == 0) mbar_init(sm.bar, 1);
    __syncthreads();
    if (a.tma_ok) {
        if (tid == 0) {
            const uint32_t bytes = (uint32_t)align_up(TN * (int)sizeof(real), 16);
            mbar_expect_tx(sm.bar, VARIANT == V_SMPPI ? 2 * bytes : bytes);
            tma_bulk_g2s(sm.Uraw, a.U, bytes, sm.bar);
            if (VARIANT == V_SMPPI) tma_bulk_g2s(sm.Araw, a.A, bytes, sm.bar);
        }
    } else {
        for (int j = tid; j < TN; j += BD) {
            sm.Uraw[j] = a.U[j];
            if (VARIANT == V_SMPPI) sm.Araw[j] = a.A[j];
        }
    }
    if (VARIANT == V_KMPPI)
        for (int j = tid; j < R; j += BD) sm.thraw[j] = a.theta[j];
}

template <typename real, int VARIANT, int NU>
__device__ void stage_finish(const KArgs<real>& a, Smem<real>& sm) {
    typedef Ops<real> O;
    const int tid = threadIdx.x, BD = blockDim.x;
    const int T = a.T, S = a.S, R = a.R, TN = a.TN;
    if (a.tma_ok) mbar_wait(sm.bar, 0);
    __syncthreads();
    for (int j = tid; j < TN; j += BD) {
        const int t = j / NU, n = j - t * NU;
        sm.Us[j] = a.shift ? (t + 1 < T ? sm.Uraw[j + NU] : a.u_init[n]) : sm.Uraw[j];               // mppi.py:237-238
        if (VARIANT == V_SMPPI) sm.As[j] = a.shift ? (t + 1 < T ? sm.Araw[j + NU] : sm.Araw[j]) : sm.Araw[j];  // :492-493
    }
    if (VARIANT == V_KMPPI) {
        for (int j = tid; j < R; j += BD) {
            const int s = j / NU, n = j - s * NU;
            if (a.shift) {                                                                 // mppi.py:619
                real acc = O::mul(sm.Wsh[s * S], sm.thraw[n]);
                for (int q = 1; q < S; ++q) acc = O::add(acc, O::mul(sm.Wsh[s * S + q], sm.thraw[q * NU + n]));
                sm.ths[j] = acc;
            } else {
                sm.ths[j] = sm.thraw[j];
            }
        }
    }
    __syncthreads();
}

template <typename real, int VARIANT, int NU>
__device__ void stage_nominal(const KArgs<real>& a, Smem<real>& sm) {
    stage_issue<real, VARIANT, NU>(a, sm);
    stage_finish<real, VARIANT, NU>(a, sm);
}

// ---- stage A: standard normals into the tile ------------------------------------------------------
// (thread -> sample s = tid % BS, chunk lane g = tid / BS: the tps threads of a sample split its
// Philox chunks)
// the rarely-taken sources of normals, out of line so that they do not sit in the hot path's instruction stream:
// injected z (parity tests), the torch-compatible stream (one Philox call per element), recording of the draws (z_out)
// G: instantiated separately for the global-tile kernels (their tile is in global memory): a shared copy of an out-of-line
// function would lose the shared-memory stores the compiler gives it when every caller passes a shared-memory tile
template <typename real, bool G = false>
__device__ __noinline__ void fill_normals_rare(const KArgs<real>& a, real* rows, int LD, int tile, bool active, unsigned long long kg, int nvalid) {
    const int tid = threadIdx.x, BD = blockDim.x, R = a.R;
    const int BS = BD / a.tps, s_ = tid % BS, g_ = tid / BS;
    if (a.z != nullptr) {
        const size_t base = (size_t)tile * BS * R;
        const int count = nvalid * R;
        for (int e = tid; e < count; e += BD) {
            const int s = e / R, j = e - s * R;
            rows[j * LD + s] = a.z[base + e];
        }
        __syncthreads();
    } else if (a.torch_total > 0 && active) {
        // torch-compatible stream: one Philox call per element (the ATen kernel scatters each call's
        // outputs `total` elements apart), 4x the generator work of the native stream
        constexpr int UN = TorchNormal<real>::UNROLL;
        real* col = rows + s_;
        const unsigned long long off = a.offset_dev != nullptr ? __ldcg(a.offset_dev) : a.offset;
        for (int j = g_; j < R; j += a.tps) {
            const unsigned long long li = kg * (unsigned long long)R + (unsigned long long)j;
            const unsigned long long idx = li % a.torch_total, m = li / a.torch_total;
            col[j * LD] = TorchNormal<real>::one(a.seed, idx, off + m / UN, (int)(m % UN));
        }
    }
}
template <typename real, bool G = false>
__device__ __noinline__ void record_normals(const KArgs<real>& a, const real* rows, int LD, int tile, int nvalid) {
    const int tid = threadIdx.x, BD = blockDim.x, R = a.R, BS = BD / a.tps;
    __syncthreads();
    const size_t base = (size_t)tile * BS * R;
    const int count = nvalid * R;
    for (int e = tid; e < count; e += BD) {
        const int s = e / R, j = e - s * R;
        a.z_out[base + e] = rows[j * LD + s];
    }
    __syncthreads();
}

template <typename real, bool GTILE = false>
__device__ void fill_normals(const KArgs<real>& a, Smem<real>& sm, int tile, bool active, unsigned long long kg, int nvalid) {
    const int tid = threadIdx.x, BD = blockDim.x, R = a.R, LD = sm.LD;
    const int BS = BD / a.tps, s_ = tid % BS, g_ = tid / BS;
    if (a.z != nullptr || a.torch_total > 0) {
        fill_normals_rare<real, GTILE>(a, sm.rows, LD, tile, active, kg, nvalid);
    } else if (active) {
        constexpr int PER = Normals<real>::PER_CALL;
        real* col = sm.rows + s_;
        const unsigned long long off = a.offset_dev != nullptr ? __ldcg(a.offset_dev) : a.offset;
        for (int c = g_; c * PER < R; c += a.tps) {
            real tmp[PER];
            Normals<real>::draw(a.seed, kg, off + (unsigned long long)c, tmp);
#pragma unroll
            for (int q = 0; q < PER; ++q)
                if (c * PER + q < R) col[(c * PER + q) * LD] = tmp[q];
        }
    }
    if (a.z_out != nullptr) record_normals<real, GTILE>(a, sm.rows, LD, tile, nvalid);
}

// value that overrides the sampled action before the clamp: null action (mppi.py:390-392) or a
// SpecificActionSampler row (mppi.py:393-399); returns true if overridden
template <typename real>
__device__ __forceinline__ bool override_value(const KArgs<real>& a, unsigned long long kg, int j, real& p) {
    if (a.null_action && kg == 0ull) { p = (real)0; return true; }
    if (a.override_rows != nullptr) {
        const long long r = (long long)kg - a.override_start;
        if (r >= 0 && r < a.n_override) { p = a.override_rows[(size_t)r * a.TN + j]; return true; }
    }
    return false;
}

// ---- stage B: colour + nominal + clamp, in place in this thread's column --------------------------
// TILE2 (fused / resident kernels): a second tile `rows2` of T*nu rows per sample keeps what the serial rollout thread
// would otherwise recompute per step — SMPPI: the effective noise eps = (v - A)/dt - U (one IEEE division per element,
// needed by the action cost and by the softmin fold); KMPPI: the interpolated, clamped trajectory (interp_column).
template <typename real, int VARIANT, int NU, bool TILE2 = false>
__device__ __forceinline__ void transform_column(const KArgs<real>& a, Smem<real>& sm, unsigned long long kg) {
    typedef Ops<real> O;
    const NoiseModel<real>& nm = a.nm;
    const int LD = sm.LD;
    const int BS = blockDim.x / a.tps, s_ = threadIdx.x % BS, g_ = threadIdx.x / BS;
    real* col = sm.rows + s_;
    if (VARIANT == V_KMPPI) {
        for (int s = g_; s < a.S; s += a.tps) {                                           // mppi.py:660-664
            real zr[NU], e[NU];
#pragma unroll
            for (int n = 0; n < NU; ++n) zr[n] = col[(s * NU + n) * LD];
            colour<real, NU>(nm, zr, e);
#pragma unroll
            for (int n = 0; n < NU; ++n)
                col[(s * NU + n) * LD] = clamp<real>(O::add(sm.ths[s * NU + n], e[n]), nm.u_min[n], nm.u_max[n]);
        }
    } else {
        for (int t = g_; t < a.T; t += a.tps) {
            real zr[NU], e[NU];
#pragma unroll
            for (int n = 0; n < NU; ++n) zr[n] = col[(t * NU + n) * LD];
            colour<real, NU>(nm, zr, e);
#pragma unroll
            for (int n = 0; n < NU; ++n) {
                real p = O::add(sm.Us[t * NU + n], e[n]);                                 // mppi.py:380 / :544
                if (VARIANT == V_SMPPI) {
                    p = O::add(sm.As[t * NU + n], O::mul(p, nm.delta_t));                 // mppi.py:548
                    override_value<real>(a, kg, t * NU + n, p);                           // mppi.py:549
                    p = clamp<real>(p, nm.a_min[n], nm.a_max[n]);                         // mppi.py:550
                    if (TILE2)                                                            // mppi.py:552
                        sm.rows2[(t * NU + n) * LD + s_] = O::sub(O::div(O::sub(p, sm.As[t * NU + n]), nm.delta_t), sm.Us[t * NU + n]);
                } else {
                    override_value<real>(a, kg, t * NU + n, p);                           // mppi.py:381
                    p = clamp<real>(p, nm.u_min[n], nm.u_max[n]);                         // mppi.py:383
                }
                col[(t * NU + n) * LD] = p;
            }
        }
    }
}

// KMPPI, TILE2: interpolate this sample's control points onto the horizon ONCE, with all its tps threads
// (mppi.py:665-668: W @ theta_k, specific actions, clamp), after the barrier that completes the control-point tile
template <typename real, int NU>
__device__ __forceinline__ void interp_column(const KArgs<real>& a, Smem<real>& sm, unsigned long long kg) {
    typedef Ops<real> O;
    const int LD = sm.LD, S = a.S;
    const int BS = blockDim.x / a.tps, s_ = threadIdx.x % BS, g_ = threadIdx.x / BS;
    const real* col = sm.rows + s_;
    for (int t = g_; t < a.T; t += a.tps) {
#pragma unroll
        for (int n = 0; n < NU; ++n) {
            real acc = O::mul(sm.Ws[t * S], col[n * LD]);
            for (int s = 1; s < S; ++s) acc = O::add(acc, O::mul(sm.Ws[t * S + s], col[(s * NU + n) * LD]));
            override_value<real>(a, kg, t * NU + n, acc);
            sm.rows2[(t * NU + n) * LD + s_] = clamp<real>(acc, a.nm.u_min[n], a.nm.u_max[n]);
        }
    }
}

// perturbed action at step t for this thread (KMPPI interpolates the control points: mppi.py:665-668)
template <typename real, int VARIANT, int NU, bool TILE2 = false>
__device__ __forceinline__ void action_at(const KArgs<real>& a, const Smem<real>& sm, unsigned long long kg, int t, real* v) {
    typedef Ops<real> O;
    const int LD = sm.LD;
    const real* col = sm.rows + (threadIdx.x % (blockDim.x / a.tps));
    if (VARIANT == V_KMPPI && TILE2) {
        const real* col2 = sm.rows2 + (threadIdx.x % (blockDim.x / a.tps));
#pragma unroll
        for (int n = 0; n < NU; ++n) v[n] = col2[(t * NU + n) * LD];
    } else if (VARIANT == V_KMPPI) {
        const int S = a.S;
#pragma unroll
        for (int n = 0; n < NU; ++n) {
            real acc = O::mul(sm.Ws[t * S], col[n * LD]);
            for (int s = 1; s < S; ++s) acc = O::add(acc, O::mul(sm.Ws[t * S + s], col[(s * NU + n) * LD]));
            override_value<real>(a, kg, t * NU + n, acc);
            v[n] = clamp<real>(acc, a.nm.u_min[n], a.nm.u_max[n]);
        }
    } else {
#pragma unroll
        for (int n = 0; n < NU; ++n) v[n] = col[(t * NU + n) * LD];
    }
}

// effective noise entering the action cost at step t (mppi.py:385 / :552 / :670)
template <typename real, int VARIANT, int NU, bool TILE2 = false>
__device__ __forceinline__ void noise_at(const KArgs<real>& a, const Smem<real>& sm, int t, const real* v, real* eps) {
    typedef Ops<real> O;
#pragma unroll
    for (int n = 0; n < NU; ++n) {
        if (VARIANT == V_SMPPI && TILE2)
            eps[n] = sm.rows2[(t * NU + n) * sm.LD + (threadIdx.x % (blockDim.x / a.tps))];
        else if (VARIANT == V_SMPPI)
            eps[n] = O::sub(O::div(O::sub(v[n], sm.As[t * NU + n]), a.nm.delta_t), sm.Us[t * NU + n]);
        else
            eps[n] = O::sub(v[n], sm.Us[t * NU + n]);
    }
}

// the weighted quantity for row j given the stored tile value (the thing the softmin averages)
template <typename real, int VARIANT>
__device__ __forceinline__ real eps_of(const NoiseModel<real>& nm, real val, real us, real as_or_ths) {
    typedef Ops<real> O;
    if (VARIANT == V_MPPI) return O::sub(val, us);                                          // mppi.py:385
    if (VARIANT == V_SMPPI) return O::sub(O::div(O::sub(val, as_or_ths), nm.delta_t), us);  // mppi.py:552
    return O::sub(val, as_or_ths);                                                          // mppi.py:664
}

// ---- peer exchange over NVLink mailboxes (LL-style 8-byte records: payload32 | flag32) ----------
// relaxed.sys, not volatile: the words are self-validating, so nothing orders one against another — and ptxas completes
// every volatile access before it issues the next (a thread polling 8 words paid 8 L2 round trips per sweep; the same
// serialisation made a 32-record combine from shared memory cost 1.5 us)
__device__ __forceinline__ void st_peer(unsigned long long* p, unsigned long long v) {
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_poll(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

// value i of the action as flagged 8-byte word(s) in pinned host memory (float: 1 word, double: 2)
template <typename real>
__device__ __forceinline__ void host_store(unsigned long long* box, int i, real v, unsigned long long epoch);
template <>
__device__ __forceinline__ void host_store<float>(unsigned long long* box, int i, float v, unsigned long long epoch) {
    st_peer(box + i, ((epoch & 0xffffffffull) << 32) | (unsigned long long)__float_as_uint(v));
}
template <>
__device__ __forceinline__ void host_store<double>(unsigned long long* box, int i, double v, unsigned long long epoch) {
    const unsigned long long bits = (unsigned long long)__double_as_longlong(v);
    st_peer(box + 2 * i, ((epoch & 0xffffffffull) << 32) | (bits & 0xffffffffull));
    st_peer(box + 2 * i + 1, ((epoch & 0xffffffffull) << 32) | (bits >> 32));
}

// ---- final update from (beta, eta, numerators) with the post-shift nominal in shared memory -----
// ENV (the batched fused kernels, MPPI): a.T is the environment's horizon h_e, and only its first h_e * nu rows take the
// update; the rows past it keep the post-shift nominal, u_init (the fold ran over all R rows, their numerators unused).
template <typename real, int VARIANT, bool ENV = false>
__device__ void finish_update(const KArgs<real>& a, const double* numd, const real* Us, const real* As, real* ths,
                              const real* Ws, int nu) {
    typedef Ops<real> O;
    const int tid = threadIdx.x, BD = blockDim.x;
    const int TN = a.TN, R = a.R;
    const int HN = ENV ? a.T * nu : TN;
    const double eta = numd[1];
    const double inv_eta = 1.0 / eta;
    // nominal_used: U | A | theta slots, as sampled from (post-shift, pre-update)
    for (int j = tid; j < TN; j += BD) {
        a.nominal_used[j] = Us[j];
        if (VARIANT == V_SMPPI) a.nominal_used[TN + j] = As[j];
    }
    if (VARIANT == V_KMPPI)
        for (int j = tid; j < R; j += BD) a.nominal_used[2 * TN + j] = ths[j];
    if (tid == 0) {
        a.stats[0] = numd[0];
        a.stats[1] = eta;
        if (a.offset_dev != nullptr && blockIdx.y == 0) *a.offset_dev += a.offset_inc;   // every sampler of this command is done
    }
    // Host delivery: each action value goes out as self-validating 8-byte words (payload32 | epoch32), so
    // the host sees a value as soon as its own store lands — no system-wide fence, no separate flag.
    unsigned long long* hact = a.host_mailbox;
    if (VARIANT == V_MPPI) {
        for (int j = tid; j < TN; j += BD) {
            const real un = ENV && j >= HN ? Us[j] : O::add(Us[j], (real)(numd[2 + j] * inv_eta));   // mppi.py:270
            a.U[j] = un;
            if (j < a.upc * nu) {                                                          // mppi.py:271-275
                a.action_out[j] = un;
                if (hact != nullptr) host_store<real>(hact, j, un, a.host_epoch);
            }
        }
    } else if (VARIANT == V_SMPPI) {
        for (int j = tid; j < TN; j += BD) {
            const real un = O::add(Us[j], (real)(numd[2 + j] * inv_eta));                // mppi.py:529
            const real an = O::add(As[j], O::mul(un, a.nm.delta_t));                       // mppi.py:531
            a.U[j] = un;
            a.A[j] = an;
            if (j < a.upc * nu) {                                                          // mppi.py:533-537
                a.action_out[j] = an;
                if (hact != nullptr) host_store<real>(hact, j, an, a.host_epoch);
            }
        }
    } else {
        __syncthreads();
        for (int j = tid; j < R; j += BD) {
            const real tn = O::add(ths[j], (real)(numd[2 + j] * inv_eta));              // mppi.py:681
            ths[j] = tn;
            a.theta[j] = tn;
        }
        __syncthreads();
        const int S = a.S;
        for (int j = tid; j < TN; j += BD) {                                               // mppi.py:682  U = W theta
            const int t = j / nu, n = j - t * nu;
            real acc = O::mul(Ws[t * S], ths[n]);
            for (int s = 1; s < S; ++s) acc = O::add(acc, O::mul(Ws[t * S + s], ths[s * nu + n]));
            a.U[j] = acc;
            if (j < a.upc * nu) {
                a.action_out[j] = acc;
                if (hact != nullptr) host_store<real>(hact, j, acc, a.host_epoch);
            }
        }
    }
}

// =================================================================================================
// Warp-fold tail: the softmin reduction of every command kernel (fused_command_kernel, the resident kernel, the
// tensor-core MLP kernels, softmin_update_kernel) without CTA-wide barriers in the fold, a thread-block-cluster stage
// through distributed shared memory, and a finisher that works on a handful of records.
//
//   per tile   each ROLLOUT WARP folds its 32 samples into its own running record (beta_w, eta_w, V_w[R]) — shuffles
//              only, fp64 accumulation, record in shared memory (warp-private: no barrier)
//   per CTA    the warp records go to the cluster LEADER's shared memory (st.shared::cluster), one cluster barrier
//   leader     combines cluster_size x warps records into ONE cluster record and publishes it: to the L2 workspace
//              (ticket among the leaders — 16 atomics instead of 128 at BASELINE config 2), or, on a sharded controller
//              in direct mode, straight into every peer GPU's mailbox over NVLink
//   finisher   (last leader) combines the n_clusters (x world) records and writes the update
// Every combination is in fixed record order and fp64, so the result does not depend on scheduling and is bit-identical
// on all ranks of a sharded controller.   Reference lines: mppi.py:254-259, 268-270 (and the SMPPI / KMPPI forms).
// =================================================================================================
__device__ __forceinline__ uint32_t cluster_nctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ uint32_t mapa_shared(uint32_t addr, uint32_t cta_rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(cta_rank));
    return r;
}
__device__ __forceinline__ void st_dsmem_f64(uint32_t addr, double v) {
    asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(addr), "d"(v) : "memory");
}
__device__ __forceinline__ void cluster_arrive_relaxed() { asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_arrive_release() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait_acquire() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }

#define MPPI_XCHG_PARITY_WORDS 65536       // 8-byte words per epoch parity of a peer mailbox (mppi_xchg_bytes = 2 x this x 8)

// doubles of the finisher's staging area: every record it polls (LL mode: xw x npub cluster records; sharded rank-record
// mode: one per rank); a single GPU in ticket mode stages nothing
__host__ __device__ inline int fused_xstage_doubles(bool sharded, int world, int npub, int R) {
    const int xw = sharded ? world : 1;
    return (npub > 1 || sharded) ? xw * npub * (R + 2) : 0;
}

// the `nb` argument of make_layout for the warp-fold tail: the records combine_records reads from the L2 workspace
// (ticket mode: the grid's NC cluster records), 1 when they arrive as flagged words (LL mode) or there is one cluster
__host__ __device__ inline int fused_layout_nb(int NC, int npub) { return (NC > 1 && npub != NC) ? NC : 1; }

// this CTA's running warp records: (beta = +inf, eta = 0, V = 0); call before the first barrier of the kernel
template <typename real>
__device__ __forceinline__ void warp_records_init(const KArgs<real>& a, Smem<real>& sm) {
    const int RW = a.R + 2, n = (blockDim.x / a.tps >> 5) * RW;
    for (int i = threadIdx.x; i < n; i += blockDim.x) sm.wrec[i] = (i % RW == 0) ? (double)INFINITY : 0.0;
}

// ---- per tile: fold this warp's 32 samples into its running record (rollout warps only; warp-synchronous) ----------
// The tile forms: `rows` holds what transform_column left there (v, or KMPPI's control points), and SMPPI's effective
// noise is read from `rows2` (TILE2) or derived from `rows` with eps_of (kernels without the second tile); EPS_DIRECT:
// `rows` holds the effective noise itself (softmin_update_kernel, every variant).
template <typename real, int VARIANT, bool TILE2 = true, bool EPS_DIRECT = false>
__device__ __forceinline__ void warp_fold(const KArgs<real>& a, Smem<real>& sm, real c_tot, bool active, int nvalid) {
    typedef Ops<real> O;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int R = a.R, LD = sm.LD, i0 = w * 32;
    double* rec = sm.wrec + (size_t)w * (R + 2);
    const real nfl = a.nm.neg_inv_lambda;
    // the 32 columns this warp reads below were written by its own lanes (one sample per thread: no CTA barrier in
    // between) — order them
    __syncwarp();
    const real cmin = warp_min<real>(active ? c_tot : O::inf());
    const real beta_run = (real)rec[0];                 // a value of type `real`, kept in a double slot
    const real beta_new = cmin < beta_run ? cmin : beta_run;
    if (beta_new == O::inf()) return;                   // warp-uniform: no sample of this warp has a cost yet
    const real wgt = active ? O::exp_(nfl * (c_tot - beta_new)) : (real)0;                       // mppi.py:12-13, 256
    const double resc = (beta_run == O::inf()) ? 0.0 : (double)O::exp_(nfl * (beta_run - beta_new));
    const double eta_tile = (double)warp_sum<real>(wgt);
    const int nv = min(32, nvalid - i0);
    for (int jb = 0; jb < R; jb += 32) {
        const int j = jb + lane;
        const bool jv = j < R;
        const int jc = jv ? j : 0;
        constexpr bool eps_in_tile = EPS_DIRECT || (VARIANT == V_SMPPI && TILE2);
        const real us = (eps_in_tile || VARIANT == V_KMPPI) ? (real)0 : sm.Us[jc];
        const real a2 = eps_in_tile ? (real)0 : VARIANT == V_SMPPI ? sm.As[jc] : (VARIANT == V_KMPPI ? sm.ths[jc] : (real)0);
        // SMPPI with TILE2: the tile of effective noise (rows2, written once by transform_column) — no division here
        const real* row = (VARIANT == V_SMPPI && TILE2 && !EPS_DIRECT ? sm.rows2 : sm.rows) + (size_t)jc * LD + i0;
        // the 32 products of a warp are added in the controller's precision (as the reference's einsum does, in its own
        // order); everything ACROSS warps, CTAs and GPUs is fp64 (measured: an fp64 inner sum costs the large-K
        // geometry, where every warp folds, 5 us per command through F2F.F64 / DADD issue)
        // The trip count is the constant 32, in batches of FB: each batch's shuffles and tile loads are issued together,
        // ahead of its FFMAs, so only the chain on `acc` is serial (with a run-time count every iteration waited on its
        // own shuffle and load).  Columns i >= nv (a partial last warp) are read — they lie inside the tile — but never
        // added: their shared memory is stale, and 0 * NaN is not 0.  FB keeps a batch's values in 16 registers, and the
        // batch loop stays rolled: fully unrolled, ptxas held every batch at once and spilled under the 64-register cap of
        // the two-CTA-per-SM kernels (and in the global-tile softmin kernel).
        constexpr int FB = sizeof(real) == 8 ? 4 : 8;
        real acc = (real)0;
#pragma unroll 1
        for (int ib = 0; ib < 32; ib += FB) {
            real wv[FB], ev[FB];
#pragma unroll
            for (int u = 0; u < FB; ++u) {
                wv[u] = __shfl_sync(0xffffffffu, wgt, ib + u);
                ev[u] = row[ib + u];
            }
#pragma unroll
            for (int u = 0; u < FB; ++u) {
                const real e = eps_in_tile ? ev[u] : eps_of<real, VARIANT>(a.nm, ev[u], us, a2);
                if (ib + u < nv) acc += wv[u] * e;                                              // mppi.py:268
            }
        }
        if (jv) rec[2 + j] = rec[2 + j] * resc + (double)acc;
    }
    __syncwarp();                    // every lane has read the running record
    if (lane == 0) {
        rec[0] = (double)beta_new;
        rec[1] = rec[1] * resc + eta_tile;
    }
    __syncwarp();
}

// ---- fixed-order fp64 combination of records (beta_q, eta_q, V_q[R]) -----------------------------------------------
//   beta = min beta_q ; s_q = exp(nfl (beta_q - beta)) ; eta = sum s_q eta_q ; V[j] = sum s_q V_q[j]   -> numd[0 .. R+2)
// CTA-wide (every thread calls it; three barriers).  Record q is recs[q * (R+2) ..] in shared or global memory (generic
// pointer, volatile loads: L2 for global).  Threads are (group g = tid / 64, column jl = tid % 64): group g adds the
// records q = g, g + nG, ... for its columns (column 0 = eta, column 1 + j = V[j]) into part2[g][..], the groups are added
// in order — the result does not depend on timing.  Deliberately SMALL and out of line (one copy for every call site):
// the tail runs once per command on a cold instruction cache, where instruction count, not arithmetic, sets its time
// (ncu: `no_instruction` is the third-largest stall of the kernel).
template <typename real>
__device__ __forceinline__ void combine_records_body(const double* recs, int nrec, int R, double nfl, double* part2, double* sq,
                                                     double* numd) {
    typedef Ops<real> O;
    const int RW = R + 2, C = R + 1;                      // columns: eta, V[0..R)
    const int tid = threadIdx.x, BD = blockDim.x, nG = BD >> 6, g = tid >> 6, jl = tid & 63, nw = BD >> 5;
    // beta: ONE load per thread (record tid; more only for grids above blockDim records), warp minima through sq[]
    const double b_mine = tid < nrec ? recs[(size_t)tid * RW] : (double)INFINITY;
    double b = b_mine;
    for (int q = tid + BD; q < nrec; q += BD) b = fmin(b, recs[(size_t)q * RW]);
    b = warp_min<double>(b);
    if ((tid & 31) == 0) part2[tid >> 5] = b;
    __syncthreads();
    double beta = part2[0];
    for (int w = 1; w < nw; ++w) beta = fmin(beta, part2[w]);
    // the rescale factors in the controller's precision (exact for equal betas; beta_q - beta is exact in fp64)
    if (tid < nrec) sq[tid] = (double)O::exp_((real)(nfl * (b_mine - beta)));
    for (int q = tid + BD; q < nrec; q += BD) sq[q] = (double)O::exp_((real)(nfl * (recs[(size_t)q * RW] - beta)));
    __syncthreads();
    if (tid == 0) numd[0] = beta;
    // the loads of a batch are issued together, THEN used: written as `acc += sq[q] * recs[..]` in one loop, ptxas keeps
    // every volatile load next to its DFMA and a thread waits one L2 round trip per record (K = 131072: 293 records in
    // the L2 workspace, 42 per thread — 9 us; batched: 6 round trips)
    constexpr int UB = 8;
    for (int j = jl; j < C; j += 64) {
        double acc = 0.0;
        const double* col = recs + 1 + j;
        for (int q0 = g; q0 < nrec; q0 += nG * UB) {
            double v[UB];
#pragma unroll
            for (int u = 0; u < UB; ++u) {
                const int q = q0 + u * nG;
                v[u] = q < nrec ? col[(unsigned)(q * RW)] : 0.0;
            }
#pragma unroll
            for (int u = 0; u < UB; ++u) {
                const int q = q0 + u * nG;
                if (q < nrec) acc += sq[q] * v[u];
            }
        }
        part2[g * C + j] = acc;
    }
    __syncthreads();
    for (int j = tid; j < C; j += BD) {
        double t = part2[j];
        for (int w = 1; w < nG; ++w) t += part2[(size_t)w * C + j];
        numd[1 + j] = t;
    }
    __syncthreads();
}
template <typename real>
__device__ __noinline__ void combine_records(const double* recs, int nrec, int R, double nfl, double* part2, double* sq,
                                             double* numd) {
    combine_records_body<real>(recs, nrec, R, nfl, part2, sq, numd);
}

// ---- the same combination for records in the L2 workspace (ticket mode: grids of hundreds of CTAs) ---------------------
// ld.global.cg loads (L2; no SM of this launch has the lines in L1), UB of them in flight per thread before the first is
// used.  The volatile form above leaves one L2 round trip per record on the critical path — at K = 131072 (293 records,
// 42 per thread) that was 9 us of a 47 us command.
template <typename real>
__device__ __noinline__ void combine_global(const double* recs, int nrec, int R, double nfl, double* part2, double* sq, double* numd) {
    typedef Ops<real> O;
    const int RW = R + 2, C = R + 1;
    const int tid = threadIdx.x, BD = blockDim.x, nG = BD >> 6, g = tid >> 6, jl = tid & 63, nw = BD >> 5;
    double b = (double)INFINITY;
    for (int q = tid; q < nrec; q += BD) b = fmin(b, __ldcg(recs + (size_t)q * RW));
    b = warp_min<double>(b);
    if ((tid & 31) == 0) part2[tid >> 5] = b;
    __syncthreads();
    double beta = part2[0];
    for (int w = 1; w < nw; ++w) beta = fmin(beta, part2[w]);
    for (int q = tid; q < nrec; q += BD) {
        const double bq = __ldcg(recs + (size_t)q * RW);
        sq[q] = bq == (double)INFINITY ? 0.0 : (double)O::exp_((real)(nfl * (bq - beta)));
    }
    __syncthreads();
    if (tid == 0) numd[0] = beta;
    constexpr int UB = 8;
    for (int j = jl; j < C; j += 64) {
        double acc = 0.0;
        const double* col = recs + 1 + j;
        for (int q0 = g; q0 < nrec; q0 += nG * UB) {
            double v[UB];
#pragma unroll
            for (int u = 0; u < UB; ++u) {
                const int q = q0 + u * nG;
                v[u] = q < nrec ? __ldcg(col + (size_t)q * RW) : 0.0;
            }
#pragma unroll
            for (int u = 0; u < UB; ++u) {
                const int q = q0 + u * nG;
                if (q < nrec) acc += sq[q] * v[u];
            }
        }
        part2[g * C + j] = acc;
    }
    __syncthreads();
    for (int j = tid; j < C; j += BD) {
        double t = part2[j];
        for (int w = 1; w < nG; ++w) t += part2[w * C + j];
        numd[1 + j] = t;
    }
    __syncthreads();
}

// ---- the same combination for at most 64 records, with one CTA barrier ------------------------------------------------
// Column j's sum runs as two chains, acc0 over the even records and acc1 over the odd ones, each in ascending order, added
// at the end as acc0 + acc1.  The chains are independent, so they run on different warps: work item u = (column block
// u >> 1, chain u & 1) belongs to warp u mod W, W = min(warps, 2 x column blocks): two warps at C <= 32.  The W warps
// compute beta each, and the rescale factors once (warps 0 and 1: records lane and 32 + lane) into sq[]; a named barrier
// among them publishes the factors, and a second one hands the odd chains' sums (in part[]) to the warps that add them to
// the even chains' sums, which already sit in numd.  A chain issues the loads of UB records and factors together, then
// their UB DFMAs: only the chain itself is serial.  The other warps of the CTA go straight to the one CTA barrier at the
// end.  This is the form the tail uses at every size that matters for latency: 16 warp records per cluster and 32 cluster
// records per GPU at BASELINE config 2 — the barrier-and-scratch form above cost 2.3 + 2.9 us there (every warp of the
// CTA walks its ~600 instructions, contending with the co-resident CTA at large K), this one a fraction.
// sq holds nrec doubles and part C (the callers pass the layout's sqd and part2).
// Named barrier 1 is reserved for the combining warps of combine_narrow_body (barrier 0 is __syncthreads); a kernel that
// runs this tail must not use id 1 for anything else.
#define MPPI_TAIL_NAMED_BARRIER 1
__device__ __forceinline__ void combine_narrow_bar(int nthreads) {
    asm volatile("barrier.sync.aligned %0, %1;" ::"n"(MPPI_TAIL_NAMED_BARRIER), "r"(nthreads) : "memory");
}
template <typename real>
__device__ __forceinline__ void combine_narrow_body(const double* recs, int nrec, int R, double nfl, double* sq, double* part,
                                                    double* numd) {
    typedef Ops<real> O;
    const int RW = R + 2, C = R + 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    // W >= 2 because every plan has at least two warps per CTA (plan_geometry: BS * tps >= 64): warps 0 and 1 write the
    // factors of records 0..31 and 32..63, and part (the layout's part2, nw * R doubles) holds C = R + 1 doubles
    const int W = min(nw, 2 * ((C + 31) >> 5));
    if (warp < W) {
        const double b0 = lane < nrec ? recs[lane * RW] : (double)INFINITY;
        const double b1 = lane + 32 < nrec ? recs[(lane + 32) * RW] : (double)INFINITY;
        const double beta = warp_min<double>(fmin(b0, b1));
        // in the controller's precision (exact for equal betas; beta_q - beta is exact in fp64); an empty record weighs 0
        if (warp < 2 && warp * 32 + lane < nrec) {
            const double bq = warp == 0 ? b0 : b1;
            sq[warp * 32 + lane] = bq == (double)INFINITY ? 0.0 : (double)O::exp_((real)(nfl * (bq - beta)));
        }
        combine_narrow_bar(W * 32);
        constexpr int UB = 8;
        for (int u = warp; u < 2 * ((C + 31) >> 5); u += W) {
            const int h = u & 1, j = (u >> 1) * 32 + lane;
            const double* col = recs + 1 + (j < C ? j : 0);
            double acc = 0.0;
            for (int q0 = h; q0 < nrec; q0 += 2 * UB) {
                double v[UB], s[UB];
#pragma unroll
                for (int k = 0; k < UB; ++k) {
                    const int q = q0 + 2 * k;
                    v[k] = q < nrec ? col[q * RW] : 0.0;
                    s[k] = q < nrec ? sq[q] : 0.0;
                }
#pragma unroll
                for (int k = 0; k < UB; ++k)
                    if (q0 + 2 * k < nrec) acc += s[k] * v[k];
            }
            if (j < C) (h ? part[j] : numd[1 + j]) = acc;
        }
        combine_narrow_bar(W * 32);
        for (int j = warp * 32 + lane; j < C; j += W * 32) numd[1 + j] = numd[1 + j] + part[j];
        if (threadIdx.x == 0) numd[0] = beta;
    }
    __syncthreads();
}
template <typename real>
__device__ __noinline__ void combine_narrow(const double* recs, int nrec, int R, double nfl, double* sq, double* part, double* numd) {
    combine_narrow_body<real>(recs, nrec, R, nfl, sq, part, numd);
}
#define MPPI_COMBINE_NARROW_MAX 64

// INLINE: the combination's code in the caller's instruction stream (the single-GPU LL tail, see warp_tail), else one
// out-of-line copy per form that every call site of the kernel shares
template <typename real, bool INLINE = false>
__device__ __forceinline__ void combine(Smem<real>& sm, const double* recs, int nrec, int R, double nfl) {
    if (INLINE) {
        if (nrec <= MPPI_COMBINE_NARROW_MAX) combine_narrow_body<real>(recs, nrec, R, nfl, sm.sqd, sm.part2, sm.numd);
        else combine_records_body<real>(recs, nrec, R, nfl, sm.part2, sm.sqd, sm.numd);
    } else {
        if (nrec <= MPPI_COMBINE_NARROW_MAX) combine_narrow<real>(recs, nrec, R, nfl, sm.sqd, sm.part2, sm.numd);
        else combine_records<real>(recs, nrec, R, nfl, sm.part2, sm.sqd, sm.numd);
    }
}

// ---- record mailboxes: records of (R+2) doubles as LL words (payload32 | flag32), record r at word r * 2 (R+2) ------
// a.peers[g], g < xw, are the mailboxes the record goes to: every rank's (sharded controller, over NVLink) or just this
// GPU's own (single GPU: a region of the workspace) — self-validating words need no fence and no ticket, the finisher
// sees a record one store-to-poll latency after it was written.
static __device__ __forceinline__ void xchg_publish_body(unsigned long long* const* peers, int xw, unsigned long long epoch,
                                                         unsigned int parity_words, int rec_index, int R, const double* src) {
    const int nwords = 2 * (R + 2);
    const uint32_t flag = (uint32_t)(epoch & 0x7fffffffull) | 0x80000000u;
    const size_t off = (size_t)(epoch & 1ull) * parity_words + (size_t)rec_index * nwords;
    for (int i = threadIdx.x; i < nwords; i += blockDim.x) {
        const unsigned long long bits = (unsigned long long)__double_as_longlong(src[i >> 1]);
        const uint32_t half = (i & 1) ? (uint32_t)(bits >> 32) : (uint32_t)bits;
        const unsigned long long word = ((unsigned long long)flag << 32) | half;
        for (int g = 0; g < xw; ++g) st_peer(peers[g] + off + i, word);
    }
    // (measured and rejected: a system-scope fence after the remote stores, meant to push the posted NVLink writes out
    // sooner, costs 4.5 us per command at two GPUs — 24.2 against 19.7 us back to back)
}
static __device__ __noinline__ void xchg_publish_words(unsigned long long* const* peers, int xw, unsigned long long epoch, unsigned int parity_words,
                                                int rec_index, int R, const double* src) {
    xchg_publish_body(peers, xw, epoch, parity_words, rec_index, R, src);
}
template <typename real, bool INLINE = false>
__device__ __forceinline__ void xchg_publish(const KArgs<real>& a, int xw, int rec_index, const double* src) {
    if (INLINE) xchg_publish_body(a.peers, xw, a.epoch, a.xchg_parity_words, rec_index, a.R, src);
    else xchg_publish_words(a.peers, xw, a.epoch, a.xchg_parity_words, rec_index, a.R, src);
}
// all threads of the CTA; nrec records from this rank's own mailbox into sm.xstage (doubles), PB polls in flight per
// thread.  Returns 0, or 1 on timeout.
static __device__ __forceinline__ int xchg_collect_body(const unsigned long long* mine, unsigned long long epoch,
                                                        unsigned long long timeout_ns, int nwords, uint32_t* dst) {
    constexpr int PB = 8;
    const int BD = blockDim.x;
    const uint32_t flag = (uint32_t)(epoch & 0x7fffffffull) | 0x80000000u;
    __shared__ int s_timeout;
    if (threadIdx.x == 0) s_timeout = 0;
    __syncthreads();
    unsigned long long t0 = 0;
    for (int base = threadIdx.x; base < nwords; base += BD * PB) {
        unsigned int pending = 0;
#pragma unroll
        for (int u = 0; u < PB; ++u)
            if (base + u * BD < nwords) pending |= 1u << u;
        unsigned int spins = 0;
        while (pending) {
            unsigned long long w[PB];
#pragma unroll
            for (int u = 0; u < PB; ++u)
                if (pending & (1u << u)) w[u] = ld_poll(mine + base + u * BD);
#pragma unroll
            for (int u = 0; u < PB; ++u)
                if ((pending & (1u << u)) && (uint32_t)(w[u] >> 32) == flag) {
                    dst[base + u * BD] = (uint32_t)w[u];
                    pending &= ~(1u << u);
                }
            if (pending && (++spins & 255u) == 0) {
                unsigned long long now;
                asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
                if (t0 == 0) t0 = now;
                if (now - t0 > timeout_ns || s_timeout) {
                    s_timeout = 1;
                    break;
                }
            }
        }
    }
    __syncthreads();
    return s_timeout;
}
static __device__ __noinline__ int xchg_collect_words(const unsigned long long* mine, unsigned long long epoch, unsigned long long timeout_ns,
                                               int nwords, uint32_t* dst) {
    return xchg_collect_body(mine, epoch, timeout_ns, nwords, dst);
}
template <typename real, bool INLINE = false>
__device__ __forceinline__ int xchg_collect(const KArgs<real>& a, Smem<real>& sm, int own, int nrec) {
    const unsigned long long* mine = a.peers[own] + (size_t)(a.epoch & 1ull) * a.xchg_parity_words;
    uint32_t* dst = reinterpret_cast<uint32_t*>(sm.xstage);
    if (INLINE) return xchg_collect_body(mine, a.epoch, a.xchg_timeout_ns, nrec * 2 * (a.R + 2), dst);
    return xchg_collect_words(mine, a.epoch, a.xchg_timeout_ns, nrec * 2 * (a.R + 2), dst);
}

// a peer never delivered: report it (device stats, pinned host word) and return a DEFINED action — the nominal the
// command sampled around, not updated.  This rank's U then lags its peers by one update: the host raises on the next
// command (mppi.py reads the status word), it does not continue silently.
template <typename real, int VARIANT>
__device__ void xchg_timed_out(const KArgs<real>& a, Smem<real>& sm, int nu) {
    const real* nom = VARIANT == V_SMPPI ? sm.As : sm.Us;
    for (int j = threadIdx.x; j < a.upc * nu; j += blockDim.x) {
        a.action_out[j] = nom[j];
        if (a.host_mailbox != nullptr) host_store<real>(a.host_mailbox, j, nom[j], a.host_epoch);
    }
    if (threadIdx.x == 0) {
        a.stats[3] = -6.0;     // MPPI_ERR_TIMEOUT
        if (a.xchg_status_host != nullptr) {
            *reinterpret_cast<volatile long long*>(a.xchg_status_host) = -6;
            __threadfence_system();
        }
        *a.ticket = 0u;
    }
}
template <typename real, int VARIANT>
__device__ __noinline__ void xchg_timed_out_rare(const KArgs<real>& a, Smem<real>& sm, int nu) {
    xchg_timed_out<real, VARIANT>(a, sm, nu);
}

// ---- the tail: returns true in the CTA that finished the command --------------------------------------------------
// PERSISTENT (resident kernel): the grid outlives the command, so the non-leader CTAs of a cluster complete the barrier
// phase (arrive + wait) instead of exiting after their arrive.
// LL1: the launch is known to be single-GPU LL mode (NC > 1 clusters, every cluster record published to this GPU's own
// mailbox; fused_command_kernel_ll).  Then the tail is one path — cluster stage, combine, publish, collect, combine,
// finish_update — and its combines, publish and collect are inlined into it: the finisher runs on a cold instruction
// cache (the L2 flushed between commands), where every jump into out-of-line code that no SM has fetched yet waits on
// memory while the rest of the GPU idles.  Only the timeout report stays out of line.
// ENV: the batched fused kernels (finish_update<..., ENV>).
template <typename real, int VARIANT, int NU, bool PERSISTENT = false, bool LL1 = false, bool ENV = false>
__device__ bool warp_tail(const KArgs<real>& a, Smem<real>& sm) {
    const int tid = threadIdx.x, BD = blockDim.x, lane = tid & 31, warp = tid >> 5;
    const int R = a.R, RW = R + 2;
    const int nrw = (BD / a.tps) >> 5;                       // rollout warps = records per CTA
    const int cs = (int)cluster_nctarank();                  // cluster dims are (cs, 1, 1)
    const int cr = blockIdx.x % cs, cid = blockIdx.x / cs, NC = gridDim.x / cs;
    const double nfl = (double)a.nm.neg_inv_lambda;
    const bool sharded = !LL1 && a.world > 1 && !a.export_partial;
    const int xw = sharded ? a.world : 1;                    // ranks whose records the finisher combines
    const int xr = sharded ? a.rank : 0;                     // this rank's slot among them
    // LL mode: the cluster records go out as flagged words (to this GPU's mailbox, and every peer's on a sharded
    // controller); the leader of cluster 0 polls for all xw x NC of them — no fence, no ticket.  Otherwise (grids whose
    // records do not fit the finisher's staging area): records to the L2 workspace, ticket among the leaders.
    const bool ll = LL1 || (NC > 1 && a.xchg_npub == NC);
    __shared__ int s_is_last;

    // (1) warp records -> the cluster leader's shared memory
    if (cs > 1) {
        if (!PERSISTENT) cluster_wait_acquire();             // phase 0 (arrived at kernel entry): every CTA of the cluster runs
        if (cr != 0 && warp < nrw) {
            const uint32_t dst = mapa_shared(smem_u32(sm.wrec), 0) + (uint32_t)(((cr * nrw + warp) * RW) * 8);
            const double* rec = sm.wrec + (size_t)warp * RW;
            for (int i = lane; i < RW; i += 32) st_dsmem_f64(dst + i * 8, rec[i]);
        }
        cluster_arrive_release();
        if (cr != 0) {
            if (PERSISTENT) cluster_wait_acquire();
            return false;
        }
        cluster_wait_acquire();
    } else {
        __syncthreads();
    }
    stamp(a.dbg, 6);

    // (2) leader: cs x nrw warp records -> one cluster record in sm.numd
    {
        combine<real, LL1>(sm, sm.wrec, cs * nrw, R, nfl);
    }
    stamp(a.dbg, 9);
    // (3) publish the cluster record
    if (ll) {
        xchg_publish<real, LL1>(a, xw, xr * NC + cid, sm.numd);
        if (cid != 0) return false;                          // the leader of cluster 0 finishes the command
    } else if (NC > 1) {
        for (int i = tid; i < RW; i += BD) a.crec[(size_t)cid * RW + i] = sm.numd[i];
        __syncthreads();        // every thread's stores precede thread 0's release (one MEMBAR per leader)
        if (tid == 0) {
            unsigned int t;
            asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], %2;" : "=r"(t) : "l"(a.ticket), "r"(1u) : "memory");
            s_is_last = (t == (unsigned int)NC - 1);
        }
        __syncthreads();
        if (!s_is_last) return false;
        if (tid == 0) *a.ticket = 0u;   // self-reset: the next launch needs no memset
    }
    stamp(a.dbg, 8);

    // (4) finisher: all records -> (beta, eta, numerators) in sm.numd
    if (ll) {
        if (xchg_collect<real, LL1>(a, sm, xr, xw * NC)) {
            if (LL1) xchg_timed_out_rare<real, VARIANT>(a, sm, NU);
            else xchg_timed_out<real, VARIANT>(a, sm, NU);
            return true;
        }
        stamp(a.dbg, 12);
        combine<real, LL1>(sm, sm.xstage, xw * NC, R, nfl);
    } else if (NC > 1) {
        combine_global<real>(a.crec, NC, R, nfl, sm.part2, sm.sqd, sm.numd);
    }
    stamp(a.dbg, 10);
    if (!LL1 && a.export_partial) {   // library-collective route: caller all-gathers, mppi_apply_partials finishes
        const int TN = a.TN;
        for (int j = tid; j < RW; j += BD) a.partial_out[j] = sm.numd[j];
        for (int j = tid; j < TN; j += BD) {
            a.nominal_used[j] = sm.Us[j];
            if (VARIANT == V_SMPPI) a.nominal_used[TN + j] = sm.As[j];
        }
        if (VARIANT == V_KMPPI)
            for (int j = tid; j < R; j += BD) a.nominal_used[2 * TN + j] = sm.ths[j];
        if (tid == 0) {
            a.stats[0] = sm.numd[0];
            a.stats[1] = sm.numd[1];
            a.stats[3] = 0.0;
        }
        return true;
    }
    if (sharded && !ll) {
        // rank-record mode: this rank's combined record is its one published record
        xchg_publish<real>(a, xw, xr, sm.numd);
        if (xchg_collect<real>(a, sm, xr, xw)) {
            xchg_timed_out<real, VARIANT>(a, sm, NU);
            return true;
        }
        combine<real>(sm, sm.xstage, xw, R, nfl);
    }
    stamp(a.dbg, 11);
    finish_update<real, VARIANT, ENV>(a, sm.numd, sm.Us, sm.As, sm.ths, sm.Ws, NU);
    if (tid == 0) a.stats[3] = 0.0;
    return true;
}

// ---- per-environment view of the kernel arguments (batched launches) -------------------------------
// The argument block lives in constant (parameter) space; a batched CTA needs its environment's
// pointers, so it builds an adjusted copy in shared memory once and every stage reads that copy.
// ENV (the batched fused kernels): the environment's own noise model replaces `nm` where env_nm is set, and its own
// horizon h_e replaces `T` where env_horizon is set.  Only `T` changes: TN, R and every stride and layout derived from them
// stay the plan's, so the environment's rows are the first h_e * nu of the plan's.
template <typename real, int NXv, int NUv, bool ENV = false>
__device__ void make_env_args(const KArgs<real>& in, KArgs<real>* out) {
    const int tid = threadIdx.x, BD = blockDim.x;
    const uint32_t* src = reinterpret_cast<const uint32_t*>(&in);
    uint32_t* dst = reinterpret_cast<uint32_t*>(out);
    for (int i = tid; i < (int)(sizeof(KArgs<real>) / 4); i += BD) dst[i] = src[i];
    __syncthreads();
    if (ENV && in.env_nm != nullptr) {
        static_assert(sizeof(NoiseModel<real>) % 4 == 0, "word copy of the noise model");
        const uint32_t* nsrc = reinterpret_cast<const uint32_t*>(in.env_nm + blockIdx.y);
        uint32_t* ndst = reinterpret_cast<uint32_t*>(&out->nm);
        for (int i = tid; i < (int)(sizeof(NoiseModel<real>) / 4); i += BD) ndst[i] = nsrc[i];
    }
    if (tid == 0) {
        const long long e = blockIdx.y;
        const long long K = in.K, TN = in.TN, R = in.R;
        out->U = in.U + e * in.env_u_stride;
        if (in.cost_total) out->cost_total = in.cost_total + e * K;
        if (in.action_out) out->action_out = in.action_out + e * in.upc * NUv;
        if (in.nominal_used) out->nominal_used = in.nominal_used + e * (3 * TN + 4);
        if (in.stats) out->stats = in.stats + e * 4;
        if (in.state_dev) out->state_dev = in.state_dev + e * NXv;
        if (in.ticket) {
            const long long off = e * in.env_ws_stride;
            out->ticket = reinterpret_cast<unsigned int*>(reinterpret_cast<unsigned char*>(in.ticket) + off);
            out->crec = reinterpret_cast<double*>(reinterpret_cast<unsigned char*>(in.crec) + off);
            if (in.world == 1 || in.export_partial)      // this GPU's own record mailbox lives in the environment's workspace
                out->peers[0] = reinterpret_cast<unsigned long long*>(reinterpret_cast<unsigned char*>(in.peers[0]) + off);
        }
        if (ENV) {
            if (in.env_horizon != nullptr) out->T = in.env_horizon[e];
        } else if (in.out_pa) {
            out->out_pa = in.out_pa + e * K * TN;
        }
        if (in.out_noise) out->out_noise = in.out_noise + e * K * TN;
        if (in.out_cost_init) out->out_cost_init = in.out_cost_init + e * K;
        if (in.in_cost) out->in_cost = in.in_cost + e * K;
        if (in.in_eps) out->in_eps = in.in_eps + e * K * R;
    }
    __syncthreads();
}

// ---- Rollouts.  A model with a fast range (FastRange, mppi_math.cuh) checks in_fast_range on x_0; when it holds, the
// sample's rollout runs on the model's fast step and cost, inlined; when it does not (a start far out, or a non-finite
// one), on the exact forms, out of line.  Every other model runs the exact forms inline.

// the rollout thread's state at t = 0 (mppi.py:303-305): the controller's state, or the sample's own (state_per_sample)
template <typename real, int NX>
__device__ __forceinline__ void initial_state(const KArgs<real>& a, int k, real* x) {
    if (a.state_dev != nullptr) {
        const real* sp = a.state_dev + (a.state_per_sample ? (size_t)k * NX : 0);
#pragma unroll
        for (int i = 0; i < NX; ++i) x[i] = sp[i];
    } else {
#pragma unroll
        for (int i = 0; i < NX; ++i) x[i] = a.x0[i];
    }
}

// what a sample's rollout loop carries from step to step besides its actions: the state, the running-cost sum (single
// loop only), the action cost and the SMPPI smoothness cost
template <typename real, int NX> struct RolloutCarry {
    real x[NX];
    real roll, pert, smooth;
};

// step t's action cost (mppi.py:409, 415) added to pert and, for SMPPI, the step's smoothness (mppi.py:559-562) added to
// smooth; vprev carries the previous perturbed action from step to step (zeros before t = 0)
template <typename real, int VARIANT, int NU>
__device__ __forceinline__ void action_terms(const NoiseModel<real>& nm, const real* us, int t, const real* v, const real* eps,
                                             real& pert, real& smooth, real* vprev) {
    typedef Ops<real> O;
    pert = O::add(pert, action_cost_term<real, NU>(nm, eps, us));
    if (VARIANT == V_SMPPI) {
        if (t > 0) {
#pragma unroll
            for (int n = 0; n < NU; ++n) {
                const real d = O::mul(nm.u_scale, O::sub(v[n], vprev[n]));    // mppi.py:559
                smooth = O::add(smooth, O::mul(d, d));
            }
        }
#pragma unroll
        for (int n = 0; n < NU; ++n) vprev[n] = v[n];
    }
}

// the sample's total cost from its rollout cost, action cost and SMPPI smoothness, stored to cost_total[k]
template <typename real, int VARIANT>
__device__ __forceinline__ real sample_total(const KArgs<real>& a, int k, real roll, real pert, real smooth) {
    typedef Ops<real> O;
    real c_tot = O::add(roll, pert);                                                  // mppi.py:416
    if (VARIANT == V_SMPPI) c_tot = O::add(c_tot, O::mul(smooth, a.nm.w_smooth));    // mppi.py:562,569
    a.cost_total[k] = c_tot;
    return c_tot;
}

// the recurrence of the split-cost rollout on the sample's rollout thread: every x_t to the sample's column of xs, the
// action cost (and SMPPI smoothness) accumulated alongside.  FAST: the model's fast step.
template <class Model, typename real, int VARIANT, bool FAST>
__device__ __forceinline__ void split_recurrence(const KArgs<real>& a, const typename Model::template P<real>& mp, const Smem<real>& sm,
                                                 unsigned long long kg, real* xcol, int BS, int T, real* x, real& pert, real& smooth) {
    typedef Ops<real> O;
    constexpr int NX = Model::NX, NU = Model::NU;
    const NoiseModel<real>& nm = a.nm;
    real vprev[NU];
#pragma unroll
    for (int n = 0; n < NU; ++n) vprev[n] = (real)0;
MPPI_UNROLL_N(MPPI_ROLLOUT_UNROLL)
    for (int t = 0; t < T; ++t) {
        real v[NU], u[NU], eps[NU];
        action_at<real, VARIANT, NU, true>(a, sm, kg, t, v);
        noise_at<real, VARIANT, NU, true>(a, sm, t, v, eps);
#pragma unroll
        for (int n = 0; n < NU; ++n) u[n] = O::mul(nm.u_scale, v[n]);            // mppi.py:313
        model_step<Model, real, FAST>(mp, x, u, t);                               // mppi.py:314
#pragma unroll
        for (int i = 0; i < NX; ++i) xcol[(t * NX + i) * BS] = x[i];
        action_terms<real, VARIANT, NU>(nm, sm.Us + t * NU, t, v, eps, pert, smooth, vprev);
    }
}

// The tiles a rollout reads (the first, the second and the nominal sequence), for the out-of-line rollouts: passing the
// whole Smem would keep all of its pointers live in the caller up to the call.
template <typename real> struct RolloutTiles {
    real *rows, *rows2, *Us;
    int LD;
    __device__ __forceinline__ RolloutTiles(const Smem<real>& sm) : rows(sm.rows), rows2(sm.rows2), Us(sm.Us), LD(sm.LD) {}
    __device__ __forceinline__ Smem<real> smem() const {
        Smem<real> sm;
        sm.rows = rows;
        sm.rows2 = rows2;
        sm.Us = Us;
        sm.LD = LD;
        return sm;
    }
};

// split_recurrence on the exact step, out of line (DESIGN §4.2 item 4: the straight path stays compact on a cold
// instruction cache).  The carry goes in and out by value, so that the inlined fast path keeps it in registers.
template <class Model, typename real, int VARIANT>
__device__ __noinline__ RolloutCarry<real, Model::NX> split_recurrence_rare(const KArgs<real>& a, const typename Model::template P<real>& mp,
                                                                            const RolloutTiles<real> tiles, unsigned long long kg, real* xcol,
                                                                            RolloutCarry<real, Model::NX> c) {
    split_recurrence<Model, real, VARIANT, false>(a, mp, tiles.smem(), kg, xcol, blockDim.x / a.tps, a.T, c.x, c.pert, c.smooth);
    return c;
}

// the T running costs of a split-cost rollout, spread over the sample's tps threads: cost_t overwrites x_t[0] in xs
template <class Model, typename real, int VARIANT, bool FAST>
__device__ __forceinline__ void split_costs(const KArgs<real>& a, const typename Model::template P<real>& mp, const Smem<real>& sm,
                                            unsigned long long kg, real* xcol, int tid, int BS, int T) {
    typedef Ops<real> O;
    constexpr int NX = Model::NX, NU = Model::NU;
MPPI_UNROLL_N(2)
    for (int t = tid / BS; t < T; t += a.tps) {      // independent across t: two in flight per thread
        real v[NU], u[NU], xt[NX];
        action_at<real, VARIANT, NU, true>(a, sm, kg, t, v);
#pragma unroll
        for (int n = 0; n < NU; ++n) u[n] = O::mul(a.nm.u_scale, v[n]);
#pragma unroll
        for (int i = 0; i < NX; ++i) xt[i] = xcol[(t * NX + i) * BS];
        xcol[(t * NX) * BS] = model_cost<Model, real, FAST>(mp, xt, u, t);      // mppi.py:318
    }
}

// ---- stage C', split-cost rollout as a function: recurrence on the rollout thread | running costs on all tps
// threads of the sample | ordered sum.  Returns the sample's total cost on its rollout thread (+inf elsewhere) and
// stores it to cost_total[k].  Contains two CTA barriers: every thread must call it.
// Shared by fused_command_kernel<..., SPLIT = true> and the resident kernel (mppi_resident.cuh).
// A model with a fast range has every thread of the sample read x_0 and check in_fast_range, so that its running costs
// take the form its recurrence took; other models read x_0 on the rollout thread only.
template <class Model, typename real, int VARIANT>
__device__ __forceinline__ real split_cost_rollout(const KArgs<real>& a, const typename Model::template P<real>& mp, Smem<real>& sm,
                                                   int k, unsigned long long kg, bool in_range, bool active) {
    static_assert(ModelCopies<Model>::value == 1, "models with COPIES > 1 run the single-loop rollout (copies_rollout)");
    typedef Ops<real> O;
    constexpr int NX = Model::NX;
    constexpr bool FR = FastRange<Model, real>::value;
    const int tid = threadIdx.x, BS = blockDim.x / a.tps, T = a.T;
    real c_tot = O::inf();
    real* xcol = sm.xs + (tid % BS);
    RolloutCarry<real, NX> c;
    c.pert = (real)0;
    c.smooth = (real)0;
    if constexpr (FR) {
        // the fast path reads its sizes where it uses them, the form its kernels (C2, C5) are tuned in
        bool fast = false;
        if (in_range) {
            initial_state<real, NX>(a, k, c.x);
            fast = Model::template in_fast_range<real>(mp, c.x, T);
        }
        if (active) {
            if (fast) split_recurrence<Model, real, VARIANT, true>(a, mp, sm, kg, xcol, blockDim.x / a.tps, a.T, c.x, c.pert, c.smooth);
            else c = split_recurrence_rare<Model, real, VARIANT>(a, mp, RolloutTiles<real>(sm), kg, xcol, c);
        }
        __syncthreads();
        if (in_range) {
            const int tid_ = threadIdx.x, BS_ = blockDim.x / a.tps, T_ = a.T;
            if (fast) split_costs<Model, real, VARIANT, true>(a, mp, sm, kg, xcol, tid_, BS_, T_);
            else split_costs<Model, real, VARIANT, false>(a, mp, sm, kg, xcol, tid_, BS_, T_);
        }
    } else {
        if (active) {
            initial_state<real, NX>(a, k, c.x);
            split_recurrence<Model, real, VARIANT, false>(a, mp, sm, kg, xcol, BS, T, c.x, c.pert, c.smooth);
        }
        __syncthreads();
        if (in_range) split_costs<Model, real, VARIANT, false>(a, mp, sm, kg, xcol, tid, BS, T);
    }
    __syncthreads();
    if (active) {
        real roll = (real)0;
        for (int t = 0; t < T; ++t) roll = O::add(roll, xcol[(t * NX) * BS]);         // mppi.py:319, t = 0..T-1
        if (Model::template has_terminal<real>(mp)) roll = O::add(roll, Model::template terminal<real>(mp, c.x));
        c_tot = sample_total<real, VARIANT>(a, k, roll, c.pert, c.smooth);
    }
    return c_tot;
}

// the single-loop rollout on the sample's rollout thread: dynamics, running cost, action cost (and SMPPI smoothness)
// per step.  FAST: the model's fast step and cost.
template <class Model, typename real, int VARIANT, bool FAST>
__device__ __forceinline__ void single_loop(const KArgs<real>& a, const typename Model::template P<real>& mp, const Smem<real>& sm,
                                            unsigned long long kg, int T, real* x, real& roll, real& pert, real& smooth) {
    typedef Ops<real> O;
    constexpr int NU = Model::NU;
    const NoiseModel<real>& nm = a.nm;
    real vprev[NU];
#pragma unroll
    for (int n = 0; n < NU; ++n) vprev[n] = (real)0;
    // The running cost of the state reached at step t-1 and the dynamics of step t both depend only on x_t, so the
    // unrolled loop issues them back to back: the single resident warp gets two independent dependency chains.  The
    // arithmetic and the order of every accumulation are exactly the reference's (cost summed t = 0..T-1).
MPPI_UNROLL_N(MPPI_ROLLOUT_UNROLL)
    for (int t = 0; t < T; ++t) {
        real v[NU], u[NU], eps[NU];
        action_at<real, VARIANT, NU, true>(a, sm, kg, t, v);
        noise_at<real, VARIANT, NU, true>(a, sm, t, v, eps);
#pragma unroll
        for (int n = 0; n < NU; ++n) u[n] = O::mul(nm.u_scale, v[n]);            // mppi.py:313
        model_step<Model, real, FAST>(mp, x, u, t);                               // mppi.py:314
        roll = O::add(roll, model_cost<Model, real, FAST>(mp, x, u, t));          // mppi.py:318-319
        action_terms<real, VARIANT, NU>(nm, sm.Us + t * NU, t, v, eps, pert, smooth, vprev);
    }
}

// single_loop on the exact step and cost, out of line (as split_recurrence_rare)
template <class Model, typename real, int VARIANT, bool G = false>      // G: as fill_normals_rare
__device__ __noinline__ RolloutCarry<real, Model::NX> single_loop_rare(const KArgs<real>& a, const typename Model::template P<real>& mp,
                                                                       const RolloutTiles<real> tiles, unsigned long long kg,
                                                                       RolloutCarry<real, Model::NX> c) {
    single_loop<Model, real, VARIANT, false>(a, mp, tiles.smem(), kg, a.T, c.x, c.roll, c.pert, c.smooth);
    return c;
}

// ---- stage C, the single-loop rollout (mppi.py:297-332) + action cost (mppi.py:409,415) [+ smoothness :559-562] on the
// sample's rollout thread: stores cost_total[k] and returns it.  T: the horizon as the kernel read it at entry; a model with
// a fast range reads it here instead (the form its kernels are tuned in: scripts/sass_rollout_loop.py).
template <class Model, typename real, int VARIANT, bool GTILE = false>
__device__ __forceinline__ real single_loop_rollout(const KArgs<real>& a, const typename Model::template P<real>& mp,
                                                    const Smem<real>& sm, int k, unsigned long long kg, int T) {
    typedef Ops<real> O;
    RolloutCarry<real, Model::NX> c;
    initial_state<real, Model::NX>(a, k, c.x);
    c.roll = (real)0;
    c.pert = (real)0;
    c.smooth = (real)0;
    if constexpr (FastRange<Model, real>::value) {
        if (Model::template in_fast_range<real>(mp, c.x, a.T)) single_loop<Model, real, VARIANT, true>(a, mp, sm, kg, a.T, c.x, c.roll, c.pert, c.smooth);
        else c = single_loop_rare<Model, real, VARIANT, GTILE>(a, mp, RolloutTiles<real>(sm), kg, c);
    } else {
        single_loop<Model, real, VARIANT, false>(a, mp, sm, kg, T, c.x, c.roll, c.pert, c.smooth);
    }
    if (Model::template has_terminal<real>(mp)) c.roll = O::add(c.roll, Model::template terminal<real>(mp, c.x));
    return sample_total<real, VARIANT>(a, k, c.roll, c.pert, c.smooth);
}

// one step's costs c[0..M-1] of the M copies (mppi.py:362-364): cs[m] += c[m], and var += var_m(c) * disc with the
// two-pass unbiased variance of cost_accumulate_kernel (mean = sum_m c / M, then sum_m (c - mean)^2 / (M - 1)).
// Models with copies at run time: M is the arrays' capacity and the first n <= M copies are folded.
template <typename real, int M>
__device__ __forceinline__ void copies_fold(real* cs, real& var, const real* c, real disc, const int n = M) {
    typedef Ops<real> O;
    real mean = c[0];
#pragma unroll
    for (int m = 1; m < M; ++m)
        if (m < n) mean = O::add(mean, c[m]);
    mean = O::div(mean, (real)n);
    real ss = (real)0;
#pragma unroll
    for (int m = 0; m < M; ++m) {
        if (m >= n) break;
        const real d = O::sub(c[m], mean);
        ss = O::add(ss, O::mul(d, d));
    }
    var = O::add(var, O::mul(O::div(ss, (real)(n - 1)), disc));
#pragma unroll
    for (int m = 0; m < M; ++m)
        if (m < n) cs[m] = O::add(cs[m], c[m]);
}

// ---- stage C'', rollout of a model with COPIES = M > 1 (rollout_samples, mppi.py:334-373), on the sample's rollout
// thread.  The M copies share the sample's action sequence, noise and action cost; their recurrences are M independent
// chains, interleaved in registers.  Per copy the running costs are summed t = 0..T-1, the discounted variance over the
// copies is accumulated per step, then cost = (mean_m(cost_m + terminal_m) + var * rollout_var_cost) + perturbation
// (+ SMPPI smoothness), in the reference's order (mppi.py:369-372, 415-416).  Stores cost_total[k] and returns it.
// A model with copies at run time (PendulumMLPEnsembleModel: a network per copy) rolls out mc = Model::copies(P) <= M
// copies, and the loops over them stay rolled (UNR = 1): its step is inlined once, and the per-copy arrays live in
// local memory (a few L1 accesses per copy and step, against the step's 1,184 FMAs).
template <class Model, typename real, int VARIANT>
__device__ __forceinline__ real copies_rollout(const KArgs<real>& a, const typename Model::template P<real>& mp, Smem<real>& sm,
                                               int k, unsigned long long kg) {
    typedef Ops<real> O;
    constexpr int NX = Model::NX, NU = Model::NU, M = ModelCopies<Model>::value;
    constexpr int UNR = CopiesAtRunTime<Model>::value ? 1 : M;
    const int mc = model_copies<Model, real>(mp);
    const NoiseModel<real>& nm = a.nm;
    const int T = a.T;
    real x[M][NX];
    initial_state<real, NX>(a, k, x[0]);
    real cs[M];
#pragma unroll
    for (int m = 0; m < M; ++m) {
        cs[m] = (real)0;
#pragma unroll
        for (int i = 0; i < NX; ++i) x[m][i] = x[0][i];
    }
    real var = (real)0, pert = (real)0, smooth = (real)0;
    real vprev[NU];
#pragma unroll
    for (int n = 0; n < NU; ++n) vprev[n] = (real)0;
    for (int t = 0; t < T; ++t) {
        real v[NU], u[NU], eps[NU], c[M];
        action_at<real, VARIANT, NU, true>(a, sm, kg, t, v);
        noise_at<real, VARIANT, NU, true>(a, sm, t, v, eps);
#pragma unroll
        for (int n = 0; n < NU; ++n) u[n] = O::mul(nm.u_scale, v[n]);                // mppi.py:355
        MPPI_UNROLL_N(UNR)
        for (int m = 0; m < mc; ++m) {
            model_step<Model, real>(mp, x[m], u, t, m);                                 // mppi.py:357
            c[m] = model_cost<Model, real>(mp, x[m], u, t, m);                          // mppi.py:362
        }
        copies_fold<real, M>(cs, var, c, __ldg(a.var_disc + t), mc);                     // mppi.py:363-364
        action_terms<real, VARIANT, NU>(nm, sm.Us + t * NU, t, v, eps, pert, smooth, vprev);
    }
    if (Model::template has_terminal<real>(mp)) {
        MPPI_UNROLL_N(UNR)
        for (int m = 0; m < mc; ++m) cs[m] = O::add(cs[m], model_terminal<Model, real>(mp, x[m], m));  // mppi.py:369-370
    }
    real mean = cs[0];
#pragma unroll
    for (int m = 1; m < M; ++m)
        if (m < mc) mean = O::add(mean, cs[m]);
    mean = O::div(mean, (real)mc);                                                        // mppi.py:371
    return sample_total<real, VARIANT>(a, k, O::add(mean, O::mul(var, a.var_cost)), pert, smooth);   // mppi.py:372
}

// =================================================================================================
// The fused command kernel
// =================================================================================================
// SPLIT (threads_per_sample > 1 only, i.e. problems too small to fill the machine): the rollout is the one
// phase a sample's helper threads cannot share — the state recurrence is serial.  But only the DYNAMICS are:
// the running cost of step t depends on x_t alone.  So the rollout thread runs the bare recurrence and parks
// every x_t in shared memory (xs[T*NX][BS]); then all tps threads of the sample evaluate the T running costs
// in parallel (in place: cost_t overwrites x_t[0]); then the rollout thread adds them up in the reference's
// order t = 0..T-1.  Same operations, same rounding, same summation order as the fused loop — the single
// resident warp just stops carrying the cost's ~45 instructions per step on its critical path.
//
// MINB: minimum resident CTAs per SM promised to ptxas.  The split-cost kernels (one CTA per SM by construction) get 1: the
// whole register file.  The single-loop kernels of the analytic models get 2 = a 64-register cap (20 B of spill): the
// two-CTA-per-SM geometry of large K needs it, and without the promise the out-of-line tail functions push ptxas to 128
// registers and one CTA per SM (measured at K = 131072: 42 -> 53 us).  The MLP's step keeps 64 activations live: it gets
// the whole register file (one CTA per SM) — under the cap it spilled 340 B per thread.  So do models with COPIES > 1:
// at M = 8 (the test models of tests/ensemble_models.py) the M states, costs and cost sums of copies_rollout spilled
// 42-62 B (fp32) and 458-578 B (fp64) of stores per thread under the cap; without it fp32 takes 122-124 registers and
// does not spill, fp64 takes 128 and spills 4-62 B.
template <class Model> struct FusedMinBlocks {
    static constexpr int value = ModelCopies<Model>::value > 1 ? 1 : MPPI_FUSED_MIN_BLOCKS;
};
template <> struct FusedMinBlocks<PendulumMLPModel> { static constexpr int value = 1; };

// LL1: the tail of warp_tail<..., LL1 = true> (fused_command_kernel_ll below)
// GTILE: the tiles in this CTA's workspace slice (fused_command_kernel_gtile below; single loop only)
template <class Model, typename real, int VARIANT, bool BATCHED, bool SPLIT, bool LL1, bool GTILE = false>
__device__ __forceinline__ void fused_command_body(const KArgs<real>& a_in, const typename Model::template P<real>& mp) {
    static_assert(!(GTILE && (SPLIT || LL1)), "the global-tile kernel runs the single-loop rollout");
    typedef Ops<real> O;
    constexpr int NX = Model::NX, NU = Model::NU;
    extern __shared__ __align__(16) unsigned char smem[];
    const int tid = threadIdx.x, BD = blockDim.x;
    __shared__ __align__(16) unsigned char a_env_raw[BATCHED ? sizeof(KArgs<real>) : 16];
    if (BATCHED) make_env_args<real, NX, NU, true>(a_in, reinterpret_cast<KArgs<real>*>(a_env_raw));
    const KArgs<real>& a = BATCHED ? *reinterpret_cast<const KArgs<real>*>(a_env_raw) : a_in;
    const int BS = BD / a.tps;
    const int xst = fused_xstage_doubles(a.world > 1 && !a.export_partial, a.world, a.xchg_npub, a.R);
    const int cs_ = (int)cluster_nctarank(), NC_ = (int)gridDim.x / cs_;
    // the layout is the plan's (a_in.T): with per-environment horizons a.T is this environment's h_e
    const SmemLayout L = make_layout<real>(VARIANT, a_in.T, NU, a.S, a.R, BD, BS, fused_layout_nb(NC_, a.xchg_npub),
                                           layout_extra(VARIANT != V_MPPI, SPLIT ? NX : 0, cs_, xst), GTILE);
    Smem<real> sm(smem, L);
    if (GTILE) gtile_bind<real>(a, sm, VARIANT != V_MPPI);
    const int T = a.T;
    warp_records_init<real>(a, sm);      // published by the barrier in stage_issue
    // phase 0 of the cluster barrier: "this CTA has started" — the tail waits for it before the first store into the
    // leader's shared memory (distributed shared memory may only be touched once its CTA is known to be running)
    if (cs_ > 1) cluster_arrive_relaxed();

    stamp(a.dbg, 0);
    // Programmatic dependent launch: this grid may be resident while the previous kernel on the stream is
    // still finishing.  Let our own successor start early too, draw the first tile's normals (pure
    // compute into shared memory), and only then wait for the predecessor's memory to be visible.
    // (GTILE: the first tile is global memory that the previous command's CTAs may still be folding from — nothing is
    // written before the wait)
    const bool early_fill = !GTILE && a.pdl && a.z == nullptr && a.z_out == nullptr && blockIdx.x < a.n_tiles;
    if (a.pdl) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    if (early_fill) {
        const int k0 = blockIdx.x * BS + (tid % BS);
        fill_normals<real, GTILE>(a, sm, blockIdx.x, k0 < a.K, (unsigned long long)(a.k_offset + k0), min(BS, a.K - blockIdx.x * BS));
    }
    if (a.pdl) asm volatile("griddepcontrol.wait;" ::: "memory");
    if constexpr (GTILE) stage_issue_gtile<real, VARIANT, NU>(a, sm);
    else stage_issue<real, VARIANT, NU>(a, sm);
    stamp(a.dbg, 1);
    bool staged = false;

    for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
        const int k = tile * BS + (tid % BS);
        const bool in_range = k < a.K;
        const bool active = in_range && tid < BS;      // the rollout thread of sample k
        const int nvalid = min(BS, a.K - tile * BS);
        const unsigned long long kg = (unsigned long long)(a.k_offset + k);

        if (!(early_fill && tile == blockIdx.x)) fill_normals<real, GTILE>(a, sm, tile, in_range, kg, nvalid);
        if (!staged) {   // the nominal sequence is first needed now; its TMA copy flew during the draws
            stage_finish<real, VARIANT, NU>(a, sm);
            staged = true;
        } else if (a.tps > 1) {
            __syncthreads();
        }
        if (tile == blockIdx.x) stamp(a.dbg, 2);
        if (in_range) transform_column<real, VARIANT, NU, true>(a, sm, kg);
        if (a.tps > 1) __syncthreads();
        if (VARIANT == V_KMPPI) {      // the control points of the sample are complete: interpolate them onto the horizon
            if (in_range) interp_column<real, NU>(a, sm, kg);
            if (a.tps > 1) __syncthreads();
        }
        if (tile == blockIdx.x) stamp(a.dbg, 3);

        real c_tot = O::inf();
        if constexpr (SPLIT) {
            // C'. split rollout: recurrence (rollout thread) | running costs (all tps threads) | ordered sum
            c_tot = split_cost_rollout<Model, real, VARIANT>(a, mp, sm, k, kg, in_range, active);
        } else if constexpr (ModelCopies<Model>::value > 1) {
            // C''. M copies of the sample's rollout, interleaved in registers
            if (active) c_tot = copies_rollout<Model, real, VARIANT>(a, mp, sm, k, kg);
        } else if (active) {
            // C. the single loop
            c_tot = single_loop_rollout<Model, real, VARIANT, GTILE>(a, mp, sm, k, kg, T);
        }
        if (tile == blockIdx.x) stamp(a.dbg, 4);
        // D. every rollout warp folds its 32 samples into its own running record (no CTA barrier)
        if (tid < BS) warp_fold<real, VARIANT>(a, sm, c_tot, active, nvalid);
        if (tile == blockIdx.x) stamp(a.dbg, 5);
        if (tile + (int)gridDim.x < a.n_tiles) __syncthreads();      // the tile is refilled by the next pass
    }
    if (!staged) stage_finish<real, VARIANT, NU>(a, sm);
    warp_tail<real, VARIANT, NU, false, LL1, BATCHED>(a, sm);
    stamp(a.dbg, 7);
}

template <class Model, typename real, int VARIANT, bool BATCHED, bool SPLIT = false, int MINB = (SPLIT ? 1 : FusedMinBlocks<Model>::value)>
__global__ void __launch_bounds__(512, MINB) fused_command_kernel(const __grid_constant__ KArgs<real> a_in,
                                                            const __grid_constant__ typename Model::template P<real> mp) {
    fused_command_body<Model, real, VARIANT, BATCHED, SPLIT, false>(a_in, mp);
}

// The split-cost kernel of single-GPU plans in LL mode (the host selects it: NC > 1 clusters, every cluster record in this
// GPU's own mailbox, no peers, no export): its tail is the one path that geometry runs, inlined (warp_tail, LL1).  Every
// other plan keeps fused_command_kernel, whose tail serves all modes through shared out-of-line code.
template <class Model, typename real, int VARIANT>
__global__ void __launch_bounds__(512, 1) fused_command_kernel_ll(const __grid_constant__ KArgs<real> a_in,
                                                                  const __grid_constant__ typename Model::template P<real> mp) {
    fused_command_body<Model, real, VARIANT, false, true, true>(a_in, mp);
}

// The single-loop kernel with its tiles in the workspace (MPPI_FLAG_GLOBAL_TILE): horizons whose R x (BS+1) tile does not
// fit in shared memory.  Same stages, same functions, same order of operations — only the tile pointers differ.
template <class Model, typename real, int VARIANT, bool BATCHED>
__global__ void __launch_bounds__(512, FusedMinBlocks<Model>::value) fused_command_kernel_gtile(
    const __grid_constant__ KArgs<real> a_in, const __grid_constant__ typename Model::template P<real> mp) {
    fused_command_body<Model, real, VARIANT, BATCHED, false, false, true>(a_in, mp);
}

// Batched environments with their own model parameters (mppi_plan_set_env_params): environment blockIdx.y's parameter
// block is read in place, through L1, from the n_env blocks packed env_stride bytes apart (16-byte aligned, as the plant
// blocks of a closed loop) — in place of the one block the other kernels take as a __grid_constant__ argument.
// GTILE: the global-tile form.
template <class Model, typename real, bool GTILE>
__device__ __forceinline__ void fused_command_env_body(const KArgs<real>& a_in, const unsigned char* __restrict__ env_mp,
                                                       long long env_stride) {
    typedef typename Model::template P<real> P;
    const P& mp = *reinterpret_cast<const P*>(env_mp + (size_t)blockIdx.y * (size_t)env_stride);
    fused_command_body<Model, real, V_MPPI, true, false, false, GTILE>(a_in, mp);
}
template <class Model, typename real, bool GTILE>
__global__ void __launch_bounds__(512, 1) fused_command_kernel_env(
    const __grid_constant__ KArgs<real> a_in, const unsigned char* __restrict__ env_mp, long long env_stride) {
    fused_command_env_body<Model, real, GTILE>(a_in, env_mp, env_stride);
}

#ifdef __CUDACC_RTC__
// A user model (NVRTC, one module per dtype and controller variant) exports its fused_command_kernel_ll under one unmangled
// name, which mppi_user_model_register looks up beside the kernels it is given by name.
#define MPPI_USER_KERNEL_LL(Model, real, VARIANT)                                                                            \
    extern "C" __global__ void __launch_bounds__(512, 1) mppi_user_fused_command_kernel_ll(                                 \
        const __grid_constant__ mppi::KArgs<real> a_in, const __grid_constant__ Model::P<real> mp) {                         \
        mppi::fused_command_body<Model, real, VARIANT, false, true, true>(a_in, mp);                                         \
    }
// ... and its global-tile kernels (mppi_user_model_register looks them up by these names): the single-loop kernel, and for
// MPPI_Batched (MPPI variant, one copy) the batched one
#define MPPI_USER_KERNEL_GTILE(Model, real, VARIANT)                                                                         \
    extern "C" __global__ void __launch_bounds__(512, mppi::FusedMinBlocks<Model>::value) mppi_user_fused_command_kernel_gtile( \
        const __grid_constant__ mppi::KArgs<real> a_in, const __grid_constant__ Model::P<real> mp) {                         \
        mppi::fused_command_body<Model, real, VARIANT, false, false, false, true>(a_in, mp);                                 \
    }
#define MPPI_USER_KERNEL_GTILE_BATCHED(Model, real)                                                                          \
    extern "C" __global__ void __launch_bounds__(512, mppi::FusedMinBlocks<Model>::value)                                    \
        mppi_user_fused_command_kernel_gtile_batched(const __grid_constant__ mppi::KArgs<real> a_in,                         \
                                                     const __grid_constant__ Model::P<real> mp) {                            \
        mppi::fused_command_body<Model, real, mppi::V_MPPI, true, false, false, true>(a_in, mp);                             \
    }
// ... and, for MPPI_Batched, the batched kernels with per-environment model parameters (fused_command_kernel_env)
#define MPPI_USER_KERNEL_ENV_BATCHED(Model, real)                                                                            \
    extern "C" __global__ void __launch_bounds__(512, 1)                                                                     \
        mppi_user_fused_command_kernel_env(const __grid_constant__ mppi::KArgs<real> a_in,                                   \
                                           const unsigned char* __restrict__ env_mp, long long env_stride) {                 \
        mppi::fused_command_env_body<Model, real, false>(a_in, env_mp, env_stride);                                          \
    }                                                                                                                        \
    extern "C" __global__ void __launch_bounds__(512, 1)                                                                     \
        mppi_user_fused_command_kernel_env_gtile(const __grid_constant__ mppi::KArgs<real> a_in,                             \
                                                 const unsigned char* __restrict__ env_mp, long long env_stride) {           \
        mppi::fused_command_env_body<Model, real, true>(a_in, env_mp, env_stride);                                           \
    }
#endif

// =================================================================================================
// Generic path, part 1: sample + perturb with coalesced write-out (mppi.py:375-385, 409, 415;
// SMPPI :539-562; KMPPI :657-670).  Also used to materialise noise/perturbed_action lazily.
// =================================================================================================
// GTILE: the tiles in this CTA's workspace slice (sample_kernel_gtile)
template <typename real, int VARIANT, int NU, bool GTILE>
__device__ __forceinline__ void sample_body(const KArgs<real>& a_in) {
    typedef Ops<real> O;
    extern __shared__ __align__(16) unsigned char smem[];
    const int tid = threadIdx.x, BD = blockDim.x;
    __shared__ __align__(16) unsigned char a_env_raw[sizeof(KArgs<real>)];
    if (a_in.n_env > 1) make_env_args<real, 0, NU>(a_in, reinterpret_cast<KArgs<real>*>(a_env_raw));
    const KArgs<real>& a = a_in.n_env > 1 ? *reinterpret_cast<const KArgs<real>*>(a_env_raw) : a_in;
    const int BS = BD / a.tps;
    const SmemLayout L = make_layout<real>(VARIANT, a.T, NU, a.S, a.R, BD, BS, 1, VARIANT == V_KMPPI, GTILE);
    Smem<real> sm(smem, L);
    if (GTILE) gtile_bind<real>(a, sm, VARIANT == V_KMPPI);
    const NoiseModel<real>& nm = a.nm;
    const int T = a.T, R = a.R, TN = a.TN, LD = sm.LD;

    if constexpr (GTILE) {
        stage_issue_gtile<real, VARIANT, NU>(a, sm);
        stage_finish<real, VARIANT, NU>(a, sm);
    } else {
        stage_nominal<real, VARIANT, NU>(a, sm);
    }
    if (blockIdx.x == 0 && a.nominal_used != nullptr) {
        for (int j = tid; j < TN; j += BD) {
            a.nominal_used[j] = sm.Us[j];
            if (VARIANT == V_SMPPI) a.nominal_used[TN + j] = sm.As[j];
        }
        if (VARIANT == V_KMPPI)
            for (int j = tid; j < R; j += BD) a.nominal_used[2 * TN + j] = sm.ths[j];
    }

    for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
        const int k = tile * BS + (tid % BS);
        const bool in_range = k < a.K;
        const bool active = in_range && tid < BS;
        const int nvalid = min(BS, a.K - tile * BS);
        const unsigned long long kg = (unsigned long long)(a.k_offset + k);
        fill_normals<real, GTILE>(a, sm, tile, in_range, kg, nvalid);
        if (a.tps > 1) __syncthreads();
        if (in_range) transform_column<real, VARIANT, NU>(a, sm, kg);
        if (a.tps > 1) __syncthreads();
        if (active) {
            real pert = (real)0, smooth = (real)0;
            real vprev[NU];
#pragma unroll
            for (int n = 0; n < NU; ++n) vprev[n] = (real)0;
            for (int t = 0; t < T; ++t) {
                real v[NU], eps[NU];
                action_at<real, VARIANT, NU>(a, sm, kg, t, v);
                noise_at<real, VARIANT, NU>(a, sm, t, v, eps);
                action_terms<real, VARIANT, NU>(nm, sm.Us + t * NU, t, v, eps, pert, smooth, vprev);
                if (VARIANT == V_KMPPI) {
#pragma unroll
                    for (int n = 0; n < NU; ++n) sm.rows2[(t * NU + n) * LD + tid] = v[n];
                }
            }
            if (a.out_cost_init != nullptr) {
                real c0 = pert;
                if (VARIANT == V_SMPPI) c0 = O::add(c0, O::mul(smooth, nm.w_smooth));
                a.out_cost_init[k] = c0;
            }
        }
        __syncthreads();
        // coalesced write-out of the tile: (K,T,nu) row-major == [sample][j]
        {
            const real* vt = (VARIANT == V_KMPPI) ? sm.rows2 : sm.rows;
            const size_t base = (size_t)tile * BS * TN;
            const int count = nvalid * TN;
            for (int e = tid; e < count; e += BD) {
                const int s = e / TN, j = e - s * TN;
                const real val = vt[j * LD + s];
                if (a.out_pa != nullptr) a.out_pa[base + e] = val;
                if (a.out_noise != nullptr) {
                    real ep;
                    if (VARIANT == V_SMPPI) ep = O::sub(O::div(O::sub(val, sm.As[j]), nm.delta_t), sm.Us[j]);
                    else ep = O::sub(val, sm.Us[j]);
                    a.out_noise[base + e] = ep;
                }
            }
            if (VARIANT == V_KMPPI && a.out_noise_theta != nullptr) {
                const size_t base2 = (size_t)tile * BS * R;
                const int count2 = nvalid * R;
                for (int e = tid; e < count2; e += BD) {
                    const int s = e / R, j = e - s * R;
                    a.out_noise_theta[base2 + e] = O::sub(sm.rows[j * LD + s], sm.ths[j]);
                }
            }
        }
        __syncthreads();
    }
}
template <typename real, int VARIANT, int NU>
__global__ void __launch_bounds__(512) sample_kernel(const __grid_constant__ KArgs<real> a_in) {
    sample_body<real, VARIANT, NU, false>(a_in);
}
template <typename real, int VARIANT, int NU>
__global__ void __launch_bounds__(512) sample_kernel_gtile(const __grid_constant__ KArgs<real> a_in) {
    sample_body<real, VARIANT, NU, true>(a_in);
}

// Step t of an open-loop replay of the action rows pa: u = u_scale * pa[t] (mppi.py:313 / :445), then the model's step — FAST: its
// fast form, which a replay takes throughout when in_fast_range holds for its start state and length, as the command's
// rollouts do.  The states kernel (get_rollouts, the states along a command's rollouts) and the plant step of a closed
// loop (a one-row replay) both step through here, so a closed loop's plant is get_rollouts(x, U=u[None]) bit for bit.
template <class Model, typename real, bool FAST>
__device__ __forceinline__ void replay_step(const typename Model::template P<real>& mp, real* x, real* u, const real* pa,
                                            real u_scale, int t, int m) {
    for (int n = 0; n < Model::NU; ++n) u[n] = Ops<real>::mul(u_scale, pa[t * Model::NU + n]);   // mppi.py:313 / :445
    model_step<Model, real, FAST>(mp, x, u, t, m);
}

// the states of sample k's replay from x, on the model's fast step (FAST) or not
template <class Model, typename real, bool FAST>
__device__ __forceinline__ void replay_states(const KArgs<real>& a, const typename Model::template P<real>& mp, real* x, const real* pa,
                                              real* states, int k, int m) {
    for (int t = 0; t < a.T; ++t) {
        real u[Model::NU];
        replay_step<Model, real, FAST>(mp, x, u, pa, a.nm.u_scale, t, m);
        for (int i = 0; i < Model::NX; ++i) states[((size_t)k * a.T + t) * Model::NX + i] = x[i];
    }
}

// states along the rollout of given perturbed actions (mppi.py:307-322), for registered models.
// pa_stride = elements between consecutive samples' action sequences: T*nu for a (K,T,nu) tensor, 0 when every
// sample replays the SAME (T,nu) sequence (get_rollouts, mppi.py:425-448).
// Models with COPIES > 1: blockIdx.y is the copy, states are (gridDim.y, K, T, nx) (mppi.py:345, 366).
template <class Model, typename real>
__global__ void states_kernel(const real* __restrict__ pa, real* __restrict__ states, const KArgs<real> a,
                              const typename Model::template P<real> mp, long long pa_stride) {
    constexpr int NX = Model::NX;
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= a.K) return;
    int m = 0;
    if constexpr (ModelCopies<Model>::value > 1) {
        m = blockIdx.y;
        states += (size_t)m * a.K * a.T * NX;
    }
    pa += (size_t)k * (size_t)pa_stride;
    real x[NX];
    initial_state<real, NX>(a, k, x);
    if constexpr (FastRange<Model, real>::value) {      // the fast step where the command's rollouts take it
        if (Model::template in_fast_range<real>(mp, x, a.T)) {
            replay_states<Model, real, true>(a, mp, x, pa, states, k, 0);
            return;
        }
    }
    replay_states<Model, real, false>(a, mp, x, pa, states, k, m);
}

// One plant step of a closed-loop episode (mppi_plan_closed_loop), one thread per environment: after the command of
// control step s wrote its action row, x_{s+1} = step(x_s, u_scale * u_s) with the environment's plant parameter block
// (the replay of get_rollouts(x_s, U=u_s[None])), plus the disturbance row; the running cost of the reached state with
// the same (scaled) action, t = 0, as a rollout scores its first step (mppi.py:313-319).
template <typename real> struct PlantStepArgs {
    const real* x;                  // (n_env, nx) state row s
    real* x_next;                   // (n_env, nx) state row s + 1
    const real* u;                  // (n_env, nu) action row s (the command's action_out)
    const real* w;                  // (n_env, nx) disturbance row s, or nullptr
    real* cost;                     // (n_env) cost row s, or nullptr
    const unsigned char* plants;    // n_plant parameter blocks (Model::P<real>), plant_stride bytes apart
    long long plant_stride;
    int n_env, n_plant;
    real u_scale;
};
// x_{s+1} and the cost of environment e, on the model's fast step or not (the caller's in_fast_range choice)
template <class Model, typename real, bool FAST>
__device__ __forceinline__ void plant_step_env(const PlantStepArgs<real>& a, const typename Model::template P<real>& mp, real* x, int e) {
    typedef Ops<real> O;
    constexpr int NX = Model::NX, NU = Model::NU;
    real u[NU];
    replay_step<Model, real, FAST>(mp, x, u, a.u + (size_t)e * NU, a.u_scale, 0, 0);
    if (a.w != nullptr)
        for (int i = 0; i < NX; ++i) x[i] = O::add(x[i], a.w[(size_t)e * NX + i]);
    for (int i = 0; i < NX; ++i) a.x_next[(size_t)e * NX + i] = x[i];
    // the cost of the state reached, disturbance included: on the model's general form (its fast form is bit-identical
    // only inside the range in_fast_range vouched for, which a disturbance may leave)
    if (a.cost != nullptr) a.cost[e] = model_cost<Model, real>(mp, x, u, 0);                  // mppi.py:318, t = 0
}
template <class Model, typename real>
__device__ __forceinline__ void plant_step_body(const PlantStepArgs<real>& a) {
    constexpr int NX = Model::NX;
    // launched behind the command (programmatic dependent launch): let the next command start drawing its noise, then
    // wait until this command's action row is written.  Without the launch attribute both are no-ops.
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a.n_env) return;
    const typename Model::template P<real>& mp = *reinterpret_cast<const typename Model::template P<real>*>(
        a.plants + (size_t)(a.n_plant > 1 ? e : 0) * (size_t)a.plant_stride);
    real x[NX];
    for (int i = 0; i < NX; ++i) x[i] = a.x[(size_t)e * NX + i];
    if constexpr (FastRange<Model, real>::value) {      // as the states kernel chooses for a one-row replay
        if (Model::template in_fast_range<real>(mp, x, 1)) {
            plant_step_env<Model, real, true>(a, mp, x, e);
            return;
        }
    }
    plant_step_env<Model, real, false>(a, mp, x, e);
}
template <class Model, typename real>
__global__ void __launch_bounds__(128) plant_step_kernel(const PlantStepArgs<real> a) {
    plant_step_body<Model, real>(a);
}

#ifdef __CUDACC_RTC__
// A user model exports its plant step under one unmangled name, which mppi_user_model_register looks up (step-dependent
// models have none: a per-step schedule has no step index in a closed loop)
#define MPPI_USER_KERNEL_PLANT(Model, real)                                                                                  \
    extern "C" __global__ void __launch_bounds__(128) mppi_user_plant_step_kernel(const mppi::PlantStepArgs<real> a) {       \
        mppi::plant_step_body<Model, real>(a);                                                                               \
    }
#endif

// =================================================================================================
// Generic path, part 2: softmin + weighted update from materialised cost_total (K) and eps (K,R)
// (mppi.py:254-259, 268-270).  HBM-bound: reads 4*K*(R+1) bytes once, coalesced.
// The warp-fold tail runs without clusters and with one published record per rank (xchg_npub = 1): ticket mode on one
// GPU, rank-record mode on a sharded controller.  Never LL mode: a single-GPU stepped command does not advance the
// record epoch, and CUDA-graph replays repeat one, so LL records of the previous command would pass for this one's.
// =================================================================================================
// GTILE: the tile in this CTA's workspace slice (softmin_update_kernel_gtile)
template <typename real, int VARIANT, int NU, bool GTILE>
__device__ __forceinline__ void softmin_update_body(const KArgs<real>& a_in) {
    typedef Ops<real> O;
    extern __shared__ __align__(16) unsigned char smem[];
    const int tid = threadIdx.x, BD = blockDim.x;
    const int BS = BD / a_in.tps;
    const int xst = fused_xstage_doubles(a_in.world > 1 && !a_in.export_partial, a_in.world, 1, a_in.R);
    const SmemLayout L = make_layout<real>(VARIANT, a_in.T, NU, a_in.S, a_in.R, BD, BS, fused_layout_nb(gridDim.x, 1),
                                           layout_extra(0, 0, 1, xst), GTILE);
    // batched environments: the per-environment argument view sits behind the layout (the host adds its size), so that
    // one environment pays no shared memory for it and this kernel plans every horizon the fused kernel does
    KArgs<real>* a_env = reinterpret_cast<KArgs<real>*>(smem + L.total);
    if (a_in.n_env > 1) make_env_args<real, 0, NU>(a_in, a_env);
    const KArgs<real>& a = a_in.n_env > 1 ? *a_env : a_in;
    Smem<real> sm(smem, L);
    if (GTILE) gtile_bind<real>(a, sm, 0);
    const int R = a.R, TN = a.TN, LD = sm.LD;
    warp_records_init<real>(a, sm);
    // post-shift nominal comes from nominal_used (written by sample_kernel)
    for (int j = tid; j < TN; j += BD) {
        sm.Us[j] = a.nominal_used[j];
        if (VARIANT == V_SMPPI) sm.As[j] = a.nominal_used[TN + j];
    }
    if (VARIANT == V_KMPPI) {
        for (int j = tid; j < R; j += BD) sm.ths[j] = a.nominal_used[2 * TN + j];
        if (!GTILE)
            for (int j = tid; j < a.T * a.S; j += BD) sm.Ws[j] = a.W[j];
    }
    for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
        const int k = tile * BS + tid;
        const bool active = tid < BS && k < a.K;
        const int nvalid = min(BS, a.K - tile * BS);
        const size_t base = (size_t)tile * BS * R;
        const int count = nvalid * R;
        __syncthreads();      // the previous tile is folded before the tile is refilled
        for (int e = tid; e < count; e += BD) {
            const int s = e / R, j = e - s * R;
            sm.rows[j * LD + s] = a.in_eps[base + e];
        }
        const real c = active ? a.in_cost[k] : O::inf();
        __syncthreads();
        if (tid < BS) warp_fold<real, VARIANT, false, true>(a, sm, c, active, nvalid);
    }
    warp_tail<real, VARIANT, NU>(a, sm);
}
template <typename real, int VARIANT, int NU>
__global__ void __launch_bounds__(512) softmin_update_kernel(const __grid_constant__ KArgs<real> a_in) {
    softmin_update_body<real, VARIANT, NU, false>(a_in);
}
template <typename real, int VARIANT, int NU>
__global__ void __launch_bounds__(512) softmin_update_kernel_gtile(const __grid_constant__ KArgs<real> a_in) {
    softmin_update_body<real, VARIANT, NU, true>(a_in);
}

// omega_k = exp(-(c_k - beta)/lambda) / eta from the stats a command left behind (mppi.py:256-258)
template <typename real>
__global__ void omega_kernel(const real* __restrict__ cost, real* __restrict__ omega, const double* __restrict__ stats,
                             real neg_inv_lambda, int K) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= K) return;
    const real beta = (real)stats[0];
    const real inv_eta = (real)(1.0 / stats[1]);
    omega[k] = inv_eta * Ops<real>::exp_(neg_inv_lambda * (cost[k] - beta));
}

// cost[m,k] += c[m,k]  (mppi.py:319 / 363); M>1: var_acc[k] += var_m(c[:,k]) * discount (mppi.py:364)
template <typename real>
__global__ void cost_accumulate_kernel(real* __restrict__ cost, const real* __restrict__ c, real* __restrict__ var_acc,
                                       int M, int K, real discount) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= K) return;
    real mean = (real)0;
    for (int m = 0; m < M; ++m) {
        const real v = c[(size_t)m * K + k];
        cost[(size_t)m * K + k] += v;
        mean += v;
    }
    if (var_acc != nullptr && M > 1) {
        mean /= (real)M;
        real ss = (real)0;
        for (int m = 0; m < M; ++m) {
            const real d = c[(size_t)m * K + k] - mean;
            ss += d * d;
        }
        var_acc[k] += ss / (real)(M - 1) * discount;
    }
}

// ---- finish from all-gathered partials (library-collective route) --------------------------------
template <typename real, int VARIANT>
__global__ void apply_partials_kernel(const KArgs<real> a, const double* partials, int nu) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int tid = threadIdx.x, BD = blockDim.x;
    const int TN = a.TN, R = a.R, T = a.T, S = a.S;
    real* Us = reinterpret_cast<real*>(smem);
    real* As = Us + TN;
    real* ths = As + TN;
    real* Ws = ths + R;
    double* numd = reinterpret_cast<double*>(smem + align_up((2 * TN + R + T * S) * (int)sizeof(real), 16));
    for (int j = tid; j < TN; j += BD) {
        Us[j] = a.nominal_used[j];
        As[j] = (VARIANT == V_SMPPI) ? a.nominal_used[TN + j] : (real)0;
    }
    if (VARIANT == V_KMPPI) {
        for (int j = tid; j < R; j += BD) ths[j] = a.nominal_used[2 * TN + j];
        for (int j = tid; j < T * S; j += BD) Ws[j] = a.W[j];
    }
    const double nfl = (double)a.nm.neg_inv_lambda;
    double beta = partials[0];
    for (int g = 1; g < a.world; ++g) beta = fmin(beta, partials[(size_t)g * (R + 2)]);
    for (int j = tid; j < R + 1; j += BD) {
        double acc = 0.0;
        for (int g = 0; g < a.world; ++g) {
            const double* rec = partials + (size_t)g * (R + 2);
            acc += exp(nfl * (rec[0] - beta)) * rec[1 + j];
        }
        numd[1 + j] = acc;
    }
    if (tid == 0) numd[0] = beta;
    __syncthreads();
    finish_update<real, VARIANT>(a, numd, Us, As, ths, Ws, nu);
    if (tid == 0) a.stats[3] = 0.0;
}

#endif  // __CUDACC__

}  // namespace mppi
