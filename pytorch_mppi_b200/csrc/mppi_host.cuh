// mppi_host.cuh — host side shared by the translation units of the library: parameter validation, launch geometry,
// argument packing, plans, and the per-model launch/plan templates.  The library is built from several translation
// units (mppi_b200.cu: C ABI + the model-independent kernels; mppi_model_tu.cu compiled once per (model, dtype):
// the fused / resident / states kernels of that model) so that it compiles in parallel; everything here has
// internal linkage (anonymous namespace) except the few declarations in namespace mppi_host that cross units.
#pragma once
#include <cuda_runtime.h>
#include <new>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <type_traits>

#include "../../include/mppi_b200.h"
#include "mppi_fused.cuh"
#include "mppi_model_tensors.h"
#include "mppi_resident.cuh"
#include "mppi_resident_host.h"

using namespace mppi;

namespace mppi_host {

// last error text of the calling thread (one definition, in mppi_b200.cu)
extern thread_local char g_cuda_err[512];

#define MPPI_MODEL_BLOCK_BYTES 12288     // largest Model::P<real> a kernel takes by value (the MLP's weights: 10 KB in fp64)

struct Geometry {
    int BD, BS, tps, nb, smem, occ, regs;   // BD = BS * tps threads per CTA, BS samples per tile
    int cluster;                            // thread-block-cluster size of the launch (1: none); nb is a multiple of it
    int npub;                               // sharded controllers: records published per rank and command (0: not sharded)
};

// Resident mode: the host side of the protocol (struct Resident, res_*) is csrc/mppi_resident_host.h; this file supplies its
// backend (cooperative launch / stream synchronise / stream query).
struct ResidentDevice {
    unsigned long long* host_box = nullptr;
    unsigned long long* board = nullptr;
    void* action_dev = nullptr;
    cudaStream_t stream = nullptr;
    unsigned long long idle_ns = 0;
};

struct ModelKernels;

struct Plan {
    MppiFusedParams p;
    const ModelKernels* mk;            // the model's kernels and parameter packer (mppi_plan_set_model_params re-packs)
    const void* kernel;
    const void* res_kernel;            // resident_command_kernel<Model, real, V>, or nullptr when this plan cannot run resident
    Resident res;
    ResidentDevice resdev;
    Geometry g;
    int is_double, nx, upc_nu, pdl;
    unsigned long long epoch, host_epoch;
    unsigned long long res_epoch_off;  // resident mode: record-mailbox epoch of command seq = res_epoch_off + seq
    alignas(16) unsigned char kargs[sizeof(KArgs<double>)];
    alignas(16) unsigned char mparams[MPPI_MODEL_BLOCK_BYTES];
    MppiTensorRef tensors[MPPI_MAX_MODEL_TENSORS];   // the plan's copy of p.model_tensors (p.model_tensors points here)
    // per-environment model parameters (mppi_plan_set_env_params): the kernel that reads them and the packed blocks in
    // the caller's scratch (env_kernel nullptr: the plan's own block, `kernel`)
    const void* env_kernel;
    const unsigned char* env_mp;
    long long env_stride;
};

// What one (model, dtype) pair contributes: its kernels (as launchable handles) and how to pack its parameter block.
// The six registry units (mppi_model_tu.cu) each export one statically; a user model compiled at run time with NVRTC
// (mppi_user_model_register) gets one on the heap.  Everything that selects and launches kernels (mppi_fused_host.cuh)
// works on this descriptor, so it is compiled once, not per model.
struct ModelKernels {
    int nx, nu;
    int is_double;
    int is_mlp;                      // 1 PendulumMLP, 2 its ensemble: no split-cost / resident variants; tensor-core
                                     // kernels in `tc`
    int np;                          // run-time user models: reals in the parameter block (P = { real v[np]; })
    int param_bytes;                 // sizeof(Model::P<real>)
    void (*load)(const ModelKernels* self, void* dst, const double* blob, const double* ext, int n_ext);
    const void* fused[3];            // fused_command_kernel<Model, real, V, false, false>, V = MPPI / SMPPI / KMPPI
    const void* split[3];            // ... SPLIT = true (nullptr: not available)
    const void* split_ll[3];         // fused_command_kernel_ll<Model, real, V>: split-cost, single-GPU LL tail (or nullptr)
    const void* batched;             // fused_command_kernel<Model, real, V_MPPI, true>
    const void* resident[3];         // resident_command_kernel<Model, real, V> (nullptr: not available)
    const void* resident_stamped;    // the one instantiation with %globaltimer stamps, or nullptr
    const void* states;              // states_kernel<Model, real>
    const void* gtile[3];            // fused_command_kernel_gtile<Model, real, V, false> (nullptr: not available)
    const void* gtile_batched;       // fused_command_kernel_gtile<Model, real, V_MPPI, true>
    const void* tc[3][2][2];         // mlp_tc_command_kernel<V, SPLIT = 2 - mode, FAST>, [V][mode - 1][fast]; fp32 MLP only
                                     // (the ensemble: mlp_ens_tc_command_kernel)
    void* library;                   // run-time user models: the cudaLibrary_t that owns the kernels
    int copies;                      // run-time user models: the COPIES their kernels were compiled with (0 or 1: none)
    int n_tensors;                   // run-time user models: device tensor views behind the parameters (mppi_model_tensors.h)
    int32_t tensor_dtype[MPPI_MAX_MODEL_TENSORS], tensor_ndim[MPPI_MAX_MODEL_TENSORS];
    const void* plant;               // plant_step_kernel<Model, real>: closed-loop episodes (nullptr: the PendulumMLP models,
                                     // step-dependent user models)
    const void* env_batched;         // fused_command_kernel_env<Model, real, false>: MPPI_Batched with per-environment model
                                     // parameters (nullptr: the PendulumMLP models)
    const void* env_gtile_batched;   // fused_command_kernel_env<Model, real, true>
};
}  // namespace mppi_host

using namespace mppi_host;

namespace {

inline int cuda_fail(cudaError_t e, const char* what) {
    snprintf(g_cuda_err, sizeof(g_cuda_err), "%s: %s (%s)", what, cudaGetErrorName(e), cudaGetErrorString(e));
    return MPPI_ERR_CUDA;
}
inline int unsupported_at(const char* why, const char* file, int line) {
    const char* base = strrchr(file, '/');
    snprintf(g_cuda_err, sizeof(g_cuda_err), "%s (%s:%d)", why, base ? base + 1 : file, line);
    return MPPI_ERR_UNSUPPORTED;
}
#define UNSUPPORTED(why) unsupported_at(why, __FILE__, __LINE__)
#define CK(call)                                              \
    do {                                                      \
        cudaError_t _e = (call);                              \
        if (_e != cudaSuccess) return cuda_fail(_e, #call);   \
    } while (0)

struct DevInfo {
    int sm_count = 0;
    int max_smem_optin = 0;
};
inline int get_dev_info(DevInfo& d) {
    static thread_local int cached_dev = -1;
    static thread_local DevInfo cached;
    int dev = 0;
    CK(cudaGetDevice(&dev));
    if (dev != cached_dev) {
        CK(cudaDeviceGetAttribute(&cached.sm_count, cudaDevAttrMultiProcessorCount, dev));
        CK(cudaDeviceGetAttribute(&cached.max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
        cached_dev = dev;
    }
    d = cached;
    return MPPI_OK;
}

inline int validate(const MppiFusedParams* p, bool fused = false) {
    if (p == nullptr) return MPPI_ERR_BAD_ARG;
    if (p->struct_size != sizeof(MppiFusedParams)) return MPPI_ERR_ABI;
    if (p->K <= 0 || p->T <= 0 || p->nu <= 0 || p->nu > MPPI_MAX_NU || p->nx <= 0) return MPPI_ERR_BAD_ARG;
    if (fused && p->nx > MPPI_MAX_NX) return MPPI_ERR_BAD_ARG;      // state by value; the per-step entry points never touch the state
    if (p->variant < 0 || p->variant > 2) return MPPI_ERR_BAD_ARG;
    if (p->dtype != MPPI_F32 && p->dtype != MPPI_F64) return MPPI_ERR_BAD_ARG;
    if (p->variant == MPPI_VARIANT_KMPPI && (p->S <= 0 || p->W == nullptr || p->theta == nullptr)) return MPPI_ERR_BAD_ARG;
    if (p->variant == MPPI_VARIANT_SMPPI && (p->A == nullptr || p->T < 2)) return MPPI_ERR_BAD_ARG;
    if ((p->flags & MPPI_FLAG_SHIFT) && p->variant == MPPI_VARIANT_KMPPI && p->Wshift == nullptr) return MPPI_ERR_BAD_ARG;
    if (p->lambda_ <= 0.0) return MPPI_ERR_BAD_ARG;
    if (p->world < 0 || p->world > MPPI_MAX_RANKS) return MPPI_ERR_BAD_ARG;
    if (p->u_per_command < 1 || p->u_per_command > p->T) return MPPI_ERR_BAD_ARG;
    return MPPI_OK;
}

inline int rows_of(const MppiFusedParams* p) { return (p->variant == MPPI_VARIANT_KMPPI ? p->S : p->T) * p->nu; }

// MPPI_OK if p->model_tensors match the tensors the model was compiled to read (none for every other model).  No CUDA call.
inline int check_model_tensors(const ModelKernels* mk, const MppiTensorRef* refs, int n) {
    return mppi_tensors::check_refs(mk->tensor_dtype, mk->tensor_ndim, mk->n_tensors, refs, n);
}

// The tensor views of a user model's block (checked references: check_model_tensors).
inline void load_model_tensors(const ModelKernels* mk, const MppiTensorRef* refs, void* dst) {
    if (mk->n_tensors > 0) mppi_tensors::pack_views(dst, mk->np, mk->is_double ? 8 : 4, refs, mk->n_tensors);
}

// The model's parameter block for these parameters (the packer of its unit).  The ensemble's block also carries the
// device weight table and the copy count, which are not doubles of model_params; a user model's, its tensor views.
inline void load_model_params(const ModelKernels* mk, const MppiFusedParams* p, void* dst) {
    mk->load(mk, dst, p->model_params, p->model_params_ext, p->n_model_params_ext);
    load_model_tensors(mk, p->model_tensors, dst);
    if (p->model == MPPI_MODEL_PENDULUM_MLP_ENSEMBLE) {
        if (mk->is_double) PendulumMLPEnsembleModel::bind<double>(*reinterpret_cast<PendulumMLPEnsembleModel::P<double>*>(dst), p->model_weights, p->rollout_samples);
        else PendulumMLPEnsembleModel::bind<float>(*reinterpret_cast<PendulumMLPEnsembleModel::P<float>*>(dst), p->model_weights, p->rollout_samples);
    }
}

template <typename real> void fill_noise_model(const MppiFusedParams* p, NoiseModel<real>& nm) {
    for (int i = 0; i < MPPI_MAX_NU; ++i) {
        nm.mu[i] = (real)p->noise_mu[i];
        nm.u_min[i] = (real)p->u_min[i];
        nm.u_max[i] = (real)p->u_max[i];
        nm.a_min[i] = (real)p->action_min[i];
        nm.a_max[i] = (real)p->action_max[i];
    }
    for (int i = 0; i < MPPI_MAX_NU * MPPI_MAX_NU; ++i) {
        nm.L[i] = (real)p->chol[i];
        nm.Sinv[i] = (real)p->sigma_inv[i];
    }
    nm.lambda_ = (real)p->lambda_;
    nm.neg_inv_lambda = (real)(-(1.0 / p->lambda_));   // mppi.py:256: -factor * (cost - beta), factor = 1/lambda
    nm.u_scale = (real)p->u_scale;
    nm.w_smooth = (real)p->w_action_seq_cost;
    nm.delta_t = (real)p->delta_t;
    nm.diag = (p->flags & MPPI_FLAG_DIAG_SIGMA) ? 1 : 0;
    nm.abs_cost = (p->flags & MPPI_FLAG_ABS_COST) ? 1 : 0;
}

// ticket + the records of the warp-fold tail's ticket mode: one of (R + 2) doubles per cluster (at most one per CTA)
// ... followed by this GPU's own record mailbox (single-GPU LL mode): two epoch parities of MPPI_LL_LOCAL_WORDS flagged words
// (MPPI_LL_STAGE_BYTES / MPPI_LL_LOCAL_WORDS: mppi_fused.cuh)
// ... followed, for the global-tile kernels, by one tile slice per CTA (gtile_slice_bytes; ws_gtile_bytes below)
// Every environment's workspace of a batched plan (env_ws_stride apart) starts MPPI_WS_ALIGN-aligned, so its ticket, records
// (doubles), mailbox words and tile slices are aligned as environment 0's are.
#define MPPI_WS_ALIGN 256
inline uint64_t ws_partials_bytes(int nb, int R) { return (16 + (uint64_t)nb * (uint64_t)(R + 2) * 8 + 255) / 256 * 256; }
inline uint64_t ws_bytes(int nb, int R) { return ws_partials_bytes(nb, R) + 2ull * MPPI_LL_LOCAL_WORDS * 8; }

#define MPPI_MAX_CTAS_PER_SM 16                            // plan_geometry's grid cap
// The largest grid any kernel of these dimensions can be planned with, on any route: tiles hold at least 32 samples, the
// planner caps grids at MPPI_MAX_CTAS_PER_SM CTAs per SM, and the fused command pads its grid to a multiple of its
// cluster size (8 at most).  A workspace of ws_bytes of this grid (MppiLaunchInfo.workspace_bytes) serves every geometry.
inline int max_planned_grid(const MppiFusedParams* p, int sm_count) {
    const long long K = p->K_geom > p->K ? p->K_geom : p->K;
    const long long tiles = (K + 31) / 32, cap = (long long)sm_count * MPPI_MAX_CTAS_PER_SM;
    const long long nb = tiles < cap ? tiles : cap;
    return (int)((nb + 7) / 8 * 8);
}

// Global-tile plans: the samples whose tiles are in flight at once (grid x samples per tile) are capped at
// MPPI_GTILE_SAMPLES_PER_SM per SM, so the tile slices stay bounded at large K (a grid-stride CTA reuses its slice).
#define MPPI_GTILE_SAMPLES_PER_SM 128
inline int gtile_grid_cap(int sm_count, int BS) {
    const int nb = sm_count * MPPI_GTILE_SAMPLES_PER_SM / BS;
    return nb > 1 ? nb : 1;
}
// The tile slices of any global-tile plan of these dimensions (per environment): at most min(K + 511, cap) samples in
// flight, one slice per CTA of at least 32 samples.  rows2 (T*nu per sample) only where a kernel of the variant has it:
// SMPPI (fused) and KMPPI (fused and sampling); MPPI's slices hold `rows` alone.  A multiple of MPPI_WS_ALIGN, as ws_bytes
// is: the workspace of a batched plan's environment e starts e x (ws_bytes + ws_gtile_bytes) bytes in (env_ws_stride).
inline uint64_t ws_gtile_bytes(const MppiFusedParams* p, int sm_count) {
    const long long K = p->K_geom > p->K ? p->K_geom : p->K;
    long long n = (long long)sm_count * MPPI_GTILE_SAMPLES_PER_SM;
    if (K + 511 < n) n = K + 511;
    const int es = p->dtype == MPPI_F64 ? 8 : 4;
    const long long per_sample = rows_of(p) + (p->variant != MPPI_VARIANT_MPPI ? (long long)p->T * p->nu : 0);
    const uint64_t bytes = (uint64_t)n * (uint64_t)per_sample * es + (uint64_t)(n / 32 + 1) * 256;
    return (bytes + MPPI_WS_ALIGN - 1) / MPPI_WS_ALIGN * MPPI_WS_ALIGN;
}
// ... and the slices of a planned grid
inline uint64_t ws_gtile_plan_bytes(const MppiFusedParams* p, int nb, int BS, int rows2) {
    return (uint64_t)nb * (uint64_t)gtile_slice_bytes(rows_of(p), p->T * p->nu, rows2, BS, p->dtype == MPPI_F64 ? 8 : 4);
}

inline unsigned long long xchg_timeout_ns() {
    // how long a shard waits for its peers' records before giving up (rank skew: a GC pause, a JIT build, a lazy module
    // load on another rank); MPPI_B200_XCHG_TIMEOUT_S overrides the 20 s default
    const char* e = getenv("MPPI_B200_XCHG_TIMEOUT_S");
    double sec = (e != nullptr && atof(e) > 0) ? atof(e) : 20.0;
    return (unsigned long long)(sec * 1e9);
}

template <typename real> int fill_kargs(const MppiFusedParams* p, KArgs<real>& a, int BS, int nb, int tps = 1) {
    memset(&a, 0, sizeof(a));
    fill_noise_model<real>(p, a.nm);
    for (int i = 0; i < MPPI_MAX_NU; ++i) a.u_init[i] = (real)p->u_init[i];
    for (int i = 0; i < MPPI_MAX_NX; ++i) a.x0[i] = (real)p->state[i];
    a.state_dev = (p->flags & MPPI_FLAG_STATE_DEVICE) ? (const real*)p->state_dev : nullptr;
    a.state_per_sample = (p->flags & MPPI_FLAG_STATE_PER_SAMPLE) ? 1 : 0;
    a.U = (real*)p->U;
    a.A = (real*)p->A;
    a.theta = (real*)p->theta;
    a.W = (const real*)p->W;
    a.Wshift = (const real*)p->Wshift;
    a.cost_total = (real*)p->cost_total;
    a.action_out = (real*)p->action_out;
    a.nominal_used = (real*)p->nominal_used;
    a.stats = (double*)p->stats;
    a.z = (const real*)p->z;
    a.z_out = (real*)p->z_out;
    a.K = p->K;
    a.T = p->T;
    a.S = p->S;
    a.R = rows_of(p);
    a.TN = p->T * p->nu;
    a.upc = p->u_per_command;
    a.n_tiles = (p->K + BS - 1) / BS;
    a.tps = tps;
    a.k_offset = p->k_offset;
    a.seed = p->seed;
    a.offset = p->offset;
    a.shift = (p->flags & MPPI_FLAG_SHIFT) ? 1 : 0;
    a.null_action = (p->flags & MPPI_FLAG_NULL_ACTION) ? 1 : 0;
    a.pdl = (p->flags & MPPI_FLAG_PDL) ? 1 : 0;
    const int es = (int)sizeof(real);
    const bool padded = (p->flags & MPPI_FLAG_NOMINAL_PADDED) || ((a.TN * es) % 16 == 0);
    a.tma_ok = padded && ((uintptr_t)p->U % 16 == 0) && (p->variant != MPPI_VARIANT_SMPPI || (uintptr_t)p->A % 16 == 0);
    // workspace carve
    if (p->workspace != nullptr) {
        unsigned char* w = (unsigned char*)p->workspace;
        a.ticket = (unsigned int*)w;
        a.crec = (double*)(w + 16);
    }
    a.xchg_npub = 1;
    a.xchg_parity_words = MPPI_XCHG_PARITY_WORDS;
    a.xchg_timeout_ns = xchg_timeout_ns();
    a.xchg_status_host = (long long*)p->xchg_status_host;
    a.rank = p->rank;
    a.world = p->world <= 0 ? 1 : p->world;
    a.epoch = p->epoch;
    a.export_partial = (p->flags & MPPI_FLAG_EXPORT_PARTIAL) ? 1 : 0;
    a.partial_out = (double*)p->partial_out;
    a.torch_total = p->torch_rng_total;
    a.offset_dev = (unsigned long long*)p->offset_dev;
    a.offset_inc = p->offset_inc;
    a.n_env = p->n_env > 1 ? p->n_env : 1;
    a.env_u_stride = p->env_u_stride;
    a.env_ws_stride = (long long)p->env_ws_stride;
    a.dbg = (unsigned long long*)p->debug_clocks;
    a.host_mailbox = (unsigned long long*)p->host_mailbox;
    a.host_epoch = p->host_epoch;
    bool any_peer = false;
    for (int g = 0; g < MPPI_MAX_RANKS; ++g) {
        a.peers[g] = (unsigned long long*)p->peer_slots[g];
        any_peer = any_peer || p->peer_slots[g] != nullptr;
    }
    if (p->rollout_samples > 1) {
        a.var_disc = (const real*)p->var_discount;
        a.var_cost = (real)p->rollout_var_cost;
    }
    if (!any_peer || a.export_partial) a.world = a.export_partial ? a.world : 1;
    if (p->workspace != nullptr && (a.world == 1 || a.export_partial)) {
        // not sharded in-kernel: the record mailbox is this GPU's own, behind the partials in the workspace
        a.peers[0] = (unsigned long long*)((unsigned char*)p->workspace + ws_partials_bytes(nb, a.R));
        a.xchg_parity_words = MPPI_LL_LOCAL_WORDS;
    }
    return MPPI_OK;
}

// launch configuration with the optional attributes: programmatic dependent launch, thread-block clusters (cluster, 1, 1)
inline void launch_config(cudaLaunchConfig_t& cfg, cudaLaunchAttribute* at, int nb, int BD, int smem, cudaStream_t stream, bool pdl,
                          int ny, int cluster) {
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(nb, ny);
    cfg.blockDim = dim3(BD);
    cfg.dynamicSmemBytes = (size_t)smem;
    cfg.stream = stream;
    int n = 0;
    if (pdl) {
        at[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[n].val.programmaticStreamSerializationAllowed = 1;
        ++n;
    }
    if (cluster > 1) {
        at[n].id = cudaLaunchAttributeClusterDimension;
        at[n].val.clusterDim.x = (unsigned)cluster;
        at[n].val.clusterDim.y = 1;
        at[n].val.clusterDim.z = 1;
        ++n;
    }
    cfg.attrs = at;
    cfg.numAttrs = n;
}

inline cudaError_t launch_raw(const void* kernel, int nb, int BD, int smem, cudaStream_t stream, void** argv, bool pdl, int ny = 1,
                              int cluster = 1) {
    if (!pdl && cluster <= 1) return cudaLaunchKernel(kernel, dim3(nb, ny), dim3(BD), argv, (size_t)smem, stream);
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute at[3];
    launch_config(cfg, at, nb, BD, smem, stream, pdl, ny, cluster);
    return cudaLaunchKernelExC(&cfg, kernel, argv);
}

template <typename... Args>
int launch_kernel(void (*kernel)(Args...), int nb, int BD, int smem, cudaStream_t stream, int ny, Args... args) {
    void* argv[] = {(void*)&args...};
    cudaError_t e = cudaLaunchKernel((const void*)kernel, dim3(nb, ny), dim3(BD), argv, (size_t)smem, stream);
    if (e != cudaSuccess) {
        snprintf(g_cuda_err, sizeof(g_cuda_err), "launch grid=%d block=%d smem=%d: %s (%s)", nb, BD, smem,
                 cudaGetErrorName(e), cudaGetErrorString(e));
        return MPPI_ERR_CUDA;
    }
    return MPPI_OK;
}

// LL mode identifies a command's records by its epoch tag: a launch captured into a CUDA graph would replay one tag.
inline int refuse_capture(cudaStream_t stream, const Geometry& g) {
    if (g.npub <= 1) return MPPI_OK;
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(stream, &st) == cudaSuccess && st != cudaStreamCaptureStatusNone)
        return UNSUPPORTED("the fused command cannot be captured into a CUDA graph (its reduction records carry a per-command tag); "
                           "launch it directly — it is one kernel — or set MPPI_B200_XCHG_DIRECT=0");
    return MPPI_OK;
}

struct GeomKey {
    const void* kernel;
    int dev, variant, K, T, nu, S, bt, tp, gb, r2, grid_recs, ne, xb;
    bool operator==(const GeomKey& o) const {
        return kernel == o.kernel && dev == o.dev && variant == o.variant && K == o.K && T == o.T && nu == o.nu && S == o.S &&
               bt == o.bt && tp == o.tp && gb == o.gb && r2 == o.r2 && grid_recs == o.grid_recs && ne == o.ne && xb == o.xb;
    }
};

// Launch geometry for (kernel, dimensions).  The occupancy / attribute queries cost microseconds, so
// the last few results are cached per thread: a steady-state command() pays only the lookup.
// grid_records: the kernel's finisher rescales one record per CTA of the grid (the warp-fold tail in ticket mode without
// clusters: softmin_update_kernel), so the layout grows with the grid; the fused routes size their final layout themselves.
// extra_bytes: dynamic shared memory the kernel uses behind the layout (the ensemble wgmma kernel's per-copy tiles).
// gtile: a global-tile kernel (layout without the tiles, grid capped by gtile_grid_cap)
template <typename real, typename KernelT>
int plan_geometry(KernelT kernel, const MppiFusedParams* p, int need_rows2, bool grid_records, Geometry& g,
                  int extra_bytes = 0, bool gtile = false) {
    static thread_local GeomKey keys[8];
    static thread_local Geometry vals[8];
    static thread_local int n_cached = 0, next_slot = 0;
    int dev = 0;
    CK(cudaGetDevice(&dev));
    const GeomKey key{(const void*)kernel, dev, p->variant, p->K, p->T, p->nu, p->S, p->block_threads, p->threads_per_sample,
                      p->grid_blocks, need_rows2, grid_records ? 1 : 0, p->n_env > 1 ? p->n_env : 1, extra_bytes};
    for (int i = 0; i < n_cached; ++i)
        if (keys[i] == key) {
            g = vals[i];
            return MPPI_OK;
        }
    DevInfo di;
    int rc = get_dev_info(di);
    if (rc) return rc;
    const int R = rows_of(p);
    // BS samples per tile; tps threads share one sample's sampling/transform work.
    //
    // Automatic geometry (block_threads == 0): blocks are statically assigned tiles (determinism:
    // the reduction order must not depend on scheduling), so the finish time follows the most
    // loaded SM.  Enumerate BS in steps of a warp and j = resident CTAs per SM, size the grid as
    // min(n_tiles, SMs*j), and keep the candidate with the smallest worst-case samples per SM
    // (ties: fewer passes, then more threads).
    int BS = p->block_threads;
    int tps = p->threads_per_sample;
    int grid_hint = 0;
    if (BS <= 0) {
        cudaFuncAttributes fa0;
        CK(cudaFuncGetAttributes(&fa0, kernel));
        const int dyn0 = di.max_smem_optin - (int)fa0.sharedSizeBytes;
        CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn0));
        long long best_load = -1;
        int best_bs = 128, best_passes = 0, best_grid = 0;
        // latency hiding needs ~24 resident warps per SM when the problem is large enough to supply them
        const long long per_sm = ((long long)p->K + di.sm_count - 1) / di.sm_count;
        const long long want_threads = per_sm < 768 ? per_sm : 768;
        // 64-sample tiles let K < 128 x SMs reach every SM; 32-sample tiles are tried only when no larger tile fits in
        // shared memory (the R x (BS+1) noise tile of long horizons at nu = 3..4), so no geometry that fits changes
        auto next_bs = [&](int bs) { return bs == 32 ? 0 : bs < 512 ? bs + (bs < 128 ? 64 : 32) : (best_load < 0 ? 32 : 0); };
        for (int bs = 64; bs != 0; bs = next_bs(bs)) {
            SmemLayout Lc = make_layout<real>(p->variant, p->T, p->nu, p->S, R, bs, bs, grid_records ? di.sm_count * 4 : 1, need_rows2, gtile);
            Lc.total += extra_bytes;
            if (Lc.total > dyn0) continue;
            int occ_c = 0;
            CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_c, kernel, bs, Lc.total));
            if (occ_c < 1) continue;
            const int nt = (p->K + bs - 1) / bs;
            for (int j = 1; j <= occ_c && j <= 8; ++j) {
                int nbc = nt < di.sm_count * j ? nt : di.sm_count * j;
                if (gtile && nbc > gtile_grid_cap(di.sm_count, bs)) nbc = gtile_grid_cap(di.sm_count, bs);   // as below
                const int passes = (nt + nbc - 1) / nbc;
                const int bps = (nbc + di.sm_count - 1) / di.sm_count;
                long long load = (long long)bps * passes * bs;
                const long long resident = (long long)bps * bs;
                if (resident < want_threads) load = load * want_threads / resident;   // under-occupied: proportionally slower
                const bool better = best_load < 0 || load < best_load ||
                                    (load == best_load && (passes < best_passes || (passes == best_passes && bs > best_bs)));
                if (better) {
                    best_load = load;
                    best_bs = bs;
                    best_passes = passes;
                    best_grid = nbc;
                }
            }
        }
        BS = best_bs;
        grid_hint = best_grid;
    }
    if (BS % 32 != 0 || BS < 32 || BS > 512) return MPPI_ERR_BAD_ARG;
    const int n_tiles = (p->K + BS - 1) / BS;
    int cap = di.sm_count * MPPI_MAX_CTAS_PER_SM;     // workspaces are sized for it: max_planned_grid
    cudaFuncAttributes fa;
    CK(cudaFuncGetAttributes(&fa, kernel));
    const int dyn_limit = di.max_smem_optin - (int)fa.sharedSizeBytes;   // static + dynamic <= opt-in maximum
    // The layout may depend on the grid (grid_records: one rescale factor per CTA in shared memory) and the
    // grid on the occupancy the layout allows: iterate from an optimistic guess to a fixed point.
    if (gtile && gtile_grid_cap(di.sm_count, BS) < cap) cap = gtile_grid_cap(di.sm_count, BS);
    int nb = n_tiles < cap ? n_tiles : cap;
    if (tps <= 0) {
        // helper threads only pay off while an SM hosts a single small CTA
        tps = 1;
        const int envs = p->n_env > 1 ? p->n_env : 1;
        if ((long long)n_tiles * envs <= di.sm_count) tps = 512 / BS >= 8 ? 8 : (512 / BS >= 4 ? 4 : (512 / BS >= 2 ? 2 : 1));
        // each helper thread's warp adds per-warp partial rows to the tile: fewer helpers where all of them do not fit
        // (the optimistic grid's layout is the largest of the fixed-point iteration below)
        while (tps > 1 && BS * tps > 64 && make_layout<real>(p->variant, p->T, p->nu, p->S, R, BS * tps, BS,
                                                             grid_records ? nb : 1, need_rows2, gtile).total + extra_bytes > dyn_limit)
            tps >>= 1;
    }
    while (tps > 1 && BS * tps > 512) tps >>= 1;
    // at least two warps per CTA: the fused command's record combines (combine_records / combine_global) split the
    // threads into groups of 64 columns, and a one-warp CTA would have none (32-sample tiles run two threads per sample)
    if (BS * tps < 64) tps = 64 / BS;
    if (tps != 1 && tps != 2 && tps != 4 && tps != 8) return MPPI_ERR_BAD_ARG;
    const int BD = BS * tps;
    // The attribute is a per-kernel LIMIT (setting a smaller value later lowers it), so raise it
    // once to the device maximum; the carve-out actually used follows each launch's request.
    CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn_limit));
    int occ = 0;
    SmemLayout L;
    for (int it = 0; it < 4; ++it) {
        L = make_layout<real>(p->variant, p->T, p->nu, p->S, R, BD, BS, grid_records ? nb : 1, need_rows2, gtile);
        L.total += extra_bytes;
        if (L.total > dyn_limit)
            return gtile ? UNSUPPORTED("global-tile plan: the per-CTA vectors (nominal sequence, softmin records) do not fit in shared memory")
                         : UNSUPPORTED("shared-memory tile does not fit");
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, BD, L.total));
        if (occ < 1) return UNSUPPORTED("kernel does not fit on an SM with this block size");
        int nb2 = n_tiles < di.sm_count * occ ? n_tiles : di.sm_count * occ;
        if (nb2 > cap) nb2 = cap;
        if (p->grid_blocks > 0 && p->grid_blocks < nb2) nb2 = p->grid_blocks;
        if (grid_hint > 0 && grid_hint < nb2) nb2 = grid_hint;
        if (nb2 == nb) break;
        nb = nb2;
    }
    L = make_layout<real>(p->variant, p->T, p->nu, p->S, R, BD, BS, grid_records ? nb : 1, need_rows2, gtile);
    L.total += extra_bytes;
    g.BS = BS;
    g.tps = tps;
    g.BD = BD;
    g.nb = nb;
    g.smem = L.total;
    g.occ = occ;
    g.regs = fa.numRegs;
    g.cluster = 1;
    g.npub = 0;
    keys[next_slot] = key;
    vals[next_slot] = g;
    next_slot = (next_slot + 1) % 8;
    if (n_cached < 8) ++n_cached;
    return MPPI_OK;
}

}  // namespace

