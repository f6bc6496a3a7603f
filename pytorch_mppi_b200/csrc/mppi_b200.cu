// mppi_b200.cu — C-ABI entry points (include/mppi_b200.h) and kernel dispatch.
// Built with: nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -shared -Xcompiler -fPIC
// No torch types cross this boundary; the Python side binds it with ctypes.
//
// Translation units of the library (built in parallel by pytorch_mppi_b200/build.py):
//   mppi_b200.cu        this file: the C ABI, the model-independent kernels (sampling, softmin update, cost
//                       accumulation, omega, apply-partials), plan commands, resident-mode backend, peer mailboxes
//   mppi_model_tu.cu    compiled once per (registered model, dtype): fused / resident / states kernels of that model
#include "mppi_fused_host.cuh"

namespace mppi_host {
thread_local char g_cuda_err[512] = "";

// one getter per (model, dtype) translation unit (mppi_model_tu.cu)
const ModelKernels* model_kernels_pendulum_f32();
const ModelKernels* model_kernels_pendulum_f64();
const ModelKernels* model_kernels_linear_point_f32();
const ModelKernels* model_kernels_linear_point_f64();
const ModelKernels* model_kernels_pendulum_mlp_f32();
const ModelKernels* model_kernels_pendulum_mlp_f64();
const ModelKernels* model_kernels_pendulum_mlp_ensemble_f32();
const ModelKernels* model_kernels_pendulum_mlp_ensemble_f64();
}  // namespace mppi_host

namespace {

// a user model compiled at run time (mppi_user_model_register): its descriptor travels in MppiFusedParams.user_model
struct UserModelHandle {
    uint32_t magic;
    ModelKernels mk;
};
constexpr uint32_t kUserMagic = 0x4d505049u;   // "MPPI"

// the (model, dtype) descriptor that serves these parameters, or nullptr
const ModelKernels* find_kernels(const MppiFusedParams* p, int* rc) {
    *rc = MPPI_ERR_UNSUPPORTED;
    const bool f32 = p->dtype == MPPI_F32;
    typedef const ModelKernels* (*Getter)();
    Getter get = nullptr;
    switch (p->model) {
        case MPPI_MODEL_PENDULUM: get = f32 ? model_kernels_pendulum_f32 : model_kernels_pendulum_f64; break;
        case MPPI_MODEL_LINEAR_POINT: get = f32 ? model_kernels_linear_point_f32 : model_kernels_linear_point_f64; break;
        case MPPI_MODEL_PENDULUM_MLP:
            if (p->n_model_params_ext < PendulumMLPModel::N_EXT || p->model_params_ext == nullptr) {
                *rc = MPPI_ERR_BAD_ARG;
                return nullptr;
            }
            get = f32 ? model_kernels_pendulum_mlp_f32 : model_kernels_pendulum_mlp_f64;
            break;
        case MPPI_MODEL_PENDULUM_MLP_ENSEMBLE:
            if (p->model_weights == nullptr) {
                *rc = MPPI_ERR_BAD_ARG;
                return nullptr;
            }
            get = f32 ? model_kernels_pendulum_mlp_ensemble_f32 : model_kernels_pendulum_mlp_ensemble_f64;
            break;
        case MPPI_MODEL_USER: {
            const UserModelHandle* h = reinterpret_cast<const UserModelHandle*>(p->user_model);
            if (h == nullptr || h->magic != kUserMagic || h->mk.is_double != (f32 ? 0 : 1)) {
                *rc = MPPI_ERR_BAD_ARG;
                return nullptr;
            }
            return &h->mk;
        }
    }
    return get != nullptr ? get() : nullptr;
}

// rollout_samples M > 1 (mppi.py:334-373) on the fused route: only a user model compiled with M copies, or the ensemble
// of M networks, makes its copies differ (another registered model's M rollouts would be identical).  No CUDA call.
int check_rollout_samples(const MppiFusedParams* p, const ModelKernels* mk) {
    if (p->rollout_samples < 0) return MPPI_ERR_BAD_ARG;
    const int M = p->rollout_samples > 1 ? p->rollout_samples : 1;
    if (p->model == MPPI_MODEL_PENDULUM_MLP_ENSEMBLE)
        return M >= 2 && M <= MPPI_MAX_COPIES && p->var_discount != nullptr ? MPPI_OK : MPPI_ERR_BAD_ARG;
    if (M > 1 && p->model != MPPI_MODEL_USER)
        return UNSUPPORTED("rollout_samples > 1 on the fused route needs a user model compiled with that many copies");
    const int copies = mk->copies > 1 ? mk->copies : 1;
    if (M != copies || (M > 1 && p->var_discount == nullptr)) return MPPI_ERR_BAD_ARG;
    return MPPI_OK;
}

// the checks every route that packs the model's parameter block makes first: rollout copies and tensors.  No CUDA call.
int check_model_args(const MppiFusedParams* p, const ModelKernels* mk) {
    const int rc = check_rollout_samples(p, mk);
    return rc ? rc : check_model_tensors(mk, p->model_tensors, p->n_model_tensors);
}

template <typename real>
inline void plan_update(Plan* pl, const double* state, const void* state_dev, uint32_t flags, uint64_t seed, uint64_t offset,
                        const void* z, void* action_out, void* host_mailbox) {
    KArgs<real>* a = reinterpret_cast<KArgs<real>*>(pl->kargs);
    if (state != nullptr)
        for (int i = 0; i < pl->nx; ++i) a->x0[i] = (real)state[i];
    a->state_dev = (flags & MPPI_FLAG_STATE_DEVICE) ? (const real*)state_dev : nullptr;
    a->state_per_sample = (flags & MPPI_FLAG_STATE_PER_SAMPLE) ? 1 : 0;
    a->shift = (flags & MPPI_FLAG_SHIFT) ? 1 : 0;
    a->seed = seed;
    a->offset = offset;
    a->z = (const real*)z;
    a->action_out = (real*)action_out;
    // one epoch per command on whichever route it takes: the tag of its reduction records (and, sharded, of the exchange)
    if (pl->res.armed && pl->res_epoch_off + pl->res.seq > pl->epoch) pl->epoch = pl->res_epoch_off + pl->res.seq;
    a->epoch = ++pl->epoch;
    a->host_mailbox = (unsigned long long*)host_mailbox;
    if (host_mailbox != nullptr) a->host_epoch = ++pl->host_epoch;
}

inline int plan_launch(Plan* pl, cudaStream_t stream) {
    int rc = refuse_capture(stream, pl->g);
    if (rc) return rc;
    void* argv[3] = {(void*)pl->kargs, (void*)pl->mparams, nullptr};
    const void* kernel = pl->kernel;
    if (pl->env_kernel != nullptr) {      // per-environment parameter blocks in place of the plan's one
        kernel = pl->env_kernel;
        argv[1] = (void*)&pl->env_mp;
        argv[2] = (void*)&pl->env_stride;
    }
    cudaError_t e = launch_raw(kernel, pl->g.nb, pl->g.BD, pl->g.smem, stream, argv, pl->pdl != 0, pl->p.n_env > 1 ? pl->p.n_env : 1,
                               pl->g.cluster);
    if (e != cudaSuccess) {
        snprintf(g_cuda_err, sizeof(g_cuda_err), "plan launch grid=%d block=%d smem=%d cluster=%d: %s (%s)", pl->g.nb, pl->g.BD, pl->g.smem, pl->g.cluster,
                 cudaGetErrorName(e), cudaGetErrorString(e));
        return MPPI_ERR_CUDA;
    }
    return MPPI_OK;
}

// one command on a plan: the per-command checks, the argument update and the launch
int plan_command(Plan* pl, const double* state, const void* state_dev, uint32_t flags, uint64_t seed, uint64_t offset, const void* z,
                 void* action_out, void* host_mailbox, cudaStream_t stream) {
    if (pl == nullptr || action_out == nullptr) return MPPI_ERR_BAD_ARG;
    if (state == nullptr && !(flags & MPPI_FLAG_STATE_DEVICE)) return MPPI_ERR_BAD_ARG;
    if (pl->p.n_env > 1 && !(flags & MPPI_FLAG_STATE_DEVICE)) return MPPI_ERR_BAD_ARG;   // states are (n_env, nx) on the device
    if (pl->is_double) plan_update<double>(pl, state, state_dev, flags, seed, offset, z, action_out, host_mailbox);
    else plan_update<float>(pl, state, state_dev, flags, seed, offset, z, action_out, host_mailbox);
    return plan_launch(pl, stream);
}

// ---- closed-loop episodes (mppi_plan_closed_loop, mppi_plan_closed_loop_plant) ------------------------------
// one packed parameter block in the plant scratch: the model's block rounded up to 16 bytes (alignment of every block)
inline uint64_t plant_block_bytes(const ModelKernels* mk) { return ((uint64_t)mk->param_bytes + 15) / 16 * 16; }

// n rows of n_params doubles in the model's own layout (the first MPPI_MODEL_PARAM_DOUBLES are its model_params,
// zero-padded, the rest its model_params_ext), packed with the model's loader into n blocks plant_block_bytes apart;
// everything else a block holds (a user model's tensor views, the ensemble's weight table) comes from `p`
void pack_param_rows(const ModelKernels* mk, const MppiFusedParams* p, const double* rows, int n, int n_params, unsigned char* dst) {
    MppiFusedParams pp = *p;
    const uint64_t bb = plant_block_bytes(mk);
    for (int i = 0; i < n; ++i) {
        const double* row = rows + (size_t)i * n_params;
        for (int j = 0; j < MPPI_MODEL_PARAM_DOUBLES; ++j) pp.model_params[j] = j < n_params ? row[j] : 0.0;
        pp.model_params_ext = n_params > MPPI_MODEL_PARAM_DOUBLES ? row + MPPI_MODEL_PARAM_DOUBLES : nullptr;
        pp.n_model_params_ext = n_params > MPPI_MODEL_PARAM_DOUBLES ? n_params - MPPI_MODEL_PARAM_DOUBLES : 0;
        load_model_params(mk, &pp, dst + (size_t)i * bb);
    }
}

// The plant of a closed loop: its kernels and the parameters its blocks are packed from.  Without a plant descriptor,
// the plan's model and parameters; with one, the plan's parameters with the plant's model, handle and tensors in place
// of the plan's (find_kernels then picks the plant's kernels of the plan's dtype).  No CUDA call.
struct PlantOf {
    const ModelKernels* mk;
    MppiFusedParams p;
};
int resolve_plant(const Plan* pl, const MppiPlantModel* pm, PlantOf* out) {
    if (pm != nullptr) {      // what can be checked without the plan
        if (pm->struct_size != sizeof(MppiPlantModel)) return MPPI_ERR_ABI;
        if (pm->reserved != 0 || pm->n_model_tensors < 0) return MPPI_ERR_BAD_ARG;
        if (pm->model == MPPI_MODEL_PENDULUM_MLP || pm->model == MPPI_MODEL_PENDULUM_MLP_ENSEMBLE)
            return UNSUPPORTED("closed loop: a PendulumMLP model is learned, not a plant (it has no plant step)");
        if (pm->model != MPPI_MODEL_PENDULUM && pm->model != MPPI_MODEL_LINEAR_POINT && pm->model != MPPI_MODEL_USER)
            return MPPI_ERR_BAD_ARG;
        if (pm->model == MPPI_MODEL_USER &&
            (pm->user_model == nullptr || reinterpret_cast<const UserModelHandle*>(pm->user_model)->magic != kUserMagic))
            return MPPI_ERR_BAD_ARG;
    }
    if (pl == nullptr) return MPPI_ERR_BAD_ARG;
    out->mk = pl->mk;
    out->p = pl->p;
    if (pm == nullptr) return MPPI_OK;
    MppiFusedParams& pp = out->p;
    pp.model = pm->model;
    pp.user_model = pm->model == MPPI_MODEL_USER ? const_cast<void*>(pm->user_model) : nullptr;
    pp.model_tensors = pm->model_tensors;
    pp.n_model_tensors = pm->n_model_tensors;
    pp.model_params_ext = nullptr;
    pp.n_model_params_ext = 0;
    pp.model_weights = nullptr;
    pp.rollout_samples = 0;
    int rc = MPPI_OK;
    out->mk = find_kernels(&pp, &rc);
    if (out->mk == nullptr) return rc;
    if (out->mk->nx != pl->nx || out->mk->nu != pl->p.nu) return MPPI_ERR_BAD_ARG;
    if (out->mk->plant == nullptr)
        return UNSUPPORTED("closed loop: the plant has no plant step (a step-dependent user model: a closed loop has no horizon index)");
    return check_model_tensors(out->mk, pm->model_tensors, pm->n_model_tensors);
}

// the reasons a closed loop is refused, before any CUDA call (MPPI_OK: none); `plant` resolved by resolve_plant
int check_closed_loop(const Plan* pl, const MppiClosedLoop* cl, const PlantOf& plant, bool own_plant) {
    if (pl == nullptr || cl == nullptr) return MPPI_ERR_BAD_ARG;
    if (cl->struct_size != sizeof(MppiClosedLoop)) return MPPI_ERR_ABI;
    const int n_env = pl->p.n_env > 1 ? pl->p.n_env : 1;
    if (cl->steps < 1 || cl->states == nullptr || cl->actions == nullptr || cl->plant_blocks == nullptr) return MPPI_ERR_BAD_ARG;
    if ((uintptr_t)cl->plant_blocks % 16 != 0 || cl->n_plant_params < 0) return MPPI_ERR_BAD_ARG;
    if (cl->n_plant != 1 && cl->n_plant != n_env) return MPPI_ERR_BAD_ARG;
    if (cl->plant_params == nullptr && (cl->n_plant != 1 || own_plant)) return MPPI_ERR_BAD_ARG;
    if (plant.mk->plant == nullptr)
        return UNSUPPORTED("closed loop: this model has no plant step (the PendulumMLP models, step-dependent user models): "
                           "name the plant apart (mppi_plan_closed_loop_plant)");
    if (pl->p.u_per_command != 1) return UNSUPPORTED("closed loop: u_per_command must be 1 (the plant applies one action per command)");
    if (pl->p.world > 1 || (pl->p.flags & MPPI_FLAG_EXPORT_PARTIAL)) return UNSUPPORTED("closed loop: not available on sharded controllers");
    if (pl->p.z_out != nullptr) return UNSUPPORTED("closed loop: the plan records the noise it draws (z_out)");
    if (pl->p.offset_dev != nullptr) return UNSUPPORTED("closed loop: the plan reads its Philox counter from the device (offset_dev)");
    if (pl->res.armed) return UNSUPPORTED("closed loop: a resident grid is armed on this plan (mppi_resident_stop first)");
    return MPPI_OK;
}

// A plant named apart from the plan's model always comes with plant_params (check_closed_loop): the plan's own block and
// its per-environment blocks serve only the plan's model.
template <typename real>
int closed_loop_t(Plan* pl, const MppiClosedLoop* cl, const PlantOf& plant, cudaStream_t stream) {
    const ModelKernels* mk = plant.mk;
    const int n_env = pl->p.n_env > 1 ? pl->p.n_env : 1;
    const int nx = mk->nx, nu = mk->nu;
    const uint64_t bb = plant_block_bytes(mk);
    PlantStepArgs<real> ps;
    ps.plants = (const unsigned char*)cl->plant_blocks;
    ps.plant_stride = (long long)bb;
    ps.n_env = n_env;
    ps.n_plant = cl->n_plant;
    if (cl->plant_params == nullptr && pl->env_kernel != nullptr) {
        // per-environment model parameters: environment e's plant is its own model, the blocks its commands read
        ps.plants = pl->env_mp;
        ps.n_plant = n_env;
    } else {
        // the plant blocks, packed once per call with the plant's loader (a user model's views: the plant's tensors —
        // the plan's when the plant is the plan's model)
        unsigned char* host = new (std::nothrow) unsigned char[bb * cl->n_plant];
        if (host == nullptr) return MPPI_ERR_BAD_ARG;
        memset(host, 0, bb * cl->n_plant);
        if (cl->plant_params == nullptr) memcpy(host, pl->mparams, mk->param_bytes);
        else pack_param_rows(mk, &plant.p, cl->plant_params, cl->n_plant, cl->n_plant_params, host);
        // pageable source: the copy has taken the data when the call returns
        const cudaError_t ce = cudaMemcpyAsync(cl->plant_blocks, host, bb * cl->n_plant, cudaMemcpyHostToDevice, stream);
        delete[] host;
        if (ce != cudaSuccess) return cuda_fail(ce, "closed loop: plant block copy");
    }
    ps.u_scale = reinterpret_cast<const KArgs<real>*>(pl->kargs)->nm.u_scale;      // get_rollouts' u_scale (mppi.py:445)
    void* argv[1] = {(void*)&ps};
    real* states = (real*)cl->states;
    real* actions = (real*)cl->actions;
    const real* w = (const real*)cl->disturbance;
    const size_t xrow = (size_t)n_env * nx, urow = (size_t)n_env * nu;
    for (int s = 0; s < cl->steps; ++s) {
        real* xs = states + (size_t)s * xrow;
        real* us = actions + (size_t)s * urow;
        plan_update<real>(pl, nullptr, xs, MPPI_FLAG_SHIFT | MPPI_FLAG_STATE_DEVICE, cl->seed, cl->offset + (uint64_t)s * cl->offset_stride,
                          nullptr, us, nullptr);
        int rc = plan_launch(pl, stream);
        if (rc) return rc;
        ps.x = xs;
        ps.x_next = xs + xrow;
        ps.u = us;
        ps.w = w != nullptr ? w + (size_t)s * xrow : nullptr;
        ps.cost = cl->costs != nullptr ? (real*)cl->costs + (size_t)s * n_env : nullptr;
        // with the plan's PDL attribute: none on the tensor-core plans (select_tensor_core_route clears MPPI_FLAG_PDL)
        const cudaError_t e = launch_raw(mk->plant, (n_env + 127) / 128, 128, 0, stream, argv, pl->pdl != 0);
        if (e != cudaSuccess) return cuda_fail(e, "closed loop: plant step launch");
    }
    return MPPI_OK;
}

// ---- per-environment settings (mppi_plan_set_env_params) -------------------------------------------------
// scratch: n_env parameter blocks (plant_block_bytes apart), then n_env noise models
inline uint64_t env_nm_bytes(const Plan* pl) {
    return pl->is_double ? sizeof(NoiseModel<double>) : sizeof(NoiseModel<float>);
}
inline uint64_t env_scratch_bytes(const Plan* pl) {
    return (uint64_t)pl->p.n_env * (plant_block_bytes(pl->mk) + env_nm_bytes(pl));
}

// the reasons the settings are refused, before any CUDA call (MPPI_OK: none)
int check_env_params(const Plan* pl, const MppiEnvParams* ep) {
    if (pl == nullptr || ep == nullptr) return MPPI_ERR_BAD_ARG;
    if (ep->struct_size != sizeof(MppiEnvParams)) return MPPI_ERR_ABI;
    if (pl->p.n_env <= 1) return UNSUPPORTED("per-environment settings: the plan has one environment (MPPI_Batched only)");
    if (pl->p.world > 1 || (pl->p.flags & MPPI_FLAG_EXPORT_PARTIAL))
        return UNSUPPORTED("per-environment settings: not available on sharded controllers");
    if (ep->n_env != pl->p.n_env || ep->n_model_params < 0 || ep->reserved != 0) return MPPI_ERR_BAD_ARG;
    if ((ep->chol == nullptr) != (ep->sigma_inv == nullptr)) return MPPI_ERR_BAD_ARG;
    if (ep->lambda_ != nullptr)
        for (int e = 0; e < ep->n_env; ++e)
            if (!(ep->lambda_[e] > 0.0) || !isfinite(ep->lambda_[e])) return MPPI_ERR_BAD_ARG;
    if (ep->model_params != nullptr) {
        const bool gtile = (pl->p.flags & MPPI_FLAG_GLOBAL_TILE) != 0;
        if ((gtile ? pl->mk->env_gtile_batched : pl->mk->env_batched) == nullptr)
            return UNSUPPORTED("per-environment model parameters: this model has no per-environment kernel (the PendulumMLP models)");
    }
    const bool any = ep->lambda_ || ep->chol || ep->noise_mu || ep->model_params;
    if (any && (ep->scratch == nullptr || (uintptr_t)ep->scratch % 16 != 0 || ep->scratch_bytes < env_scratch_bytes(pl)))
        return MPPI_ERR_BAD_ARG;
    return MPPI_OK;
}

template <typename real>
int set_env_params_t(Plan* pl, const MppiEnvParams* ep, cudaStream_t stream) {
    KArgs<real>* a = reinterpret_cast<KArgs<real>*>(pl->kargs);
    const bool has_nm = ep->lambda_ || ep->chol || ep->noise_mu;
    if (!has_nm && ep->model_params == nullptr) {      // back to the plan's shared values
        a->env_nm = nullptr;
        pl->env_kernel = nullptr;
        pl->env_mp = nullptr;
        return MPPI_OK;
    }
    const int n_env = pl->p.n_env;
    const uint64_t bb = plant_block_bytes(pl->mk), mp_bytes = (uint64_t)n_env * bb;
    const void* env_kernel = nullptr;
    if (ep->model_params != nullptr) {
        // the per-environment kernel runs the plan's geometry (same tiles, grid and clusters, so the same reduction order):
        // its shared-memory limit is raised as the plan's kernel's was.  Its registers are not capped for two 512-thread
        // CTAs per SM (the cap spills); fewer resident CTAs than the plan counted on cost time, not correctness: only an
        // environment's finisher waits, for CTAs of its own environment dispatched before it.
        env_kernel = (pl->p.flags & MPPI_FLAG_GLOBAL_TILE) ? pl->mk->env_gtile_batched : pl->mk->env_batched;
        DevInfo di;
        int rc = get_dev_info(di);
        if (rc) return rc;
        cudaFuncAttributes fa;
        CK(cudaFuncGetAttributes(&fa, env_kernel));
        CK(cudaFuncSetAttribute(env_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, di.max_smem_optin - (int)fa.sharedSizeBytes));
        int occ = 0;
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, env_kernel, pl->g.BD, pl->g.smem));
        if (occ < 1) return UNSUPPORTED("per-environment model parameters: the per-environment kernel does not fit the plan's CTA");
    }
    unsigned char* host = new (std::nothrow) unsigned char[env_scratch_bytes(pl)];
    if (host == nullptr) return MPPI_ERR_BAD_ARG;
    memset(host, 0, env_scratch_bytes(pl));
    if (ep->model_params != nullptr) pack_param_rows(pl->mk, &pl->p, ep->model_params, n_env, ep->n_model_params, host);
    NoiseModel<real>* nms = reinterpret_cast<NoiseModel<real>*>(host + mp_bytes);
    if (has_nm) {
        // environment e's noise model: the plan's parameters with e's values, through the plan's own fill_noise_model
        MppiFusedParams pe = pl->p;
        for (int e = 0; e < n_env; ++e) {
            if (ep->lambda_ != nullptr) pe.lambda_ = ep->lambda_[e];
            if (ep->noise_mu != nullptr) memcpy(pe.noise_mu, ep->noise_mu + (size_t)e * MPPI_MAX_NU, sizeof(pe.noise_mu));
            if (ep->chol != nullptr) {
                const size_t nn = MPPI_MAX_NU * MPPI_MAX_NU;
                memcpy(pe.chol, ep->chol + (size_t)e * nn, sizeof(pe.chol));
                memcpy(pe.sigma_inv, ep->sigma_inv + (size_t)e * nn, sizeof(pe.sigma_inv));
                bool diag = true;
                for (int i = 0; i < MPPI_MAX_NU; ++i)
                    for (int j = 0; j < MPPI_MAX_NU; ++j) diag = diag && (i == j || pe.chol[i * MPPI_MAX_NU + j] == 0.0);
                pe.flags = diag ? (pe.flags | MPPI_FLAG_DIAG_SIGMA) : (pe.flags & ~(uint32_t)MPPI_FLAG_DIAG_SIGMA);
            }
            fill_noise_model<real>(&pe, nms[e]);
        }
    }
    // pageable source: the copy has taken the data when the call returns; commands enqueued before it have read the old
    // blocks by the time it lands (stream order)
    const cudaError_t ce = cudaMemcpyAsync(ep->scratch, host, env_scratch_bytes(pl), cudaMemcpyHostToDevice, stream);
    delete[] host;
    if (ce != cudaSuccess) return cuda_fail(ce, "per-environment settings: block copy");
    const unsigned char* scratch = (const unsigned char*)ep->scratch;
    a->env_nm = has_nm ? reinterpret_cast<const NoiseModel<real>*>(scratch + mp_bytes) : nullptr;
    pl->env_kernel = env_kernel;
    pl->env_mp = env_kernel != nullptr ? scratch : nullptr;
    pl->env_stride = (long long)bb;
    return MPPI_OK;
}

// ---- per-environment horizons (mppi_plan_set_env_horizon) ------------------------------------------------
inline uint64_t env_horizon_bytes(const Plan* pl) { return ((uint64_t)pl->p.n_env * sizeof(int32_t) + 15) / 16 * 16; }

// the reasons the horizons are refused, before any CUDA call (MPPI_OK: none)
int check_env_horizon(const Plan* pl, const int32_t* h, const void* scratch) {
    if (pl == nullptr) return MPPI_ERR_BAD_ARG;
    if (pl->p.n_env <= 1) return UNSUPPORTED("per-environment horizons: the plan has one environment (MPPI_Batched only)");
    if (pl->p.world > 1 || (pl->p.flags & MPPI_FLAG_EXPORT_PARTIAL))
        return UNSUPPORTED("per-environment horizons: not available on sharded controllers");
    if (pl->mk->is_mlp) return UNSUPPORTED("per-environment horizons: not available for the PendulumMLP models (their batched kernels fix their own tiles)");
    if (h == nullptr) return MPPI_OK;
    const int lo = pl->p.u_per_command > 1 ? pl->p.u_per_command : 1;
    for (int e = 0; e < pl->p.n_env; ++e)
        if (h[e] < lo || h[e] > pl->p.T) return MPPI_ERR_BAD_ARG;
    if (scratch == nullptr || (uintptr_t)scratch % 16 != 0) return MPPI_ERR_BAD_ARG;
    return MPPI_OK;
}

template <typename real>
int set_env_horizon_t(Plan* pl, const int32_t* h, void* scratch, cudaStream_t stream) {
    KArgs<real>* a = reinterpret_cast<KArgs<real>*>(pl->kargs);
    if (h == nullptr) {      // back to the plan's T
        a->env_horizon = nullptr;
        return MPPI_OK;
    }
    // pageable source: the copy has taken the data when the call returns; commands enqueued before it have read the old
    // horizons by the time it lands (stream order)
    const cudaError_t ce = cudaMemcpyAsync(scratch, h, (size_t)pl->p.n_env * sizeof(int32_t), cudaMemcpyHostToDevice, stream);
    if (ce != cudaSuccess) return cuda_fail(ce, "per-environment horizons: copy");
    a->env_horizon = (const int*)scratch;
    return MPPI_OK;
}

// ---- resident mode: the device backend of csrc/mppi_resident_host.h ---------------------------------
template <typename real>
int resident_launch_t(Plan* pl, uint64_t seed, uint64_t offset_pred, int shift_pred, uint64_t seq_start, uint32_t gen) {
    ResidentDevice& d = pl->resdev;
    KArgs<real> a = *reinterpret_cast<KArgs<real>*>(pl->kargs);
    a.seed = seed;
    a.z = nullptr;
    a.z_out = nullptr;
    a.state_dev = nullptr;
    a.action_out = (real*)d.action_dev;
    a.host_mailbox = d.host_box + RES_BOX_ACTION;
    a.pdl = 0;
    ResidentArgs ra;
    memset(&ra, 0, sizeof(ra));
    ra.host_cmd = d.host_box + RES_BOX_RECORD;
    ra.host_status = d.host_box + RES_BOX_DONE;
    ra.board = d.board;
    ra.seq_start = seq_start;
    ra.offset_pred = offset_pred;
    ra.idle_ns = d.idle_ns;
    ra.epoch_off = pl->res_epoch_off;
    ra.gen = gen;
    ra.shift_pred = shift_pred;
    ra.n_words = 3 + pl->nx * (pl->is_double ? 2 : 1);
    DevInfo di;
    int rc = get_dev_info(di);
    if (rc) return rc;
    // the launch route's grid (one tile per CTA, padded to the cluster size) and cluster size: same reduction tree, same
    // bits.  If the driver refuses cooperative + cluster together, the grid is launched without clusters (its results
    // then agree with the launch route to fp64 rounding of the reduction order instead of bit for bit).
    const MppiFusedParams& pp = pl->p;
    cudaFuncAttributes fa;
    CK(cudaFuncGetAttributes(&fa, pl->res_kernel));
    const int dyn_limit = di.max_smem_optin - (int)fa.sharedSizeBytes;
    CK(cudaFuncSetAttribute(pl->res_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn_limit));
    CK(cudaMemsetAsync(d.board, 0, MPPI_RES_BOARD_WORDS * sizeof(unsigned long long), d.stream));
    void* argv[3] = {(void*)&a, (void*)pl->mparams, (void*)&ra};
    cudaError_t e = cudaErrorInvalidConfiguration;
    for (int cs = pl->g.cluster; cs >= 1; cs = (cs > 1 ? 1 : 0)) {
        const int nb = cs > 1 ? pl->g.nb : a.n_tiles;
        const int smem = make_layout<real>(pp.variant, pp.T, pp.nu, pp.S, a.R, pl->g.BD, pl->g.BS, fused_layout_nb(nb / cs, a.xchg_npub),
                                           layout_extra(pp.variant != MPPI_VARIANT_MPPI, pl->nx, cs, fused_xstage_doubles(false, 1, a.xchg_npub, a.R))).total;
        if (smem > dyn_limit) return UNSUPPORTED("resident kernel: shared-memory tile does not fit");
        // cooperative: every CTA is resident or the launch fails — the CTAs wait for each other through the board
        cudaLaunchConfig_t cfg;
        cudaLaunchAttribute at[3];
        launch_config(cfg, at, nb, pl->g.BD, smem, d.stream, false, 1, cs);
        at[cfg.numAttrs].id = cudaLaunchAttributeCooperative;
        at[cfg.numAttrs].val.cooperative = 1;
        ++cfg.numAttrs;
        e = cudaLaunchKernelExC(&cfg, pl->res_kernel, argv);
        if (e == cudaSuccess) break;
        cudaGetLastError();
    }
    if (e != cudaSuccess) return cuda_fail(e, "resident launch");
    return MPPI_OK;
}
int resident_be_launch(void* ctx, uint64_t seed, uint64_t offset_pred, int shift_pred, uint64_t seq_start, uint32_t gen) {
    Plan* pl = reinterpret_cast<Plan*>(ctx);
    return pl->is_double ? resident_launch_t<double>(pl, seed, offset_pred, shift_pred, seq_start, gen)
                         : resident_launch_t<float>(pl, seed, offset_pred, shift_pred, seq_start, gen);
}
int resident_be_drain(void* ctx) {
    Plan* pl = reinterpret_cast<Plan*>(ctx);
    CK(cudaStreamSynchronize(pl->resdev.stream));
    return MPPI_OK;
}
int resident_be_health(void* ctx) {
    Plan* pl = reinterpret_cast<Plan*>(ctx);
    cudaError_t q = cudaStreamQuery(pl->resdev.stream);
    if (q != cudaSuccess && q != cudaErrorNotReady) return cuda_fail(q, "cudaStreamQuery while waiting for the resident grid");
    return MPPI_OK;
}
static_assert(MPPI_RES_CMD_SHIFT == (unsigned)RES_CMD_SHIFT && MPPI_RES_CMD_STOP == (unsigned)RES_CMD_STOP, "record flags: host and device disagree");
static_assert((int)RES_ERR_BAD_ARG == (int)MPPI_ERR_BAD_ARG && (int)RES_ERR_TIMEOUT == (int)MPPI_ERR_TIMEOUT, "status codes of the protocol header");

// ---- generic path: sample / softmin -------------------------------------------------------------
// MPPI_FLAG_GLOBAL_TILE: the global-tile kernels, whose tile slices follow the record mailbox in the workspace
inline bool gtile_of(const MppiFusedParams* p) { return (p->flags & MPPI_FLAG_GLOBAL_TILE) != 0; }
inline int check_gtile_workspace(const MppiFusedParams* p, const Geometry& g, int rows2) {
    const uint64_t need = ws_bytes(g.nb, rows_of(p)) + ws_gtile_plan_bytes(p, g.nb, g.BS, rows2);
    if (p->workspace == nullptr || p->workspace_bytes < need) return MPPI_ERR_WORKSPACE;
    if (p->n_env > 1 && (p->env_ws_stride < need || p->env_ws_stride % MPPI_WS_ALIGN != 0 ||
                         p->workspace_bytes < p->env_ws_stride * (uint64_t)p->n_env))
        return MPPI_ERR_WORKSPACE;
    return MPPI_OK;
}

template <typename real, int V, int NU>
int plan_sample(const MppiFusedParams* p, Geometry& g) {
    if (!gtile_of(p)) return plan_geometry<real>(sample_kernel<real, V, NU>, p, V == V_KMPPI, false, g);
    if (const char* why = gtile_refusal(nullptr, p)) return UNSUPPORTED(why);
    int rc = plan_geometry<real>(sample_kernel_gtile<real, V, NU>, p, V == V_KMPPI, false, g, 0, true);
    return rc ? rc : check_gtile_workspace(p, g, V == V_KMPPI);
}

template <typename real, int V, int NU>
int run_sample(const MppiFusedParams* p, KArgs<real>& a_extra, cudaStream_t stream) {
    auto kernel = gtile_of(p) ? sample_kernel_gtile<real, V, NU> : sample_kernel<real, V, NU>;
    Geometry g;
    int rc = plan_sample<real, V, NU>(p, g);
    if (rc) return rc;
    KArgs<real> a;
    fill_kargs<real>(p, a, g.BS, g.nb, g.tps);
    a.out_pa = a_extra.out_pa;
    a.out_noise = a_extra.out_noise;
    a.out_noise_theta = a_extra.out_noise_theta;
    a.out_cost_init = a_extra.out_cost_init;
    a.override_rows = a_extra.override_rows;
    a.n_override = a_extra.n_override;
    a.override_start = a_extra.override_start;
    if (a_extra.shift < 0) {   // materialise from nominal_used: no shift, plain loads
        a.U = (real*)p->nominal_used;
        a.A = a.U + a.TN;
        a.theta = a.U + 2 * a.TN;
        a.shift = 0;
        a.tma_ok = 0;
        a.nominal_used = nullptr;
    }
    return launch_kernel(kernel, g.nb, g.BD, g.smem, stream, a.n_env, a);
}

template <typename real, int V> int run_sample_nu(const MppiFusedParams* p, KArgs<real>& e, cudaStream_t s) {
    switch (p->nu) {
        case 1: return run_sample<real, V, 1>(p, e, s);
        case 2: return run_sample<real, V, 2>(p, e, s);
        case 3: return run_sample<real, V, 3>(p, e, s);
        case 4: return run_sample<real, V, 4>(p, e, s);
    }
    return MPPI_ERR_UNSUPPORTED;
}

template <typename real>
int run_sample_any(const MppiFusedParams* p, void* pa, void* noise, void* noise_theta, void* cost_init, const void* ovr,
                   int n_ovr, int ovr_start, bool from_nominal_used, cudaStream_t s) {
    KArgs<real> e;
    memset(&e, 0, sizeof(e));
    e.out_pa = (real*)pa;
    e.out_noise = (real*)noise;
    e.out_noise_theta = (real*)noise_theta;
    e.out_cost_init = (real*)cost_init;
    e.override_rows = (const real*)ovr;
    e.n_override = n_ovr;
    e.override_start = ovr_start;
    e.shift = from_nominal_used ? -1 : 0;
    switch (p->variant) {
        case MPPI_VARIANT_MPPI: return run_sample_nu<real, V_MPPI>(p, e, s);
        case MPPI_VARIANT_SMPPI: return run_sample_nu<real, V_SMPPI>(p, e, s);
        case MPPI_VARIANT_KMPPI: return run_sample_nu<real, V_KMPPI>(p, e, s);
    }
    return MPPI_ERR_BAD_ARG;
}

// check_ws = false: the geometry alone (mppi_fused_query asks before the caller has a workspace)
template <typename real, int V, int NU>
int plan_softmin(const MppiFusedParams* p, Geometry& g, bool check_ws = true) {
    // the warp-fold tail without clusters, one record per rank: its layout as softmin_update_kernel builds it
    const int xst = fused_xstage_doubles(sharded_in_kernel(p), p->world, 1, rows_of(p));
    const int env_bytes = p->n_env > 1 ? (int)sizeof(KArgs<real>) : 0;
    if (gtile_of(p)) {
        if (const char* why = gtile_refusal(nullptr, p)) return UNSUPPORTED(why);
        int rc = plan_geometry<real>(softmin_update_kernel_gtile<real, V, NU>, p, layout_extra(0, 0, 1, xst), true, g, env_bytes, true);
        return rc ? rc : check_gtile_workspace(p, g, 0);
    }
    int rc = plan_geometry<real>(softmin_update_kernel<real, V, NU>, p, layout_extra(0, 0, 1, xst), true, g, env_bytes);
    if (rc || !check_ws) return rc;
    const uint64_t need_ws = ws_bytes(g.nb, rows_of(p));
    if (p->workspace == nullptr || p->workspace_bytes < need_ws) return MPPI_ERR_WORKSPACE;
    if (p->n_env > 1 && (p->env_ws_stride < need_ws || p->env_ws_stride % MPPI_WS_ALIGN != 0 ||
                         p->workspace_bytes < p->env_ws_stride * (uint64_t)p->n_env))
        return MPPI_ERR_WORKSPACE;
    return MPPI_OK;
}

template <typename real, int V, int NU>
int run_softmin(const MppiFusedParams* p, const void* cost, const void* eps, cudaStream_t stream) {
    auto kernel = gtile_of(p) ? softmin_update_kernel_gtile<real, V, NU> : softmin_update_kernel<real, V, NU>;
    Geometry g;
    int rc = plan_softmin<real, V, NU>(p, g);
    if (rc) return rc;
    KArgs<real> a;
    fill_kargs<real>(p, a, g.BS, g.nb, g.tps);
    a.in_cost = (const real*)cost;
    a.in_eps = (const real*)eps;
    if (a.world > 1 && rows_of(p) > MPPI_XCHG_MAX_R) return UNSUPPORTED("T*nu exceeds the peer mailbox record size");
    return launch_kernel(kernel, g.nb, g.BD, g.smem, stream, a.n_env, a);
}

template <typename real, int V> int run_softmin_nu(const MppiFusedParams* p, const void* c, const void* e, cudaStream_t s) {
    switch (p->nu) {
        case 1: return run_softmin<real, V, 1>(p, c, e, s);
        case 2: return run_softmin<real, V, 2>(p, c, e, s);
        case 3: return run_softmin<real, V, 3>(p, c, e, s);
        case 4: return run_softmin<real, V, 4>(p, c, e, s);
    }
    return MPPI_ERR_UNSUPPORTED;
}
template <typename real> int run_softmin_any(const MppiFusedParams* p, const void* c, const void* e, cudaStream_t s) {
    switch (p->variant) {
        case MPPI_VARIANT_MPPI: return run_softmin_nu<real, V_MPPI>(p, c, e, s);
        case MPPI_VARIANT_SMPPI: return run_softmin_nu<real, V_SMPPI>(p, c, e, s);
        case MPPI_VARIANT_KMPPI: return run_softmin_nu<real, V_KMPPI>(p, c, e, s);
    }
    return MPPI_ERR_BAD_ARG;
}

// the larger dynamic shared memory of the sampling and softmin plans of these dimensions (mppi_fused_query, model == 0);
// 0 if either does not fit
template <typename real, int V, int NU> int stepped_smem(const MppiFusedParams* p) {
    Geometry gs, gu;
    if (plan_sample<real, V, NU>(p, gs) != MPPI_OK) return 0;
    if (plan_softmin<real, V, NU>(p, gu, false) != MPPI_OK) return 0;
    return gs.smem > gu.smem ? gs.smem : gu.smem;
}
template <typename real> int stepped_smem_any(const MppiFusedParams* p) {
    const int V = p->variant, nu = p->nu;
#define MPPI_STEPPED_SMEM_NU(VV)                                      \
    switch (nu) {                                                      \
        case 1: return stepped_smem<real, VV, 1>(p);                   \
        case 2: return stepped_smem<real, VV, 2>(p);                   \
        case 3: return stepped_smem<real, VV, 3>(p);                   \
        case 4: return stepped_smem<real, VV, 4>(p);                   \
    }
    if (V == V_MPPI) { MPPI_STEPPED_SMEM_NU(V_MPPI) }
    else if (V == V_SMPPI) { MPPI_STEPPED_SMEM_NU(V_SMPPI) }
    else { MPPI_STEPPED_SMEM_NU(V_KMPPI) }
#undef MPPI_STEPPED_SMEM_NU
    return 0;
}

template <typename real, int V>
int run_apply(const MppiFusedParams* p, const void* partials, cudaStream_t stream) {
    KArgs<real> a;
    fill_kargs<real>(p, a, 128, 1);
    a.world = p->world <= 0 ? 1 : p->world;
    const int smem = align_up((2 * a.TN + a.R + a.T * a.S) * (int)sizeof(real), 16) + (a.R + 2) * 8 + 16;
    apply_partials_kernel<real, V><<<1, 128, smem, stream>>>(a, (const double*)partials, p->nu);
    CK(cudaGetLastError());
    return MPPI_OK;
}

}  // namespace

// =================================================================================================
extern "C" {

int mppi_b200_abi_version(void) { return MPPI_B200_ABI_VERSION; }

uint64_t mppi_abi_layout(int which) {
    switch (which) {
        case 0: return sizeof(MppiFusedParams);
        case 1: return offsetof(MppiFusedParams, seed);
        case 2: return offsetof(MppiFusedParams, state);
        case 3: return offsetof(MppiFusedParams, U);
        case 4: return offsetof(MppiFusedParams, rank);
        case 5: return offsetof(MppiFusedParams, partial_out);
        case 6: return sizeof(MppiLaunchInfo);
        case 7: return offsetof(MppiFusedParams, model_weights);
        case 8: return offsetof(MppiFusedParams, model_tensors);
        case 9: return sizeof(MppiClosedLoop);
        case 10: return offsetof(MppiClosedLoop, states);
        case 11: return offsetof(MppiClosedLoop, plant_params);
        case 12: return offsetof(MppiClosedLoop, plant_blocks);
        case 13: return sizeof(MppiEnvParams);
        case 14: return offsetof(MppiEnvParams, chol);
        case 15: return offsetof(MppiEnvParams, model_params);
        case 16: return offsetof(MppiEnvParams, scratch);
        case 17: return sizeof(MppiPlantModel);
        case 18: return offsetof(MppiPlantModel, model_tensors);
    }
    return 0;
}

const char* mppi_status_string(int s) {
    switch (s) {
        case MPPI_OK: return "ok";
        case MPPI_ERR_BAD_ARG: return "bad argument";
        case MPPI_ERR_UNSUPPORTED: return "unsupported (model, variant, dtype, size) combination";
        case MPPI_ERR_WORKSPACE: return "workspace too small";
        case MPPI_ERR_CUDA: return "CUDA error";
        case MPPI_ERR_ABI: return "MppiFusedParams size mismatch (ABI)";
        case MPPI_ERR_TIMEOUT: return "peer exchange timed out";
    }
    return "unknown status";
}

const char* mppi_last_cuda_error(void) { return g_cuda_err; }

int mppi_fused_query(const MppiFusedParams* p, MppiLaunchInfo* out) {
    if (out == nullptr) return MPPI_ERR_BAD_ARG;
    memset(out, 0, sizeof(*out));
    int rc = validate(p);
    if (rc) return rc;
    if (p->model == 0) {      // the per-step entry points: only the workspace mppi_softmin_update needs
        if (gtile_of(p))
            if (const char* why = gtile_refusal(nullptr, p)) return UNSUPPORTED(why);
        DevInfo di;
        if ((rc = get_dev_info(di)) != MPPI_OK) return rc;
        out->sm_count = di.sm_count;
        out->workspace_bytes = ws_bytes(max_planned_grid(p, di.sm_count), rows_of(p));
        if (gtile_of(p)) {
            out->workspace_bytes += ws_gtile_bytes(p, di.sm_count);
            out->global_tile = 1;
        } else {
            out->smem_bytes = p->dtype == MPPI_F32 ? stepped_smem_any<float>(p) : stepped_smem_any<double>(p);
        }
        return MPPI_OK;
    }
    if ((rc = validate(p, true)) != MPPI_OK) return rc;
    const ModelKernels* mk = find_kernels(p, &rc);
    if (mk == nullptr) return rc;
    if ((rc = check_model_args(p, mk)) != MPPI_OK) return rc;
    return mk->is_double ? query_fused<double>(mk, p, out) : query_fused<float>(mk, p, out);
}

// a one-shot plan, with the record tags of a plan-less command: one process-wide counter on a single GPU (or with
// EXPORT_PARTIAL), the caller's epoch on an in-kernel sharded controller (every rank issues the same sequence)
int mppi_fused_command(const MppiFusedParams* p, void* stream) {
    void* plan = nullptr;
    int rc = mppi_plan_create(p, &plan);
    if (rc) return rc;
    Plan* pl = reinterpret_cast<Plan*>(plan);
    static unsigned long long s_epoch = 0;
    // plan_update pre-increments both tags
    pl->epoch = sharded_in_kernel(p) ? p->epoch - 1 : __atomic_add_fetch(&s_epoch, 1ull, __ATOMIC_RELAXED) - 1;
    pl->host_epoch = p->host_epoch - 1;
    rc = plan_command(pl, p->state, p->state_dev, p->flags, p->seed, p->offset, p->z, p->action_out, p->host_mailbox, (cudaStream_t)stream);
    delete pl;
    return rc;
}

int mppi_plan_create(const MppiFusedParams* p, void** plan_out) {
    if (plan_out == nullptr) return MPPI_ERR_BAD_ARG;
    int rc = validate(p, true);
    if (rc) return rc;
    Plan* pl = new (std::nothrow) Plan();
    if (pl == nullptr) return MPPI_ERR_BAD_ARG;
    const ModelKernels* mk = find_kernels(p, &rc);
    if (mk != nullptr) rc = check_model_args(p, mk);
    if (mk != nullptr && rc == MPPI_OK) rc = mk->is_double ? build_plan<double>(mk, p, pl) : build_plan<float>(mk, p, pl);
    if (rc) {
        delete pl;
        return rc;
    }
    *plan_out = pl;
    return MPPI_OK;
}

int mppi_plan_destroy(void* plan) {
    if (plan == nullptr) return MPPI_ERR_BAD_ARG;
    Plan* pl = reinterpret_cast<Plan*>(plan);
    if (pl->res.armed) mppi_resident_stop(plan);      // the resident grid reads this controller's buffers
    delete pl;
    return MPPI_OK;
}

int mppi_plan_command(void* plan, const double* state, const void* state_dev, uint32_t flags, uint64_t seed, uint64_t offset,
                      const void* z, void* action_out, void* stream) {
    return plan_command(reinterpret_cast<Plan*>(plan), state, state_dev, flags, seed, offset, z, action_out, nullptr, (cudaStream_t)stream);
}

// the plan's parameter block is a kernel argument: it is copied at every launch, so a launch already enqueued keeps the
// values it was launched with; a resident grid holds the block of its own launch for as long as it stays
int mppi_plan_set_model_params(void* plan, const double* model_params, const double* ext, int32_t n_ext) {
    Plan* pl = reinterpret_cast<Plan*>(plan);
    if (pl == nullptr || model_params == nullptr || n_ext < 0 || (n_ext > 0 && ext == nullptr)) return MPPI_ERR_BAD_ARG;
    if (pl->mk->is_mlp && ((pl->mk->is_mlp == 1 && n_ext < PendulumMLPModel::N_EXT) || model_params[2] != pl->p.model_params[2] ||
                           model_params[3] != pl->p.model_params[3]))
        return MPPI_ERR_BAD_ARG;      // the weights are required, and [2] / [3] selected the plan's kernel
    if (pl->res.armed) return UNSUPPORTED("the resident grid holds the parameters it was launched with: stop it first");
    memcpy(pl->p.model_params, model_params, sizeof(pl->p.model_params));
    pl->p.model_params_ext = ext;
    pl->p.n_model_params_ext = n_ext;
    load_model_params(pl->mk, &pl->p, pl->mparams);
    return MPPI_OK;
}

// as mppi_plan_set_model_params, for the tensor views only (the parameters stay as they are)
int mppi_plan_set_model_tensors(void* plan, const MppiTensorRef* refs, int32_t n) {
    Plan* pl = reinterpret_cast<Plan*>(plan);
    if (pl == nullptr || check_model_tensors(pl->mk, refs, n) != MPPI_OK) return MPPI_ERR_BAD_ARG;
    if (pl->res.armed) return UNSUPPORTED("the resident grid holds the tensors it was launched with: stop it first");
    if (n > 0) memcpy(pl->tensors, refs, sizeof(MppiTensorRef) * n);
    load_model_tensors(pl->mk, pl->tensors, pl->mparams);
    return MPPI_OK;
}

uint64_t mppi_plan_model_block_bytes(void* plan) {
    const Plan* pl = reinterpret_cast<const Plan*>(plan);
    return pl == nullptr ? 0 : plant_block_bytes(pl->mk);
}

uint64_t mppi_plant_block_bytes(void* plan, const MppiPlantModel* plant) {
    PlantOf po;
    return resolve_plant(reinterpret_cast<const Plan*>(plan), plant, &po) == MPPI_OK ? plant_block_bytes(po.mk) : 0;
}

int mppi_plan_closed_loop_plant(void* plan, const MppiClosedLoop* cl, const MppiPlantModel* plant, void* stream) {
    Plan* pl = reinterpret_cast<Plan*>(plan);
    PlantOf po;
    int rc = resolve_plant(pl, plant, &po);
    if (rc == MPPI_OK) rc = check_closed_loop(pl, cl, po, plant != nullptr);
    if (rc) return rc;
    return pl->is_double ? closed_loop_t<double>(pl, cl, po, (cudaStream_t)stream) : closed_loop_t<float>(pl, cl, po, (cudaStream_t)stream);
}

int mppi_plan_closed_loop(void* plan, const MppiClosedLoop* cl, void* stream) {
    return mppi_plan_closed_loop_plant(plan, cl, nullptr, stream);
}

uint64_t mppi_plan_env_scratch_bytes(void* plan) {
    const Plan* pl = reinterpret_cast<const Plan*>(plan);
    return pl == nullptr ? 0 : env_scratch_bytes(pl);
}

int mppi_plan_set_env_params(void* plan, const MppiEnvParams* ep, void* stream) {
    Plan* pl = reinterpret_cast<Plan*>(plan);
    const int rc = check_env_params(pl, ep);
    if (rc) return rc;
    return pl->is_double ? set_env_params_t<double>(pl, ep, (cudaStream_t)stream) : set_env_params_t<float>(pl, ep, (cudaStream_t)stream);
}

uint64_t mppi_plan_env_horizon_bytes(void* plan) {
    const Plan* pl = reinterpret_cast<const Plan*>(plan);
    return pl == nullptr ? 0 : env_horizon_bytes(pl);
}

int mppi_plan_set_env_horizon(void* plan, const int32_t* horizon_host, void* scratch, void* stream) {
    Plan* pl = reinterpret_cast<Plan*>(plan);
    const int rc = check_env_horizon(pl, horizon_host, scratch);
    if (rc) return rc;
    return pl->is_double ? set_env_horizon_t<double>(pl, horizon_host, scratch, (cudaStream_t)stream)
                         : set_env_horizon_t<float>(pl, horizon_host, scratch, (cudaStream_t)stream);
}

int mppi_plan_command_host(void* plan, const double* state, uint32_t flags, uint64_t seed, uint64_t offset, const void* z,
                           void* action_out_dev, void* host_mailbox, void* action_host_out, void* stream) {
    Plan* pl = reinterpret_cast<Plan*>(plan);
    if (pl == nullptr || state == nullptr || host_mailbox == nullptr || action_host_out == nullptr || action_out_dev == nullptr)
        return MPPI_ERR_BAD_ARG;
    int rc = plan_command(pl, state, nullptr, flags, seed, offset, z, action_out_dev, host_mailbox, (cudaStream_t)stream);
    if (rc) return rc;
    // every action value arrives as self-validating 8-byte word(s): payload32 | (epoch & 0xffffffff) << 32
    volatile unsigned long long* box = reinterpret_cast<volatile unsigned long long*>(host_mailbox);
    const unsigned long long want = pl->host_epoch & 0xffffffffull;
    const int nwords = pl->upc_nu * (pl->is_double ? 2 : 1);
    unsigned long long spins = 0;
    for (int w = 0; w < nwords; ++w) {
        while ((box[w] >> 32) != want) {
#if defined(__x86_64__)
            __builtin_ia32_pause();
#endif
            if ((++spins & 0xFFFFF) == 0) {       // every ~1M spins: has the stream died or finished without publishing?
                cudaError_t q = cudaStreamQuery((cudaStream_t)stream);
                if (q != cudaSuccess && q != cudaErrorNotReady) return cuda_fail(q, "cudaStreamQuery while waiting for the mailbox");
                if (q == cudaSuccess && (box[w] >> 32) != want) return MPPI_ERR_TIMEOUT;
            }
        }
    }
    // the action is returned in the controller's own dtype (f32 words or f64 double-words)
    if (pl->is_double) {
        unsigned long long* out = reinterpret_cast<unsigned long long*>(action_host_out);
        for (int i = 0; i < pl->upc_nu; ++i) out[i] = (box[2 * i] & 0xffffffffull) | (box[2 * i + 1] << 32);
    } else {
        uint32_t* out = reinterpret_cast<uint32_t*>(action_host_out);
        for (int i = 0; i < pl->upc_nu; ++i) out[i] = (uint32_t)box[i];
    }
    return MPPI_OK;
}

// The record epochs a resident session used (res_epoch_off + seq, stop records included) become the plan's own: the
// workspace still holds records with those tags, so neither the next session nor a launch-route command may reuse them.
inline void fold_resident_epochs(Plan* pl) {
    if (pl->res_epoch_off + pl->res.seq > pl->epoch) pl->epoch = pl->res_epoch_off + pl->res.seq;
}

int mppi_resident_start(void* plan, void* host_box, void* board_dev, void* action_out_dev, uint64_t idle_us, void* stream) {
    Plan* pl = reinterpret_cast<Plan*>(plan);
    if (pl == nullptr || host_box == nullptr || board_dev == nullptr || action_out_dev == nullptr || idle_us == 0)
        return MPPI_ERR_BAD_ARG;
    if (pl->p.flags & MPPI_FLAG_GLOBAL_TILE)
        return UNSUPPORTED("resident mode keeps its tiles in shared memory: not available on a global-tile plan (tile_memory)");
    if (pl->res_kernel == nullptr)
        return UNSUPPORTED("resident mode needs a plan on the split-cost rollout (one tile per SM, one environment, single GPU)");
    if (pl->p.z_out != nullptr) return UNSUPPORTED("resident mode does not record the noise it draws (z_out)");
    if (pl->res.launched) {                 // re-arming: the old grid leaves first (it polls the box that is about to be cleared)
        int rc = res_halt(pl->res);
        if (rc) return rc;
    }
    fold_resident_epochs(pl);
    ResidentDevice& d = pl->resdev;
    d.host_box = reinterpret_cast<unsigned long long*>(host_box);
    d.board = reinterpret_cast<unsigned long long*>(board_dev);
    d.action_dev = action_out_dev;
    d.idle_ns = idle_us * 1000ull;
    d.stream = (cudaStream_t)stream;
    const ResidentBackend be{pl, resident_be_launch, resident_be_drain, resident_be_health};
    const int rc_arm = res_arm(pl->res, host_box, pl->nx, pl->upc_nu, pl->is_double, be, 0);
    // resident commands continue the plan's epochs: command seq carries epoch res_epoch_off + seq
    pl->res_epoch_off = pl->epoch - pl->res.seq;
    return rc_arm;
}

int mppi_resident_command(void* plan, const double* state, uint32_t flags, uint64_t seed, uint64_t offset, void* action_host_out) {
    Plan* pl = reinterpret_cast<Plan*>(plan);
    if (pl == nullptr) return MPPI_ERR_BAD_ARG;
    return res_command(pl->res, state, (flags & MPPI_FLAG_SHIFT) ? 1 : 0, seed, offset, action_host_out, 0);
}

int mppi_resident_sync(void* plan) {
    Plan* pl = reinterpret_cast<Plan*>(plan);
    return pl == nullptr ? (int)MPPI_ERR_BAD_ARG : res_sync(pl->res);
}

int mppi_resident_stop(void* plan) {
    Plan* pl = reinterpret_cast<Plan*>(plan);
    if (pl == nullptr) return MPPI_ERR_BAD_ARG;
    const int rc = res_stop(pl->res);
    fold_resident_epochs(pl);
    return rc;
}

// ---- user models compiled at run time ----------------------------------------------------------------------------------
// The Python side compiles `mppi_fused.cuh + mppi_resident.cuh + the user's model header` with NVRTC (in process, no
// toolkit) into a cubin and hands it over with the lowered names of the kernels; they are loaded as a cudaLibrary_t and
// wrapped in a ModelKernels table exactly like a registry unit's.  `names`: 5 entries, nullptr = not built:
//   [0] fused (this variant)  [1] split-cost  [2] batched (MPPI variant only)  [3] resident  [4] states
// and the kernels a module exports under fixed names (LL, global-tile, plant step)
namespace {
void user_load(const ModelKernels* mk, void* dst, const double* blob, const double* ext, int n_ext) {
    for (int i = 0; i < mk->np; ++i) {
        const double v = i < MPPI_MODEL_PARAM_DOUBLES ? blob[i] : ((ext != nullptr && i - MPPI_MODEL_PARAM_DOUBLES < n_ext) ? ext[i - MPPI_MODEL_PARAM_DOUBLES] : 0.0);
        if (mk->is_double) reinterpret_cast<double*>(dst)[i] = v;
        else reinterpret_cast<float*>(dst)[i] = (float)v;
    }
}
}  // namespace

int mppi_user_model_register(const void* cubin, uint64_t cubin_bytes, int32_t nx, int32_t nu, int32_t n_params, int32_t dtype,
                             int32_t variant, const char* const* names, void** handle_out) {
    if (cubin == nullptr || cubin_bytes == 0 || names == nullptr || handle_out == nullptr) return MPPI_ERR_BAD_ARG;
    if (nx < 1 || nx > MPPI_MAX_NX || nu < 1 || nu > MPPI_MAX_NU || n_params < 1 || variant < 0 || variant > 2) return MPPI_ERR_BAD_ARG;
    if (dtype != MPPI_F32 && dtype != MPPI_F64) return MPPI_ERR_BAD_ARG;
    const int es = dtype == MPPI_F64 ? 8 : 4;
    if (n_params * es > MPPI_MODEL_BLOCK_BYTES) return UNSUPPORTED("user model has too many parameters");
    cudaLibrary_t lib = nullptr;
    CK(cudaLibraryLoadData(&lib, cubin, nullptr, nullptr, 0, nullptr, nullptr, 0));
    UserModelHandle* h = new (std::nothrow) UserModelHandle();
    if (h == nullptr) return MPPI_ERR_BAD_ARG;
    memset(h, 0, sizeof(*h));
    h->magic = kUserMagic;
    ModelKernels& mk = h->mk;
    mk.nx = nx;
    mk.nu = nu;
    mk.is_double = dtype == MPPI_F64;
    mk.np = n_params;
    mk.param_bytes = n_params * es;
    mk.load = user_load;
    mk.library = (void*)lib;
    const void** slots[5] = {&mk.fused[variant], &mk.split[variant], &mk.batched, &mk.resident[variant], &mk.states};
    for (int i = 0; i < 5; ++i) {
        if (names[i] == nullptr) continue;
        cudaKernel_t k = nullptr;
        cudaError_t e = cudaLibraryGetKernel(&k, lib, names[i]);
        if (e != cudaSuccess) {
            cudaLibraryUnload(lib);
            delete h;
            return cuda_fail(e, names[i]);
        }
        *slots[i] = (const void*)k;
    }
    if (mk.split[variant] != nullptr) {
        // its single-GPU LL form, which the module exports under a fixed name (MPPI_USER_KERNEL_LL in mppi_fused.cuh)
        cudaKernel_t k = nullptr;
        cudaError_t e = cudaLibraryGetKernel(&k, lib, "mppi_user_fused_command_kernel_ll");
        if (e != cudaSuccess) {
            cudaLibraryUnload(lib);
            delete h;
            return cuda_fail(e, "mppi_user_fused_command_kernel_ll");
        }
        mk.split_ll[variant] = (const void*)k;
    }
    // its global-tile kernels, exported under fixed names (MPPI_USER_KERNEL_GTILE / _BATCHED in mppi_fused.cuh), and beside
    // the batched kernel its per-environment forms (MPPI_USER_KERNEL_ENV_BATCHED)
    const bool b = mk.batched != nullptr;
    const char* gnames[4] = {"mppi_user_fused_command_kernel_gtile", b ? "mppi_user_fused_command_kernel_gtile_batched" : nullptr,
                             b ? "mppi_user_fused_command_kernel_env" : nullptr, b ? "mppi_user_fused_command_kernel_env_gtile" : nullptr};
    const void** gslots[4] = {&mk.gtile[variant], &mk.gtile_batched, &mk.env_batched, &mk.env_gtile_batched};
    for (int i = 0; i < 4; ++i) {
        if (gnames[i] == nullptr) continue;
        cudaKernel_t k = nullptr;
        cudaError_t e = cudaLibraryGetKernel(&k, lib, gnames[i]);
        if (e != cudaSuccess) {
            cudaLibraryUnload(lib);
            delete h;
            return cuda_fail(e, gnames[i]);
        }
        *gslots[i] = (const void*)k;
    }
    // its closed-loop plant step, where the module has one (MPPI_USER_KERNEL_PLANT; none for step-dependent models)
    {
        cudaKernel_t k = nullptr;
        if (cudaLibraryGetKernel(&k, lib, "mppi_user_plant_step_kernel") == cudaSuccess) mk.plant = (const void*)k;
        else cudaGetLastError();      // absent: closed loops of this model are refused
    }
    if (mk.fused[variant] == nullptr || mk.states == nullptr) {
        cudaLibraryUnload(lib);
        delete h;
        return MPPI_ERR_BAD_ARG;
    }
    *handle_out = h;
    return MPPI_OK;
}

int mppi_user_model_release(void* handle) {
    UserModelHandle* h = reinterpret_cast<UserModelHandle*>(handle);
    if (h == nullptr || h->magic != kUserMagic) return MPPI_ERR_BAD_ARG;
    if (h->mk.library != nullptr) cudaLibraryUnload((cudaLibrary_t)h->mk.library);
    h->magic = 0;
    delete h;
    return MPPI_OK;
}

int mppi_user_model_set_copies(void* handle, int32_t copies) {
    UserModelHandle* h = reinterpret_cast<UserModelHandle*>(handle);
    if (h == nullptr || h->magic != kUserMagic || copies < 1 || copies > MPPI_MAX_COPIES) return MPPI_ERR_BAD_ARG;
    const ModelKernels& mk = h->mk;
    bool others = mk.batched != nullptr;
    for (int v = 0; v < 3; ++v) others = others || mk.split[v] != nullptr || mk.resident[v] != nullptr;
    if (copies > 1 && others) return MPPI_ERR_BAD_ARG;     // those kernels roll out one copy per sample
    h->mk.copies = copies;
    return MPPI_OK;
}

int mppi_user_model_set_tensors(void* handle, int32_t n, const int32_t* dtypes, const int32_t* ndims) {
    UserModelHandle* h = reinterpret_cast<UserModelHandle*>(handle);
    if (h == nullptr || h->magic != kUserMagic || n < 0 || n > MPPI_MAX_MODEL_TENSORS) return MPPI_ERR_BAD_ARG;
    if (n > 0 && (dtypes == nullptr || ndims == nullptr)) return MPPI_ERR_BAD_ARG;
    for (int i = 0; i < n; ++i)
        if (!mppi_tensors::known_dtype(dtypes[i]) || ndims[i] < 1 || ndims[i] > 4) return MPPI_ERR_BAD_ARG;
    ModelKernels& mk = h->mk;
    const int bytes = mppi_tensors::block_bytes(mk.np, mk.is_double ? 8 : 4, n);
    if (bytes > MPPI_MODEL_BLOCK_BYTES) return UNSUPPORTED("user model parameter block (parameters and tensor views) too large");
    for (int i = 0; i < n; ++i) {
        mk.tensor_dtype[i] = dtypes[i];
        mk.tensor_ndim[i] = ndims[i];
    }
    mk.n_tensors = n;
    mk.param_bytes = bytes;
    return MPPI_OK;
}

uint64_t mppi_plan_epoch(void* plan) {
    Plan* pl = reinterpret_cast<Plan*>(plan);
    if (pl == nullptr) return 0;
    const unsigned long long res = pl->res.armed ? pl->res_epoch_off + pl->res.seq : 0;
    return res > pl->epoch ? res : pl->epoch;
}

uint64_t mppi_resident_launches(void* plan) {
    Plan* pl = reinterpret_cast<Plan*>(plan);
    return pl == nullptr ? 0 : pl->res.launches;
}

int mppi_apply_partials(const MppiFusedParams* p, const void* partials, void* stream) {
    int rc = validate(p);
    if (rc) return rc;
    if (partials == nullptr || p->nominal_used == nullptr || p->stats == nullptr || p->U == nullptr || p->action_out == nullptr)
        return MPPI_ERR_BAD_ARG;
    cudaStream_t s = (cudaStream_t)stream;
    if (p->dtype == MPPI_F32) {
        switch (p->variant) {
            case MPPI_VARIANT_MPPI: return run_apply<float, V_MPPI>(p, partials, s);
            case MPPI_VARIANT_SMPPI: return run_apply<float, V_SMPPI>(p, partials, s);
            case MPPI_VARIANT_KMPPI: return run_apply<float, V_KMPPI>(p, partials, s);
        }
    } else {
        switch (p->variant) {
            case MPPI_VARIANT_MPPI: return run_apply<double, V_MPPI>(p, partials, s);
            case MPPI_VARIANT_SMPPI: return run_apply<double, V_SMPPI>(p, partials, s);
            case MPPI_VARIANT_KMPPI: return run_apply<double, V_KMPPI>(p, partials, s);
        }
    }
    return MPPI_ERR_BAD_ARG;
}

// two epoch parities of MPPI_XCHG_PARITY_WORDS flagged 8-byte words: world x records x 2 (R+2) words per command
uint64_t mppi_xchg_bytes(void) { return (uint64_t)2 * MPPI_XCHG_PARITY_WORDS * sizeof(unsigned long long); }

int mppi_xchg_create(void** mailbox, void* ipc_handle_out_64B) {
    if (mailbox == nullptr || ipc_handle_out_64B == nullptr) return MPPI_ERR_BAD_ARG;
    void* ptr = nullptr;
    CK(cudaMalloc(&ptr, mppi_xchg_bytes()));
    CK(cudaMemset(ptr, 0, mppi_xchg_bytes()));
    CK(cudaDeviceSynchronize());
    cudaIpcMemHandle_t h;
    CK(cudaIpcGetMemHandle(&h, ptr));
    static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
    memcpy(ipc_handle_out_64B, &h, 64);
    *mailbox = ptr;
    return MPPI_OK;
}

int mppi_xchg_open(const void* ipc_handle_64B, void** peer_mailbox) {
    if (ipc_handle_64B == nullptr || peer_mailbox == nullptr) return MPPI_ERR_BAD_ARG;
    cudaIpcMemHandle_t h;
    memcpy(&h, ipc_handle_64B, 64);
    void* ptr = nullptr;
    CK(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
    *peer_mailbox = ptr;
    return MPPI_OK;
}

int mppi_xchg_close(void* peer_mailbox) {
    if (peer_mailbox == nullptr) return MPPI_ERR_BAD_ARG;
    CK(cudaIpcCloseMemHandle(peer_mailbox));
    return MPPI_OK;
}

int mppi_xchg_destroy(void* mailbox) {
    if (mailbox == nullptr) return MPPI_ERR_BAD_ARG;
    CK(cudaFree(mailbox));
    return MPPI_OK;
}

int mppi_materialize(const MppiFusedParams* p, void* perturbed_action, void* noise, void* noise_theta, void* states,
                     void* stream) {
    int rc = validate(p);
    if (rc) return rc;
    if (p->nominal_used == nullptr) return MPPI_ERR_BAD_ARG;
    cudaStream_t s = (cudaStream_t)stream;
    if (states != nullptr && perturbed_action == nullptr) return MPPI_ERR_BAD_ARG;
    rc = p->dtype == MPPI_F32
             ? run_sample_any<float>(p, perturbed_action, noise, noise_theta, nullptr, nullptr, 0, 0, true, s)
             : run_sample_any<double>(p, perturbed_action, noise, noise_theta, nullptr, nullptr, 0, 0, true, s);
    if (rc || states == nullptr) return rc;
    const ModelKernels* mk = find_kernels(p, &rc);
    if (mk == nullptr) return rc;
    if ((rc = check_model_args(p, mk)) != MPPI_OK) return rc;
    return mk->is_double ? run_states<double>(mk, p, perturbed_action, states, s) : run_states<float>(mk, p, perturbed_action, states, s);
}

int mppi_rollout_states(const MppiFusedParams* p, const void* start_states, const void* actions, int64_t actions_stride,
                        int32_t n_rollouts, int32_t T, void* states_out, void* stream) {
    if (p == nullptr || start_states == nullptr || actions == nullptr || states_out == nullptr) return MPPI_ERR_BAD_ARG;
    if (p->struct_size != sizeof(MppiFusedParams)) return MPPI_ERR_ABI;
    if (n_rollouts < 1 || T < 1 || actions_stride < 0) return MPPI_ERR_BAD_ARG;
    if (p->dtype != MPPI_F32 && p->dtype != MPPI_F64) return MPPI_ERR_BAD_ARG;
    cudaStream_t s = (cudaStream_t)stream;
    int rc = MPPI_ERR_UNSUPPORTED;
    const ModelKernels* mk = find_kernels(p, &rc);
    if (mk == nullptr) return rc;
    if ((rc = check_model_tensors(mk, p->model_tensors, p->n_model_tensors)) != MPPI_OK) return rc;
    return mk->is_double ? run_rollout_states<double>(mk, p, start_states, actions, actions_stride, n_rollouts, T, states_out, s)
                         : run_rollout_states<float>(mk, p, start_states, actions, actions_stride, n_rollouts, T, states_out, s);
}

int mppi_sample_perturb(const MppiFusedParams* p, void* perturbed_action, void* noise, void* noise_theta, void* cost_init,
                        const void* override_rows, int32_t n_override, int32_t override_start, void* stream) {
    int rc = validate(p);
    if (rc) return rc;
    if (p->U == nullptr || perturbed_action == nullptr || noise == nullptr || p->nominal_used == nullptr) return MPPI_ERR_BAD_ARG;
    cudaStream_t s = (cudaStream_t)stream;
    return p->dtype == MPPI_F32 ? run_sample_any<float>(p, perturbed_action, noise, noise_theta, cost_init, override_rows,
                                                        n_override, override_start, false, s)
                                : run_sample_any<double>(p, perturbed_action, noise, noise_theta, cost_init, override_rows,
                                                         n_override, override_start, false, s);
}

int mppi_cost_accumulate(void* cost, const void* c, void* var_acc, int32_t M, int32_t K, double discount, int32_t dtype,
                         void* stream) {
    if (cost == nullptr || c == nullptr || M < 1 || K < 1) return MPPI_ERR_BAD_ARG;
    cudaStream_t s = (cudaStream_t)stream;
    const int BD = 256, nb = (K + BD - 1) / BD;
    if (dtype == MPPI_F32)
        cost_accumulate_kernel<float><<<nb, BD, 0, s>>>((float*)cost, (const float*)c, (float*)var_acc, M, K, (float)discount);
    else if (dtype == MPPI_F64)
        cost_accumulate_kernel<double><<<nb, BD, 0, s>>>((double*)cost, (const double*)c, (double*)var_acc, M, K, discount);
    else
        return MPPI_ERR_BAD_ARG;
    CK(cudaGetLastError());
    return MPPI_OK;
}

int mppi_softmin_update(const MppiFusedParams* p, const void* cost_total, const void* eps, void* stream) {
    int rc = validate(p);
    if (rc) return rc;
    if (cost_total == nullptr || eps == nullptr || p->nominal_used == nullptr || p->U == nullptr || p->action_out == nullptr ||
        p->stats == nullptr)
        return MPPI_ERR_BAD_ARG;
    cudaStream_t s = (cudaStream_t)stream;
    return p->dtype == MPPI_F32 ? run_softmin_any<float>(p, cost_total, eps, s) : run_softmin_any<double>(p, cost_total, eps, s);
}

int mppi_omega(const void* cost_total, void* omega_out, const void* stats, double lambda_, int32_t K, int32_t dtype,
               void* stream) {
    if (cost_total == nullptr || omega_out == nullptr || stats == nullptr || K < 1 || lambda_ <= 0) return MPPI_ERR_BAD_ARG;
    cudaStream_t s = (cudaStream_t)stream;
    const int BD = 256, nb = (K + BD - 1) / BD;
    if (dtype == MPPI_F32)
        omega_kernel<float><<<nb, BD, 0, s>>>((const float*)cost_total, (float*)omega_out, (const double*)stats,
                                              (float)(-(1.0 / lambda_)), K);
    else if (dtype == MPPI_F64)
        omega_kernel<double><<<nb, BD, 0, s>>>((const double*)cost_total, (double*)omega_out, (const double*)stats,
                                               -(1.0 / lambda_), K);
    else
        return MPPI_ERR_BAD_ARG;
    CK(cudaGetLastError());
    return MPPI_OK;
}

}  // extern "C"
