// mppi_fused_host.cuh — kernel selection, launch geometry and plans of the fused command, for ANY model: the
// model enters through a ModelKernels descriptor (kernel handles + parameter packing), so this is compiled once, in
// mppi_b200.cu, and serves the registry models and NVRTC-compiled user models alike.
#pragma once
#include "mppi_host.cuh"

namespace {

// ---- fused command ----------------------------------------------------------------------------
// PENDULUM_MLP in fp32 with model_params[3] != 0: the wgmma kernel (mppi_mlp_tc.cuh).  One CTA = 256 threads = 128
// samples (two threads per sample) = two warpgroups of 64 accumulator rows; it does not take part in PDL.
inline bool select_tensor_core_route(const ModelKernels* mk, const MppiFusedParams* p, MppiFusedParams& p_tc, const void*& kernel) {
    if (mk->is_mlp && !mk->is_double) {
        int mode = (int)p->model_params[3];            // 1: hi/lo-split bf16 operands ("3 x bf16"), 2: plain bf16, 3: automatic
        // automatic (the Python default): the tensor-core kernel with split operands — the parity route — wherever it
        // exists (fp32, one environment)
        if (mode == 3) mode = 1;
        const int fast = p->model_params[2] != 0.0 ? 1 : 0;
        if ((mode == 1 || mode == 2) && p->n_env <= 1 && mk->tc[p->variant][mode - 1][fast] != nullptr) {
            p_tc = *p;
            p_tc.block_threads = 128;                   // samples per tile
            p_tc.threads_per_sample = 2;
            p_tc.flags &= ~(uint32_t)MPPI_FLAG_PDL;
            kernel = mk->tc[p->variant][mode - 1][fast];
            // co-residency is bounded by shared memory: ask for the largest carve-out
            cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
            return true;
        }
    }
    return false;
}

// ---- kernel + launch geometry of one fused command -------------------------------------------------------------------
// What is decided here, once per plan:
//   kernel     fused_command_kernel<Model, real, V, batched, split>  (or the wgmma kernel, select_tensor_core_route)
//   geometry   tile size / helper threads / grid (plan_geometry), planned for K_geom samples on sharded controllers so
//              that every rank launches the same grid
//   split      MPPI_FLAG_SPLIT_COST honoured: problems small enough to run with helper threads (threads_per_sample > 1)
//              take the split-cost rollout if its per-step state buffer fits in shared memory
//   cluster    thread-block-cluster size of the warp-fold tail: 8 / 4 / 2 when the whole grid is one wave of at most
//              one CTA per SM and all its clusters are co-resident (cudaOccupancyMaxActiveClusters), else 1
//   npub       sharded controllers: the records a rank publishes to its peers per command — its cluster records when
//              their staging (world x clusters x (R+2) doubles) is small (direct mode), else its one combined record
//   ll         split-cost plans of one GPU whose clusters all publish to its own mailbox (LL mode) run
//              fused_command_kernel_ll, the instantiation whose tail is that one path, inlined (mppi_fused.cuh, warp_tail)
//   gtile      MPPI_FLAG_GLOBAL_TILE: fused_command_kernel_gtile, tiles in per-CTA workspace slices — single loop, one GPU,
//              no clusters (the padded grid of a cluster would outgrow the slices ws_gtile_bytes sizes), and ticket mode
//              where the finisher's LL staging does not fit next to the (R+2)-sized records
struct FusedChoice {
    const void* kernel;
    Geometry g;
    int split;
    int ll;
    int gtile;
};

// the reasons a global-tile plan is refused, before any CUDA call (nullptr: none)
inline const char* gtile_refusal(const ModelKernels* mk, const MppiFusedParams* p) {
    if (mk != nullptr && mk->is_mlp)
        return "global-tile plans: the PendulumMLP kernels fix their own tiles (tile_memory='shared' only)";
    if (p->world > 1 || (p->flags & MPPI_FLAG_EXPORT_PARTIAL))
        return "global-tile plans: not available on sharded controllers (the peer mailbox caps T*nu at 1024)";
    return nullptr;
}

// the rank records of a command are exchanged with peers inside the kernel (else they stay in this GPU's own mailbox)
inline bool sharded_in_kernel(const MppiFusedParams* p) {
    bool any_peer = false;
    for (int g = 0; g < MPPI_MAX_RANKS; ++g) any_peer = any_peer || p->peer_slots[g] != nullptr;
    return p->world > 1 && any_peer && !(p->flags & MPPI_FLAG_EXPORT_PARTIAL);
}

template <typename real>
int choose_fused(const ModelKernels* mk, const MppiFusedParams*& p, MppiFusedParams& p_tc, FusedChoice& c) {
    if (p->nx != mk->nx || p->nu != mk->nu) return MPPI_ERR_BAD_ARG;
    const int V = p->variant;
    const bool batched = p->n_env > 1;
    if (batched && (V != V_MPPI || p->world > 1)) return UNSUPPORTED("batched environments: MPPI variant, single GPU only");
    const bool gtile = (p->flags & MPPI_FLAG_GLOBAL_TILE) != 0;
    if (gtile) {
        if (const char* why = gtile_refusal(mk, p)) return UNSUPPORTED(why);
    }
    const void* kernel = gtile ? (batched ? mk->gtile_batched : mk->gtile[V]) : (batched ? mk->batched : mk->fused[V]);
    if (kernel == nullptr) return UNSUPPORTED("this model was built without the kernel of this controller variant");
    const bool tc_route = !gtile && select_tensor_core_route(mk, p, p_tc, kernel);
    if (tc_route) p = &p_tc;
    const int R = rows_of(p);
    const int world = p->world <= 0 ? 1 : p->world;
    const bool sharded = sharded_in_kernel(p);
    MppiFusedParams pg = *p;
    if (p->K_geom > p->K) pg.K = p->K_geom;
    Geometry g;
    int rc;
    const int xst1 = sharded ? world * (R + 2) : 0;          // staging of the rank-record exchange
    // SMPPI: effective-noise tile, KMPPI: interpolated-trajectory tile (the tensor-core kernels have neither)
    const int tile2 = V != V_MPPI && !tc_route;
    // the ensemble's tensor-core kernel keeps every copy's network and step buffers behind the layout
    const int ens_bytes = tc_route && mk->is_mlp == 2 ? PendulumMLPEnsembleModel::tc_smem_bytes(p->rollout_samples) : 0;
    rc = plan_geometry<real>(kernel, &pg, layout_extra(tile2, 0, 1, xst1), false, g, ens_bytes, gtile);
    if (rc) return rc;
    int split = 0;
    if (mk->split[V] != nullptr && !gtile) {      // (the MLP has none: its step is the network, the cost is nothing)
        if (!batched && (p->flags & MPPI_FLAG_SPLIT_COST) && g.tps > 1) {
            const void* k2 = mk->split[V];
            MppiFusedParams p2 = pg;
            p2.block_threads = g.BS;
            p2.threads_per_sample = g.tps;
            p2.grid_blocks = g.nb;
            Geometry g2;
            if (plan_geometry<real>(k2, &p2, layout_extra(tile2, mk->nx, 1, xst1), false, g2) == MPPI_OK &&
                g2.BS == g.BS && g2.tps == g.tps) {
                kernel = k2;
                g = g2;
                split = 1;
            }
        }
    }
    // ---- cluster size and exchange mode ------------------------------------------------------------------------------
    DevInfo di;
    rc = get_dev_info(di);
    if (rc) return rc;
    int want = 8;
    if (const char* e = getenv("MPPI_B200_CLUSTER")) want = atoi(e);
    cudaFuncAttributes fa;
    CK(cudaFuncGetAttributes(&fa, kernel));
    const int envs = batched ? p->n_env : 1;
    const bool may_ll = split && !sharded && !(p->flags & MPPI_FLAG_EXPORT_PARTIAL) && mk->split_ll[V] != nullptr;
    const void* chosen = kernel;
    g.cluster = 0;
    g.npub = 1;
    for (int cs = 8; cs >= 1; cs >>= 1) {
        if (cs > want && cs > 1) continue;
        if (gtile && cs > 1) continue;
        const int nbp = (g.nb + cs - 1) / cs * cs;
        if (cs > 2 && nbp > di.sm_count) continue;                        // 8 / 4: one wave of at most one CTA per SM (pairs pack anywhere)
        if (cs > 1 && (g.nb < 2 || nbp > di.sm_count * g.occ)) continue;
        const int NC = nbp / cs;
        // LL mode: the finisher (leader of cluster 0) stages every rank's cluster records: xw x NC x (R+2) doubles
        const int xw = sharded ? world : 1;
        int npub = 1;
        if (NC > 1 && (long long)xw * NC * (R + 2) * 8 <= MPPI_LL_STAGE_BYTES) npub = NC;
        if (const char* e = getenv("MPPI_B200_XCHG_DIRECT"))
            if (atoi(e) == 0) npub = 1;
        int xst = fused_xstage_doubles(sharded, world, npub, R);
        const void* kc = may_ll && NC > 1 && npub == NC ? mk->split_ll[V] : kernel;
        CK(cudaFuncGetAttributes(&fa, kc));
        const int dyn_limit = di.max_smem_optin - (int)fa.sharedSizeBytes;
        if (kc != kernel) CK(cudaFuncSetAttribute(kc, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn_limit));
        int smem = make_layout<real>(p->variant, p->T, p->nu, p->S, R, g.BD, g.BS, fused_layout_nb(NC, npub),
                                     layout_extra(tile2, split ? mk->nx : 0, cs, xst), gtile).total + ens_bytes;
        if (gtile && smem > dyn_limit && npub > 1) {       // ticket mode: the cluster records stay in the L2 workspace
            npub = 1;
            xst = fused_xstage_doubles(sharded, world, npub, R);
            smem = make_layout<real>(p->variant, p->T, p->nu, p->S, R, g.BD, g.BS, fused_layout_nb(NC, npub),
                                     layout_extra(tile2, 0, cs, xst), true).total;
        }
        if (smem > dyn_limit) continue;
        if (cs > 1) {
            cudaLaunchConfig_t cfg;
            cudaLaunchAttribute at[3];
            launch_config(cfg, at, nbp, g.BD, smem, nullptr, (p->flags & MPPI_FLAG_PDL) != 0, envs, cs);
            int max_clusters = 0;
            if (cudaOccupancyMaxActiveClusters(&max_clusters, kc, &cfg) != cudaSuccess) {
                cudaGetLastError();
                continue;
            }
            if (getenv("MPPI_B200_DEBUG_GEOM"))
                fprintf(stderr, "[mppi_b200] cluster %d: grid %d, smem %d, max active clusters %d (need %d)\n", cs, nbp, smem, max_clusters, NC * envs);
            if (max_clusters < NC * envs) continue;                       // a cluster left for a second wave doubles the time
        }
        g.cluster = cs;
        g.nb = nbp;
        g.smem = smem;
        g.npub = npub;
        g.regs = fa.numRegs;
        chosen = kc;
        break;
    }
    if (g.cluster == 0)
        return gtile ? UNSUPPORTED("global-tile plan: the per-CTA vectors (nominal sequence, softmin records) do not fit in shared memory")
                     : UNSUPPORTED("shared-memory tile does not fit");
    c = FusedChoice{chosen, g, split, chosen != kernel, gtile ? 1 : 0};
    return MPPI_OK;
}

template <typename real> void finish_kargs(const MppiFusedParams* p, const FusedChoice& c, KArgs<real>& a) {
    fill_kargs<real>(p, a, c.g.BS, c.g.nb, c.g.tps);
    a.xchg_npub = c.g.npub > 0 ? c.g.npub : 1;
}

// MppiLaunchInfo of the plan these parameters would make (no launch)
template <typename real> int query_fused(const ModelKernels* mk, const MppiFusedParams* p, MppiLaunchInfo* info) {
    MppiFusedParams p_tc;
    FusedChoice c;
    int rc = choose_fused<real>(mk, p, p_tc, c);
    if (rc) return rc;
    DevInfo di;
    if ((rc = get_dev_info(di)) != MPPI_OK) return rc;
    KArgs<real> a;
    finish_kargs<real>(p, c, a);
    const Geometry& g = c.g;
    info->block_threads = g.BD;
    info->threads_per_sample = g.tps;
    info->grid_blocks = g.nb;
    info->smem_bytes = g.smem;
    info->regs_per_thread = g.regs;
    info->max_blocks_per_sm = g.occ;
    info->sm_count = di.sm_count;
    info->workspace_bytes = ws_bytes(max_planned_grid(p, di.sm_count), rows_of(p)) + (c.gtile ? ws_gtile_bytes(p, di.sm_count) : 0);
    info->tma_staging = a.tma_ok;
    info->split_cost = c.split;
    info->cluster_size = g.cluster;
    info->xchg_records = g.npub;
    info->ll_tail = c.ll;
    info->global_tile = c.gtile;
    return MPPI_OK;
}

// Every check of the buffers and strides a command uses happens here, once per plan.
template <typename real> int build_plan(const ModelKernels* mk, const MppiFusedParams* p, Plan* pl) {
    const bool batched = p->n_env > 1;
    const int V = p->variant;
    MppiFusedParams p_tc;
    FusedChoice c;
    int rc = choose_fused<real>(mk, p, p_tc, c);
    if (rc) return rc;
    pl->g = c.g;
    if (p->U == nullptr || p->cost_total == nullptr || p->nominal_used == nullptr || p->stats == nullptr || p->workspace == nullptr)
        return MPPI_ERR_BAD_ARG;
    const uint64_t need_ws = ws_bytes(pl->g.nb, rows_of(p)) + (c.gtile ? ws_gtile_plan_bytes(p, pl->g.nb, pl->g.BS, V != V_MPPI) : 0);
    if (p->workspace_bytes < need_ws) return MPPI_ERR_WORKSPACE;
    if (batched && (p->env_ws_stride < need_ws || p->env_ws_stride % MPPI_WS_ALIGN != 0 ||
                    p->workspace_bytes < p->env_ws_stride * (uint64_t)p->n_env || p->env_u_stride < p->T * p->nu))
        return MPPI_ERR_WORKSPACE;
    if (mk->param_bytes > (int)sizeof(pl->mparams)) return UNSUPPORTED("model parameter block too large");
    KArgs<real>* a = reinterpret_cast<KArgs<real>*>(pl->kargs);
    finish_kargs<real>(p, c, *a);
    if (a->world > 1 && rows_of(p) > MPPI_XCHG_MAX_R) return UNSUPPORTED("T*nu exceeds the peer mailbox record size");
    if (a->export_partial && p->partial_out == nullptr) return MPPI_ERR_BAD_ARG;
    load_model_params(mk, p, pl->mparams);
    pl->mk = mk;
    pl->kernel = c.kernel;
    pl->res_kernel = nullptr;
    // resident mode runs the split-cost rollout with one tile per CTA: exactly the single-GPU plans that took it, with
    // the launch route's grid and cluster size (mppi_resident.cuh)
    if (c.split && !batched && !a->export_partial && a->world == 1 && a->n_tiles <= pl->g.nb && pl->g.nb <= a->n_tiles + pl->g.cluster - 1) {
        pl->res_kernel = mk->resident[V];
        // the one instantiation with %globaltimer stamps (a profiling aid, scripts/resident_timeline.py)
        if (pl->res_kernel != nullptr && p->debug_clocks != nullptr && V == V_MPPI && mk->resident_stamped != nullptr)
            pl->res_kernel = mk->resident_stamped;
    }
    pl->is_double = sizeof(real) == 8;
    pl->nx = mk->nx;
    pl->upc_nu = p->u_per_command * p->nu;
    pl->pdl = (p->flags & MPPI_FLAG_PDL) ? 1 : 0;
    pl->epoch = p->epoch;
    pl->res_epoch_off = 0;
    pl->host_epoch = p->host_epoch;      // monotonic across re-plans: a stale mailbox tag of an earlier plan can never match
    pl->p = *p;
    // mppi_plan_set_model_params re-packs the whole block from pl->p: the tensor references it reads are the plan's own
    if (mk->n_tensors > 0) memcpy(pl->tensors, p->model_tensors, sizeof(MppiTensorRef) * mk->n_tensors);
    pl->p.model_tensors = pl->tensors;
    return MPPI_OK;
}

template <typename real>
int launch_states(const ModelKernels* mk, const MppiFusedParams* p, KArgs<real>& a, int n, const void* actions, void* states,
                  long long stride, cudaStream_t stream, int copies = 1) {
    alignas(16) unsigned char mp[MPPI_MODEL_BLOCK_BYTES];
    if (mk->param_bytes > (int)sizeof(mp)) return UNSUPPORTED("model parameter block too large");
    load_model_params(mk, p, mp);
    const real* pa = (const real*)actions;
    real* st = (real*)states;
    void* argv[5] = {(void*)&pa, (void*)&st, (void*)&a, (void*)mp, (void*)&stride};
    cudaError_t e = cudaLaunchKernel(mk->states, dim3((n + 127) / 128, copies), dim3(128), argv, 0, stream);
    if (e != cudaSuccess) return cuda_fail(e, "states launch");
    return MPPI_OK;
}

// states along the rollouts of the last command's perturbed actions (mppi.py:307-322); every copy's with
// rollout_samples = M > 1 (mppi.py:366): (M,K,T,nx)
template <typename real>
int run_states(const ModelKernels* mk, const MppiFusedParams* p, const void* pa, void* states, cudaStream_t stream) {
    if (p->nx != mk->nx || p->nu != mk->nu) return MPPI_ERR_BAD_ARG;
    KArgs<real> a;
    fill_kargs<real>(p, a, 128, 1);
    return launch_states<real>(mk, p, a, p->K, pa, states, (long long)p->T * p->nu, stream,
                               p->rollout_samples > 1 ? p->rollout_samples : 1);
}

// get_rollouts (mppi.py:425-448): n start states, each rolled through an action sequence
template <typename real>
int run_rollout_states(const ModelKernels* mk, const MppiFusedParams* p, const void* start_states, const void* actions, long long stride,
                       int n, int T, void* states, cudaStream_t stream) {
    if (p->nx != mk->nx || p->nu != mk->nu) return MPPI_ERR_BAD_ARG;
    KArgs<real> a;
    memset(&a, 0, sizeof(a));
    a.nm.u_scale = (real)p->u_scale;
    a.K = n;
    a.T = T;
    a.state_dev = (const real*)start_states;
    a.state_per_sample = 1;
    return launch_states<real>(mk, p, a, n, actions, states, stride, stream);
}

}  // namespace

