// mppi_model_tu.cu — one translation unit per (registered model, dtype): the fused command kernels
// (fused_command_kernel<Model, real, V, ...>, all variants and instantiations), the resident command kernels, the
// states kernel and the closed-loop plant step of that model — and, for the fp32 MLP, the wgmma kernels.  The unit contains no launch logic: it
// exports ONE symbol, mppi_host::model_kernels_<model>_<dtype>(), a table of kernel handles plus the parameter packer,
// which the generic host code in mppi_b200.cu (mppi_fused_host.cuh) works on.
//
// Compiled several times by pytorch_mppi_b200/build.py:
//     nvcc ... -DMPPI_TU_MODEL=<1 pendulum | 2 linear point | 3 pendulum MLP | 4 pendulum MLP ensemble> -DMPPI_TU_F64=<0|1> -c
// (user models are compiled at run time with NVRTC and registered with mppi_user_model_register — same kernels, same table).
#include "mppi_host.cuh"
#include "mppi_mlp_tc.cuh"

#ifndef MPPI_TU_MODEL
#error "MPPI_TU_MODEL must be defined (see pytorch_mppi_b200/build.py)"
#endif
#ifndef MPPI_TU_F64
#error "MPPI_TU_F64 must be 0 or 1"
#endif

#if MPPI_TU_F64
typedef double TuReal;
#define MPPI_TU_SUFFIX f64
#else
typedef float TuReal;
#define MPPI_TU_SUFFIX f32
#endif

#if MPPI_TU_MODEL == 1
typedef mppi::PendulumModel TuModel;
#define MPPI_TU_NAME pendulum
#elif MPPI_TU_MODEL == 2
typedef mppi::LinearPointModel TuModel;
#define MPPI_TU_NAME linear_point
#elif MPPI_TU_MODEL == 3
typedef mppi::PendulumMLPModel TuModel;
#define MPPI_TU_NAME pendulum_mlp
#elif MPPI_TU_MODEL == 4
typedef mppi::PendulumMLPEnsembleModel TuModel;
#define MPPI_TU_NAME pendulum_mlp_ensemble
#else
#error "unknown MPPI_TU_MODEL"
#endif

#define MPPI_TU_CAT2(a, b, c) model_kernels_##a##_##b
#define MPPI_TU_CAT(a, b) MPPI_TU_CAT2(a, b, )
#define MPPI_TU_GETTER MPPI_TU_CAT(MPPI_TU_NAME, MPPI_TU_SUFFIX)

namespace {

constexpr bool kIsMlp = MPPI_TU_MODEL == 3;
constexpr bool kIsEnsemble = MPPI_TU_MODEL == 4;   // copies at run time: no split-cost, batched or resident kernels
typedef TuModel::P<TuReal> TuParams;
static_assert(sizeof(TuParams) <= MPPI_MODEL_BLOCK_BYTES, "model parameter block too large");

void tu_load(const ModelKernels*, void* dst, const double* blob, const double* ext, int n_ext) {
    TuModel::load<TuReal>(*reinterpret_cast<TuParams*>(dst), blob, ext, n_ext);
}

template <int V> const void* split_kernel() {
    if constexpr (kIsMlp || kIsEnsemble) return nullptr;      // its step is the network; the cost is nothing
    else return (const void*)fused_command_kernel<TuModel, TuReal, V, false, true>;
}
template <int V> const void* split_ll_kernel() {
    if constexpr (kIsMlp || kIsEnsemble) return nullptr;
    else return (const void*)fused_command_kernel_ll<TuModel, TuReal, V>;
}
const void* batched_kernel() {
    if constexpr (kIsEnsemble) return nullptr;                // MPPI_Batched has no rollout_samples
    else return (const void*)fused_command_kernel<TuModel, TuReal, V_MPPI, true>;
}
template <int V> const void* resident_kernel() {
    if constexpr (kIsMlp || kIsEnsemble) return nullptr;
    else return (const void*)resident_command_kernel<TuModel, TuReal, V>;
}
const void* stamped_resident_kernel() {
    if constexpr (MPPI_TU_MODEL == 1 && !MPPI_TU_F64) return (const void*)resident_command_kernel<TuModel, TuReal, V_MPPI, true>;
    else return nullptr;
}
// global-tile kernels (MPPI_FLAG_GLOBAL_TILE): not for the MLP models, whose kernels fix their own tiles
template <int V> const void* gtile_kernel() {
    if constexpr (kIsMlp || kIsEnsemble) return nullptr;
    else return (const void*)fused_command_kernel_gtile<TuModel, TuReal, V, false>;
}
const void* gtile_batched_kernel() {
    if constexpr (kIsMlp || kIsEnsemble) return nullptr;
    else return (const void*)fused_command_kernel_gtile<TuModel, TuReal, V_MPPI, true>;
}
// the plant step of closed-loop episodes: not for the MLP models (a learned model is not the plant it approximates)
const void* plant_kernel() {
    if constexpr (kIsMlp || kIsEnsemble) return nullptr;
    else return (const void*)plant_step_kernel<TuModel, TuReal>;
}
// MPPI_Batched with per-environment model parameters: not for the MLP models (their 1,250-weight blocks)
template <bool GTILE> const void* env_kernel() {
    if constexpr (kIsMlp || kIsEnsemble) return nullptr;
    else return (const void*)fused_command_kernel_env<TuModel, TuReal, GTILE>;
}
template <int V, int SPLIT, int FAST> const void* tc_kernel() {
    if constexpr (kIsMlp && !MPPI_TU_F64) return (const void*)mlp_tc_command_kernel<V, SPLIT, FAST>;
    else if constexpr (kIsEnsemble && !MPPI_TU_F64) return (const void*)mlp_ens_tc_command_kernel<V, SPLIT, FAST>;
    else return nullptr;
}

const ModelKernels g_kernels = {
    TuModel::NX, TuModel::NU, MPPI_TU_F64, kIsMlp ? 1 : (kIsEnsemble ? 2 : 0), 0, (int)sizeof(TuParams), tu_load,
    {(const void*)fused_command_kernel<TuModel, TuReal, V_MPPI, false>, (const void*)fused_command_kernel<TuModel, TuReal, V_SMPPI, false>,
     (const void*)fused_command_kernel<TuModel, TuReal, V_KMPPI, false>},
    {split_kernel<V_MPPI>(), split_kernel<V_SMPPI>(), split_kernel<V_KMPPI>()},
    {split_ll_kernel<V_MPPI>(), split_ll_kernel<V_SMPPI>(), split_ll_kernel<V_KMPPI>()},
    batched_kernel(),
    {resident_kernel<V_MPPI>(), resident_kernel<V_SMPPI>(), resident_kernel<V_KMPPI>()},
    stamped_resident_kernel(),
    (const void*)states_kernel<TuModel, TuReal>,
    {gtile_kernel<V_MPPI>(), gtile_kernel<V_SMPPI>(), gtile_kernel<V_KMPPI>()},
    gtile_batched_kernel(),
    {{{tc_kernel<V_MPPI, 1, 0>(), tc_kernel<V_MPPI, 1, 1>()}, {tc_kernel<V_MPPI, 0, 0>(), tc_kernel<V_MPPI, 0, 1>()}},
     {{tc_kernel<V_SMPPI, 1, 0>(), tc_kernel<V_SMPPI, 1, 1>()}, {tc_kernel<V_SMPPI, 0, 0>(), tc_kernel<V_SMPPI, 0, 1>()}},
     {{tc_kernel<V_KMPPI, 1, 0>(), tc_kernel<V_KMPPI, 1, 1>()}, {tc_kernel<V_KMPPI, 0, 0>(), tc_kernel<V_KMPPI, 0, 1>()}}},
    nullptr, 0, 0, {}, {},
    plant_kernel(),
    env_kernel<false>(),
    env_kernel<true>(),
};

}  // namespace

namespace mppi_host {
const ModelKernels* MPPI_TU_GETTER() { return &g_kernels; }
}  // namespace mppi_host
