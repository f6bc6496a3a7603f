/*
 * mppi_b200.h — C ABI of the H100-native MPPI rollout-and-reweight engine.
 *
 * The reference (UM-ARM-Lab/pytorch_mppi) is pure Python and has no FFI; the drop-in boundary is
 * its Python class API (SURVEY.md §8b).  This header is the boundary *below* that API: the Python
 * controllers in pytorch_mppi_b200/ bind these symbols with ctypes (INTEGRATION.md shows the stub a
 * reference maintainer would add to mppi.py to do the same).  Every entry point
 *   - takes plain pointers / sizes / a cudaStream_t passed as void*  (no torch types),
 *   - never allocates or frees caller-visible memory (buffers are caller-owned device memory),
 *   - launches asynchronously on the given stream and returns 0 or a negative MppiStatus,
 *   - is not re-entrant per controller (one controller <-> one stream, as the reference).
 *
 * Each entry point cites the reference code it replaces (file:line into
 * reference src/pytorch_mppi/mppi.py).
 */
#ifndef MPPI_B200_H
#define MPPI_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MPPI_B200_ABI_VERSION 3

#define MPPI_MAX_NU 4            /* control dimension supported by the fused registry            */
#define MPPI_MAX_NX 8            /* state dimension supported by the fused registry              */
#define MPPI_MODEL_PARAM_DOUBLES 48
#define MPPI_MAX_RANKS 8         /* GPUs of one NVSwitch box                                     */
#define MPPI_MAX_COPIES 8        /* rollout_samples of a user model compiled with copies (registers) */
#define MPPI_MAX_MODEL_TENSORS 8 /* device tensors a user model's bodies may read                */

typedef enum MppiStatus {
    MPPI_OK = 0,
    MPPI_ERR_BAD_ARG = -1,        /* null pointer / out-of-range dimension / unknown enum        */
    MPPI_ERR_UNSUPPORTED = -2,    /* (model, variant, dtype) not in the compiled registry        */
    MPPI_ERR_WORKSPACE = -3,      /* workspace too small (see mppi_fused_query)                  */
    MPPI_ERR_CUDA = -4,           /* a CUDA runtime call failed; see mppi_last_cuda_error()      */
    MPPI_ERR_ABI = -5,            /* struct_size does not match this library                     */
    MPPI_ERR_TIMEOUT = -6         /* peer exchange timed out (reported via the status word)      */
} MppiStatus;

typedef enum MppiVariant { MPPI_VARIANT_MPPI = 0, MPPI_VARIANT_SMPPI = 1, MPPI_VARIANT_KMPPI = 2 } MppiVariant;
typedef enum MppiDType { MPPI_F32 = 0, MPPI_F64 = 1, MPPI_U8 = 2, MPPI_I32 = 3 } MppiDType;   /* U8 / I32: tensor elements only */

/* A read-only device tensor a user model's bodies read (CudaModel(tensors=...)): contiguous, row-major, element type
 * `dtype` (MPPI_F32 / MPPI_F64 / MPPI_U8 / MPPI_I32), 1 <= ndim <= 4, shape[d] > 0 for d < ndim, at most 2^31 - 1
 * elements.  Its data must outlive every command that may read it. */
typedef struct MppiTensorRef {
    const void* data;
    int32_t dtype;
    int32_t ndim;
    int64_t shape[4];
} MppiTensorRef;

/* Registry of analytic models whose dynamics + running cost are compiled into the fused kernel.
 * (The reference takes arbitrary Python callables, mppi.py:147-157; arbitrary callables use the
 * per-step entry points further down.) */
typedef enum MppiModel {
    MPPI_MODEL_PENDULUM = 1,      /* reference tests/pendulum.py:30-60                      */
    MPPI_MODEL_LINEAR_POINT = 2,  /* tests/test_mppi.py:24-51 and tests/smooth_mppi.py:29-142    */
    MPPI_MODEL_PENDULUM_MLP = 3,  /* tests/pendulum_approximate.py:47-67 (3-32-32-2 tanh residual MLP) */
    MPPI_MODEL_PENDULUM_MLP_ENSEMBLE = 4,  /* rollout_samples = M networks of PENDULUM_MLP's shape, one per copy
                                              (a bootstrapped ensemble of learned dynamics); weights in model_weights */
    MPPI_MODEL_USER = 100         /* a user-written model compiled at run time and registered with
                                     mppi_user_model_register (see pytorch_mppi_b200.models.CudaModel): the
                                     reference accepts arbitrary Python callables (mppi.py:63-64) — this is the
                                     compiled equivalent for analytic dynamics/costs                           */
} MppiModel;

/* model_params layouts (doubles):
 *  PENDULUM     : [0]=g [1]=m [2]=l [3]=dt [4]=max_torque [5]=max_speed [6]=w_thdot(0.1)
 *  LINEAR_POINT : [0..3]=B(2x2 row-major) [4..5]=goal [6..9]=Q [10]=has_R [11..14]=R
 *                 [15]=terminal_scale [16]=n_hills(<=3) then per hill h at 17+7h:
 *                 Qh(4) centre(2) height(1)
 *  PENDULUM_MLP : [0]=max_torque [1]=w_thdot [2]=tanh_mode(0 exp-based, 1 MUFU.TANH) [3]=tensor_cores (0 = FFMA kernel;
 *                 wgmma kernel, fp32 accumulate: 1 = hi/lo-split bf16 operands, 2 = plain bf16; 3 = automatic:
 *                 mode 1 wherever that kernel exists — fp32, one environment — else the FFMA kernel); the 1,250 weights go in
 *                 model_params_ext: W1 (32x3 row-major), b1 (32), W2 (32x32), b2 (32), W3 (2x32), b3 (2)
 *  PENDULUM_MLP_ENSEMBLE : [0..3] as PENDULUM_MLP.  The M = rollout_samples (2..MPPI_MAX_COPIES) networks' weights are
 *                 NOT in model_params_ext but in the device buffer model_weights: (M, 1250) in the controller dtype, row
 *                 m = network m in PENDULUM_MLP's model_params_ext order.  Copy m of every sample is rolled out through
 *                 network m.  No split-cost, batched or resident kernels.
 */

enum {
    MPPI_FLAG_SHIFT = 1u << 0,            /* shift_nominal_trajectory before sampling (mppi.py:232-238, 249-250) */
    MPPI_FLAG_NULL_ACTION = 1u << 1,      /* sample_null_action: global sample 0 is zeroed before the clamp (:390-392) */
    MPPI_FLAG_ABS_COST = 1u << 2,         /* noise_abs_cost (:190-191, 196-197)                                  */
    MPPI_FLAG_DIAG_SIGMA = 1u << 3,       /* diagonal covariance fast path (:131-136, 188-193, 204-205)          */
    MPPI_FLAG_STATE_DEVICE = 1u << 4,     /* read the state from state_dev instead of the by-value copy          */
    MPPI_FLAG_STATE_PER_SAMPLE = 1u << 5, /* state_dev is (K,nx): one start state per sample (:302-303)          */
    MPPI_FLAG_EXPORT_PARTIAL = 1u << 6,   /* multi-GPU, library collective: write this rank's (beta,eta,V) to
                                             partial_out and do NOT update U (mppi_apply_partials finishes)    */
    MPPI_FLAG_NOMINAL_PADDED = 1u << 7,   /* U (and A) are 16-byte aligned allocations padded to a multiple of
                                             16 bytes: lets the kernel stage them with one TMA bulk copy        */
    MPPI_FLAG_PDL = 1u << 8,              /* programmatic dependent launch: the kernel may start while the previous
                                             kernel on the stream is finishing; it draws its Philox normals (shared
                                             memory only) and touches global memory only after griddepcontrol.wait */
    MPPI_FLAG_WIDE_REGS = 1u << 10,       /* retired (accepted and ignored; the bit stays reserved): round 1's opt-in
                                             instantiation without the 64-register cap.  The split-cost kernels have the
                                             whole register file anyway, the single-loop kernels of large K need the cap. */
    MPPI_FLAG_SPLIT_COST = 1u << 9,       /* small problems (threads_per_sample > 1): the rollout thread runs the bare state
                                             recurrence, the sample's helper threads evaluate the T running costs in
                                             parallel from the stored states, summed in the reference's order (same
                                             operations and rounding as the single-loop rollout; see mppi_fused.cuh)  */
    MPPI_FLAG_GLOBAL_TILE = 1u << 11      /* keep the noise tiles (and KMPPI's W / Wshift) in a per-CTA slice of the
                                             workspace instead of shared memory: horizons whose tile does not fit.  Read
                                             by mppi_fused_query, mppi_plan_create, mppi_sample_perturb,
                                             mppi_softmin_update and mppi_materialize; single-loop kernels (split-cost
                                             off), one GPU, not for resident mode or the PendulumMLP models           */
};

/* One `command()` of a registered analytic model: replaces, in one launch,
 *   shift_nominal_trajectory            mppi.py:232-238 (SMPPI :489-493, KMPPI :617-619)
 *   _compute_perturbed_action_and_noise mppi.py:375-385 (SMPPI :539-552, KMPPI :657-670)
 *   _compute_rollout_costs_single       mppi.py:297-332
 *   _compute_total_cost_batch           mppi.py:407-417 (SMPPI :554-570)
 *   _compute_weighting                  mppi.py:254-259
 *   the einsum update in _command       mppi.py:268-270 (SMPPI :527-531, KMPPI :679-682)
 * All pointers are device pointers of element type `dtype` unless noted. */
typedef struct MppiFusedParams {
    uint32_t struct_size;        /* sizeof(MppiFusedParams), ABI check                                  */
    int32_t variant;             /* MppiVariant                                                         */
    int32_t model;               /* MppiModel                                                           */
    int32_t dtype;               /* MppiDType                                                           */
    int32_t K;                   /* samples rolled out by THIS rank                                     */
    int32_t T;                   /* horizon                                                             */
    int32_t nx, nu;              /* must match the model                                                */
    int32_t S;                   /* KMPPI: number of support points (else 0)                            */
    int32_t u_per_command;       /* rows of the action sequence copied to action_out                    */
    uint32_t flags;              /* MPPI_FLAG_*                                                         */
    int32_t block_threads;       /* samples per CTA tile (multiple of 32, <= 512); 0 = library default  */
    int32_t grid_blocks;         /* 0 = library default (<= SMs * resident CTAs)                        */
    int32_t threads_per_sample;  /* 1/2/4 threads share one sample's sampling work; 0 = library default */
    int64_t k_offset;            /* global index of this rank's first sample (keys the RNG, null action)*/
    uint64_t seed, offset;       /* Philox4x32-10 key / counter base (see oracle/philox_oracle.py)      */
    double lambda_;              /* temperature                                                         */
    double u_scale;
    double noise_mu[MPPI_MAX_NU];
    double chol[MPPI_MAX_NU * MPPI_MAX_NU];      /* row-major lower Cholesky factor L of noise_sigma; diag: sqrt on the diagonal */
    double sigma_inv[MPPI_MAX_NU * MPPI_MAX_NU]; /* row-major inverse covariance                                         */
    double u_min[MPPI_MAX_NU], u_max[MPPI_MAX_NU];
    double u_init[MPPI_MAX_NU];
    double action_min[MPPI_MAX_NU], action_max[MPPI_MAX_NU];   /* SMPPI (mppi.py:464-477)              */
    double w_action_seq_cost, delta_t;                         /* SMPPI (mppi.py:456-459)              */
    double model_params[MPPI_MODEL_PARAM_DOUBLES];
    double state[MPPI_MAX_NX];   /* start state by value: no host->device copy on the hot path          */
    const void* state_dev;       /* optional device state, (nx) or (K,nx)                               */
    void* U;                     /* (T,nu) in/out nominal controls (SMPPI: control derivative)          */
    void* A;                     /* SMPPI: (T,nu) in/out action_sequence                                */
    void* theta;                 /* KMPPI: (S,nu) in/out control points                                 */
    const void* W;               /* KMPPI: (T,S)  k(Hs,Tk) k(Tk,Tk)^-1                                  */
    const void* Wshift;          /* KMPPI: (S,S)  k(Tk+1,Tk) k(Tk,Tk)^-1                                */
    void* cost_total;            /* (K) out                                                             */
    void* action_out;            /* (u_per_command,nu) out                                              */
    void* nominal_used;          /* out, 3*(T*nu) elements: U | A | theta as used for sampling (post-shift,
                                    pre-update); lets noise/perturbed_action be materialised lazily     */
    void* stats;                 /* out, 4 doubles: beta, eta, (reserved), status word                  */
    const void* z;               /* optional injected standard normals (K,T,nu) / KMPPI (K,S,nu); NULL = Philox */
    void* z_out;                 /* optional: the standard normals actually used, same shape            */
    void* workspace;             /* caller-owned scratch, zero-initialised ONCE by the caller           */
    uint64_t workspace_bytes;
    /* ---- multi-GPU (K sharded over ranks; SURVEY.md §8e) ---- */
    int32_t rank, world;
    uint64_t epoch;              /* strictly increasing per command; keys the peer-exchange flags        */
    void* peer_slots[MPPI_MAX_RANKS];   /* in-kernel exchange: pointer to every rank's mailbox (own included),
                                           from mppi_xchg_*; all NULL = no in-kernel exchange            */
    void* partial_out;           /* MPPI_FLAG_EXPORT_PARTIAL: (2 + R) doubles out                        */
    /* ---- batched environments (MPPI_Batched, mppi.py:691-873): n_env independent problems sharing one noise
     * stream, launched as gridDim.y = n_env.  Buffers are (n_env, ...) with these strides; state_dev is
     * (n_env, nx) on the device.  n_env <= 1 means a single problem.  MPPI variant only. */
    int32_t n_env;
    int32_t env_u_stride;        /* ELEMENTS between consecutive environments' U (>= T*nu, 16-byte multiple for TMA) */
    uint64_t env_ws_stride;      /* BYTES between consecutive environments' workspace slices (a multiple of 256)   */
    void* host_mailbox;          /* optional PINNED HOST memory (device-visible under UVA), u_per_command*nu 8-byte
                                    words (x2 for f64): the kernel stores every action value as a self-validating
                                    word, payload32 | (host_epoch & 0xffffffff) << 32, so the host spins on the
                                    words themselves instead of issuing a D2H copy or a stream synchronise      */
    uint64_t host_epoch;
    uint64_t torch_rng_total;    /* 0: the engine's own stream (one Philox subsequence per sample).  > 0: reproduce the
                                    stream of `torch.randn(K,T,nu, device="cuda")` (ATen/native/cuda/
                                    DistributionTemplates.h:50-100): element li of the flat (K,T,nu) tensor comes from
                                    thread idx = li % total, loop slot (li / total), with total = 256 * grid — so a
                                    reference controller on device="cuda" and this engine draw identical noise from
                                    the same (seed, offset).  `offset` is then the generator offset / 4.            */
    void* offset_dev;            /* optional DEVICE u64: when set, the Philox counter base is read from here instead of
                                    `offset`, and the finishing kernel adds `offset_inc` to it — lets a captured CUDA
                                    graph of a whole command draw fresh noise on every replay                       */
    uint64_t offset_inc;
    const double* model_params_ext;   /* HOST pointer: extra model parameters (e.g. MLP weights), read at call /
                                         plan-creation time; NULL if the model needs none                    */
    int32_t n_model_params_ext;
    int32_t K_geom;              /* 0, or the sample count the launch geometry is planned for (>= K): every shard of a
                                    multi-GPU controller passes the LARGEST shard so that all ranks launch the same
                                    grid and publish the same number of records per command                */
    void* debug_clocks;          /* optional profiling aid: (grid_blocks, 16) uint64 %globaltimer stamps (ns) at
                                    phase boundaries of each CTA's first tile; NULL on the product path   */
    void* xchg_status_host;      /* optional pinned HOST int64: the kernel stores MPPI_ERR_TIMEOUT there when a peer
                                    exchange timed out (the caller checks it before the next command)      */
    void* user_model;            /* model == MPPI_MODEL_USER: handle from mppi_user_model_register (a model compiled at
                                    run time); required                                                     */
    /* ---- rollout_samples M > 1 (mppi.py:334-373): each sample's actions are rolled out through M copies of the
     * dynamics; cost = mean over copies + rollout_var_cost * sum_t var_discount[t] * var_m(c_{m,t}).  Fused route: user
     * models compiled with M copies only (mppi_user_model_set_copies); registered models: MPPI_ERR_UNSUPPORTED. */
    int32_t rollout_samples;     /* 0 or 1: one rollout per sample                                                  */
    double rollout_var_cost;
    const void* var_discount;    /* (T) device buffer of the controller dtype: rollout_var_discount ** arange(T)
                                    (mppi.py:174-175); required when rollout_samples > 1                        */
    /* ---- device tensors of a user model (mppi_user_model_set_tensors): HOST array of n_model_tensors references, in
     * the order and with the dtypes / ndims the model was compiled with; read at call / plan-creation time (a plan keeps
     * its own copy).  0 / NULL for every other model. */
    const MppiTensorRef* model_tensors;
    int32_t n_model_tensors;
    const void* model_weights;   /* model == MPPI_MODEL_PENDULUM_MLP_ENSEMBLE: (rollout_samples, 1250) DEVICE buffer of
                                    the controller dtype, one network per row (see the model_params layouts); read by
                                    every command, so it must outlive the plan.  Required for that model, else unused */
} MppiFusedParams;

typedef struct MppiLaunchInfo {
    int32_t block_threads, grid_blocks;
    int32_t smem_bytes, regs_per_thread;
    int32_t max_blocks_per_sm, sm_count;
    uint64_t workspace_bytes;    /* workspace for these dimensions, per environment: enough for any grid they can be
                                    planned with, so one allocation serves every route and geometry         */
    int32_t tma_staging;         /* 1 if the nominal sequence is staged with cp.async.bulk (TMA)         */
    int32_t threads_per_sample;
    int32_t split_cost;          /* 1 if MPPI_FLAG_SPLIT_COST was honoured for these dimensions          */
    int32_t wide_regs;           /* always 0 (MPPI_FLAG_WIDE_REGS is retired)                            */
    int32_t cluster_size;        /* thread-block-cluster size of the launch (1 = no cluster): the CTAs of a cluster
                                    reduce their softmin partials through distributed shared memory        */
    int32_t xchg_records;        /* sharded controllers: records each rank publishes per command (its cluster records
                                    in direct mode, 1 = the rank's combined record); 0 = not sharded       */
    int32_t ll_tail;             /* 1 if the command runs the split-cost kernel specialised for one GPU in LL mode (every
                                    cluster record through this GPU's own mailbox): its softmin tail is inlined   */
    int32_t global_tile;         /* 1 if the plan keeps its tiles in the workspace (MPPI_FLAG_GLOBAL_TILE); fills the
                                    struct's trailing padding, so sizeof stays 64                           */
} MppiLaunchInfo;

int mppi_b200_abi_version(void);
/* Layout probe for foreign-language mirrors of MppiFusedParams: which=0 sizeof, 1 offsetof(seed),
 * 2 offsetof(state), 3 offsetof(U), 4 offsetof(rank), 5 offsetof(partial_out), 6 sizeof(MppiLaunchInfo),
 * 7 offsetof(model_weights), 8 offsetof(model_tensors); and of MppiClosedLoop: 9 sizeof, 10 offsetof(states),
 * 11 offsetof(plant_params), 12 offsetof(plant_blocks); and of MppiEnvParams: 13 sizeof, 14 offsetof(chol),
 * 15 offsetof(model_params), 16 offsetof(scratch); and of MppiPlantModel: 17 sizeof, 18 offsetof(model_tensors). */
uint64_t mppi_abi_layout(int which);
const char* mppi_status_string(int status);
const char* mppi_last_cuda_error(void);

/* Launch geometry / scratch needs for these parameters (no launch).  With model == 0 (no fused model: the per-step
 * entry points further down) only sm_count, workspace_bytes, global_tile and smem_bytes are filled in: smem_bytes is the
 * larger dynamic shared memory of the sampling and softmin kernels' plans, 0 if either does not fit (then only
 * MPPI_FLAG_GLOBAL_TILE runs these dimensions). */
int mppi_fused_query(const MppiFusedParams* p, MppiLaunchInfo* out);
/* The fused command (see struct comment) as a one-shot plan: mppi_plan_create, one command with the struct's state /
 * state_dev / flags / seed / offset / z / action_out / host_mailbox, mppi_plan_destroy.  `stream` is a cudaStream_t. */
int mppi_fused_command(const MppiFusedParams* p, void* stream);

/* ---- Plans: the steady-state fast path ----------------------------------------------------------
 * A plan freezes everything a fused command derives from an MppiFusedParams (kernel selection, launch
 * geometry, the pre-cast kernel argument block, the checks of its buffers, workspace and strides) so
 * that one command costs one short call.
 * Per command only the start state, the RNG counter / injected-noise pointer, the flags that vary
 * (SHIFT, STATE_DEVICE, STATE_PER_SAMPLE) and the action destination change.  The multi-GPU epoch is
 * advanced inside the plan (every rank issues the same sequence of commands). */
int mppi_plan_create(const MppiFusedParams* p, void** plan_out);
int mppi_plan_destroy(void* plan);
/* One command(); `state` = nx host doubles (by value into the launch) or NULL with `state_dev` set. */
int mppi_plan_command(void* plan, const double* state, const void* state_dev, uint32_t flags, uint64_t seed,
                      uint64_t offset, const void* z, void* action_out, void* stream);
/* One command() for a host-resident control loop: launches, then spins (in C) on the pinned-host
 * mailbox the kernel stores the flagged action words into, and returns the action in
 * `action_host_out` (u_per_command*nu elements of the controller dtype).  No D2H memcpy call, no stream synchronise.
 * `host_mailbox`: u_per_command*nu*8 bytes (x2 for f64) of zero-initialised pinned host memory. */
int mppi_plan_command_host(void* plan, const double* state, uint32_t flags, uint64_t seed, uint64_t offset,
                           const void* z, void* action_out_dev, void* host_mailbox, void* action_host_out, void* stream);
/* New model parameters for the plan's following commands, without re-planning: `model_params`
 * (MPPI_MODEL_PARAM_DOUBLES doubles, the layout of MppiFusedParams.model_params) and `ext` / `n_ext` (host doubles, as
 * model_params_ext) are packed with the model's loader exactly as at plan creation, and the plan's copy of the
 * parameters is updated.  Nothing else changes: no kernel selection, geometry, allocation or CUDA call.  Commands
 * already launched keep the values they were launched with (kernel arguments are copied at launch).  This is how a
 * time-varying problem (a moving target, a reference trajectory) follows its data from one control step to the next.
 * PENDULUM_MLP: [2] and [3] selected the plan's kernel and must stay as they are, and the weights are required.
 * MPPI_ERR_BAD_ARG: null plan or model_params, n_ext < 0, ext NULL with n_ext > 0.  MPPI_ERR_UNSUPPORTED while a
 * resident grid is armed (its parameters are frozen; mppi_resident_stop first). */
int mppi_plan_set_model_params(void* plan, const double* model_params, const double* ext, int32_t n_ext);
/* New device tensors for a user model's plan (MppiFusedParams.model_tensors): the plan re-packs only the tensor views of
 * its parameter block — no kernel selection, geometry, allocation or CUDA call.  The count, dtypes and ndims must be the
 * model's; shapes and data pointers may change.  Commands already launched keep the views they were launched with.
 * Edits of a tensor's contents need no call: a command reads them in stream order.
 * MPPI_ERR_BAD_ARG: null plan, refs NULL with n > 0, or a reference the model's signature refuses (see
 * mppi_user_model_set_tensors).  MPPI_ERR_UNSUPPORTED while a resident grid is armed. */
int mppi_plan_set_model_tensors(void* plan, const MppiTensorRef* refs, int32_t n);

/* ---- Closed-loop episodes: the receding-horizon loop without returning to the host -----------------
 * `steps` control steps of a plan's controller against a plant, enqueued on the stream in one call.  Step s is the plan's
 * command (mppi_plan_command with flags SHIFT | STATE_DEVICE, state_dev = states row s, action_out = actions row s, Philox
 * (seed, offset + s * offset_stride)), then one plant step on that action: states row s + 1 = the model's step of row s
 * under u_scale * action — what mppi_rollout_states replays for a one-row sequence — plus disturbance row s, and costs
 * row s = the model's running cost of row s + 1 with that action (t = 0).  The plant is the plan's model (copy 0 of a model
 * with copies) with its own parameter block per environment.  Both launches of every step use programmatic dependent
 * launch where the plan does (MPPI_FLAG_PDL).  The plan's epochs advance once per command, as through mppi_plan_command.
 * All buffers are device memory of the controller dtype, n_env = 1 for a single-environment plan. */
typedef struct MppiClosedLoop {
    uint32_t struct_size;                   /* sizeof(MppiClosedLoop), ABI check                                       */
    int32_t steps;                          /* >= 1                                                                    */
    uint64_t seed, offset, offset_stride;   /* command s draws (seed, offset + s * offset_stride)                      */
    void* states;                           /* (steps+1, n_env, nx): row 0 read, rows 1..steps written                 */
    void* actions;                          /* (steps, n_env, nu) written                                              */
    void* costs;                            /* (steps, n_env) written, or NULL                                         */
    const void* disturbance;                /* (steps, n_env, nx) or NULL                                              */
    const double* plant_params;             /* HOST (n_plant, n_plant_params) doubles in the model's own layout (model_params
                                               followed by model_params_ext), or NULL = the plan's parameters          */
    int32_t n_plant, n_plant_params;        /* n_plant: 1 or n_env                                                     */
    void* plant_blocks;                     /* caller-owned DEVICE scratch, n_plant * mppi_plan_model_block_bytes(plan)
                                               bytes, 16-byte aligned; written once per call (stream-ordered)          */
} MppiClosedLoop;
/* Bytes one packed model parameter block takes in MppiClosedLoop.plant_blocks (a multiple of 16); 0 for a null plan. */
uint64_t mppi_plan_model_block_bytes(void* plan);
/* A plant row's first MPPI_MODEL_PARAM_DOUBLES doubles are its model_params (zero-padded), the rest its model_params_ext;
 * a user model's plant reads the plan's device tensors.
 * MPPI_ERR_ABI: struct_size.  MPPI_ERR_BAD_ARG: null plan / cl / states / actions / plant_blocks, steps < 1, n_plant not 1
 * or n_env, n_plant_params < 0, plant_params NULL with n_plant > 1.
 * MPPI_ERR_UNSUPPORTED: models without a plant step (PENDULUM_MLP / _ENSEMBLE, step-dependent user models),
 * u_per_command != 1, sharded plans (world > 1 or EXPORT_PARTIAL), plans that record their noise (z_out) or draw it from a
 * device counter (offset_dev), a resident grid armed.  All checked before any CUDA call. */
int mppi_plan_closed_loop(void* plan, const MppiClosedLoop* cl, void* stream);

/* The plant of a closed loop named apart from the plan's model: the controller plans with its own model (a learned
 * PENDULUM_MLP network, an ensemble, a simpler analytic model) while the episode follows this one.  Its nx and nu are the
 * plan's; its kernels are the plan's dtype. */
typedef struct MppiPlantModel {
    uint32_t struct_size;                 /* sizeof(MppiPlantModel), ABI check                                    */
    int32_t model;                        /* MPPI_MODEL_PENDULUM, _LINEAR_POINT or _USER                          */
    const void* user_model;               /* MPPI_MODEL_USER: handle compiled for the plan's dtype, else NULL     */
    const MppiTensorRef* model_tensors;   /* HOST array of the plant's own tensors (user models), or NULL         */
    int32_t n_model_tensors, reserved;    /* reserved: 0                                                          */
} MppiPlantModel;
/* Bytes one packed parameter block of this plant takes in MppiClosedLoop.plant_blocks (a multiple of 16); plant NULL: the
 * plan's model, as mppi_plan_model_block_bytes.  0 for arguments mppi_plan_closed_loop_plant refuses. */
uint64_t mppi_plant_block_bytes(void* plan, const MppiPlantModel* plant);
/* mppi_plan_closed_loop against `plant` (NULL: the plan's model, exactly mppi_plan_closed_loop): states row s + 1 = the
 * plant's step of row s under u_scale * action, plus disturbance row s; costs row s = the plant's running cost.  With a
 * plant, plant_params is required: n_plant rows of n_plant_params doubles in the plant's own layout, packed into
 * plant_blocks (n_plant * mppi_plant_block_bytes bytes); a user plant reads its own tensors, and replays copy 0 of a model
 * with copies.  The plan's model need not have a plant step, and per-environment model parameters of the plan
 * (mppi_plan_set_env_params) stay the controller's.
 * MPPI_ERR_ABI: struct_size of cl or plant.  MPPI_ERR_BAD_ARG: those of mppi_plan_closed_loop, an unknown model, a user
 * model whose handle is NULL, not a handle or compiled for the other dtype, reserved != 0, plant nx / nu not the plan's,
 * tensors the plant's signature refuses, plant_params NULL.  MPPI_ERR_UNSUPPORTED: a PENDULUM_MLP / _ENSEMBLE plant or a
 * plant without a plant step (step-dependent user models), and those of mppi_plan_closed_loop but the plan's model's own
 * plant step.  All checked before any CUDA call. */
int mppi_plan_closed_loop_plant(void* plan, const MppiClosedLoop* cl, const MppiPlantModel* plant, void* stream);

/* ---- Per-environment settings of a batched plan (n_env > 1) ---------------------------------------
 * Environment e of a batched plan may have its own temperature, noise covariance, noise mean and model parameters; the
 * K standard normals stay shared.  Every array is optional (NULL: the plan's value applies to every environment) and
 * HOST memory, read during the call.  Each environment's noise model is built exactly as the plan's: the plan's parameters
 * with that environment's values substituted.  An environment's covariance counts as diagonal (MPPI_FLAG_DIAG_SIGMA)
 * when its Cholesky factor is: a diagonal factor is the one of a diagonal covariance, so diagonal and full covariances
 * may be mixed.  The packed blocks go to `scratch` with one stream-ordered copy; commands enqueued before the call keep the
 * values they were launched with, the following commands (and mppi_plan_closed_loop, whose plants with plant_params NULL
 * are then the per-environment models) use the new ones.  No new plan: kernel and geometry stay; with model parameters
 * the plan runs the batched kernel that reads one parameter block per environment.  All pointers NULL: back to the plan's
 * shared values. */
typedef struct MppiEnvParams {
    uint32_t struct_size;                   /* sizeof(MppiEnvParams), ABI check                                        */
    int32_t n_env;                          /* the plan's n_env                                                        */
    const double* lambda_;                  /* (n_env) temperatures > 0, or NULL                                       */
    const double* chol;                     /* (n_env, MPPI_MAX_NU, MPPI_MAX_NU) lower Cholesky factors of the noise
                                               covariances, as MppiFusedParams.chol (diagonal: sqrt on the diagonal); NULL
                                               or set together with sigma_inv                                          */
    const double* sigma_inv;                /* (n_env, MPPI_MAX_NU, MPPI_MAX_NU) inverse covariances, or NULL           */
    const double* noise_mu;                 /* (n_env, MPPI_MAX_NU) noise means, or NULL                               */
    const double* model_params;             /* (n_env, n_model_params) in the model's own layout (model_params followed
                                               by model_params_ext, as MppiClosedLoop.plant_params), or NULL; a user
                                               model's blocks read the plan's device tensors                           */
    int32_t n_model_params;
    int32_t reserved;                       /* 0                                                                       */
    void* scratch;                          /* caller-owned DEVICE memory, mppi_plan_env_scratch_bytes(plan) bytes,
                                               16-byte aligned, kept for as long as the plan runs with these settings;
                                               NULL when every array is NULL                                           */
    uint64_t scratch_bytes;
} MppiEnvParams;
/* Bytes of MppiEnvParams.scratch for this plan (n_env parameter blocks and noise models); 0 for a null plan. */
uint64_t mppi_plan_env_scratch_bytes(void* plan);
/* MPPI_ERR_ABI: struct_size.  MPPI_ERR_BAD_ARG: null plan / ep, n_env not the plan's, a temperature <= 0 or not finite,
 * only one of chol / sigma_inv, n_model_params < 0, reserved != 0, scratch NULL / misaligned / smaller than
 * mppi_plan_env_scratch_bytes.  MPPI_ERR_UNSUPPORTED: single-environment plans, sharded plans, model parameters of the
 * PENDULUM_MLP models (no per-environment kernel).  All checked before any CUDA call. */
int mppi_plan_set_env_params(void* plan, const MppiEnvParams* ep, void* stream);

/* Per-environment horizons of a batched plan: environment e rolls out h_e <= T steps (T: the plan's horizon), so it is the
 * single-environment MPPI command with horizon h_e on the first h_e * nu rows of the shared standard normals — rollout,
 * running and action costs over t < h_e, its update added to its first h_e rows, and the shift moving rows 1..h_e-1 up
 * with u_init into row h_e-1.  Rows h_e.. of its nominal sequence are left at the post-shift nominal, u_init when they
 * held it.  `horizon_host`: (n_env) HOST int32 values with u_per_command <= h_e <= T, read during the call; NULL: back to T
 * for every environment.  The values go to `scratch` (caller-owned DEVICE memory, mppi_plan_env_horizon_bytes(plan)
 * bytes, 16-byte aligned, kept for as long as the plan runs with these horizons; may be NULL with horizon_host NULL) with
 * one stream-ordered copy: commands enqueued before the call keep the horizons they were launched with.  No new plan:
 * kernel, geometry, tiles and strides stay the plan's. */
uint64_t mppi_plan_env_horizon_bytes(void* plan);   /* 0 for a null plan */
/* MPPI_ERR_BAD_ARG: null plan, a horizon < 1, < u_per_command or > T, scratch NULL / misaligned.  MPPI_ERR_UNSUPPORTED:
 * single-environment plans, sharded plans, the PENDULUM_MLP models (their batched kernels fix their own tiles).  All
 * checked before any CUDA call. */
int mppi_plan_set_env_horizon(void* plan, const int32_t* horizon_host, void* scratch, void* stream);

/* ---- Resident mode: command() without a kernel launch ---------------------------------------------
 * For a host control loop (mppi.py:240-252 called once per control step).  One cooperative launch leaves the
 * command's grid on the SMs; each following command is a record (flags, Philox counter, start state) written into
 * pinned host memory that the grid polls, and the action comes back the way mppi_plan_command_host returns it.
 * The grid prepares the next command's noise and perturbed actions while the host turns around, and leaves by
 * itself after `idle_us` without a command (the next command relaunches it), so a device-wide synchronise is
 * never blocked for longer than that.  Results are bit-identical to mppi_plan_command_host with the same
 * (state, flags, seed, offset).  Available for plans that run the split-cost rollout (one tile per SM;
 * MPPI_FLAG_SPLIT_COST honoured — MppiLaunchInfo.split_cost) of single-GPU controllers (one environment, no peers, no
 * EXPORT_PARTIAL); others: MPPI_ERR_UNSUPPORTED.
 *
 *   host_box      pinned host memory, zero-initialised, 64 + u_per_command*nu (x2 for f64) 8-byte words:
 *                 [0,32) command record | [32] sequence number of the last finished command | [33] exit word |
 *                 [64,..) action words (payload32 | seq32 << 32)
 *   board_dev     device memory, 128 8-byte words (the record re-published for all CTAs + the done word)
 *   action_out_dev device (u_per_command,nu) of the controller dtype (the action as on the launch route)
 *   stream        a NON-BLOCKING stream used for nothing else: work on other streams is not ordered against the
 *                 resident grid; call mppi_resident_sync before reading U / cost_total / stats, mppi_resident_stop
 *                 before writing U or launching mppi_plan_command on the same controller.
 * While resident, the controller's parameters are frozen (they are kernel arguments of the resident launch). */
int mppi_resident_start(void* plan, void* host_box, void* board_dev, void* action_out_dev, uint64_t idle_us, void* stream);
/* One command(): `state` = nx host doubles; flags: MPPI_FLAG_SHIFT is read; returns the action in action_host_out
 * (u_per_command*nu elements of the controller dtype). */
int mppi_resident_command(void* plan, const double* state, uint32_t flags, uint64_t seed, uint64_t offset,
                          void* action_host_out);
/* Wait until everything the last command wrote to device memory (U, cost_total, nominal_used, stats) is complete. */
int mppi_resident_sync(void* plan);
/* Send the grid away and wait for it; mppi_plan_destroy does this too. */
int mppi_resident_stop(void* plan);
/* Kernel launches made by resident mode so far (the first command, and each wake-up after an idle exit). */
uint64_t mppi_resident_launches(void* plan);

/* Multi-GPU, library-collective route: after every rank exported its partial and the caller
 * all-gathered them (NCCL), finish the update on each rank: beta=min, rescale, U += sum/eta
 * (mppi.py:254-259, 268-270 across shards).  `partials` is (world, 2+R) doubles on device. */
int mppi_apply_partials(const MppiFusedParams* p, const void* partials, void* stream);

/* Peer mailboxes for the in-kernel NVLink exchange.  The library owns these small buffers
 * (cudaMalloc + cudaIpc), because IPC handles must cover a whole allocation. */
/* A user-written analytic model compiled at run time (the reference's plugin surface is arbitrary Python callables,
 * mppi.py:63-64; analytic ones can be given as CUDA C++ bodies — pytorch_mppi_b200.models.CudaModel — and are compiled
 * with NVRTC in process).  `cubin` is the compiled module, `names` the lowered names of its kernels:
 * [0] fused_command_kernel<UserModel, real, variant, false, false>   [1] ... split-cost (or NULL)
 * [2] ... batched, MPPI variant (or NULL)   [3] resident_command_kernel<UserModel, real, variant> (or NULL)
 * [4] states_kernel<UserModel, real>.  A module with a split-cost kernel also exports its single-GPU LL form as
 * `mppi_user_fused_command_kernel_ll` (MPPI_USER_KERNEL_LL).  A module may export its closed-loop plant step as
 * `mppi_user_plant_step_kernel` (MPPI_USER_KERNEL_PLANT; without it mppi_plan_closed_loop is unsupported for the model).
 * The handle goes into MppiFusedParams.user_model with model = MPPI_MODEL_USER. */
int mppi_user_model_register(const void* cubin, uint64_t cubin_bytes, int32_t nx, int32_t nu, int32_t n_params, int32_t dtype,
                             int32_t variant, const char* const* names, void** handle_out);
int mppi_user_model_release(void* handle);
/* The copy count a user model's kernels were compiled with (CudaModel(copies=M): its bodies take the copy index m; 1 by
 * default).  Plans of the model require rollout_samples == copies.  A model with copies > 1 has no split-cost, batched
 * or resident kernels (names[1..3] NULL), so its commands run the single-loop rollout and resident mode is refused.
 * MPPI_ERR_BAD_ARG: bad handle, copies outside 1..MPPI_MAX_COPIES, or copies > 1 with any of those kernels. */
int mppi_user_model_set_copies(void* handle, int32_t copies);
/* The device tensors a user model's kernels were compiled to read (CudaModel(tensors=...)): their count (0..
 * MPPI_MAX_MODEL_TENSORS), element types and ndims, in the order of the views in its parameter block
 * `struct P { real v[n_params]; View t0; ...; }`, View = { const T* data; int32_t shape[4]; } (24 bytes, 8-aligned).
 * The shapes and pointers come with every plan (MppiFusedParams.model_tensors), which must then match this signature:
 * same count, dtypes and ndims, non-null data, positive dimensions, at most 2^31 - 1 elements (else MPPI_ERR_BAD_ARG).
 * MPPI_ERR_BAD_ARG: bad handle, n outside 0..MPPI_MAX_MODEL_TENSORS, NULL arrays with n > 0, an unknown dtype or an ndim
 * outside 1..4.  MPPI_ERR_UNSUPPORTED: the parameter block would exceed the largest block a kernel takes. */
int mppi_user_model_set_tensors(void* handle, int32_t n, const int32_t* dtypes, const int32_t* ndims);
/* Highest command epoch this plan has used (the tag of its reduction records, shared by the launch and resident routes);
 * pass it as MppiFusedParams.epoch when re-creating the plan so that stale records can never match. */
uint64_t mppi_plan_epoch(void* plan);
int mppi_xchg_create(void** mailbox, void* ipc_handle_out_64B);       /* local mailbox + its IPC handle */
int mppi_xchg_open(const void* ipc_handle_64B, void** peer_mailbox);  /* map a peer's mailbox           */
int mppi_xchg_close(void* peer_mailbox);
int mppi_xchg_destroy(void* mailbox);
uint64_t mppi_xchg_bytes(void);

/* ---- API-visible intermediates, produced on demand (off the hot path) -------------------------
 * The reference stores noise / perturbed_action (mppi.py:383-385) and, with a terminal cost,
 * states / actions (mppi.py:307-322) on every command.  The fused kernel keeps them in shared
 * memory only; these entry points regenerate them from (seed, offset | z) and nominal_used. */
int mppi_materialize(const MppiFusedParams* p, void* perturbed_action /*(K,T,nu)*/, void* noise /*(K,T,nu)*/,
                     void* noise_theta /*KMPPI (K,S,nu) or NULL*/,
                     void* states /*(K,T,nx), (M,K,T,nx) with rollout_samples = M > 1, or NULL*/, void* stream);

/* get_rollouts (mppi.py:425-448) for a registered model: `n_rollouts` start states (n_rollouts,nx) on the device, each
 * rolled T steps through u_scale * actions[t] — one (T,nu) sequence replayed by every rollout (actions_stride = 0) or a
 * sequence per rollout (actions_stride = elements between them, e.g. T*nu) — into states_out (n_rollouts,T,nx).
 * Only model, dtype, nx, nu, u_scale and the model parameters of `p` are read; a model with copies rolls out copy 0. */
int mppi_rollout_states(const MppiFusedParams* p, const void* start_states, const void* actions, int64_t actions_stride,
                        int32_t n_rollouts, int32_t T, void* states_out, void* stream);

/* ---- Per-step entry points for arbitrary Python dynamics/cost callables ------------------------
 * The T-loop stays in Python (mppi.py:312-322); sampling, cost accumulation and the softmin update
 * are kernels. */

/* mppi.py:375-385 + 186-199 + 415 (SMPPI :539-562, KMPPI :657-670): fills perturbed_action, noise
 * (and noise_theta) and initialises cost_init[k] = sum_t U . action_cost (+ SMPPI smoothness).
 * `override` (n_override,T,nu) rows replace samples [override_start, ...) before the clamp
 * (SpecificActionSampler, mppi.py:393-399). */
int mppi_sample_perturb(const MppiFusedParams* p, void* perturbed_action, void* noise, void* noise_theta,
                        void* cost_init, const void* override_rows, int32_t n_override, int32_t override_start,
                        void* stream);
/* mppi.py:318-319 / 362-364: cost[m,k] += c[m,k]; M>1 also var_acc[k] += var_m(c) * discount. */
int mppi_cost_accumulate(void* cost /*(M,K)*/, const void* c /*(M*K)*/, void* var_acc /*(K) or NULL*/,
                         int32_t M, int32_t K, double discount, int32_t dtype, void* stream);
/* mppi.py:254-259 + 268-270 from materialised tensors: cost_total (K) and eps = noise (K,T,nu)
 * (KMPPI: noise_theta (K,S,nu)).  Reads the post-shift nominal from p->nominal_used (written by
 * mppi_sample_perturb), writes p->U / A / theta, p->action_out and p->stats. */
int mppi_softmin_update(const MppiFusedParams* p, const void* cost_total, const void* eps, void* stream);
/* omega (mppi.py:256-258) from cost_total and the (beta, eta) a command left in `stats`. */
int mppi_omega(const void* cost_total, void* omega_out, const void* stats, double lambda_, int32_t K, int32_t dtype,
               void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MPPI_B200_H */
