"""ctypes binding of the C-ABI library (include/mppi_b200.h -> csrc/libmppi_b200.so).

The library is built in-tree by ``pytorch_mppi_b200.build`` (nvcc, sm_90a).  There is NO fallback:
if the shared object is missing or a symbol is absent, importing the controllers raises.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MPPI_B200_LIB") or os.path.join(HERE, "csrc", "libmppi_b200.so")

MPPI_MAX_NU = 4
MPPI_MAX_NX = 8
MPPI_MODEL_PARAM_DOUBLES = 48
MPPI_MAX_RANKS = 8
MPPI_MAX_COPIES = 8
MPPI_MAX_MODEL_TENSORS = 8
ABI_VERSION = 3

# enums
VARIANT_MPPI, VARIANT_SMPPI, VARIANT_KMPPI = 0, 1, 2
F32, F64 = 0, 1
U8, I32 = 2, 3                       # element types of model tensors only
MODEL_PENDULUM, MODEL_LINEAR_POINT, MODEL_PENDULUM_MLP = 1, 2, 3
MODEL_PENDULUM_MLP_ENSEMBLE = 4
MODEL_USER = 100
FLAG_SHIFT = 1 << 0
FLAG_NULL_ACTION = 1 << 1
FLAG_ABS_COST = 1 << 2
FLAG_DIAG_SIGMA = 1 << 3
FLAG_STATE_DEVICE = 1 << 4
FLAG_STATE_PER_SAMPLE = 1 << 5
FLAG_EXPORT_PARTIAL = 1 << 6
FLAG_NOMINAL_PADDED = 1 << 7
FLAG_PDL = 1 << 8
FLAG_SPLIT_COST = 1 << 9
FLAG_WIDE_REGS = 1 << 10
FLAG_GLOBAL_TILE = 1 << 11

STATUS = {0: "ok", -1: "bad argument", -2: "unsupported", -3: "workspace too small", -4: "CUDA error",
          -5: "ABI mismatch", -6: "peer exchange timeout"}


class MppiTensorRef(C.Structure):
    """Mirror of `struct MppiTensorRef`: one device tensor a user model's bodies read."""
    _fields_ = [
        ("data", C.c_void_p),
        ("dtype", C.c_int32),
        ("ndim", C.c_int32),
        ("shape", C.c_int64 * 4),
    ]


class MppiFusedParams(C.Structure):
    """Mirror of `struct MppiFusedParams` (include/mppi_b200.h).  Field order and types must match;
    tests/test_cabi.py checks sizeof/offsetof against the library."""
    _fields_ = [
        ("struct_size", C.c_uint32),
        ("variant", C.c_int32),
        ("model", C.c_int32),
        ("dtype", C.c_int32),
        ("K", C.c_int32),
        ("T", C.c_int32),
        ("nx", C.c_int32),
        ("nu", C.c_int32),
        ("S", C.c_int32),
        ("u_per_command", C.c_int32),
        ("flags", C.c_uint32),
        ("block_threads", C.c_int32),
        ("grid_blocks", C.c_int32),
        ("threads_per_sample", C.c_int32),
        ("k_offset", C.c_int64),
        ("seed", C.c_uint64),
        ("offset", C.c_uint64),
        ("lambda_", C.c_double),
        ("u_scale", C.c_double),
        ("noise_mu", C.c_double * MPPI_MAX_NU),
        ("chol", C.c_double * (MPPI_MAX_NU * MPPI_MAX_NU)),
        ("sigma_inv", C.c_double * (MPPI_MAX_NU * MPPI_MAX_NU)),
        ("u_min", C.c_double * MPPI_MAX_NU),
        ("u_max", C.c_double * MPPI_MAX_NU),
        ("u_init", C.c_double * MPPI_MAX_NU),
        ("action_min", C.c_double * MPPI_MAX_NU),
        ("action_max", C.c_double * MPPI_MAX_NU),
        ("w_action_seq_cost", C.c_double),
        ("delta_t", C.c_double),
        ("model_params", C.c_double * MPPI_MODEL_PARAM_DOUBLES),
        ("state", C.c_double * MPPI_MAX_NX),
        ("state_dev", C.c_void_p),
        ("U", C.c_void_p),
        ("A", C.c_void_p),
        ("theta", C.c_void_p),
        ("W", C.c_void_p),
        ("Wshift", C.c_void_p),
        ("cost_total", C.c_void_p),
        ("action_out", C.c_void_p),
        ("nominal_used", C.c_void_p),
        ("stats", C.c_void_p),
        ("z", C.c_void_p),
        ("z_out", C.c_void_p),
        ("workspace", C.c_void_p),
        ("workspace_bytes", C.c_uint64),
        ("rank", C.c_int32),
        ("world", C.c_int32),
        ("epoch", C.c_uint64),
        ("peer_slots", C.c_void_p * MPPI_MAX_RANKS),
        ("partial_out", C.c_void_p),
        ("n_env", C.c_int32),
        ("env_u_stride", C.c_int32),
        ("env_ws_stride", C.c_uint64),
        ("host_mailbox", C.c_void_p),
        ("host_epoch", C.c_uint64),
        ("torch_rng_total", C.c_uint64),
        ("offset_dev", C.c_void_p),
        ("offset_inc", C.c_uint64),
        ("model_params_ext", C.c_void_p),
        ("n_model_params_ext", C.c_int32),
        ("K_geom", C.c_int32),
        ("debug_clocks", C.c_void_p),
        ("xchg_status_host", C.c_void_p),
        ("user_model", C.c_void_p),
        ("rollout_samples", C.c_int32),
        ("rollout_var_cost", C.c_double),
        ("var_discount", C.c_void_p),
        ("model_tensors", C.c_void_p),
        ("n_model_tensors", C.c_int32),
        ("model_weights", C.c_void_p),
    ]


class MppiLaunchInfo(C.Structure):
    _fields_ = [
        ("block_threads", C.c_int32),
        ("grid_blocks", C.c_int32),
        ("smem_bytes", C.c_int32),
        ("regs_per_thread", C.c_int32),
        ("max_blocks_per_sm", C.c_int32),
        ("sm_count", C.c_int32),
        ("workspace_bytes", C.c_uint64),
        ("tma_staging", C.c_int32),
        ("threads_per_sample", C.c_int32),
        ("split_cost", C.c_int32),
        ("wide_regs", C.c_int32),
        ("cluster_size", C.c_int32),
        ("xchg_records", C.c_int32),
        ("ll_tail", C.c_int32),
        ("global_tile", C.c_int32),
    ]


class MppiClosedLoop(C.Structure):
    """Mirror of `struct MppiClosedLoop`: one closed-loop episode of a plan (mppi_plan_closed_loop)."""
    _fields_ = [
        ("struct_size", C.c_uint32),
        ("steps", C.c_int32),
        ("seed", C.c_uint64),
        ("offset", C.c_uint64),
        ("offset_stride", C.c_uint64),
        ("states", C.c_void_p),
        ("actions", C.c_void_p),
        ("costs", C.c_void_p),
        ("disturbance", C.c_void_p),
        ("plant_params", C.c_void_p),
        ("n_plant", C.c_int32),
        ("n_plant_params", C.c_int32),
        ("plant_blocks", C.c_void_p),
    ]


class MppiPlantModel(C.Structure):
    """Mirror of `struct MppiPlantModel`: the plant of a closed loop, named apart from the plan's model
    (mppi_plan_closed_loop_plant)."""
    _fields_ = [
        ("struct_size", C.c_uint32),
        ("model", C.c_int32),
        ("user_model", C.c_void_p),
        ("model_tensors", C.c_void_p),
        ("n_model_tensors", C.c_int32),
        ("reserved", C.c_int32),
    ]


class MppiEnvParams(C.Structure):
    """Mirror of `struct MppiEnvParams`: per-environment settings of a batched plan (mppi_plan_set_env_params)."""
    _fields_ = [
        ("struct_size", C.c_uint32),
        ("n_env", C.c_int32),
        ("lambda_", C.c_void_p),
        ("chol", C.c_void_p),
        ("sigma_inv", C.c_void_p),
        ("noise_mu", C.c_void_p),
        ("model_params", C.c_void_p),
        ("n_model_params", C.c_int32),
        ("reserved", C.c_int32),
        ("scratch", C.c_void_p),
        ("scratch_bytes", C.c_uint64),
    ]


# every symbol include/mppi_b200.h declares: (name, restype, argtypes)
_P = C.POINTER(MppiFusedParams)
SYMBOLS = [
    ("mppi_b200_abi_version", C.c_int, []),
    ("mppi_status_string", C.c_char_p, [C.c_int]),
    ("mppi_last_cuda_error", C.c_char_p, []),
    ("mppi_abi_layout", C.c_uint64, [C.c_int]),
    ("mppi_fused_query", C.c_int, [_P, C.POINTER(MppiLaunchInfo)]),
    ("mppi_fused_command", C.c_int, [_P, C.c_void_p]),
    ("mppi_plan_create", C.c_int, [_P, C.POINTER(C.c_void_p)]),
    ("mppi_plan_destroy", C.c_int, [C.c_void_p]),
    ("mppi_plan_command", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint64, C.c_uint64, C.c_void_p,
                                    C.c_void_p, C.c_void_p]),
    ("mppi_plan_command_host", C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_void_p]),
    ("mppi_plan_set_model_params", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32]),
    ("mppi_plan_set_model_tensors", C.c_int, [C.c_void_p, C.c_void_p, C.c_int32]),
    ("mppi_plan_model_block_bytes", C.c_uint64, [C.c_void_p]),
    ("mppi_plan_closed_loop", C.c_int, [C.c_void_p, C.POINTER(MppiClosedLoop), C.c_void_p]),
    ("mppi_plant_block_bytes", C.c_uint64, [C.c_void_p, C.POINTER(MppiPlantModel)]),
    ("mppi_plan_closed_loop_plant", C.c_int, [C.c_void_p, C.POINTER(MppiClosedLoop), C.POINTER(MppiPlantModel), C.c_void_p]),
    ("mppi_plan_env_scratch_bytes", C.c_uint64, [C.c_void_p]),
    ("mppi_plan_set_env_params", C.c_int, [C.c_void_p, C.POINTER(MppiEnvParams), C.c_void_p]),
    ("mppi_plan_env_horizon_bytes", C.c_uint64, [C.c_void_p]),
    ("mppi_plan_set_env_horizon", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("mppi_resident_start", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    ("mppi_resident_command", C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint64, C.c_uint64, C.c_void_p]),
    ("mppi_resident_sync", C.c_int, [C.c_void_p]),
    ("mppi_resident_stop", C.c_int, [C.c_void_p]),
    ("mppi_resident_launches", C.c_uint64, [C.c_void_p]),
    ("mppi_plan_epoch", C.c_uint64, [C.c_void_p]),
    ("mppi_user_model_register", C.c_int, [C.c_void_p, C.c_uint64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                           C.POINTER(C.c_char_p), C.POINTER(C.c_void_p)]),
    ("mppi_user_model_release", C.c_int, [C.c_void_p]),
    ("mppi_user_model_set_copies", C.c_int, [C.c_void_p, C.c_int32]),
    ("mppi_user_model_set_tensors", C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    ("mppi_apply_partials", C.c_int, [_P, C.c_void_p, C.c_void_p]),
    ("mppi_xchg_create", C.c_int, [C.POINTER(C.c_void_p), C.c_void_p]),
    ("mppi_xchg_open", C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    ("mppi_xchg_close", C.c_int, [C.c_void_p]),
    ("mppi_xchg_destroy", C.c_int, [C.c_void_p]),
    ("mppi_xchg_bytes", C.c_uint64, []),
    ("mppi_materialize", C.c_int, [_P, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("mppi_rollout_states", C.c_int, [_P, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    ("mppi_sample_perturb", C.c_int, [_P, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                      C.c_int32, C.c_void_p]),
    ("mppi_cost_accumulate", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_double, C.c_int32,
                                       C.c_void_p]),
    ("mppi_softmin_update", C.c_int, [_P, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("mppi_omega", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_int32, C.c_int32, C.c_void_p]),
]

_lib = None
_variants = {}


class MppiLibraryError(RuntimeError):
    pass


def load(path=None):
    """Load the shared library (or a user-model variant at `path`) and bind every declared symbol;
    raises if anything is missing."""
    global _lib
    if path is None:
        if _lib is not None:
            return _lib
        path = LIB_PATH
    elif path in _variants:
        return _variants[path]
    if not os.path.exists(path):
        raise MppiLibraryError(
            f"{path} not found: build it with `python -m pytorch_mppi_b200.build` "
            "(nvcc, sm_90a). pytorch_mppi_b200 has no CPU or eager-PyTorch fallback.")
    lib = C.CDLL(path)
    for name, restype, argtypes in SYMBOLS:
        try:
            fn = getattr(lib, name)
        except AttributeError as e:
            raise MppiLibraryError(f"{path} does not export `{name}`; rebuild the library") from e
        fn.restype = restype
        fn.argtypes = argtypes
    v = lib.mppi_b200_abi_version()
    if v != ABI_VERSION:
        raise MppiLibraryError(f"ABI version mismatch: library {v}, python {ABI_VERSION}")
    if lib.mppi_abi_layout(0) != C.sizeof(MppiFusedParams):
        raise MppiLibraryError("MppiFusedParams layout differs between the ctypes mirror and the library")
    if path == LIB_PATH:
        _lib = lib
    else:
        _variants[path] = lib
    return lib


def check(rc, what="mppi call"):
    if rc != 0:
        lib = load()
        msg = lib.mppi_status_string(rc).decode()
        if rc in (-4, -2):
            msg += ": " + lib.mppi_last_cuda_error().decode()
        raise MppiLibraryError(f"{what} failed: {msg} ({rc})")
