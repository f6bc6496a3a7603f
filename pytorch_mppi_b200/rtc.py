"""Run-time compilation of user-written analytic models with NVRTC (in process; no nvcc, no toolkit at run time).

`CudaModel` (models.py) turns the user's `step` / `cost` / `terminal` bodies into a `struct mppi::UserModel`; this module
compiles `csrc/mppi_fused.cuh + csrc/mppi_resident.cuh + that struct` for sm_90a — the SAME kernel templates the
registry models are built from — and returns the cubin with the lowered names of the instantiated kernels, which the
C library loads (`mppi_user_model_register`: cudaLibraryLoadData + cudaLibraryGetKernel).  Compiled modules are cached
on disk under csrc/_user/ keyed by the hash of everything they are built from, so a model compiles once (a few
seconds) and a cached cubin needs no NVRTC at all.

NVRTC is bound with ctypes (8 entry points); the library is looked up in the CUDA toolkit, then in the wheel torch
ships (nvidia-cuda-nvrtc), then on the loader path.
"""
from __future__ import annotations

import ctypes as C
import glob
import hashlib
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
CACHE = os.path.join(CSRC, "_user")
ARCH = "sm_90a"
_KERNEL_HEADERS = ("mppi_fused.cuh", "mppi_math.cuh", "mppi_resident.cuh")

_nvrtc = None


class RtcError(RuntimeError):
    pass


def _load_nvrtc():
    global _nvrtc
    if _nvrtc is not None:
        return _nvrtc
    cands = sorted(glob.glob("/usr/local/cuda*/lib64/libnvrtc.so.1[0-9]"), reverse=True)
    try:
        import nvidia  # the namespace package of torch's CUDA wheels
        for root in nvidia.__path__:
            cands += sorted(glob.glob(os.path.join(root, "cuda_nvrtc", "lib", "libnvrtc.so.1[0-9]")), reverse=True)
    except ImportError:
        pass
    cands += ["libnvrtc.so.12", "libnvrtc.so"]
    last = None
    for path in cands:
        try:
            lib = C.CDLL(path)
        except OSError as e:
            last = e
            continue
        lib.nvrtcCreateProgram.argtypes = [C.POINTER(C.c_void_p), C.c_char_p, C.c_char_p, C.c_int, C.c_void_p, C.c_void_p]
        lib.nvrtcCompileProgram.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_char_p)]
        lib.nvrtcAddNameExpression.argtypes = [C.c_void_p, C.c_char_p]
        lib.nvrtcGetLoweredName.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_char_p)]
        lib.nvrtcGetProgramLogSize.argtypes = [C.c_void_p, C.POINTER(C.c_size_t)]
        lib.nvrtcGetProgramLog.argtypes = [C.c_void_p, C.c_char_p]
        lib.nvrtcGetCUBINSize.argtypes = [C.c_void_p, C.POINTER(C.c_size_t)]
        lib.nvrtcGetCUBIN.argtypes = [C.c_void_p, C.c_char_p]
        lib.nvrtcDestroyProgram.argtypes = [C.POINTER(C.c_void_p)]
        _nvrtc = lib
        return lib
    raise RtcError(f"libnvrtc not found (tried {cands}): {last}")


def _sources_hash() -> str:
    h = hashlib.sha1(ARCH.encode())
    for name in _KERNEL_HEADERS:
        with open(os.path.join(CSRC, name), "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def kernel_names(real: str, variant: int, copies: int = 1):
    """Name expressions of the kernels one (dtype, controller variant) needs, in mppi_user_model_register's order:
    fused, split-cost, batched (MPPI variant only), resident, states.  A model with copies > 1 has only the fused
    (single-loop) and states kernels: the split-cost rollout and the kernels built on it roll out one copy per sample,
    and MPPI_Batched has no rollout_samples.  A module with the split-cost kernel also exports its single-GPU LL form
    under a fixed unmangled name (MPPI_USER_KERNEL_LL, added by compile_user_model), and every module its global-tile kernels
    (MPPI_USER_KERNEL_GTILE, and MPPI_USER_KERNEL_GTILE_BATCHED where the batched kernel exists)."""
    m = "mppi::UserModel"
    one = copies == 1
    return [f"&mppi::fused_command_kernel<{m}, {real}, {variant}, false, false>",
            f"&mppi::fused_command_kernel<{m}, {real}, {variant}, false, true>" if one else None,
            f"&mppi::fused_command_kernel<{m}, {real}, 0, true>" if variant == 0 and one else None,
            f"&mppi::resident_command_kernel<{m}, {real}, {variant}>" if one else None,
            f"&mppi::states_kernel<{m}, {real}>"]


def compile_user_model(header_text: str, real: str, variant: int, copies: int = 1, plant: bool = True):
    """-> (cubin bytes, [lowered kernel name or None] x 5).  Cached on disk.  `plant`: also export the closed-loop plant
    step (MPPI_USER_KERNEL_PLANT; step-dependent models have none)."""
    src = '#include "mppi_fused.cuh"\n#include "mppi_resident.cuh"\n' + header_text + "\n"
    if copies == 1:   # the split-cost kernel's single-GPU LL form, under the name mppi_user_model_register looks up
        src += f"MPPI_USER_KERNEL_LL(mppi::UserModel, {real}, {variant})\n"
    # the global-tile kernels (tile_memory='global' / 'auto' past the shared-memory edge), also under fixed names
    src += f"MPPI_USER_KERNEL_GTILE(mppi::UserModel, {real}, {variant})\n"
    if variant == 0 and copies == 1:
        src += f"MPPI_USER_KERNEL_GTILE_BATCHED(mppi::UserModel, {real})\n"
        # MPPI_Batched with per-environment model parameters (set_env_params)
        src += f"MPPI_USER_KERNEL_ENV_BATCHED(mppi::UserModel, {real})\n"
    if plant:         # the plant step of closed-loop episodes (run_closed_loop)
        src += f"MPPI_USER_KERNEL_PLANT(mppi::UserModel, {real})\n"
    # keyed by the whole program (model, exported kernels) and the kernel headers it includes: a module built before a
    # kernel was added is never reused
    tag = hashlib.sha1(f"{src}|{real}|{variant}|{copies}|{_sources_hash()}".encode()).hexdigest()[:20]
    cubin_path = os.path.join(CACHE, f"rtc_{tag}.cubin")
    names_path = os.path.join(CACHE, f"rtc_{tag}.json")
    if os.path.exists(cubin_path) and os.path.exists(names_path):
        with open(cubin_path, "rb") as f, open(names_path) as g:
            return f.read(), json.load(g)
    lib = _load_nvrtc()
    prog = C.c_void_p()
    if lib.nvrtcCreateProgram(C.byref(prog), src.encode(), b"mppi_user_model.cu", 0, None, None) != 0:
        raise RtcError("nvrtcCreateProgram failed")
    try:
        exprs = kernel_names(real, variant, copies)
        for e in exprs:
            if e is not None and lib.nvrtcAddNameExpression(prog, e.encode()) != 0:
                raise RtcError(f"nvrtcAddNameExpression({e}) failed")
        # -default-device: the model structs' parameter packers (`load`) are host code in the nvcc build; here they are
        # never called (the library packs user-model parameters generically) and NVRTC has no host side
        opts = [f"--gpu-architecture={ARCH}", "-default-device", "-std=c++17", "-lineinfo", f"-I{CSRC}"]
        arr = (C.c_char_p * len(opts))(*[o.encode() for o in opts])
        rc = lib.nvrtcCompileProgram(prog, len(opts), arr)
        n = C.c_size_t()
        lib.nvrtcGetProgramLogSize(prog, C.byref(n))
        log = C.create_string_buffer(max(n.value, 1))
        lib.nvrtcGetProgramLog(prog, log)
        if rc != 0:
            raise RtcError("NVRTC could not compile the user model:\n" + log.value.decode(errors="replace")[-6000:])
        lib.nvrtcGetCUBINSize(prog, C.byref(n))
        cubin = C.create_string_buffer(n.value)
        if lib.nvrtcGetCUBIN(prog, cubin) != 0:
            raise RtcError("nvrtcGetCUBIN failed")
        lowered = []
        for e in exprs:
            if e is None:
                lowered.append(None)
                continue
            p = C.c_char_p()
            if lib.nvrtcGetLoweredName(prog, e.encode(), C.byref(p)) != 0:
                raise RtcError(f"nvrtcGetLoweredName({e}) failed")
            lowered.append(p.value.decode())
        data = cubin.raw
    finally:
        lib.nvrtcDestroyProgram(C.byref(prog))
    # several processes (one per GPU) may compile the same model at the same time: both files appear atomically, the
    # names first — a reader that finds the cubin finds complete names
    os.makedirs(CACHE, exist_ok=True)
    tmp = names_path + f".{os.getpid()}.tmp"
    with open(tmp, "w") as g:
        json.dump(lowered, g)
    os.replace(tmp, names_path)
    tmp = cubin_path + f".{os.getpid()}.tmp"
    with open(tmp, "wb") as f:
        f.write(data)
    os.replace(tmp, cubin_path)
    return data, lowered
