"""In-tree build of the C-ABI CUDA library for sm_90a:  python -m pytorch_mppi_b200.build [--force] [-v]

nvcc cross-compiles without a GPU.  The library is several translation units compiled in parallel (one per
registered model x dtype plus the C-ABI / model-independent unit) and linked into ONE shared object, which stays
in-tree (git-ignored) so that a copy of the built tree carries the native code its tests load.
Objects are cached under csrc/_obj/ keyed by the hash of everything they are compiled from, so touching one
kernel header rebuilds only the units that include it.
"""
from __future__ import annotations

import concurrent.futures
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(CSRC, "_obj")
OUT = os.path.join(CSRC, "libmppi_b200.so")
STAMP = OUT + ".stamp"
PUBLIC_HEADER = os.path.join(os.path.dirname(HERE), "include", "mppi_b200.h")


def _h(*names):
    return [os.path.join(CSRC, n) for n in names]


COMMON_HEADERS = _h("mppi_host.cuh", "mppi_fused.cuh", "mppi_math.cuh", "mppi_resident.cuh", "mppi_resident_host.h",
                    "mppi_model_tensors.h") + [PUBLIC_HEADER]
MODEL_HEADERS = COMMON_HEADERS + _h("mppi_mlp_tc.cuh")
CABI_HEADERS = COMMON_HEADERS + _h("mppi_fused_host.cuh")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC"]

# name -> (source, extra defines, headers it depends on)
UNITS = {"cabi": ("mppi_b200.cu", [], CABI_HEADERS)}
for _mid, _mname in ((1, "pendulum"), (2, "linear_point"), (3, "pendulum_mlp"), (4, "pendulum_mlp_ensemble")):
    for _f64 in (0, 1):
        UNITS[f"model_{_mname}_{'f64' if _f64 else 'f32'}"] = (
            "mppi_model_tu.cu", [f"-DMPPI_TU_MODEL={_mid}", f"-DMPPI_TU_F64={_f64}"], MODEL_HEADERS)


def _unit_hash(src, defines, headers):
    h = hashlib.sha1(" ".join(NVCC_FLAGS + defines).encode())
    for d in [os.path.join(CSRC, src), *headers]:
        with open(d, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def source_hash() -> str:
    """Hash of everything the library is compiled from (sources, headers, flags).  File times are not used: the
    copy that ships a built tree to a GPU machine need not keep them, and a spurious rebuild there costs
    GPU minutes."""
    h = hashlib.sha1()
    for name in sorted(UNITS):
        h.update(_unit_hash(*UNITS[name]).encode())
    return h.hexdigest()


def needs_build() -> bool:
    if not (os.path.exists(OUT) and os.path.exists(STAMP)):
        return True
    with open(STAMP) as f:
        return f.read().strip() != source_hash()


def _compile_unit(name, src, defines, headers, verbose=False):
    """Compile one unit into csrc/_obj/<name>.o unless an object with the same input hash is already there."""
    os.makedirs(OBJ, exist_ok=True)
    obj = os.path.join(OBJ, name + ".o")
    stamp = obj + ".stamp"
    want = _unit_hash(src, defines, headers)
    if os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read().strip() == want:
        return obj, ""
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc, *NVCC_FLAGS, *defines, "-c", os.path.join(CSRC, src), "-o", obj]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for unit {name}:\n{' '.join(cmd)}\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(want)
    return obj, r.stderr


def _link(objs, out):
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC", "-o", out, *objs]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{' '.join(cmd)}\n{r.stdout}\n{r.stderr}")


def _compile_all(units, verbose=False):
    jobs = min(len(units), int(os.environ.get("MPPI_B200_BUILD_JOBS", str(os.cpu_count() or 4))))
    objs, logs = {}, {}
    with concurrent.futures.ThreadPoolExecutor(max_workers=max(jobs, 1)) as ex:
        futs = {ex.submit(_compile_unit, name, *spec, verbose): name for name, spec in units.items()}
        for fut in concurrent.futures.as_completed(futs):
            objs[futs[fut]], logs[futs[fut]] = fut.result()
    if verbose:
        for name in sorted(logs):
            if logs[name]:
                print(f"==== {name}\n{logs[name]}")
    return [objs[n] for n in sorted(objs)]


class _BuildLock:
    """One builder at a time per tree: the ranks of a multi-GPU job that all find the library stale must not run nvcc
    into the same object files.  (flock on a file next to the library; released when the process ends, whatever happens.)"""

    def __enter__(self):
        import fcntl
        os.makedirs(OBJ, exist_ok=True)
        self._f = open(os.path.join(OBJ, ".build.lock"), "w")
        fcntl.flock(self._f, fcntl.LOCK_EX)
        return self

    def __exit__(self, *exc):
        import fcntl
        fcntl.flock(self._f, fcntl.LOCK_UN)
        self._f.close()
        return False


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return OUT
    with _BuildLock():
        if not force and not needs_build():        # another process built it while this one waited
            return OUT
        return _build_locked(force, verbose)


def _build_locked(force: bool, verbose: bool) -> str:
    h = source_hash()          # of the sources as compiled (taken before nvcc runs)
    if force:
        for name in UNITS:
            try:
                os.unlink(os.path.join(OBJ, name + ".o.stamp"))
            except OSError:
                pass
    objs = _compile_all(UNITS, verbose)
    tmp = OUT + f".{os.getpid()}.tmp"
    _link(objs, tmp)
    os.replace(tmp, OUT)
    with open(STAMP, "w") as f:
        f.write(h)
    # everything cached for user models was built from the previous sources: drop it (it is keyed by the source hash and
    # would never be used again, but it travels with every snapshot of the tree)
    udir = os.path.join(CSRC, "_user")
    if os.path.isdir(udir):
        for name in os.listdir(udir):
            try:
                os.unlink(os.path.join(udir, name))
            except OSError:
                pass
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
