"""Recipe for oracle/_ref/: an importable copy of the UNMODIFIED reference package, for use as a checker / CPU baseline.

TEST INFRASTRUCTURE ONLY (like everything under oracle/).  Run in the build container, where /root/reference exists:

    python oracle/make_ref.py

It copies the reference's pure-Python package files where they lie (`/root/reference/src/pytorch_mppi/{__init__,mppi}.py`)
and its own test-suite (`/root/reference/tests/test_mppi.py`, used by tests/test_gpu_ref_suite.py) into `oracle/_ref/`,
and writes the `arm_pytorch_utilities` stand-in next to them (tests/golden/_shim; the real dependency is not
vendored with the reference and there is no network).  `oracle/_ref/` is git-ignored — reference sources never enter
the history — but it travels with a copy of the working tree to a GPU machine, where `bench.py --impl reference`
and the `cpu_baseline` leg time it (kind "reference") and the reference's own tests run against the engine.
Nothing in the product imports it.
"""
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ.get("MPPI_REFERENCE_ROOT", "/root/reference")
OUT = os.path.join(HERE, "_ref")


def available() -> bool:
    return os.path.exists(os.path.join(OUT, "pytorch_mppi", "mppi.py"))


def make(force: bool = False) -> bool:
    """Returns True if oracle/_ref is in place afterwards (False: no reference tree here and none built earlier)."""
    src = os.path.join(REF, "src", "pytorch_mppi")
    if not os.path.isdir(src):
        return available()
    if available() and not force:
        return True
    pkg = os.path.join(OUT, "pytorch_mppi")
    os.makedirs(pkg, exist_ok=True)
    for name in ("__init__.py", "mppi.py"):
        shutil.copyfile(os.path.join(src, name), os.path.join(pkg, name))
    shim_src = os.path.join(ROOT, "tests", "golden", "_shim", "arm_pytorch_utilities")
    shim_dst = os.path.join(OUT, "arm_pytorch_utilities")
    os.makedirs(shim_dst, exist_ok=True)
    shutil.copyfile(os.path.join(shim_src, "__init__.py"), os.path.join(shim_dst, "__init__.py"))
    tests_dst = os.path.join(OUT, "tests")
    os.makedirs(tests_dst, exist_ok=True)
    shutil.copyfile(os.path.join(REF, "tests", "test_mppi.py"), os.path.join(tests_dst, "test_mppi.py"))
    # The same suite pointed at the ENGINE: the one-line device constant patched to CUDA (the engine has no CPU path),
    # and `pytorch_mppi` resolved to an alias package that re-exports pytorch_mppi_b200 (tests/test_gpu_ref_suite.py).
    with open(os.path.join(tests_dst, "test_mppi.py")) as f:
        text = f.read()
    assert text.count('DEVICE = "cpu"') == 1, "the reference suite's device constant moved"
    with open(os.path.join(tests_dst, "test_mppi_engine.py"), "w") as f:
        f.write(text.replace('DEVICE = "cpu"', 'DEVICE = "cuda"'))
    alias = os.path.join(OUT, "engine_alias", "pytorch_mppi")
    os.makedirs(alias, exist_ok=True)
    with open(os.path.join(alias, "__init__.py"), "w") as f:
        f.write("# alias written by oracle/make_ref.py: the reference's test-suite imports `pytorch_mppi`\n"
                "from pytorch_mppi_b200 import *  # noqa: F401,F403\n"
                "from pytorch_mppi_b200 import MPPI, SMPPI, KMPPI, MPPI_Batched  # noqa: F401\n")
    with open(os.path.join(alias, "mppi.py"), "w") as f:
        f.write("from pytorch_mppi_b200.mppi import *  # noqa: F401,F403\n"
                "from pytorch_mppi_b200.mppi import RBFKernel, SpecificActionSampler, TimeKernel  # noqa: F401\n")
    return True


def import_reference():
    """The live reference module (`pytorch_mppi.mppi`) from oracle/_ref, or None if it was never built."""
    if not available():
        return None
    if OUT not in sys.path:
        sys.path.insert(0, OUT)
    import importlib
    return importlib.import_module("pytorch_mppi.mppi")


if __name__ == "__main__":
    ok = make(force="--force" in sys.argv)
    print("oracle/_ref:", "ready" if ok else "reference tree not found (nothing built)")
