"""GPU: the reference's OWN test-suite (its tests/test_mppi.py, 73 tests; its CI gate is
.github/workflows/tests.yml:28-29) run against the engine.

`oracle/make_ref.py` (run by build() where the reference sources are available) writes an engine-pointed copy of that file into
the git-ignored `oracle/_ref/tests/test_mppi_engine.py` — identical except for the one-line `DEVICE = "cpu"` ->
`"cuda"` (the engine has no CPU path) — and an alias package so that `from pytorch_mppi import MPPI, ...` resolves to
`pytorch_mppi_b200`.  This test runs it in a subprocess and checks the outcome test by test: everything must pass except
the entries of EXPECTED_FAIL, each with the reason it cannot hold for a CUDA-only engine.  The per-test report is
written to tests/_reports/ref_suite_report.txt (tests/reports.py).
"""
import os
import re
import subprocess
import sys

import pytest

from tests import reports

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SUITE = os.path.join(ROOT, "oracle", "_ref", "tests", "test_mppi_engine.py")
ALIAS = os.path.join(ROOT, "oracle", "_ref", "engine_alias")

# test id (Class::name) -> why it cannot pass against this engine.
EXPECTED_FAIL = {
}


def test_reference_suite_against_the_engine():
    if not os.path.exists(SUITE):
        pytest.skip("oracle/_ref not built (python oracle/make_ref.py where the reference sources are available)")
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([ALIAS, ROOT, env.get("PYTHONPATH", "")])
    r = subprocess.run([sys.executable, "-m", "pytest", SUITE, "-q", "-rA", "--no-header", "-p", "no:cacheprovider",
                        "--rootdir", os.path.dirname(SUITE), "-c", os.devnull],
                       capture_output=True, text=True, timeout=1800, cwd=os.path.dirname(SUITE), env=env)
    out = r.stdout + "\n" + r.stderr
    results = {}
    for m in re.finditer(r"^(PASSED|FAILED|ERROR|SKIPPED|XFAIL|XPASS)\s+\S*test_mppi_engine\.py::(\S+)", out, re.M):
        results[m.group(2)] = m.group(1)
    try:
        assert len(results) >= 70, f"suite did not run: {out[-3000:]}"
        bad = {k: v for k, v in results.items() if v not in ("PASSED", "SKIPPED") and k not in EXPECTED_FAIL}
        stale = [k for k in EXPECTED_FAIL if results.get(k) == "PASSED"]
        assert not bad, f"unexpected failures against the engine: {bad}\n{out[-4000:]}"
        assert not stale, f"listed as expected failures but passing: {stale}"
    finally:
        n_pass = sum(v == "PASSED" for v in results.values())
        lines = [f"reference suite against pytorch_mppi_b200: {n_pass} passed of {len(results)}"]
        lines += [f"{results[k]:8s} {k}" + (f"    # expected: {EXPECTED_FAIL[k]}" if k in EXPECTED_FAIL else "") for k in sorted(results)]
        reports.write("ref_suite_report.txt", "\n".join(lines) + "\n\n---- raw tail ----\n" + out[-6000:])
