"""The measurement scripts under scripts/: each imports without running anything, only scripts/timing.py takes a time
or reads the card, and scripts/README.md lists exactly the scripts there are.  No GPU needed."""
import ast
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPTS = os.path.join(ROOT, "scripts")


def python_sources():
    return sorted(os.path.relpath(os.path.join(d, f), SCRIPTS)
                  for d, _, fs in os.walk(SCRIPTS) for f in fs if f.endswith(".py"))


def test_every_script_imports_without_running():
    # in a fresh interpreter with no CUDA device visible: a script that measured, or read its arguments, at import
    # raises there
    probe = """
import importlib.util, json, os, sys, traceback
root, scripts = sys.argv[1], sys.argv[2]
sys.path[:0] = [scripts, root]
failed = {}
for name in sys.argv[3:]:
    spec = importlib.util.spec_from_file_location("script_" + name[:-3].replace(os.sep, "_"), os.path.join(scripts, name))
    try:
        spec.loader.exec_module(importlib.util.module_from_spec(spec))
    except BaseException:
        failed[name] = traceback.format_exc(limit=-2)
print(json.dumps(failed))
"""
    scripts = [s for s in python_sources() if os.sep not in s]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONDONTWRITEBYTECODE="1")
    python = [sys.executable, "-s"] if sys.flags.no_user_site else [sys.executable]
    r = subprocess.run([*python, "-c", probe, ROOT, SCRIPTS, *scripts], capture_output=True, text=True, env=env,
                       cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr
    failed = json.loads(r.stdout.strip().splitlines()[-1])
    assert not failed, "\n".join(f"{k}:\n{v}" for k, v in failed.items())


def test_every_script_ends_in_a_main_guard():
    for name in python_sources():
        if name == "timing.py":
            continue
        last = ast.parse(open(os.path.join(SCRIPTS, name)).read()).body[-1]
        assert isinstance(last, ast.If) and ast.unparse(last.test) == "__name__ == '__main__'", name


def test_only_timing_module_times():
    """CUDA events, elapsed_time, perf_counter and the card query belong to scripts/timing.py alone."""
    banned = {"Event", "elapsed_time", "perf_counter", "perf_counter_ns"}
    for name in python_sources():
        if name == "timing.py":
            continue
        for node in ast.walk(ast.parse(open(os.path.join(SCRIPTS, name)).read())):
            used = (node.attr if isinstance(node, ast.Attribute) else node.id if isinstance(node, ast.Name)
                    else node.name if isinstance(node, ast.alias) else None)
            assert used not in banned, f"{name}:{getattr(node, 'lineno', '')} uses {used}; time through scripts/timing.py"
            if isinstance(node, ast.Constant) and isinstance(node.value, str):
                assert not node.value.startswith("nvidia-smi"), f"{name}:{node.lineno} queries the card; use timing.card()"


def test_readme_lists_every_script():
    readme = open(os.path.join(SCRIPTS, "README.md")).read()
    listed = set()
    for line in readme.splitlines():
        if line.startswith("|") and not line.startswith("|---"):
            listed |= set(re.findall(r"`([\w/]+\.(?:py|cu))", line.split("|")[1]))
    present = set(python_sources()) | {os.path.relpath(os.path.join(d, f), SCRIPTS)
                                       for d, _, fs in os.walk(SCRIPTS) for f in fs if f.endswith(".cu")}
    assert present - listed == set(), "not in scripts/README.md"
    assert listed - present == set(), "named in scripts/README.md but missing"
