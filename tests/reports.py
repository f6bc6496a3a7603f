"""Diagnostic reports of the GPU tests (measured parity errors, host-loop latencies, the reference suite's per-test
outcome), written to tests/_reports/ (git-ignored) inside the tree the tests run from.  A report that cannot be
written is dropped: it never fails a test."""
import json
import os

DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_reports")


def write(name: str, text: str) -> None:
    try:
        os.makedirs(DIR, exist_ok=True)
        with open(os.path.join(DIR, name), "w") as f:
            f.write(text)
    except OSError:
        pass


_WORST = {}


def worst(name: str, key: str, err) -> None:
    """Keeps the largest `err` seen under `key` in the JSON report `name`, across every test module of the session."""
    table = _WORST.setdefault(name, {})
    table[key] = max(table.get(key, 0.0), float(err))
    write(name, json.dumps(table, indent=1, sort_keys=True))
