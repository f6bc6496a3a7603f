"""Diagnostic reports of the GPU tests (measured parity errors, host-loop latencies, the reference suite's per-test
outcome), written to tests/_reports/ (git-ignored) inside the tree the tests run from.  A report that cannot be
written is dropped: it never fails a test."""
import os

DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_reports")


def write(name: str, text: str) -> None:
    try:
        os.makedirs(DIR, exist_ok=True)
        with open(os.path.join(DIR, name), "w") as f:
            f.write(text)
    except OSError:
        pass
