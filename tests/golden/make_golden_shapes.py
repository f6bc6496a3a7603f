"""Generate tests/golden/shape_*.npz (tests/golden/shape_cases.py) by running the LIVE reference with the torch twins of
tests/shape_models.py on injected standard-normal draws, and pin the oracle bit for bit against it: the cases go through
make_golden.py's runners, which assert `torch.equal(oracle, reference)` on every intermediate they write.

Run only where the reference sources are available:

    python tests/golden/make_golden_shapes.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import run_batched_case, run_case  # noqa: E402  (puts the reference and the repository on sys.path)
from tests.golden.shape_cases import SHAPE_BATCHED_CASES, SHAPE_CASES  # noqa: E402


def main():
    torch.set_num_threads(1)   # fixed reduction order inside ATen sums
    only = set(sys.argv[1:])
    for table, runner in ((SHAPE_CASES, run_case), (SHAPE_BATCHED_CASES, run_batched_case)):
        for name, case in table.items():
            if only and name not in only:
                continue
            path = os.path.join(HERE, f"{name}.npz")
            np.savez_compressed(path, **runner(name, case))
            print(f"{name}: oracle == reference over {case['steps']} step(s); wrote {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
