"""Tiny driver for ncu: n commands of one bench.py workload, built exactly as bench.py builds it.
usage: prof_workload.py <workload> [n]"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import pytorch_mppi_b200 as eng  # noqa: E402


def main():
    wl = bench.WORKLOADS[sys.argv[1]]
    n = int(sys.argv[2]) if len(sys.argv) > 2 else 30
    dev = torch.device("cuda", 0)
    ctrl = bench.make_engine(eng, wl, wl["K"], dev, None, "p2p")
    x = torch.tensor(wl["x0"], device=dev)
    for _ in range(n):
        a = ctrl.command(x)
    torch.cuda.synchronize()
    li = ctrl.launch_info
    print("done", a.tolist(), "grid", li.grid_x, "block", li.block_threads, "split", li.split_cost, "cluster", li.cluster_size)


if __name__ == "__main__":
    main()
