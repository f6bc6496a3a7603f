"""Cold against warm phase timeline of one bench.py command (%globaltimer stamps 0-12 of the fused kernel).
usage: phase_clocks_cold.py [workload] [reps]          (default: pendulum_c2, 30 repetitions)

The controller is bench.py's (make_engine, same seed), the state a device tensor as bench.py passes it.  Each repetition
stamps one command twice, in alternation:
  warm  the command right after the previous one (instructions and data still in L2)
  cold  the command right after the 256 MiB zero_() that bench.py runs before every timed step
Each phase is reported as the median over the repetitions of its duration on the finisher (CTA 0, the leader of
cluster 0), warm, cold and cold - warm.  Transform, warp fold and the cluster combine touch no global memory (the tile
and the records live in shared memory): what they gain when cold is instruction fetch.  So is what the tail (stamps
6 -> 11) gains, beyond the collect's polls of the mailbox words."""
import os
import sys

import numpy as np
import torch

import timing

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import pytorch_mppi_b200 as eng  # noqa: E402

# (label, stamp at the start, stamp at the end) on the finisher's path; "start" is the earliest CTA's stamp 0
PHASES = [("launch -> CTA 0 start", "t0", 0), ("fill normals of tile 0, PDL wait, TMA issue", 0, 1),
          ("nominal staged (TMA wait, shift)", 1, 2),
          ("transform", 2, 3), ("rollout (state load, recurrence, costs)", 3, 4), ("warp fold", 4, 5),
          ("cluster barrier (DSMEM records)", 5, 6), ("cluster combine", 6, 9), ("publish", 9, 8),
          ("collect (waits for the last cluster)", 8, 12), ("final combine", 12, 10), ("-> finish_update", 10, 11),
          ("finish_update", 11, 7)]
TAIL = [p[0] for p in PHASES if p[1] in (6, 9, 8, 12, 10, 11)]
MEM_FREE = ["transform", "warp fold", "cluster combine"]


def one(ctrl, x_dev, dbg, cold):
    dbg.zero_()
    if cold:
        timing.flush_l2()
    else:
        torch.cuda.synchronize()
    ctrl.command(x_dev)
    torch.cuda.synchronize()
    d = dbg.cpu().numpy().astype(np.int64)
    t = {"t0": d[:, 0].min()}
    for s in range(13):
        t[s] = d[0, s]
    out = {name: (t[b] - t[a]) / 1e3 for name, a, b in PHASES}
    out["command (t0 -> CTA 0 exit)"] = (t[7] - t["t0"]) / 1e3
    out["last CTA folded (t0 -> max stamp 5)"] = (d[:, 5].max() - t["t0"]) / 1e3
    return out


def main():
    wl_name = sys.argv[1] if len(sys.argv) > 1 else "pendulum_c2"
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 30
    wl = bench.WORKLOADS[wl_name]
    dev = torch.device("cuda", 0)
    ctrl = bench.make_engine(eng, wl, wl["K"], dev, None, "p2p")
    x_dev = torch.tensor(wl["x0"], dtype=torch.float32, device=dev)
    for _ in range(5):
        ctrl.command(x_dev)
    torch.cuda.synchronize()
    info = ctrl.launch_info
    dbg = torch.zeros(info.grid_blocks, 16, dtype=torch.int64, device=dev)
    ctrl._debug_clocks = dbg
    ctrl._dirty = True
    ctrl.command(x_dev)
    torch.cuda.synchronize()

    runs = {False: [], True: []}
    for _ in range(reps):
        for cold in (False, True):
            runs[cold].append(one(ctrl, x_dev, dbg, cold))
    names = list(runs[False][0])
    med = {c: {n: float(np.median([r[n] for r in runs[c]])) for n in names} for c in (False, True)}
    print(f"{wl_name}: {timing.card()}; grid {info.grid_blocks} x {info.block_threads} threads, "
          f"cluster {info.cluster_size}, split {info.split_cost}, records {info.xchg_records}, "
          f"ll_tail {getattr(info, 'll_tail', 0)}; median of {reps} repetitions")
    print(f"{'phase (CTA 0)':44s} {'warm us':>8s} {'cold us':>8s} {'cold-warm':>9s}")
    for n in names:
        print(f"{n:44s} {med[False][n]:8.2f} {med[True][n]:8.2f} {med[True][n] - med[False][n]:9.2f}")
    tail = sum(med[True][n] - med[False][n] for n in TAIL)
    mem_free = sum(med[True][n] - med[False][n] for n in MEM_FREE if n not in TAIL)
    print(f"tail stages (stamps 6 -> 11) cold - warm: {tail:.2f} us; other memory-free phases: {mem_free:.2f} us; "
          f"together {tail + mem_free:.2f} us")


if __name__ == "__main__":
    main()
