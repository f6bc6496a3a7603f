"""Where a resident command's time goes: %globaltimer stamps from the debug instantiation of the resident kernel
(resident_command_kernel<PendulumModel, float, V_MPPI, false, STAMPS = true>, chosen when the plan carries debug_clocks)
plus the host's own round-trip clock.  usage: resident_timeline.py [K] [T] [n]      (NOT under ncu)

Stamp slots (csrc/mppi_resident.cuh): 14 previous update visible | 0 prepared, polling | 13 (CTA 0) record seen in host
memory | 1 record seen by this CTA (board) | 2 decoded | 3 rolled out | 4 folded | 6 ticket taken | 8 / 10 / 11 finisher:
partials acquired / eta / numerators | 12 finisher: action stored, fence done, done word written."""
import os
import sys

import numpy as np
import torch

import timing

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402


def main():
    K = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
    T = int(sys.argv[2]) if len(sys.argv) > 2 else 30
    n = int(sys.argv[3]) if len(sys.argv) > 3 else 200
    pend = eng.Pendulum()
    ctrl = eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), num_samples=K, horizon=T,
                    u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda", rng_seed=1)
    x = [3.14159, 1.0]
    ctrl.command_host(x)
    nb = ctrl.launch_info.grid_blocks
    dbg = torch.zeros(nb, 16, dtype=torch.int64, device="cuda")
    ctrl._debug_clocks = dbg
    ctrl._dirty = True

    SLOTS = [(14, "previous update visible"), (0, "prepared, polling"), (13, "CTA 0: record seen (host memory)"),
             (1, "record seen (board)"), (2, "decoded"), (3, "rolled out"), (4, "folded"), (6, "ticket taken"),
             (8, "finisher: partials acquired"), (10, "finisher: eta"), (11, "finisher: numerators"),
             (12, "finisher: action + fence + done")]
    rows = {s: [] for s, _ in SLOTS}
    host_us = []
    side = torch.cuda.Stream()
    with ctrl.resident(idle_us=50000):
        for _ in range(50):
            ctrl.command_host(x)
        for _ in range(n):
            host_us.append(timing.host_us(lambda: ctrl.command_host(x), 1, warm=0))
            ctrl.cost_total                       # waits for the finisher's done word: every stamp of this command is written
            with torch.cuda.stream(side):         # the resident grid keeps its own stream; this copy must not wait for it
                d = dbg.to("cpu", non_blocking=False).numpy().astype(np.int64)
            ref = d[0, 13]                        # CTA 0 saw the record in host memory
            for s, _ in SLOTS:
                col = d[:, s]
                col = col[col > 0]
                if len(col):
                    rows[s].append(((col.min() - ref) / 1e3, (np.median(col) - ref) / 1e3, (col.max() - ref) / 1e3))
    print(f"K={K} T={T} grid={nb} block={ctrl.launch_info.block_threads}: {n} resident commands, launches={ctrl.resident_launches}")
    print(f"host round trip (command_host, Python): median {np.median(host_us):.2f} us, min {np.min(host_us):.2f}")
    print("GPU side, microseconds relative to CTA 0 seeing the record (median over commands of the per-command min / median / max over CTAs):")
    for s, name in SLOTS:
        if rows[s]:
            a = np.array(rows[s])
            print(f"  {name:36s} {np.median(a[:, 0]):8.2f} {np.median(a[:, 1]):8.2f} {np.median(a[:, 2]):8.2f}")


if __name__ == "__main__":
    main()
