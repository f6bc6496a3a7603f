"""Phase timeline of the sharded fused kernel (%globaltimer stamps), one process per GPU:
   python -m torch.distributed.run --nproc-per-node N scripts/phase_clocks_multi.py [K_per_gpu] [T]
Prints, per rank, the stamps of the finisher CTA relative to the EARLIEST kernel start over all ranks (the GPUs' global
timers are synchronised to well under a microsecond on one NVSwitch box; the offsets printed first show by how much)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402


def main():
    K = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
    T = int(sys.argv[2]) if len(sys.argv) > 2 else 30
    rank = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", device_id=dev)
    world = dist.get_world_size()
    pend = eng.Pendulum()
    ctrl = eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), num_samples=K * world, horizon=T, u_min=torch.tensor(-2.0),
                    u_max=torch.tensor(2.0), device=dev, rng_seed=1, process_group=dist.group.WORLD)
    x = [3.14159, 1.0]
    for _ in range(20):
        ctrl.command(x)
    nb = ctrl.launch_info.grid_blocks
    dbg = torch.zeros(nb, 16, dtype=torch.int64, device=dev)
    ctrl._debug_clocks = dbg
    ctrl._dirty = True
    names = {0: "start", 3: "transformed", 4: "rolled", 5: "folded", 6: "tail entered (cluster barrier)", 9: "cluster record combined",
             8: "L: record published", 12: "L: all records collected", 10: "L: records combined", 11: "L: numerators", 7: "CTA exit"}
    for rep in range(4):
        dbg.zero_()
        dist.barrier()
        torch.cuda.synchronize()
        for _ in range(3):           # back to back: the last one is measured in steady state
            dbg.zero_()
            ctrl.command(x)
        torch.cuda.synchronize()
        d = dbg.cpu().numpy().astype(np.int64)
        t_start = torch.tensor([int(d[:, 0][d[:, 0] > 0].min())], dtype=torch.int64, device=dev)
        starts = [torch.zeros_like(t_start) for _ in range(world)]
        dist.all_gather(starts, t_start)
        t0 = int(t_start.item())      # per rank: the GPUs' global timers are NOT synchronised (measured: 0.4 s apart)
        lines = [f"rep {rep} rank {rank}: start offset {(int(t_start.item()) - t0) / 1e3:.2f} us  grid={nb} cluster={ctrl.launch_info.cluster_size} records={ctrl.launch_info.xchg_records}"]
        for slot, n in names.items():
            col = d[:, slot]
            col = col[col > 0]
            if len(col):
                lines.append(f"    {n:32s} min {(col.min() - t0) / 1e3:7.2f}  median {(np.median(col) - t0) / 1e3:7.2f}  max {(col.max() - t0) / 1e3:7.2f}")
        for r in range(world):
            if r == rank and rep >= 2:
                print("\n".join(lines), flush=True)
            dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
