"""Why does a sharded command cost more back to back than its isolated timeline says?  Per rank (torchrun):
host enqueue time per command() (no synchronise: the first 400 calls after a sync fit the launch queue), device time
per command back to back (CUDA events over 2000), with and without programmatic dependent launch, and the same for an
unsharded controller on the same GPU.   usage: torchrun --nproc-per-node N scripts/b2b_multi_diag.py [K_per_gpu] [T]"""
import os
import sys

import torch
import torch.distributed as dist

import timing

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def run(tag, pdl, sharded, K, T, dev, x):
    os.environ["MPPI_B200_PDL"] = "1" if pdl else "0"
    import pytorch_mppi_b200 as eng
    pend = eng.Pendulum()
    torch.manual_seed(0)
    U0 = torch.randn(T, 1) * 3.16
    kw = dict(num_samples=K * (dist.get_world_size() if sharded else 1), horizon=T, u_min=torch.tensor(-2.0),
              u_max=torch.tensor(2.0), device=dev, rng_seed=1, U_init=U0)
    if sharded:
        kw["process_group"] = dist.group.WORLD
    c = eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), **kw)
    for _ in range(50):
        c.command(x)
    torch.cuda.synchronize()
    dist.barrier()
    host_us = timing.host_us(lambda: c.command(x), 400, warm=0)
    torch.cuda.synchronize()
    dist.barrier()
    dev_us = timing.back_to_back_us(lambda: c.command(x), 2000, warm=0, reps=1)
    li = c.launch_info
    print(f"rank {dist.get_rank()} {tag:28s} host enqueue {host_us:6.2f} us/command   device back to back {dev_us:6.2f} us/command   "
          f"grid {li.grid_blocks} cluster {li.cluster_size} records {li.xchg_records}", flush=True)
    dist.barrier()


def main():
    K = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
    T = int(sys.argv[2]) if len(sys.argv) > 2 else 30
    rank = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", device_id=dev)
    if rank == 0:
        print(timing.card(), flush=True)
    x = torch.tensor([3.14159, 1.0], device=dev)
    args = (K, T, dev, x)
    run("unsharded, PDL", True, False, *args)
    run("unsharded, no PDL", False, False, *args)
    run("sharded, PDL", True, True, *args)
    run("sharded, no PDL", False, True, *args)
    os.environ["MPPI_B200_XCHG_DIRECT"] = "0"
    run("sharded rank-record, PDL", True, True, *args)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
