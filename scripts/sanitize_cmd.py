"""Driver for compute-sanitizer (memcheck / racecheck / synccheck): a few commands of every kernel family, small sizes.
usage: sanitize_cmd.py [fused|tc|resident|batched|stepped|multi]      (multi: torchrun --nproc-per-node 2)"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng  # noqa: E402


def main():
    what = sys.argv[1] if len(sys.argv) > 1 else "fused"
    dev = "cuda"
    pend = eng.Pendulum()
    nav = eng.LinearPoint.toy2d_nav()

    def pendulum(K=2048, T=15, **kw):
        return eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), num_samples=K, horizon=T, u_min=torch.tensor(-2.0),
                        u_max=torch.tensor(2.0), device=dev, rng_seed=3, **kw)

    if what == "fused":
        ctrls = [pendulum(), pendulum(K=4096 + 37, T=12),
                 eng.SMPPI(nav.dynamics, nav.running_cost, 2, torch.eye(2), num_samples=1024, horizon=12, device=dev, rng_seed=1,
                           terminal_state_cost=nav.terminal_cost, w_action_seq_cost=5.0, action_max=torch.tensor([1.0, 1.0])),
                 eng.KMPPI(nav.dynamics, nav.running_cost, 2, torch.eye(2), num_samples=1024, horizon=12, device=dev, rng_seed=1,
                           terminal_state_cost=nav.terminal_cost, num_support_pts=4, kernel=eng.RBFKernel(sigma=2))]
        for c in ctrls:
            x = [3.0, 0.5] if c.nu == 1 else [-3.0, -2.0]
            for _ in range(3):
                a = c.command(x)
            ah = c.command_host(x)
            torch.cuda.synchronize()
            print(type(c).__name__, c.launch_info.grid_blocks, c.launch_info.cluster_size, float(a.abs().sum()), float(ah.abs().sum()))
        big = pendulum(K=70000, T=10)          # multi-tile grid: ticket mode
        for _ in range(2):
            big.command([3.0, 0.5])
        torch.cuda.synchronize()
        print("big", big.launch_info.grid_blocks, big.launch_info.cluster_size, big.launch_info.xchg_records)
    elif what == "tc":
        torch.manual_seed(25)
        net = torch.nn.Sequential(torch.nn.Linear(3, 32), torch.nn.Tanh(), torch.nn.Linear(32, 32), torch.nn.Tanh(), torch.nn.Linear(32, 2)).to(dev)
        for mode in ("bf16x3", "bf16"):
            m = eng.PendulumMLP(net, tensor_cores=mode)
            c = eng.MPPI(m.dynamics, m.running_cost, 2, torch.tensor(1.0), num_samples=1024, horizon=8, u_min=torch.tensor(-2.0),
                         u_max=torch.tensor(2.0), device=dev, rng_seed=1)
            for _ in range(2):
                a = c.command([3.0, 0.5])
            torch.cuda.synchronize()
            print("tc", mode, c.launch_info.grid_blocks, c.launch_info.block_threads, float(a))
    elif what == "resident":
        c = pendulum(K=4096, T=12)
        c.start_resident(idle_us=500000)
        for i in range(100):
            a = c.command_host([3.0, 0.5 + 0.001 * i])
        c.stop_resident()
        torch.cuda.synchronize()
        print("resident", c.resident_launches, float(a))
    elif what == "batched":
        lin = eng.LinearPoint.unit_test_env()
        c = eng.MPPI_Batched(lin.dynamics, lin.running_cost, 2, torch.eye(2), num_envs=4, num_samples=300, horizon=8, device=dev, rng_seed=1)
        for _ in range(2):
            a = c.command(torch.zeros(4, 2, device=dev))
        torch.cuda.synchronize()
        print("batched", a.shape)
    elif what == "stepped":
        lin = eng.LinearPoint.unit_test_env()
        c = eng.MPPI(lambda s, a: lin.dynamics(s, a), lambda s, a: lin.running_cost(s, a), 2, torch.eye(2), num_samples=300, horizon=6,
                     device=dev, rng_seed=1, rollout_samples=2, rollout_var_cost=0.5)
        for _ in range(2):
            a = c.command([0.0, 0.0])
        torch.cuda.synchronize()
        print("stepped", a)
    elif what == "multi":
        import torch.distributed as dist
        rank = int(os.environ["LOCAL_RANK"])
        torch.cuda.set_device(rank)
        dev = torch.device("cuda", rank)
        dist.init_process_group("nccl", device_id=dev)
        c = eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), num_samples=8192, horizon=15, u_min=torch.tensor(-2.0),
                     u_max=torch.tensor(2.0), device=dev, rng_seed=3, process_group=dist.group.WORLD)
        for _ in range(3):
            a = c.command([3.0, 0.5])
        torch.cuda.synchronize()
        print("multi", rank, c.launch_info.xchg_records, float(a))
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
