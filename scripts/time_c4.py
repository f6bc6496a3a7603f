"""BASELINE config 4 (MLP dynamics, K=32768, T=30): fused route vs stepped route, device time per command."""
import os, sys, copy
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_mppi_b200 as eng
torch.manual_seed(25)
net = torch.nn.Sequential(torch.nn.Linear(3, 32), torch.nn.Tanh(), torch.nn.Linear(32, 32), torch.nn.Tanh(), torch.nn.Linear(32, 2)).cuda()
K, T = 32768, 30
def run(name, dyn, cost, n, **kw):
    c = eng.MPPI(dyn, cost, 2, torch.tensor(1.0), num_samples=K, horizon=T, u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0),
                 device="cuda", rng_seed=1, **kw)
    x = [3.0, 0.5]
    for _ in range(5): c.command(x)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): c.command(x)
    e1.record(); torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / n * 1e3
    info = getattr(c, "launch_info", None)
    geo = "" if info is None or c._model is None else f" grid={info.grid_blocks} block={info.block_threads} regs={info.regs_per_thread} smem={info.smem_bytes} occ={info.max_blocks_per_sm}"
    print(f"{name}: {us:.1f} us/command -> {K*T/us/1e3:.2f} G rollout-steps/s, {2368*K*T/us/1e6:.2f} TFLOP/s of MLP math{geo}")
for fast in (False, True):
    m = eng.PendulumMLP(net, fast_tanh=fast)
    run(f"fused   fp32 fast_tanh={fast}", m.dynamics, m.running_cost, 50)
    for bt in (128, 256):
        run(f"fused   fp32 fast_tanh={fast} bt={bt}", m.dynamics, m.running_cost, 50, block_threads=bt)
for mode in ("bf16x3", "bf16"):
    for fast in (False, True):
        m = eng.PendulumMLP(net, fast_tanh=fast, tensor_cores=mode)
        run(f"fused   wgmma {mode} fast_tanh={fast}", m.dynamics, m.running_cost, 50)
m = eng.PendulumMLP(net)
run("stepped fp32 (torch MLP, Python T-loop)", lambda s, a: m.dynamics(s, a), lambda s, a: m.running_cost(s, a), 10)
c = eng.MPPI(lambda s, a: m.dynamics(s, a), lambda s, a: m.running_cost(s, a), 2, torch.tensor(1.0), num_samples=K, horizon=T,
             u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda", rng_seed=1)
c.compile()
x = [3.0, 0.5]
for _ in range(5): c.command(x)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(20): c.command(x)
e1.record(); torch.cuda.synchronize()
print(f"stepped fp32 + compile() (CUDA graph replay): {e0.elapsed_time(e1)/20*1e3:.1f} us/command")
