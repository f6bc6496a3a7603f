"""GPU diagnostic: per-case parity table + quick command() timing.  usage: gpu_diag.py [out.txt] (default: stdout only)"""
import os
import sys
import traceback

import numpy as np
import torch

import timing

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.golden.cases import BASE, CASES  # noqa: E402
from tests.golden.replay import OracleRunner, load  # noqa: E402

out = None


def P(*a):
    s = " ".join(str(x) for x in a)
    print(s, flush=True)
    if out is not None:
        out.write(s + "\n")
        out.flush()


def parity():
    for route in ("fused", "stepped"):
        for name in sorted(CASES):
            case, gold = load(name)
            if route not in BASE.routes(name, case):
                continue
            try:
                run = OracleRunner(case, gold)
                ctrl = BASE.engine(case, gold, run.stream.U0, route)
                errs, cerrs = [], []
                for step in range(case["steps"]):
                    z = run.stream.next_z()
                    ctrl.inject_noise(z)
                    xg = torch.from_numpy(gold[f"x_{step}"]).to(run.prob.dtype)
                    ctrl.command(xg.numpy())
                    errs.append(float(np.abs(ctrl.U.cpu().numpy() - gold[f"U_{step}"]).max()))
                    if f"cost_total_{step}" in gold:
                        c = ctrl.cost_total.cpu().numpy()
                        cerrs.append(float(np.abs(c - gold[f"cost_total_{step}"]).max() / np.abs(gold[f"cost_total_{step}"]).max()))
                    ctrl.U = torch.from_numpy(gold[f"U_{step}"])
                    if case["variant"] == "smppi":
                        ctrl.action_sequence = torch.from_numpy(gold[f"A_{step}"])
                    if case["variant"] == "kmppi":
                        ctrl.theta = torch.from_numpy(gold[f"theta_{step}"])
                info = getattr(ctrl, "launch_info", None)
                geo = "" if info is None else f"grid={info.grid_blocks} block={info.block_threads} smem={info.smem_bytes} regs={info.regs_per_thread} occ={info.max_blocks_per_sm} tma={info.tma_staging}"
                P(f"{route:8s} {name:28s} maxUerr={max(errs):.3e} relCostErr={max(cerrs) if cerrs else float('nan'):.3e} {geo}")
            except Exception:
                P(f"{route:8s} {name:28s} EXCEPTION\n{traceback.format_exc()}")

    # fp32 noise-floor table at C2 (SURVEY §8d): engine32 vs ref32, engine32 vs ref64, ref32 vs ref64
    try:
        case, g32 = load("pendulum_c2_f32")
        _, g64 = load("pendulum_c2_f64")
        run = OracleRunner(case)
        ctrl = BASE.engine(case, g32, run.stream.U0, "fused")
        ctrl.inject_noise(run.stream.next_z())
        ctrl.command(np.asarray(case["x0"]))
        Ue = ctrl.U.cpu().numpy().astype(np.float64)
        P("C2 step0: err(engine32,ref32)=%.3e err(engine32,ref64)=%.3e err(ref32,ref64)=%.3e" % (
            np.abs(Ue - g32["U_0"]).max(), np.abs(Ue - g64["U_0"]).max(), np.abs(g32["U_0"].astype(np.float64) - g64["U_0"]).max()))
    except Exception:
        P("noise floor table EXCEPTION\n" + traceback.format_exc())


def timings():
    import pytorch_mppi_b200 as eng
    pend = eng.Pendulum()
    for K, T, bt, tps in ((16384, 30, 0, 0), (16384, 30, 128, 1), (16384, 30, 128, 2), (16384, 30, 128, 4), (16384, 30, 64, 4), (16384, 30, 64, 2), (16384, 30, 32, 4), (16384, 30, 256, 2),
                          (131072, 50, 0, 0), (131072, 50, 128, 2), (131072, 50, 256, 1), (131072, 50, 512, 1), (1 << 20, 50, 0, 0), (1 << 20, 50, 128, 1), (1 << 20, 50, 512, 1)):
        try:
            ctrl = eng.MPPI(pend.dynamics, pend.running_cost, 2, torch.tensor(10.0), num_samples=K, horizon=T,
                            u_min=torch.tensor(-2.0), u_max=torch.tensor(2.0), device="cuda", rng_seed=1, block_threads=bt, threads_per_sample=tps)
            x = [3.14159, 1.0]
            n = 200 if K <= 131072 else 50

            def window():
                for _ in range(n):
                    ctrl.command(x)
                torch.cuda.synchronize()
            dev = timing.back_to_back_us(lambda: ctrl.command(x), n)
            wall = timing.host_us(window, 1, warm=0) / n
            info = ctrl.launch_info
            P(f"time K={K} T={T} bt={bt} tps={tps}->{info.threads_per_sample}: device {dev:.2f} us/command, wall {wall:.2f} us/command, grid={info.grid_blocks} block={info.block_threads} occ={info.max_blocks_per_sm} -> {K*T/dev:.1f} M rollout-steps/s")
            # e2e: host state in, action to host
            P(f"     e2e (host state -> action.cpu()): {timing.host_us(lambda: ctrl.command(x).cpu(), n):.2f} us/command")
            P(f"     e2e (command_host, pinned mailbox):  {timing.host_us(lambda: ctrl.command_host(x), n):.2f} us/command")
        except Exception:
            P(f"time K={K} EXCEPTION\n{traceback.format_exc()}")


def main():
    global out
    out = open(sys.argv[1], "w") if len(sys.argv) > 1 else None
    P(timing.card(), torch.__version__)
    parity()
    timings()
    if out is not None:
        out.close()


if __name__ == "__main__":
    main()
