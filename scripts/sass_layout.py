"""Instruction layout of a command kernel, read from the SASS of a built library (no GPU needed: cuobjdump).
usage: sass_layout.py [lib.so] [kernel-substring ...]
  default kernels: the two split-cost pendulum fp32 MPPI kernels — fused_command_kernel_ll (what C2 runs: one GPU, LL
  mode) and fused_command_kernel<..., split-cost> (every other split-cost plan)

For each kernel: its total size, the size of its body (the kernel's own code; the out-of-line functions it calls follow
it), and the CALL sites in the body — all of them, and those of the tail (from the first cluster-barrier wait, where
warp_tail starts, to the end of the body), with the size of each routine a tail call jumps to."""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "pytorch_mppi_b200", "csrc", "libmppi_b200.so")
    wants = sys.argv[2:] or ["fused_command_kernel_llINS_13PendulumModelEfLi0EE",
                             "fused_command_kernelINS_13PendulumModelEfLi0ELb0ELb1ELi1E"]

    txt = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in txt.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;", line)
        if cur is not None and m:
            cur.append((int(m.group(1), 16), re.sub(r"\s+", " ", m.group(2))))

    for want in wants:
        names = [k for k in funcs if want in k]
        if not names:
            sys.exit(f"no kernel matching {want!r} in {lib}")
        code = funcs[names[0]]
        end = code[-1][0] + 16
        calls = [(a, int(m.group(1), 16)) for a, ins in code for m in [re.search(r"\bCALL\.\S+ 0x([0-9a-f]+)", ins)] if m]
        targets = sorted({t for _, t in calls})
        body_end = targets[0] if targets else end
        waits = [a for a, ins in code if "CGABAR_WAIT" in ins and a < body_end]
        tail_start = waits[0] if waits else None
        bounds = targets + [end]
        size_of = {t: bounds[i + 1] - t for i, t in enumerate(targets)}
        print(f"{names[0]}")
        print(f"  total {len(code)} instructions ({end / 1024:.1f} KB), body {body_end // 16} instructions ({body_end / 1024:.1f} KB), "
              f"out-of-line routines {len(targets)} ({(end - body_end) / 1024:.1f} KB)")
        print(f"  CALL sites in the body: {len(calls)}")
        if tail_start is None:
            print("  no cluster-barrier wait in the body: tail not located")
            continue
        tail = [(a, t) for a, t in calls if a >= tail_start]
        print(f"  tail {tail_start:#x} .. {body_end:#x} ({(body_end - tail_start) // 16} instructions): {len(tail)} CALL sites")
        for a, t in tail:
            print(f"    {a:#07x} -> {t:#x} ({size_of[t] // 16} instructions)")


if __name__ == "__main__":
    main()
