"""What the pendulum's rollout recurrence loop contains, read from the SASS of a built library (no GPU needed: cuobjdump).
usage: sass_rollout_loop.py [lib.so] [kernel-substring]
  default kernel: the C2 command kernel, fused_command_kernel_ll<PendulumModel, float, MPPI> (split-cost, single-GPU LL tail)

The recurrence loop is the innermost backward branch whose body multiplies by 2/pi (the sine's quadrant); between its
head and its back-edge the script counts every instruction, the float <-> int conversions (F2I, I2F, I2FP), the
convergence barriers (BSSY, BSYNC), the branches other than the back-edge, the calls and the constant-bank loads."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "pytorch_mppi_b200", "csrc", "libmppi_b200.so")
    want = sys.argv[2] if len(sys.argv) > 2 else "fused_command_kernel_llINS_13PendulumModelEfLi0EE"

    txt = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    code, cur = [], None
    for line in txt.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;", line)
        if cur is not None and want in cur and m:
            code.append((int(m.group(1), 16), re.sub(r"\s+", " ", m.group(2))))
        elif cur is not None and want not in cur and code:
            break
    if not code:
        sys.exit(f"no kernel matching {want!r} in {lib}")

    loops = []
    for i, (addr, ins) in enumerate(code):
        m = re.search(r"\bBRA (?:`\(\.L_x_\d+\) )?0x([0-9a-f]+)", ins) or re.search(r"\bBRA 0x([0-9a-f]+)", ins)
        if m and int(m.group(1), 16) < addr:
            head = int(m.group(1), 16)
            body = [c for c in code if head <= c[0] <= addr]
            if any("0.63661974668502807617" in c[1] for c in body):
                loops.append((addr - head, head, addr, body))
    if not loops:
        sys.exit("no backward branch around the 2/pi multiply: the recurrence loop was not found")
    _, head, back, body = min(loops)

    def opcode(ins):
        return re.sub(r"^@!?U?P[T\d]+ ", "", ins).split(" ")[0]

    ops = collections.Counter(opcode(ins) for _, ins in body)
    count = lambda *names: sum(n for op, n in ops.items() if op.split(".")[0] in names)  # noqa: E731
    branches = [ins for a, ins in body if opcode(ins).startswith("BRA") and a != back]
    print(f"kernel {want} in {lib}")
    print(f"recurrence loop {head:#x} .. {back:#x} (back-edge): {len(body)} instructions")
    print(f"  F2I/I2F/I2FP conversions: {count('F2I', 'I2F', 'I2FP')}")
    print(f"  BSSY/BSYNC:               {count('BSSY', 'BSYNC')}")
    print(f"  branches (not the back-edge): {len(branches)}")
    print(f"  calls:                    {count('CALL')}")
    print(f"  LDC (constant-bank loads): {count('LDC')}")
    print("  opcodes: " + ", ".join(f"{op} {n}" for op, n in sorted(ops.items(), key=lambda kv: -kv[1])))


if __name__ == "__main__":
    main()
