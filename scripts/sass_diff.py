"""Compare the SASS of every kernel two builds of the library have in common (instructions and encodings, column
alignment ignored).  usage: sass_diff.py old.so new.so      (no GPU needed: cuobjdump)

Used in round 1 to show that adding the resident kernels (and the `bool` return of publish_and_finish they needed) left
all 130 kernels of the last fully GPU-tested library byte-identical."""
import re
import subprocess
import sys


def kernels(path):
    txt = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    out, cur = {}, None
    for line in txt.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            out[cur] = []
        elif cur is not None and "/*" in line:
            out[cur].append(re.sub(r"\s+", " ", line.strip()))
    return out


def main():
    old, new = kernels(sys.argv[1]), kernels(sys.argv[2])
    missing = [k for k in old if k not in new]
    differing = [k for k in old if k in new and old[k] != new[k]]
    print(f"{len(old)} kernels in {sys.argv[1]}, {len(new)} in {sys.argv[2]}: {len(missing)} missing, {len(differing)} differing, "
          f"{len(new) - len(old) + len(missing)} new")
    for k in missing:
        print("missing  ", subprocess.run(["c++filt", k], capture_output=True, text=True).stdout.strip()[:160])
    for k in differing:
        print("differing", subprocess.run(["c++filt", k], capture_output=True, text=True).stdout.strip()[:160])
    sys.exit(1 if missing or differing else 0)


if __name__ == "__main__":
    main()
