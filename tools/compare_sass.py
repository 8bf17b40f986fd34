"""Compare the SASS of two builds of libmppi_b200.so kernel by kernel, e.g. a change against its parent commit:

    python tools/compare_sass.py OLD.so NEW.so \
        [--rename 'rollout_kernel_ar_ws<mppib::plugins::ARStandardCost, =rollout_kernel_ar_ws<']

Each kernel's instructions are read with `cuobjdump -sass`, without addresses and encodings, and matched by demangled
name. --rename FROM=TO rewrites a substring of NEW's names, for example to drop a template argument a change added (the
cost parameter of rollout_kernel_ar_ws), so that the old and new instantiations pair up. Prints one line per kernel of
OLD (SAME / DIFF / MISSING) and exits 1 if any differs. Needs the CUDA toolkit's cuobjdump and binutils' c++filt; no GPU."""
import argparse
import os
import re
import subprocess
import sys


def kernels(so):
    cuobjdump = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    text = subprocess.run([cuobjdump, "-sass", so], capture_output=True, text=True, check=True).stdout
    parts = re.split(r"\n\s*Function : (\S+)\n", text)
    names = [parts[i] for i in range(1, len(parts), 2)]
    demangled = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True,
                               check=True).stdout.splitlines()
    out = {}
    for name, body in zip(demangled, parts[2::2]):
        lines = []
        for line in body.splitlines():
            line = re.sub(r"/\*[0-9a-f]{4,}\*/", "", line)
            line = re.sub(r"/\* 0x[0-9a-f]+ \*/", "", line).strip()
            if line and not line.startswith("."):
                lines.append(line)
        out[name] = lines
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--rename", action="append", default=[], metavar="FROM=TO")
    a = ap.parse_args()
    old = kernels(a.old)
    new = {}
    for name, body in kernels(a.new).items():
        for rule in a.rename:
            src, dst = rule.split("=", 1)
            name = name.replace(src, dst)
        new[name] = body
    differ = 0
    for name in sorted(old):
        state = "MISSING" if name not in new else ("SAME" if new[name] == old[name] else "DIFF")
        differ += state != "SAME"
        print(f"{state:8s}{len(old[name]):7d} {name[:160]}")
    print(f"{len(old) - differ} of {len(old)} kernels identical")
    sys.exit(1 if differ else 0)


if __name__ == "__main__":
    main()
