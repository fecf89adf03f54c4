#!/usr/bin/env python3
"""Compare the SASS of every kernel in two builds of one object file, e.g. before and after a change that must leave existing kernels
untouched:

    python scripts/compare_sass.py old/mlp_fused.o new/mlp_fused.o

Instruction text is compared with addresses and column padding removed. A kernel template that gained a trailing `bool` parameter
(`mlp_forward_kernel<W, GENERIC_ACT, BWD, PRE, WIDE>`, `fused_ws_kernel<D, F, TRAIN, GENERIC_ACT, PDF>`, `mlp_wgrad_kernel<W, WIDE>`) is matched to its old name
when the new parameter is false. Exit code 1 if any old
kernel is missing or differs.

Build both objects from the same source path (e.g. stash the change, build, unstash, build): kernels in an anonymous namespace
carry a hash of the path in their mangled names, so objects built from two checkouts report every such kernel MISSING."""
import re
import subprocess
import sys


def functions(obj):
    out = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    fs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            fs[cur] = []
        elif cur is not None:
            fs[cur].append(" ".join(re.sub(r"/\*[0-9a-f]{4,}\*/", "", line).split()))
    return fs


def old_name(name):
    return re.sub(r"(I(?:L[jb]\d+E)+)Lb0E(E)", r"\1\2", name)


def main():
    old, new = functions(sys.argv[1]), functions(sys.argv[2])
    # a kernel whose name is unchanged is matched by that name first (old_name would strip its own trailing false parameter)
    by_old_name = {**{old_name(k): v for k, v in new.items()}, **new}
    bad = 0
    for name, sass in old.items():
        if by_old_name.get(name) != sass:
            print("DIFFERENT" if name in by_old_name else "MISSING", name)
            bad += 1
    added = [k for k in new if k not in old and old_name(k) not in old]
    print(f"{len(old) - bad} of {len(old)} kernels identical; {len(added)} new: {' '.join(added)}")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
