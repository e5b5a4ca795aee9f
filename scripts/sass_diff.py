#!/usr/bin/env python
"""Kernel-by-kernel SASS comparison of two builds of the library, without a GPU:

    cuobjdump -sass <old libeat_b200.so> > old.sass
    cuobjdump -sass <new libeat_b200.so> > new.sass
    python scripts/sass_diff.py old.sass new.sass [--drop-last-arg dw_slide_kernel dw_tile_kernel]

Every kernel of the old build must have a kernel of the same (demangled) name in the new one with the same instructions.
--drop-last-arg names kernel templates that gained a trailing template parameter with a default: the new instance whose
last argument equals the default ("…, 2>" for DyReLU-B's pieces) stands for the old name.  Prints the counts of identical,
differing, missing and added kernels; exits 1 if any old kernel differs or is missing."""
import argparse
import collections
import re
import subprocess
import sys


def parse(path):
    per, cur = collections.OrderedDict(), None
    for line in open(path):
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            per[cur] = []
        elif cur is not None and re.match(r"\s*/\*[0-9a-f]{4}\*/", line):
            per[cur].append(re.sub(r"^\s*/\*[0-9a-f]+\*/\s*", "", line).strip())
    names = subprocess.run(["c++filt"], input="\n".join(per), capture_output=True, text=True).stdout.splitlines()
    return {d: per[k] for k, d in zip(per, names)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--drop-last-arg", nargs="*", default=["dw_slide_kernel", "dw_tile_kernel"])
    ap.add_argument("--default", default="2")
    a = ap.parse_args()
    old, new = parse(a.old), parse(a.new)
    pats = [re.compile(rf"({re.escape(k)}<[^>]*), {re.escape(a.default)}>") for k in a.drop_last_arg]

    def as_old(name):
        for p in pats:
            name = p.sub(r"\1>", name)
        return name
    mapped = {}
    for d, v in new.items():
        mapped.setdefault(as_old(d), []).append(v)
    same, differ, missing = 0, [], []
    for d, v in old.items():
        cands = mapped.get(d)
        if cands is None:
            missing.append(d)
        elif any(c == v for c in cands):
            same += 1
        else:
            differ.append(d)
    added = len(new) - same - len(differ)           # new kernels that stand for no old one
    for d in differ:
        print("differs:", d[:200])
    for d in missing:
        print("missing:", d[:200])
    print(f"old kernels {len(old)}, new kernels {len(new)}: identical SASS {same}, differing {len(differ)}, "
          f"missing {len(missing)}, added {added}")
    sys.exit(1 if differ or missing else 0)


if __name__ == "__main__":
    main()
