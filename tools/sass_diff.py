"""Compare the SASS of kernels between two builds of one source file, by kernel name with template arguments dropped or
mapped, e.g. that the AA = false instantiations of the projection kernels compile to the instructions of the build before the
anti-aliased mode existed (DESIGN.md section 4):

    python tools/sass_diff.py parent/project_bwd.o new/project_bwd.o \
        --map 'project_bwd_views_kernelILi12ELi5EE=project_bwd_views_kernelILi12ELi5ELb0EE' ...

Each object's SASS (cuobjdump -sass) is split per function; instruction text is compared with addresses and comments
removed.  Exit status 1 if any mapped pair differs."""
import argparse
import re
import subprocess
import sys

CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"


def functions(obj):
    out = subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
            continue
        if name is None:
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s*(.*?)\s*;", line)
        if m:
            funcs[name].append(re.sub(r"\s+", " ", m.group(1)))
    return funcs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--map", action="append", default=[], help="OLD_SUBSTRING=NEW_SUBSTRING of the mangled names")
    a = ap.parse_args()
    fo, fn = functions(a.old), functions(a.new)
    bad = 0
    for spec in a.map:
        o, n = spec.split("=", 1)
        ko = [k for k in fo if o in k]
        kn = [k for k in fn if n in k]
        if len(ko) != 1 or len(kn) != 1:
            print(f"{spec}: expected one function on each side, got {ko} / {kn}")
            bad += 1
            continue
        same = fo[ko[0]] == fn[kn[0]]
        print(f"{'same' if same else 'DIFFERENT'}  {len(fo[ko[0]])} / {len(fn[kn[0]])} instructions  {ko[0]} -> {kn[0]}")
        bad += not same
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
