"""Instruction-by-instruction comparison of the kernels of two builds of libdspgn.so (cuobjdump -sass; addresses and
the encoding comments dropped).  Use it to show that a change leaves a kernel's machine code as it was.

  python tools/sass_diff.py OLD.so NEW.so [--rename OLD_MANGLED=NEW_MANGLED ...]

--rename pairs a kernel whose mangled name changed (e.g. a kernel that became a template instantiation).  Prints each
kernel that differs and a summary line; exits 1 if any kernel of OLD differs or is missing in NEW.
"""
import argparse
import re
import subprocess
import sys


def kernels(so):
    out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
    fs, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            name = m.group(1)
            fs[name] = []
        elif name and "/*" in line:
            fs[name].append(re.sub(r"/\*[0-9a-f]{4,}\*/", "", line).strip())
    return fs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--rename", nargs="*", default=[], metavar="OLD=NEW")
    args = ap.parse_args()
    ren = dict(r.split("=", 1) for r in args.rename)
    a, b = kernels(args.old), kernels(args.new)
    same, bad = 0, 0
    for n, ins in a.items():
        m = ren.get(n, n)
        if m not in b:
            print("missing in new:", n)
            bad += 1
        elif ins != b[m]:
            print(f"differs: {n} ({len(ins)} -> {len(b[m])} instructions)")
            bad += 1
        else:
            same += 1
    new_only = sorted(set(b) - {ren.get(n, n) for n in a})
    print(f"identical: {same}, different or missing: {bad}, only in new: {new_only}")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
