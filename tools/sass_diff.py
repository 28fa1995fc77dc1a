"""Checks that every kernel of a baseline build compiles to the same SASS in this tree's build.

    python tools/sass_diff.py --base REV        # exports git revision REV to a temporary directory and builds it there
    python tools/sass_diff.py --base-dir DIR    # a tree that is already built

Both trees are built with gaussianformer_b200/csrc/build.py.  For every object file of the baseline, every function
`cuobjdump -sass` lists (kernels and non-inlined device functions) must have the same instructions, offsets and
encodings in this tree's object of the same name.  Functions only this tree has are listed as new.  Exits 1 on any
difference.  Needs nvcc and cuobjdump, no GPU.
"""
import argparse
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join("gaussianformer_b200", "csrc")
CUOBJDUMP = os.path.join(os.path.dirname(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")), "cuobjdump")


def build(tree):
    subprocess.run([sys.executable, "-m", "gaussianformer_b200.csrc.build", "--force"], cwd=tree, check=True)


def functions(obj):
    """{function name: SASS text} of one object file"""
    out = subprocess.run([CUOBJDUMP, "-sass", obj], check=True, capture_output=True, text=True).stdout
    # anonymous namespaces are named after a hash of the source's path: two checkouts differ there only
    out = re.sub(r"_GLOBAL__N__[0-9a-f]+_", "_GLOBAL__N__", out)
    funcs, name, body = {}, None, []
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                funcs[name] = "\n".join(body)
            name, body = m.group(1), []
        elif name:
            body.append(line.rstrip())
    if name:
        funcs[name] = "\n".join(body)
    return funcs


def compare(base_tree, new_tree):
    changed, same, new = [], 0, []
    base_dir, new_dir = os.path.join(base_tree, CSRC), os.path.join(new_tree, CSRC)
    for obj in sorted(f for f in os.listdir(base_dir) if f.endswith(".o")):
        old = functions(os.path.join(base_dir, obj))
        cur = functions(os.path.join(new_dir, obj))
        for name, sass in old.items():
            if cur.get(name) == sass:
                same += 1
            else:
                changed.append(f"{obj}: {name}" + ("" if name in cur else " (missing)"))
        new += [f"{obj}: {n}" for n in cur if n not in old]
    for obj in sorted(f for f in os.listdir(new_dir) if f.endswith(".o")):
        if not os.path.exists(os.path.join(base_dir, obj)):
            new += [f"{obj}: {n}" for n in functions(os.path.join(new_dir, obj))]
    return changed, same, new


def main():
    ap = argparse.ArgumentParser()
    g = ap.add_mutually_exclusive_group(required=True)
    g.add_argument("--base", help="git revision to compare against")
    g.add_argument("--base-dir", help="an already built tree to compare against")
    ap.add_argument("--no-build", action="store_true", help="use this tree's objects as they are")
    args = ap.parse_args()
    if not args.no_build:
        build(ROOT)
    with tempfile.TemporaryDirectory() as tmp:
        base = args.base_dir
        if base is None:
            base = tmp
            archive = subprocess.run(["git", "archive", args.base], cwd=ROOT, check=True, capture_output=True).stdout
            subprocess.run(["tar", "-x", "-C", tmp], input=archive, check=True)
            build(tmp)
        changed, same, new = compare(base, ROOT)
    print(f"{same} functions with identical SASS")
    for n in new:
        print("new:", n)
    for c in changed:
        print("CHANGED:", c)
    return 1 if changed else 0


if __name__ == "__main__":
    sys.exit(main())
