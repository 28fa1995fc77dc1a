"""Builds an alternative libgf_b200 with extra nvcc flags for A/B measurements:
    python tools/build_variant.py timing -DGF_RENDER_TIMING
writes gaussianformer_b200/csrc/variants/libgf_b200_timing.so; select it with GF_B200_LIB=<path>."""
import os, subprocess, sys
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from gaussianformer_b200.csrc import build as B
name, extra = sys.argv[1], sys.argv[2:]
out_dir = os.path.join(B.HERE, "variants", name)
os.makedirs(out_dir, exist_ok=True)
objs, procs = [], []
for src in B.SOURCES:
    obj = os.path.join(out_dir, src.replace(".cu", ".o"))
    cmd = [B.NVCC] + B.FLAGS + extra + (["-ccbin", B.HOST_CXX] if B.HOST_CXX else []) + ["-c", os.path.join(B.HERE, src), "-o", obj]
    procs.append(subprocess.Popen(cmd)); objs.append(obj)
assert all(p.wait() == 0 for p in procs)
lib = os.path.join(B.HERE, "variants", f"libgf_b200_{name}.so")
subprocess.run([B.NVCC, "-shared", "-o", lib] + (["-ccbin", B.HOST_CXX] if B.HOST_CXX else []) + objs + ["-lcudart"], check=True)
for o in objs: os.remove(o)
print(lib)
