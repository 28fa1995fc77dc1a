"""Static SASS opcode histograms of the main kernels (cuobjdump -sass of the in-tree library; modifiers stripped).
    python tools/sass_hist.py"""
import collections, os, re, subprocess, sys
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
LIB = os.path.join(ROOT, "gaussianformer_b200", "csrc", "libgf_b200.so")
KERNELS = [("render_tile_kernel<18,false>", "_ZN2gf18render_tile_kernelILi18ELb0EEEvNS_12RenderParamsE"),
           ("render_tile_kernel<18,true>", "_ZN2gf18render_tile_kernelILi18ELb1EEEvNS_12RenderParamsE"),
           ("backward_bin_kernel<18,false>", "backward_bin_kernelILi18ELb0"),
           ("backward_bin_kernel<18,true>", "backward_bin_kernelILi18ELb1"),
           ("pack_mask_kernel", "pack_mask_kernel"), ("list_kernel", "list_kernel"),
           ("daf_fast_kernel<fwd>", "daf_fast_kernelILb0"), ("daf_fast_kernel<bwd>", "daf_fast_kernelILb1"),
           ("daf_fused_kernel<fwd>", "daf_fused_kernelILb0"), ("daf_fused_kernel<bwd>", "daf_fused_kernelILb1")]
sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
funcs, cur = {}, None
for line in sass.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = m.group(1); funcs[cur] = []
    elif cur and re.match(r"\s+/\*[0-9a-f]{4,}\*/", line):
        body = re.sub(r"/\*.*?\*/", "", line).strip()
        body = re.sub(r"^@!?U?P\d+\s+", "", body)
        if body:
            funcs[cur].append(body.split()[0].split(".")[0].rstrip(";"))
print("SASS opcode histograms (static instruction counts per kernel, cuobjdump -sass of the in-tree library; modifiers stripped).")
print("What to look for: render = LDGSTS (cp.async ring) + SYNCS (mbarrier) + FFMA2 + MUFU, no tensor / TMA opcodes (SIMT by measurement, DESIGN.md 4.1);")
print("backward_bin = UTMALDG (cp.async.bulk.tensor.3d tile copies) + SYNCS + REDG/ATOMG (raw-sum accumulation) + SHFL (8-lane transposing reduction).\n")
for name, key in KERNELS:
    hit = [f for f in funcs if key in f]
    if not hit:
        continue
    ops = collections.Counter(funcs[hit[0]])
    print(f"== {name}: {sum(ops.values())} instructions")
    items = [f"{k}:{v}" for k, v in ops.most_common()]
    for i in range(0, len(items), 16):
        print("  ".join(items[i:i + 16]))
    print()
