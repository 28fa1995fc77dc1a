"""C-ABI backward timing: python tools/time_bwd.py [config] [batch]"""
import os, sys
import torch
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from gaussianformer_b200 import _lib  # noqa: E402
from gaussianformer_b200.splat import _make_desc, splat_backward_raw, splat_forward_raw  # noqa: E402
from gaussianformer_b200.synthetic import make_splat_inputs  # noqa: E402

cfg = sys.argv[1] if len(sys.argv) > 1 else "gs25600_solid"
B = int(sys.argv[2]) if len(sys.argv) > 2 else 1
parts = [make_splat_inputs(cfg, seed=s, perturb=False) for s in range(B)]
kw, variant = parts[0][0], parts[0][2]
t = {k: torch.cat([p[1][k] for p in parts], 0).cuda().contiguous() for k in parts[0][1]}
G, N = t["means"].shape[1], t["pts"].shape[1]
prob = variant == "prob"
desc = _make_desc(G, N, 18, kw["H"], kw["W"], kw["D"], _lib.GF_SPLAT_PROB if prob else _lib.GF_SPLAT_BASE, 1, 9, kw["pc_min"],
                  kw["grid_size"], float(kw["scale_multiplier"]), 1 if prob else 0, B, 0)
cov = t["cov"].reshape(B, G, 9)
(lg, bl, de, pr), _ = splat_forward_raw(desc, t["pts"], t["means"], t["opa"], t["sem"], cov, scales=t["scales"])
gen = torch.Generator(device="cuda").manual_seed(0)
g = (torch.randn(lg.shape, device="cuda", generator=gen),
     torch.randn(B, N, device="cuda", generator=gen) if prob else None, torch.randn(B, N, device="cuda", generator=gen) if prob else None)
saved = (lg, bl, pr) if prob else (None, None, None)
run = lambda: splat_backward_raw(desc, t["pts"], t["means"], t["opa"], t["sem"], cov, g, saved, scales=t["scales"])
for _ in range(3):
    out = run()
torch.cuda.synchronize()
a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
a.record()
for _ in range(10):
    run()
b.record()
torch.cuda.synchronize()
print(f"{cfg} B={B}: {a.elapsed_time(b) / 10:.4f} ms per call, {a.elapsed_time(b) / 10 / B:.4f} ms per sample; |g_means| {float(out[0].abs().sum()):.6e}")
