"""Sampling-op experiments on one GPU: the L2 -> SM gather roof (random 512-byte rows of the 88 MB feature table) and the
product kernel against it on the uncorrelated and on the projected (correlated) workload.  Prints one JSON object."""
import ctypes, json, os, sys
import torch
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from gaussianformer_b200 import _lib  # noqa: E402
from gaussianformer_b200.ops import DeformableAggregationFunction as DAF  # noqa: E402
from gaussianformer_b200.synthetic import make_daf_inputs, make_daf_inputs_projected  # noqa: E402

dev = torch.device("cuda")
L_ = _lib.lib()
stream = lambda: ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def timeit(fn, reps=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


out = {}
# ---- L2 -> SM gather roof ----
fms, loc, w = make_daf_inputs(seed=0)
feat, shape, start = DAF.feature_maps_format([f.to(dev) for f in fms])
feat = feat.contiguous()
rows = feat.numel() // 128
n = 4_000_000
sink = torch.zeros(4, device=dev)
for name, nrows in (("table_88MB", rows), ("table_16MB", 32768)):
    idx = torch.randint(0, nrows, (n,), device=dev, dtype=torch.int32)
    ms = timeit(lambda: _lib.check(L_.gf_debug_gather_probe(ctypes.c_void_p(feat.data_ptr()), ctypes.c_void_p(idx.data_ptr()), n, 128,
                                                            ctypes.c_void_p(sink.data_ptr()), stream())))
    out["gather_probe_" + name] = {"ms": ms, "gbs": n * 512 / (ms * 1e-3) / 1e9, "rows": n, "row_bytes": 512}
roof = out["gather_probe_table_88MB"]["gbs"]


def run_case(tag, fms, loc, w):
    feat, shape, start = DAF.feature_maps_format([f.to(dev) for f in fms])
    feat = feat.contiguous()
    loc, w = loc.to(dev), w.to(dev)
    vis = ((loc > 0) & (loc < 1)).all(-1)
    pairs = int(vis.sum()) * shape.shape[0]
    gathered = pairs * 4 * 512
    # the op's own rows as a plain gather: every visible (camera, level) pair's four (clamped) corner rows, in the op's order
    B, P, M, _ = loc.shape
    F = feat.shape[2]
    rows_all = []
    for l in range(shape.shape[0]):
        h, wd = int(shape[l, 0]), int(shape[l, 1])
        x_im, y_im = loc[..., 0] * wd - 0.5, loc[..., 1] * h - 0.5
        x0, y0 = torch.floor(x_im).long(), torch.floor(y_im).long()
        base = (torch.arange(B, device=dev)[:, None, None] * M + torch.arange(M, device=dev)[None, None, :]) * F + int(start[l])
        for dy, dx in ((0, 0), (0, 1), (1, 0), (1, 1)):
            rows_all.append(base + (y0 + dy).clamp(0, h - 1) * wd + (x0 + dx).clamp(0, wd - 1))
    rows_t = torch.stack(rows_all, -1).reshape(B, P, M, shape.shape[0], 4)     # [B,P,M,L,4]
    idx_same = rows_t[vis].reshape(-1).to(torch.int32).contiguous()           # visible (point, camera): all levels, 4 corners
    sink2 = torch.zeros(4, device=dev)
    ms_same = timeit(lambda: _lib.check(L_.gf_debug_gather_probe(ctypes.c_void_p(feat.data_ptr()), ctypes.c_void_p(idx_same.data_ptr()),
                                                                  idx_same.numel(), 128, ctypes.c_void_p(sink2.data_ptr()), stream())))
    ms = timeit(lambda: DAF.apply(feat, shape, start, loc, w))
    out[tag] = {"visible_pairs": pairs, "visible_fraction": float(vis.float().mean()), "gather_bytes": gathered,
                "fwd_ms": ms, "gather_gbs": gathered / (ms * 1e-3) / 1e9, "frac_of_uniform_88MB_probe": gathered / (ms * 1e-3) / 1e9 / roof,
                "same_rows_probe_ms": ms_same, "same_rows_probe_gbs": idx_same.numel() * 512 / (ms_same * 1e-3) / 1e9,
                "frac_of_same_rows_probe": ms_same / ms}


run_case("uncorrelated", fms, loc, w)
run_case("projected", *make_daf_inputs_projected(seed=0))
print(json.dumps(out))
