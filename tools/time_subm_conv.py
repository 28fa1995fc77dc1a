"""Times the submanifold sparse convolution (gaussianformer_b200.ops.subm_conv3d) against a PyTorch gather-GEMM-scatter
on the same GPU over the same voxel-level rulebook (per offset: index_select of the representative rows, mm,
index_add_ into the voxel accumulators, then every row reads its voxel; spconv itself is not timed),
forward and forward + backward, on

    gs25600_uniform     GaussianFormer-1, 25 600 rows, 200 x 200 x 16, k = 5, one layer without bias
    gs25600_clustered   the same rows drawn on a ground plane and box faces (synthetic.make_subm_conv_inputs)
    gs144000            GaussianFormer-1, 144 000 uniform rows
    gf2_gs25600_stack   GaussianFormer-2, 25 600 rows, 100 x 100 x 8, three layers with bias (LayerNorm/ReLU left out)

The rulebook is built once per workload and reused, as SparseConv3D reuses it across its layers; the rulebook build is
timed on its own.  The routes alternate over --regions regions of --iters calls each, CUDA events around every region,
and the median per-call time is reported with the voxel-pair count (the pairs both routes multiply), the achieved
GFLOP/s (2 * 128 * 128 FLOP per voxel pair and layer; 3x that for forward + backward) against the 67 TFLOP/s FP32 data-sheet figure, and the card's name and power
limit read in the same run.

    python tools/time_subm_conv.py --out DIR [--iters 10] [--regions 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gaussianformer_b200.ops import build_rulebook, subm_conv3d  # noqa: E402
from gaussianformer_b200.synthetic import make_subm_conv_inputs  # noqa: E402

PEAK_FP32 = 67e12
WORKLOADS = {
    "gs25600_uniform": (25600, (200, 200, 16), False, 1, False),
    "gs25600_clustered": (25600, (200, 200, 16), True, 1, False),
    "gs144000": (144000, (200, 200, 16), False, 1, False),
    "gf2_gs25600_stack": (25600, (100, 100, 8), False, 3, True),
}


def torch_rulebook(idx, spatial, k):
    """The op's rulebook restated with PyTorch on the device, built once outside the timed regions: rep [M] (the lowest
    row of each occupied voxel, voxels in (b, x, y, z) order), slot [N] and per-offset voxel-level pairs
    (dst slots, src slots), the same pairs the device kernels run over"""
    X, Y, Z = spatial
    i = idx.long()
    key = ((i[:, 0] * X + i[:, 1]) * Y + i[:, 2]) * Z + i[:, 3]
    n = idx.shape[0]
    table = torch.full(((int(i[:, 0].max()) + 1) * X * Y * Z + 1,), n, dtype=torch.long, device=idx.device)
    table.scatter_reduce_(0, key, torch.arange(n, device=idx.device), "amin")
    vkey, slot = torch.unique(key, return_inverse=True)
    rep = table[vkey]
    vox = torch.stack([vkey // (X * Y * Z), vkey // (Y * Z) % X, vkey // Z % Y, vkey % Z], 1)
    p = (k - 1) // 2
    pairs = []
    for o in range(k ** 3):
        q = vox[:, 1:] + torch.tensor([o // (k * k) - p, (o // k) % k - p, o % k - p], device=idx.device)
        inside = ((q >= 0) & (q < torch.tensor(spatial, device=idx.device))).all(1)
        qk = ((vox[:, 0] * X + q[:, 0]) * Y + q[:, 1]) * Z + q[:, 2]
        row = table[torch.where(inside, qk, table.numel() - 1)]
        hit = row < n
        pairs.append((torch.nonzero(hit)[:, 0], slot[row[hit]]))
    return rep, slot, pairs


def torch_layer(x, w, b, rb, k):
    """one layer as a gather-GEMM-scatter over the voxel-level pairs: per offset index_select of the representative
    rows, mm, index_add_ into the voxel accumulators; then every row reads its voxel"""
    rep, slot, pairs = rb
    acc = torch.zeros(len(rep), w.shape[0], device=x.device) if b is None else b.expand(len(rep), -1).clone()
    for o, (dst, src) in enumerate(pairs):
        wo = w[:, o // (k * k), (o // k) % k, o % k, :]
        acc = acc.index_add(0, dst, x.index_select(0, rep[src]).mm(wo.t()))
    return acc.index_select(0, slot)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--regions", type=int, default=5)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    torch.backends.cuda.matmul.allow_tf32 = False
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    results = {"gpu": smi, "workloads": {}}
    for name, (n, spatial, clustered, layers, with_bias) in WORKLOADS.items():
        f, idx, w, b = make_subm_conv_inputs(n, spatial, clustered=clustered, seed=0)
        x, idx = f.cuda(), idx.cuda()
        ws = [(w * (1 + 0.1 * j)).cuda().requires_grad_() for j in range(layers)]
        bs = [b.cuda().requires_grad_() if with_bias else None for _ in range(layers)]
        rb = build_rulebook(idx, spatial, 1, 5, validate=False)
        trb = torch_rulebook(idx, spatial, 5)
        npairs = sum(int(d.numel()) for d, _ in trb[2])
        g = torch.randn_like(x)

        def device(grad):
            h = x.detach().requires_grad_(grad)
            for w_, b_ in zip(ws, bs):
                h = subm_conv3d(h, idx, w_, b_, spatial, 1, rulebook=rb)
            if grad:
                h.backward(g)

        def pytorch(grad):
            h = x.detach().requires_grad_(grad)
            for w_, b_ in zip(ws, bs):
                h = torch_layer(h, w_, b_, trb, 5)
            if grad:
                h.backward(g)

        def rulebook(grad):
            build_rulebook(idx, spatial, 1, 5, validate=False)

        res = {"rows": n, "voxels": len(trb[0]), "voxel_pairs": npairs, "layers": layers}
        for grad in (False, True):
            routes = {"device": device, "pytorch": pytorch} if grad else \
                {"device": device, "pytorch": pytorch, "rulebook": rulebook}
            for fn in routes.values():
                fn(grad)
            torch.cuda.synchronize()
            times = {r: [] for r in routes}
            for _ in range(args.regions):
                for r, fn in routes.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.iters):
                        fn(grad)
                    e1.record()
                    torch.cuda.synchronize()
                    times[r].append(e0.elapsed_time(e1) / args.iters)
            flop = 2 * 128 * 128 * npairs * layers * (3 if grad else 1)
            for r, t in times.items():
                med = sorted(t)[len(t) // 2]
                key = f"{'fwd_bwd' if grad else 'fwd'}_{r}"
                res[key + "_ms"] = round(med, 4)
                if r != "rulebook":
                    res[key + "_gflops"] = round(flop / med / 1e6, 1)
                    res[key + "_share_of_fp32_peak"] = round(flop / med / 1e-3 / PEAK_FP32, 4)
        results["workloads"][name] = res
        print(name, json.dumps(res), flush=True)
    with open(os.path.join(args.out, "time_subm_conv.json"), "w") as fh:
        json.dump(results, fh, indent=1)
    print(json.dumps(results))


if __name__ == "__main__":
    main()
