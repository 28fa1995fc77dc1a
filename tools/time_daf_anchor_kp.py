"""Times the anchor key-point generator on one GPU, device against PyTorch, on the same inputs:

  generator  SparseGaussian3DKeyPointsGenerator (learnable_fc + gf_daf_anchor_key_points) against the reference's
             generator in PyTorch (learnable_fc + the lines of deformable_module.py:51-90, as restated in
             tests/daf_anchor_oracle.py), forward (no grad) and forward + backward (torch.autograd.grad to the anchor
             and the learnable_fc weight)
  chain      anchor -> aggregated feature: the module + deformable_aggregation_from_key_points against the PyTorch
             generator + the reference's project_points (deformable_module.py:287-305) + permute feeding
             deformable_aggregation_fused; forward and forward + backward (to the anchor, the learnable_fc weight,
             the feature table and the weight logits)

Workloads: GaussianFormer-1 (25 600 anchors, 7 + 2 key points) and GaussianFormer-2 (6 400, 7 + 6), B = 1, 6 cameras,
4 levels of 1600x864 / 8..64, C = 128, 4 groups, fp32.  Within a workload the two routes alternate in each of
--regions regions with CUDA events around --iters calls; the median region is reported with the spread.  Also times
the two kernels alone and records the card's name, power limit and max SM clock.

    python tools/time_daf_anchor_kp.py --out DIR        # writes DIR/time_daf_anchor_kp.json
"""
import argparse
import json
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import daf_anchor_oracle as ao  # noqa: E402
from gaussianformer_b200.ops import DeformableAggregationFunction as DAF  # noqa: E402
from gaussianformer_b200.ops import SparseGaussian3DKeyPointsGenerator, anchor_key_points  # noqa: E402
from gaussianformer_b200.ops import deformable_aggregation_from_key_points, deformable_aggregation_fused  # noqa: E402
from gaussianformer_b200.synthetic import ANCHOR_FIX_SCALE, make_anchor_kp_inputs, make_daf_kp_inputs  # noqa: E402
from time_daf_bwd import gpu_info, time_group  # noqa: E402
from time_daf_kp import project_points  # noqa: E402


def workload(config, dev="cuda"):
    d = make_anchor_kp_inputs(config, seed=0)
    A, Kl = d["anchor"].shape[1], d["num_learnable"]
    K = len(ANCHOR_FIX_SCALE) + Kl
    m = SparseGaussian3DKeyPointsGenerator(embed_dims=128, num_learnable_pts=Kl,
                                           learnable_fixed_scale=d["learnable_fixed_scale"], fix_scale=ANCHOR_FIX_SCALE,
                                           pc_range=d["pc_range"], scale_range=d["scale_range"]).to(dev)
    m.load_state_dict({"learnable_fc.weight": d["weight"], "learnable_fc.bias": d["bias"]})
    fms, _, _, _, wlog, _ = make_daf_kp_inputs(num_anchor=A, num_pts=K, seed=1)
    table, shape, start = DAF.feature_maps_format([f.to(dev) for f in fms])
    anchor = d["anchor"].to(dev).requires_grad_()
    table = table.detach().requires_grad_()
    wlog = wlog.to(dev).requires_grad_()
    inst = d["instance_feature"].to(dev)
    P, wh = d["projection_mat"].to(dev), d["image_wh"].to(dev)
    M = P.shape[1]

    def gen(route):
        if route == "device":
            return m(anchor, inst)
        logits = m.learnable_fc(inst).reshape(1, A, Kl, 3)
        return ao.reference_generator(anchor, logits, ANCHOR_FIX_SCALE, d["pc_range"], d["scale_range"],
                                      d["learnable_fixed_scale"])

    def chain(route):
        kp = gen(route)
        if route == "device":
            return deformable_aggregation_from_key_points(table, shape, start, kp, P, wh, wlog)
        pts, mask = project_points(kp, P, wh)
        loc = pts.permute(0, 2, 3, 1, 4).reshape(1, A * K, M, 2)
        return deformable_aggregation_fused(table, shape, start, loc, wlog, mask.permute(0, 2, 3, 1))

    leaves = {"generator": [anchor, m.learnable_fc.weight], "chain": [anchor, m.learnable_fc.weight, table, wlog]}
    gen_g = torch.randn(1, A, K, 3, device=dev, generator=torch.Generator(device=dev).manual_seed(2))
    chain_g = torch.randn(1, A, 128, device=dev, generator=torch.Generator(device=dev).manual_seed(3))
    kernels = (anchor.detach(), d["logits"].to(dev), m.fix_scale, d["pc_range"], d["scale_range"],
               d["learnable_fixed_scale"])
    return {"generator": (gen, gen_g), "chain": (chain, chain_g)}, leaves, kernels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    assert args.regions >= 3
    os.makedirs(args.out, exist_ok=True)
    res = {"gpu": gpu_info(), "iters": args.iters, "regions": args.regions}
    routes = ("device", "pytorch")
    for config in ("gs25600_solid", "prob_gs6400"):
        stages, leaves, kern = workload(config)
        r = {}
        for stage, (fn, g) in stages.items():
            with torch.no_grad():
                r[stage + "_forward"] = time_group({rt: (lambda rt=rt: fn(rt)) for rt in routes},
                                                   args.iters, args.regions, args.warmup)
            r[stage + "_fwd_bwd"] = time_group(
                {rt: (lambda rt=rt: torch.autograd.grad(fn(rt), leaves[stage], g)) for rt in routes},
                args.iters, args.regions, args.warmup)
        a, lg, fix, pcr, scr, lfs = kern
        a, lg = a.requires_grad_(), lg.requires_grad_()
        gk = torch.randn(a.shape[0], a.shape[1], fix.shape[0] + lg.shape[2], 3, device="cuda")
        r["kernels_alone"] = time_group({
            "gf_daf_anchor_key_points": lambda: anchor_key_points(a.detach(), lg.detach(), fix, pcr, scr, lfs),
            "forward_and_backward": lambda: torch.autograd.grad(anchor_key_points(a, lg, fix, pcr, scr, lfs),
                                                                [a, lg], gk)},
            args.iters * 5, args.regions, args.warmup)
        res[config] = r
        print(config, {k: {rt: round(v[rt]["median_ms"], 4) for rt in v} for k, v in r.items()},
              "spread", {k: {rt: round(max(v[rt]["regions_ms"]) - min(v[rt]["regions_ms"]), 4) for rt in v}
                         for k, v in r.items()}, flush=True)
        del stages, leaves, kern
        torch.cuda.empty_cache()
    path = os.path.join(args.out, "time_daf_anchor_kp.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print("gpu", res["gpu"])
    print("wrote", path)


if __name__ == "__main__":
    main()
