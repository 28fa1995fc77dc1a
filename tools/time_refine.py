"""Times the Gaussian refinement on one GPU, device against PyTorch, on the same inputs:

  arithmetic  gaussian_refine against the reference's lines after ``layers`` (refine_module.py:72-123,
              refine_module_v2.py:64-108, as restated in tests/refine_oracle.py), on the same MLP output
  module      the whole module with its MLP: SparseGaussian3DRefinementModule(V2) against the same ``layers`` followed
              by the PyTorch restatement

each forward (no grad) and forward + backward (torch.autograd.grad of every output to the MLP output and the anchor,
for the module also to every MLP parameter).  Workloads: the three shipped setups of synthetic.REFINE_CONFIGS at
B = 1, embed_dims 128, fp32.  Each is timed two ways:

  eager   the calls as a training step makes them: Python, autograd and launches included
  graph   the same calls captured once in a CUDA graph and replayed: the device time alone, without the host

Within a workload the two routes alternate in each of --regions regions with CUDA events around a block of calls.  A
block lasts about --region-seconds (at least 20 calls), since the eager calls are host-bound and a short window
measures the scheduler as much as the call.  The median region is reported with the spread, max - min over the
regions.  Records the card's name, power limit and max SM clock.

    python tools/time_refine.py --out DIR        # writes DIR/time_refine.json
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import refine_oracle as ro  # noqa: E402
from gaussianformer_b200.ops import (SparseGaussian3DRefinementModule, SparseGaussian3DRefinementModuleV2,  # noqa: E402
                                     gaussian_refine)
from gaussianformer_b200.synthetic import REFINE_CONFIGS, make_refine_inputs  # noqa: E402
from time_daf_bwd import gpu_info, time_group  # noqa: E402


def workload(config, dev="cuda"):
    d = make_refine_inputs(config, seed=0)
    cfg = dict(d["config"], variant=d["variant"])
    cls = SparseGaussian3DRefinementModuleV2 if d["variant"] == "v2" else SparseGaussian3DRefinementModule
    torch.manual_seed(0)
    m = cls(**d["config"]).to(dev)
    if d["variant"] == "v2":
        cfg["unit_xyz_buffer"] = m.unit_xyz          # the reference multiplies by its device buffer
    out = d["out"].to(dev).requires_grad_()
    anchor = d["anchor"].to(dev).requires_grad_()
    inst, embed = d["instance_feature"].to(dev), d["anchor_embed"].to(dev)
    v1 = d["variant"] == "v1"
    args = dict(variant=d["variant"], pc_range=cfg["pc_range"], scale_range=cfg["scale_range"],
                unit_xyz=cfg["unit_xyz"], refine_prefix=len(cfg["refine_manual"]) if v1 else 0,
                restrict_xyz=cfg.get("restrict_xyz", False), include_opa=cfg["include_opa"],
                semantic_dim=cfg["semantic_dim"], semantics_activation=cfg["semantics_activation"])

    def flat(new_anchor, g):
        """the outputs in one order for both routes, the empty ones left out"""
        g = g._asdict() if hasattr(g, "_asdict") else g
        return [new_anchor] + [g[k] for k in ro.OUTPUTS[1:] if g.get(k) is not None and g[k].numel()]

    def arithmetic(route):
        if route == "device":
            return flat(*gaussian_refine(out, anchor, **args))
        return flat(*ro.reference_refine(out, anchor, cfg))

    def module(route):
        if route == "device":
            return flat(*m(inst, anchor, embed))
        return flat(*ro.reference_refine(m.layers(inst + embed), anchor, cfg))

    with torch.no_grad():
        shapes = [t.shape for t in arithmetic("device")]
    gen = torch.Generator(device=dev).manual_seed(1)
    ups = [torch.randn(s, device=dev, generator=gen) for s in shapes]
    leaves = {"arithmetic": [out, anchor], "module": [anchor] + list(m.parameters())}
    return {"arithmetic": arithmetic, "module": module}, leaves, ups


def graphed(fn):
    """fn captured in a CUDA graph (after a warm-up on a side stream, as capture requires); returns its replay"""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    torch.cuda.synchronize()
    return g.replay


def calls_per_region(variants, seconds):
    """the number of calls that makes the slowest variant's block last about `seconds` (at least 20)"""
    worst = 0.0
    for fn in variants.values():
        fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        worst = max(worst, (time.perf_counter() - t0) / 5)
    return max(20, int(seconds / worst))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--region-seconds", type=float, default=0.25)
    ap.add_argument("--regions", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    assert args.regions >= 3
    os.makedirs(args.out, exist_ok=True)
    res = {"gpu": gpu_info(), "region_seconds": args.region_seconds, "regions": args.regions}
    routes = ("device", "pytorch")
    for config in REFINE_CONFIGS:
        stages, leaves, ups = workload(config)
        r = {}
        for stage, fn in stages.items():
            def forward(rt, fn=fn):
                with torch.no_grad():
                    return fn(rt)

            def fwd_bwd(rt, fn=fn, stage=stage):
                return torch.autograd.grad(fn(rt), leaves[stage], ups)

            for what, call in (("forward", forward), ("fwd_bwd", fwd_bwd)):
                eager = {rt: (lambda rt=rt, call=call: call(rt)) for rt in routes}
                for mode, variants in (("eager", eager), ("graph", {rt: graphed(f) for rt, f in eager.items()})):
                    n = calls_per_region(variants, args.region_seconds)
                    t = time_group(variants, n, args.regions, args.warmup)
                    for v in t.values():
                        v["calls_per_region"] = n
                    r[f"{stage}_{what}_{mode}"] = t
        res[config] = r
        for k, v in r.items():
            print(config, k, {rt: (round(v[rt]["median_ms"], 4),
                                   round(max(v[rt]["regions_ms"]) - min(v[rt]["regions_ms"]), 4)) for rt in v},
                  flush=True)
        del stages, leaves, ups
        torch.cuda.empty_cache()
    path = os.path.join(args.out, "time_refine.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print("gpu", res["gpu"])
    print("wrote", path)


if __name__ == "__main__":
    main()
