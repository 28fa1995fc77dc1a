"""Times the occupancy loss of one supervised layer: the PyTorch restatement of the reference's OccupancyLoss as written
(tests/occ_loss_oracle.py: boolean gathers, a present test per class, torch.sort per class) against the device op
(gaussianformer_b200.loss.occupancy_loss, validate=False), forward and forward + backward, on

    gf1      GaussianFormer-1: logits, 200 x 200 x 16 voxels x 18 classes, B = 1
    gf1_b4   the same at B = 4 (one pooled call, as the reference's batch)
    gf2      GaussianFormer-2: probabilities at the same grid, B = 1

with 10 x CE + 1 x Lovasz, lovasz_ignore = 17, occ_mask = label != 0 and make_occ_loss_inputs' labels.  One process;
the routes alternate over --regions regions of --iters calls each, CUDA events around every region, and the median
per-call time is reported with |V|, the card's name and power limit, and the host synchronisations one call of each
route makes (torch.cuda.set_sync_debug_mode("warn")).

    python tools/time_occ_loss.py --out DIR [--iters 20] [--regions 5] [--n 640000]
"""
import argparse
import json
import os
import subprocess
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import occ_loss_oracle as olo  # noqa: E402
from gaussianformer_b200.loss import occupancy_loss  # noqa: E402
from gaussianformer_b200.synthetic import make_occ_loss_inputs  # noqa: E402

MANUAL = [1.01552756, 1.06897009, 1.30013094, 1.07253735, 0.94637502, 1.10087012, 1.26960524, 1.06258364, 1.189019,
          1.06217292, 1.00595144, 0.85706115, 1.03923299, 0.90867526, 0.8936431, 0.85486129, 0.8527829, 0.5]
KW = dict(ce_weight=10.0, lovasz_weight=1.0, lovasz_ignore=17)


def routes(x, labels, mask, w, use_softmax):
    def torch_route(grad):
        xx = x.detach().requires_grad_(grad)
        loss = olo.restatement(xx, labels, mask, w, use_softmax=use_softmax, **KW)[0]
        if grad:
            loss.backward()

    def device_route(grad):
        xx = x.detach().requires_grad_(grad)
        loss = occupancy_loss(xx, labels, mask, class_weights=w, use_softmax=use_softmax, validate=False, **KW)
        if grad:
            loss.backward()

    return {"pytorch": torch_route, "device": device_route}


def syncs(fn, grad):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn(grad)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    return sum("synchroniz" in str(r.message) for r in rec)


def time_region(fn, grad, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn(grad)
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--n", type=int, default=640000, help="voxels per sample")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_occ_loss.py measures on a CUDA device; none is available")
    os.makedirs(args.out, exist_ok=True)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    res = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi[0] if smi else None, "iters": args.iters,
           "regions": args.regions, "workloads": {}}
    w18 = torch.tensor(MANUAL)
    w = (18 * w18 / w18.abs().sum()).cuda()
    for name, B, use_softmax in (("gf1", 1, True), ("gf1_b4", 4, True), ("gf2", 1, False)):
        pred, labels, mask = make_occ_loss_inputs(B, args.n, 18, use_softmax, seed=0, ignore_share=0.0)
        x, labels, mask = pred.cuda().transpose(1, 2), labels.cuda(), mask.cuda()
        nv = int((mask & (labels != 17)).sum())
        fns = routes(x, labels, mask, w, use_softmax)
        r = {"B": B, "N": args.n, "num_v": nv}
        for grad in (False, True):
            tag = "fwd_bwd" if grad else "fwd"
            for rn, fn in fns.items():
                for _ in range(args.warmup):
                    fn(grad)
                r[f"{rn}_{tag}_syncs"] = syncs(fn, grad)
            times = {rn: [] for rn in fns}
            for _ in range(args.regions):
                for rn, fn in fns.items():
                    times[rn].append(time_region(fn, grad, args.iters))
            for rn in fns:
                r[f"{rn}_{tag}_ms"] = sorted(times[rn])[len(times[rn]) // 2]
                r[f"{rn}_{tag}_all_ms"] = times[rn]
        res["workloads"][name] = r
        print(name, {k: (round(v, 4) if isinstance(v, float) else v) for k, v in r.items() if "all" not in k},
              flush=True)
        del x, labels, mask, fns
        torch.cuda.empty_cache()
    print("gpu", res["gpu"], "|", res["nvidia_smi"])
    path = os.path.join(args.out, "time_occ_loss.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", path)


if __name__ == "__main__":
    main()
