"""The Gaussian refinement on the GPU: the kernels against the fp64 oracle (refine_oracle) for the three shipped setups
at full size and at B = 2, the option values and crafted edges; gradient parity with the fp32 PyTorch restatement;
reproducibility, gradient subsets, half inputs, strides, CUDA-graph replay, no host synchronisation, the errors; and
four refinement layers chained through the key-point generator and the splat against the same chain in PyTorch."""
import copy

import numpy as np
import pytest
import torch
from torch import nn

import helpers as h
import refine_oracle as ro
from gaussianformer_b200._lib import GfError
from gaussianformer_b200.ops import (GaussianPrediction, SparseGaussian3DKeyPointsGenerator,
                                     SparseGaussian3DRefinementModule, gaussian_refine)
from gaussianformer_b200.splat import LocalAggregator
from gaussianformer_b200.synthetic import ANCHOR_FIX_SCALE, REFINE_CONFIGS, make_refine_inputs
from test_daf_anchor_kp_gpu import assert_within_oracle
from test_refine_cpu import CASES, _grads

pytestmark = pytest.mark.gpu

CONFIGS = list(REFINE_CONFIGS)


def _args(cfg):
    v1 = cfg["variant"] == "v1"
    return dict(variant=cfg["variant"], pc_range=cfg["pc_range"], scale_range=cfg["scale_range"],
                unit_xyz=cfg["unit_xyz"], refine_prefix=len(cfg.get("refine_manual") or []) if v1 else 0,
                restrict_xyz=cfg.get("restrict_xyz", False) if v1 else False, include_opa=cfg["include_opa"],
                semantic_dim=cfg["semantic_dim"], semantics_activation=cfg["semantics_activation"])


def _outputs(new_anchor, gp):
    res = dict(new_anchor=new_anchor, **gp._asdict())
    return {k: v for k, v in res.items() if v is not None}


def _run(out, anchor, cfg, grads=None):
    """device outputs {name: CPU tensor} and, with grads ({name: CPU tensor or None}), (grad_out, grad_anchor)"""
    o = out.cuda().requires_grad_()
    a = anchor.cuda().requires_grad_()
    res = _outputs(*gaussian_refine(o, a, **_args(cfg)))
    if grads is None:
        return {k: v.detach().cpu() for k, v in res.items()}, None
    used = [k for k in res if grads.get(k) is not None]
    torch.autograd.backward([res[k] for k in used], [grads[k].cuda() for k in used])
    return {k: v.detach().cpu() for k, v in res.items()}, (o.grad.cpu(), a.grad.cpu())


def check_against_oracle(out, anchor, cfg, grads, what):
    got, (go, ga) = _run(out, anchor, cfg, grads)
    want, wabs = ro.refine(out.numpy(), anchor.numpy(), cfg)
    assert set(got) == set(want)
    for k in want:
        assert_within_oracle(got[k].numpy(), want[k], wabs[k], f"{what} {k}", True)
    g = {k: (None if v is None else v.numpy()) for k, v in grads.items()}
    wo, woa, wa, waa = ro.refine_backward(out.numpy(), anchor.numpy(), cfg, g)
    assert_within_oracle(go.numpy(), wo, woa, f"{what} grad out", False)
    assert_within_oracle(ga.numpy(), wa, waa, f"{what} grad anchor", False)
    r = 3 if cfg["variant"] == "v2" else len(cfg.get("refine_manual") or [])
    assert (ga[..., r:] == 0).all() and not torch.signbit(ga[..., r:]).any()
    return got, go, ga


def _inputs(config, B, A=None, seed=0, margin=False):
    d = make_refine_inputs(config, batch=B, num_anchor=A, seed=seed, margin=margin)
    return d["out"], d["anchor"], dict(d["config"], variant=d["variant"])


SIZES = [(c, 1, None) for c in CONFIGS] + [(c, 2, 3000) for c in CONFIGS]


@pytest.mark.parametrize("config,B,A", SIZES, ids=[f"{c}-B{b}" for c, b, _ in SIZES])
def test_shipped_setups_against_the_oracle(config, B, A):
    out, anchor, cfg = _inputs(config, B, A, seed=1)
    check_against_oracle(out, anchor, cfg, _grads(out, anchor, cfg, seed=2), f"{config} B={B}")


@pytest.mark.parametrize("case", [c for c in CASES if c not in CONFIGS])
def test_options_and_crafted_edges_against_the_oracle(case):
    out, anchor, cfg = CASES[case]()
    _, go, _ = check_against_oracle(out, anchor, cfg, _grads(out, anchor, cfg), case)
    if case == "crafted":                                   # the clamps' gates on the device
        through = go[0] - _grads(out, anchor, cfg)["new_anchor"][0]
        assert (through[0, [0, 1, 3, 4, 10]] != 0).all() and (through[1, [0, 2, 3, 10]] == 0).all()
        assert torch.isfinite(go).all()


@pytest.mark.parametrize("config", CONFIGS)
def test_gradient_parity_with_the_fp32_restatement(config):
    out, anchor, cfg = _inputs(config, 1, seed=3, margin=True)
    grads = _grads(out, anchor, cfg, seed=4)
    _, (go, ga) = _run(out, anchor, cfg, grads)
    o = out.cuda().requires_grad_()
    a = anchor.cuda().requires_grad_()
    na, g = ro.reference_refine(o, a, cfg)
    ref = dict(new_anchor=na, **g)
    torch.autograd.backward([ref[k] for k in ref], [grads[k].cuda() for k in ref])
    wo, _, wa, _ = ro.refine_backward(out.numpy(), anchor.numpy(), cfg, {k: v.numpy() for k, v in grads.items()})
    h.assert_grad_parity(go.numpy(), wo, o.grad.cpu().numpy(), what=f"{config} grad out")
    h.assert_grad_parity(ga.numpy(), wa, a.grad.cpu().numpy(), what=f"{config} grad anchor")


def test_bit_reproducible_and_independent_of_the_batch():
    out, anchor, cfg = _inputs("prob_gs25600", 2, 3000, seed=5)
    grads = _grads(out, anchor, cfg, seed=6)
    first = _run(out, anchor, cfg, grads)
    for _ in range(2):
        again = _run(out, anchor, cfg, grads)
        assert all(torch.equal(first[0][k], again[0][k]) for k in first[0])
        assert all(torch.equal(x, y) for x, y in zip(first[1], again[1]))
    for b in range(2):
        alone = _run(out[b:b + 1], anchor[b:b + 1], cfg, {k: v[b:b + 1] for k, v in grads.items()})
        assert all(torch.equal(alone[0][k][0], first[0][k][b]) for k in first[0])
        assert all(torch.equal(x[0], y[b]) for x, y in zip(alone[1], first[1]))


@pytest.mark.parametrize("config,subset", [("gs25600_solid", ("means", "semantics")),
                                           ("gs144000", ("new_anchor",)),
                                           ("prob_gs25600", ("scales", "rotations", "delta_means")),
                                           ("prob_gs25600", ("original_means", "opacities"))])
def test_gradient_subsets(config, subset):
    """outputs outside the subset do not reach the loss: their gradients are None, counted as zero and not read"""
    out, anchor, cfg = _inputs(config, 2, 2000, seed=7)
    grads = {k: (v if k in subset else None) for k, v in _grads(out, anchor, cfg, seed=8).items()}
    check_against_oracle(out, anchor, cfg, grads, f"{config} {subset}")


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_half_inputs_equal_the_upcast_inputs(dtype):
    out, anchor, cfg = _inputs("gs25600_solid", 2, 2000, seed=9)
    out, anchor = out.to(dtype), anchor.to(dtype)
    grads = _grads(out.float(), anchor.float(), cfg, seed=10)
    o = out.cuda().requires_grad_()
    a = anchor.cuda().requires_grad_()
    res = _outputs(*gaussian_refine(o, a, **_args(cfg)))
    torch.autograd.backward(list(res.values()), [grads[k].cuda() for k in res])
    full, (go, ga) = _run(out.float(), anchor.float(), cfg, grads)
    for k, v in res.items():
        assert v.dtype == torch.float32 and torch.equal(v.detach().cpu(), full[k]), k
    assert o.grad.dtype == dtype and a.grad.dtype == dtype
    assert torch.equal(o.grad.cpu(), go.to(dtype)) and torch.equal(a.grad.cpu(), ga.to(dtype))


def test_non_contiguous_inputs():
    out, anchor, cfg = _inputs("gs144000", 2, 2000, seed=11)
    wide = torch.cat([out, torch.randn(2, 2000, 4)], -1).cuda()[..., :28]              # row stride 32
    anchor_t = anchor.transpose(0, 1).contiguous().cuda().transpose(0, 1)               # [B, A, D] of an [A, B, D]
    res = _outputs(*gaussian_refine(wide, anchor_t, **_args(cfg)))
    want, _ = _run(out, anchor, cfg)
    assert all(torch.equal(res[k].cpu(), want[k]) for k in want)


def test_cuda_graph_replay_with_new_inputs():
    out, anchor, cfg = _inputs("prob_gs25600", 2, 3000, seed=12)
    o = out.cuda().requires_grad_()
    a = anchor.cuda().requires_grad_()
    grads = _grads(out, anchor, cfg, seed=13)
    up = {k: v.cuda() for k, v in grads.items()}

    def step():
        o.grad = a.grad = None
        res = _outputs(*gaussian_refine(o, a, **_args(cfg)))
        torch.autograd.backward(list(res.values()), [up[k] for k in res])
        return [v.detach() for v in res.values()] + [o.grad, a.grad]

    step()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step()
    torch.cuda.synchronize()
    for seed in (14, 15):
        new_o, new_a, _ = _inputs("prob_gs25600", 2, 3000, seed=seed)
        with torch.no_grad():
            o.copy_(new_o.cuda())
            a.copy_(new_a.cuda())
        graph.replay()
        torch.cuda.synchronize()
        vals, (go, ga) = _run(new_o, new_a, cfg, grads)
        eager = list(vals.values()) + [go, ga]
        assert all(torch.equal(x.cpu(), y) for x, y in zip(static, eager))


def test_no_host_synchronisation():
    out, anchor, cfg = _inputs("gs25600_solid", 1, 4000, seed=16)
    o = out.cuda().requires_grad_()
    a = anchor.cuda().requires_grad_()
    up = {k: v.cuda() for k, v in _grads(out, anchor, cfg, seed=17).items()}
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        res = _outputs(*gaussian_refine(o, a, **_args(cfg)))
        torch.autograd.backward(list(res.values()), [up[k] for k in res])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert torch.isfinite(o.grad).all()


def test_errors():
    out, anchor, cfg = _inputs("gs25600_solid", 1, 64, seed=18)
    o, a = out.cuda(), anchor.cuda()
    gaussian_refine(o, a, **_args(cfg))
    with pytest.raises(RuntimeError, match="CUDA-only"):
        gaussian_refine(o.cpu(), a, **_args(cfg))
    with pytest.raises(ValueError, match="agree in B and A"):
        gaussian_refine(o, a[:, :32], **_args(cfg))
    with pytest.raises(ValueError, match="variant"):
        gaussian_refine(o, a, **dict(_args(cfg), variant="v3"))
    with pytest.raises(GfError, match="expected 10 \\+ include_opa \\+ semantic_dim"):
        gaussian_refine(o[..., :27], a, **_args(cfg))
    with pytest.raises(GfError, match="refine_prefix=3 exceeds"):
        gaussian_refine(o, a[..., :2], **_args(cfg))
    wide = torch.randn(1, 64, 10 + 1 + 33, device="cuda")
    with pytest.raises(GfError, match="compiled maximum"):
        gaussian_refine(wide, a, **dict(_args(cfg), semantic_dim=33))


# ------------------------------------------------------------------------------------------------ end to end
E2E_LAYERS, E2E_ANCHORS = 4, 1024
# GaussianFormer-1's empty Gaussian (config/nuscenes_gs25600_solid.py:179-184, gaussian_head.py:43-48,96-102)
EMPTY_MEAN, EMPTY_SCALE, EMPTY_SCALAR, EMPTY_LABEL = (0.0, 0.0, -1.0), (100.0, 100.0, 8.0), 10.0, 17


def _chain(layers, encoder, generator, agg, anchor, inst, pts, w_kp, w_logits, refine, dtype):
    """E2E_LAYERS refinement layers: anchor_embed = encoder(anchor) (a stand-in for the anchor encoder), the layer's
    new_anchor feeds the key-point generator and its Gaussians, with the empty Gaussian appended as GaussianHead does,
    the splat; the loss weighs key points and logits with fixed random weights.  ``refine(layer, inst, anchor, embed)``
    -> (new_anchor, GaussianPrediction); the generator and the splat always see fp32."""
    loss = 0
    dev = anchor.device
    for i, layer in enumerate(layers):
        new_anchor, gp = refine(layer, inst, anchor, encoder(anchor))
        kp = generator(new_anchor.float(), inst.float())
        B, G = gp.means.shape[:2]
        sem = torch.cat([gp.semantics, torch.zeros_like(gp.semantics[..., :1])], -1)
        empty_sem = torch.zeros(B, 1, sem.shape[-1], dtype=sem.dtype, device=dev)
        empty_sem[..., EMPTY_LABEL] = EMPTY_SCALAR
        t = lambda v: torch.tensor(v, dtype=gp.means.dtype, device=dev).expand(B, 1, len(v))     # noqa: E731
        logits = agg.forward_from_srt(
            pts, torch.cat([gp.means, t(EMPTY_MEAN)], 1).float(),
            torch.cat([gp.opacities[..., 0], torch.ones(B, 1, dtype=sem.dtype, device=dev)], 1).float(),
            torch.cat([sem, empty_sem], 1).float(), torch.cat([gp.scales, t(EMPTY_SCALE)], 1).float(),
            torch.cat([gp.rotations, t((1.0, 0.0, 0.0, 0.0))], 1).float())
        loss = loss + (kp.to(dtype) * w_kp[i].to(dtype)).sum() + (logits.to(dtype) * w_logits[i].to(dtype)).sum()
        anchor = new_anchor
    return loss


def test_four_layers_end_to_end_against_the_pytorch_chain():
    """The device op against the PyTorch restatement over four chained layers (GaussianFormer-1, gs25600_solid
    settings, 1 024 anchors), gradients of instance_feature, the initial anchor and every MLP parameter held to
    assert_grad_parity, the fp64 chain (MLP and refinement in fp64) being the reference and the fp32 one the floor.
    The splat runs on a 4 m grid: every Gaussian's box then has a radius of one voxel and the voxel centres it gains
    or loses when an ulp moves its mean across a voxel face lie > 4 sigma away, so the chains do not diverge there."""
    d = make_refine_inputs("gs25600_solid", batch=1, num_anchor=E2E_ANCHORS, seed=20, margin=True)
    cfg = dict(d["config"], variant="v1")
    D = d["out"].shape[-1]
    torch.manual_seed(21)
    layers = nn.ModuleList([SparseGaussian3DRefinementModule(phi_activation="sigmoid", **d["config"])
                            for _ in range(E2E_LAYERS)]).cuda()
    encoder = nn.Linear(D, 128).cuda()
    generator = SparseGaussian3DKeyPointsGenerator(embed_dims=128, num_learnable_pts=2, fix_scale=ANCHOR_FIX_SCALE,
                                                   pc_range=cfg["pc_range"], scale_range=cfg["scale_range"]).cuda()
    agg = LocalAggregator(scale_multiplier=3, H=25, W=25, D=2, pc_min=[-50.0, -50.0, -5.0], grid_size=4.0).cuda()
    pts = agg.grid_points("cuda")
    gen = torch.Generator().manual_seed(22)
    w_kp = [torch.randn(1, E2E_ANCHORS, 9, 3, generator=gen).cuda() for _ in range(E2E_LAYERS)]
    w_logits = [torch.randn(pts.shape[1], 18, generator=gen).cuda() for _ in range(E2E_LAYERS)]

    def device(layer, inst, anchor, embed):
        return layer(inst, anchor, embed)

    def pytorch(layer, inst, anchor, embed):
        na, g = ro.reference_refine(layer.layers(inst + embed), anchor, cfg)
        return na, GaussianPrediction(**g)

    results = {}
    for name, refine, dtype in (("device", device, torch.float32), ("fp32", pytorch, torch.float32),
                                ("fp64", pytorch, torch.float64)):
        ls, enc = (layers, encoder) if dtype == torch.float32 else (copy.deepcopy(layers).double(),
                                                                    copy.deepcopy(encoder).double())
        inst = d["instance_feature"].cuda().to(dtype).requires_grad_()
        anchor = d["anchor"].cuda().to(dtype).requires_grad_()
        for p in ls.parameters():
            p.grad = None
        _chain(ls, enc, generator, agg, anchor, inst, pts, w_kp, w_logits, refine, dtype).backward()
        grads = dict(instance_feature=inst.grad, anchor=anchor.grad,
                     **{f"mlp {k}": p.grad for k, p in ls.named_parameters()})
        results[name] = {k: v.detach().double().cpu().numpy() for k, v in grads.items()}
    for k in results["device"]:
        assert np.isfinite(results["device"][k]).all(), k
        h.assert_grad_parity(results["device"][k], results["fp64"][k], results["fp32"][k], what=f"end to end {k}")
