"""ABI 2 features of the splat op on the GPU: the batched launch (gf_splat_desc.batch / pts_shared), the inverse
covariance built inside the pack kernel from scales + rotations with its own backward (SURVEY.md 8f-1), and the
render epilogue's class-major logits, arg-max and softmax cross-entropy partial sums (SURVEY.md 8f-3)."""
import numpy as np
import pytest
import torch

import helpers as h

pytestmark = pytest.mark.gpu


def _batch_of(cfg, seeds, perturb, over=None, per_axis=False):
    kws, inps = [], []
    for s in seeds:
        kw, inp, variant = h.splat_case(cfg, s, perturb, over, per_axis=per_axis)
        kws.append(kw); inps.append(inp)
    cat = {k: torch.cat([i[k] for i in inps], 0) for k in inps[0]}
    return kws[0], inps, cat, variant


@pytest.mark.parametrize("cfg,per_axis,over", [
    ("tiny", False, None),
    ("tiny", False, dict(dims=(37, 21, 6), pc_min=(-9.0, -5.0, -1.5))),    # ragged bins, scalar stores
    ("tiny_prob", False, None),
    ("tiny_prob", True, None),
    ("gs25600_solid", False, dict(G=1500)),                                 # full grid, whole-grid Gaussian per sample
])
def test_batched_launch_equals_per_sample_calls(cfg, per_axis, over):
    """B distinct samples in ONE call (forward and backward) == B separate calls, bit for bit in the forward."""
    kw, inps, cat, variant = _batch_of(cfg, (21, 22, 23), True, over, per_axis)
    m = h.make_module(kw, variant)
    tb = h.to_dev(cat, requires_grad=True)
    outb = m(tb["pts"], tb["means"], tb["opa"], tb["sem"], tb["scales"], tb["cov"])
    outb = (outb,) if variant == "base" else tuple(outb)
    gen = torch.Generator().manual_seed(5)
    gs = [torch.randn(o.shape, generator=gen).cuda() for o in outb]
    torch.autograd.backward(list(outb), gs)
    for b, inp in enumerate(inps):
        t = h.to_dev(inp, requires_grad=True)
        out = m(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"])
        out = (out,) if variant == "base" else tuple(out)
        for o, ob in zip(out, outb):
            assert torch.equal(o, ob[b]), (cfg, b)
        torch.autograd.backward(list(out), [g[b] for g in gs])
        for k in ("means", "opa", "sem", "cov"):
            ref = t[k].grad[0].cpu().numpy()
            h.assert_close(tb[k].grad[b].cpu().numpy(), ref, rtol=1e-4, atol=1e-5 * max(1.0, float(np.abs(ref).max())),
                           what=f"{cfg} batch grad {k}[{b}]")


def test_shared_points_and_forward_on_grid_batch():
    kw, inps, cat, variant = _batch_of("gs25600_solid", (31, 32), False, dict(G=800))
    m = h.make_module(kw, variant)
    t = h.to_dev(cat)
    full = m(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"])
    grid = m.forward_on_grid(t["means"], t["opa"], t["sem"], t["scales"], t["cov"])     # pts_shared = 1
    assert full.shape == grid.shape == (2, 640000, 18)
    assert torch.equal(full, grid)


@pytest.mark.parametrize("cfg", ["tiny", "tiny_prob"])
def test_in_kernel_inverse_covariance_and_its_backward(cfg):
    """forward_from_srt: Sigma^-1 = R^T diag(1/s^2) R inside the pack kernel; backward: d/dscales, d/drotations from the
    srt kernel.  Values: against the reference's CPU inverse (gaussian_head.py:111-119) fed through the standard entry
    point.  Gradients of all five leaves: every sample against the fp64 chain of tests/srt_oracle.py with
    helpers.assert_grad_parity (srt_oracle.check_grads)."""
    import srt_oracle as so
    from gaussianformer_b200.synthetic import inverse_covariance
    kw, inps, cat, variant = _batch_of(cfg, (41, 42), True)
    B, G = cat["means"].shape[:2]
    gen = torch.Generator().manual_seed(2)
    rots = torch.randn(B, G, 4, generator=gen) * 1.7            # un-normalised on purpose
    m = h.make_module(kw, variant)
    t = h.to_dev(cat)
    # values: against the reference's numerical inverse fed through the standard entry point
    ref_cov = inverse_covariance(cat["scales"], rots).float().cuda()
    out_ref = m(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], ref_cov)
    leaves = {k: t[k].clone().requires_grad_(True) for k in ("means", "opa", "sem", "scales")}
    leaves["rotations"] = rots.cuda().requires_grad_(True)
    out = m.forward_from_srt(t["pts"], leaves["means"], leaves["opa"], leaves["sem"], leaves["scales"], leaves["rotations"])
    first = out if variant == "base" else out[0]
    first_ref = out_ref if variant == "base" else out_ref[0]
    h.assert_close(first.detach().cpu().numpy(), first_ref.cpu().numpy(), rtol=1e-3, atol=1e-4, what="logits from s, r")
    # gradients: against the fp64 chain, per sample
    outs = (out,) if variant == "base" else tuple(out)
    gs = [torch.randn(o.shape, generator=gen) for o in outs]
    torch.autograd.backward(list(outs), [x.cuda() for x in gs])
    for b, inp in enumerate(inps):
        mine_out = [o[b].detach().cpu().numpy() for o in outs]
        chains = so.srt_chains(kw, inp, inp["scales"][0], rots[b], variant, tuple(x[b].numpy() for x in gs),
                               op_outputs=mine_out[:2])
        so.check_grads({k: v.grad[b].cpu().numpy() for k, v in leaves.items()}, chains[0][1], chains[1][1],
                       f"{cfg} sample {b}")
    r1, s1 = leaves["rotations"], leaves["scales"]
    assert float(r1.grad.abs().max()) > 0 and torch.isfinite(s1.grad).all()
    # the gradient of an un-normalised quaternion is orthogonal to it (F.normalize)
    dots = (r1.grad * r1.detach()).sum(-1).abs().max()
    assert float(dots) <= 1e-3 * float(r1.grad.abs().max()) * float(r1.detach().abs().max()) + 1e-6


@pytest.mark.parametrize("over", [None, dict(dims=(37, 21, 6), pc_min=(-9.0, -5.0, -1.5))])
def test_fused_epilogue_outputs(over):
    """forward_eval: [B,C,N] logits, arg-max and the CE_ssc_loss from per-CTA partial sums == PyTorch on the op's
    own [N,C] logits (loss/occupancy_loss.py:164-178: CrossEntropyLoss(weight, ignore_index=255, 'mean'))."""
    kw, inps, cat, variant = _batch_of("tiny", (51, 52, 53), True, over)
    m = h.make_module(kw, variant)
    t = h.to_dev(cat)
    logits = m(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"])           # [B,N,C]
    B, N, C = logits.shape
    gen = torch.Generator().manual_seed(9)
    labels = torch.randint(0, C, (B, N), generator=gen)
    labels[torch.rand(B, N, generator=gen) < 0.2] = 255
    cw = torch.rand(C, generator=gen) + 0.5
    r = m.forward_eval(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"], labels=labels.cuda(),
                       class_weights=cw.cuda(), layout="cn")
    assert r["logits"] is None and r["pred_occ"].shape == (B, C, N)
    assert torch.equal(r["pred_occ"], logits.transpose(1, 2))
    first = (logits == logits.max(dim=2, keepdim=True).values).float().argmax(dim=2)
    assert torch.equal(r["final_occ"].long(), first)
    want = torch.nn.functional.cross_entropy(logits.double().transpose(1, 2), labels.cuda(), weight=cw.double().cuda(),
                                             ignore_index=255, reduction="mean")
    assert abs(float(r["ce_loss"]) - float(want)) <= 2e-5 * abs(float(want)) + 1e-6, (float(r["ce_loss"]), float(want))
    # unweighted, and the [N,C] layout through the same entry point
    r2 = m.forward_eval(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"], labels=labels.cuda(), layout="nc")
    want2 = torch.nn.functional.cross_entropy(logits.double().transpose(1, 2), labels.cuda(), ignore_index=255)
    assert torch.equal(r2["logits"], logits) and r2["pred_occ"] is None
    assert abs(float(r2["ce_loss"]) - float(want2)) <= 2e-5 * abs(float(want2)) + 1e-6
    # layout=None: nothing but the prediction (and the loss) leaves the kernel
    r3 = m.forward_eval(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"], layout=None)
    assert r3["logits"] is None and r3["pred_occ"] is None and torch.equal(r3["final_occ"], r["final_occ"])


def test_misaligned_tensors_take_the_scalar_path():
    """Tensors whose storage offset breaks the 16-byte alignment of the vector loads / stores (ADVICE r01) are
    handled by the scalar accesses of the same kernels: same results, no fault."""
    kw, inp, variant = h.splat_case("tiny", 61, True)
    m = h.make_module(kw, variant)
    t = h.to_dev(inp)
    ref = m(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"])
    buf = torch.empty(t["pts"].numel() + 1, device="cuda")
    pts_odd = buf[1:].view_as(t["pts"])
    pts_odd.copy_(t["pts"])
    assert pts_odd.data_ptr() % 16 == 4
    out = m(pts_odd, t["means"], t["opa"], t["sem"], t["scales"], t["cov"])
    assert torch.equal(out, ref)


def test_module_follows_its_buffer_and_attributes():
    """The reference reads self.pc_min and its attributes on every call; a checkpoint that carries another origin,
    or an attribute changed after the first forward, must take effect (ADVICE r01)."""
    kw, inp, variant = h.splat_case("tiny", 62, True)
    m = h.make_module(kw, variant)
    t = h.to_dev(inp)
    a = m(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"])
    shift = torch.tensor([[0.5, 0.0, 0.0]])
    sd = {"pc_min": m.pc_min.cpu() + shift}
    m.load_state_dict(sd)
    b = m(t["pts"] + shift.cuda(), t["means"] + shift.cuda(), t["opa"], t["sem"], t["scales"], t["cov"])
    h.assert_close(b.cpu().numpy(), a.cpu().numpy(), what="shifted origin + shifted inputs")
    m.scale_multiplier = 1                      # smaller boxes -> fewer contributions -> a different result
    c = m(t["pts"] + shift.cuda(), t["means"] + shift.cuda(), t["opa"], t["sem"], t["scales"], t["cov"])
    assert not torch.equal(b, c)


def test_prob_outputs_are_independent_tensors():
    kw, inp, variant = h.splat_case("tiny_prob", 63, True)
    m = h.make_module(kw, variant)
    t = h.to_dev(inp, requires_grad=True)
    lg, bl, de = m(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"])
    de.clamp_(max=0.5)                          # an in-place edit of one output (ADVICE r01) ...
    (lg.sum() + bl.sum()).backward()            # ... must not invalidate what backward saved
    assert torch.isfinite(t["means"].grad).all()
