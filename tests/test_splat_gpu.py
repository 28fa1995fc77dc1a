"""Parity of the sm_90a splat kernels (through the public modules -> C ABI) against the oracle,
and the committed reference-op goldens.
Tolerance: |new - ref| <= 1e-5 + 1e-4*|ref| elementwise in fp32 (helpers.RTOL/ATOL)."""
import os

import numpy as np
import pytest
import torch

import helpers as h

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _run(kw, inp, variant, requires_grad=False, validate=True):
    m = h.make_module(kw, variant, validate=validate)
    t = h.to_dev(inp, requires_grad=requires_grad)
    out = m(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"])
    return m, t, out


@pytest.mark.parametrize("cfg,seed,perturb,over", [
    ("tiny", 0, False, None),
    ("tiny", 1, True, None),
    ("tiny", 2, True, dict(dims=(37, 21, 6), pc_min=(-9.0, -5.0, -1.5))),      # D % 4 != 0, ragged bins
    ("tiny", 3, False, dict(dims=(16, 8, 40), pc_min=(-4.0, -2.0, -10.0))),     # several z chunks; > 32 levels: no z-level mask in the record
    ("tiny", 5, False, dict(dims=(16, 8, 32), pc_min=(-4.0, -2.0, -8.0))),      # two z chunks, z-level mask uses all 32 bits
    ("tiny", 6, False, dict(dims=(12, 8, 24), pc_min=(-3.0, -2.0, -6.0))),      # second chunk half empty
    ("tiny", 4, True, dict(G=1)),
    ("gs25600_solid", 0, True, dict(G=3000)),                                   # full grid + empty Gaussian
])
def test_base_forward_vs_oracle(cfg, seed, perturb, over):
    kw, inp, variant = h.splat_case(cfg, seed, perturb, over)
    _, _, out = _run(kw, inp, variant)
    ref = h.oracle_forward(kw, inp, variant)
    h.assert_close(out.cpu().numpy(), ref["logits"], what="logits")
    h.assert_argmax_parity(out.cpu().numpy(), ref["logits"])


@pytest.mark.parametrize("cfg,seed,perturb,per_axis,over", [
    ("tiny_prob", 0, False, False, None),
    ("tiny_prob", 2, True, True, None),
    ("tiny_prob", 5, True, False, dict(dims=(19, 30, 10), pc_min=(-5.0, -7.0, -2.5))),
    ("prob_gs6400", 0, True, False, dict(G=400)),
])
def test_prob_forward_vs_oracle(cfg, seed, perturb, per_axis, over):
    kw, inp, variant = h.splat_case(cfg, seed, perturb, over, per_axis=per_axis)
    _, _, (lg, bl, de) = _run(kw, inp, variant)
    ref = h.oracle_forward(kw, inp, variant)
    z = ref["probability"]
    stable = np.abs(z - 1e-9) > 1e-10      # voxels on the fallback switch may take either branch
    h.assert_close(lg.cpu().numpy()[stable], ref["logits"][stable], what="logits")
    h.assert_close(bl.cpu().numpy(), ref["bin_logits"], what="bin_logits")
    h.assert_close(de.cpu().numpy(), ref["density"], what="density")


def test_base_backward_vs_oracle():
    kw, inp, variant = h.splat_case("gs25600_solid", 3, True, dict(G=2000))
    _, t, out = _run(kw, inp, variant, requires_grad=True)
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(7))
    out.backward(g.cuda())
    h.check_module_grads(t, kw, inp, variant, (g.numpy(),), what="base")


@pytest.mark.parametrize("per_axis", [False, True])
def test_prob_backward_vs_oracle(per_axis):
    kw, inp, variant = h.splat_case("prob_gs6400", 1, True, dict(G=300), per_axis=per_axis)
    _, t, (lg, bl, de) = _run(kw, inp, variant, requires_grad=True)
    gen = torch.Generator().manual_seed(9)
    g = (torch.randn(lg.shape, generator=gen), torch.randn(bl.shape, generator=gen), torch.randn(de.shape, generator=gen))
    torch.autograd.backward([lg, bl, de], [x.cuda() for x in g])
    # feed the oracle the saved outputs of the op under test (as the reference's backward receives them)
    from gaussianformer_b200 import splat as S  # noqa: F401
    ref_f = h.oracle_forward(kw, inp, variant, "f32")
    saved = dict(logits=lg.detach().cpu().numpy(), bin_logits=bl.detach().cpu().numpy(),
                 probability=ref_f["probability"])
    h.check_module_grads(t, kw, inp, variant, tuple(x.numpy() for x in g), what="prob", saved_from=saved)


def test_generic_points_path():
    """Arbitrary points: shuffled order, duplicates in one voxel, N != H*W*D (reference debug.py usage)."""
    kw, inp, variant = h.splat_case("tiny", 6, True)
    gen = torch.Generator().manual_seed(0)
    pts = inp["pts"][0]
    idx = torch.cat([torch.randperm(pts.shape[0], generator=gen)[:7000], torch.arange(50)])
    inp = dict(inp, pts=pts[idx][None].contiguous())
    _, _, out = _run(kw, inp, variant)
    ref = h.oracle_forward(kw, inp, variant)
    h.assert_close(out.cpu().numpy(), ref["logits"], what="generic logits")
    # same N as the grid but permuted: the tile kernel must detect it and hand over
    perm = torch.randperm(pts.shape[0], generator=gen)
    inp2 = dict(inp, pts=pts[perm][None].contiguous())
    _, _, out2 = _run(kw, inp2, variant)
    ref2 = h.oracle_forward(kw, inp2, variant)
    h.assert_close(out2.cpu().numpy(), ref2["logits"], what="permuted logits")


def test_backward_properties_full_size():
    """BASELINE config 2 at full size, forward and backward tied together without an oracle run:
    (i) Euler identities -- the output is linear in the opacities and in the class vectors, so
        <G, out> == <opa, dL/dopa> == <sem, dL/dsem> for any upstream G;
    (ii) the backward is linear in the upstream gradient;
    (iii) the covariance gradient lives on the six gathered entries of the 3x3 only;
    (iv) a finite difference along a random direction of the means matches <dL/dmeans, direction>."""
    kw, inp, variant = h.splat_case("gs25600_solid", 5, True)
    m = h.make_module(kw, variant)
    t = h.to_dev(inp, requires_grad=True)
    out = m(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"])
    gen = torch.Generator(device="cuda").manual_seed(11)
    g1 = torch.randn(out.shape, device="cuda", generator=gen)
    g2 = torch.randn(out.shape, device="cuda", generator=gen)
    wrt = [t["means"], t["opa"], t["sem"], t["cov"]]
    a = torch.autograd.grad(out, wrt, g1, retain_graph=True)
    b = torch.autograd.grad(out, wrt, g2, retain_graph=True)
    c = torch.autograd.grad(out, wrt, g1 + 2 * g2, retain_graph=True)
    inner = float((g1.double() * out.detach().double()).sum())
    via_opa = float((t["opa"].detach().double() * a[1].double()).sum())
    via_sem = float((t["sem"].detach().double() * a[2].double()).sum())
    assert abs(via_opa - inner) <= 1e-4 * abs(inner) + 1e-3, (via_opa, inner)
    assert abs(via_sem - inner) <= 1e-4 * abs(inner) + 1e-3, (via_sem, inner)
    for x, y, z, name in zip(a, b, c, ("means", "opa", "sem", "cov")):
        ref = (x.double() + 2 * y.double()).cpu().numpy()
        h.assert_close(z.cpu().numpy(), ref, rtol=1e-3, atol=h.grad_tolerance(ref), what=f"linearity of grad {name}")
    gcov = a[3].reshape(-1, 9)
    assert float(gcov[:, [3, 6, 7]].abs().max()) == 0.0
    # directional finite difference in float64-accumulated loss
    d = torch.randn(t["means"].shape, device="cuda", generator=gen)
    d[:, -1] = 0                                        # keep the whole-grid "empty" Gaussian put
    # the integer box follows the mean's voxel: only move means that cannot cross a voxel face (the op is
    # discontinuous there, like the reference)
    frac = ((t["means"].detach() - m.pc_min.view(1, 1, 3)) / m.grid_size) % 1.0
    d = d * ((frac > 0.1) & (frac < 0.9)).all(dim=-1, keepdim=True)
    eps = 1e-3
    with torch.no_grad():
        lp = (m(t["pts"], t["means"] + eps * d, t["opa"], t["sem"], t["scales"], t["cov"]).double() * g1.double()).sum()
        lm = (m(t["pts"], t["means"] - eps * d, t["opa"], t["sem"], t["scales"], t["cov"]).double() * g1.double()).sum()
    fd = float((lp - lm) / (2 * eps))
    an = float((a[0].double() * d.double()).sum())
    assert abs(fd - an) <= 2e-2 * max(abs(an), abs(fd)) + 1e-2, (fd, an)


def test_backward_generic_points_and_unaligned_gradients():
    """Backward paths off the fast lane: points not in voxel order (voxel -> point map), a subset of the grid
    (empty voxels), and upstream gradients whose storage is only 4- or 8-byte aligned (narrow row loads)."""
    import oracle
    kw, inp, variant = h.splat_case("tiny", 11, True)
    gen = torch.Generator().manual_seed(3)
    pts = inp["pts"][0]
    perm = torch.randperm(pts.shape[0], generator=gen)
    for idx, offset in ((perm, 0), (perm[: pts.shape[0] // 2], 0), (torch.arange(pts.shape[0]), 1),
                        (torch.arange(pts.shape[0]), 2)):
        inp2 = dict(inp, pts=pts[idx][None].contiguous())
        _, t, out = _run(kw, inp2, variant, requires_grad=True)
        g = torch.randn(out.shape, generator=gen)
        flat = torch.empty(g.numel() + offset, device="cuda")
        g_dev = flat[offset:].view_as(g)          # storage offset of `offset` floats
        g_dev.copy_(g)
        assert g_dev.data_ptr() % 16 == 4 * offset
        out.backward(g_dev)
        h.check_module_grads(t, kw, inp2, variant, (g.numpy(),), what=f"(N={len(idx)}, offset={offset})")


def test_reference_asserts_are_raised():
    kw, inp, variant = h.splat_case("tiny", 0)
    bad = dict(inp, means=inp["means"].clone())
    bad["means"][0, 3, 0] = 1e3                       # mean outside the grid
    with pytest.raises(AssertionError):
        _run(kw, bad, variant)
    bad = dict(inp, scales=inp["scales"] * 0.0)       # radii.min() < 1
    with pytest.raises(AssertionError):
        _run(kw, bad, variant)
    bad = dict(inp, pts=inp["pts"].clone())
    bad["pts"][0, 5] = -1e3                           # point outside the grid
    with pytest.raises(AssertionError):
        _run(kw, bad, variant)


def test_batched_and_linearity_properties_full_size():
    """BASELINE config 2 at full size: size-independent properties (no oracle run needed).
    (i) the op is linear in opacity: out(2*opa) == 2*out(opa) up to fp32 rounding;
    (ii) splitting the Gaussian set in two and adding the halves reproduces the whole;
    (iii) a batch of 2 equals two single calls."""
    kw, inp, variant = h.splat_case("gs25600_solid", 0, True)
    m = h.make_module(kw, variant)
    t = h.to_dev(inp)
    out = m(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"])
    out2 = m(t["pts"], t["means"], 2 * t["opa"], t["sem"], t["scales"], t["cov"])
    h.assert_close(out2.cpu().numpy(), 2 * out.cpu().numpy(), what="opacity linearity")
    G = t["means"].shape[1]
    halves = []
    for sl in (slice(0, G // 2), slice(G // 2, G)):
        halves.append(m(t["pts"], t["means"][:, sl], t["opa"][:, sl], t["sem"][:, sl], t["scales"][:, sl], t["cov"][:, sl]))
    h.assert_close((halves[0] + halves[1]).cpu().numpy(), out.cpu().numpy(), rtol=2e-4, what="additivity over Gaussians")
    b2 = {k: torch.cat([v, v.flip(1) if k != "pts" else v], 0) for k, v in t.items()}
    outb = m(b2["pts"], b2["means"], b2["opa"], b2["sem"], b2["scales"], b2["cov"])
    assert outb.shape == (2,) + tuple(out.shape)
    assert torch.equal(outb[0], out)


@pytest.mark.parametrize("fixture,cfg,seed,perturb,per_axis", [
    ("ref_splat_base_tiny", "tiny", 0, False, False),
    ("ref_splat_base_tiny_perturb", "tiny", 1, True, False),
    ("ref_splat_prob_tiny", "tiny_prob", 0, False, False),
    ("ref_splat_probfast_tiny", "tiny_prob", 2, True, True),
])
def test_vs_reference_goldens(fixture, cfg, seed, perturb, per_axis):
    path = os.path.join(GOLD, fixture + ".npz")
    if not os.path.exists(path):
        pytest.skip("golden fixture not generated yet")
    gold = np.load(path)
    kw, inp, variant = h.splat_case(cfg, seed, perturb, per_axis=per_axis)
    _, t, out = _run(kw, inp, variant, requires_grad=True)
    gen = torch.Generator().manual_seed(int(gold["grad_seed"]))
    if variant == "base":
        h.assert_close(out.detach().cpu().numpy(), gold["logits"], what="logits vs reference op")
        g_base = torch.randn(out.shape, generator=gen)
        out.backward(g_base.cuda())
    else:
        lg, bl, de = out
        z = gold["probability"]
        stable = np.abs(z - 1e-9) > 1e-10
        h.assert_close(lg.detach().cpu().numpy()[stable], gold["logits"][stable], what="logits vs reference op")
        h.assert_close(bl.detach().cpu().numpy(), gold["bin_logits"], what="bin vs reference op")
        h.assert_close(de.detach().cpu().numpy(), gold["density"], what="density vs reference op")
        g = [torch.randn(lg.shape, generator=gen), torch.randn(bl.shape, generator=gen), torch.randn(de.shape, generator=gen)]
        torch.autograd.backward([lg, bl, de], [x.cuda() for x in g])
    import oracle
    golden = {"means": gold["means_grad"], "opa": gold["opacity_grad"], "sem": gold["semantics_grad"],
              "cov": oracle.cov6_grad_to_3x3(gold["cov_grad"])}
    if variant == "base":
        grads_np, saved = (g_base.numpy(),), None
    else:   # the reference's backward received the reference's own forward outputs
        grads_np = tuple(x.numpy() for x in g)
        saved = dict(logits=gold["logits"], bin_logits=gold["bin_logits"], probability=gold["probability"])
    h.check_module_grads(t, kw, inp, variant, grads_np, what=fixture, saved_from=saved, golden=golden)


def test_vs_reference_golden_mid_size():
    """The mid-size reference-op golden (full config-2 grid, 2000 Gaussians + the whole-grid one)."""
    path = os.path.join(GOLD, "ref_splat_base_mid.npz")
    if not os.path.exists(path):
        pytest.skip("mid-size golden not generated yet")
    gold = np.load(path)
    kw, inp, variant = h.splat_case("gs25600_solid", 7, False, dict(G=2000))
    _, t, out = _run(kw, inp, variant, requires_grad=True)
    stride = int(gold["row_stride"])
    got = out.detach().cpu().numpy()
    h.assert_close(got[::stride], gold["logits_rows"], what="sampled logits rows vs reference op")
    tol = h.ATOL * got.shape[0] + h.RTOL * gold["logits_abs_colsum"]
    assert np.all(np.abs(got.astype(np.float64).sum(0) - gold["logits_colsum"]) <= tol)
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(int(gold["grad_seed"])))
    out.backward(g.cuda())
    import oracle
    golden = {"means": gold["means_grad"], "opa": gold["opacity_grad"], "sem": gold["semantics_grad"],
              "cov": oracle.cov6_grad_to_3x3(gold["cov_grad"])}
    h.check_module_grads(t, kw, inp, variant, (g.numpy(),), what="mid golden", golden=golden)


def test_fused_argmax_matches_logits():
    kw, inp, variant = h.splat_case("gs25600_solid", 2, True, dict(G=2000))
    m = h.make_module(kw, variant)
    t = h.to_dev(inp)
    logits, occ = m.forward_with_occupancy(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"])
    ref = m(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"])
    assert torch.equal(logits, ref)
    assert occ.dtype == torch.uint8 and occ.shape == (logits.shape[0],)
    picked = logits.gather(1, occ.long()[:, None])[:, 0]
    assert torch.equal(picked, logits.max(dim=1).values)          # a maximiser ...
    first = (logits == logits.max(dim=1, keepdim=True).values).float().argmax(dim=1)
    assert torch.equal(occ.long(), first)                          # ... and the lowest-index one
    # stray points (permuted order) go through the per-point path and must report their arg-max too
    perm = torch.randperm(t["pts"].shape[1], generator=torch.Generator().manual_seed(0)).cuda()
    lg2, occ2 = m.forward_with_occupancy(t["pts"][:, perm].contiguous(), t["means"], t["opa"], t["sem"], t["scales"], t["cov"])
    first2 = (lg2 == lg2.max(dim=1, keepdim=True).values).float().argmax(dim=1)
    assert torch.equal(occ2.long(), first2)


@pytest.mark.parametrize("C", [16, 17, 19, 20])
@pytest.mark.parametrize("variant", ["base", "prob"])
def test_other_class_counts(C, variant):
    """The reference hard-codes 18 classes (src/config.h:15); the library is compiled for 16..20."""
    cfg = "tiny" if variant == "base" else "tiny_prob"
    kw, inp, _ = h.splat_case(cfg, 9, True)
    G = inp["sem"].shape[1]
    sem = torch.rand(1, G, C, generator=torch.Generator().manual_seed(C))
    inp = dict(inp, sem=sem)
    m = h.make_module(kw, variant)
    t = h.to_dev(inp, requires_grad=True)
    out = m(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"])
    ref = h.oracle_forward(kw, inp, variant)
    first = out if variant == "base" else out[0]
    stable = np.ones(first.shape[0], bool) if variant == "base" else np.abs(ref["probability"] - 1e-9) > 1e-10
    h.assert_close(first.detach().cpu().numpy()[stable], ref["logits"][stable], what=f"C={C} logits")
    gen = torch.Generator().manual_seed(1)
    if variant == "base":
        g = (torch.randn(first.shape, generator=gen),)
        first.backward(g[0].cuda())
        saved = None
    else:
        g = (torch.randn(out[0].shape, generator=gen), torch.randn(out[1].shape, generator=gen),
             torch.randn(out[2].shape, generator=gen))
        torch.autograd.backward(list(out), [x.cuda() for x in g])
        saved = dict(logits=out[0].detach().cpu().numpy(), bin_logits=out[1].detach().cpu().numpy(),
                     probability=h.oracle_forward(kw, inp, variant, "f32")["probability"])
    h.check_module_grads(t, kw, inp, variant, tuple(x.numpy() for x in g), what=f"C={C}", saved_from=saved)


def test_forward_from_scales_and_rotations():
    """The closed-form device-side Sigma^-1 (forward_from_srt) against the reference's route
    (Cov = (S R)^T (S R), numerical inverse on the CPU): same logits, and gradients reach scales/rotations."""
    from gaussianformer_b200.splat import inverse_covariance_from_srt
    from gaussianformer_b200.synthetic import inverse_covariance
    kw, inp, variant = h.splat_case("tiny", 13, True)
    gen = torch.Generator().manual_seed(2)
    G = inp["means"].shape[1]
    rots = torch.randn(1, G, 4, generator=gen)
    scales = inp["scales"]
    ref_cov = inverse_covariance(scales, rots)                       # CPU inverse, like the reference
    dev_cov = inverse_covariance_from_srt(scales.cuda(), rots.cuda())
    h.assert_close(dev_cov.cpu().numpy(), ref_cov.numpy(), rtol=1e-4, atol=1e-4 * float(ref_cov.abs().max()), what="Sigma^-1")
    m = h.make_module(kw, variant)
    t = h.to_dev(dict(inp, cov=ref_cov))
    out_ref = m(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"])
    s_d = scales.cuda().requires_grad_(True)
    r_d = rots.cuda().requires_grad_(True)
    out = m.forward_from_srt(t["pts"], t["means"], t["opa"], t["sem"], s_d, r_d)
    h.assert_close(out.detach().cpu().numpy(), out_ref.cpu().numpy(), rtol=1e-3, atol=1e-4, what="logits from s, r")
    out.sum().backward()
    assert s_d.grad is not None and r_d.grad is not None
    assert torch.isfinite(s_d.grad).all() and torch.isfinite(r_d.grad).all() and float(r_d.grad.abs().max()) > 0


def test_miou_is_unchanged():
    """North star: mIoU on SurroundOcc-shaped synthetic inputs is unchanged.  SURVEY.md 8(d) recipe: labels = arg-max
    of the fp64 oracle with 10 % of the voxels re-drawn (seed 1), mask = label != 0; the fused arg-max of the CUDA
    path and the oracle's arg-max are scored with the reference's MeanIoU (misc/metric_util.py:35-111).  The
    gs144000-style sample (N(0,1) class vectors, no empty Gaussian) is used because its arg-max spreads over all 18
    classes (on gs25600_solid the empty Gaussian's 10*e_17 wins every voxel and the score degenerates).
    Gates (BASELINE.md): no arg-max difference on a numerically decided voxel; MeanIoU equal within 1e-4 points over the
    decided voxels; over ALL voxels (numerical ties included) within 1e-4 + K x the measured distance between the
    oracle's own fp32 and fp64 builds (the fp32 floor of the arithmetic on this sample, printed).
    The full-size op-vs-op version of this test is tests/test_parity_full_gpu.py (0 differences against the reference
    op on configs 2, 3 and 4)."""
    from gaussianformer_b200.metric import miou_parity, synthetic_labels
    kw, inp, variant = h.splat_case("gs144000", 5, False, dict(G=20000))
    m = h.make_module(kw, variant)
    t = h.to_dev(inp)
    logits, occ = m.forward_with_occupancy(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"])
    ref = h.oracle_forward(kw, inp, variant)["logits"]
    ref32 = h.oracle_forward(kw, inp, variant, "f32")["logits"]
    h.assert_argmax_parity(logits.cpu().numpy(), ref)
    C = ref.shape[1]
    labels, mask = synthetic_labels(ref, C)
    tie = torch.as_tensor(h.tie_voxels(ref))
    am, am64, am32 = occ.cpu().long(), torch.as_tensor(ref.argmax(1)), torch.as_tensor(ref32.argmax(1))
    assert int(((am != am64) & ~tie).sum()) == 0
    r_dec = miou_parity(am, am64, labels, mask & ~tie, C)
    r_all = miou_parity(am, am64, labels, mask, C)
    floor = miou_parity(am32, am64, labels, mask, C)
    print("mIoU all voxels", r_all, "fp32-vs-fp64 oracle floor", floor["abs_diff"], "flips", int((am != am64).sum()),
          "oracle fp32 flips", int((am32 != am64).sum()), "tie voxels", int(tie.sum()))
    assert r_dec["abs_diff"] <= 1e-4, r_dec
    assert r_all["abs_diff"] <= 1e-4 + h.K_FLOOR * floor["abs_diff"], (r_all, floor)
    assert int((am != am64).sum()) <= max(64, h.K_FLOOR * int((am32 != am64).sum()))
    assert r_all["ref"][0] > 50.0            # the labels are a meaningful target (10 % noise), not a degenerate score


def test_forward_on_grid_is_forward_on_the_voxel_centres():
    kw, inp, variant = h.splat_case("gs25600_solid", 7, False, dict(G=1500))
    m = h.make_module(kw, variant)
    t = h.to_dev(inp)
    a = m(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"])
    b = m.forward_on_grid(t["means"], t["opa"], t["sem"], t["scales"], t["cov"])
    assert torch.equal(m.grid_points(a.device), t["pts"])      # the synthetic points ARE the loader's voxel centres
    assert torch.equal(a, b)
    assert "_grid_pts" not in m.state_dict() and list(m.state_dict().keys()) == ["pc_min"]
