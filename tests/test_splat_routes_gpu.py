"""Every kernel route of the splat op against the fp64 oracle, for all three variants.

The op picks its kernels from the inputs.  Forward: the tile kernel for points in canonical voxel order (point n in
voxel n), the same kernel re-evaluating stray points in place (N == H*W*D, not canonical), and render_points_kernel
for N != H*W*D.  Backward: the bin-centric kernel (N == H*W*D, D % 4 == 0, aligned points and logits gradient), its
hand-over to the Gaussian-centric chain when it finds a stray point, and that chain called directly (voxel map ->
small -> big boxes).  The shipped configs feed voxel centres in grid order, so the rest of the suite mostly runs the
tile and bin kernels; here every case is built to take one of the other routes, and every case that reaches the
Gaussian-centric chain holds a clipped box of more than kBigBox = 2048 voxels, so that backward_big_kernel has queued
work.  Gates: helpers.assert_close for the outputs, helpers.check_module_grads for the four gradients."""
import numpy as np
import pytest
import torch

import helpers as h
import oracle

pytestmark = pytest.mark.gpu

K_BIG_BOX = 2048   # splat_bwd_common.cuh kBigBox: larger clipped boxes go to backward_big_kernel's queue

# per variant: (config, seed, overrides, per-axis radii), each with at least one clipped box above K_BIG_BOX voxels
BASE_INPUTS = {
    "base": ("tiny", 0, dict(with_empty=True), False),                 # + the whole-grid Gaussian (10 000 voxels)
    "prob": ("tiny_prob", 3, {}, False),                                # 31 boxes above 2048 voxels
    "prob_fast": ("tiny_prob", 3, dict(scale_multiplier=6), True),      # per-axis radii: at 4 the largest box is 2040
}
VARIANTS = list(BASE_INPUTS)
D16 = dict(dims=(24, 12, 16), pc_min=(-6.0, -3.0, -4.0))        # one 16-deep z chunk per bin
RAGGED = dict(dims=(37, 21, 6), pc_min=(-9.0, -5.0, -1.5))      # D % 4 != 0: scalar tile path, no bin kernel


def _case(variant, over=None, seed=None, perturb=True, C=None):
    cfg, s, base_over, per_axis = BASE_INPUTS[variant]
    kw, inp, v = h.splat_case(cfg, s if seed is None else seed, perturb, {**base_over, **(over or {})},
                              per_axis=per_axis)
    assert v == variant
    if C is not None:
        G = inp["sem"].shape[1]
        inp = dict(inp, sem=torch.rand(1, G, C, generator=torch.Generator().manual_seed(C)))
    return kw, inp


def _clipped_box_volumes(kw, inp, variant):
    _, _, mi, radii, _, dims = h.oracle_prep(kw, inp, variant)
    r = radii.reshape(len(mi), -1)
    lo = np.maximum(mi - r, 0)
    hi = np.minimum(mi + r, np.asarray(dims) - 1)
    return np.prod(np.maximum(hi - lo + 1, 0), axis=1)


def _assert_big_box(kw, inp, variant):
    vol = _clipped_box_volumes(kw, inp, variant)
    assert (vol > K_BIG_BOX).any(), f"no clipped box above {K_BIG_BOX} voxels (largest {vol.max()}): " \
                                    "backward_big_kernel would have no queued work"


def _index(kw, x, y, z):
    return (x * kw["W"] + y) * kw["D"] + z


def _outputs(out):
    return (out,) if isinstance(out, torch.Tensor) else tuple(out)


def _upstream(outs, seed, offset=0):
    """Random upstream gradients (CPU) and their device copies; the logits gradient starts ``offset`` floats into
    its storage (offset 1: 4-byte aligned only)."""
    gen = torch.Generator().manual_seed(seed)
    g = [torch.randn(o.shape, generator=gen) for o in outs]
    dev = [x.cuda() for x in g]
    if offset:
        flat = torch.empty(g[0].numel() + offset, device="cuda")
        dev[0] = flat[offset:].view_as(g[0])
        dev[0].copy_(g[0])
        assert dev[0].data_ptr() % 16 == 4 * offset
    return g, dev


def _check_forward(outs, ref, variant, what, rtol=h.RTOL, atol=h.ATOL):
    lg = outs[0].detach().cpu().numpy()
    if variant == "base":
        h.assert_close(lg, ref["logits"], rtol, atol, what=f"{what} logits")
        return
    stable = np.abs(ref["probability"] - 1e-9) > 1e-10      # voxels on the fallback switch may take either branch
    h.assert_close(lg[stable], ref["logits"][stable], rtol, atol, what=f"{what} logits")
    h.assert_close(outs[1].detach().cpu().numpy(), ref["bin_logits"], rtol, atol, what=f"{what} bin_logits")
    h.assert_close(outs[2].detach().cpu().numpy(), ref["density"], rtol, atol, what=f"{what} density")


def _saved(outs, kw, inp, variant):
    """what the oracle's prob backward receives: the op's own forward outputs (probability: the fp32 oracle's)"""
    if variant == "base":
        return None
    return dict(logits=outs[0].detach().cpu().numpy(), bin_logits=outs[1].detach().cpu().numpy(),
                probability=h.oracle_forward(kw, inp, variant, "f32")["probability"])


def _check_vs_oracle(kw, inp, variant, what, offset=0, call=None, big_box=None, seed=7):
    """One batched call through the public module, forward and backward; every sample's outputs and four gradients
    against the oracle.  ``call(m, t)``: the entry point (default: forward on ``t["pts"]``); ``big_box``: the samples
    that must reach backward_big_kernel (default: all)."""
    m = h.make_module(kw, variant)
    t = h.to_dev(inp, requires_grad=True)
    call = call or (lambda m, t: m(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"]))
    outs = _outputs(call(m, t))
    g, dev = _upstream(outs, seed, offset)
    torch.autograd.backward(list(outs), dev)
    B = inp["means"].shape[0]
    for b in range(B):
        one = {k: v[b:b + 1] for k, v in inp.items()}
        if big_box is None or b in big_box:
            _assert_big_box(kw, one, variant)
        pick = (lambda x: x[b]) if B > 1 else (lambda x: x)
        mine = [pick(o) for o in outs]
        ref = h.oracle_forward(kw, one, variant)
        _check_forward(mine, ref, variant, f"{what} sample {b}")
        h.check_module_grads(t, kw, one, variant, tuple(pick(x).numpy() for x in g), what=f"{what} sample {b}",
                             saved_from=_saved(mine, kw, one, variant), sample=b)


# ------------------------------------------------------------------------------------------------ route matrix
ROUTES = {
    # name: (grid overrides, class count, point order, logits-gradient offset)
    "permuted": (None, None, "permuted", 0),             # in-place stray re-evaluation; bin kernel -> fallback
    "swapped_pair": (D16, None, "swapped_pair", 0),      # one stray pair at z >= 8 must send the call to the fallback
    "subset_dups": (None, None, "subset_dups", 0),       # N != H*W*D: render_points_kernel, Gaussian-centric backward
    "ragged": (RAGGED, None, "canonical", 0),            # D % 4 != 0: scalar tile path, Gaussian-centric backward
    "misaligned_grad": (None, None, "batch_of_2", 1),    # 4-byte aligned logits gradient: narrow row loads
    "permuted_C17": (None, 17, "permuted", 0),           # odd class count: narrow pair loop
    "subset_dups_C19": (None, 19, "subset_dups", 0),
}
POINTS_KERNEL = {"permuted": False, "swapped_pair": False, "subset_dups": True, "ragged": False,
                 "misaligned_grad": False, "permuted_C17": False, "subset_dups_C19": True}
BIN_KERNEL = {"permuted": True, "swapped_pair": True, "subset_dups": False, "ragged": False,
              "misaligned_grad": False, "permuted_C17": True, "subset_dups_C19": False}


def _route_inputs(variant, route):
    over, C, order, offset = ROUTES[route]
    kw, inp = _case(variant, over, C=C)
    pts = inp["pts"][0]
    N = pts.shape[0]
    gen = torch.Generator().manual_seed(17)
    if order == "permuted":
        idx = torch.randperm(N, generator=gen)
    elif order == "subset_dups":      # a random 60 % of the points + 40 of them again (two points in one voxel)
        sub = torch.randperm(N, generator=gen)[: N * 3 // 5]
        idx = torch.cat([sub, sub[:40]])
    elif order == "swapped_pair":     # both in the first bin, at z 9 and 14 of its 16 levels
        idx = torch.arange(N)
        a, b = _index(kw, 1, 2, 9), _index(kw, 6, 1, 14)
        idx[a], idx[b] = b, a
    elif order == "batch_of_2":
        # A single sample's outputs are squeezed views, and autograd hands the op a fresh (aligned) gradient for
        # them; the outputs of a batch are the op's own tensors, so a misaligned upstream gradient reaches the op.
        _, other = _case(variant, over, seed=BASE_INPUTS[variant][1] + 40, C=C)
        return kw, {k: torch.cat([inp[k], other[k]], 0) for k in inp}, offset
    else:
        idx = None
    if idx is not None:
        inp = dict(inp, pts=pts[idx][None].contiguous())
    return kw, inp, offset


@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("variant", VARIANTS)
def test_route_vs_oracle(variant, route):
    kw, inp, offset = _route_inputs(variant, route)
    _check_vs_oracle(kw, inp, variant, f"{variant}/{route}", offset=offset, big_box=(0,))


def _empty_supertile_inputs(variant):
    """N == H*W*D with one stray point: the point stored for voxel (16, 5, 9) lies in voxel (7, 8, 8), which then
    holds two points (the backward uses the larger index, like the oracle).  No Gaussian reaches x >= 16, so the bin
    that stores the stray point belongs to a 16-column supertile without any candidate Gaussian; its bin must still
    find the stray point."""
    cfg, seed, base_over, per_axis = BASE_INPUTS[variant]
    over = {**base_over, "dims": (48, 16, 16), "pc_min": (-12.0, -4.0, -4.0), "with_empty": False}
    kw, inp, _ = h.splat_case(cfg, seed, True, over, per_axis=per_axis)
    gs, pc, mult = kw["grid_size"], kw["pc_min"], kw["scale_multiplier"]
    means, scales, cov = inp["means"].clone(), inp["scales"].clone(), inp["cov"].clone()
    r_max = int(np.ceil(float(scales.max()) * mult / gs))
    x_vox = max(15 - r_max, 0)                 # mean voxels 0..x_vox along x: every box ends at x <= 15
    means[..., 0] = pc[0] + (means[..., 0] - pc[0]) / (kw["H"] * gs) * ((x_vox + 1) * gs)
    s = 7.6 * gs / mult                        # one Gaussian with radius 8 around voxel (7, 8, 8): box x 0..15, 4096 voxels
    means[0, 0] = torch.tensor([pc[0] + 7.5 * gs, pc[1] + 8.5 * gs, pc[2] + 8.5 * gs])
    scales[0, 0] = s
    cov[0, 0] = torch.eye(3) / (s * s)
    pts = inp["pts"].clone()
    pts[0, _index(kw, 16, 5, 9)] = pts[0, _index(kw, 7, 8, 8)]     # the centre voxel of the wide Gaussian
    inp = dict(inp, means=means, scales=scales, cov=cov, pts=pts)
    _, _, mi, radii, _, _ = h.oracle_prep(kw, inp, variant)
    assert (mi[:, 0] + radii.reshape(len(mi), -1)[:, 0]).max() <= 15
    return kw, inp


@pytest.mark.parametrize("variant", VARIANTS)
def test_stray_point_in_a_supertile_without_gaussians(variant):
    kw, inp = _empty_supertile_inputs(variant)
    _check_vs_oracle(kw, inp, variant, f"{variant}/empty supertile")


# ------------------------------------------------------------------------------------------------ batches, entry points
def _mixed_batch(variant):
    """sample 0 in canonical order (bin kernel), sample 1 permuted (Gaussian-centric fallback), other Gaussians"""
    kw, a = _case(variant, seed=BASE_INPUTS[variant][1] + 20)
    _, b = _case(variant)
    perm = torch.randperm(b["pts"].shape[1], generator=torch.Generator().manual_seed(5))
    b = dict(b, pts=b["pts"][:, perm].contiguous())
    return kw, {k: torch.cat([a[k], b[k]], 0) for k in a}


@pytest.mark.parametrize("variant", VARIANTS)
def test_mixed_batch_canonical_and_permuted(variant):
    kw, inp = _mixed_batch(variant)
    _check_vs_oracle(kw, inp, variant, f"{variant}/mixed batch", big_box=(1,))


def _grid_batch(variant):
    kw, a = _case(variant, perturb=False)
    _, b = _case(variant, perturb=False, seed=BASE_INPUTS[variant][1] + 30)
    return kw, {k: torch.cat([a[k], b[k]], 0) for k in a}


def _on_grid(m, t):
    assert torch.equal(m.grid_points(t["means"].device)[0], t["pts"][0])   # the oracle gets the same voxel centres
    return m.forward_on_grid(t["means"], t["opa"], t["sem"], t["scales"], t["cov"])


@pytest.mark.parametrize("variant", VARIANTS)
def test_forward_on_grid_batch_vs_oracle(variant):
    """pts_shared = 1: one [N,3] point array for both samples (the bin kernel's point tile row is then 0 + bin x)."""
    kw, inp = _grid_batch(variant)
    _check_vs_oracle(kw, inp, variant, f"{variant}/on grid", call=_on_grid, big_box=())


@pytest.mark.parametrize("variant", VARIANTS)
def test_forward_from_srt_generic_route(variant):
    """forward_from_srt on permuted points: the Gaussian-centric chain writes the gradient of Sigma^-1 (stride 6) and
    srt_grad_kernel maps it to scales and rotations.  Reference: the fp64 chain of tests/srt_oracle.py (Sigma^-1, the
    oracle and autograd through the closed form R^T diag(1/s^2) R in float64), with the gates of
    test_splat_srt_gpu.check_srt; under use_deterministic_algorithms the deterministic backward."""
    import test_splat_srt_gpu as srt
    kw, inp = _case(variant)
    G = inp["means"].shape[1]
    gen = torch.Generator().manual_seed(23)
    rots = torch.randn(1, G, 4, generator=gen) * 1.5
    perm = torch.randperm(inp["pts"].shape[1], generator=gen)
    inp = dict(inp, pts=inp["pts"][:, perm].contiguous())
    srt.check_srt(kw, inp, rots, variant, f"{variant}/srt", det=torch.are_deterministic_algorithms_enabled())


# ------------------------------------------------------------------------------------------------ permutation invariance
@pytest.mark.parametrize("variant", VARIANTS)
def test_permutation_invariance_full_grid(variant):
    """Full 200x200x16 grid, one point per voxel, no oracle: permuting the points and the upstream rows alike permutes
    the forward rows (stray points are re-evaluated by render_one_point, whose arithmetic differs from the tile
    kernel's column path: elementwise gate) and leaves every Gaussian gradient unchanged up to fp32 reordering.  The
    canonical call runs the bin kernel, the permuted one its Gaussian-centric fallback."""
    cfg, over = ("gs25600_solid", dict(G=1500)) if variant == "base" else ("prob_gs6400", dict(G=400))
    kw, inp, v = h.splat_case(cfg, 4, True, over, per_axis=variant == "prob_fast")
    assert v == variant
    m = h.make_module(kw, variant)
    N = inp["pts"].shape[1]
    perm = torch.randperm(N, generator=torch.Generator().manual_seed(8)).cuda()
    results = []
    for order in (None, perm):
        t = h.to_dev(inp, requires_grad=True)
        pts = t["pts"] if order is None else t["pts"][:, order].contiguous()
        outs = _outputs(m(pts, t["means"], t["opa"], t["sem"], t["scales"], t["cov"]))
        if order is None:
            g, dev = _upstream(outs, 3)
        torch.autograd.backward(list(outs), dev if order is None else [x[order] for x in dev])
        results.append(([o.detach() for o in outs], [t[k].grad[0].cpu().numpy() for k in ("means", "opa", "sem", "cov")]))
    (oc, gc), (op, gp) = results
    rows = [x[perm] for x in oc]
    keep = torch.ones(N, dtype=torch.bool, device="cuda")
    if variant != "base":    # rows on the probability switch (the uniform fallback row) may take either branch
        C = rows[0].shape[1]
        fallback = torch.full((C,), 1.0 / (C - 1), device="cuda")
        fallback[-1] = 0
        keep = ~((rows[0] == fallback).all(1) | (op[0] == fallback).all(1))
    h.assert_close(op[0][keep].cpu().numpy(), rows[0][keep].cpu().numpy(), what=f"{variant} permuted logits")
    for name, a, b in zip(("bin_logits", "density"), op[1:], rows[1:]):
        h.assert_close(a.cpu().numpy(), b.cpu().numpy(), what=f"{variant} permuted {name}")
    for name, a, b in zip(("means", "opa", "sem", "cov"), gp, gc):
        h.assert_close(a, b, rtol=1e-3, atol=h.grad_tolerance(b), what=f"{variant} permuted grad {name}")


# ------------------------------------------------------------------------------------------------ integer preparation
EDGE_GRIDS = {
    "gs0.5": dict(grid_size=0.5),
    "gs0.4": dict(grid_size=0.4),
    "gs0.4_ragged": dict(grid_size=0.4, **RAGGED),
}


def _faces(pc, gs, k):
    """fp32 lower face pc + k * gs of voxel k (the arithmetic of the voxel-centre grid)"""
    return (np.asarray(k).astype(np.float32) * np.float32(gs) + np.float32(pc)).astype(np.float32)


def _edge_inputs(variant, grid):
    """Voxel centres with a quarter of the coordinates moved onto their voxel's lower face and a quarter one ulp below
    it; points of voxel 0 moved into (pc_min - grid_size, pc_min); the means likewise on faces and one ulp below."""
    kw, inp = _case(variant, EDGE_GRIDS[grid], perturb=False)
    dims, gs, pc = (kw["H"], kw["W"], kw["D"]), kw["grid_size"], kw["pc_min"]
    rng = np.random.default_rng(11)
    pts = inp["pts"][0].numpy().copy()
    vox = np.stack(np.unravel_index(np.arange(len(pts)), dims), 1)
    means = inp["means"][0].numpy().copy()
    mvox = np.clip(((means - np.float32(pc)) / np.float32(gs)).astype(np.int32), 0, np.asarray(dims) - 1)
    for a in range(3):
        face = _faces(pc[a], gs, vox[:, a])
        kind = rng.integers(0, 4, len(pts))
        pts[:, a] = np.where(kind == 0, face, np.where(kind == 1, np.nextafter(face, np.float32(-np.inf)), pts[:, a]))
        low = (vox[:, a] == 0) & (kind == 2)
        pts[low, a] = np.float32(pc[a]) - rng.uniform(0.05, 0.95, int(low.sum())).astype(np.float32) * np.float32(gs)
        mface = _faces(pc[a], gs, mvox[:, a])
        mkind = rng.integers(0, 3, len(means))
        means[:, a] = np.where(mkind == 0, mface, np.where(mkind == 1, np.nextafter(mface, np.float32(-np.inf)),
                                                           means[:, a]))
    return kw, dict(inp, pts=torch.from_numpy(pts)[None], means=torch.from_numpy(means)[None])


def _reference_raises(kw, inp, variant):
    a = {k: v[0].numpy() for k, v in inp.items()}
    try:
        oracle.host_prep(a["pts"], a["means"], a["scales"], kw["pc_min"], kw["grid_size"], kw["scale_multiplier"],
                         radii_min=None if variant == "base" else 1, per_axis=variant == "prob_fast",
                         dims=(kw["H"], kw["W"], kw["D"]))
    except AssertionError:
        return True
    return False


def _op_raises(m, inp):
    t = h.to_dev(inp)
    try:
        m(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"])
    except AssertionError:
        return True
    return False


@pytest.mark.parametrize("grid", list(EDGE_GRIDS))
@pytest.mark.parametrize("variant", ["base", "prob"])
def test_points_and_means_on_voxel_faces(variant, grid):
    """The voxel index is the reference's fp32 truncation of (p - pc_min) / grid_size.  On faces a shortcut would
    disagree with it: with grid_size 0.4 some face coordinates truncate into the voxel below, so the points are
    N == H*W*D but not canonical (one voxel doubly occupied, its neighbour empty)."""
    kw, inp = _edge_inputs(variant, grid)
    assert not _reference_raises(kw, inp, variant)
    _check_vs_oracle(kw, inp, variant, f"{variant}/{grid} faces")
    # validate=True raises exactly where the reference's asserts fire: the grid's outer faces and one ulp off them
    kw, inp = _case(variant, EDGE_GRIDS[grid], perturb=False)
    dims, gs, pc = (kw["H"], kw["W"], kw["D"]), kw["grid_size"], kw["pc_min"]
    m = h.make_module(kw, variant)
    verdicts = []
    for a in range(3):
        upper = _faces(pc[a], gs, dims[a])
        outside = _faces(pc[a], gs, -1)
        for value in (upper, np.nextafter(upper, np.float32(-np.inf)), outside, np.nextafter(outside, np.float32(np.inf))):
            for key, row in (("pts", len(inp["pts"][0]) - 1), ("means", 1)):
                bad = dict(inp, **{key: inp[key].clone()})
                bad[key][0, row, a] = float(value)
                want = _reference_raises(kw, bad, variant)
                assert _op_raises(m, bad) == want, f"{key}[{row}, {a}] = {float(value)!r}: reference raises: {want}"
                verdicts.append(want)
    assert any(verdicts) and not all(verdicts)


# ------------------------------------------------------------------------------------------------ route check
def _kernel_names(run):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    return {e.name for e in prof.events()}


def _fwd_bwd(kw, inp, variant, offset=0):
    def run():
        m = h.make_module(kw, variant)
        t = h.to_dev(inp, requires_grad=True)
        outs = _outputs(m(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"]))
        torch.autograd.backward(list(outs), _upstream(outs, 1, offset)[1])
    return run


def test_cases_take_the_route_they_name():
    """The cases above cover their routes only while the kernel selection stays as it is (e.g. the bin kernel needs
    the driver's tensor-map encoder).  Kernel names recorded with torch.profiler (CUDA activity only)."""
    cases = []
    for variant in VARIANTS:
        for route in ROUTES:
            kw, inp, offset = _route_inputs(variant, route)
            cases.append((f"{variant}/{route}", _fwd_bwd(kw, inp, variant, offset), POINTS_KERNEL[route], BIN_KERNEL[route]))
        kw, inp = _empty_supertile_inputs(variant)
        cases.append((f"{variant}/empty supertile", _fwd_bwd(kw, inp, variant), False, True))
        kw, inp = _mixed_batch(variant)
        cases.append((f"{variant}/mixed batch", _fwd_bwd(kw, inp, variant), False, True))
    for variant in ("base", "prob"):
        kw, inp = _edge_inputs(variant, "gs0.4_ragged")
        cases.append((f"{variant}/faces ragged", _fwd_bwd(kw, inp, variant), False, False))
        kw, inp = _edge_inputs(variant, "gs0.4")
        cases.append((f"{variant}/faces", _fwd_bwd(kw, inp, variant), False, True))
    wrong = []
    for what, run, points_kernel, bin_kernel in cases:
        names = _kernel_names(run)
        assert any("render_" in n for n in names), \
            f"{what}: the profiler recorded no render kernel (recorded: {sorted(names)[:20]})"
        got = (any("render_points_kernel" in n for n in names), any("backward_bin_kernel" in n for n in names))
        if got != (points_kernel, bin_kernel):
            wrong.append(f"{what}: render_points_kernel {got[0]} (want {points_kernel}), "
                         f"backward_bin_kernel {got[1]} (want {bin_kernel})")
    assert not wrong, "\n".join(wrong)
