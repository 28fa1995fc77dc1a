"""The splat op's scales-and-rotations route (``forward_from_srt``) against the fp64 oracle of the whole chain
(tests/srt_oracle.py): Sigma^-1 built in the pack kernel and the backward's loaders, the [G,6] gradient of Sigma^-1 the
backward kernels write into the workspace, and srt_grad_kernel's map of it to dL/dscales and dL/drotations.

Every case calls the public ``forward_from_srt`` with all five leaves requiring grad and backpropagates random upstream
gradients.  Gates: helpers.assert_close for the outputs, helpers.assert_grad_parity for the five gradients (the fp32
chain supplies the floor; srt_oracle.check_grads).  Each case prints one ``[srt]`` report line: the worst output error as
a fraction of its tolerance, the gradient entries that took the floor rule and the share of dL/dscales an all-zero
answer would pass.

That share is below 1 % on every case but the flat and needle Gaussians at the prob scale range, where it reaches
30-90 %.  A floor measured per Gaussian row does not help there: the prob determinant of such a Sigma^-1 amplifies the
fp32 rounding of its entries, and the fp32 oracle fed the best fp32 Sigma^-1 there is (the fp64 one rounded once) already
misses a 4x per-row floor on up to 29 of 576 dL/dscales entries."""
import time

import numpy as np
import pytest
import torch

import helpers as h
import srt_oracle as so
import test_splat_routes_gpu as routes
from test_splat_deterministic_gpu import deterministic

pytestmark = pytest.mark.gpu

LEAVES = ("means", "opa", "sem", "scales", "rotations")
MODES = ["atomic", "deterministic"]


def _rotations(B, G, seed, scale=1.5):
    return torch.randn(B, G, 4, generator=torch.Generator().manual_seed(seed)) * scale


def _run(kw, inp, rots, variant, det=False, seed=29, scales=None, rotations=None):
    """forward_from_srt + autograd.  Returns (outputs on the CPU, CPU upstream gradients, leaf gradients on the CPU).
    ``scales`` / ``rotations``: device tensors to pass instead of fresh contiguous leaves (their gradients are then the
    caller's to read)."""
    m = h.make_module(kw, variant)
    t = h.to_dev(inp)
    leaves = {k: t[k].clone().requires_grad_(True) for k in ("means", "opa", "sem", "scales")}
    leaves["rotations"] = rots.cuda().requires_grad_(True)
    s = leaves["scales"] if scales is None else scales
    r = leaves["rotations"] if rotations is None else rotations
    with deterministic(det):
        outs = routes._outputs(m.forward_from_srt(t["pts"], leaves["means"], leaves["opa"], leaves["sem"], s, r))
        g, dev = routes._upstream(outs, seed)
        torch.autograd.backward(list(outs), dev)
    grads = {k: None if v.grad is None else v.grad.cpu() for k, v in leaves.items()}
    return [o.detach().cpu() for o in outs], g, grads


def check_srt(kw, inp, rots, variant, what, det=False, big_box=None):
    """One batched forward_from_srt call, every sample against its own fp64 chain.  ``big_box``: the samples that must
    hold a clipped box above kBigBox (default: all)."""
    outs, g, grads = _run(kw, inp, rots, variant, det)
    B = inp["means"].shape[0]
    reports = []
    for b in range(B):
        one = {k: v[b:b + 1] for k, v in inp.items()}
        if big_box is None or b in big_box:
            routes._assert_big_box(kw, one, variant)
        pick = (lambda x: x[b]) if B > 1 else (lambda x: x)
        mine = [pick(o).numpy() for o in outs]
        chains = so.srt_chains(kw, one, inp["scales"][b], rots[b], variant, tuple(pick(x).numpy() for x in g),
                               op_outputs=mine[:2])
        reports.append(so.check_sample(mine, {k: grads[k][b].numpy() for k in LEAVES}, chains, variant,
                                       f"{what} sample {b}"))
    return reports


# ------------------------------------------------------------------------------------------------ route matrix
ROUTES = ["canonical", "permuted", "swapped_pair", "subset_dups", "ragged", "permuted_C17"]


def _route_inputs(variant, route):
    """(kw, inp, samples that must reach the big-box queue): the inputs of test_splat_routes_gpu's route matrix"""
    if route == "canonical":              # tile kernel forward, bin kernel backward
        kw, inp = routes._case(variant)
        return kw, inp, ()
    kw, inp, _ = routes._route_inputs(variant, route)
    return kw, inp, (0,)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("variant", routes.VARIANTS)
def test_srt_route_vs_fp64_chain(variant, route, mode):
    kw, inp, big = _route_inputs(variant, route)
    rots = _rotations(1, inp["means"].shape[1], 23)
    check_srt(kw, inp, rots, variant, f"{variant}/{route}/{mode}", det=mode == "deterministic", big_box=big)


# ------------------------------------------------------------------------------------------------ batches
def _two_canonical(variant):
    """two canonical samples with different Gaussians: both take the bin kernel"""
    kw, a = routes._case(variant)
    _, b = routes._case(variant, seed=routes.BASE_INPUTS[variant][1] + 30)
    return kw, {k: torch.cat([a[k], b[k]], 0) for k in a}, ()


BATCHES = {
    "two_canonical": _two_canonical,
    "mixed": lambda variant: routes._mixed_batch(variant) + ((1,),),   # bin kernel + Gaussian-centric chain
}


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("batch", list(BATCHES))
@pytest.mark.parametrize("variant", routes.VARIANTS)
def test_srt_batch_vs_fp64_chain(variant, batch, mode):
    """B = 2 with different Gaussians and different quaternions per sample: srt_grad_kernel and the stride-6 writers
    must narrow the workspace and the quaternions to each sample"""
    kw, inp, big = BATCHES[batch](variant)
    rots = _rotations(2, inp["means"].shape[1], 31)
    assert not torch.equal(rots[0], rots[1])
    check_srt(kw, inp, rots, variant, f"{variant}/{batch}/{mode}", det=mode == "deterministic", big_box=big)


# ------------------------------------------------------------------------------------------------ quaternions
def _quaternion_zoo(G, seed):
    """The identity, axis-aligned 90 and 180 degree rotations (R with exact zeros), the same with w < 0 and with norms
    far from 1; the rest random directions with w < 0 in half of them and norms log-uniform in [1e-4, 1e4]."""
    gen = torch.Generator().manual_seed(seed)
    special = torch.tensor([
        [1, 0, 0, 0], [1, 1, 0, 0], [1, 0, 1, 0], [1, 0, 0, 1],           # identity, 90 degrees about x, y, z
        [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1],                          # 180 degrees about x, y, z
        [-1, 0, 0, 0], [-1, 1, 0, 0], [-1, 0, 0, 1], [0, 0, -1, 0],        # w < 0 / negated
        [1e-4, 0, 0, 0], [0, 0, 0, 1e4], [3e-3, 0, 3e-3, 0], [0, -2e3, 0, 0],
    ], dtype=torch.float32)
    q = torch.randn(G, 4, generator=gen)
    q = q / q.norm(dim=1, keepdim=True)
    q[:, 0] = torch.where(torch.rand(G, generator=gen) < 0.5, -q[:, 0].abs(), q[:, 0])
    q = q * torch.exp(torch.empty(G, 1).uniform_(np.log(1e-4), np.log(1e4), generator=gen))
    n = min(len(special), G)
    q[:n] = special[:n]
    return q


@pytest.mark.parametrize("route", ["canonical", "permuted"])
@pytest.mark.parametrize("variant", routes.VARIANTS)
def test_srt_quaternion_norms_and_axis_rotations(variant, route):
    kw, inp, big = _route_inputs(variant, route)
    rots = _quaternion_zoo(inp["means"].shape[1], 41)[None]
    norms = rots.norm(dim=-1)
    assert float(norms.min()) < 1e-3 and float(norms.max()) > 1e3 and (rots[..., 0] < 0).sum() > 10
    check_srt(kw, inp, rots, variant, f"{variant}/{route}/quaternion zoo", big_box=big)


@pytest.mark.parametrize("route", ["canonical", "permuted"])
@pytest.mark.parametrize("variant", routes.VARIANTS)
def test_srt_quaternion_sign_and_power_of_two_scale(variant, route):
    """Exact properties, in deterministic mode: -q gives the same outputs and the other gradients bit for bit and
    exactly the negated dL/dq; 2^k q (k per Gaussian in [-24, 24]) gives the same outputs and gradients and dL/dq scaled
    by exactly 2^-k, because the norm and its reciprocal scale exactly."""
    kw, inp, _ = _route_inputs(variant, route)
    G = inp["means"].shape[1]
    q = _rotations(1, G, 43)
    k = torch.randint(-24, 25, (1, G, 1), generator=torch.Generator().manual_seed(44)).float()
    runs = {name: _run(kw, inp, rq, variant, det=True) for name, rq in
            (("q", q), ("-q", -q), ("2^k q", q * torch.exp2(k)))}
    outs, _, grads = runs["q"]
    for name, (o, _, gr) in runs.items():
        for a, b in zip(o, outs):
            assert torch.equal(a, b), f"{variant}/{route} {name}: outputs differ"
        for leaf in ("means", "opa", "sem", "scales"):
            assert torch.equal(gr[leaf], grads[leaf]), f"{variant}/{route} {name}: grad {leaf} differs"
    assert float(grads["rotations"].abs().max()) > 0
    assert torch.equal(runs["-q"][2]["rotations"], -grads["rotations"]), f"{variant}/{route}: dL/d(-q) != -dL/dq"
    scaled = grads["rotations"].double() * torch.exp2(-k.double())
    assert torch.equal(runs["2^k q"][2]["rotations"].double(), scaled), f"{variant}/{route}: dL/d(2^k q) != 2^-k dL/dq"


# ------------------------------------------------------------------------------------------------ flat and needle
SHAPE_FAMILIES = {
    # name: (variant, config, seed, overrides, per-axis radii, bottom of the flat Gaussians)
    "tiny": ("base", "tiny", 0, dict(with_empty=True), False, 0.08),   # 0.08 - 0.64 + the whole-grid Gaussian
    "prob_range": ("prob", "tiny_prob", 3, dict(scale_range=(0.01, 3.2)), False, 0.1),    # prob_gs6400's range, x4
    "prob_range_per_axis": ("prob_fast", "tiny_prob", 3, dict(scale_range=(0.01, 3.2)), True, 0.1),
}


def _shaped_inputs(family, shape):
    """Every Gaussian (but the whole-grid one) flat -- two axes near the top of the config's scale range, one near its
    bottom -- or a needle -- one near the top, two near the bottom -- on randomly chosen axes; points permuted, so the
    Gaussian-centric chain runs and its big-box queue has work.

    The prob variants' flat Gaussians stop at a bottom of 0.1: the prob determinant det(Sigma^-1) = 1/(s0 s1 s2)^2 is
    evaluated in fp32 from entries up to 1/s_min^2 (by the reference op as by this one), and with s = (3.2, 3.2, 0.01)
    its cancellation leaves no correct digit -- the fp32 chain itself returns NaN gradients there.  Needles keep the
    full range: their determinant loses far less."""
    variant, cfg, seed, over, per_axis, flat_bottom = SHAPE_FAMILIES[family]
    kw, inp, v = h.splat_case(cfg, seed, True, over, per_axis=per_axis)
    assert v == variant
    lo, hi = over.get("scale_range", (0.08, 0.64))
    if shape == "flat":
        lo = flat_bottom
    G = inp["means"].shape[1] - (1 if over.get("with_empty") else 0)
    gen = torch.Generator().manual_seed(7)
    top = hi * (1 - 0.05 * torch.rand(G, 3, generator=gen))
    bottom = lo * (1 + 0.05 * torch.rand(G, 3, generator=gen))
    n_top = 2 if shape == "flat" else 1
    axes = torch.argsort(torch.rand(G, 3, generator=gen), dim=1) < n_top
    scales = inp["scales"].clone()
    scales[0, :G] = torch.where(axes, top, bottom)
    scales[0, 0] = top[0]       # one round Gaussian at the top of the range: per-axis needles alone hold no big box
    perm = torch.randperm(inp["pts"].shape[1], generator=gen)
    return kw, dict(inp, scales=scales, pts=inp["pts"][:, perm].contiguous()), variant


@pytest.mark.parametrize("shape", ["flat", "needle"])
@pytest.mark.parametrize("family", list(SHAPE_FAMILIES))
def test_srt_flat_and_needle_gaussians(family, shape):
    kw, inp, variant = _shaped_inputs(family, shape)
    rots = _rotations(1, inp["means"].shape[1], 47)
    check_srt(kw, inp, rots, variant, f"{family}/{shape}")


# ------------------------------------------------------------------------------------------------ full size
FULL = {
    # name: (config, seed, variant)
    "gs25600_solid": ("gs25600_solid", 0, "base"),    # with the whole-grid Gaussian, s = (100, 100, 8), q = (1, 0, 0, 0)
    "prob_gs6400": ("prob_gs6400", 0, "prob"),
}


@pytest.mark.parametrize("case", list(FULL))
def test_srt_full_size_vs_fp64_chain(case):
    cfg, seed, variant = FULL[case]
    kw, inp, v = h.splat_case(cfg, seed, False)
    assert v == variant
    G = inp["means"].shape[1]
    rots = _rotations(1, G, 53)
    if cfg == "gs25600_solid":
        assert inp["scales"][0, -1].tolist() == [100.0, 100.0, 8.0]
        rots[0, -1] = torch.tensor([1.0, 0.0, 0.0, 0.0])
    start = time.perf_counter()
    check_srt(kw, inp, rots, variant, f"full {case}", big_box=())
    print(f"[srt] full {case}: {time.perf_counter() - start:.1f} s")


# ------------------------------------------------------------------------------------------------ caller's layout
@pytest.mark.parametrize("variant", routes.VARIANTS)
def test_srt_scales_and_rotations_as_anchor_views(variant):
    """Scales and quaternions as non-contiguous column views of one [B, G, 28] anchor-like leaf, as a head slices them
    from its anchor: outputs and the gradient landing in the leaf equal the contiguous call bit for bit (deterministic
    mode), and the other columns of the leaf get none."""
    kw, inp = routes._mixed_batch(variant)
    B, G = inp["means"].shape[:2]
    rots = _rotations(B, G, 59)
    anchor = torch.randn(B, G, 28, generator=torch.Generator().manual_seed(60))
    anchor[..., 3:6] = inp["scales"]
    anchor[..., 6:10] = rots
    leaf = anchor.cuda().requires_grad_(True)
    s, r = leaf[..., 3:6], leaf[..., 6:10]
    assert not s.is_contiguous() and not r.is_contiguous()
    outs_v, _, grads_v = _run(kw, inp, rots, variant, det=True, scales=s, rotations=r)
    outs_c, _, grads_c = _run(kw, inp, rots, variant, det=True)
    for a, b in zip(outs_v, outs_c):
        assert torch.equal(a, b)
    for leaf_name in ("means", "opa", "sem"):
        assert torch.equal(grads_v[leaf_name], grads_c[leaf_name]), leaf_name
    g = leaf.grad.cpu()
    assert torch.equal(g[..., 3:6], grads_c["scales"]) and torch.equal(g[..., 6:10], grads_c["rotations"])
    assert float(g[..., 3:10].abs().max()) > 0
    assert not g[..., :3].any() and not g[..., 10:].any()


# ------------------------------------------------------------------------------------------------ route check
def test_srt_cases_take_the_route_they_name():
    """The route matrix above covers its kernels only while the kernel selection stays as it is: render_points_kernel
    for subset_dups, backward_bin_kernel for the canonical and the N == H*W*D routes, and srt_grad_kernel on all.
    Kernel names recorded with torch.profiler (CUDA activity only)."""
    points_kernel = dict(routes.POINTS_KERNEL, canonical=False, mixed=False)
    bin_kernel = dict(routes.BIN_KERNEL, canonical=True, mixed=True)
    wrong = []
    for variant in routes.VARIANTS:
        cases = [(route,) + _route_inputs(variant, route)[:2] for route in ROUTES]
        kw, inp, _ = BATCHES["mixed"](variant)
        cases.append(("mixed", kw, inp))
        for route, kw, inp in cases:
            rots = _rotations(inp["means"].shape[0], inp["means"].shape[1], 23)
            names = routes._kernel_names(lambda: _run(kw, inp, rots, variant))
            got = (any("render_points_kernel" in n for n in names), any("backward_bin_kernel" in n for n in names),
                   any("srt_grad_kernel" in n for n in names))
            want = (points_kernel[route], bin_kernel[route], True)
            if got != want:
                wrong.append(f"{variant}/{route}: render_points_kernel, backward_bin_kernel, srt_grad_kernel: {got}, "
                             f"want {want}")
    assert not wrong, "\n".join(wrong)
