"""The splat op on grids deeper than one 16-level z chunk, against the fp64 oracle, for all three variants.

The render kernel and the bin-centric backward cut every column into z chunks of kBinZ = 16 levels (launch grid
(nzc, nby, nbx * B), nzc = ceil(D / 16)).  With D <= 16 the z chunk of a bin is always 0: the z term of the
deterministic slot index (rz), the z coordinate of the TMA tile loads, the zero fill of a partial last chunk and the
per-chunk row counts of the slot finish never leave their first value.  Here every grid has two or three chunks and a
small H x W, so that the fp64 oracle stays cheap:

  D32          two full chunks; the base record's z-level mask uses all 32 bits
  D20          the second chunk has 4 levels: the tile loads run past D and are zero-filled
  D24          the second chunk is half empty
  D48          three chunks, no z-level mask in the record, and one Gaussian whose box spans all three; the base
               variant's whole-grid Gaussian covers 8 x 6 x 3 = 144 bins, more than kWarpSlots = 128, so the CTA-wide
               slot finish sums its rows of every chunk
  D36_ragged   H % 8 != 0 and W % 4 != 0 as well: ragged bins in all three axes

Every case is one batched forward and backward through the public module; every sample's outputs and four gradients
pass helpers.assert_close / helpers.check_module_grads (test_splat_routes_gpu._check_vs_oracle).  The inputs are
guarded: boxes that straddle a chunk boundary, a box over three chunks on D48, the whole-grid Gaussian's slot rows above
128, and a clipped box above kBigBox voxels wherever the Gaussian-centric chain runs."""
import numpy as np
import pytest
import torch

import helpers as h
import test_splat_deterministic_gpu as det
import test_splat_routes_gpu as routes
from gaussianformer_b200 import _lib

pytestmark = pytest.mark.gpu

BIN = (8, 4, 16)     # common.cuh kBinX, kBinY, kBinZ
K_WARP_SLOTS = 128   # splat_backward_bin.cu kWarpSlots: a Gaussian with more slot rows is summed by the whole CTA

# pc_min centres the grid on the origin: the whole-grid Gaussian of the base inputs (mean (0, 0, -1)) lies inside it
GRIDS = {
    "D32": dict(dims=(16, 12, 32), pc_min=(-4.0, -3.0, -8.0)),
    "D20": dict(dims=(16, 12, 20), pc_min=(-4.0, -3.0, -5.0)),
    "D24": dict(dims=(16, 12, 24), pc_min=(-4.0, -3.0, -6.0)),
    "D48": dict(dims=(64, 24, 48), pc_min=(-16.0, -6.0, -12.0)),
    "D36_ragged": dict(dims=(21, 10, 36), pc_min=(-5.25, -2.5, -9.0)),
}
# both points of the swapped pair in z chunk 1 or later, in different bins
STRAY_PAIRS = {"D20": ((1, 2, 16), (9, 5, 19)), "D48": ((1, 2, 17), (10, 5, 40))}

CASES = {
    # name: (grid, point order, batch, class count, deterministic, slot budget)
    **{f"canonical_{g}": (g, "canonical", 1, None, False, None) for g in GRIDS},        # bin kernel, atomics
    **{f"det_{g}": (g, "canonical", 1, None, True, None) for g in GRIDS},               # bin kernel, slot rows
    **{f"overflow_{g}": (g, "canonical", 1, None, True, 1) for g in ("D20", "D48")},    # slot overflow -> fallback
    **{f"stray_{g}": (g, "stray_pair", 1, None, False, None) for g in STRAY_PAIRS},     # bin kernel hands over
    **{f"stray_det_{g}": (g, "stray_pair", 1, None, True, None) for g in STRAY_PAIRS},
    **{f"subset_dups_{g}": (g, "subset_dups", 1, None, False, None) for g in ("D48", "D36_ragged")},
    "b2_D36_ragged": ("D36_ragged", "canonical", 2, None, False, None),                # B * H tensor-map rows
    "b2_det_D36_ragged": ("D36_ragged", "canonical", 2, None, True, None),
    "b2_shared_D24": ("D24", "shared", 2, None, False, None),                          # one [N, 3] point array
    "b2_shared_det_D48": ("D48", "shared", 2, None, True, None),
    "C17_D32": ("D32", "canonical", 1, 17, False, None),                               # odd C: narrow row loads
    "C19_D32_permuted": ("D32", "permuted", 1, 19, False, None),                       # odd C, Gaussian-centric
}
WANT_WORD = {"canonical": _lib.GF_DEBUG_ROUTE_BIN, "shared": _lib.GF_DEBUG_ROUTE_BIN,
             "stray_pair": _lib.GF_DEBUG_ROUTE_STRAY_POINTS, "permuted": _lib.GF_DEBUG_ROUTE_STRAY_POINTS,
             "subset_dups": _lib.GF_DEBUG_ROUTE_GAUSSIAN}


def _with_tall_gaussian(kw, inp):
    """Gaussian 0 becomes an isotropic one of radius 10 voxels centred on z level 24: its box spans levels 14..34,
    three z chunks, without covering the whole grid."""
    gs, pc, mult = kw["grid_size"], kw["pc_min"], kw["scale_multiplier"]
    means, scales, cov = inp["means"].clone(), inp["scales"].clone(), inp["cov"].clone()
    s = 9.5 * gs / mult
    means[0, 0] = torch.tensor([pc[0] + (kw["H"] // 2 + 0.5) * gs, pc[1] + (kw["W"] // 2 + 0.5) * gs, pc[2] + 24.5 * gs])
    scales[0, 0] = s
    cov[0, 0] = torch.eye(3) / (s * s)
    return dict(inp, means=means, scales=scales, cov=cov)


def _grid_inputs(variant, grid, order, seed=None, C=None):
    kw, inp = routes._case(variant, GRIDS[grid], seed=seed, perturb=order != "shared", C=C)
    assert (kw["H"], kw["W"], kw["D"]) == GRIDS[grid]["dims"]
    if grid == "D48":
        inp = _with_tall_gaussian(kw, inp)
    pts = inp["pts"][0]
    N = pts.shape[0]
    gen = torch.Generator().manual_seed(17)
    idx = None
    if order == "stray_pair":
        a, b = (routes._index(kw, *v) for v in STRAY_PAIRS[grid])
        idx = torch.arange(N)
        idx[a], idx[b] = b, a
    elif order == "subset_dups":      # a random 60 % of the points + 40 of them again (two points in one voxel)
        sub = torch.randperm(N, generator=gen)[: N * 3 // 5]
        idx = torch.cat([sub, sub[:40]])
    elif order == "permuted":
        idx = torch.randperm(N, generator=gen)
    if idx is not None:
        inp = dict(inp, pts=pts[idx][None].contiguous())
    return kw, inp


def _inputs(variant, case):
    """(kw, inputs with the batch dimension, entry point for _check_vs_oracle)"""
    grid, order, B, C, _, _ = CASES[case]
    base_seed = routes.BASE_INPUTS[variant][1]
    parts = [_grid_inputs(variant, grid, order, seed=base_seed + 70 * b, C=C) for b in range(B)]
    kw = parts[0][0]
    inp = {k: torch.cat([p[1][k] for p in parts], 0) for k in parts[0][1]}
    return kw, inp, routes._on_grid if order == "shared" else None


def _clipped_boxes(kw, one, variant):
    """[G, 3] first and last voxel of every Gaussian's box clipped to the grid"""
    _, _, mi, radii, _, dims = h.oracle_prep(kw, one, variant)
    r = radii.reshape(len(mi), -1)
    return np.maximum(mi - r, 0), np.minimum(mi + r, np.asarray(dims) - 1)


def _assert_guards(kw, inp, variant, grid):
    """The inputs reach what this file is about: boxes over chunk boundaries (one that does not span the whole depth),
    three chunks on D48, and on the base variant's D48 grid more than kWarpSlots slot rows for one Gaussian."""
    D = kw["D"]
    for b in range(inp["means"].shape[0]):
        lo, hi = _clipped_boxes(kw, {k: v[b:b + 1] for k, v in inp.items()}, variant)
        chunks = hi[:, 2] // BIN[2] - lo[:, 2] // BIN[2] + 1
        partial = (lo[:, 2] > 0) | (hi[:, 2] < D - 1)
        assert (chunks[partial] >= 2).any(), f"{grid} sample {b}: no box straddles a z-chunk boundary"
        if grid == "D48":
            assert (chunks[partial] >= 3).any(), f"{grid} sample {b}: no box covers three z chunks"
            if variant == "base":
                rows = np.prod(hi // BIN - lo // BIN + 1, axis=1)
                assert rows.max() > K_WARP_SLOTS, f"{grid} sample {b}: most slot rows {rows.max()}"


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("variant", routes.VARIANTS)
def test_deep_grid_vs_oracle(variant, case):
    grid, order, B, _, deterministic, budget = CASES[case]
    kw, inp, call = _inputs(variant, case)
    _assert_guards(kw, inp, variant, grid)
    # the Gaussian-centric chain must have work for backward_big_kernel wherever it produces the gradients
    fallback = order not in ("canonical", "shared") or budget is not None
    with det.plan(slot_budget=-1 if budget is None else budget), det.deterministic(deterministic):
        routes._check_vs_oracle(kw, inp, variant, f"{variant}/{case}", call=call, big_box=None if fallback else ())
        if deterministic:
            det._repeatable(kw, inp, variant, f"{variant}/{case}", call=call)
            want = _lib.GF_DEBUG_ROUTE_SLOT_OVERFLOW if budget is not None else WANT_WORD[order]
            pts = inp["pts"][0] if order == "shared" else inp["pts"]
            assert det._route_words(kw, dict(inp, pts=pts), variant) == [want] * B


# ------------------------------------------------------------------------------------------------ forward
@pytest.mark.parametrize("grid", ["D32", "D48"])
@pytest.mark.parametrize("variant", routes.VARIANTS)
def test_forward_on_voxel_centres_vs_oracle(variant, grid):
    """Unperturbed voxel centres: the render kernel's column form (base: with the record's z-level mask up to 32
    levels) and, for the base variant, the bulk write-out of whole z chunks from an aligned logits tensor."""
    kw, inp = routes._case(variant, GRIDS[grid], perturb=False)
    m = h.make_module(kw, variant)
    t = h.to_dev(inp)
    outs = routes._outputs(m(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"]))
    assert outs[0].data_ptr() % 16 == 0
    routes._check_forward(outs, h.oracle_forward(kw, inp, variant), variant, f"{variant}/{grid} voxel centres")


@pytest.mark.parametrize("grid", ["D32", "D36_ragged"])
def test_fused_argmax_and_class_major_logits(grid):
    """forward_eval on a deep grid: the [C, N] logits are the [N, C] logits transposed, bit for bit, the fused arg-max
    is their lowest-index maximiser, and both agree with the oracle."""
    kw, inp = routes._case("base", GRIDS[grid], perturb=False)
    m = h.make_module(kw, "base")
    t = h.to_dev(inp)
    args = (t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"])
    nc = m.forward_eval(*args, layout="nc")
    cn = m.forward_eval(*args, layout="cn")
    logits = nc["logits"][0]
    assert torch.equal(cn["pred_occ"][0], logits.t())
    assert torch.equal(cn["final_occ"], nc["final_occ"])
    first = (logits == logits.max(dim=1, keepdim=True).values).float().argmax(dim=1)
    assert torch.equal(nc["final_occ"][0].long(), first)
    ref = h.oracle_forward(kw, inp, "base")["logits"]
    h.assert_close(logits.cpu().numpy(), ref, what=f"{grid} logits")
    h.assert_argmax_parity(logits.cpu().numpy(), ref)


# ------------------------------------------------------------------------------------------------ route check
def test_cases_take_the_route_they_name():
    """Every case above runs the kernels it is named for: the bin-centric kernel (backward_bin_kernel, or
    backward_bin_slots_kernel under the deterministic switch) whenever N == H*W*D, render_points_kernel otherwise.
    Kernel names recorded with torch.profiler (CUDA activity only)."""
    wrong = []
    for variant in routes.VARIANTS:
        for case, (grid, order, B, C, deterministic, budget) in CASES.items():
            kw, inp, call = _inputs(variant, case)
            call = call or (lambda m, t: m(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"]))

            def run():
                m = h.make_module(kw, variant)
                t = h.to_dev(inp, requires_grad=True)
                outs = routes._outputs(call(m, t))
                torch.autograd.backward(list(outs), routes._upstream(outs, 1)[1])

            with det.plan(slot_budget=-1 if budget is None else budget), det.deterministic(deterministic):
                for _ in range(3):   # a capture now and then lacks the forward's kernels: take it again
                    names = routes._kernel_names(run)
                    if any("render_" in n for n in names):
                        break
            points = order == "subset_dups"
            want = {"render_tile_kernel": not points, "render_points_kernel": points,
                    "backward_bin_kernel": not points and not deterministic,
                    "backward_bin_slots_kernel": not points and deterministic}
            got = {k: any(k in n for n in names) for k in want}
            if got != want:
                wrong.append(f"{variant}/{case}: ran {got}, want {want}")
    assert not wrong, "\n".join(wrong)
