"""The render tile kernel writes the [N, C] logits of a CTA through a shared-memory tile and bulk copies when the
logits tensor is 16-byte aligned, D is a multiple of the 16-voxel z chunk and no point of the CTA is stray; otherwise it
stores them directly.  Both routes must write the same bytes: every case renders the same inputs once into an aligned
logits tensor (bulk copies wherever they apply) and once into a view that starts 4 bytes into its storage (direct
stores everywhere), and compares the results byte for byte.  Outputs start as NaN, so a row neither route writes
fails as well."""
import ctypes

import pytest
import torch

import helpers as h
from gaussianformer_b200 import _lib
from gaussianformer_b200.splat import _forward_ws_bytes, _make_desc, _ptr

pytestmark = pytest.mark.gpu


def _render(desc, t, misalign):
    """One gf_splat_forward call; the logits go to a [B, N, C] view ``misalign`` floats into its storage."""
    B, N, C = desc.batch, desc.N, desc.C
    flat = torch.full((B * N * C + misalign,), float("nan"), device="cuda")
    logits = flat[misalign:].view(B, N, C)
    assert (logits.data_ptr() % 16 == 0) == (misalign == 0)
    extra = [torch.full((B, N), float("nan"), device="cuda") for _ in range(3)] \
        if desc.variant == _lib.GF_SPLAT_PROB else [None] * 3
    ws_bytes = _forward_ws_bytes(desc)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    ins = _lib.SplatInputs(_ptr(t["pts"]), None, _ptr(t["means"]), None, _ptr(t["opa"]), _ptr(t["sem"]),
                           _ptr(t["cov"]), None, _ptr(t["scales"]))
    outs = _lib.SplatOutputs(_ptr(logits), *(_ptr(e) for e in extra))
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(_lib.lib().gf_splat_forward(ctypes.byref(desc), ctypes.byref(ins), ctypes.byref(outs), _ptr(ws),
                                           ws_bytes, stream))
    torch.cuda.synchronize()
    return [logits.clone()] + [e for e in extra if e is not None]


def _case(cfg, dims, B, variant="base", stray=False):
    over = dict(dims=dims, pc_min=(-0.25 * dims[0], -0.25 * dims[1], -0.25 * dims[2]))
    samples = [h.splat_case(cfg, seed, False, over)[:2] for seed in range(B)]
    kw = samples[0][0]
    t = {k: torch.cat([inp[k] for _, inp in samples], 0).cuda().contiguous() for k in samples[0][1]}
    G, N, C = t["means"].shape[1], t["pts"].shape[1], t["sem"].shape[2]
    assert N == kw["H"] * kw["W"] * kw["D"]
    if stray:   # swap two points of sample B-1 that lie in different bins: both leave canonical voxel order
        a, b = 5, (9 * kw["W"] + 6) * kw["D"] + 3
        t["pts"][B - 1, [a, b]] = t["pts"][B - 1, [b, a]].clone()
    t["cov"] = t["cov"].reshape(B, G, 9).contiguous()
    prob = variant == "prob"
    desc = _make_desc(G, N, C, kw["H"], kw["W"], kw["D"], _lib.GF_SPLAT_PROB if prob else _lib.GF_SPLAT_BASE, 1, 9,
                      kw["pc_min"], kw["grid_size"], float(kw["scale_multiplier"]), 1 if prob else 0, B, 0)
    return desc, t


CASES = {
    "b3_d16": ("tiny", (24, 12, 16), 3, "base", False),
    "d32": ("tiny", (16, 8, 32), 1, "base", False),
    "hw_ragged": ("tiny", (21, 10, 16), 2, "base", False),   # H % 8 != 0 and W % 4 != 0: partial bins at both edges
    "stray": ("tiny", (24, 12, 16), 2, "base", True),
    "prob_d16": ("tiny_prob", (24, 12, 16), 2, "prob", False),
}


@pytest.mark.parametrize("name", list(CASES))
def test_bulk_store_matches_direct_stores(name):
    desc, t = _case(*CASES[name])
    bulk = _render(desc, t, 0)
    direct = _render(desc, t, 1)
    for i, (x, y) in enumerate(zip(bulk, direct)):
        assert not torch.isnan(x).any(), f"{name}: output {i} has rows no route wrote"
        assert torch.equal(x.view(torch.int32), y.view(torch.int32)), f"{name}: output {i} differs between the routes"
