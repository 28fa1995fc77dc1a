"""fp16 / bf16 feature tables in the deformable-aggregation op: the format kernel moves half maps bit-exactly, the
sampling kernels give bit-identical outputs to the fp32 route on the upcast table, and the table's gradient is the
fp32 gradient rounded once to the table's dtype.  The last test runs without a GPU: the C ABI rejects an unknown
table dtype before it touches the CUDA runtime."""
import ctypes

import numpy as np
import pytest
import torch

import helpers as h
import oracle
from gaussianformer_b200 import _lib
from gaussianformer_b200.ops import DeformableAggregationFunction as DAF
from gaussianformer_b200.ops import deformable_aggregation_fused, fused_supported
from gaussianformer_b200.synthetic import make_daf_fused_inputs, make_daf_inputs

gpu = pytest.mark.gpu
DTYPES = [torch.float16, torch.bfloat16]
_MANT_EMIN = {torch.float16: (10, -14), torch.bfloat16: (7, -126)}   # stored mantissa bits, least normal exponent


def _ulp(x, dtype):
    """Spacing of `dtype` at |x| (subnormal spacing below the normal range)."""
    mant, emin = _MANT_EMIN[dtype]
    a = np.abs(np.asarray(x, np.float64))
    e = np.floor(np.log2(np.where(a > 0, a, 1.0)))
    e = np.maximum(np.where(a > 0, e, emin), emin)
    return np.exp2(e - mant)


def assert_half_grad(mine, ref64, ref32, dtype, what):
    """The fp32 gradient gate (helpers.assert_grad_parity) widened by one ulp of the table's dtype: the fp32 sum is
    rounded to that dtype once."""
    assert mine.dtype == dtype, f"{what}: dtype {mine.dtype}, want {dtype}"
    mine = mine.float().cpu().numpy().astype(np.float64)
    ref64 = np.asarray(ref64, np.float64)
    floor = float(np.abs(np.asarray(ref32, np.float64) - ref64).max())
    tol = np.maximum(h.ATOL + h.RTOL * np.abs(ref64), h.K_FLOOR * floor) + _ulp(ref64, dtype)
    bad, _, i = h.outside_tolerance(mine, ref64, tol)
    if bad.any():
        raise AssertionError(f"{what}: {int(bad.sum())}/{bad.size} outside the fp32 gate + 1 ulp; worst at {i}: "
                             f"got {mine[i]!r} want {ref64[i]!r}")


@gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("channels,levels", [
    (128, ((108, 200), (54, 100), (27, 50), (14, 25))),    # BASELINE config-2 maps (1 sample x 6 cameras)
    (24, ((5, 7), (3, 3), (1, 1))),                         # ragged: nothing divides the tile or vector sizes
    (130, ((9, 13),)),
])
def test_half_feature_maps_format_is_the_reference_layout(dtype, channels, levels):
    gen = torch.Generator().manual_seed(5)
    bs, cams = (1, 6) if channels == 128 else (2, 3)
    maps = [torch.randn(bs, cams, channels, h_, w_, generator=gen).to(dtype).cuda().requires_grad_(True)
            for h_, w_ in levels]
    col, shape, start = DAF.feature_maps_format(maps)
    assert col.dtype == dtype and col.is_contiguous()
    assert col.shape == (bs, cams, sum(h_ * w_ for h_, w_ in levels), channels)
    ref_col = torch.cat([m.detach().reshape(bs, cams, channels, -1) for m in maps], dim=-1).permute(0, 1, 3, 2)
    assert torch.equal(col.detach(), ref_col)
    g = torch.randn(col.shape, generator=gen).to(dtype).cuda()
    col.backward(g)
    back = DAF.feature_maps_format([g, shape, start], inverse=True)
    for m, b in zip(maps, back):
        assert m.grad.dtype == dtype and torch.equal(m.grad, b.contiguous())


@gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("embed,groups,levels,cams", [
    (128, 4, ((12, 20), (6, 10), (3, 5)), 3),     # fast kernel
    (256, 8, ((9, 7), (5, 4)), 3),                # two channel slices per warp
    (16, 4, ((7, 12), (4, 6), (2, 3)), 3),        # general kernel
    (24, 3, ((5, 5),), 3),
    (128, 4, ((10, 16), (8, 12), (6, 9), (4, 6), (3, 4), (2, 2)), 6),   # 36 (camera, level) pairs: general kernel
    (128, 64, ((12, 20), (6, 10), (3, 5)), 3),    # 2 channels per group: general kernel
])
def test_half_daf_forward_backward_vs_oracle(dtype, embed, groups, levels, cams):
    fms, loc, w = make_daf_inputs(num_anchor=64, num_pts=5, batch=2, num_cams=cams, embed_dims=embed,
                                  num_groups=groups, levels=levels, visible_p=0.5, seed=3)
    loc[0, 0, 0] = torch.tensor([0.0, 0.5]); loc[0, 1, 0] = torch.tensor([1.0, 0.5])
    loc[0, 2, 0] = torch.tensor([0.004, 0.996]); loc[0, 3, 1] = torch.tensor([0.999, 0.001])
    loc[1, 2, 2] = torch.tensor([0.5, 0.0]); loc[1, 4, 2] = torch.tensor([float("nan"), 0.5])
    table, shape, start = DAF.feature_maps_format([f.to(dtype).cuda() for f in fms])
    assert table.dtype == dtype
    table = table.detach().requires_grad_()
    loc_d, w_d = loc.cuda().requires_grad_(), w.cuda().requires_grad_()
    out = DAF.apply(table, shape, start, loc_d, w_d)
    assert out.dtype == torch.float32
    assert torch.equal(out.detach(), DAF.apply(table.detach().float(), shape, start, loc.cuda(), w.cuda()))
    f_np, s_np, st_np = table.detach().float().cpu().numpy(), shape.cpu().numpy(), start.cpu().numpy()
    h.assert_close(out.detach().cpu().numpy(), oracle.daf_forward(f_np, s_np, st_np, loc.numpy(), w.numpy(), "f64"),
                   what="half daf out")
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(11))
    out.backward(g.cuda())
    rf, rl, rw = oracle.daf_backward(f_np, s_np, st_np, loc.numpy(), w.numpy(), g.numpy(), "f64")
    rf32, rl32, rw32 = oracle.daf_backward(f_np, s_np, st_np, loc.numpy(), w.numpy(), g.numpy(), "f32")
    assert_half_grad(table.grad, rf, rf32, dtype, "half grad feat")
    h.assert_grad_parity(w_d.grad.cpu().numpy(), rw, rw32, what="half grad weights")
    h.assert_grad_parity(loc_d.grad.cpu().numpy(), rl, rl32, what="half grad loc")


@gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("embed,groups,levels,masks", [
    (128, 4, ((12, 20), (6, 10), (3, 5)), "both"),
    (128, 4, ((12, 20), (6, 10), (3, 5)), "point"),
    (128, 4, ((12, 20), (6, 10), (3, 5)), "none"),
    (256, 8, ((9, 7), (5, 4)), "both"),
    (128, 1, ((5, 5),), "point"),
])
def test_half_daf_fused_forward_backward_vs_oracle(dtype, embed, groups, levels, masks):
    B, A, K, M = 2, 40, 5, 3
    fms, loc, logits, pm, wm = make_daf_fused_inputs(num_anchor=A, num_pts=K, batch=B, num_cams=M, embed_dims=embed,
                                                     num_groups=groups, levels=levels, visible_p=0.5, seed=21,
                                                     attn_drop=0.15)
    loc[0, 2, 0] = torch.tensor([0.004, 0.996]); loc[0, 3, 1] = torch.tensor([0.999, 0.001])
    loc[1, 4, 2] = torch.tensor([float("nan"), 0.5])
    pm = ((loc > 0) & (loc < 1)).all(-1).reshape(B, A, K, M).contiguous()
    pm[0, 0] = False                                     # an anchor no camera sees
    wm[0, 1, :, :, :, 0] = False                         # a group with every entry dropped
    logits[1, 2, 0, 0, 0, 0] = 30.0                      # a dominant entry
    if masks == "point":
        wm = None
    elif masks == "none":
        pm = wm = None
    assert fused_supported(embed, groups, M, len(levels))
    pm_d = None if pm is None else pm.cuda()
    wm_d = None if wm is None else wm.cuda()
    table, shape, start = DAF.feature_maps_format([f.to(dtype).cuda() for f in fms])
    table = table.detach().requires_grad_()
    loc_d, lg_d = loc.cuda().requires_grad_(), logits.cuda().requires_grad_()
    out = deformable_aggregation_fused(table, shape, start, loc_d, lg_d, pm_d, wm_d)
    assert out.dtype == torch.float32
    assert torch.equal(out.detach(), deformable_aggregation_fused(table.detach().float(), shape, start, loc.cuda(),
                                                                  logits.cuda(), pm_d, wm_d))
    f_np, s_np, st_np = table.detach().float().cpu().numpy(), shape.cpu().numpy(), start.cpu().numpy()
    pm_np = None if pm is None else pm.numpy()
    wm_np = None if wm is None else wm.numpy()
    ref = oracle.daf_fused_forward(f_np, s_np, st_np, loc.numpy(), logits.numpy(), pm_np, wm_np, "f64")
    h.assert_close(out.detach().cpu().numpy(), ref, what="half fused daf out")
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(5))
    out.backward(g.cuda())
    rf, rl, rw = oracle.daf_fused_backward(f_np, s_np, st_np, loc.numpy(), logits.numpy(), g.numpy(), pm_np, wm_np, "f64")
    rf32, rl32, rw32 = oracle.daf_fused_backward(f_np, s_np, st_np, loc.numpy(), logits.numpy(), g.numpy(), pm_np, wm_np,
                                                 "f32")
    assert_half_grad(table.grad, rf, rf32, dtype, "half fused grad feat")
    h.assert_grad_parity(lg_d.grad.cpu().numpy(), rw, rw32, what="half fused grad logits")
    h.assert_grad_parity(loc_d.grad.cpu().numpy(), rl, rl32, what="half fused grad loc")


@gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_half_full_size_forward_equals_the_fp32_route(dtype):
    """BASELINE config-2 shape (25 600 anchors x 9 key points, 6 cameras, 4 levels, C = 128), both ops."""
    fms, loc, w = make_daf_inputs(seed=0)
    table, shape, start = DAF.feature_maps_format([f.to(dtype).cuda() for f in fms])
    assert table.dtype == dtype
    loc_d, w_d = loc.cuda(), w.cuda()
    assert torch.equal(DAF.apply(table, shape, start, loc_d, w_d), DAF.apply(table.float(), shape, start, loc_d, w_d))
    fms, loc, logits, pm, _ = make_daf_fused_inputs(seed=0)
    table, shape, start = DAF.feature_maps_format([f.to(dtype).cuda() for f in fms])
    loc_d, lg_d, pm_d = loc.cuda(), logits.cuda(), pm.cuda()
    assert torch.equal(deformable_aggregation_fused(table, shape, start, loc_d, lg_d, pm_d),
                       deformable_aggregation_fused(table.float(), shape, start, loc_d, lg_d, pm_d))


@gpu
def test_autocast_route_samples_the_half_maps():
    """Under autocast the FPN hands fp16 maps to the op.  The table stays fp16 through feature_maps_format and the op
    (the op saves it, not an fp32 copy); outputs equal the reference's route (cat/permute + .float()) bit for bit and
    the upstream parameters get the same gradients."""
    B, M, Cin, C = 2, 3, 32, 128
    levels = ((12, 20), (6, 10), (3, 5))
    gen = torch.Generator().manual_seed(7)
    xs = [torch.randn(B * M, Cin, h_, w_, generator=gen).cuda() for h_, w_ in levels]
    conv = torch.nn.Conv2d(Cin, C, 1).cuda()
    _, loc, w = make_daf_inputs(num_anchor=64, num_pts=5, batch=B, num_cams=M, embed_dims=C, num_groups=4,
                                levels=levels, visible_p=0.5, seed=8)
    loc, w = loc.cuda(), w.cuda()
    g = torch.randn(B, loc.shape[1], C, generator=gen).cuda()
    with torch.autocast("cuda", torch.float16):
        maps = [conv(x).reshape(B, M, C, *x.shape[-2:]) for x in xs]
        assert all(m.dtype == torch.float16 for m in maps)
        table, shape, start = DAF.feature_maps_format(maps)
        out = DAF.apply(table, shape, start, loc, w)
        ref_table = torch.cat([m.reshape(B, M, C, -1) for m in maps], dim=-1).permute(0, 1, 3, 2).float()
        ref = DAF.apply(ref_table, shape, start, loc, w)
    assert table.dtype == torch.float16 and out.dtype == torch.float32
    assert out.grad_fn.saved_tensors[0].dtype == torch.float16
    assert ref.grad_fn.saved_tensors[0].dtype == torch.float32
    assert torch.equal(out, ref)
    params = [conv.weight, conv.bias]
    mine = torch.autograd.grad((out * g).sum(), params, retain_graph=True)
    want = torch.autograd.grad((ref * g).sum(), params)
    for name, a, b in zip(("weight", "bias"), mine, want):
        b = b.cpu().numpy()
        h.assert_close(a.cpu().numpy(), b, rtol=1e-3, atol=h.grad_tolerance(b), what="autocast grad conv " + name)


def test_ex_entry_points_reject_an_unknown_dtype():
    """Runs without a GPU: the dtype is checked before any CUDA runtime call."""
    from gaussianformer_b200.csrc import build
    build.build()
    L = _lib.lib()
    d = _lib.DafDesc(1, 1, 4, 128, 1, 8, 4)
    fd = _lib.DafFusedDesc(d, 2)
    fmt = _lib.DafFormatDesc(1, 128, 1)
    calls = {
        "gf_daf_forward_ex": lambda: L.gf_daf_forward_ex(ctypes.byref(d), 7, *[None] * 7),
        "gf_daf_backward_ex": lambda: L.gf_daf_backward_ex(ctypes.byref(d), 7, *[None] * 10),
        "gf_daf_fused_forward_ex": lambda: L.gf_daf_fused_forward_ex(ctypes.byref(fd), 7, *[None] * 10),
        "gf_daf_fused_backward_ex": lambda: L.gf_daf_fused_backward_ex(ctypes.byref(fd), 7, *[None] * 14),
        "gf_daf_format_ex": lambda: L.gf_daf_format_ex(ctypes.byref(fmt), 7, None, None, 0, None),
    }
    for name, call in calls.items():
        assert call() == _lib.GF_ERR_INVALID_ARG, name
        msg = L.gf_last_error().decode()
        assert "dtype 7" in msg, (name, msg)
