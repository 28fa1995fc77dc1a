"""The anchor key-point generator on the GPU: the kernels against the fp64 oracle (daf_anchor_oracle) at both shipped
configs and on crafted cases, reproducibility, the module + deformable_aggregation_from_key_points against the
reference's composition, half anchors, CUDA-graph replay and the argument errors."""
import numpy as np
import pytest
import torch

import daf_anchor_oracle as ao
import helpers as h
from gaussianformer_b200.ops import DeformableAggregationFunction as DAF
from gaussianformer_b200.ops import SparseGaussian3DKeyPointsGenerator, anchor_key_points
from gaussianformer_b200.ops import deformable_aggregation_from_key_points as daf_kp
from gaussianformer_b200.synthetic import ANCHOR_FIX_SCALE, make_anchor_kp_inputs, make_daf_kp_inputs
from gaussianformer_b200.synthetic import reference_fused_composition
from test_daf_anchor_kp_cpu import _crafted
from test_daf_key_points_gpu import _ulps, literal_project_points

pytestmark = pytest.mark.gpu

CONFIGS = ["gs25600_solid", "prob_gs6400"]


def _inputs(config, seed=0, B=2):
    """B = 2 with different anchors per sample"""
    d = make_anchor_kp_inputs(config, batch=B, seed=seed)
    return d["anchor"], d["logits"], d["fix_scale"], d["pc_range"], d["scale_range"], d["learnable_fixed_scale"]


def _run(anchor, logits, fix, pcr, scr, lfs, g=None):
    a = anchor.cuda().requires_grad_()
    lg = None if logits is None else logits.cuda().requires_grad_()
    kp = anchor_key_points(a, lg, fix.cuda(), pcr, scr, lfs)
    if g is None:
        return kp.detach(), None, None
    kp.backward(g.cuda())
    return kp.detach(), a.grad, None if lg is None else lg.grad


def assert_within_oracle(got, d64, dabs, what, midpoint_aware):
    """got within 1 fp32 ulp of float(d64) -- for the forward only where d64 lies within 2^-40 x dabs of a midpoint
    between two fp32 values, otherwise equal -- except where d64 is below 2^-24 x dabs (cancellation: the last bits of
    fp64 exp decide the rounding), which is held to |got - d64| <= 2^-40 x dabs."""
    got = np.asarray(got, np.float32)
    d64, dabs = np.asarray(d64, np.float64), np.asarray(dabs, np.float64)
    r32 = d64.astype(np.float32)
    ulps = _ulps(got, r32)
    cancel = np.abs(d64) < 2.0 ** -24 * dabs
    if midpoint_aware:
        other = np.nextafter(r32, np.where(d64 > r32, np.float32(np.inf), np.float32(-np.inf))).astype(np.float64)
        near = np.abs(d64 - (r32.astype(np.float64) + other) / 2) <= 2.0 ** -40 * dabs
        close = (ulps == 0) | ((ulps <= 1) & near)
    else:
        close = ulps <= 1
    ok = np.where(cancel, np.abs(got.astype(np.float64) - d64) <= 2.0 ** -40 * dabs, close)
    assert ok.all(), f"{what}: {int((~ok).sum())} of {ok.size} entries outside the gate, first at {np.argwhere(~ok)[0]}"
    return int(cancel.sum())


CASES = {c: (lambda c=c: _inputs(c, seed=1)) for c in CONFIGS}
CASES["crafted"] = _crafted


@pytest.mark.parametrize("case", list(CASES))
def test_forward_and_backward_against_the_oracle(case):
    anchor, logits, fix, pcr, scr, lfs = CASES[case]()
    g = torch.randn(anchor.shape[0], anchor.shape[1], len(fix) + logits.shape[2], 3,
                    generator=torch.Generator().manual_seed(3))
    kp, ga, gl = _run(anchor, logits, fix, pcr, scr, lfs, g)
    _, kp64, kp_abs = ao.key_points(anchor.numpy(), fix.numpy(), logits.numpy(), pcr, scr, lfs)
    assert_within_oracle(kp.cpu().numpy(), kp64, kp_abs, f"{case} key points", True)
    want_a, abs_a, want_l, abs_l = ao.key_points_backward(anchor.numpy(), fix.numpy(), logits.numpy(), pcr, scr, lfs,
                                                          g.numpy())
    ga, gl = ga.cpu().numpy(), gl.cpu().numpy()
    assert (ga[..., 10:] == 0).all() and not np.signbit(ga[..., 10:]).any()
    assert_within_oracle(ga, want_a, abs_a, f"{case} grad anchor", False)
    assert_within_oracle(gl, want_l, abs_l, f"{case} grad learnable", False)
    if case == "crafted":                                   # the clamp's gate on the device
        assert (ga[0, 0, [0, 1, 3, 4]] != 0).all() and (ga[0, 1, [0, 2, 3]] == 0).all()
        assert (gl[0, 0, 0, :2] != 0).all() and gl[0, 0, 0, 2] == 0 and gl[0, 1, 1, 0] == 0
        assert np.isfinite(ga).all()


def test_fixed_points_only():
    """num_learnable_pts = 0 / no instance_feature, and the default fix_scale ((0, 0, 0),)"""
    anchor, logits, fix, pcr, scr, lfs = _inputs("gs25600_solid", seed=2)
    d = make_anchor_kp_inputs("gs25600_solid", batch=2, seed=2)
    m = SparseGaussian3DKeyPointsGenerator(embed_dims=128, num_learnable_pts=2, fix_scale=ANCHOR_FIX_SCALE,
                                           pc_range=pcr, scale_range=scr).cuda()
    a = anchor.cuda()
    kp = m(a)                                               # instance_feature=None: the 7 fixed points only
    assert kp.shape == (2, 25600, 7, 3)
    assert torch.equal(kp, m(a, d["instance_feature"].cuda())[:, :, :7])
    for fix0 in (fix, torch.zeros(1, 3)):
        g = torch.randn(2, 25600, len(fix0), 3, generator=torch.Generator().manual_seed(4))
        kp, ga, gl = _run(anchor, None, fix0, pcr, scr, lfs, g)
        assert gl is None
        _, kp64, kp_abs = ao.key_points(anchor.numpy(), fix0.numpy(), None, pcr, scr, lfs)
        assert_within_oracle(kp.cpu().numpy(), kp64, kp_abs, "fixed only", True)
        want, wabs, _, _ = ao.key_points_backward(anchor.numpy(), fix0.numpy(), None, pcr, scr, lfs, g.numpy())
        assert_within_oracle(ga.cpu().numpy(), want, wabs, "fixed only grad", False)
    m0 = SparseGaussian3DKeyPointsGenerator(pc_range=pcr, scale_range=scr).cuda()
    assert m0(a).shape == (2, 25600, 1, 3)


def test_gradients_are_bit_reproducible():
    anchor, logits, fix, pcr, scr, lfs = _inputs("prob_gs6400", seed=5)
    g = torch.randn(2, 6400, 13, 3, generator=torch.Generator().manual_seed(6))
    first = _run(anchor, logits, fix, pcr, scr, lfs, g)
    for _ in range(2):
        again = _run(anchor, logits, fix, pcr, scr, lfs, g)
        assert all(torch.equal(x, y) for x, y in zip(first, again))
    for b in range(2):
        alone = _run(anchor[b:b + 1], logits[b:b + 1], fix, pcr, scr, lfs, g[b:b + 1])
        assert all(torch.equal(x[0], y[b]) for x, y in zip(alone, first))


@pytest.mark.parametrize("config", CONFIGS)
def test_module_into_the_op_against_the_reference_composition(config):
    """SparseGaussian3DKeyPointsGenerator -> deformable_aggregation_from_key_points against the reference's generator
    -> literal fp32 project_points -> reference_fused_composition around DAF.apply, both differentiated by autograd.
    The reference generator runs in fp64 and its key points are rounded to fp32 once: evaluated in fp32 it rounds
    coordinates of up to 50 m to ~4e-6 m, which moves a sample by ~1e-3 px and the output by up to ~4e-4, more than
    the key-point test's tolerances, which then apply unchanged.  make_anchor_kp_inputs' margins keep every gate, mask
    and cell decision away from fp32 rounding."""
    d = make_anchor_kp_inputs(config, batch=1, seed=7, margin=True)
    A, Kl = d["anchor"].shape[1], d["num_learnable"]
    K = 7 + Kl
    fms, _, _, _, wlog, _ = make_daf_kp_inputs(num_anchor=A, num_pts=K, seed=8)
    M = wlog.shape[3]
    P, wh = d["projection_mat"].cuda(), d["image_wh"].cuda()
    up = torch.randn(1, A, 128, generator=torch.Generator().manual_seed(9)).cuda()
    outs, grads = [], []
    for mine in (True, False):
        m = SparseGaussian3DKeyPointsGenerator(embed_dims=128, num_learnable_pts=Kl,
                                               learnable_fixed_scale=d["learnable_fixed_scale"],
                                               fix_scale=ANCHOR_FIX_SCALE, pc_range=d["pc_range"],
                                               scale_range=d["scale_range"], phi_activation="sigmoid").cuda()
        m.load_state_dict({"learnable_fc.weight": d["weight"], "learnable_fc.bias": d["bias"]})
        feat, shape, start = DAF.feature_maps_format([f.cuda() for f in fms])
        feat = feat.detach().contiguous().requires_grad_()
        anchor = d["anchor"].cuda().requires_grad_()
        lg = wlog.cuda().requires_grad_()
        inst = d["instance_feature"].cuda()
        if mine:
            out = daf_kp(feat, shape, start, m(anchor, inst), P, wh, lg)
        else:
            logits = m.learnable_fc(inst).reshape(1, A, Kl, 3)
            kp = ao.reference_generator(anchor.double(), logits.double(), ANCHOR_FIX_SCALE, d["pc_range"],
                                        d["scale_range"], d["learnable_fixed_scale"]).float()
            pts, mask = literal_project_points(kp, P, wh)
            loc = pts.permute(0, 2, 3, 1, 4).reshape(1, A * K, M, 2)
            out = reference_fused_composition(DAF.apply, feat, shape, start, loc, lg, mask.permute(0, 2, 3, 1))
        out.backward(up)
        outs.append(out.detach().cpu().numpy())
        grads.append([t.grad.cpu().numpy() for t in (anchor, m.learnable_fc.weight, feat, lg)])
    h.assert_close(outs[0], outs[1], atol=1e-4, what="output vs the reference composition")
    for name, a, b in zip(("anchor", "learnable_fc weight", "feat", "weight logits"), grads[0], grads[1]):
        h.assert_close(a, b, rtol=1e-3, atol=h.grad_tolerance(b), what="grad " + name)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_half_anchors_equal_the_upcast_anchors(dtype):
    anchor, logits, fix, pcr, scr, lfs = _inputs("prob_gs6400", seed=10)
    anchor, logits = anchor.to(dtype), logits.to(dtype)
    g = torch.randn(2, 6400, 13, 3, generator=torch.Generator().manual_seed(11))
    half = _run(anchor, logits, fix, pcr, scr, lfs, g)
    full = _run(anchor.float(), logits.float(), fix, pcr, scr, lfs, g)
    assert half[0].dtype == torch.float32 and torch.equal(half[0], full[0])
    assert half[1].dtype == dtype and half[2].dtype == dtype
    assert torch.equal(half[1], full[1].to(dtype)) and torch.equal(half[2], full[2].to(dtype))


def test_non_contiguous_anchors():
    anchor, logits, fix, pcr, scr, lfs = _inputs("gs25600_solid", seed=12)
    wide = torch.cat([anchor, torch.randn(2, 25600, 4)], -1).cuda()[..., :28]        # row stride 32
    kp = anchor_key_points(wide, logits.cuda(), fix.cuda(), pcr, scr, lfs)
    assert torch.equal(kp, _run(anchor, logits, fix, pcr, scr, lfs)[0])


def test_cuda_graph_replay_with_new_anchors():
    anchor, logits, fix, pcr, scr, lfs = _inputs("prob_gs6400", seed=13)
    a = anchor.cuda().requires_grad_()
    lg = logits.cuda().requires_grad_()
    fix_d = fix.cuda()
    up = torch.randn(2, 6400, 13, 3, generator=torch.Generator().manual_seed(14)).cuda()

    def step():
        a.grad = lg.grad = None
        kp = anchor_key_points(a, lg, fix_d, pcr, scr, lfs)
        kp.backward(up)
        return kp.detach(), a.grad, lg.grad

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
    for seed in (15, 16):
        new_a, new_l, _, _, _, _ = _inputs("prob_gs6400", seed=seed)
        with torch.no_grad():
            a.copy_(new_a.cuda())
            lg.copy_(new_l.cuda())
        graph.replay()
        torch.cuda.synchronize()
        eager = _run(new_a, new_l, fix, pcr, scr, lfs, up.cpu())
        assert all(torch.equal(x, y) for x, y in zip(static, eager))


def test_errors():
    anchor, logits, fix, pcr, scr, lfs = _inputs("gs25600_solid", seed=17)
    a, lg, f = anchor[:, :64].cuda(), logits[:, :64].cuda(), fix.cuda()
    anchor_key_points(a, lg, f, pcr, scr, lfs)
    with pytest.raises(RuntimeError, match="CUDA-only"):
        anchor_key_points(a.cpu(), lg, f, pcr, scr, lfs)
    with pytest.raises(ValueError, match="D >= 10"):
        anchor_key_points(a[..., :9], lg, f, pcr, scr, lfs)
    with pytest.raises(ValueError, match="learnable_logits"):
        anchor_key_points(a, lg[:, :32], f, pcr, scr, lfs)
    with pytest.raises(ValueError, match="learnable_logits"):
        anchor_key_points(a, lg[..., :2], f, pcr, scr, lfs)
    with pytest.raises(ValueError, match="fix_scale"):
        anchor_key_points(a, lg, f[:, :2], pcr, scr, lfs)
    with pytest.raises(Exception, match="num_fixed \\+ num_learnable"):
        anchor_key_points(a, None, f[:0], pcr, scr, lfs)
