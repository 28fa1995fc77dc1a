"""The device occupancy loss (gf_occ_loss, gaussianformer_b200.loss) against the fp64 oracle and the PyTorch
restatement of the reference (tests/occ_loss_oracle.py): values, the Lovasz sort order, gradients evaluated in the
device's own order, layouts, determinism, no host synchronisation, CUDA-graph replay, validation and the chain from
the splat."""
import ctypes

import numpy as np
import pytest
import torch

import helpers as h
import occ_loss_oracle as olo
from gaussianformer_b200 import _lib
from gaussianformer_b200.loss import OccupancyLoss, occupancy_loss
from gaussianformer_b200.synthetic import make_occ_labels, make_occ_loss_inputs

pytestmark = pytest.mark.gpu

MANUAL = [1.01552756, 1.06897009, 1.30013094, 1.07253735, 0.94637502, 1.10087012, 1.26960524, 1.06258364, 1.189019,
          1.06217292, 1.00595144, 0.85706115, 1.03923299, 0.90867526, 0.8936431, 0.85486129, 0.8527829, 0.5, 0.7, 1.2]
CE_W, LOV_W = 10.0, 1.0


def _weights(C):
    w = torch.tensor(MANUAL[:C])
    return (C * w / w.abs().sum()).float()


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _abi(x, labels, mask, w, use_softmax, lovasz_ignore=17, empty_label=None, grad=True, ws=None):
    """One gf_occ_loss call on x [B, C, N] (either layout): (loss[3], grad in x's strides, workspace, desc)"""
    from gaussianformer_b200.loss import _layout
    layout, x = _layout(x)
    B, C, N = x.shape
    d = _lib.OccLossDesc(B, N, C, 0 if use_softmax else 1, layout, 255, lovasz_ignore,
                         -1 if empty_label is None else empty_label, 1.0, CE_W, LOV_W)
    L = _lib.lib()
    nbytes = L.gf_occ_loss_workspace_bytes(ctypes.byref(d))
    assert nbytes > 0
    if ws is None:
        ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    loss = torch.empty(3, device="cuda")
    g = torch.empty_strided(x.shape, x.stride(), device="cuda") if grad else None
    m = None if mask is None else mask.view(torch.uint8)
    _lib.check(L.gf_occ_loss(ctypes.byref(d), _ptr(x), _ptr(labels), _ptr(m), _ptr(w), _ptr(loss), _ptr(g), _ptr(ws),
                             nbytes, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return loss, g, ws, d


def _order(d, ws):
    """{present class: positions in V in the device's sorted order}, |V|"""
    nvox = d.batch * d.N
    order = np.zeros((d.C, max(nvox, 1)), np.int32)
    nv = ctypes.c_int32()
    present = np.zeros(d.C, np.uint8)
    _lib.check(_lib.lib().gf_debug_occ_loss_order(ctypes.byref(d), _ptr(ws),
                                                  ctypes.c_void_p(torch.cuda.current_stream().cuda_stream),
                                                  order.ctypes.data_as(ctypes.c_void_p), ctypes.byref(nv),
                                                  present.ctypes.data_as(ctypes.c_void_p)))
    return {c: order[c, :nv.value].copy() for c in range(d.C) if present[c]}, nv.value


def _inputs(B, N, C, use_softmax, seed, with_mask):
    pred, labels, mask = make_occ_loss_inputs(B, N, C, use_softmax, seed, ignore_share=0.01, duplicate_share=0.02)
    return pred.cuda(), labels.cuda(), (mask.cuda() if with_mask else None)


CASES = (
    [("tiny", 1, 4000, 18, sm, mk, em, lay) for sm in (True, False) for mk, em, lay in
     ((True, None, "voxel"), (False, None, "class"), (True, 17, "voxel"), (False, 17, "class"))] +
    [(name, B, 640000, 18, sm, True, None, "voxel") for name, B in (("full", 1), ("full_b2", 2)) for sm in (True, False)] +
    [(f"c{C}", B, N, C, sm, mk, em, lay) for C, B, N in ((17, 2, 20000), (20, 1, 50000)) for sm in (True, False)
     for mk, em, lay in ((True, None, "voxel"), (False, 17, "class"))]
)


@pytest.mark.parametrize("name,B,N,C,use_softmax,with_mask,empty,layout", CASES,
                         ids=[f"{c[0]}-{'logits' if c[4] else 'probs'}-{'mask' if c[5] else 'nomask'}-"
                              f"{'empty' if c[6] is not None else 'all'}-{c[7]}" for c in CASES])
def test_against_oracle(name, B, N, C, use_softmax, with_mask, empty, layout):
    pred, labels, mask = _inputs(B, N, C, use_softmax, seed=B * 7 + C, with_mask=with_mask)
    x = pred.transpose(1, 2)
    if layout == "class":
        x = x.contiguous()
    w = _weights(C).cuda()
    loss, grad, ws, d = _abi(x, labels, mask, w, use_softmax, empty_label=empty)
    order, nv = _order(d, ws)
    assert (grad.stride() == x.stride())
    xn, yn = x.cpu().numpy(), labels.cpu().numpy()
    mn = None if mask is None else mask.cpu().numpy()
    kw = dict(use_softmax=use_softmax, lovasz_ignore=17, empty_label=empty, ce_weight=CE_W, lovasz_weight=LOV_W)
    ref = olo.oracle(xn, yn, mn, w.cpu().numpy(), **kw)
    assert nv == len(ref["V"]) and sorted(order) == ref["present"]

    # values: the fp64 oracle, and the fp32 restatement as written (unstable sort, syncing gathers)
    got = loss.cpu().numpy().astype(np.float64)
    for i, key in enumerate(("loss", "ce", "lovasz")):
        assert abs(got[i] - ref[key]) <= 1e-5 + 1e-4 * abs(ref[key]), (key, got[i], ref[key])
    rest = [float(v) for v in olo.restatement(x, labels, mask, w, **kw)]
    for i, key in enumerate(("loss", "ce", "lovasz")):
        dist = abs(rest[i] - ref[key])
        assert abs(got[i] - rest[i]) <= max(1e-5 + 1e-4 * abs(ref[key]), 4 * dist), (key, got[i], rest[i], ref[key])

    # order: a permutation of V along which the fp64 errors never rise by more than 2^-20, exact ties ascending
    for c, o in order.items():
        assert np.array_equal(np.sort(o), np.arange(nv)), c
        e = ref["errors"][c][o]
        assert (np.diff(e) <= 2.0 ** -20).all(), (c, float(np.diff(e).max()))
        s = np.argsort(e, kind="stable")
        tie = e[s][1:] == e[s][:-1]
        assert (o[s][1:][tie] > o[s][:-1][tie]).all(), c
        if not use_softmax:   # fp32 errors are the same bits on both sides: torch's stable sort gives the same order
            V = torch.as_tensor(ref["V"], device="cuda")
            xv = x.transpose(1, 2).reshape(-1, C)[V, c]
            e32 = ((labels.reshape(-1)[V] == c).float() - xv).abs()
            assert np.array_equal(torch.sort(e32, descending=True, stable=True).indices.cpu().numpy(), o), c

    # gradients per entry: the fp64 oracle in the device's order, floor = the fp32 restatement in that order
    ref_o = olo.oracle(xn, yn, mn, w.cpu().numpy(), order=order, **kw)
    x32 = x.detach().clone().requires_grad_()
    olo.restatement(x32, labels, mask, w, order=order, **kw)[0].backward()
    g32 = x32.grad.cpu().numpy()
    mine = grad.cpu().numpy()
    h.assert_grad_parity(mine, ref_o["grad"], g32, what=f"{name} grad")
    if not use_softmax:
        x_as = x.detach().clone().requires_grad_()
        olo.restatement(x_as, labels, mask, w, **kw)[0].backward()
        h.assert_grad_parity(mine, x_as.grad.cpu().numpy(), ref_o["grad"], what=f"{name} grad vs restatement autograd")


def test_gradient_layout_follows_pred():
    C = 18
    pred, labels, mask = _inputs(2, 3000, C, True, 1, True)
    crit = OccupancyLoss(num_classes=C, balance_cls_weight=True, manual_class_weight=MANUAL[:C],
                         use_sem_geo_scal_loss=False, lovasz_ignore=17,
                         multi_loss_weights=dict(loss_voxel_ce_weight=CE_W, loss_voxel_lovasz_weight=LOV_W)).cuda()
    leaf = pred.clone().requires_grad_()            # the splat's contiguous [B, N, C]
    sem = leaf.transpose(1, 2)
    seen = []
    sem.register_hook(lambda g: seen.append(g.stride()))
    crit(dict(pred_occ=[sem], sampled_xyz=None, sampled_label=labels, occ_mask=mask)).backward()
    assert seen == [sem.stride()] and leaf.grad.is_contiguous()
    cm = pred.transpose(1, 2).contiguous().requires_grad_()     # forward_eval's class-major [B, C, N]
    crit(dict(pred_occ=[cm], sampled_xyz=None, sampled_label=labels, occ_mask=mask)).backward()
    assert cm.grad.is_contiguous()
    torch.testing.assert_close(cm.grad, leaf.grad.transpose(1, 2), rtol=0, atol=0)


@pytest.mark.parametrize("use_softmax", [True, False])
def test_bit_reproducible(use_softmax):
    pred, labels, mask = _inputs(1, 640000, 18, use_softmax, 5, True)
    w = _weights(18).cuda()
    a = _abi(pred.transpose(1, 2), labels, mask, w, use_softmax)
    b = _abi(pred.transpose(1, 2), labels, mask, w, use_softmax)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_module_never_synchronises_and_layers_average():
    C = 18
    pred, labels, mask = _inputs(1, 640000, C, True, 2, True)
    crit = OccupancyLoss(weight=1.5, num_classes=C, balance_cls_weight=True, manual_class_weight=MANUAL[:C],
                         use_sem_geo_scal_loss=False, lovasz_ignore=17,
                         multi_loss_weights=dict(loss_voxel_ce_weight=CE_W, loss_voxel_lovasz_weight=LOV_W)).cuda()
    crit.validate = False
    layers = [(pred * s).requires_grad_() for s in (1.0, 0.5)]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = crit(dict(pred_occ=[p.transpose(1, 2) for p in layers], sampled_xyz=None, sampled_label=labels,
                         occ_mask=mask))
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    w = _weights(C).cuda()
    parts = [_abi(p.detach().transpose(1, 2), labels, mask, w, True) for p in layers]
    want = 1.5 * (parts[0][0][0] + parts[1][0][0]) / 2
    torch.testing.assert_close(loss.detach(), want, rtol=1e-6, atol=0)
    for p, (_, g, _, _) in zip(layers, parts):
        torch.testing.assert_close(p.grad, 1.5 / 2 * g.transpose(1, 2), rtol=1e-6, atol=1e-12)


@pytest.mark.parametrize("use_softmax", [True, False])
def test_cuda_graph_replay_matches_eager(use_softmax):
    C, B, N = 18, 2, 100000
    pred, labels, mask = _inputs(B, N, C, use_softmax, 3, True)
    w = _weights(C).cuda()
    x = pred.transpose(1, 2)
    static = [x.clone(memory_format=torch.preserve_format), labels.clone(), mask.clone()]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        out = _abi(static[0], static[1], static[2], w, use_softmax)   # warm-up; allocates the workspace
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = _abi(static[0], static[1], static[2], w, use_softmax, ws=out[2])
    for seed in (11, 12):
        p2, l2, m2 = _inputs(B, N, C, use_softmax, seed, True)
        static[0].copy_(p2.transpose(1, 2))
        static[1].copy_(l2)
        static[2].copy_(m2)
        graph.replay()
        eager = _abi(p2.transpose(1, 2), l2, m2, w, use_softmax)
        torch.cuda.synchronize()
        assert torch.equal(out[0], eager[0]) and torch.equal(out[1], eager[1])


def test_validation_raises_on_out_of_range_label():
    C = 18
    pred, labels, mask = _inputs(1, 5000, C, True, 4, True)
    x = pred.transpose(1, 2)
    kw = dict(class_weights=_weights(C).cuda(), ce_weight=CE_W, lovasz_weight=LOV_W, lovasz_ignore=17, validate=True)
    occupancy_loss(x, labels, mask, **kw)                  # 255 and 17 are allowed
    bad = labels.clone()
    bad[0, torch.nonzero(mask[0])[0, 0]] = 40
    with pytest.raises(ValueError, match="outside"):
        occupancy_loss(x, bad, mask, **kw)
    masked_out = labels.clone()
    masked_out[0, torch.nonzero(~mask[0])[0, 0]] = 40      # outside the pool: not an error
    occupancy_loss(x, masked_out, mask, **kw)


def test_chain_from_the_splat():
    kw, inp, variant = h.splat_case("tiny", 1, True)
    m = h.make_module(kw, variant)
    t = h.to_dev(inp, requires_grad=True)
    out = m(t["pts"], t["means"], t["opa"], t["sem"], t["scales"], t["cov"])
    lg = out if out.dim() == 3 else out[None]
    _, N, C = lg.shape
    labels = make_occ_labels(1, N, C, seed=3, ignore_share=0.01).cuda()
    mask = labels != 0
    crit = OccupancyLoss(num_classes=C, balance_cls_weight=True, manual_class_weight=MANUAL[:C],
                         use_sem_geo_scal_loss=False, lovasz_ignore=17,
                         multi_loss_weights=dict(loss_voxel_ce_weight=CE_W, loss_voxel_lovasz_weight=LOV_W)).cuda()
    crit(dict(pred_occ=[lg.transpose(1, 2)], sampled_xyz=None, sampled_label=labels, occ_mask=mask)).backward()
    x = lg.detach().transpose(1, 2)
    w = crit.class_weights
    _, _, ws, d = _abi(x, labels, mask, w, True)
    order, _ = _order(d, ws)
    ref = olo.oracle(x.cpu().numpy(), labels.cpu().numpy(), mask.cpu().numpy(), w.cpu().numpy(), use_softmax=True,
                     lovasz_ignore=17, ce_weight=CE_W, lovasz_weight=LOV_W, order=order)
    g = ref["grad"][0].T.reshape(out.shape)
    h.check_module_grads(t, kw, inp, variant, (g,), what="splat <- occupancy loss")
