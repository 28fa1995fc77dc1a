"""The device submanifold sparse convolution (gf_subm_conv_*, gaussianformer_b200.ops.sparse_conv) against the oracle
(tests/subm_conv_oracle.py): the rulebook exactly, the output and the three gradients under the gradient parity gate,
on tiny grids and on GaussianFormer's grids, and the properties the contract promises: duplicate rows, zero gradient
off the representatives, bit reproducibility, no host synchronisation, CUDA-graph replay and the SparseConv3D module."""
import ctypes

import numpy as np
import pytest
import torch
from torch import nn

import helpers as h
import subm_conv_oracle as sco
from gaussianformer_b200 import _lib
from gaussianformer_b200.ops import SparseConv3D, build_rulebook, subm_conv3d
from gaussianformer_b200.synthetic import make_subm_conv_inputs

pytestmark = pytest.mark.gpu

GF1, GF2 = (200, 200, 16), (100, 100, 8)
# name: (rows per sample, spatial, batch, k, clustered, invalid, duplicates_of, bias)
CASES = {
    "tiny_k3": (300, (9, 8, 7), 1, 3, False, 0, None, True),
    "tiny_k5": (300, (9, 8, 7), 1, 5, False, 0, None, False),
    "tiny_k1": (200, (6, 6, 6), 1, 1, False, 0, None, True),
    "b2_densities": ((600, 60), (10, 9, 8), 2, 3, False, 0, None, True),
    "duplicates": (400, (8, 8, 6), 2, 5, False, 0, 6, True),
    "invalid_rows": (400, (8, 8, 6), 2, 3, False, 25, 7, True),
    "gs25600_uniform": (25600, GF1, 1, 5, False, 0, None, False),
    "gs25600_clustered": (25600, GF1, 1, 5, True, 0, None, False),
    "gs144000_uniform": (144000, GF1, 1, 5, False, 0, None, False),
    "gs144000_clustered": (144000, GF1, 1, 5, True, 0, None, False),
    "prob_gs6400": (6400, GF2, 1, 5, False, 0, None, True),
    "prob_gs25600": (25600, GF2, 1, 5, False, 0, None, True),
    "prob_gs25600_clustered_b2": (25600, GF2, 2, 5, True, 0, None, True),
}
SMALL = [n for n, c in CASES.items() if c[1] not in (GF1, GF2)]


def _case(name, seed=0):
    n, spatial, batch, k, clustered, invalid, dup, with_bias = CASES[name]
    f, idx, w, b = make_subm_conv_inputs(n, spatial, batch=batch, clustered=clustered, seed=seed, kernel_size=k,
                                         invalid=invalid, duplicates_of=dup)
    return f, idx, w, (b if with_bias else None), spatial, batch, k


def _neighbors(rb):
    d = rb.desc
    N, K = d.num_rows, d.kernel_size ** 3
    m = ctypes.c_int32()
    slot, rep, nbr = np.zeros(N, np.int32), np.zeros(N, np.int32), np.zeros((N, K), np.int32)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)   # noqa: E731
    _lib.check(_lib.lib().gf_debug_subm_conv_neighbors(ctypes.byref(d), ctypes.c_void_p(rb.workspace.data_ptr()),
                                                       ctypes.c_void_p(torch.cuda.current_stream().cuda_stream),
                                                       ctypes.byref(m), p(slot), p(rep), p(nbr)))
    return m.value, slot, rep[:m.value], nbr[:m.value]


@pytest.mark.parametrize("name", SMALL + ["gs25600_clustered", "prob_gs25600_clustered_b2"])
def test_rulebook_matches_the_oracle(name):
    f, idx, w, b, spatial, batch, k = _case(name)
    rb = build_rulebook(idx.cuda(), spatial, batch, k, validate=False)
    ref = sco.rulebook(idx.numpy(), spatial, batch, k)
    m, slot, rep, nbr = _neighbors(rb)
    assert m == len(ref["rep"])
    np.testing.assert_array_equal(slot, ref["slot"])
    np.testing.assert_array_equal(rep, ref["rep"])
    np.testing.assert_array_equal(nbr, ref["nbr"])
    status = int(rb.workspace[:4].view(torch.int32).item())
    assert bool(status & _lib.GF_FLAG_INDEX_OUT_OF_RANGE) == bool((~ref["valid"]).any())


def _device(f, idx, w, b, spatial, batch, k, g, rulebook=None):
    x = f.cuda().requires_grad_()
    wt = w.cuda().requires_grad_()
    bt = None if b is None else b.cuda().requires_grad_()
    out = subm_conv3d(x, idx.cuda(), wt, bt, spatial, batch, rulebook=rulebook, validate=False)
    out.backward(g.cuda())
    return out.detach(), x.grad, wt.grad, (None if bt is None else bt.grad)


@pytest.mark.parametrize("name", list(CASES))
def test_parity_with_the_oracle(name):
    f, idx, w, b, spatial, batch, k = _case(name, seed=1)
    n_rows = f.shape[0]
    g = torch.randn(n_rows, 128, generator=torch.Generator().manual_seed(2))
    rb = sco.rulebook(idx.numpy(), spatial, batch, k)
    counts = np.bincount(rb["slot"][rb["valid"]])
    if name == "duplicates":
        assert (counts >= 3).sum() >= 5
    if name == "invalid_rows":
        assert (~rb["valid"]).sum() > 0
    if name == "b2_densities":
        assert len(np.unique(rb["voxels"][:, 0])) == 2
    mine = [t.double().cpu().numpy() if t is not None else None for t in _device(f, idx, w, b, spatial, batch, k, g)]
    if n_rows <= 1000:
        r64 = [sco.forward(f.numpy(), w.numpy(), None if b is None else b.numpy(), rb)] + \
            list(sco.backward(f.numpy(), w.numpy(), g.numpy(), rb))
        r32 = [sco.forward(f.numpy(), w.numpy(), None if b is None else b.numpy(), rb, np.float32)] + \
            list(sco.backward(f.numpy(), w.numpy(), g.numpy(), rb, np.float32))
    else:
        args = (f.numpy(), w.numpy(), None if b is None else b.numpy(), g.numpy(), rb)
        r64 = sco.torch_reference(*args, torch.float64, "cuda")
        r32 = sco.torch_reference(*args, torch.float32, "cuda")
    for what, a, e64, e32 in zip(("out", "grad_features", "grad_weight", "grad_bias"), mine, r64, r32):
        if a is None:
            continue
        h.assert_grad_parity(a, e64, e32, what=f"{name} {what}")
    assert not mine[0][~rb["valid"]].any()


def test_duplicates_bit_identical_and_zero_gradient_off_representatives():
    f, idx, w, b, spatial, batch, k = _case("invalid_rows", seed=3)
    rb = sco.rulebook(idx.numpy(), spatial, batch, k)
    g = torch.randn(f.shape[0], 128, generator=torch.Generator().manual_seed(4))
    out, gx, _, _ = (t.cpu().numpy() for t in _device(f, idx, w, b, spatial, batch, k, g))
    slot = rb["slot"]
    for s in np.nonzero(np.bincount(slot[rb["valid"]]) >= 2)[0]:
        rows = np.nonzero(slot == s)[0]
        assert (out[rows] == out[rows[0]]).all()
    not_rep = np.ones(len(slot), bool)
    not_rep[rb["rep"]] = False
    assert not_rep.sum() > 0 and (gx[not_rep] == 0).all()
    assert (out[~rb["valid"]] == 0).all()


@pytest.mark.parametrize("name", ["duplicates", "gs144000_clustered", "prob_gs25600"])
def test_two_calls_are_bit_identical(name):
    f, idx, w, b, spatial, batch, k = _case(name, seed=5)
    g = torch.randn(f.shape[0], 128, generator=torch.Generator().manual_seed(6))
    first = _device(f, idx, w, b, spatial, batch, k, g)
    rb = build_rulebook(idx.cuda(), spatial, batch, k, validate=False)
    second = _device(f, idx, w, b, spatial, batch, k, g, rulebook=rb)
    third = _device(f, idx, w, b, spatial, batch, k, g, rulebook=rb)
    for a, c, d in zip(first, second, third):
        if a is not None:
            assert torch.equal(a, c) and torch.equal(a, d)


def test_no_host_synchronisation():
    f, idx, w, b, spatial, batch, k = _case("prob_gs6400", seed=7)
    x, i, wt, bt = f.cuda().requires_grad_(), idx.cuda(), w.cuda().requires_grad_(), b.cuda().requires_grad_()
    g = torch.randn_like(x)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        rb = build_rulebook(i, spatial, batch, k, validate=False)
        out = subm_conv3d(x, i, wt, bt, spatial, batch, rulebook=rb)
        out.backward(g)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_cuda_graph_replay_matches_eager():
    f, idx, w, b, spatial, batch, k = _case("gs25600_clustered", seed=8)
    x, i, wt = f.cuda(), idx.cuda(), w.cuda()
    g = torch.randn_like(x)
    L = _lib.lib()
    rb = build_rulebook(i, spatial, batch, k, validate=False)
    d = rb.desc

    def step(out, gx, gw, gb):
        ptr = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None   # noqa: E731
        s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        _lib.check(L.gf_subm_conv_rulebook(ctypes.byref(d), ptr(rb.indices), ptr(rb.workspace),
                                           rb.workspace.numel(), s))
        _lib.check(L.gf_subm_conv_forward(ctypes.byref(d), ptr(rb.workspace), ptr(x), ptr(wt), None, ptr(out), s))
        _lib.check(L.gf_subm_conv_backward(ctypes.byref(d), ptr(rb.workspace), ptr(x), ptr(wt), ptr(g), ptr(gx),
                                           ptr(gw), ptr(gb), s))

    eager = [torch.empty_like(x), torch.empty_like(x), torch.empty_like(wt), torch.empty(128, device="cuda")]
    step(*eager)
    graphed = [torch.full_like(t, float("nan")) for t in eager]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step(*graphed)   # warm-up outside capture
    torch.cuda.current_stream().wait_stream(side)
    for t in graphed:
        t.fill_(float("nan"))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step(*graphed)
    graph.replay()
    graph.replay()
    torch.cuda.synchronize()
    for a, e in zip(graphed, eager):
        assert torch.equal(a, e)


def _conv_restated(x, w, b, rb_np):
    """the contract as torch gathers on the oracle's rulebook (differentiable, any dtype, on the CPU)"""
    k = rb_np["k"]
    rep, slot = torch.as_tensor(rb_np["rep"]), torch.as_tensor(rb_np["slot"])
    acc = torch.zeros(len(rep), w.shape[0], dtype=x.dtype) if b is None else b.expand(len(rep), -1).clone()
    for o, (dst, src) in enumerate(rb_np["pairs"]):
        wo = w[:, o // (k * k), (o // k) % k, o % k, :]
        acc = acc.index_add(0, torch.as_tensor(dst), x[rep[torch.as_tensor(src)]] @ wo.T)
    assert rb_np["valid"].all()
    return acc[slot]


def _reference_module(mod, feat, g, rb_np, dtype):
    """the reference SparseConv3D's forward restated in `dtype` on the CPU with spconv replaced by the oracle's
    contract, and its autograd backward for the output gradient g: (out, {parameter: grad}, grad of feat)"""
    P = {n: p.detach().cpu().to(dtype).requires_grad_() for n, p in mod.named_parameters()}
    B, G, Cc = feat.shape
    x0 = feat.detach().cpu().to(dtype).requires_grad_()
    x = x0.flatten(0, 1)
    if isinstance(mod.layer, nn.Sequential):
        for j in (0, 3, 6):
            y = _conv_restated(x, P[f"layer.{j}.weight"], P[f"layer.{j}.bias"], rb_np)
            x = torch.relu(torch.nn.functional.layer_norm(y, (Cc,), P[f"layer.{j + 1}.weight"],
                                                          P[f"layer.{j + 1}.bias"]))
    else:
        x = _conv_restated(x, P["layer.weight"], None, rb_np)
    y = x.reshape(B, G, Cc)
    if "output_proj.weight" in P:
        y = y @ P["output_proj.weight"].T + P["output_proj.bias"]
    y.backward(g.cpu().to(dtype))
    return (y.detach().double().numpy(), {n: p.grad.double().numpy() for n, p in P.items()},
            x0.grad.double().numpy())


@pytest.mark.parametrize("multi", [False, True])
def test_sparse_conv3d_module_matches_the_reference_restatement(multi):
    pc = [-50.0, -50.0, -5.0, 50.0, 50.0, 3.0]
    torch.manual_seed(9)
    kw = dict(use_multi_layer=True, grid_size=[1.0] * 3) if multi else dict(use_out_proj=True, grid_size=[0.5] * 3)
    gs = kw.pop("grid_size")
    mod = SparseConv3D(128, 128, pc, gs, kernel_size=5, phi_activation="sigmoid", **kw).cuda()
    B, G = 2, 3000
    gen = torch.Generator().manual_seed(10)
    anchor = torch.randn(B, G, 11, generator=gen) * 1.5
    anchor[1, :, :3] = anchor[1, :, :3] * 0.3       # the second sample denser
    anchor[:, ::7, :3] = anchor[:, 1::7, :3][:, :anchor[:, ::7].shape[1]]   # shared voxels
    feat = torch.randn(B, G, 128, generator=gen)
    anchor, feat = anchor.cuda(), feat.cuda().requires_grad_()
    out = mod(feat, anchor)
    idx = mod.voxel_indices(anchor)
    # the reference's expression, op for op, on the same fp32 tensors
    a = anchor[..., :3]
    xyz = torch.sigmoid(torch.clamp(a, -9.21, 9.21))
    xyz = torch.stack([xyz[..., 0] * (pc[3] - pc[0]) + pc[0], xyz[..., 1] * (pc[4] - pc[1]) + pc[1],
                       xyz[..., 2] * (pc[5] - pc[2]) + pc[2]], dim=-1).flatten(0, 1)
    ref_idx = ((xyz - mod.pc_range[None, :3]) / mod.grid_size[None, :]).to(torch.int32)
    assert torch.equal(idx[:, 1:], ref_idx)
    rb_np = sco.rulebook(idx.cpu().numpy(), mod.spatial_shape, B, 5)
    assert (np.bincount(rb_np["slot"]) >= 2).any()
    g = torch.randn(B, G, 128, generator=torch.Generator().manual_seed(11)).cuda()
    out.backward(g)
    out64, grads64, feat64 = _reference_module(mod, feat, g, rb_np, torch.float64)
    out32, grads32, feat32 = _reference_module(mod, feat, g, rb_np, torch.float32)
    h.assert_grad_parity(out.detach().double().cpu().numpy(), out64, out32, what=f"multi={multi} out")
    h.assert_grad_parity(feat.grad.double().cpu().numpy(), feat64, feat32, what=f"multi={multi} grad feat")
    for n, p in mod.named_parameters():
        h.assert_grad_parity(p.grad.double().cpu().numpy(), grads64[n], grads32[n], what=f"multi={multi} grad {n}")
    feat = feat.detach()
    sd = mod.state_dict()
    twin = SparseConv3D(128, 128, pc, gs, kernel_size=5, **kw).cuda()
    twin.load_state_dict(sd, strict=True)
    mod.load_state_dict(twin.state_dict(), strict=True)
    assert torch.equal(twin(feat, anchor), out.detach())
