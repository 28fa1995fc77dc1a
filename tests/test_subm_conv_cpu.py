"""CPU checks of the submanifold sparse convolution: the numpy oracle against F.conv3d on unique indices (offset order,
cross-correlation, weight layout), its gradients against autograd through an fp64 torch gather restatement, the
duplicate- and invalid-row semantics, the ctypes desc layout and every refusal of the C ABI (all before any CUDA
call, so they run without a GPU)."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import subm_conv_oracle as sco
from gaussianformer_b200 import _lib
from gaussianformer_b200.synthetic import make_subm_conv_inputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C = 128


def _unique_case(k, seed=0, spatial=(6, 5, 4), batch=2, n=40):
    f, idx, w, b = make_subm_conv_inputs(n, spatial, batch=batch, seed=seed, kernel_size=k)
    _, first = np.unique(idx.numpy(), axis=0, return_index=True)
    keep = np.sort(first)
    return f[keep].double(), idx[keep], w.double(), b.double()


@pytest.mark.parametrize("k", [1, 3, 5])
def test_oracle_equals_dense_conv3d_on_unique_indices(k):
    spatial, batch = (6, 5, 4), 2
    f, idx, w, b = _unique_case(k, seed=k, spatial=spatial, batch=batch)
    rb = sco.rulebook(idx.numpy(), spatial, batch, k)
    out = sco.forward(f.numpy(), w.numpy(), b.numpy(), rb)
    dense = torch.zeros(batch, C, *spatial, dtype=torch.float64)
    i = idx.long()
    dense[i[:, 0], :, i[:, 1], i[:, 2], i[:, 3]] = f
    ref = F.conv3d(dense, w.permute(0, 4, 1, 2, 3), b, padding=(k - 1) // 2)
    ref = ref[i[:, 0], :, i[:, 1], i[:, 2], i[:, 3]]
    np.testing.assert_allclose(out, ref.numpy(), rtol=1e-12, atol=1e-12)


def _restatement(x, w, b, rb, k):
    """the contract as fp64 torch gathers: out[i] = b + sum_o W_o x[rep(nbr(slot(i), o))]"""
    rep = torch.as_tensor(rb["rep"])
    nbr = torch.as_tensor(rb["nbr"])
    acc = b.expand(len(rep), -1).clone()
    for o in range(k ** 3):
        hit = nbr[:, o] >= 0
        wo = w[:, o // (k * k), (o // k) % k, o % k, :]
        acc = acc.index_add(0, torch.nonzero(hit)[:, 0], x[rep[nbr[hit, o]]] @ wo.T)
    slot = torch.as_tensor(rb["slot"])
    valid = torch.as_tensor(rb["valid"])
    return torch.where(valid[:, None], acc[slot.clamp(min=0)], torch.zeros((), dtype=x.dtype))


@pytest.mark.parametrize("k", [3, 5])
def test_oracle_gradients_equal_autograd_with_duplicates_and_invalid_rows(k):
    spatial, batch = (7, 6, 5), 2
    f, idx, w, b = make_subm_conv_inputs(160, spatial, batch=batch, seed=10 + k, kernel_size=k, invalid=6,
                                         duplicates_of=9)
    rb = sco.rulebook(idx.numpy(), spatial, batch, k)
    counts = np.bincount(rb["slot"][rb["valid"]])
    assert counts.max() >= 3 and (~rb["valid"]).sum() > 0
    g = torch.randn(f.shape[0], C, dtype=torch.float64, generator=torch.Generator().manual_seed(k))
    x = f.double().requires_grad_()
    wt = w.double().requires_grad_()
    bt = b.double().requires_grad_()
    out = _restatement(x, wt, bt, rb, k)
    np.testing.assert_allclose(sco.forward(f.numpy(), w.numpy(), b.numpy(), rb), out.detach().numpy(), rtol=1e-12,
                               atol=1e-12)
    (out * g).sum().backward()
    gx, gw, gb = sco.backward(f.numpy(), w.numpy(), g.numpy(), rb)
    np.testing.assert_allclose(gx, x.grad.numpy(), rtol=1e-11, atol=1e-11)
    np.testing.assert_allclose(gw, wt.grad.numpy(), rtol=1e-11, atol=1e-11)
    np.testing.assert_allclose(gb, bt.grad.numpy(), rtol=1e-11, atol=1e-11)


def test_duplicate_and_invalid_row_semantics():
    spatial, batch, k = (5, 5, 5), 1, 3
    f, idx, w, b = make_subm_conv_inputs(30, spatial, batch=batch, seed=3, kernel_size=k)
    idx = idx.numpy().copy()
    idx[7] = idx[2]                       # rows 2 and 7 share a voxel: rep = 2
    idx[11] = idx[2]
    idx[4] = (0, 5, 0, 0)                 # x out of range
    idx[5] = (1, 0, 0, 0)                 # batch out of range
    idx[6] = (0, 0, -1, 0)
    rb = sco.rulebook(idx, spatial, batch, k)
    assert not rb["valid"][[4, 5, 6]].any() and (rb["slot"][[4, 5, 6]] == -1).all()
    s = rb["slot"][2]
    assert rb["slot"][7] == s == rb["slot"][11] and rb["rep"][s] == 2
    out = sco.forward(f.numpy(), w.numpy(), b.numpy(), rb)
    assert (out[[4, 5, 6]] == 0).all()
    assert (out[7] == out[2]).all() and (out[11] == out[2]).all()
    g = np.random.default_rng(0).standard_normal(out.shape)
    gx, gw, gb = sco.backward(f.numpy(), w.numpy(), g, rb)
    assert (gx[[4, 5, 6, 7, 11]] == 0).all() and np.abs(gx[2]).sum() > 0
    np.testing.assert_allclose(gb, g[rb["valid"]].sum(0), rtol=1e-12)
    # features of a non-representative row do not enter the output
    f2 = f.numpy().copy()
    f2[7] += 100.0
    np.testing.assert_array_equal(sco.forward(f2, w.numpy(), b.numpy(), rb), out)


def test_desc_layout_follows_the_header():
    src = open(os.path.join(ROOT, "include", "gf_b200.h")).read()
    body = re.search(r"typedef struct gf_subm_conv_desc \{(.*?)\} gf_subm_conv_desc;", src, flags=re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in filter(None, (d.strip() for d in body.split(";"))):
        first, *rest = decl.split(",")
        names += [first.split()[-1]] + [r.strip() for r in rest]
    assert names == [n for n, _ in _lib.SubmConvDesc._fields_]
    assert all(t is ctypes.c_int32 for _, t in _lib.SubmConvDesc._fields_)


def _desc(**kw):
    d = dict(batch=1, num_rows=1000, X=200, Y=200, Z=16, kernel_size=5, c_in=C, c_out=C)
    d.update(kw)
    return _lib.SubmConvDesc(*[d[n] for n, _ in _lib.SubmConvDesc._fields_])


def test_workspace_query_and_formula():
    L = _lib.lib()
    d = _desc(num_rows=144000)
    nbytes = L.gf_subm_conv_workspace_bytes(ctypes.byref(d))
    V, N, K, P = 200 * 200 * 16, 144000, 125, _lib.GF_SUBM_DW_PIECES
    formula = 8 * V + 4 * N * (8 + 2 * K + 2 * C) + 4 * K * C * C * (1 + P)
    assert formula <= nbytes <= formula + 256 * 1024   # alignment, sort histogram, scan and bias partials
    assert nbytes < 512 * 2 ** 20


BAD_DESCS = [
    (dict(kernel_size=4), _lib.GF_ERR_INVALID_ARG), (dict(kernel_size=7), _lib.GF_ERR_INVALID_ARG),
    (dict(kernel_size=0), _lib.GF_ERR_INVALID_ARG), (dict(c_in=64), _lib.GF_ERR_UNSUPPORTED),
    (dict(c_out=256), _lib.GF_ERR_UNSUPPORTED), (dict(num_rows=0), _lib.GF_ERR_INVALID_ARG),
    (dict(batch=0), _lib.GF_ERR_INVALID_ARG), (dict(Z=-1), _lib.GF_ERR_INVALID_ARG),
    (dict(batch=2, X=2048, Y=2048, Z=256), _lib.GF_ERR_UNSUPPORTED),          # B*X*Y*Z >= 2^31
    (dict(num_rows=2 ** 24), _lib.GF_ERR_UNSUPPORTED),                         # N*C >= 2^31
    (dict(num_rows=17_200_000, kernel_size=5), _lib.GF_ERR_UNSUPPORTED),       # N*k^3 >= 2^31
    (dict(X=2 ** 21, Y=2 ** 21, Z=2 ** 21), _lib.GF_ERR_UNSUPPORTED),          # 2^63 voxels: no 64-bit wrap
    (dict(batch=2 ** 30, X=2 ** 30, Y=2 ** 30, Z=2 ** 30), _lib.GF_ERR_UNSUPPORTED),
]

FAKE = ctypes.c_void_p(1 << 20)   # aligned, never dereferenced: every call below fails before any CUDA call


@pytest.mark.parametrize("kw,code", BAD_DESCS)
def test_bad_desc_is_refused_before_any_cuda_call(kw, code):
    L = _lib.lib()
    d = _desc(**kw)
    assert L.gf_subm_conv_workspace_bytes(ctypes.byref(d)) == 0
    assert L.gf_subm_conv_rulebook(ctypes.byref(d), FAKE, FAKE, 1 << 40, None) == code
    assert L.gf_subm_conv_forward(ctypes.byref(d), FAKE, FAKE, FAKE, None, FAKE, None) == code
    assert L.gf_subm_conv_backward(ctypes.byref(d), FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, None) == code
    assert "subm conv" in L.gf_last_error().decode()


def test_null_and_workspace_refusals():
    L = _lib.lib()
    d = _desc()
    nbytes = L.gf_subm_conv_workspace_bytes(ctypes.byref(d))
    ws = _lib.GF_ERR_WORKSPACE
    inv = _lib.GF_ERR_INVALID_ARG
    assert L.gf_subm_conv_rulebook(None, FAKE, FAKE, nbytes, None) == inv
    assert L.gf_subm_conv_rulebook(ctypes.byref(d), None, FAKE, nbytes, None) == inv
    assert L.gf_subm_conv_rulebook(ctypes.byref(d), ctypes.c_void_p((1 << 20) + 4), FAKE, nbytes, None) == inv
    assert L.gf_subm_conv_rulebook(ctypes.byref(d), FAKE, FAKE, nbytes - 1, None) == ws
    assert L.gf_subm_conv_rulebook(ctypes.byref(d), FAKE, None, nbytes, None) == ws
    assert L.gf_subm_conv_rulebook(ctypes.byref(d), FAKE, ctypes.c_void_p((1 << 20) + 128), nbytes, None) == ws
    assert L.gf_subm_conv_forward(ctypes.byref(d), None, FAKE, FAKE, None, FAKE, None) == ws
    for i in range(3):
        args = [FAKE, FAKE, FAKE]
        args[i] = None
        assert L.gf_subm_conv_forward(ctypes.byref(d), FAKE, args[0], args[1], None, args[2], None) == inv
    assert L.gf_subm_conv_backward(ctypes.byref(d), FAKE, FAKE, FAKE, None, FAKE, FAKE, FAKE, None) == inv
    assert L.gf_subm_conv_backward(ctypes.byref(d), FAKE, FAKE, None, FAKE, FAKE, None, None, None) == inv
    assert L.gf_subm_conv_backward(ctypes.byref(d), FAKE, None, FAKE, FAKE, None, FAKE, None, None) == inv
    assert L.gf_subm_conv_backward(ctypes.byref(d), None, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, None) == ws


def test_cpu_tensors_are_refused():
    from gaussianformer_b200.ops import build_rulebook
    with pytest.raises(RuntimeError, match="CUDA-only"):
        build_rulebook(torch.zeros(4, 4, dtype=torch.int32), (4, 4, 4), 1, 3)


def test_module_state_dict_keys_follow_the_reference():
    from gaussianformer_b200.ops import SparseConv3D
    pc = [-50.0, -50.0, -5.0, 50.0, 50.0, 3.0]
    single = SparseConv3D(128, 128, pc, [0.5] * 3, use_out_proj=True, kernel_size=5, phi_activation="sigmoid",
                          xyz_coordinate="cartesian")
    assert sorted(single.state_dict()) == ["grid_size", "layer.weight", "output_proj.bias", "output_proj.weight",
                                           "pc_range"]
    assert tuple(single.layer.weight.shape) == (128, 5, 5, 5, 128) and single.spatial_shape == (200, 200, 16)
    multi = SparseConv3D(128, 128, pc, [1.0] * 3, kernel_size=5, use_multi_layer=True)
    keys = sorted(multi.state_dict())
    assert keys == sorted(["grid_size", "pc_range"] + [f"layer.{i}.{n}" for i in range(9) if i % 3 != 2
                                                       for n in ("weight", "bias")])
    assert multi.spatial_shape == (100, 100, 8)


def test_torch_reference_equals_the_oracle():
    spatial, batch, k = (7, 6, 5), 2, 3
    f, idx, w, b = make_subm_conv_inputs(160, spatial, batch=batch, seed=4, kernel_size=k, invalid=3, duplicates_of=7)
    rb = sco.rulebook(idx.numpy(), spatial, batch, k)
    g = np.random.default_rng(1).standard_normal((f.shape[0], C))
    ref = [sco.forward(f.numpy(), w.numpy(), b.numpy(), rb)] + list(sco.backward(f.numpy(), w.numpy(), g, rb))
    mine = sco.torch_reference(f.numpy(), w.numpy(), b.numpy(), g, rb, torch.float64, "cpu")
    for a, e in zip(mine, ref):
        np.testing.assert_allclose(a, e, rtol=1e-12, atol=1e-12)


def test_misaligned_tensors_are_refused_before_any_cuda_call():
    L = _lib.lib()
    d = _desc()
    inv = _lib.GF_ERR_INVALID_ARG
    odd = ctypes.c_void_p((1 << 20) + 4)
    assert L.gf_subm_conv_forward(ctypes.byref(d), FAKE, odd, FAKE, None, FAKE, None) == inv
    assert L.gf_subm_conv_forward(ctypes.byref(d), FAKE, FAKE, FAKE, None, odd, None) == inv
    assert "16-byte aligned" in L.gf_last_error().decode()
    assert L.gf_subm_conv_backward(ctypes.byref(d), FAKE, odd, FAKE, FAKE, FAKE, FAKE, FAKE, None) == inv
    assert L.gf_subm_conv_backward(ctypes.byref(d), FAKE, FAKE, FAKE, odd, FAKE, FAKE, FAKE, None) == inv
    assert L.gf_subm_conv_backward(ctypes.byref(d), FAKE, FAKE, FAKE, FAKE, odd, FAKE, FAKE, None) == inv


def test_module_grid_follows_loaded_buffers():
    from gaussianformer_b200.ops import SparseConv3D
    pc = [-50.0, -50.0, -5.0, 50.0, 50.0, 3.0]
    coarse = SparseConv3D(128, 128, pc, [1.0] * 3, kernel_size=3)
    fine = SparseConv3D(128, 128, [-40.0, -40.0, -1.0, 40.0, 40.0, 5.4], [0.5] * 3, kernel_size=3)
    assert coarse.spatial_shape == (100, 100, 8) and fine.spatial_shape == (160, 160, 12)
    coarse.load_state_dict(fine.state_dict(), strict=True)
    assert coarse.spatial_shape == (160, 160, 12)
