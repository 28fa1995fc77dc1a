"""CPU-only: the fp64 oracle of the anchor key-point generator (daf_anchor_oracle) against the reference generator
(deformable_module.py:51-90, get_rotation_matrix, safe_sigmoid) restated in fp64 torch, its gradients against fp64
autograd through those lines, crafted edge cases, the gf_daf_kps_desc layout, the argument checks of
gf_daf_anchor_key_points / _backward (before any CUDA call) and the module's reference-shaped state dict."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import daf_anchor_oracle as ao
from gaussianformer_b200 import _lib
from gaussianformer_b200.csrc import build
from gaussianformer_b200.ops import SparseGaussian3DKeyPointsGenerator
from gaussianformer_b200.synthetic import make_anchor_kp_inputs
from daf_anchor_oracle import reference_generator

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _case(config, seed=0, A=300, B=2):
    d = make_anchor_kp_inputs(config, batch=B, num_anchor=A, seed=seed)
    return d["anchor"], d["logits"], d["fix_scale"], d["pc_range"], d["scale_range"], d["learnable_fixed_scale"]


def _crafted():
    """anchor and learnable logits at and beyond the clamp, a quaternion of norm below 1e-12, a NaN-free rest"""
    anchor, logits, fix, pcr, scr, lfs = _case("prob_gs6400", seed=3, A=8, B=1)
    c = np.float32(9.21)
    anchor[0, 0, 0], anchor[0, 0, 1], anchor[0, 0, 3], anchor[0, 0, 4] = float(c), -float(c), float(c), -float(c)
    anchor[0, 1, 0] = float(np.nextafter(c, np.float32(10)))
    anchor[0, 1, 3] = -float(np.nextafter(c, np.float32(10)))
    anchor[0, 1, 2] = 20.0
    anchor[0, 2, 6:10] = torch.tensor([1e-14, -2e-14, 3e-14, 0.5e-14])
    anchor[0, 3, 6:10] = torch.tensor([0.0, 0.0, 0.0, 0.0])
    logits[0, 0, 0] = torch.tensor([float(c), -float(c), 30.0])
    logits[0, 1, 1] = torch.tensor([-float(np.nextafter(c, np.float32(10))), 0.0, 1e-7])
    return anchor, logits, fix, pcr, scr, lfs


CASES = {"gs25600_solid": lambda: _case("gs25600_solid", 1), "prob_gs6400": lambda: _case("prob_gs6400", 2),
         "crafted": _crafted}


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_forward_matches_the_reference_lines_in_fp64(case):
    anchor, logits, fix, pcr, scr, lfs = CASES[case]()
    _, got, got_abs = ao.key_points(anchor.numpy(), fix.numpy(), logits.numpy(), pcr, scr, lfs)
    want = reference_generator(anchor.double(), logits.double(), fix, pcr, scr, lfs).numpy()
    assert np.isfinite(want).all()
    assert (np.abs(got - want) <= 1e-12 * got_abs).all()


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_backward_matches_fp64_autograd(case):
    anchor, logits, fix, pcr, scr, lfs = CASES[case]()
    a = anchor.double().requires_grad_()
    lg = logits.double().requires_grad_()
    kp = reference_generator(a, lg, fix, pcr, scr, lfs)
    g = torch.randn(kp.shape, generator=torch.Generator().manual_seed(4)).float()
    kp.backward(g.double())
    ga, ga_abs, gl, gl_abs = ao.key_points_backward(anchor.numpy(), fix.numpy(), logits.numpy(), pcr, scr, lfs,
                                                    g.numpy())
    for what, got, got_abs, want in (("anchor", ga, ga_abs, a.grad.numpy()), ("logits", gl, gl_abs, lg.grad.numpy())):
        assert np.isfinite(want).all(), what
        assert (np.abs(got - want) <= 1e-12 * np.maximum(np.abs(want), got_abs)).all(), what
    assert (ga[..., 10:] == 0).all()
    if case == "crafted":
        c = ga[0]
        assert (c[0, [0, 1, 3, 4]] != 0).all()                       # at +-9.21f the gradient passes
        assert (c[1, [0, 2, 3]] == 0).all()                         # beyond it it does not
        assert (gl[0, 0, 0, :2] != 0).all() and gl[0, 0, 0, 2] == 0 and gl[0, 1, 1, 0] == 0
        assert np.abs(c[2, 6:10]).max() > 1e6                       # norm below 1e-12: divided by the epsilon
        assert np.isfinite(c[3, 6:10]).all()


def test_no_learnable_points_and_the_default_fix_scale():
    anchor, _, _, pcr, scr, _ = _case("gs25600_solid", 5, A=50)
    fix = np.zeros((1, 3), np.float32)                               # fix_scale=None: ((0, 0, 0),)
    kp, kp64, _ = ao.key_points(anchor.numpy(), fix, None, pcr, scr)
    want = reference_generator(anchor.double(), None, fix, pcr, scr, 1.0).numpy()
    np.testing.assert_allclose(kp64, want, rtol=1e-13)
    assert kp.shape == (2, 50, 1, 3)
    g = np.ones((2, 50, 1, 3), np.float32)
    ga, _, gl, _ = ao.key_points_backward(anchor.numpy(), fix, None, pcr, scr, 1.0, g)
    assert gl is None and (ga[..., 3:10] == 0).all() and (ga[..., :3] != 0).all()   # a zero offset moves nothing


# ------------------------------------------------------------------------------------------------ C ABI and module
@pytest.fixture(scope="module")
def L():
    build.build()
    return _lib.lib()


def test_kps_desc_layout_follows_the_header():
    src = open(os.path.join(ROOT, "include", "gf_b200.h")).read()
    body = re.search(r"typedef struct gf_daf_kps_desc \{(.*?)\} gf_daf_kps_desc;", src, flags=re.S).group(1)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            ctype, first = decl.split(None, 1)
            fields += [(n.strip().split("[")[0], ctype, int(n.split("[")[1].rstrip("]")) if "[" in n else 1)
                       for n in first.split(",")]
    want = [(name, {"int32_t": ctypes.c_int32, "float": ctypes.c_float}[ctype], n) for name, ctype, n in fields]
    got = [(name, t._type_ if hasattr(t, "_length_") else t, getattr(t, "_length_", 1))
           for name, t in _lib.DafKpsDesc._fields_]
    assert got == want
    assert ctypes.sizeof(_lib.DafKpsDesc) == 4 * (5 + 9)


FAKE = ctypes.c_void_p(256)                              # never dereferenced: every call below stops at a check


def _desc(B=1, A=4, D=28, Kf=7, Kl=2):
    d = _lib.DafKpsDesc()
    d.batch, d.num_anchors, d.anchor_dim, d.num_fixed, d.num_learnable = B, A, D, Kf, Kl
    return d


def _fwd(L, d, anchor=FAKE, fix=FAKE, logits=FAKE, kp=FAKE):
    return L.gf_daf_anchor_key_points(ctypes.byref(d) if d is not None else None, anchor, fix, logits, kp, None)


def _bwd(L, d, anchor=FAKE, fix=FAKE, logits=FAKE, gkp=FAKE, ga=FAKE, gl=FAKE):
    return L.gf_daf_anchor_key_points_backward(ctypes.byref(d) if d is not None else None, anchor, fix, logits, gkp,
                                               ga, gl, None)


@pytest.mark.parametrize("field", ["batch", "num_anchors", "anchor_dim", "num_fixed", "num_learnable"])
def test_negative_sizes_are_refused(L, field):
    d = _desc()
    setattr(d, field, -1)
    for call in (_fwd, _bwd):
        assert call(L, d) == _lib.GF_ERR_INVALID_ARG
        assert b"negative size" in L.gf_last_error()


def test_short_anchors_no_key_points_and_null_desc_are_refused(L):
    for call in (_fwd, _bwd):
        assert call(L, _desc(D=9)) == _lib.GF_ERR_INVALID_ARG
        assert b"anchor_dim" in L.gf_last_error()
        assert call(L, _desc(Kf=0, Kl=0)) == _lib.GF_ERR_INVALID_ARG
        assert b"num_fixed + num_learnable" in L.gf_last_error()
        assert call(L, None) == _lib.GF_ERR_INVALID_ARG
        assert b"desc is NULL" in L.gf_last_error()


@pytest.mark.parametrize("field", ["anchor", "fix", "logits", "kp"])
def test_null_pointers_are_refused_for_non_empty_work(L, field):
    assert _fwd(L, _desc(), **{field: None}) == _lib.GF_ERR_INVALID_ARG
    assert b"NULL" in L.gf_last_error()


@pytest.mark.parametrize("field", ["anchor", "fix", "logits", "gkp", "ga", "gl"])
def test_backward_null_pointers_are_refused_for_non_empty_work(L, field):
    assert _bwd(L, _desc(), **{field: None}) == _lib.GF_ERR_INVALID_ARG
    assert b"NULL" in L.gf_last_error()


def test_empty_work_needs_no_pointers(L):
    assert _fwd(L, _desc(B=0), None, None, None, None) == _lib.GF_OK
    assert _fwd(L, _desc(A=0, Kf=0, Kl=0), None, None, None, None) == _lib.GF_OK
    assert _bwd(L, _desc(A=0), None, None, None, None, None, None) == _lib.GF_OK


def test_more_than_2_31_key_points_are_refused(L):
    A = (1 << 31) // 9 + 1                               # B * A * K >= 2^31
    for call in (_fwd, _bwd):
        assert call(L, _desc(A=A)) == _lib.GF_ERR_UNSUPPORTED
        assert b"2^31" in L.gf_last_error()
        assert call(L, _desc(B=3, A=A // 3 + 1)) == _lib.GF_ERR_UNSUPPORTED
        assert call(L, _desc(B=1 << 20, A=1 << 20)) == _lib.GF_ERR_UNSUPPORTED     # B * A itself past 2^31


def reference_shaped_state_dict(embed_dims, Kl):
    """the state dict of the reference module: learnable_fc only (its fix_scale is a numpy attribute)"""
    return {"learnable_fc.weight": torch.randn(3 * Kl, embed_dims), "learnable_fc.bias": torch.randn(3 * Kl)}


@pytest.mark.parametrize("Kl,lfs", [(2, 1), (6, 6.0)])
def test_module_loads_a_reference_state_dict_strictly(Kl, lfs):
    m = SparseGaussian3DKeyPointsGenerator(embed_dims=128, phi_activation="sigmoid", xyz_coordinate="cartesian",
                                           num_learnable_pts=Kl, learnable_fixed_scale=lfs,
                                           fix_scale=[[0, 0, 0], [0.45, 0, 0], [-0.45, 0, 0], [0, 0.45, 0],
                                                      [0, -0.45, 0], [0, 0, 0.45], [0, 0, -0.45]],
                                           pc_range=[-50.0, -50.0, -5.0, 50.0, 50.0, 3.0], scale_range=[0.08, 0.64])
    sd = reference_shaped_state_dict(128, Kl)
    assert set(m.state_dict()) == set(sd)
    m.load_state_dict(sd, strict=True)
    assert torch.equal(m.learnable_fc.weight, sd["learnable_fc.weight"])
    assert m.num_pts == 7 + Kl and m.fix_scale.dtype == torch.float32 and m.fix_scale.shape == (7, 3)
    m.init_weight()
    assert (m.learnable_fc.bias == 0).all() and m.learnable_fc.weight.abs().max() <= (6 / (128 + 3 * Kl)) ** 0.5


def test_module_defaults_and_activations():
    m = SparseGaussian3DKeyPointsGenerator(pc_range=[0] * 6, scale_range=[0, 1])
    assert m.num_pts == 1 and m.state_dict() == {} and m.fix_scale.tolist() == [[0.0, 0.0, 0.0]]
    for kw in ({"xyz_activation": "none"}, {"scale_activation": "exp"}):
        with pytest.raises(ValueError, match="sigmoid"):
            SparseGaussian3DKeyPointsGenerator(pc_range=[0] * 6, scale_range=[0, 1], **kw)
