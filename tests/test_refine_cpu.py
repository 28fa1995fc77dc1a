"""CPU-only: the fp64 oracle of the Gaussian refinement (refine_oracle) against the reference's lines
(refine_module.py:72-123, refine_module_v2.py:64-108) restated in fp64 torch, its gradients against fp64 autograd
through those lines, for the three shipped setups, the other option values and crafted edges; the gf_refine_desc
layout, the argument checks of gf_gaussian_refine / _backward (before any CUDA call) and reference-shaped state dicts."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import refine_oracle as ro
from gaussianformer_b200 import _lib
from gaussianformer_b200.csrc import build
from gaussianformer_b200.ops import SparseGaussian3DRefinementModule, SparseGaussian3DRefinementModuleV2
from gaussianformer_b200.synthetic import REFINE_CONFIGS, make_refine_inputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIGS = list(REFINE_CONFIGS)


def oracle_cfg(d, **changes):
    """the oracle's cfg of make_refine_inputs' dict d, with option values changed"""
    cfg = dict(d["config"], variant=d["variant"])
    cfg.update(changes)
    return cfg


def reshape_inputs(d, cfg):
    """out and anchor of d cut or padded to cfg's out_dim (the anchor keeps d's width unless it is narrower)"""
    D = 10 + int(cfg["include_opa"]) + cfg["semantic_dim"]
    out = d["out"]
    if out.shape[-1] < D:
        out = torch.cat([out, torch.randn(*out.shape[:2], D - out.shape[-1], generator=torch.Generator().manual_seed(1))],
                        -1)
    return out[..., :D].contiguous(), d["anchor"]


def _case(config, seed=0, A=400, B=2, **changes):
    d = make_refine_inputs(config, batch=B, num_anchor=A, seed=seed)
    cfg = oracle_cfg(d, **changes)
    out, anchor = reshape_inputs(d, cfg)
    return out, anchor, cfg


OPTIONS = {
    "softmax": dict(semantics_activation="softmax"),
    "no_opacity": dict(include_opa=False),
    "no_semantics": dict(semantic_dim=0, semantics=False),
    "prefix_0": dict(refine_manual=[]),
    "prefix_10": dict(refine_manual=list(range(10))),
    "prefix_28": dict(refine_manual=list(range(28))),
    "free_xyz": dict(restrict_xyz=False),
}


def _crafted():
    """logits exactly at and just beyond +-9.21f, softplus inputs exactly 20 and beyond, a zero quaternion and one of
    norm below 1e-12; V1 without the restriction and the residual, so the crafted logits reach the clamps as written"""
    out, anchor, cfg = _case("gs25600_solid", seed=3, A=8, B=1, restrict_xyz=False, refine_manual=[])
    c = float(np.float32(9.21))
    beyond = float(np.nextafter(np.float32(9.21), np.float32(10)))
    out[0, 0, [0, 1, 3, 4, 10]] = torch.tensor([c, -c, c, -c, c])
    out[0, 1, [0, 2, 3, 10]] = torch.tensor([beyond, -beyond, beyond, -beyond])
    out[0, 2, 6:10] = torch.tensor([1e-14, -2e-14, 3e-14, 0.5e-14])
    out[0, 3, 6:10] = 0.0
    out[0, 4, 11:14] = torch.tensor([20.0, float(np.nextafter(np.float32(20), np.float32(30))), 19.5])
    return out, anchor, cfg


CASES = {c: (lambda c=c: _case(c, 1)) for c in CONFIGS}
CASES.update({k: (lambda k=k: _case("gs25600_solid", 2, **v)) for k, v in OPTIONS.items()})
CASES["v2_softmax"] = lambda: _case("prob_gs25600", 4, semantics_activation="softmax")
CASES["v2_softplus_no_opacity"] = lambda: _case("prob_gs25600", 5, semantics_activation="softplus", include_opa=False)
CASES["crafted"] = _crafted


def _grads(out, anchor, cfg, seed=4):
    """a seeded fp32 gradient for every output the variant has"""
    _, g = ro.reference_refine(out.double(), anchor.double(), cfg)
    gen = torch.Generator().manual_seed(seed)
    shapes = dict(new_anchor=out.shape[-1], **{k: v.shape[-1] for k, v in g.items()})
    return {k: torch.randn(*out.shape[:2], n, generator=gen) for k, n in shapes.items()}


def _reference_outputs(out, anchor, cfg):
    na, g = ro.reference_refine(out, anchor, cfg)
    return dict(new_anchor=na, **g)


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_forward_matches_the_reference_lines_in_fp64(case):
    out, anchor, cfg = CASES[case]()
    got, got_abs = ro.refine(out.numpy(), anchor.numpy(), cfg)
    want = _reference_outputs(out.double(), anchor.double(), cfg)
    assert set(got) == set(want)
    for k, w in want.items():
        w = w.numpy()
        assert got[k].shape == w.shape, k
        assert np.isfinite(w).all(), k
        assert (np.abs(got[k] - w) <= 1e-12 * np.maximum(got_abs[k], np.abs(w))).all(), k


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_backward_matches_fp64_autograd(case):
    out, anchor, cfg = CASES[case]()
    o = out.double().requires_grad_()
    a = anchor.double().requires_grad_()
    outs = _reference_outputs(o, a, cfg)
    g = _grads(out, anchor, cfg)
    torch.autograd.backward([outs[k] for k in outs], [g[k].double() for k in outs])
    go, goa, ga, gaa = ro.refine_backward(out.numpy(), anchor.numpy(), cfg, {k: v.numpy() for k, v in g.items()})
    a_grad = np.zeros(anchor.shape) if a.grad is None else a.grad.numpy()        # prefix 0: the anchor is not read
    for what, got, got_abs, want in (("out", go, goa, o.grad.numpy()), ("anchor", ga, gaa, a_grad)):
        assert np.isfinite(want).all(), what
        assert (np.abs(got - want) <= 1e-12 * np.maximum(np.abs(want), got_abs)).all(), what
    r = 3 if cfg["variant"] == "v2" else len(cfg.get("refine_manual") or [])
    assert (ga[..., r:] == 0).all()
    if case == "crafted":
        c = go[0]
        through = c - g["new_anchor"].double().numpy()[0]            # the part that does not skip the activations
        assert (through[0, [0, 1, 3, 4, 10]] != 0).all()             # at +-9.21f the gradient passes
        assert (through[1, [0, 2, 3, 10]] == 0).all()                # beyond it it does not
        assert np.abs(c[2, 6:10]).max() > 1e6                        # norm below 1e-12: divided by the epsilon
        assert np.isfinite(c[3, 6:10]).all() and np.abs(c[3, 6:10]).max() > 1e6
        sig20 = 1 / (1 + np.exp(-20.0))
        gsem = g["semantics"].double().numpy()[0, 4]
        np.testing.assert_allclose(c[4, 11:14] - g["new_anchor"].double().numpy()[0, 4, 11:14],
                                   gsem[:3] * [sig20, 1.0, 1 / (1 + np.exp(-19.5))], rtol=1e-14)


def test_inverse_sigmoid_clamp_at_its_fp32_bounds():
    """t exactly at the fp32 bounds passes the gradient, one fp64 step beyond does not (torch.clamp's backward)"""
    t = np.array([ro.INV_LO, ro.INV_HI, np.nextafter(ro.INV_LO, 0), np.nextafter(ro.INV_HI, 1), 0.3])
    tt = torch.tensor(t, requires_grad=True)
    ro.safe_inverse_sigmoid(tt).sum().backward()
    v, dv, _ = ro.sinv(t)
    np.testing.assert_allclose(v, ro.safe_inverse_sigmoid(torch.tensor(t)).numpy(), rtol=1e-15)
    np.testing.assert_allclose(dv, tt.grad.numpy(), rtol=1e-14)
    assert (dv[:2] > 0).all() and (dv[2:4] == 0).all()


def test_v2_faces_saturate_the_inverse_sigmoid():
    """the synthetic inputs push anchors past the pc-range faces: V2's clamp blocks their xyz gradient"""
    out, anchor, cfg = _case("prob_gs25600", 6, A=4000, B=1)
    g = {k: v.numpy() for k, v in _grads(out, anchor, cfg).items() if k in ("new_anchor", "means")}
    go, _, ga, _ = ro.refine_backward(out.numpy(), anchor.numpy(), cfg, g)
    val, _ = ro.refine(out.numpy(), anchor.numpy(), cfg)
    sat = np.abs(val["new_anchor"][..., :3]) > 9.2
    assert sat.sum() > 20
    assert (go[..., :3][sat] == 0).all() and (ga[..., :3][sat] == 0).all()
    assert (go[..., :3][~sat] != 0).mean() > 0.9


# ------------------------------------------------------------------------------------------------ C ABI and module
@pytest.fixture(scope="module")
def L():
    build.build()
    return _lib.lib()


def _header_fields(src, name):
    body = re.search(r"typedef struct " + name + r" \{(.*?)\} " + name + ";", src, flags=re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in body.split(";"):
        decl = re.sub(r"^const\s+", "", decl.strip())
        if decl:
            ctype, rest = decl.split(None, 1)
            fields += [(n.strip().lstrip("*").split("[")[0], ctype, int(n.split("[")[1].rstrip("]")) if "[" in n else 1)
                       for n in rest.split(",")]
    return fields


def test_refine_structs_follow_the_header():
    src = open(os.path.join(ROOT, "include", "gf_b200.h")).read()
    want = [(n, {"int32_t": ctypes.c_int32, "float": ctypes.c_float}[t], k)
            for n, t, k in _header_fields(src, "gf_refine_desc")]
    got = [(name, t._type_ if hasattr(t, "_length_") else t, getattr(t, "_length_", 1))
           for name, t in _lib.RefineDesc._fields_]
    assert got == want
    assert ctypes.sizeof(_lib.RefineDesc) == 4 * (10 + 11)
    for name, cls in (("gf_refine_outputs", _lib.RefineOutputs), ("gf_refine_grads", _lib.RefineGrads)):
        assert [n for n, _, _ in _header_fields(src, name)] == [n for n, _ in cls._fields_] == list(ro.OUTPUTS)
    assert _lib.GF_REFINE_MAX_SEMANTICS == int(re.search(r"#define GF_REFINE_MAX_SEMANTICS (\d+)", src).group(1))


FAKE = 256                                               # never dereferenced: every call below stops at a check


def _desc(variant=0, B=1, A=4, S=17, opa=1, Da=28, r=3, restrict=1, act=2):
    d = _lib.RefineDesc()
    d.variant, d.batch, d.num_anchors, d.out_dim, d.anchor_dim = variant, B, A, 10 + opa + S, Da
    d.refine_prefix, d.restrict_xyz, d.include_opa, d.semantic_dim, d.semantics_act = r, restrict, opa, S, act
    return d


def _outputs(**null):
    return _lib.RefineOutputs(**{n: (None if n in null else FAKE) for n in ro.OUTPUTS})


def _fwd(L, d, out=FAKE, anchor=FAKE, outputs="all"):
    o = _outputs() if outputs == "all" else outputs
    return L.gf_gaussian_refine(ctypes.byref(d) if d is not None else None, out, anchor,
                                ctypes.byref(o) if o is not None else None, None)


def _bwd(L, d, out=FAKE, anchor=FAKE, go=FAKE, ga=FAKE):
    g = _lib.RefineGrads()
    return L.gf_gaussian_refine_backward(ctypes.byref(d) if d is not None else None, out, anchor, ctypes.byref(g), go,
                                         ga, None)


REFUSED = {
    "null desc": (None, _lib.GF_ERR_INVALID_ARG, b"desc is NULL"),
    "negative batch": (dict(B=-1), _lib.GF_ERR_INVALID_ARG, b"negative size"),
    "negative anchors": (dict(A=-1), _lib.GF_ERR_INVALID_ARG, b"negative size"),
    "negative anchor_dim": (dict(Da=-1, r=0), _lib.GF_ERR_INVALID_ARG, b"negative size"),
    "negative prefix": (dict(r=-1), _lib.GF_ERR_INVALID_ARG, b"negative size"),
    "unknown variant": (dict(variant=2), _lib.GF_ERR_INVALID_ARG, b"unknown variant"),
    "unknown activation": (dict(act=3), _lib.GF_ERR_INVALID_ARG, b"semantics activation"),
    "include_opa 2": (dict(opa=2), _lib.GF_ERR_INVALID_ARG, b"must be 0 or 1"),
    "prefix above anchor_dim": (dict(Da=2), _lib.GF_ERR_INVALID_ARG, b"exceeds min"),
    "prefix above out_dim": (dict(Da=40, r=29), _lib.GF_ERR_INVALID_ARG, b"exceeds min"),
    "v2 with a prefix": (dict(variant=1, restrict=0), _lib.GF_ERR_INVALID_ARG, b"V1 fields"),
    "v2 with restrict_xyz": (dict(variant=1, r=0), _lib.GF_ERR_INVALID_ARG, b"V1 fields"),
    "v2 short anchor": (dict(variant=1, r=0, restrict=0, Da=2), _lib.GF_ERR_INVALID_ARG, b"anchor_dim=2"),
    "wide semantics": (dict(S=33), _lib.GF_ERR_UNSUPPORTED, b"compiled maximum"),
    "2^31 entries": (dict(A=(1 << 31) // 28 + 1), _lib.GF_ERR_UNSUPPORTED, b"2^31"),
    "2^31 anchor entries": (dict(A=(1 << 31) // 64 + 1, Da=64), _lib.GF_ERR_UNSUPPORTED, b"2^31"),
    "2^31 anchors": (dict(B=1 << 20, A=1 << 20), _lib.GF_ERR_UNSUPPORTED, b"2^31"),
}


@pytest.mark.parametrize("case", list(REFUSED))
def test_bad_descriptors_are_refused(L, case):
    kw, code, msg = REFUSED[case]
    d = None if kw is None else _desc(**kw)
    for call in (_fwd, _bwd):
        assert call(L, d) == code, case
        assert msg in L.gf_last_error(), L.gf_last_error()


def test_out_dim_must_match_the_options(L):
    d = _desc()
    d.out_dim = 27
    for call in (_fwd, _bwd):
        assert call(L, d) == _lib.GF_ERR_INVALID_ARG
        assert b"expected 10 + include_opa + semantic_dim = 28" in L.gf_last_error()


@pytest.mark.parametrize("field", ["out", "anchor"])
def test_null_inputs_are_refused_for_non_empty_work(L, field):
    for call in (_fwd, _bwd):
        assert call(L, _desc(), **{field: None}) == _lib.GF_ERR_INVALID_ARG
        assert b"NULL" in L.gf_last_error()


@pytest.mark.parametrize("variant,field", [(0, n) for n in ro.OUTPUTS[:6]] + [(1, n) for n in ro.OUTPUTS[6:]])
def test_null_outputs_are_refused_for_non_empty_work(L, variant, field):
    d = _desc(variant, r=0, restrict=0) if variant else _desc()
    assert _fwd(L, d, outputs=_outputs(**{field: 1})) == _lib.GF_ERR_INVALID_ARG
    assert field.encode() in L.gf_last_error()
    assert _fwd(L, d, outputs=None) == _lib.GF_ERR_INVALID_ARG


@pytest.mark.parametrize("field", ["go", "ga"])
def test_backward_null_gradients_are_refused_for_non_empty_work(L, field):
    assert _bwd(L, _desc(), **{field: None}) == _lib.GF_ERR_INVALID_ARG
    assert b"NULL" in L.gf_last_error()


def test_empty_work_needs_no_pointers(L):
    for d in (_desc(B=0), _desc(A=0), _desc(1, A=0, r=0, restrict=0)):
        assert _fwd(L, d, None, None, None) == _lib.GF_OK
        assert _bwd(L, d, None, None, None, None) == _lib.GF_OK


def reference_shaped_state_dict(embed_dims, out_dim, gen):
    """the state dict of the reference modules: linear_relu_ln(embed_dims, 2, 2), Linear, mmcv Scale"""
    sd = {}
    for i in (0, 2, 5, 7):
        sd[f"layers.{i}.weight"] = torch.randn(embed_dims, embed_dims, generator=gen)
        sd[f"layers.{i}.bias"] = torch.randn(embed_dims, generator=gen)
    for i in (4, 9):
        sd[f"layers.{i}.weight"] = torch.rand(embed_dims, generator=gen)
        sd[f"layers.{i}.bias"] = torch.randn(embed_dims, generator=gen)
    sd["layers.10.weight"] = torch.randn(out_dim, embed_dims, generator=gen)
    sd["layers.10.bias"] = torch.randn(out_dim, generator=gen)
    sd["layers.11.scale"] = torch.rand(out_dim, generator=gen)
    return sd


@pytest.mark.parametrize("config", CONFIGS)
def test_modules_load_a_reference_state_dict_strictly(config):
    d = make_refine_inputs(config, num_anchor=4)
    cls = SparseGaussian3DRefinementModuleV2 if d["variant"] == "v2" else SparseGaussian3DRefinementModule
    m = cls(phi_activation="sigmoid", xyz_coordinate="cartesian", **d["config"])
    sd = reference_shaped_state_dict(128, m.output_dim, torch.Generator().manual_seed(0))
    assert set(m.state_dict()) == set(sd)
    m.load_state_dict(sd, strict=True)
    assert torch.equal(m.layers[11].scale, sd["layers.11.scale"])
    x = torch.randn(2, 3, 128)
    assert torch.equal(m.layers(x), m.layers[11](m.layers[10](m.layers[:10](x))))
    assert m.output_dim == d["out"].shape[-1] == 10 + int(m.include_opa) + m.semantic_dim
    if d["variant"] == "v2":
        assert "unit_xyz" not in m.state_dict() and m.unit_xyz.dtype == torch.float32
        assert m.unit_xyz.tolist() == d["config"]["unit_xyz"]
    else:
        assert m.refine_state == [0, 1, 2] and m.unit_sigmoid[2] == 4 * 1.0 / 8.0 * d["config"]["unit_xyz"][2]


def test_modules_refuse_other_activations_and_bad_prefixes():
    d = make_refine_inputs("gs25600_solid", num_anchor=4)
    for cls, kw in ((SparseGaussian3DRefinementModule, d["config"]),
                    (SparseGaussian3DRefinementModuleV2, make_refine_inputs("prob_gs25600", num_anchor=4)["config"])):
        for bad in ({"xyz_activation": "none"}, {"scale_activation": "exp"}):
            with pytest.raises(ValueError, match="sigmoid"):
                cls(**dict(kw, **bad))
    with pytest.raises(AssertionError):
        SparseGaussian3DRefinementModule(**dict(d["config"], refine_manual=[0, 2]))
