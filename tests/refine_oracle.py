"""fp64 numpy oracle of the Gaussian refinement (``gf_gaussian_refine`` / ``_backward``), and the reference's lines
restated in torch.

``SparseGaussian3DRefinementModule.forward`` (model/encoder/gaussian_encoder/refine_module.py:72-123) and
``SparseGaussian3DRefinementModuleV2.forward`` (refine_module_v2.py:64-108) after ``layers``, with ``safe_sigmoid`` /
``safe_inverse_sigmoid`` (model/utils/safe_ops.py) and ``cartesian`` / ``reverse_cartesian``
(model/encoder/gaussian_encoder/utils.py:26-47), in fp64 on the fp32 inputs with the constants the reference's fp32
tensors hold (9.21f, 1e-12f, the fp32 ranges and units, the fp32 inverse-sigmoid bounds).  The contract is stated in
include/gf_b200.h.

Next to every value the oracle returns the sum of the absolute values of the terms that make it (``abs``), carried
through every step: the scale of the rounding errors any fp64 evaluation of it makes.  Where a value is far below that
scale (cancellation), the GPU tests hold it to an absolute bound relative to ``abs``, as test_daf_anchor_kp_gpu.py
does.  ``cfg`` is the ``config`` dict of ``synthetic.make_refine_inputs`` plus ``variant``.
"""
import numpy as np
import torch
import torch.nn.functional as F

CLAMP = float(np.float32(9.21))              # safe_sigmoid's bound as an fp32 tensor holds it
EPS = float(np.float32(1e-12))               # F.normalize's epsilon, likewise
INV_LO = float(np.float32(1 - 0.9999))       # safe_inverse_sigmoid's bounds, likewise
INV_HI = float(np.float32(0.9999))
F32 = lambda v: float(np.float32(v))         # noqa: E731
OUTPUTS = ("new_anchor", "means", "scales", "rotations", "opacities", "semantics", "original_means", "delta_means")


def _f64(a):
    return np.asarray(a, np.float32).astype(np.float64)


def sig(v):
    """(sigmoid of the clamped logit, its derivative with the clamp's gate: bounds pass, outside and NaN do not)"""
    with np.errstate(invalid="ignore", over="ignore"):
        s = 1.0 / (1.0 + np.exp(-np.clip(v, -CLAMP, CLAMP)))
        return s, np.where((v >= -CLAMP) & (v <= CLAMP), s * (1.0 - s), 0.0)


def sinv(t):
    """(safe_inverse_sigmoid of t, its derivative with the clamp's gate, the clamped t)"""
    tc = np.clip(t, INV_LO, INV_HI)
    return np.log(tc / (1.0 - tc)), np.where((t >= INV_LO) & (t <= INV_HI), 1.0 / (tc * (1.0 - tc)), 0.0), tc


def constants(cfg):
    pc, v2 = cfg["pc_range"], cfg["variant"] == "v2"
    lo = np.array([F32(pc[i]) for i in range(3)])
    ext = np.array([F32(float(pc[i + 3]) - float(pc[i])) for i in range(3)])
    if v2:
        unit = np.array([F32(u) for u in cfg["unit_xyz"]])
    elif cfg.get("restrict_xyz"):
        unit = np.array([F32(4 * float(cfg["unit_xyz"][i]) / (float(pc[i + 3]) - float(pc[i]))) for i in range(3)])
    else:
        unit = None
    sr = cfg["scale_range"]
    return lo, ext, unit, F32(sr[0]), F32(float(sr[1]) - float(sr[0]))


def _prefix(cfg):
    return 0 if cfg["variant"] == "v2" else len(cfg.get("refine_manual") or [])


def _frame(out, anchor, cfg):
    o, a = _f64(out), _f64(anchor)
    lo, ext, unit, slo, sext = constants(cfg)
    opa = int(cfg["include_opa"])
    f = dict(lo=lo, ext=ext, unit=unit, slo=slo, sext=sext, opa=opa, s0=10 + opa, D=o.shape[-1], r=_prefix(cfg))
    x, xa = o.copy(), np.abs(o)
    if cfg["variant"] == "v1":
        if unit is not None:
            f["sr"], f["dsr"] = sig(o[..., :3])
            x[..., :3] = (2 * f["sr"] - 1) * unit
            xa[..., :3] = (2 * f["sr"] + 1) * np.abs(unit)
        r = f["r"]
        x[..., :r] += a[..., :r]
        xa[..., :r] += np.abs(a[..., :r])
    else:
        f["sr"], f["dsr"] = sig(o[..., :3])
        f["delta"], f["delta_abs"] = (2 * f["sr"] - 1) * unit, (2 * f["sr"] + 1) * np.abs(unit)
        f["sa"], f["dsa"] = sig(a[..., :3])
        f["orig"], f["orig_abs"] = f["sa"] * ext + lo, f["sa"] * ext + np.abs(lo)
        t = ((f["orig"] + f["delta"]) - lo) / ext
        t_abs = (f["orig_abs"] + f["delta_abs"] + np.abs(lo)) / ext
        axyz, f["dinv"], tc = sinv(t)
        x[..., :3] = axyz
        xa[..., :3] = np.abs(axyz) + np.where(f["dinv"] > 0, t_abs / (tc * (1 - tc)), 0.0)
    f["x"], f["xa"] = x, xa
    f["sm"], f["dsm"] = sig(x[..., :3])
    f["ss"], f["dss"] = sig(x[..., 3:6])
    q = x[..., 6:10]
    n = np.sqrt((q * q).sum(-1, keepdims=True))
    f["inv"] = 1.0 / np.maximum(n, EPS)
    f["below"] = n < EPS
    f["rot"] = q * f["inv"]
    f["rot_abs"] = xa[..., 6:10] * f["inv"] + np.abs(f["rot"]) * (xa[..., 6:10] * np.abs(q)).sum(-1, keepdims=True) * \
        f["inv"] ** 2
    return f


def refine(out, anchor, cfg):
    """-> ({output name: fp64 value}, {output name: absolute-term sums}); V1 has no original_means / delta_means"""
    f = _frame(out, anchor, cfg)
    x, xa, opa, s0 = f["x"], f["xa"], f["opa"], f["s0"]
    val, err = {}, {}
    val["new_anchor"] = np.concatenate([x[..., :6], f["rot"], x[..., 10:]], -1)
    err["new_anchor"] = np.concatenate([xa[..., :6], f["rot_abs"], xa[..., 10:]], -1)
    val["means"] = f["sm"] * f["ext"] + f["lo"]
    err["means"] = f["sm"] * f["ext"] + np.abs(f["lo"]) + 0.25 * f["ext"] * xa[..., :3]
    val["scales"] = f["slo"] + f["sext"] * f["ss"]
    err["scales"] = abs(f["slo"]) + abs(f["sext"]) * (f["ss"] + 0.25 * xa[..., 3:6])
    val["rotations"], err["rotations"] = f["rot"], f["rot_abs"]
    so, _ = sig(x[..., 10:10 + opa])
    val["opacities"], err["opacities"] = so, so + 0.25 * xa[..., 10:10 + opa]
    z, za = x[..., s0:], xa[..., s0:]
    act = cfg["semantics_activation"]
    with np.errstate(over="ignore"):
        if act == "softmax":
            e = np.exp(z - z.max(-1, keepdims=True)) if z.shape[-1] else z
            y = e / e.sum(-1, keepdims=True) if z.shape[-1] else z
            val["semantics"], err["semantics"] = y, y * (1 + za + (y * za).sum(-1, keepdims=True))
        elif act == "softplus":
            sp = np.where(z > 20.0, z, np.log1p(np.exp(np.minimum(z, 20.0))))
            val["semantics"], err["semantics"] = sp, np.abs(sp) + za
        else:
            val["semantics"], err["semantics"] = z, za
    if cfg["variant"] == "v2":
        val["original_means"], err["original_means"] = f["orig"], f["orig_abs"]
        val["delta_means"], err["delta_means"] = f["delta"], f["delta_abs"]
    return val, err


def refine_backward(out, anchor, cfg, grads):
    """``grads``: {output name: gradient or None}.  -> (grad_out, its absolute-term sums, grad_anchor, its sums), fp64"""
    f = _frame(out, anchor, cfg)
    x, opa, s0, D, r = f["x"], f["opa"], f["s0"], f["D"], f["r"]
    lead = x.shape[:-1]
    shapes = dict(new_anchor=D, means=3, scales=3, rotations=4, opacities=opa, semantics=D - s0, original_means=3,
                  delta_means=3)
    G = {n: (_f64(grads[n]) if grads.get(n) is not None else np.zeros(lead + (shapes[n],))) for n in shapes}
    Ga = {n: np.abs(v) for n, v in G.items()}
    dX, dXa = np.zeros(x.shape), np.zeros(x.shape)
    na, naa = G["new_anchor"], Ga["new_anchor"]
    dX[..., :3] = na[..., :3] + G["means"] * f["ext"] * f["dsm"]
    dXa[..., :3] = naa[..., :3] + Ga["means"] * f["ext"] * f["dsm"]
    dX[..., 3:6] = na[..., 3:6] + G["scales"] * f["sext"] * f["dss"]
    dXa[..., 3:6] = naa[..., 3:6] + Ga["scales"] * abs(f["sext"]) * f["dss"]
    gr, gra = na[..., 6:10] + G["rotations"], naa[..., 6:10] + Ga["rotations"]
    rot = f["rot"]
    dot = np.where(f["below"], 0.0, (rot * gr).sum(-1, keepdims=True))
    dota = np.where(f["below"], 0.0, (np.abs(rot) * gra).sum(-1, keepdims=True))
    dX[..., 6:10] = f["inv"] * (gr - rot * dot)
    dXa[..., 6:10] = f["inv"] * (gra + np.abs(rot) * dota)
    _, dso = sig(x[..., 10:10 + opa])
    dX[..., 10:s0] = na[..., 10:s0] + G["opacities"] * dso
    dXa[..., 10:s0] = naa[..., 10:s0] + Ga["opacities"] * dso
    z, gs, gsa = x[..., s0:], G["semantics"], Ga["semantics"]
    act = cfg["semantics_activation"]
    if act == "softmax" and z.shape[-1]:
        e = np.exp(z - z.max(-1, keepdims=True))
        y = e / e.sum(-1, keepdims=True)
        ds = y * (gs - (gs * y).sum(-1, keepdims=True))
        dsa = y * (gsa + (gsa * y).sum(-1, keepdims=True))
    elif act == "softplus":
        with np.errstate(over="ignore"):
            ez = np.exp(np.minimum(z, 20.0))
        d = np.where(z > 20.0, 1.0, ez / (ez + 1.0))
        ds, dsa = gs * d, gsa * d
    else:
        ds, dsa = gs, gsa
    dX[..., s0:] = na[..., s0:] + ds
    dXa[..., s0:] = naa[..., s0:] + dsa
    ga = np.zeros(lead + (np.shape(anchor)[-1],))
    gaa = np.zeros(ga.shape)
    go, goa = dX.copy(), dXa.copy()
    if cfg["variant"] == "v1":
        ga[..., :r], gaa[..., :r] = dX[..., :r], dXa[..., :r]
        if f["unit"] is not None:
            k = 2 * f["unit"] * f["dsr"]
            go[..., :3], goa[..., :3] = dX[..., :3] * k, dXa[..., :3] * np.abs(k)
    else:
        dsum, dsuma = dX[..., :3] * f["dinv"] / f["ext"], dXa[..., :3] * f["dinv"] / f["ext"]
        ga[..., :3] = (dsum + G["original_means"]) * f["ext"] * f["dsa"]
        gaa[..., :3] = (dsuma + Ga["original_means"]) * f["ext"] * f["dsa"]
        k = 2 * f["unit"] * f["dsr"]
        go[..., :3] = (dsum + G["delta_means"]) * k
        goa[..., :3] = (dsuma + Ga["delta_means"]) * np.abs(k)
    return go, goa, ga, gaa


# ------------------------------------------------------------- the reference's lines in torch, any dtype
def safe_sigmoid(t):
    return torch.sigmoid(torch.clamp(t, -CLAMP, CLAMP))            # safe_ops.py:7-9, the bound as fp32 holds it


def safe_inverse_sigmoid(t):
    t = torch.clamp(t, INV_LO, INV_HI)                              # safe_ops.py:11-13, likewise
    return torch.log(t / (1 - t))


def _cartesian(a, lo, ext):
    s = safe_sigmoid(a[..., :3])
    return torch.stack([s[..., i] * ext[i] + lo[i] for i in range(3)], -1)


def _activate(sem, act):
    if act == "softmax":
        return sem.softmax(dim=-1)
    if act == "softplus":
        return F.softplus(sem)
    return sem


def reference_refine(output, anchor, cfg):
    """The reference's forward after ``layers`` (refine_module.py:72-123 / refine_module_v2.py:64-108), with the
    constants as the fp32 values the reference's fp32 tensors are combined with; works in ``output``'s dtype.
    -> (new_anchor, {output name: tensor})"""
    lo, ext, unit, slo, sext = constants(cfg)
    opa = int(cfg["include_opa"])
    s0, S = 10 + opa, cfg["semantic_dim"]
    g = {}
    if cfg["variant"] == "v1":
        if unit is not None:
            p = 2 * safe_sigmoid(output[..., :3]) - 1
            output = torch.cat([torch.stack([p[..., i] * unit[i] for i in range(3)], -1), output[..., 3:]], -1)
        r = _prefix(cfg)
        if r > 0:
            output = torch.cat([output[..., :r] + anchor[..., :r], output[..., r:]], -1)
        xyz, scale = output[..., :3], output[..., 3:6]
        rot = F.normalize(output[..., 6:10], dim=-1, eps=EPS)
        new_anchor = torch.cat([xyz, scale, rot, output[..., 10:]], -1)
        g["means"] = _cartesian(xyz, lo, ext)
        sem = new_anchor[..., s0:s0 + S]
        opacity = new_anchor[..., 10:10 + opa]
    else:
        # the module's fp32 unit_xyz buffer when the caller passes it (a device tensor, as in the reference), else the
        # same values as a new tensor
        buf = cfg.get("unit_xyz_buffer")
        unit_t = output.new_tensor(unit) if buf is None else buf.to(output.dtype)
        delta = (2 * safe_sigmoid(output[..., :3]) - 1.) * unit_t[None, None]
        orig = _cartesian(anchor[..., :3], lo, ext)
        moved = orig + delta
        axyz = safe_inverse_sigmoid(torch.stack([(moved[..., i] - lo[i]) / ext[i] for i in range(3)], -1))
        scale = output[..., 3:6]
        rot = F.normalize(output[..., 6:10], 2, -1, eps=EPS)
        opacity, sem = output[..., 10:s0], output[..., s0:s0 + S]
        new_anchor = torch.cat([axyz, scale, rot, opacity, sem], -1)
        g["means"] = _cartesian(axyz, lo, ext)
        g["original_means"], g["delta_means"] = orig, delta
    g["scales"] = slo + sext * safe_sigmoid(scale)
    g["rotations"] = rot
    g["opacities"] = safe_sigmoid(opacity)
    g["semantics"] = _activate(sem, cfg["semantics_activation"])
    return new_anchor, g
