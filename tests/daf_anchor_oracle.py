"""fp64 numpy oracle of the anchor key-point generator (``gf_daf_anchor_key_points`` / ``_backward``).

``SparseGaussian3DKeyPointsGenerator.forward`` (model/encoder/gaussian_encoder/deformable_module.py:51-90) with
``get_rotation_matrix`` (model/utils/utils.py:20-69) and ``safe_sigmoid`` (model/utils/safe_ops.py:7-9), in fp64 on the
fp32 inputs, with the constants the reference's fp32 tensors hold (9.21f, 1e-12f, the fp32 ranges):

    sig(v) = 1 / (1 + exp(-clamp(v, -9.21f, 9.21f)))
    xyz    = lo + extent * sig(x[0:3]),   gs = s0 + (s1 - s0) * sig(x[3:6])
    s_k    = fix_scale[k]  |  (sig(l_k) - 0.5) * learnable_fixed_scale
    kp_k   = R(q)^T (s_k * gs) + xyz,     R of F.normalize(q), q = x[6:10]

Next to every value the oracle returns the sum of the absolute values of the terms that make it (``*_abs``): the
scale of the rounding errors any fp64 evaluation of it makes.  Where a value is far below that scale (cancellation),
two fp64 evaluations that differ in the last bits of ``exp`` may round to different fp32 values, so the GPU tests hold
such entries to an absolute bound relative to ``*_abs``.
"""
import numpy as np
import torch
import torch.nn.functional as F

CLAMP = float(np.float32(9.21))        # safe_sigmoid's bound as an fp32 tensor holds it
EPS = float(np.float32(1e-12))         # F.normalize's epsilon, likewise
F32 = lambda v: float(np.float32(v))   # noqa: E731

# R(qh)[k, l] = sum_ab QUAD[k, l, a, b] qh_a qh_b for the unit quaternion qh = (w, x, y, z)
QUAD = np.zeros((3, 3, 4, 4))
for (k, l), terms in {
        (0, 0): [(1, 0, 0), (1, 1, 1), (-1, 2, 2), (-1, 3, 3)], (0, 1): [(2, 1, 2), (-2, 0, 3)],
        (0, 2): [(2, 1, 3), (2, 0, 2)], (1, 0): [(2, 1, 2), (2, 0, 3)],
        (1, 1): [(1, 0, 0), (-1, 1, 1), (1, 2, 2), (-1, 3, 3)], (1, 2): [(2, 2, 3), (-2, 0, 1)],
        (2, 0): [(2, 1, 3), (-2, 0, 2)], (2, 1): [(2, 2, 3), (2, 0, 1)],
        (2, 2): [(1, 0, 0), (-1, 1, 1), (-1, 2, 2), (1, 3, 3)]}.items():
    for c, a, b in terms:
        QUAD[k, l, a, b] += c
DQUAD = QUAD + QUAD.transpose(0, 1, 3, 2)         # d R[k, l] / d qh_a = sum_b DQUAD[k, l, a, b] qh_b


def _f64(a):
    return np.asarray(a, np.float32).astype(np.float64)


def _sig(v):
    """(sigmoid of the clamped logit, its derivative with the clamp's gate: bounds pass, outside and NaN do not)"""
    with np.errstate(invalid="ignore"):
        s = 1.0 / (1.0 + np.exp(-np.clip(v, -CLAMP, CLAMP)))
        return s, np.where((v >= -CLAMP) & (v <= CLAMP), s * (1.0 - s), 0.0)


def _frame(anchor, fix_scale, logits, pc_range, scale_range, lfs):
    a = _f64(anchor)
    B, A = a.shape[:2]
    lo = np.array([F32(pc_range[i]) for i in range(3)])
    ext = np.array([F32(pc_range[i + 3] - pc_range[i]) for i in range(3)])
    s0, sext, lfs = F32(scale_range[0]), F32(scale_range[1] - scale_range[0]), F32(lfs)
    f = dict(ext=ext, sext=sext, lfs=lfs)
    f["sx"], f["dsx"] = _sig(a[..., 0:3])
    f["sg"], f["dsg"] = _sig(a[..., 3:6])
    f["xyz"], f["xyz_abs"] = lo + ext * f["sx"], np.abs(lo) + ext * f["sx"]
    f["gs"], f["gs_abs"] = s0 + sext * f["sg"], abs(s0) + abs(sext) * f["sg"]
    q = a[..., 6:10]
    n = np.sqrt((q * q).sum(-1))
    f["inv"] = 1.0 / np.maximum(n, EPS)
    f["below"] = n < EPS
    f["qh"] = q * f["inv"][..., None]
    f["R"] = np.einsum("klab,...a,...b->...kl", QUAD, f["qh"], f["qh"])
    f["R_abs"] = np.einsum("klab,...a,...b->...kl", np.abs(QUAD), np.abs(f["qh"]), np.abs(f["qh"]))
    fix = np.broadcast_to(_f64(fix_scale).reshape(1, 1, -1, 3), (B, A, len(fix_scale), 3))
    s, s_abs, f["dsl"] = fix, np.abs(fix), None
    if logits is not None:
        sl, f["dsl"] = _sig(_f64(logits))
        s = np.concatenate([s, (sl - 0.5) * lfs], 2)
        s_abs = np.concatenate([s_abs, (sl + 0.5) * abs(lfs)], 2)
    f["s"], f["s_abs"] = s, s_abs
    f["v"], f["v_abs"] = s * f["gs"][:, :, None], s_abs * f["gs_abs"][:, :, None]
    return f


def key_points(anchor, fix_scale, logits, pc_range, scale_range, lfs=1.0):
    """-> (key points [B, A, K, 3] rounded to fp32, the same in fp64, their absolute-term sums)"""
    f = _frame(anchor, fix_scale, logits, pc_range, scale_range, lfs)
    kp = np.einsum("...ji,...kj->...ki", f["R"], f["v"]) + f["xyz"][:, :, None]
    kp_abs = np.einsum("...ji,...kj->...ki", f["R_abs"], f["v_abs"]) + f["xyz_abs"][:, :, None]
    with np.errstate(over="ignore", invalid="ignore"):
        return kp.astype(np.float32), kp, kp_abs


def key_points_backward(anchor, fix_scale, logits, pc_range, scale_range, lfs, grad_kp):
    """-> (grad_anchor [B, A, D], its absolute-term sums, grad_logits [B, A, Kl, 3] or None, its sums), fp64"""
    f = _frame(anchor, fix_scale, logits, pc_range, scale_range, lfs)
    g = _f64(grad_kp)
    ga = np.abs(g)
    Kf = len(fix_scale)
    dv = np.einsum("...ji,...ki->...kj", f["R"], g)                        # dv_k = R g_k
    dv_abs = np.einsum("...ji,...ki->...kj", f["R_abs"], ga)
    grad = np.zeros(np.shape(anchor))
    grad_abs = np.zeros(np.shape(anchor))
    grad[..., 0:3] = g.sum(2) * f["ext"] * f["dsx"]
    grad_abs[..., 0:3] = ga.sum(2) * f["ext"] * f["dsx"]
    grad[..., 3:6] = (f["s"] * dv).sum(2) * f["sext"] * f["dsg"]
    grad_abs[..., 3:6] = (f["s_abs"] * dv_abs).sum(2) * abs(f["sext"]) * f["dsg"]
    dR = np.einsum("...kj,...ki->...ji", f["v"], g)                        # sum_k v_k g_k^T
    dR_abs = np.einsum("...kj,...ki->...ji", f["v_abs"], ga)
    dqh = np.einsum("klab,...b,...kl->...a", DQUAD, f["qh"], dR)
    dqh_abs = np.einsum("klab,...b,...kl->...a", np.abs(DQUAD), np.abs(f["qh"]), dR_abs)
    below = f["below"][..., None]
    dot = np.where(below, 0.0, (f["qh"] * dqh).sum(-1, keepdims=True))
    dot_abs = np.where(below, 0.0, (np.abs(f["qh"]) * dqh_abs).sum(-1, keepdims=True))
    inv = f["inv"][..., None]
    grad[..., 6:10] = inv * (dqh - f["qh"] * dot)
    grad_abs[..., 6:10] = inv * (dqh_abs + np.abs(f["qh"]) * dot_abs)
    gl = gl_abs = None
    if logits is not None:
        gl = f["gs"][:, :, None] * dv[:, :, Kf:] * f["lfs"] * f["dsl"]
        gl_abs = f["gs_abs"][:, :, None] * dv_abs[:, :, Kf:] * abs(f["lfs"]) * f["dsl"]
    return grad, grad_abs, gl, gl_abs


# ------------------------------------------------------------- the reference's lines in torch, any dtype
def safe_sigmoid(t):
    return torch.sigmoid(torch.clamp(t, -CLAMP, CLAMP))     # safe_ops.py:7-9, the bound as fp32 holds it


def rotation_matrix(q):
    """get_rotation_matrix (utils.py:20-69): F.normalize, then the product of the quaternion's left-multiplication
    matrix with the conjugate transpose of its right-multiplication matrix, rows and columns 1..3."""
    q = F.normalize(q, dim=-1, eps=EPS)
    w, x, y, z = q.unbind(-1)
    left = torch.stack([torch.stack(r, -1) for r in ((w, -x, -y, -z), (x, w, -z, y), (y, z, w, -x), (z, -y, x, w))], -2)
    right = torch.stack([torch.stack(r, -1) for r in ((w, -x, -y, -z), (x, w, z, -y), (y, -z, w, x), (z, y, -x, w))], -2)
    return torch.matmul(left, torch.conj(right).transpose(-1, -2))[..., 1:, 1:]


def reference_generator(anchor, logits, fix_scale, pc_range, scale_range, lfs):
    """SparseGaussian3DKeyPointsGenerator.forward (deformable_module.py:51-90) after learnable_fc, with the ranges and
    scales as the fp32 values the reference's fp32 tensors multiply by; works in the anchor's dtype."""
    bs, num_anchor = anchor.shape[:2]
    f32 = F32
    scale = anchor.new_tensor(np.asarray(fix_scale, np.float32))[None, None].tile([bs, num_anchor, 1, 1])
    if logits is not None:
        scale = torch.cat([scale, (safe_sigmoid(logits) - 0.5) * f32(lfs)], dim=-2)
    gs_scales = f32(scale_range[0]) + f32(scale_range[1] - scale_range[0]) * safe_sigmoid(anchor[..., None, 3:6])
    key_points = scale * gs_scales
    rotation_mat = rotation_matrix(anchor[..., 6:10]).transpose(-1, -2)
    key_points = torch.matmul(rotation_mat[:, :, None], key_points[..., None]).squeeze(-1)
    xyz = safe_sigmoid(anchor[..., :3])
    xyz = torch.stack([xyz[..., i] * f32(pc_range[i + 3] - pc_range[i]) + f32(pc_range[i]) for i in range(3)], -1)
    return key_points + xyz.unsqueeze(2)
