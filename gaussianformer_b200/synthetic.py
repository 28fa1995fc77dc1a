"""Seeded synthetic inputs shaped like the reference's SurroundOcc configs (no dataset needed).

Distributions follow SURVEY.md §8(d):

* grid / voxel centres — ``dataset/transform_3d.py:484-499`` (x-major, z fastest);
* scales ``lo + (hi-lo)*sigmoid(N(0,1))`` with the config's ``scale_range``
  (``config/nuscenes_gs25600_solid.py:70``, ``config/nuscenes_gs144000.py:70``,
  ``config/prob/nuscenes_gs6400.py:88``);
* inverse covariance built like ``model/head/gaussian_head.py:111-119``
  (``S``, ``R`` -> ``M = S R`` -> ``Cov = M^T M`` -> ``Cov.inverse()``), rotation from a unit
  quaternion (``model/utils/utils.py:20-69``);
* the "empty" Gaussian of the solid config — ``model/head/gaussian_head.py:43-48,96-102`` with
  ``config/nuscenes_gs25600_solid.py:179-184``.

Everything is generated on the CPU with a ``torch.Generator`` so the same seed gives the same
bytes on every box.
"""
from __future__ import annotations

import math

import torch

SPLAT_CONFIGS = {
    # name: (G, grid dims, pc_min, grid_size, scale_range, scale_multiplier, variant, empty, opa, sem)
    "tiny": dict(G=256, dims=(50, 50, 4), pc_min=(-12.5, -12.5, -1.0), grid_size=0.5,
                 scale_range=(0.08, 0.64), scale_multiplier=3, variant="base", with_empty=False,
                 include_opa=True, sem="softplus17"),
    "gs25600_solid": dict(G=25600, dims=(200, 200, 16), pc_min=(-50.0, -50.0, -5.0), grid_size=0.5,
                          scale_range=(0.08, 0.64), scale_multiplier=3, variant="base",
                          with_empty=True, include_opa=True, sem="softplus17"),
    "gs144000": dict(G=144000, dims=(200, 200, 16), pc_min=(-50.0, -50.0, -5.0), grid_size=0.5,
                     scale_range=(0.08, 0.32), scale_multiplier=3, variant="base",
                     with_empty=False, include_opa=False, sem="normal18"),
    "prob_gs6400": dict(G=6400, dims=(200, 200, 16), pc_min=(-50.0, -50.0, -5.0), grid_size=0.5,
                        scale_range=(0.01, 3.2), scale_multiplier=4, variant="prob",
                        with_empty=False, include_opa=True, sem="softmax17"),
    "tiny_prob": dict(G=192, dims=(40, 36, 8), pc_min=(-10.0, -9.0, -2.0), grid_size=0.5,
                      scale_range=(0.05, 1.2), scale_multiplier=4, variant="prob",
                      with_empty=False, include_opa=True, sem="softmax17"),
}


def voxel_centers(dims, pc_min, grid_size):
    """[H,W,D,3] voxel-centre coordinates, the ``occ_xyz`` of the reference loader."""
    H, W, D = dims
    xs = torch.arange(H, dtype=torch.float) * grid_size + 0.5 * grid_size + pc_min[0]
    ys = torch.arange(W, dtype=torch.float) * grid_size + 0.5 * grid_size + pc_min[1]
    zs = torch.arange(D, dtype=torch.float) * grid_size + 0.5 * grid_size + pc_min[2]
    return torch.stack([xs[:, None, None].expand(H, W, D), ys[None, :, None].expand(H, W, D),
                        zs[None, None, :].expand(H, W, D)], dim=-1).contiguous()


def quat_to_rotmat(q):
    """Unit-quaternion (w,x,y,z) -> 3x3 rotation, same matrix as the reference's helper."""
    q = torch.nn.functional.normalize(q, dim=-1)
    w, x, y, z = q.unbind(-1)
    rows = [
        torch.stack([w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
        torch.stack([2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)], -1),
        torch.stack([2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z], -1),
    ]
    return torch.stack(rows, dim=-2)


def inverse_covariance(scales, rotations):
    """``CovInv`` of ``GaussianHead.prepare_gaussian_args`` (computed on the CPU, like the reference)."""
    S = torch.diag_embed(scales)
    R = quat_to_rotmat(rotations)
    M = torch.matmul(S, R)
    cov = torch.matmul(M.transpose(-1, -2), M)
    return torch.linalg.inv(cov.cpu())


def make_splat_inputs(name="gs25600_solid", seed=0, perturb=False, overrides=None):
    """Returns (module_kwargs, inputs) with ``inputs`` = dict(pts, means, opa, sem, scales, cov)
    each carrying the reference's leading batch dimension of 1 (CPU float32)."""
    cfg = dict(SPLAT_CONFIGS[name])
    if overrides:
        cfg.update(overrides)
    gen = torch.Generator().manual_seed(seed)
    G = cfg["G"]
    dims, pc_min, gs = cfg["dims"], cfg["pc_min"], cfg["grid_size"]
    lo, hi = cfg["scale_range"]
    pc_min_t = torch.tensor(pc_min, dtype=torch.float)
    extent = torch.tensor(dims, dtype=torch.float) * gs

    pts = voxel_centers(dims, pc_min, gs).reshape(-1, 3)
    if perturb:  # dataset/transform_3d.py:522-525
        jitter = torch.clamp(torch.randn(pts.shape, generator=gen) / 6, -0.5, 0.5) * 0.49
        pts = pts + jitter
    means = pc_min_t + torch.rand(G, 3, generator=gen) * extent * (1 - 1e-3)
    scales = lo + (hi - lo) * torch.sigmoid(torch.randn(G, 3, generator=gen))
    rots = torch.randn(G, 4, generator=gen)
    if cfg["include_opa"]:
        opa = torch.sigmoid(torch.randn(G, generator=gen))
    else:
        opa = torch.ones(G)
    kind = cfg["sem"]
    if kind == "softplus17":
        sem = torch.nn.functional.softplus(torch.randn(G, 17, generator=gen))
        sem = torch.cat([sem, torch.zeros(G, 1)], dim=-1)
    elif kind == "softmax17":
        sem = torch.softmax(torch.randn(G, 17, generator=gen), dim=-1)
        sem = torch.cat([sem, torch.zeros(G, 1)], dim=-1)
    elif kind == "normal18":
        sem = torch.randn(G, 18, generator=gen)
    else:
        raise ValueError(kind)
    if cfg["with_empty"]:
        means = torch.cat([means, torch.tensor([[0.0, 0.0, -1.0]])], 0)
        scales = torch.cat([scales, torch.tensor([[100.0, 100.0, 8.0]])], 0)
        rots = torch.cat([rots, torch.tensor([[1.0, 0.0, 0.0, 0.0]])], 0)
        empty_sem = torch.zeros(1, 18)
        empty_sem[0, 17] = 10.0
        sem = torch.cat([sem, empty_sem], 0)
        opa = torch.cat([opa, torch.ones(1)], 0)
    cov = inverse_covariance(scales, rots)
    module_kwargs = dict(scale_multiplier=cfg["scale_multiplier"], H=dims[0], W=dims[1], D=dims[2],
                         pc_min=list(pc_min), grid_size=gs)
    inputs = dict(pts=pts[None].contiguous(), means=means[None].contiguous(),
                  opa=opa[None].contiguous(), sem=sem[None].contiguous(),
                  scales=scales[None].contiguous(), cov=cov[None].contiguous().float())
    return module_kwargs, inputs, cfg["variant"]


DAF_LEVELS_1600x864 = ((108, 200), (54, 100), (27, 50), (14, 25))


def make_daf_inputs(num_anchor=25600, num_pts=9, batch=1, num_cams=6, embed_dims=128, num_groups=4,
                    levels=DAF_LEVELS_1600x864, visible_p=0.22, seed=0):
    """Feature pyramid + sampling locations + masked-softmax weights shaped like
    ``DeformableFeatureAggregation.forward`` hands them to the op
    (``model/encoder/gaussian_encoder/deformable_module.py:161-228``)."""
    gen = torch.Generator().manual_seed(seed)
    feature_maps = [torch.randn(batch, num_cams, embed_dims, h, w, generator=gen) for h, w in levels]
    P = num_anchor * num_pts
    L = len(levels)
    inside = torch.rand(batch, P, num_cams, generator=gen) < visible_p
    loc_in = torch.rand(batch, P, num_cams, 2, generator=gen) * 0.998 + 0.001
    loc_out = 1.0 + torch.rand(batch, P, num_cams, 2, generator=gen) * 0.5
    flip = torch.rand(batch, P, num_cams, 2, generator=gen) < 0.5
    loc_out = torch.where(flip, -loc_out + 1.0, loc_out)
    loc = torch.where(inside[..., None], loc_in, loc_out).contiguous()
    # joint softmax over (pts, cams, levels) per anchor and group with invisible cams masked out
    raw = torch.randn(batch, num_anchor, num_pts, num_cams, L, num_groups, generator=gen)
    mask = inside.reshape(batch, num_anchor, num_pts, num_cams)[..., None, None].expand_as(raw)
    all_miss = mask.sum(dim=[2, 3, 4], keepdim=True) == 0
    raw = raw.masked_fill(~mask, -math.inf)
    raw = torch.where(all_miss.expand_as(raw), torch.zeros_like(raw), raw)
    w = raw.flatten(2, 4).softmax(dim=-2).reshape(batch, P, num_cams, L, num_groups)
    w = w * (1 - all_miss.expand(-1, -1, num_pts, -1, -1, -1).reshape(batch, P, 1, 1, num_groups).float())
    return feature_maps, loc, w.contiguous()


def make_daf_inputs_projected(num_anchor=25600, num_pts=9, batch=1, num_cams=6, embed_dims=128, num_groups=4,
                              levels=DAF_LEVELS_1600x864, seed=0, image_wh=(1600.0, 864.0), kp_sigma=0.3):
    """A CORRELATED sampling workload: what ``DeformableFeatureAggregation`` really feeds the op.  Anchors are 3-D
    points in the nuScenes volume; each anchor has ``num_pts`` key points scattered ``kp_sigma`` metres around it
    (``SparseGaussian3DKeyPointsGenerator``: fixed + learnable offsets scaled by the Gaussian, deformable_module.py:17-90);
    the key points are projected into ``num_cams`` pinhole cameras that look outward at 360/num_cams degree steps and
    normalised by the image size (``project_points``, deformable_module.py:287-305).  A camera sees a key point when it
    lies in front of it and inside the image; the other cameras get a location outside (0, 1) like the reference's.
    Key points of one anchor therefore land a few pixels apart (and on the same rows of the coarse levels), unlike
    ``make_daf_inputs`` whose locations are independent uniform draws.  Returns (feature_maps, loc, weights)."""
    gen = torch.Generator().manual_seed(seed)
    feature_maps = [torch.randn(batch, num_cams, embed_dims, h, w, generator=gen) for h, w in levels]
    W_img, H_img = image_wh
    P = num_anchor * num_pts
    L = len(levels)
    anchors = torch.rand(batch, num_anchor, 3, generator=gen) * torch.tensor([100.0, 100.0, 8.0]) + torch.tensor([-50.0, -50.0, -5.0])
    kps = anchors[:, :, None, :] + torch.randn(batch, num_anchor, num_pts, 3, generator=gen) * kp_sigma
    kps = kps.reshape(batch, P, 3)
    focal = 0.8 * W_img
    locs, vis = [], []
    for m in range(num_cams):
        yaw = 2 * math.pi * m / num_cams
        fwd = torch.tensor([math.cos(yaw), math.sin(yaw), 0.0])
        right = torch.tensor([math.sin(yaw), -math.cos(yaw), 0.0])
        up = torch.tensor([0.0, 0.0, 1.0])
        rel = kps - torch.tensor([0.0, 0.0, -3.2])                 # camera 1.8 m above the ground plane of the volume
        depth = (rel * fwd).sum(-1)
        u = focal * (rel * right).sum(-1) / depth.clamp(min=1e-5) + 0.5 * W_img
        v = -focal * (rel * up).sum(-1) / depth.clamp(min=1e-5) + 0.5 * H_img
        xy = torch.stack([u / W_img, v / H_img], -1)
        ok = (depth > 1e-5) & (xy > 0).all(-1) & (xy < 1).all(-1)
        xy = torch.where(ok[..., None], xy, torch.full_like(xy, 2.0))
        locs.append(xy)
        vis.append(ok)
    loc = torch.stack(locs, 2).contiguous()                          # [B, P, M, 2]
    inside = torch.stack(vis, 2)                                     # [B, P, M]
    raw = torch.randn(batch, num_anchor, num_pts, num_cams, L, num_groups, generator=gen)
    mask = inside.reshape(batch, num_anchor, num_pts, num_cams)[..., None, None].expand_as(raw)
    all_miss = mask.sum(dim=[2, 3, 4], keepdim=True) == 0
    raw = raw.masked_fill(~mask, -math.inf)
    raw = torch.where(all_miss.expand_as(raw), torch.zeros_like(raw), raw)
    w = raw.flatten(2, 4).softmax(dim=-2).reshape(batch, P, num_cams, L, num_groups)
    w = w * (1 - all_miss.expand(-1, -1, num_pts, -1, -1, -1).reshape(batch, P, 1, 1, num_groups).float())
    return feature_maps, loc, w.contiguous()


def make_daf_fused_inputs(num_anchor=25600, num_pts=9, batch=1, num_cams=6, embed_dims=128, num_groups=4,
                          levels=DAF_LEVELS_1600x864, visible_p=0.22, seed=0, attn_drop=0.0):
    """Inputs of the fused caller path (``ops.deformable_aggregation_fused``): the same pyramid and sampling
    locations as ``make_daf_inputs`` plus what ``DeformableFeatureAggregation.forward`` holds BEFORE its softmax
    (``deformable_module.py:177-212``): raw weights ``[B, A, K, M, L, Gr]``, the projection mask
    ``[B, A, K, M]`` (a camera sees the key point) and, for ``attn_drop > 0``, the training-time weight mask."""
    feature_maps, loc, _ = make_daf_inputs(num_anchor, num_pts, batch, num_cams, embed_dims, num_groups, levels,
                                           visible_p, seed)
    gen = torch.Generator().manual_seed(seed + 1000)
    L = len(levels)
    logits = torch.randn(batch, num_anchor, num_pts, num_cams, L, num_groups, generator=gen)
    point_mask = ((loc > 0) & (loc < 1)).all(-1).reshape(batch, num_anchor, num_pts, num_cams).contiguous()
    weight_mask = None
    if attn_drop > 0:
        weight_mask = torch.rand(logits.shape, generator=gen) > attn_drop
    return feature_maps, loc, logits, point_mask, weight_mask


def camera_rig(num_cams=6, image_wh=(1600.0, 864.0)):
    """The pinhole rig of ``make_daf_inputs_projected`` as ``[M, 4, 4]`` projection matrices (fp32): focal length
    0.8 W, principal point at the image centre, cameras 1.8 m above the volume floor (z = -3.2) looking outward every
    360/M degrees.  ``P @ (X, Y, Z, 1)`` gives (u z, v z, z, 1) in pixels, the convention of ``project_points``
    (deformable_module.py:287-305) before its division by ``image_wh``."""
    W_img, H_img = image_wh
    focal = 0.8 * W_img
    centre = torch.tensor([0.0, 0.0, -3.2], dtype=torch.float64)
    mats = []
    for m in range(num_cams):
        yaw = 2 * math.pi * m / num_cams
        fwd = torch.tensor([math.cos(yaw), math.sin(yaw), 0.0], dtype=torch.float64)
        right = torch.tensor([math.sin(yaw), -math.cos(yaw), 0.0], dtype=torch.float64)
        up = torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64)
        rows = torch.stack([focal * right + 0.5 * W_img * fwd, -focal * up + 0.5 * H_img * fwd, fwd])
        P = torch.eye(4, dtype=torch.float64)
        P[:3, :3] = rows
        P[:3, 3] = -(rows @ centre)
        mats.append(P)
    return torch.stack(mats).float()


def _near_a_boundary(key_points, projection_mat, image_wh, levels):
    """[B, A, K] True where the fp64 projection of a key point, in a camera with z > 0, lies within 1e-4 of the image
    border (normalised), within 1e-3 px of a bilinear cell boundary on any level, or has z within 1e-3 relative of
    1e-5 -- where an fp32 evaluation of project_points may decide a gate, mask or cell differently."""
    B, A, K, _ = key_points.shape
    X = torch.cat([key_points.double(), torch.ones(B, A, K, 1, dtype=torch.float64)], -1)      # [B, A, K, 4]
    xyz = torch.einsum("bmrc,bakc->bakmr", projection_mat.double()[:, :, :3], X)               # [B, A, K, M, 3]
    z = xyz[..., 2]
    zc = z.clamp(min=1e-5)
    uv = xyz[..., :2] / zc[..., None]
    if image_wh is not None:
        uv = uv / image_wh.double()[:, None, None]
    bad = (uv.abs() < 1e-4).any(-1) | ((uv - 1).abs() < 1e-4).any(-1) | ((z - 1e-5).abs() <= 1e-3 * 1e-5)
    for h, w in levels:
        im = uv * torch.tensor([w, h], dtype=torch.float64) - 0.5
        bad |= ((im - im.round()).abs() < 1e-3).any(-1)
    return (bad & (z > 0)).any(-1)


def make_daf_kp_inputs(num_anchor=25600, num_pts=9, batch=1, num_cams=6, embed_dims=128, num_groups=4,
                       levels=DAF_LEVELS_1600x864, seed=0, image_wh=(1600.0, 864.0), kp_sigma=0.3, attn_drop=0.0,
                       margin=False):
    """Inputs of ``ops.deformable_aggregation_from_key_points``: the pyramid, anchors and key points of
    ``make_daf_inputs_projected`` (key points ``kp_sigma`` metres around anchors in the nuScenes volume), its camera
    rig as ``projection_mat`` ``[B, M, 4, 4]`` (``camera_rig``), ``image_wh`` ``[B, M, 2]``, raw weights
    ``[B, A, K, M, L, Gr]`` and, for ``attn_drop > 0``, the training-time weight mask (else None).

    ``margin=True`` re-draws, from the same seeded generator, every key point that ``_near_a_boundary`` flags, so that
    an fp32 PyTorch ``project_points`` and the op decide every gate, mask and bilinear cell the same way.  Returns
    (feature_maps, key_points, projection_mat, image_wh, logits, weight_mask)."""
    gen = torch.Generator().manual_seed(seed)
    feature_maps = [torch.randn(batch, num_cams, embed_dims, h, w, generator=gen) for h, w in levels]
    L = len(levels)
    anchors = torch.rand(batch, num_anchor, 3, generator=gen) * torch.tensor([100.0, 100.0, 8.0]) + torch.tensor([-50.0, -50.0, -5.0])
    kps = anchors[:, :, None, :] + torch.randn(batch, num_anchor, num_pts, 3, generator=gen) * kp_sigma
    proj = camera_rig(num_cams, image_wh)[None].repeat(batch, 1, 1, 1).contiguous()
    wh = torch.tensor(image_wh, dtype=torch.float32).repeat(batch, num_cams, 1).contiguous()
    if margin:
        for _ in range(100):
            bad = _near_a_boundary(kps, proj, wh, levels)
            n = int(bad.sum())
            if n == 0:
                break
            b, a, _k = bad.nonzero(as_tuple=True)
            kps[bad] = anchors[b, a] + torch.randn(n, 3, generator=gen) * kp_sigma
        else:
            raise RuntimeError("make_daf_kp_inputs: key points near a boundary after 100 re-draws")
    logits = torch.randn(batch, num_anchor, num_pts, num_cams, L, num_groups, generator=gen)
    weight_mask = torch.rand(logits.shape, generator=gen) > attn_drop if attn_drop > 0 else None
    return feature_maps, kps.contiguous(), proj, wh, logits, weight_mask


# The key-point generator of both shipped families: fix_scale of config/_base_/model.py:88-96; GaussianFormer-1
# config/nuscenes_gs25600_solid.py:69-70,124-131, GaussianFormer-2 config/prob/nuscenes_gs6400.py:87-88,173-181.
ANCHOR_FIX_SCALE = ((0.0, 0.0, 0.0), (0.45, 0.0, 0.0), (-0.45, 0.0, 0.0), (0.0, 0.45, 0.0), (0.0, -0.45, 0.0),
                    (0.0, 0.0, 0.45), (0.0, 0.0, -0.45))
ANCHOR_KP_CONFIGS = {
    "gs25600_solid": dict(num_anchor=25600, num_learnable=2, learnable_fixed_scale=1.0,
                          pc_range=(-50.0, -50.0, -5.0, 50.0, 50.0, 3.0), scale_range=(0.08, 0.64)),
    "prob_gs6400": dict(num_anchor=6400, num_learnable=6, learnable_fixed_scale=6.0,
                        pc_range=(-50.0, -50.0, -5.0, 50.0, 50.0, 3.0), scale_range=(0.01, 3.2)),
}
ANCHOR_DIM = 28          # xyz, scale, rotation, opacity, semantics


def _key_points_fp64(anchor, logits, cfg):
    """SparseGaussian3DKeyPointsGenerator.forward in fp64 (for the margin test of make_anchor_kp_inputs only)."""
    a = anchor.double()
    sig = lambda v: torch.sigmoid(v.clamp(-9.21, 9.21))                                 # noqa: E731
    lo, hi = torch.tensor(cfg["pc_range"][:3]).double(), torch.tensor(cfg["pc_range"][3:]).double()
    s0, s1 = cfg["scale_range"]
    xyz = lo + (hi - lo) * sig(a[..., 0:3])
    gs = s0 + (s1 - s0) * sig(a[..., 3:6])
    B, A = a.shape[:2]
    s = torch.tensor(ANCHOR_FIX_SCALE, dtype=torch.float64).expand(B, A, -1, -1)
    s = torch.cat([s, (sig(logits.double()) - 0.5) * cfg["learnable_fixed_scale"]], 2)
    R = quat_to_rotmat(a[..., 6:10])
    return torch.einsum("bajk,bapj->bapk", R, s * gs[:, :, None]) + xyz[:, :, None]           # R^T v + xyz


def make_anchor_kp_inputs(config="gs25600_solid", batch=1, num_anchor=None, embed_dims=128, seed=0, margin=False,
                          num_cams=6, levels=DAF_LEVELS_1600x864, image_wh=(1600.0, 864.0)):
    """Inputs of ``ops.anchor_key_points`` / ``ops.SparseGaussian3DKeyPointsGenerator`` for one of
    ``ANCHOR_KP_CONFIGS``: anchors ``[B, A, 28]`` (xyz logits of a uniform position in pc_range, N(0, 1) scale logits,
    an un-normalised N(0, 1) quaternion, N(0, 1) opacity and semantics), an ``instance_feature`` ``[B, A, embed_dims]``,
    a seeded ``learnable_fc`` (``weight``, ``bias``, xavier-uniform) and its output ``logits`` ``[B, A, Kl, 3]``
    (fp32, on the CPU), plus the camera rig of ``make_daf_kp_inputs`` (``projection_mat``, ``image_wh``).

    ``margin=True`` keeps every anchor and learnable logit at least 1e-3 from +-9.21 (instance features are re-drawn
    for the learnable ones), and re-draws every anchor one of whose key points ``_near_a_boundary`` flags, so that an
    fp32 PyTorch generator and projection decide every gate, mask and bilinear cell as the fp64 ones do.  Returns a
    dict with those tensors and the generator's ``fix_scale``, ``pc_range``, ``scale_range``,
    ``learnable_fixed_scale`` and ``num_learnable``."""
    cfg = ANCHOR_KP_CONFIGS[config]
    A = cfg["num_anchor"] if num_anchor is None else num_anchor
    Kl = cfg["num_learnable"]
    gen = torch.Generator().manual_seed(seed)

    def draw_anchors(n):
        u = torch.rand(n, 3, generator=gen) * 0.96 + 0.02
        return torch.cat([torch.log(u / (1 - u)), torch.randn(n, ANCHOR_DIM - 3, generator=gen)], -1)

    anchor = draw_anchors(batch * A).reshape(batch, A, ANCHOR_DIM)
    feat = torch.randn(batch, A, embed_dims, generator=gen)
    bound = math.sqrt(6.0 / (embed_dims + 3 * Kl))
    weight = (torch.rand(3 * Kl, embed_dims, generator=gen) * 2 - 1) * bound
    bias = (torch.rand(3 * Kl, generator=gen) * 2 - 1) * 0.1
    logits = lambda: (feat @ weight.T + bias).reshape(batch, A, Kl, 3)                  # noqa: E731
    proj = camera_rig(num_cams, image_wh)[None].repeat(batch, 1, 1, 1).contiguous()
    wh = torch.tensor(image_wh, dtype=torch.float32).repeat(batch, num_cams, 1).contiguous()
    if margin:
        near = lambda v: ((v.abs() - 9.21).abs() < 1e-3)                                  # noqa: E731
        for _ in range(100):
            bad_f = near(logits()).flatten(2).any(-1)
            bad_a = near(anchor[..., :6]).any(-1) | _near_a_boundary(
                _key_points_fp64(anchor, logits(), cfg).float(), proj, wh, levels).any(-1)
            if not (bad_f.any() or bad_a.any()):
                break
            feat[bad_f] = torch.randn(int(bad_f.sum()), embed_dims, generator=gen)
            anchor[bad_a] = draw_anchors(int(bad_a.sum()))
        else:
            raise RuntimeError("make_anchor_kp_inputs: anchors near a boundary after 100 re-draws")
    return dict(anchor=anchor.contiguous(), instance_feature=feat.contiguous(), weight=weight, bias=bias,
                logits=logits().contiguous(), projection_mat=proj, image_wh=wh,
                fix_scale=torch.tensor(ANCHOR_FIX_SCALE), pc_range=list(cfg["pc_range"]),
                scale_range=list(cfg["scale_range"]), learnable_fixed_scale=cfg["learnable_fixed_scale"],
                num_learnable=Kl)


def reference_fused_composition(daf_apply, feat, shape, start, loc, logits, point_mask=None, weight_mask=None):
    """``deformable_module.py:213-228`` + ``:242`` in PyTorch around an op call ``daf_apply`` — what the fused entry
    point replaces (used by the tests and by bench.py to time the unfused route on the same GPU)."""
    B, A, K, M, L, Gr = logits.shape
    mask = torch.ones_like(logits, dtype=torch.bool)
    if point_mask is not None:
        mask = point_mask[..., None, None] & mask
    if weight_mask is not None:
        mask = mask & weight_mask
    all_miss = mask.sum(dim=[2, 3, 4], keepdim=True) == 0
    all_miss = all_miss.expand(-1, -1, K, M, L, -1)
    weights = logits.clone()
    weights[~mask] = -torch.inf
    weights[all_miss] = 0.
    weights = weights.flatten(2, 4).softmax(dim=-2).reshape(B, A * K, M, L, Gr)
    weights = weights * (1 - all_miss.flatten(1, 2).float())
    features = daf_apply(feat, shape, start, loc, weights).reshape(B, A, K, -1)
    return features.sum(dim=2)


# Label shares of a SurroundOcc-like occupancy target: class 17 (empty) dominates, a few percent are class 0 (others),
# the rest spread unevenly over the semantic classes 1..16.  These shares are an assumption -- real label statistics
# are not part of this repository -- chosen so that every class is present at full size and the Lovasz sort sees the
# heavy class imbalance of an occupancy grid.
OCC_EMPTY_SHARE, OCC_ZERO_SHARE = 0.88, 0.03


def make_occ_labels(batch, n, num_classes=18, seed=0, ignore_share=0.0, generator=None):
    """``[batch, n]`` int64 labels: ``OCC_EMPTY_SHARE`` of ``num_classes - 1``, ``OCC_ZERO_SHARE`` of 0, the rest over
    1..num_classes-2 with weights 1..num_classes-2 (uneven on purpose), and ``ignore_share`` of 255."""
    g = generator or torch.Generator().manual_seed(seed)
    sem = num_classes - 2
    probs = torch.tensor([OCC_ZERO_SHARE] + [(1 - OCC_EMPTY_SHARE - OCC_ZERO_SHARE) * (k + 1) / (sem * (sem + 1) / 2)
                                             for k in range(sem)] + [OCC_EMPTY_SHARE], dtype=torch.float64)
    labels = torch.multinomial(probs, batch * n, replacement=True, generator=g).reshape(batch, n)
    if ignore_share > 0:
        labels[torch.rand(batch, n, generator=g) < ignore_share] = 255
    return labels


def make_occ_loss_inputs(batch=1, n=640000, num_classes=18, use_softmax=True, seed=0, ignore_share=0.0,
                         duplicate_share=0.01, mask=True):
    """Inputs of ``occupancy_loss`` as the head hands them over: ``pred`` ``[B, N, C]`` fp32 contiguous (the splat's
    output; the loss takes ``pred.transpose(1, 2)``), logits ~ 2 N(0, 1) with the label's class raised by 1, or their
    fp32 softmax for the probability branch; ``labels`` ``[B, N]`` int64 (make_occ_labels); ``occ_mask`` ``[B, N]`` bool
    = ``labels != 0`` as the loader builds it, or None.  ``duplicate_share`` of the voxels copy the prediction and the
    label of an earlier voxel bit for bit, so the Lovasz sort meets exact ties at every size."""
    g = torch.Generator().manual_seed(seed)
    labels = make_occ_labels(batch, n, num_classes, generator=g, ignore_share=ignore_share)
    logits = 2.0 * torch.randn(batch, n, num_classes, generator=g)
    lab = labels.clamp(max=num_classes - 1)
    logits.scatter_add_(2, lab[..., None], torch.ones(batch, n, 1))
    pred = torch.softmax(logits, dim=2) if not use_softmax else logits
    ndup = int(duplicate_share * n)
    if ndup > 0 and n > 1:
        dst = torch.randperm(n, generator=g)[:ndup]
        src = (torch.rand(ndup, generator=g) * dst.float()).long()   # an earlier voxel (dst 0 copies itself)
        pred[:, dst] = pred[:, src]
        labels[:, dst] = labels[:, src]
    occ_mask = labels != 0 if mask else None
    return pred.contiguous(), labels, occ_mask


# Assumed shares of the clustered sparse-convolution anchors: trained Gaussians gather on surfaces, here a ground
# plane (SUBM_GROUND_SHARE, in the lowest SUBM_GROUND_LEVELS z levels) and the faces of SUBM_BOXES boxes (the rest).
# These are assumptions standing in for a trained model's anchors, not measured statistics.
SUBM_GROUND_SHARE, SUBM_GROUND_LEVELS, SUBM_BOXES = 0.5, 2, 24


def make_subm_conv_inputs(n, spatial, batch=1, clustered=False, seed=0, kernel_size=5, channels=128,
                          invalid=0, duplicates_of=None):
    """Inputs of ``subm_conv3d``: ``features [N, C]`` ~ N(0, 1), ``indices [N, 4]`` int32 rows ``(b, x, y, z)``
    (``n`` rows per sample, b-major, then shuffled), ``weight [C, k, k, k, C]`` and ``bias [C]`` ~ U(+-1/sqrt(k^3 C))
    as nn.Conv3d initialises them.  Voxels are uniform over the grid, or with ``clustered`` on the ground plane and box
    faces (shares above).  ``invalid`` rows get an out-of-grid coordinate or batch index; ``duplicates_of`` = m puts
    every m-th row into the voxel of one of the first N / 4m rows, about four per voxel, so that some voxels hold 3
    or more rows."""
    g = torch.Generator().manual_seed(seed)
    X, Y, Z = spatial
    rows = []
    for b in range(batch):
        nb = n if isinstance(n, int) else n[b]
        if clustered:
            ng = int(SUBM_GROUND_SHARE * nb)
            ground = torch.stack([torch.randint(0, X, (ng,), generator=g), torch.randint(0, Y, (ng,), generator=g),
                                  torch.randint(0, SUBM_GROUND_LEVELS, (ng,), generator=g)], 1)
            lo = torch.stack([torch.randint(0, X, (SUBM_BOXES,), generator=g), torch.randint(0, Y, (SUBM_BOXES,), generator=g),
                              torch.randint(0, max(1, Z // 2), (SUBM_BOXES,), generator=g)], 1)
            size = torch.stack([torch.randint(4, max(5, X // 8), (SUBM_BOXES,), generator=g),
                                torch.randint(4, max(5, Y // 8), (SUBM_BOXES,), generator=g),
                                torch.randint(2, max(3, Z // 2), (SUBM_BOXES,), generator=g)], 1)
            nf = nb - ng
            box = torch.randint(0, SUBM_BOXES, (nf,), generator=g)
            u = torch.rand(nf, 3, generator=g)
            face = torch.randint(0, 6, (nf,), generator=g)
            u[torch.arange(nf), face // 2] = (face % 2).float()            # pin one coordinate to a face
            pts = lo[box] + (u * (size[box] - 1).float()).round().long()
            pts = torch.minimum(pts, torch.tensor([X - 1, Y - 1, Z - 1]))
            xyz = torch.cat([ground, pts], 0)
        else:
            xyz = torch.stack([torch.randint(0, X, (nb,), generator=g), torch.randint(0, Y, (nb,), generator=g),
                               torch.randint(0, Z, (nb,), generator=g)], 1)
        rows.append(torch.cat([torch.full((xyz.shape[0], 1), b, dtype=torch.long), xyz], 1))
    idx = torch.cat(rows, 0)
    N = idx.shape[0]
    if duplicates_of:
        dst = torch.arange(duplicates_of, N, duplicates_of)
        idx[dst] = idx[(dst // duplicates_of) % max(1, N // (4 * duplicates_of))]   # ~4 copies of each early row
    if invalid:
        bad = torch.randperm(N, generator=g)[:invalid]
        col = torch.randint(0, 4, (invalid,), generator=g)
        lim = torch.tensor([batch, X, Y, Z])
        idx[bad, col] = torch.where(torch.rand(invalid, generator=g) < 0.5, -1 - col, lim[col] + col)
    idx = idx[torch.randperm(N, generator=g)].to(torch.int32).contiguous()
    bound = 1.0 / math.sqrt(kernel_size ** 3 * channels)
    features = torch.randn(N, channels, generator=g)
    weight = (torch.rand(channels, kernel_size, kernel_size, kernel_size, channels, generator=g) * 2 - 1) * bound
    bias = (torch.rand(channels, generator=g) * 2 - 1) * bound
    return features, idx, weight, bias


# The refinement modules of the three shipped setups: GaussianFormer-1 config/nuscenes_gs25600_solid.py:69-76,133-147
# and config/nuscenes_gs144000.py:69-76,133-147, GaussianFormer-2 config/prob/nuscenes_gs25600.py:87-94,116,183-194
# (19 200 lifted anchors + 6 400 random ones).  The anchor has the refined row's layout, so anchor_dim = out_dim.
REFINE_CONFIGS = {
    "gs25600_solid": dict(variant="v1", num_anchor=25600, unit_xyz=(4.0, 4.0, 1.0), refine_manual=[0, 1, 2],
                          restrict_xyz=True, semantics_activation="softplus", semantic_dim=17, include_opa=True,
                          pc_range=(-50.0, -50.0, -5.0, 50.0, 50.0, 3.0), scale_range=(0.08, 0.64)),
    "gs144000": dict(variant="v1", num_anchor=144000, unit_xyz=(2.0, 2.0, 0.5), refine_manual=[0, 1, 2],
                     restrict_xyz=True, semantics_activation="identity", semantic_dim=18, include_opa=False,
                     pc_range=(-50.0, -50.0, -5.0, 50.0, 50.0, 3.0), scale_range=(0.08, 0.32)),
    "prob_gs25600": dict(variant="v2", num_anchor=19200 + 6400, unit_xyz=(4.0, 4.0, 1.0), refine_manual=None,
                         restrict_xyz=False, semantics_activation="identity", semantic_dim=17, include_opa=True,
                         pc_range=(-50.0, -50.0, -5.0, 50.0, 50.0, 3.0), scale_range=(0.01, 1.8)),
}
# Shares of the drawn inputs that exercise the clamps (assumptions, not statistics of a trained model): anchors near a
# pc-range face with a delta that pushes them past it, xyz / scale / opacity logits beyond +-9.21, and semantic logits
# around the softplus threshold.
REFINE_FACE_SHARE, REFINE_BEYOND_SHARE, REFINE_HIGH_SEM_SHARE = 0.05, 0.02, 0.02


def _refine_clamp_inputs(out, anchor, cfg):
    """The fp64 values of the refinement that meet a clamp or the softplus threshold, as (value, bound) pairs, for the
    margin test of make_refine_inputs."""
    o, a = out.double(), anchor.double()
    lo = torch.tensor(cfg["pc_range"][:3], dtype=torch.float64)
    ext = torch.tensor(cfg["pc_range"][3:], dtype=torch.float64) - lo
    sig = lambda v: torch.sigmoid(v.clamp(-9.21, 9.21))                                 # noqa: E731
    unit = torch.tensor(cfg["unit_xyz"], dtype=torch.float64)
    opa = int(cfg["include_opa"])
    pairs = [(o[..., 0:6], 9.21), (o[..., 10:10 + opa], 9.21)]
    if cfg["variant"] == "v1":
        x = (2 * sig(o[..., :3]) - 1) * (4 * unit / ext) + a[..., :3]
        pairs.append((x, 9.21))
    else:
        t = (sig(a[..., :3]) * ext + lo + (2 * sig(o[..., :3]) - 1) * unit - lo) / ext
        pairs += [(a[..., :3], 9.21), (t, 1e-4), (t, 0.9999)]
    if cfg["semantics_activation"] == "softplus":
        pairs.append((o[..., 10 + opa:], 20.0))
    return pairs


def make_refine_inputs(config="gs25600_solid", batch=1, num_anchor=None, embed_dims=128, seed=0, margin=False):
    """Inputs of ``ops.gaussian_refine`` / the refinement modules for one of ``REFINE_CONFIGS``: the MLP output ``out``
    ``[B, A, D]`` and the incoming ``anchor`` ``[B, A, D]`` (fp32, on the CPU), with ``instance_feature`` and
    ``anchor_embed`` ``[B, A, embed_dims]`` for the whole module.

    Anchors: xyz logits of a position in pc_range (GaussianFormer-2: the first 3/4 near the ground, z in the lower
    half, the rest uniform), N(0, 1) scale logits, an un-normalised N(0, 1) quaternion, N(0, 1) opacity and semantics.
    ``out``: N(0, 1.5) xyz logits, N(0, 1) for the rest, semantics N(0, 3).  On top, ``REFINE_FACE_SHARE`` of the
    anchors sit within 1e-3 of a pc-range face on one axis (xyz logit beyond +-6.9) with an xyz logit in ``out`` that
    pushes them outward, so that V1's means and V2's inverse sigmoid meet their clamps; ``REFINE_BEYOND_SHARE`` of the
    xyz, scale and opacity logits are U(+-(9.21, 12)); ``REFINE_HIGH_SEM_SHARE`` of the semantic logits are U(15, 25).

    ``margin=True`` re-draws every anchor one of whose values meets a clamp (+-9.21f, V2's 1e-4 and 0.9999) or the
    softplus threshold within 1e-3, so that an fp32 evaluation decides every clamp as the fp64 one does.  The
    saturated inverse sigmoid is log(0.9999 / 1e-4) = 9.21024, beyond the sigmoid's 9.21 by construction; its gradient
    is 0 either way.  Returns a dict with those tensors and the module's constructor arguments under ``config``."""
    cfg = REFINE_CONFIGS[config]
    A = cfg["num_anchor"] if num_anchor is None else num_anchor
    opa, S = int(cfg["include_opa"]), cfg["semantic_dim"]
    D = 10 + opa + S
    gen = torch.Generator().manual_seed(seed)

    def draw(n):
        u = torch.rand(n, 3, generator=gen) * 0.96 + 0.02
        if cfg["variant"] == "v2":
            lifted = torch.arange(n) % 4 != 3                                  # 19 200 of 25 600
            u[lifted, 2] = u[lifted, 2] * 0.5
        anchor = torch.cat([torch.log(u / (1 - u)), torch.randn(n, D - 3, generator=gen)], -1)
        out = torch.cat([torch.randn(n, 3, generator=gen) * 1.5, torch.randn(n, 7 + opa, generator=gen),
                         torch.randn(n, S, generator=gen) * 3.0], -1)
        face = torch.rand(n, generator=gen) < REFINE_FACE_SHARE
        nf = int(face.sum())
        axis = torch.randint(0, 3, (nf,), generator=gen)
        side = torch.where(torch.rand(nf, generator=gen) < 0.5, -1.0, 1.0)
        rows = face.nonzero()[:, 0]
        anchor[rows, axis] = side * (6.9 + 2.2 * torch.rand(nf, generator=gen))
        out[rows, axis] = side * (1.0 + 2.0 * torch.rand(nf, generator=gen))
        cols = torch.cat([torch.arange(6), torch.arange(10, 10 + opa)])        # the clamped logits of out
        beyond = torch.rand(n, len(cols), generator=gen) < REFINE_BEYOND_SHARE
        mag = (9.21 + 2.79 * torch.rand(n, len(cols), generator=gen)) * torch.where(
            torch.rand(n, len(cols), generator=gen) < 0.5, -1.0, 1.0)
        out[:, cols] = torch.where(beyond, mag, out[:, cols])
        if S:
            high = torch.rand(n, S, generator=gen) < REFINE_HIGH_SEM_SHARE
            out[:, 10 + opa:][high] = 15.0 + 10.0 * torch.rand(int(high.sum()), generator=gen)
        return out, anchor

    out, anchor = draw(batch * A)
    if margin:
        for _ in range(100):
            bad = torch.zeros(batch * A, dtype=torch.bool)
            for v, bound in _refine_clamp_inputs(out, anchor, cfg):
                if v.numel():
                    bad |= ((v.abs() - bound).abs() < 1e-3).reshape(batch * A, -1).any(-1)
            if not bad.any():
                break
            out[bad], anchor[bad] = draw(int(bad.sum()))
        else:
            raise RuntimeError("make_refine_inputs: values near a clamp after 100 re-draws")
    module = dict(pc_range=list(cfg["pc_range"]), scale_range=list(cfg["scale_range"]),
                  unit_xyz=list(cfg["unit_xyz"]), semantics=S > 0, semantic_dim=S, include_opa=cfg["include_opa"],
                  semantics_activation=cfg["semantics_activation"], embed_dims=embed_dims)
    if cfg["variant"] == "v1":
        module.update(restrict_xyz=cfg["restrict_xyz"], refine_manual=list(cfg["refine_manual"]))
    return dict(out=out.reshape(batch, A, D).contiguous(), anchor=anchor.reshape(batch, A, D).contiguous(),
                instance_feature=torch.randn(batch, A, embed_dims, generator=gen),
                anchor_embed=torch.randn(batch, A, embed_dims, generator=gen), variant=cfg["variant"], config=module)
