"""Key points of Gaussian anchors on the device: a drop-in for ``SparseGaussian3DKeyPointsGenerator``
(``model/encoder/gaussian_encoder/deformable_module.py:17-90``).

``anchor_key_points`` is the generator's arithmetic after ``learnable_fc`` as one autograd op
(``gf_daf_anchor_key_points`` / ``gf_daf_anchor_key_points_backward``, include/gf_b200.h): fp64 inside, each key point
and each gradient rounded to fp32 once, gradients bit-reproducible.  ``SparseGaussian3DKeyPointsGenerator`` is the
module with the reference's constructor, ``learnable_fc`` and state dict around it.  The key points feed
``deformable_aggregation_from_key_points`` directly.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch
from torch import nn
from torch.autograd.function import Function, once_differentiable

from .. import _lib
from .._lib import DafKpsDesc


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _kps_desc(anchor, fix_scale, logits, pc_range, scale_range, learnable_fixed_scale):
    """The descriptor, with the constants as the fp32 values the reference's fp32 tensors are multiplied by
    (ctypes rounds each Python float to fp32 once)."""
    d = DafKpsDesc()
    d.batch, d.num_anchors, d.anchor_dim = anchor.shape
    d.num_fixed = fix_scale.shape[0]
    d.num_learnable = 0 if logits is None else logits.shape[2]
    for i in range(3):
        d.lo[i] = float(pc_range[i])
        d.extent[i] = float(pc_range[i + 3]) - float(pc_range[i])
    d.scale_lo = float(scale_range[0])
    d.scale_extent = float(scale_range[1]) - float(scale_range[0])
    d.learnable_fixed_scale = float(learnable_fixed_scale)
    return d


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


class AnchorKeyPointsFunction(Function):
    """``[B, A, Kf + Kl, 3]`` key points of ``anchor`` ``[B, A, D]``; gradients to ``anchor`` and
    ``learnable_logits``.  The backward runs on the saved fp32 inputs; nothing else is kept."""

    @staticmethod
    def forward(ctx, anchor, learnable_logits, fix_scale, pc_range, scale_range, learnable_fixed_scale):
        for t in (anchor, learnable_logits, fix_scale):
            if t is not None and not t.is_cuda:
                raise RuntimeError("anchor_key_points is CUDA-only (sm_90a); there is no CPU fallback.")
        if anchor.dim() != 3 or anchor.shape[-1] < 10:
            raise ValueError(f"anchor must be [B, A, D] with D >= 10 (xyz, scale, rotation, ...), got "
                             f"{list(anchor.shape)}")
        B, A = anchor.shape[:2]
        if fix_scale.dim() != 2 or fix_scale.shape[1] != 3:
            raise ValueError(f"fix_scale must be [Kf, 3], got {list(fix_scale.shape)}")
        if learnable_logits is not None and (learnable_logits.dim() != 4 or
                                             tuple(learnable_logits.shape[:2]) != (B, A) or
                                             learnable_logits.shape[3] != 3):
            raise ValueError(f"learnable_logits must be [B, A, Kl, 3] = [{B}, {A}, Kl, 3], got "
                             f"{list(learnable_logits.shape)}")
        ctx.dtypes = (anchor.dtype, None if learnable_logits is None else learnable_logits.dtype)
        anchor = anchor.detach().contiguous().float()
        fix_scale = fix_scale.detach().contiguous().float()
        logits = None if learnable_logits is None else learnable_logits.detach().contiguous().float()
        d = _kps_desc(anchor, fix_scale, logits, pc_range, scale_range, learnable_fixed_scale)
        dev = anchor.device
        with torch.cuda.device(dev):
            kp = torch.empty((B, A, d.num_fixed + d.num_learnable, 3), dtype=torch.float32, device=dev)
            _lib.check(_lib.lib().gf_daf_anchor_key_points(ctypes.byref(d), _ptr(anchor), _ptr(fix_scale),
                                                           _ptr(logits), _ptr(kp), _stream(dev)))
        ctx.desc = d
        ctx.has_logits = logits is not None
        ctx.save_for_backward(anchor, fix_scale, *([logits] if logits is not None else []))
        return kp

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_kp):
        anchor, fix_scale, *rest = ctx.saved_tensors
        logits = rest[0] if ctx.has_logits else None
        d = ctx.desc
        dev = anchor.device
        grad_kp = grad_kp.contiguous().float()
        with torch.cuda.device(dev):
            grad_anchor = torch.empty_like(anchor)
            grad_logits = None if logits is None else torch.empty_like(logits)
            _lib.check(_lib.lib().gf_daf_anchor_key_points_backward(
                ctypes.byref(d), _ptr(anchor), _ptr(fix_scale), _ptr(logits), _ptr(grad_kp), _ptr(grad_anchor),
                _ptr(grad_logits), _stream(dev)))
        anchor_dtype, logits_dtype = ctx.dtypes
        return (grad_anchor.to(anchor_dtype), None if grad_logits is None else grad_logits.to(logits_dtype),
                None, None, None, None)


def anchor_key_points(anchor, learnable_logits, fix_scale, pc_range, scale_range, learnable_fixed_scale=1.0):
    """``SparseGaussian3DKeyPointsGenerator.forward`` after ``learnable_fc`` (deformable_module.py:56-90):

    * ``anchor`` ``[B, A, D]``, D >= 10: xyz logits, scale logits, quaternion (w, x, y, z), then anything
    * ``learnable_logits`` ``[B, A, Kl, 3]`` — ``learnable_fc(instance_feature)`` reshaped, before the sigmoid; or None
    * ``fix_scale`` ``[Kf, 3]`` CUDA tensor; ``pc_range`` 6 numbers; ``scale_range`` 2 numbers

    Returns ``[B, A, Kf + Kl, 3]`` fp32.  Any float dtype is upcast to fp32; the gradients of ``anchor`` (columns 10 and
    up are 0) and ``learnable_logits`` come back in their dtypes.  No host synchronisation (CUDA-graph capturable)."""
    return AnchorKeyPointsFunction.apply(anchor, learnable_logits, fix_scale, pc_range, scale_range,
                                         learnable_fixed_scale)


class SparseGaussian3DKeyPointsGenerator(nn.Module):
    """Drop-in for the reference module of the same name: the same constructor (other keyword arguments, e.g.
    ``phi_activation`` or ``xyz_coordinate`` of the shipped configs, are accepted and ignored as there), the same
    ``learnable_fc`` and ``init_weight``, the same ``num_pts`` and state-dict keys (``fix_scale`` is a non-persistent
    buffer), and the same rule that without ``instance_feature`` or learnable points only the fixed points are
    returned.  The arithmetic after ``learnable_fc`` runs in ``anchor_key_points``."""

    def __init__(self, embed_dims=256, num_learnable_pts=0, learnable_fixed_scale=1, fix_scale=None, pc_range=None,
                 scale_range=None, xyz_activation="sigmoid", scale_activation="sigmoid", **kwargs):
        super().__init__()
        if xyz_activation != "sigmoid" or scale_activation != "sigmoid":
            raise ValueError(f"only the sigmoid activations are implemented (xyz_activation={xyz_activation!r}, "
                             f"scale_activation={scale_activation!r})")
        self.embed_dims = embed_dims
        self.num_learnable_pts = num_learnable_pts
        self.learnable_fixed_scale = learnable_fixed_scale
        if fix_scale is None:
            fix_scale = ((0.0, 0.0, 0.0),)
        self.register_buffer("fix_scale", torch.tensor(np.array(fix_scale), dtype=torch.float32).reshape(-1, 3),
                             persistent=False)
        self.num_pts = len(self.fix_scale) + num_learnable_pts
        if num_learnable_pts > 0:
            self.learnable_fc = nn.Linear(self.embed_dims, num_learnable_pts * 3)
        self.pc_range = pc_range
        self.scale_range = scale_range
        self.xyz_act = xyz_activation
        self.scale_act = scale_activation

    def init_weight(self):
        if self.num_learnable_pts > 0:            # mmengine xavier_init(distribution="uniform", bias=0.0)
            nn.init.xavier_uniform_(self.learnable_fc.weight, gain=1)
            nn.init.constant_(self.learnable_fc.bias, 0.0)

    def forward(self, anchor, instance_feature=None):
        logits = None
        if self.num_learnable_pts > 0 and instance_feature is not None:
            bs, num_anchor = anchor.shape[:2]
            logits = self.learnable_fc(instance_feature).reshape(bs, num_anchor, self.num_learnable_pts, 3)
        return anchor_key_points(anchor, logits, self.fix_scale, self.pc_range, self.scale_range,
                                 self.learnable_fixed_scale)
