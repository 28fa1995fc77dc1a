"""Gaussian refinement on the device: drop-ins for ``SparseGaussian3DRefinementModule``
(``model/encoder/gaussian_encoder/refine_module.py:10-123``, GaussianFormer-1) and
``SparseGaussian3DRefinementModuleV2`` (``refine_module_v2.py:11-108``, GaussianFormer-2).

``gaussian_refine`` is the modules' arithmetic after their MLP as one autograd op (``gf_gaussian_refine`` /
``gf_gaussian_refine_backward``, include/gf_b200.h): fp64 inside, each output and each gradient rounded to fp32 once,
gradients bit-reproducible, no host synchronisation.  The modules build the reference's ``layers`` (``linear_relu_ln``
and mmcv's ``Scale``, restated) around it, so a reference state dict loads strictly.
"""
from __future__ import annotations

import ctypes
from typing import NamedTuple

import numpy as np
import torch
from torch import Tensor, nn
from torch.autograd.function import Function, once_differentiable

from .. import _lib
from .._lib import REFINE_OUTPUTS, RefineDesc, RefineGrads, RefineOutputs


class GaussianPrediction(NamedTuple):
    """The reference's ``GaussianPrediction`` (model/encoder/gaussian_encoder/utils.py:62-69)."""
    means: Tensor
    scales: Tensor
    rotations: Tensor
    opacities: Tensor
    semantics: Tensor
    original_means: Tensor = None
    delta_means: Tensor = None


_ACTIVATIONS = {"softmax": _lib.GF_REFINE_SOFTMAX, "softplus": _lib.GF_REFINE_SOFTPLUS}


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _refine_desc(variant, batch, num_anchors, out_dim, anchor_dim, pc_range, scale_range, unit_xyz, refine_prefix=0,
                 restrict_xyz=False, include_opa=True, semantic_dim=0, semantics_activation="softmax"):
    """The descriptor, with the constants as the fp32 values the reference's fp32 tensors are combined with (ctypes
    rounds each Python float to fp32 once).  ``unit_xyz`` in metres; V1 with ``restrict_xyz`` divides it by the extent
    and multiplies by 4 in double first, as the reference's constructor does."""
    d = RefineDesc()
    d.variant = variant
    d.batch, d.num_anchors, d.out_dim, d.anchor_dim = batch, num_anchors, out_dim, anchor_dim
    d.refine_prefix, d.restrict_xyz = refine_prefix, int(restrict_xyz)
    d.include_opa, d.semantic_dim = int(include_opa), semantic_dim
    d.semantics_act = _ACTIVATIONS.get(semantics_activation, _lib.GF_REFINE_IDENTITY)
    for i in range(3):
        ext = float(pc_range[i + 3]) - float(pc_range[i])
        d.lo[i] = float(pc_range[i])
        d.extent[i] = ext
        if variant == _lib.GF_REFINE_V2:
            d.unit[i] = float(unit_xyz[i])
        elif restrict_xyz:
            d.unit[i] = 4 * float(unit_xyz[i]) / ext
    d.scale_lo = float(scale_range[0])
    d.scale_extent = float(scale_range[1]) - float(scale_range[0])
    return d


class GaussianRefineFunction(Function):
    """``out`` ``[B, A, D]`` and ``anchor`` ``[B, A, Da]`` -> new_anchor, means, scales, rotations, opacities,
    semantics (and for V2 original_means, delta_means).  The backward runs on the saved fp32 inputs; nothing else is
    kept.  The gradient of an output that does not reach the loss arrives as None and is not read."""

    @staticmethod
    def forward(ctx, out, anchor, desc):
        for t in (out, anchor):
            if not t.is_cuda:
                raise RuntimeError("gaussian_refine is CUDA-only (sm_90a); there is no CPU fallback.")
        ctx.set_materialize_grads(False)
        ctx.dtypes = (out.dtype, anchor.dtype)
        out = out.detach().contiguous().float()
        anchor = anchor.detach().contiguous().float()
        B, A, D = out.shape
        v2 = desc.variant == _lib.GF_REFINE_V2
        shapes = {"new_anchor": D, "means": 3, "scales": 3, "rotations": 4, "opacities": desc.include_opa,
                  "semantics": desc.semantic_dim, "original_means": 3, "delta_means": 3}
        names = REFINE_OUTPUTS if v2 else REFINE_OUTPUTS[:6]
        dev = out.device
        with torch.cuda.device(dev):
            res = {n: torch.empty((B, A, shapes[n]), dtype=torch.float32, device=dev) for n in names}
            o = RefineOutputs(**{n: _ptr(t) for n, t in res.items()})
            _lib.check(_lib.lib().gf_gaussian_refine(ctypes.byref(desc), _ptr(out), _ptr(anchor), ctypes.byref(o),
                                                     _stream(dev)))
        ctx.desc = desc
        ctx.names = names
        ctx.save_for_backward(out, anchor)
        return tuple(res[n] for n in names)

    @staticmethod
    @once_differentiable
    def backward(ctx, *grads):
        out, anchor = ctx.saved_tensors
        dev = out.device
        keep = [None if g is None else g.contiguous().float() for g in grads]
        with torch.cuda.device(dev):
            g = RefineGrads(**{n: _ptr(t) for n, t in zip(ctx.names, keep)})
            grad_out = torch.empty_like(out)
            grad_anchor = torch.empty_like(anchor)
            _lib.check(_lib.lib().gf_gaussian_refine_backward(ctypes.byref(ctx.desc), _ptr(out), _ptr(anchor),
                                                              ctypes.byref(g), _ptr(grad_out), _ptr(grad_anchor),
                                                              _stream(dev)))
        out_dtype, anchor_dtype = ctx.dtypes
        return grad_out.to(out_dtype), grad_anchor.to(anchor_dtype), None


def gaussian_refine(out, anchor, variant, pc_range, scale_range, unit_xyz=None, refine_prefix=0, restrict_xyz=False,
                    include_opa=True, semantic_dim=0, semantics_activation="softmax"):
    """The refinement modules' arithmetic after ``layers`` (refine_module.py:72-123, refine_module_v2.py:64-108):

    * ``out`` ``[B, A, 10 + include_opa + semantic_dim]``, the MLP output after ``Scale``; ``anchor`` ``[B, A, Da]``
    * ``variant``: ``"v1"`` (``SparseGaussian3DRefinementModule``) or ``"v2"`` (``...V2``)
    * ``refine_prefix``: V1's ``len(refine_manual)``; ``restrict_xyz``: V1's switch; ``unit_xyz`` in metres
    * ``semantics_activation``: ``"softmax"``, ``"softplus"`` or anything else for none

    Returns ``(new_anchor, GaussianPrediction)``, fp32; V2 fills ``original_means`` and ``delta_means``.  Any float
    dtype and any strides are accepted (upcast to fp32); the gradients of ``out`` and ``anchor`` come back in their
    dtypes.  No host synchronisation (CUDA-graph capturable)."""
    if variant not in ("v1", "v2"):
        raise ValueError(f"variant must be 'v1' or 'v2', got {variant!r}")
    if out.dim() != 3 or anchor.dim() != 3 or tuple(out.shape[:2]) != tuple(anchor.shape[:2]):
        raise ValueError(f"out [B, A, D] and anchor [B, A, Da] must agree in B and A, got {list(out.shape)} and "
                         f"{list(anchor.shape)}")
    B, A, D = out.shape
    desc = _refine_desc(_lib.GF_REFINE_V2 if variant == "v2" else _lib.GF_REFINE_V1, B, A, D, anchor.shape[2],
                        pc_range, scale_range, unit_xyz, refine_prefix, restrict_xyz, include_opa, semantic_dim,
                        semantics_activation)
    res = GaussianRefineFunction.apply(out, anchor, desc)
    return res[0], GaussianPrediction(*res[1:])


def linear_relu_ln(embed_dims, in_loops, out_loops, input_dims=None):
    """The reference's MLP block builder (model/encoder/gaussian_encoder/utils.py:49-59)."""
    if input_dims is None:
        input_dims = embed_dims
    layers = []
    for _ in range(out_loops):
        for _ in range(in_loops):
            layers.append(nn.Linear(input_dims, embed_dims))
            layers.append(nn.ReLU(inplace=True))
            input_dims = embed_dims
        layers.append(nn.LayerNorm(embed_dims))
    return layers


class Scale(nn.Module):
    """mmcv's ``Scale``: ``x * scale`` with a learnable ``scale`` (here one per channel, as the refinement modules
    build it from a list)."""

    def __init__(self, scale=1.0):
        super().__init__()
        self.scale = nn.Parameter(torch.tensor(scale, dtype=torch.float))

    def forward(self, x):
        return x * self.scale


def _check_activations(xyz_activation, scale_activation):
    if xyz_activation != "sigmoid" or scale_activation != "sigmoid":
        raise ValueError(f"only the sigmoid activations are implemented (xyz_activation={xyz_activation!r}, "
                         f"scale_activation={scale_activation!r})")


class _RefinementBase(nn.Module):
    def _setup(self, embed_dims, pc_range, scale_range, semantics, semantic_dim, include_opa, semantics_activation,
               xyz_activation, scale_activation):
        _check_activations(xyz_activation, scale_activation)
        self.embed_dims = embed_dims
        if semantics:
            assert semantic_dim is not None
        else:
            semantic_dim = 0
        self.output_dim = 10 + int(include_opa) + semantic_dim
        self.semantic_start = 10 + int(include_opa)
        self.semantic_dim = semantic_dim
        self.include_opa = include_opa
        self.semantics_activation = semantics_activation
        self.xyz_act = xyz_activation
        self.scale_act = scale_activation
        self.pc_range = pc_range
        self.scale_range = scale_range
        self.layers = nn.Sequential(*linear_relu_ln(embed_dims, 2, 2), nn.Linear(self.embed_dims, self.output_dim),
                                    Scale([1.0] * self.output_dim))

    def _refine(self, output, anchor, variant, unit_xyz, refine_prefix=0, restrict_xyz=False):
        return gaussian_refine(output, anchor, variant, self.pc_range, self.scale_range, unit_xyz, refine_prefix,
                               restrict_xyz, self.include_opa, self.semantic_dim, self.semantics_activation)


class SparseGaussian3DRefinementModule(_RefinementBase):
    """Drop-in for the GaussianFormer-1 refinement module: the reference's constructor (keywords it ignores, e.g.
    ``phi_activation`` or ``xyz_coordinate`` of the shipped configs, are accepted and ignored), ``layers`` and state-dict
    keys.  ``forward(instance_feature, anchor, anchor_embed)`` returns ``(new_anchor, GaussianPrediction)``; the
    arithmetic after ``layers`` runs in ``gaussian_refine``."""

    def __init__(self, embed_dims=256, pc_range=None, scale_range=None, restrict_xyz=False, unit_xyz=None,
                 refine_manual=None, semantics=False, semantic_dim=None, include_opa=True,
                 semantics_activation="softmax", xyz_activation="sigmoid", scale_activation="sigmoid", **kwargs):
        super().__init__()
        self._setup(embed_dims, pc_range, scale_range, semantics, semantic_dim, include_opa, semantics_activation,
                    xyz_activation, scale_activation)
        self.restrict_xyz = restrict_xyz
        self.unit_xyz = unit_xyz
        if restrict_xyz:
            assert unit_xyz is not None
            self.unit_sigmoid = [4 * unit_xyz[i] / (pc_range[i + 3] - pc_range[i]) for i in range(3)]
        assert isinstance(refine_manual, list)
        self.refine_state = refine_manual
        assert all(self.refine_state[i] == i for i in range(len(self.refine_state)))

    def forward(self, instance_feature, anchor, anchor_embed):
        output = self.layers(instance_feature + anchor_embed)
        return self._refine(output, anchor, "v1", self.unit_xyz, len(self.refine_state), self.restrict_xyz)


class SparseGaussian3DRefinementModuleV2(_RefinementBase):
    """Drop-in for the GaussianFormer-2 refinement module: the reference's constructor (ignored keywords as above),
    ``layers``, state-dict keys and non-persistent ``unit_xyz`` buffer.  ``forward`` returns ``(new_anchor,
    GaussianPrediction)`` with ``original_means`` and ``delta_means``.  The op takes ``unit_xyz`` as the constructor's
    values rounded to fp32, the values the buffer holds, so no call reads the buffer back from the device."""

    def __init__(self, embed_dims=256, pc_range=None, scale_range=None, unit_xyz=None, semantics=False,
                 semantic_dim=None, include_opa=True, semantics_activation="softmax", xyz_activation="sigmoid",
                 scale_activation="sigmoid", **kwargs):
        super().__init__()
        self._setup(embed_dims, pc_range, scale_range, semantics, semantic_dim, include_opa, semantics_activation,
                    xyz_activation, scale_activation)
        self.register_buffer("unit_xyz", torch.tensor(unit_xyz, dtype=torch.float), False)
        self._unit_xyz_host = [float(v) for v in np.asarray(unit_xyz, np.float32)]

    def forward(self, instance_feature, anchor, anchor_embed):
        output = self.layers(instance_feature + anchor_embed)
        return self._refine(output, anchor, "v2", self._unit_xyz_host)
