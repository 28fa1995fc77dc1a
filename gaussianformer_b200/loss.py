"""Occupancy loss on the device: a drop-in for the reference's ``OccupancyLoss`` (``loss/occupancy_loss.py:34-149``)
as every shipped config runs it, ``ce_weight * CE + lovasz_weight * Lovasz-softmax``.

``occupancy_loss`` is one supervised layer as one autograd op: one ``gf_occ_loss`` call (include/gf_b200.h) computes
the loss and, when a gradient is needed, the gradient too; the backward only scales that gradient.  The PyTorch
original pays a host synchronisation for every boolean gather and every present-class test; the device op pays none
(with ``validate=False``), so a training step that uses it can be captured in a CUDA graph.  Loss and gradient are
bit-reproducible from call to call.

Deviations from the reference, all documented in DESIGN.md:

* equal Lovasz errors are ordered by ascending position (a stable sort); ``torch.sort`` leaves that order open, so the
  reference's gradient on a tie is arbitrary.  The loss value and a tie group's total gradient do not depend on it;
* an empty voxel pool gives CE = NaN (PyTorch's empty mean) and Lovasz = 0, not the reference's empty tensor;
* ``balance_cls_weight=True`` needs ``manual_class_weight`` (every shipped config passes it).
"""
from __future__ import annotations

import ctypes
import os

import torch
import torch.nn.functional as F
from torch import nn
from torch.autograd.function import Function, once_differentiable

from . import _lib
from ._lib import OccLossDesc


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _layout(pred):
    """(GF_OCC_* layout, pred) for ``[B, C, N]`` pred: the splat's transposed ``[B, N, C]`` view and a contiguous
    ``[B, C, N]`` are read in place; anything else is made contiguous first."""
    B, C, N = pred.shape
    st = pred.stride()
    if (C == 1 or st[1] == 1) and (N == 1 or st[2] == C) and (B == 1 or st[0] == N * C):
        return _lib.GF_OCC_VOXEL_MAJOR, pred
    if (C == 1 or st[1] == N) and (N == 1 or st[2] == 1) and (B == 1 or st[0] == N * C):
        return _lib.GF_OCC_CLASS_MAJOR, pred
    return _lib.GF_OCC_CLASS_MAJOR, pred.contiguous()


class OccupancyLossFunction(Function):
    """Scalar loss of ``pred`` ``[B, C, N]``; the gradient comes back in ``pred``'s layout."""

    @staticmethod
    def forward(ctx, pred, labels, occ_mask, class_weights, cfg):
        ignore_index, lovasz_ignore, empty_label, use_softmax, ce_weight, lovasz_weight, validate = cfg
        for t in (pred, labels, occ_mask, class_weights):
            if t is not None and not t.is_cuda:
                raise RuntimeError("occupancy_loss is CUDA-only (sm_90a); there is no CPU fallback.")
        if pred.dim() != 3:
            raise ValueError(f"pred must be [B, C, N], got {list(pred.shape)}")
        B, C, N = pred.shape
        if tuple(labels.shape) != (B, N):
            raise ValueError(f"labels must be [B, N] = [{B}, {N}], got {list(labels.shape)}")
        if occ_mask is not None and tuple(occ_mask.shape) != (B, N):
            raise ValueError(f"occ_mask must be [B, N] = [{B}, {N}], got {list(occ_mask.shape)}")
        if class_weights.numel() != C:
            raise ValueError(f"class_weights must have C = {C} entries, got {class_weights.numel()}")
        dtype = pred.dtype
        layout, x = _layout(pred.detach().float())
        labels = labels.detach().long().contiguous()
        mask = None if occ_mask is None else occ_mask.detach().bool().contiguous().view(torch.uint8)
        w = class_weights.detach().float().contiguous()
        d = OccLossDesc()
        d.batch, d.N, d.C = B, N, C
        d.branch = _lib.GF_OCC_LOGITS if use_softmax else _lib.GF_OCC_PROBS
        d.layout = layout
        d.ignore_index, d.lovasz_ignore = int(ignore_index), int(lovasz_ignore)
        d.empty_label = -1 if empty_label is None else int(empty_label)
        d.weight, d.ce_weight, d.lovasz_weight = 1.0, float(ce_weight), float(lovasz_weight)
        L = _lib.lib()
        dev = x.device
        with torch.cuda.device(dev):
            nbytes = L.gf_occ_loss_workspace_bytes(ctypes.byref(d))
            if nbytes == 0:
                raise _lib.GfError(f"occupancy_loss: {L.gf_last_error().decode()}")
            ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            loss = torch.empty(3, dtype=torch.float32, device=dev)
            grad = torch.empty_strided(x.shape, x.stride(), dtype=torch.float32, device=dev) \
                if ctx.needs_input_grad[0] else None
            _lib.check(L.gf_occ_loss(ctypes.byref(d), _ptr(x), _ptr(labels), _ptr(mask), _ptr(w), _ptr(loss),
                                     _ptr(grad), _ptr(ws), nbytes,
                                     ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
        if validate:
            status = int(ws[:4].view(torch.int32).item())   # one host synchronisation
            if status & _lib.GF_FLAG_LABEL_OUT_OF_RANGE:
                raise ValueError(f"occupancy_loss: a label in the voxel pool is outside [0, {C}) and is neither "
                                 f"ignore_index={ignore_index} nor lovasz_ignore={lovasz_ignore}")
        ctx.dtype = dtype
        ctx.save_for_backward(grad)
        parts = loss[1:].clone()
        ctx.mark_non_differentiable(parts)
        return loss[0].clone(), parts

    @staticmethod
    @once_differentiable
    def backward(ctx, g_total, g_parts):
        (grad,) = ctx.saved_tensors
        return (grad * g_total).to(ctx.dtype), None, None, None, None


def _validate_default():
    return os.environ.get("GF_B200_VALIDATE", "1") != "0"


def occupancy_loss(pred, labels, occ_mask=None, *, class_weights, ce_weight, lovasz_weight, lovasz_ignore,
                   ignore_index=255, use_softmax=True, empty_label=None, validate=None, return_parts=False):
    """``ce_weight * CE + lovasz_weight * Lovasz`` of one supervised layer (the contract in include/gf_b200.h):

    * ``pred`` ``[B, C, N]`` CUDA, logits (``use_softmax=True``, GaussianFormer-1) or probabilities (GaussianFormer-2);
      the transposed view of the splat's ``[B, N, C]`` output is read in place, and its gradient has the same strides
    * ``labels`` ``[B, N]`` integers; ``occ_mask`` ``[B, N]`` bool or None; ``class_weights`` ``[C]``
    * ``empty_label``: voxels with this label leave the pool (the reference's ``ignore_empty``); None = off

    The voxels of all samples form one pool, as the reference's boolean indexing makes them.  Returns the scalar loss,
    or ``(loss, ce, lovasz)`` with ``return_parts`` (the parts carry no gradient).  ``validate`` (default: the
    ``GF_B200_VALIDATE`` environment variable, on unless "0") raises on a label outside ``[0, C)`` that is neither
    ignore label, at the cost of one host synchronisation; without it the op never synchronises."""
    if validate is None:
        validate = _validate_default()
    cfg = (ignore_index, lovasz_ignore, empty_label, bool(use_softmax), ce_weight, lovasz_weight, bool(validate))
    total, parts = OccupancyLossFunction.apply(pred, labels, occ_mask, class_weights, cfg)
    return (total, parts[0], parts[1]) if return_parts else total


class OccupancyLoss(nn.Module):
    """Drop-in for the reference's ``OccupancyLoss`` with its constructor keywords, ``input_dict``, ``loss_voxel`` and
    ``forward``.  The CE and Lovasz terms run in ``occupancy_loss``; the focal, dice and scal terms are not implemented
    (no shipped config turns them on) and raise."""

    def __init__(self, weight=1.0, empty_label=17, num_classes=18, use_focal_loss=False, focal_loss_args=None,
                 use_dice_loss=False, balance_cls_weight=False, multi_loss_weights=None, use_sem_geo_scal_loss=True,
                 use_lovasz_loss=True, lovasz_ignore=255, manual_class_weight=None, ignore_empty=False,
                 lovasz_use_softmax=True, input_dict=None):
        super().__init__()
        for name, on in (("use_focal_loss", use_focal_loss), ("use_dice_loss", use_dice_loss),
                         ("use_sem_geo_scal_loss", use_sem_geo_scal_loss)):
            if on:
                raise NotImplementedError(f"OccupancyLoss: {name}=True is not implemented on the device (no shipped "
                                          f"config turns it on); pass {name}=False")
        self.weight = weight
        self.input_dict = input_dict if input_dict is not None else {
            "pred_occ": "pred_occ", "sampled_xyz": "sampled_xyz", "sampled_label": "sampled_label",
            "occ_mask": "occ_mask"}
        self.loss_func = self.loss_voxel
        self.empty_label = empty_label
        self.num_classes = num_classes
        self.classes = list(range(num_classes))
        self.use_lovasz_loss = use_lovasz_loss
        self.lovasz_ignore = lovasz_ignore
        self.ignore_empty = ignore_empty
        self.lovasz_use_softmax = lovasz_use_softmax
        mlw = multi_loss_weights or {}
        self.loss_voxel_ce_weight = mlw.get("loss_voxel_ce_weight", 1.0)
        self.loss_voxel_lovasz_weight = mlw.get("loss_voxel_lovasz_weight", 1.0)
        if balance_cls_weight:
            if manual_class_weight is None:
                raise NotImplementedError("OccupancyLoss: balance_cls_weight=True needs manual_class_weight (the "
                                          "frequency-derived weights are not available)")
            w = num_classes * F.normalize(torch.tensor(manual_class_weight), 1, -1)
        else:
            w = torch.ones(num_classes)
        self.register_buffer("class_weights", w.float(), persistent=False)
        #: raise on a label outside [0, C) that is neither ignore label (one host synchronisation per layer); set
        #: False for fully asynchronous / graph-captured use
        self.validate = _validate_default()

    def loss_voxel(self, pred_occ, sampled_xyz, sampled_label, occ_mask=None):
        if occ_mask is not None:
            occ_mask = occ_mask.flatten(1)
        labels = sampled_label.flatten(1)
        tot_loss = 0.0
        for semantics in pred_occ:
            w = self.class_weights.to(semantics.device)
            tot_loss = tot_loss + occupancy_loss(
                semantics, labels, occ_mask, class_weights=w, ce_weight=self.loss_voxel_ce_weight,
                lovasz_weight=self.loss_voxel_lovasz_weight if self.use_lovasz_loss else 0.0,
                lovasz_ignore=self.lovasz_ignore, ignore_index=255, use_softmax=self.lovasz_use_softmax,
                empty_label=self.empty_label if self.ignore_empty else None, validate=self.validate)
        return tot_loss / len(pred_occ)

    def forward(self, inputs):
        return self.weight * self.loss_func(**{k: inputs[v] for k, v in self.input_dict.items()})
