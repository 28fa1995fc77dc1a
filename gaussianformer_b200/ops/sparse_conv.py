"""Submanifold sparse convolution on the device: spconv's ``SubMConv3d`` and the encoder's ``SparseConv3D``
(``model/encoder/gaussian_encoder/spconv3d_module.py:10-83``) without spconv.

``build_rulebook`` turns the ``[N, 4]`` indices into a rulebook on the device (``gf_subm_conv_rulebook``,
include/gf_b200.h); ``subm_conv3d`` runs the convolution and its backward on it, and one rulebook serves any number of
calls on the same indices.  Nothing synchronises the host (with ``validate=False``), and the output and all three
gradients are bit-reproducible from call to call.

Deviation from spconv, documented in DESIGN.md: rows that share a voxel all read the voxel's representative, the
lowest row index in it (spconv keeps one row per voxel too but leaves open which), and all get the same output.
"""
from __future__ import annotations

import ctypes
import os

import torch
from torch import nn
from torch.autograd.function import Function, once_differentiable

from .. import _lib
from .._lib import SubmConvDesc

WIDTH = 128   # c_in = c_out the op is compiled for


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _validate_default():
    return os.environ.get("GF_B200_VALIDATE", "1") != "0"


class SubmConvRulebook:
    """The device rulebook of one set of indices: the workspace ``gf_subm_conv_rulebook`` filled, and its desc.  The
    forward and backward calls use the same workspace for their scratch, so they run in the order of one stream."""

    def __init__(self, indices, spatial_shape, batch, kernel_size, validate=None):
        if not indices.is_cuda:
            raise RuntimeError("build_rulebook is CUDA-only (sm_90a); there is no CPU fallback.")
        if indices.dim() != 2 or indices.shape[1] != 4:
            raise ValueError(f"indices must be [N, 4] (b, x, y, z), got {list(indices.shape)}")
        X, Y, Z = (int(s) for s in spatial_shape)
        self.indices = indices.detach().to(torch.int32).contiguous()
        self.desc = SubmConvDesc(int(batch), int(indices.shape[0]), X, Y, Z, int(kernel_size), WIDTH, WIDTH)
        self.kernel_size = int(kernel_size)
        L = _lib.lib()
        dev = self.indices.device
        with torch.cuda.device(dev):
            nbytes = L.gf_subm_conv_workspace_bytes(ctypes.byref(self.desc))
            if nbytes == 0:
                raise _lib.GfError(f"subm_conv3d: {L.gf_last_error().decode()}")
            self.workspace = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            _lib.check(L.gf_subm_conv_rulebook(ctypes.byref(self.desc), _ptr(self.indices), _ptr(self.workspace),
                                               nbytes, _stream(dev)))
        if validate is None:
            validate = _validate_default()
        if validate:
            status = int(self.workspace[:4].view(torch.int32).item())   # one host synchronisation
            if status & _lib.GF_FLAG_INDEX_OUT_OF_RANGE:
                raise ValueError(f"subm_conv3d: a row's (b, x, y, z) lies outside batch {batch} x spatial shape "
                                 f"{(X, Y, Z)}; such rows get 0 and contribute nothing")


def build_rulebook(indices, spatial_shape, batch, kernel_size, validate=None):
    """Rulebook of ``indices`` ``[N, 4]`` int32 rows ``(b, x, y, z)`` on a ``batch x spatial_shape`` grid for an odd
    ``kernel_size <= 5``; pass it to ``subm_conv3d`` to reuse it.  ``validate`` (default: the ``GF_B200_VALIDATE``
    environment variable, on unless "0") raises on a row outside the grid, at the cost of one host synchronisation."""
    return SubmConvRulebook(indices, spatial_shape, batch, kernel_size, validate)


class SubMConv3dFunction(Function):
    """``out [N, 128] = subm_conv(features [N, 128], weight [128, k, k, k, 128], bias [128] or None)`` on a rulebook;
    the gradients come back in the inputs' dtypes."""

    @staticmethod
    def forward(ctx, features, weight, bias, rulebook):
        for t in (features, weight, bias):
            if t is not None and not t.is_cuda:
                raise RuntimeError("subm_conv3d is CUDA-only (sm_90a); there is no CPU fallback.")
        d = rulebook.desc
        k = rulebook.kernel_size
        if tuple(features.shape) != (d.num_rows, WIDTH):
            raise ValueError(f"features must be [N, {WIDTH}] = [{d.num_rows}, {WIDTH}], got {list(features.shape)}")
        if tuple(weight.shape) != (WIDTH, k, k, k, WIDTH):
            raise ValueError(f"weight must be [{WIDTH}, {k}, {k}, {k}, {WIDTH}] (spconv layout), got "
                             f"{list(weight.shape)}")
        if bias is not None and tuple(bias.shape) != (WIDTH,):
            raise ValueError(f"bias must be [{WIDTH}], got {list(bias.shape)}")
        x = features.detach().float().contiguous()
        w = weight.detach().float().contiguous()
        b = None if bias is None else bias.detach().float().contiguous()
        dev = x.device
        out = torch.empty_like(x)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().gf_subm_conv_forward(ctypes.byref(d), _ptr(rulebook.workspace), _ptr(x), _ptr(w),
                                                       _ptr(b), _ptr(out), _stream(dev)))
        ctx.rulebook = rulebook
        ctx.dtypes = (features.dtype, weight.dtype, None if bias is None else bias.dtype)
        ctx.save_for_backward(x, w)
        return out.to(features.dtype)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        x, w = ctx.saved_tensors
        rb = ctx.rulebook
        g = grad_out.float().contiguous()
        need_x, need_w, need_b = ctx.needs_input_grad[:3]
        gx = torch.empty_like(x) if need_x else None
        gw = torch.empty_like(w) if need_w else None
        gb = torch.empty(WIDTH, dtype=torch.float32, device=x.device) if need_b else None
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().gf_subm_conv_backward(ctypes.byref(rb.desc), _ptr(rb.workspace), _ptr(x), _ptr(w),
                                                        _ptr(g), _ptr(gx), _ptr(gw), _ptr(gb), _stream(x.device)))
        dx, dw, db = ctx.dtypes
        return (None if gx is None else gx.to(dx), None if gw is None else gw.to(dw),
                None if gb is None else gb.to(db), None)


def subm_conv3d(features, indices, weight, bias, spatial_shape, batch, rulebook=None, validate=None):
    """Submanifold convolution of ``features`` ``[N, 128]`` at ``indices`` ``[N, 4]`` (the contract in
    include/gf_b200.h) with ``weight`` ``[128, k, k, k, 128]`` (spconv 2.x layout) and ``bias`` ``[128]`` or None.
    ``rulebook`` (from ``build_rulebook`` on the same indices, grid and k) skips building one."""
    if rulebook is None:
        rulebook = build_rulebook(indices, spatial_shape, batch, weight.shape[1], validate)
    return SubMConv3dFunction.apply(features, weight, bias, rulebook)


class SubMConv3d(nn.Module):
    """spconv's ``SubMConv3d(in_channels, out_channels, kernel_size, stride=1, padding=(k-1)//2, bias=True)`` on
    ``(features, indices, spatial_shape, batch)``, with its parameter names and shapes (``weight [Cout, k, k, k, Cin]``,
    ``bias [Cout]``), so state dicts keep their keys."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=None, bias=True):
        super().__init__()
        if in_channels != WIDTH or out_channels != WIDTH:
            raise NotImplementedError(f"SubMConv3d is compiled for {WIDTH} -> {WIDTH} channels, got "
                                      f"{in_channels} -> {out_channels}")
        if stride != 1 or (padding is not None and padding != (kernel_size - 1) // 2):
            raise NotImplementedError("SubMConv3d: only stride 1 with padding (k - 1) // 2 (submanifold)")
        k = int(kernel_size)
        self.kernel_size = k
        self.weight = nn.Parameter(torch.empty(out_channels, k, k, k, in_channels))
        self.bias = nn.Parameter(torch.empty(out_channels)) if bias else None
        nn.init.kaiming_uniform_(self.weight.view(out_channels, -1), a=5 ** 0.5)
        if self.bias is not None:
            nn.init.uniform_(self.bias, -1 / (k ** 3 * in_channels) ** 0.5, 1 / (k ** 3 * in_channels) ** 0.5)

    def forward(self, features, indices=None, spatial_shape=None, batch=None, rulebook=None):
        return subm_conv3d(features, indices, self.weight, self.bias, spatial_shape, batch, rulebook)


class SparseConv3D(nn.Module):
    """Drop-in for the reference's ``SparseConv3D``: the same constructor keywords (unused ones such as
    ``phi_activation`` or ``xyz_coordinate`` are accepted and ignored, as there), the same state-dict keys and
    ``forward(instance_feature [B, G, C], anchor [B, G, >=3]) -> [B, G, C]``.  The voxel indices are the reference's
    fp32 expression; one rulebook per forward serves every layer of the stack.  LayerNorm, ReLU and ``output_proj``
    stay in PyTorch.

    As in the reference, ``cartesian`` uses the constructor's ``pc_range`` while the offset, the cell size and the
    grid come from the ``pc_range`` / ``grid_size`` buffers; the grid is re-derived when a state dict is loaded.  The
    class is a plain ``nn.Module`` (no mmengine dependency), so ``init_cfg`` is accepted and ignored: the parameters
    keep PyTorch's default initialisation unless a checkpoint is loaded."""

    def __init__(self, in_channels, embed_channels, pc_range, grid_size, xyz_activation="sigmoid",
                 use_out_proj=False, kernel_size=5, use_multi_layer=False, init_cfg=None, **kwargs):
        super().__init__()
        if use_multi_layer:
            self.layer = nn.Sequential(
                SubMConv3d(in_channels, embed_channels, kernel_size), nn.LayerNorm(embed_channels), nn.ReLU(True),
                SubMConv3d(embed_channels, embed_channels, kernel_size), nn.LayerNorm(embed_channels), nn.ReLU(True),
                SubMConv3d(embed_channels, embed_channels, kernel_size), nn.LayerNorm(embed_channels), nn.ReLU(True))
        else:
            self.layer = SubMConv3d(in_channels, embed_channels, kernel_size, bias=False)
        self.output_proj = nn.Linear(embed_channels, embed_channels) if use_out_proj else nn.Identity()
        self.kernel_size = int(kernel_size)
        self.pc_range_list = [float(v) for v in pc_range]
        self.use_sigmoid = xyz_activation == "sigmoid"
        self.register_buffer("pc_range", torch.tensor(pc_range, dtype=torch.float))
        self.register_buffer("grid_size", torch.tensor(grid_size, dtype=torch.float))
        self._update_grid()
        self.register_load_state_dict_post_hook(lambda module, incompatible: module._update_grid())
        #: raise on an anchor outside the grid (one host synchronisation per forward); False for asynchronous use
        self.validate = _validate_default()

    def _update_grid(self):
        """``spatial_shape`` from the ``pc_range`` and ``grid_size`` buffers, the reference's fp32 expression
        (spconv3d_module.py:75-76), evaluated on the host when the module is built and whenever a state dict is
        loaded, so that forward never synchronises"""
        pr, gs = self.pc_range.detach().cpu(), self.grid_size.detach().cpu()
        self.spatial_shape = tuple(int(v) for v in ((pr[3:] - pr[:3]) / gs).to(torch.int32).tolist())

    def voxel_indices(self, anchor):
        """``[B*G, 4]`` int32 rows (b, x, y, z): spconv3d_module.py:57-72 op for op (cartesian with safe_sigmoid or
        the clamp, minus pc_range, over grid_size, truncated)."""
        bs, g = anchor.shape[:2]
        pr = self.pc_range_list
        a = anchor[..., :3].float()
        xyz = torch.sigmoid(torch.clamp(a, -9.21, 9.21)) if self.use_sigmoid else a.clamp(min=1e-6, max=1 - 1e-6)
        xyz = torch.stack([xyz[..., 0] * (pr[3] - pr[0]) + pr[0], xyz[..., 1] * (pr[4] - pr[1]) + pr[1],
                           xyz[..., 2] * (pr[5] - pr[2]) + pr[2]], dim=-1).flatten(0, 1)
        idx = ((xyz - self.pc_range[None, :3]) / self.grid_size[None, :]).to(torch.int32)
        b = torch.arange(bs, device=idx.device, dtype=torch.int32).reshape(bs, 1, 1).expand(-1, g, -1).flatten(0, 1)
        return torch.cat([b, idx], dim=-1)

    def forward(self, instance_feature, anchor):
        bs, g, _ = instance_feature.shape
        indices = self.voxel_indices(anchor)
        rb = build_rulebook(indices, self.spatial_shape, bs, self.kernel_size, self.validate)
        x = instance_feature.flatten(0, 1)
        if isinstance(self.layer, nn.Sequential):
            for m in self.layer:
                x = m(x, rulebook=rb) if isinstance(m, SubMConv3d) else m(x)
        else:
            x = self.layer(x, rulebook=rb)
        return self.output_proj(x.unflatten(0, (bs, g)))
