"""Grid sampler — host-side mirror of the reference binding det2trt/models/functions/grid_sampler.py (:7-305):
``grid_sampler(input, grid, interpolation_mode: str, padding_mode: str, align_corners: bool)`` and its twin
``grid_sampler2`` (plugin GridSampler{2D,3D}TRT2), the same ONNX symbolics, grid channel-first ``[N, 2|3, ...]`` in the
[-10, 10] range (Appendix B of SURVEY.md).

forward() calls the sm_90a kernels through the C ABI (the reference's forward is ``aten.grid_sampler`` on
``grid.permute(...)/10``, :28-32). backward() is the reference's, statement for statement (:39-55 / :93-109): ATen's
``grid_sampler_{2,3}d_backward`` on the saved ``(input, grid/10)``, the grid gradient permuted back and scaled by 10 — it
exists for quantisation-aware training only and is not on the inference path.

TensorRT-format entries: ``grid_sampler_chw2`` (FP16 kCHW2, what the …TRT2 plugin negotiates, gridSamplerPlugin.cpp:
171-186) and ``grid_sampler_int8`` (INT8 kCHW4 with per-tensor scales) take tensors already in those packed layouts;
``pack_chw`` / ``unpack_chw`` convert from/to plain NCHW.
"""
import ctypes

import torch
from torch.autograd import Function

from .. import _lib

_MODE = {"bilinear": 0, "nearest": 1, "bicubic": 2}
_PAD = {"zeros": 0, "border": 1, "reflection": 2}


def _dims(t):
    return (ctypes.c_int * t.dim())(*t.shape)


def _launch(name, out, inp, grid, out_shape, in_shape, grid_shape, mode, pad, align, scales=None):
    nb = len(in_shape)
    od, idm, gd = ((ctypes.c_int * nb)(*s) for s in (out_shape, in_shape, grid_shape))
    if scales is None:
        _lib.call(name, inp.device, out.data_ptr(), inp.data_ptr(), grid.data_ptr(), od, idm, gd, nb, mode, pad,
                  int(bool(align)))  # fmt: skip
    else:
        so, si, sg = scales
        _lib.call(name, inp.device, out.data_ptr(), float(so), inp.data_ptr(), float(si), grid.data_ptr(), float(sg),
                  od, idm, gd, nb, mode, pad, int(bool(align)))  # fmt: skip
    return out


def _forward(input, grid, interpolation_mode, padding_mode, align_corners):
    if not input.is_cuda:
        raise RuntimeError("grid_sampler: input must be a CUDA tensor (no CPU fallback exists)")
    if input.dim() not in (4, 5) or grid.dim() != input.dim():
        raise RuntimeError("grid_sampler: input and grid must both be 4-D or 5-D")
    if grid.shape[0] != input.shape[0] or grid.shape[1] != input.dim() - 2:
        raise ValueError("grid must be [N, 2, Ho, Wo] (or [N, 3, Do, Ho, Wo]) with the input's batch size")
    if input.dtype not in (torch.float32, torch.float16):
        raise _lib.B200OpsError("grid_sampler", 1)
    input = input.contiguous()
    grid = grid.to(input.dtype).contiguous()
    out_shape = (input.shape[0], input.shape[1], *grid.shape[2:])
    out = torch.empty(out_shape, dtype=input.dtype, device=input.device)
    name = "b200_grid_sample_f32" if input.dtype == torch.float32 else "b200_grid_sample_f16"
    return _launch(name, out, input, grid, out_shape, tuple(input.shape), tuple(grid.shape), interpolation_mode,
                   padding_mode, align_corners)  # fmt: skip


def _make(op_name):
    class _GridSampler(Function):
        @staticmethod
        def symbolic(g, input, grid, interpolation_mode, padding_mode, align_corners):
            return g.op(op_name, input, grid, interpolation_mode_i=interpolation_mode, padding_mode_i=padding_mode,
                        align_corners_i=align_corners)  # fmt: skip

        @staticmethod
        def forward(ctx, input, grid, interpolation_mode, padding_mode, align_corners):
            if input.requires_grad or grid.requires_grad:
                perm = (0, 2, 3, 1) if grid.dim() == 4 else (0, 2, 3, 4, 1)
                ctx.save_for_backward(input, grid.permute(*perm) / 10)
                ctx.interpolation_mode, ctx.padding_mode, ctx.align_corners = interpolation_mode, padding_mode, align_corners
            return _forward(input, grid, interpolation_mode, padding_mode, align_corners)

        @staticmethod
        def backward(ctx, grad_outputs):
            input, grid = ctx.saved_tensors
            bwd = torch.ops.aten.grid_sampler_2d_backward if grid.dim() == 4 else torch.ops.aten.grid_sampler_3d_backward
            input_grad, grid_grad = bwd(grad_outputs.contiguous(), input, grid.to(input.dtype), ctx.interpolation_mode,
                                        ctx.padding_mode, ctx.align_corners, [True, True])
            back = (0, 3, 1, 2) if grid.dim() == 4 else (0, 4, 1, 2, 3)
            return input_grad, grid_grad.permute(*back) * 10, None, None, None

    _GridSampler.__name__ = "_" + op_name
    return _GridSampler


_GridSampler2D = _make("GridSampler2DTRT")
_GridSampler3D = _make("GridSampler3DTRT")
_GridSampler2D2 = _make("GridSampler2DTRT2")
_GridSampler3D2 = _make("GridSampler3DTRT2")


def grid_sampler(input, grid, interpolation_mode: str, padding_mode: str, align_corners: bool):
    """Plugin GridSampler2DTRT / GridSampler3DTRT (FP32, FP16). grid: [N,2,Ho,Wo] or [N,3,Do,Ho,Wo], values in
    [-10, 10] (x = -10 is the left edge, +10 the right edge). Same contract as the reference wrapper (:144-223)."""
    if grid.dim() == 4:
        return _GridSampler2D.apply(input, grid, _MODE[interpolation_mode], _PAD[padding_mode], align_corners)
    if grid.dim() == 5:
        return _GridSampler3D.apply(input, grid, _MODE[interpolation_mode], _PAD[padding_mode], align_corners)
    raise RuntimeError


def grid_sampler2(input, grid, interpolation_mode: str, padding_mode: str, align_corners: bool):
    """Plugin GridSampler2DTRT2 / GridSampler3DTRT2 (FP16 as half2). Same contract as the reference wrapper (:226-305).
    On PyTorch tensors (plain NCHW) it is numerically the same op; the packed-layout kernel is ``grid_sampler_chw2``."""
    if grid.dim() == 4:
        return _GridSampler2D2.apply(input, grid, _MODE[interpolation_mode], _PAD[padding_mode], align_corners)
    if grid.dim() == 5:
        return _GridSampler3D2.apply(input, grid, _MODE[interpolation_mode], _PAD[padding_mode], align_corners)
    raise RuntimeError


# ---- TensorRT vectorised formats ---------------------------------------------------------------------------------
def pack_chw(x: torch.Tensor, width: int) -> torch.Tensor:
    """NCHW -> TensorRT kCHW2 / kCHW4: [N, ceil(C/width), H, W, width] (channels zero-padded)."""
    n, c, h, w = x.shape
    cp = (c + width - 1) // width
    if cp * width != c:
        x = torch.cat([x, x.new_zeros(n, cp * width - c, h, w)], 1)
    return x.view(n, cp, width, h, w).permute(0, 1, 3, 4, 2).contiguous()


def unpack_chw(x: torch.Tensor, channels: int) -> torch.Tensor:
    n, cp, h, w, width = x.shape
    return x.permute(0, 1, 4, 2, 3).reshape(n, cp * width, h, w)[:, :channels].contiguous()


def _check_packed(name, input, grid, channels, width, dtype):
    """Shapes first, then device and dtype: input [N, ceil(channels / width), Hi, Wi, width], grid [N, 1, Ho, Wo, width]
    of the input's dtype. Returns (n, hi, wi, ho, wo)."""
    if input.dim() != 5 or input.shape[-1] != width or -(-channels // width) != input.shape[1]:
        raise ValueError(f"{name}: input must be [N, ceil({channels} / {width}), Hi, Wi, {width}], got {tuple(input.shape)}")
    if grid.dim() != 5 or grid.shape[0] != input.shape[0] or grid.shape[1] != 1 or grid.shape[-1] != width:
        raise ValueError(f"{name}: grid must be [{input.shape[0]}, 1, Ho, Wo, {width}], got {tuple(grid.shape)}")
    if not (input.is_cuda and grid.is_cuda) or input.dtype != dtype or grid.dtype != dtype:
        raise RuntimeError(f"{name}: input and grid must be {dtype} CUDA tensors")
    n, _, hi, wi, _ = input.shape
    return n, hi, wi, grid.shape[2], grid.shape[3]


def grid_sampler_chw2(input_chw2, grid_chw2, channels, interpolation_mode: str, padding_mode: str, align_corners: bool):
    """FP16 kCHW2 tensors: input [N, ceil(C/2), Hi, Wi, 2], grid [N, 1, Ho, Wo, 2] = (x, y). Returns kCHW2 output."""
    n, hi, wi, ho, wo = _check_packed("grid_sampler_chw2", input_chw2, grid_chw2, channels, 2, torch.float16)
    out = torch.empty(n, input_chw2.shape[1], ho, wo, 2, dtype=torch.float16, device=input_chw2.device)
    return _launch("b200_grid_sample_f16_chw2", out, input_chw2.contiguous(), grid_chw2.contiguous(),
                   (n, channels, ho, wo), (n, channels, hi, wi), (n, 2, ho, wo), _MODE[interpolation_mode],
                   _PAD[padding_mode], align_corners)  # fmt: skip


def grid_sampler_int8(input_chw4, scale_i, grid_chw4, scale_g, scale_o, channels, interpolation_mode: str,
                      padding_mode: str, align_corners: bool):
    """INT8 kCHW4 tensors with per-tensor scales (real = q*scale): input [N, ceil(C/4), Hi, Wi, 4], grid
    [N, 1, Ho, Wo, 4] = (x, y, 0, 0). Mirrors grid_sample_int8 (gridSamplerKernel.h:20-26). Returns kCHW4 int8."""
    n, hi, wi, ho, wo = _check_packed("grid_sampler_int8", input_chw4, grid_chw4, channels, 4, torch.int8)
    out = torch.empty(n, input_chw4.shape[1], ho, wo, 4, dtype=torch.int8, device=input_chw4.device)
    return _launch("b200_grid_sample_i8_chw4", out, input_chw4.contiguous(), grid_chw4.contiguous(),
                   (n, channels, ho, wo), (n, channels, hi, wi), (n, 2, ho, wo), _MODE[interpolation_mode],
                   _PAD[padding_mode], align_corners, scales=(scale_o, scale_i, scale_g))  # fmt: skip
