"""Rotate — host-side mirror of the reference binding det2trt/models/functions/rotate.py (:7-124):
``rotate(img, angle, center, interpolation="nearest")`` and its twin ``rotate2`` (plugins RotateTRT / RotateTRT2), the
same ONNX symbolics (``interpolation_i``), img ``[C, H, W]``, angle in degrees (counter-clockwise, a 0-d or 1-element
tensor), center ``(x, y)`` in pixels, zero padding.

forward() calls the sm_90a kernels through the C ABI (the reference's forward builds an affine grid with bmm and calls
``aten.grid_sampler``, :12-84). Inference path only, as in the reference (its backward raises, :86-88).

Extension ``rotate_hwc``: BEVFormer keeps prev_bev as ``[H*W, 1, C]`` and permutes it to ``[C, H, W]`` and back
around the op (det2trt/models/modules/transformer.py:296-304); ``rotate_hwc(prev_bev.view(H, W, C), …)`` rotates the
channels-last tensor directly (16-byte coalesced taps, no permutes). ``rotate`` itself takes the same shortcut when
it is handed a permuted view of a channels-last tensor, and returns the same kind of view.

TensorRT-format entries: ``rotate_chw2`` (FP16 kCHW2) and ``rotate_int8`` (INT8 kCHW4 with per-tensor scales) take
tensors already packed with ``functions.grid_sampler.pack_chw``.
"""
import ctypes

import torch
from torch.autograd import Function

from .. import _lib

_MODE = {"bilinear": 0, "nearest": 1}


def _scalars(img, angle, center, dtype):
    """angle / center as the plugin receives them: device tensors [1] / [2] of the image's float type."""
    angle = torch.as_tensor(angle, device=img.device).to(dtype).reshape(-1)
    center = torch.as_tensor(center, device=img.device).to(dtype).reshape(-1)
    if angle.numel() != 1 or center.numel() != 2:
        raise ValueError("rotate: angle must have 1 element and center 2 (x, y)")
    return angle.contiguous(), center.contiguous()


def _is_hwc_view(img):
    """True for a [C, H, W] view whose memory is a dense [H, W, C] tensor (what .view(H, W, C).permute(2, 0, 1) gives)."""
    c, h, w = img.shape
    return c > 1 and img.stride() == (1, w * c, c)


def _check_image(name, img, layout):
    """A 3-D FP32 / FP16 CUDA image (`layout` names its axes for the message)."""
    if not img.is_cuda:
        raise RuntimeError(f"{name}: img must be a CUDA tensor (no CPU fallback exists)")
    if img.dim() != 3:
        raise RuntimeError(f"{name}: img must be {layout}")
    if img.dtype not in (torch.float32, torch.float16):
        raise _lib.B200OpsError(name, 1)


def _check_packed(name, img, channels, width, dtype):
    """Shape first, then device and dtype: img [ceil(channels / width), H, W, width]. Returns the contiguous image."""
    if img.dim() != 4 or img.shape[-1] != width or -(-channels // width) != img.shape[0]:
        raise ValueError(f"{name}: img must be [ceil({channels} / {width}), H, W, {width}], got {tuple(img.shape)}")
    if not img.is_cuda or img.dtype != dtype:
        raise RuntimeError(f"{name}: img must be a {dtype} CUDA tensor")
    return img.contiguous()


def _forward(img, angle, center, interpolation):
    _check_image("rotate", img, "[C, H, W]")
    c, h, w = img.shape
    vec = 4 if img.dtype == torch.float32 else 8
    if _is_hwc_view(img) and c % vec == 0 and img.data_ptr() % 16 == 0:
        return rotate_hwc(img.permute(1, 2, 0), angle, center, interpolation).permute(2, 0, 1)
    img = img.contiguous()
    angle, center = _scalars(img, angle, center, img.dtype)
    out = torch.empty_like(img)
    name = "b200_rotate_f32" if img.dtype == torch.float32 else "b200_rotate_f16"
    _lib.call(name, img.device, out.data_ptr(), img.data_ptr(), angle.data_ptr(), center.data_ptr(),
              (ctypes.c_int * 3)(c, h, w), int(interpolation))  # fmt: skip
    return out


def _make(op_name):
    class _Rotate(Function):
        @staticmethod
        def symbolic(g, img, angle, center, interpolation):
            return g.op(op_name, img, angle, center, interpolation_i=interpolation)

        @staticmethod
        def forward(ctx, img, angle, center, interpolation):
            return _forward(img, angle, center, interpolation)

        @staticmethod
        def backward(ctx, grad_output):
            raise NotImplementedError

    _Rotate.__name__ = "_" + op_name
    return _Rotate


_Rotate = _make("RotateTRT")
_Rotate2 = _make("RotateTRT2")


def rotate(img, angle, center, interpolation="nearest"):
    """Plugin RotateTRT (FP32, FP16). Same contract as the reference wrapper (rotate.py:99-115)."""
    return _Rotate.apply(img, angle, center, _MODE[interpolation])


def rotate2(img, angle, center, interpolation="nearest"):
    """Plugin RotateTRT2 (FP16 as half2). Same contract as the reference wrapper (rotate.py:118-134). On PyTorch
    tensors (plain [C, H, W]) it is numerically the same op; the packed-layout kernel is ``rotate_chw2``."""
    return _Rotate2.apply(img, angle, center, _MODE[interpolation])


def rotate_hwc(img_hwc, angle, center, interpolation="nearest"):
    """Channels-last image [H, W, C] (dense), FP32 or FP16; returns [H, W, C]."""
    _check_image("rotate_hwc", img_hwc, "[H, W, C]")
    img_hwc = img_hwc.contiguous()
    h, w, c = img_hwc.shape
    angle, center = _scalars(img_hwc, angle, center, img_hwc.dtype)
    out = torch.empty_like(img_hwc)
    mode = _MODE[interpolation] if isinstance(interpolation, str) else int(interpolation)
    _lib.call("b200_rotate_hwc", img_hwc.device, out.data_ptr(), img_hwc.data_ptr(), angle.data_ptr(),
              center.data_ptr(), 0 if img_hwc.dtype == torch.float32 else 1, (ctypes.c_int * 3)(c, h, w), mode)  # fmt: skip
    return out


def rotate_chw2(img_chw2, channels, angle, center, interpolation="nearest"):
    """FP16 kCHW2 image [ceil(C/2), H, W, 2] (rotate_h2, rotateKernel.h:18-20). Returns kCHW2."""
    img_chw2 = _check_packed("rotate_chw2", img_chw2, channels, 2, torch.float16)
    _, h, w, _ = img_chw2.shape
    angle, center = _scalars(img_chw2, angle, center, torch.float16)
    out = torch.empty_like(img_chw2)
    _lib.call("b200_rotate_f16_h2", img_chw2.device, out.data_ptr(), img_chw2.data_ptr(), angle.data_ptr(),
              center.data_ptr(), (ctypes.c_int * 3)(channels, h, w), _MODE[interpolation])  # fmt: skip
    return out


def rotate_int8(img_chw4, scale_i, channels, angle, center, scale_o, interpolation="nearest"):
    """INT8 kCHW4 image [ceil(C/4), H, W, 4] with per-tensor scales (real = q*scale); angle / center float32 or
    float16 tensors (rotate_int8<T>, rotateKernel.h:22-26; rotatePlugin.cpp:101-111). Returns kCHW4 int8."""
    img_chw4 = _check_packed("rotate_int8", img_chw4, channels, 4, torch.int8)
    _, h, w, _ = img_chw4.shape
    adt = angle.dtype if torch.is_tensor(angle) and angle.dtype == torch.float16 else torch.float32
    angle, center = _scalars(img_chw4, angle, center, adt)
    out = torch.empty_like(img_chw4)
    _lib.call("b200_rotate_i8", img_chw4.device, out.data_ptr(), float(scale_o), img_chw4.data_ptr(), float(scale_i),
              angle.data_ptr(), center.data_ptr(), int(adt == torch.float16), (ctypes.c_int * 3)(channels, h, w),
              _MODE[interpolation])  # fmt: skip
    return out
