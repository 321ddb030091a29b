"""Modulated deformable convolution (DCNv2) — host-side mirror of the reference binding
det2trt/models/functions/modulated_deformable_conv2d.py (:13-291): ``modulated_deformable_conv2d(input, offset, mask,
weight, bias=None, stride=1, padding=0, dilation=1, groups=1, deform_groups=1)`` and its twin
``modulated_deformable_conv2d2`` (plugin …TRT2), same ONNX symbolic attributes, used by DCNv2P
(det2trt/models/modules/cnn/dcn.py:70-86: ``offset = cat(o1, o2)``, ``mask = sigmoid(mask)``).

The reference's forward calls mmcv's ``modulated_deform_conv_forward`` (:84-104) and its backward mmcv's
``modulated_deform_conv_backward`` (:107-157); here both call the sm_90a kernels behind the C ABI. The backward returns
gradients for input, offset, mask, weight and bias (``once_differentiable``, as in the reference)."""
import weakref

import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable
from torch.nn.modules.utils import _pair

from .. import _lib


def _out_extent(size, kernel, stride, padding, dilation):
    """Output length of a convolution along one axis."""
    return (size + 2 * padding - (dilation * (kernel - 1) + 1)) // stride + 1


def _forward(input, offset, mask, weight, bias, stride, padding, dilation, groups, deform_groups):
    if not input.is_cuda:
        raise RuntimeError("modulated_deformable_conv2d: input must be a CUDA tensor (no CPU fallback exists)")
    if input.dim() != 4 or weight.dim() != 4:
        raise ValueError("input must be [N,C,H,W] and weight [Co, C/groups, kh, kw]")
    dt = input.dtype
    suffix, code = _lib.float_dtype(dt, "modulated_deformable_conv2d")
    (sh, sw), (ph, pw), (dh, dw) = _pair(stride), _pair(padding), _pair(dilation)
    n, c, h, w = input.shape
    co, cig, kh, kw = weight.shape
    if cig * groups != c:
        raise ValueError("weight.shape[1] * groups must equal the input channels")
    ho, wo = _out_extent(h, kh, sh, ph, dh), _out_extent(w, kw, sw, pw, dw)
    if tuple(offset.shape) != (n, deform_groups * 2 * kh * kw, ho, wo):
        raise ValueError(f"offset must be {(n, deform_groups * 2 * kh * kw, ho, wo)}, got {tuple(offset.shape)}")
    if tuple(mask.shape) != (n, deform_groups * kh * kw, ho, wo):
        raise ValueError(f"mask must be {(n, deform_groups * kh * kw, ho, wo)}, got {tuple(mask.shape)}")
    lib = _lib.load()
    fused = (dt == torch.float16 and groups == 1 and deform_groups == 1 and c % 64 == 0 and co in (128, 256, 512)
             and kh * kw <= 9 and lib.b200_dcn_set_fused(-1) == 1)
    if fused:
        return _forward_fused_f16(lib, input, offset, mask, weight, bias, (sh, sw), (ph, pw), (dh, dw), (ho, wo))
    input, offset, mask, weight = (t.to(dt).contiguous() for t in (input, offset, mask, weight))
    bias_t = bias.to(dt).contiguous() if bias is not None else None
    ws_bytes = lib.b200_dcn_workspace_size(code, n, c, h, w, kw, kh, sw, sh, pw, ph, dw, dh)
    workspace = torch.empty(ws_bytes, dtype=torch.uint8, device=input.device)
    out = torch.empty(n, co, ho, wo, dtype=dt, device=input.device)
    _lib.call(f"b200_dcn_{suffix}", input.device, input.data_ptr(), weight.data_ptr(),
              bias_t.data_ptr() if bias_t is not None else None, offset.data_ptr(), mask.data_ptr(), out.data_ptr(),
              workspace.data_ptr(), n, c, h, w, co, kw, kh, sw, sh, pw, ph, dw, dh, groups, deform_groups, min(n, 32),
              None)  # fmt: skip
    return out


_PACKED = {}  # id(weight) -> (weakref to the weight, its _version, packed copy); entries die with their weight


def _pack(lib, weight):
    co, c, kh, kw = weight.shape
    packed = torch.empty_like(weight, memory_format=torch.contiguous_format)
    _lib.call("b200_dcn_pack_weights_f16", weight.device, weight.data_ptr(), packed.data_ptr(), co, c, kh, kw)
    return packed


def _packed_weight(lib, weight):
    """Weights permuted for the fused kernel. The permutation is constant at inference, so it is cached — but only for
    long-lived tensors the caller owns (``nn.Parameter`` / registered buffers, i.e. tensors that are not the result of
    a cast or ``.contiguous()`` made for this call), and the entry is tied to that tensor OBJECT by a weak reference:
    a freed weight takes its entry with it, so a new tensor that lands on the same address can never see stale packed
    weights. In-place updates are caught by ``_version``. Temporaries are packed on every call (a 1.2 MB kernel)."""
    cacheable = isinstance(weight, torch.nn.Parameter) or getattr(weight, "_b200_cache_packed", False)
    if not cacheable or not weight.is_contiguous() or weight.dtype != torch.float16:
        return _pack(lib, weight.to(torch.float16).contiguous())
    key = id(weight)
    hit = _PACKED.get(key)
    if hit is not None and hit[0]() is weight and hit[1] == weight._version:
        return hit[2]
    packed = _pack(lib, weight)
    _PACKED[key] = (weakref.ref(weight, lambda _r, k=key: _PACKED.pop(k, None)), weight._version, packed)
    return packed


def _forward_fused_f16(lib, input, offset, mask, weight, bias, stride, padding, dilation, out_hw):
    """FP16 fused tensor-core path: the weight permutation is cached per weight tensor, and a channels-last input is
    consumed in place (no NCHW->NHWC pre-pass)."""
    n, c, h, w = input.shape
    co, _, kh, kw = weight.shape
    dt = torch.float16
    flags = 2
    if input.is_contiguous(memory_format=torch.channels_last) and not input.is_contiguous():
        flags |= 1  # NHWC bytes already
        x = input
    else:
        x = input.contiguous()
    if x.data_ptr() % 16:  # a view at an odd storage offset: the pre-pass / gather use 128-bit loads
        x = x.clone()  # dense, so the copy keeps the memory format
    wp = _packed_weight(lib, weight)
    offset, mask = offset.to(dt).contiguous(), mask.to(dt).contiguous()
    bias_t = bias.to(dt).contiguous() if bias is not None else None
    ws_bytes = lib.b200_dcn_workspace_size(1, n, c, h, w, kw, kh, stride[1], stride[0], padding[1], padding[0],
                                           dilation[1], dilation[0])  # fmt: skip
    workspace = torch.empty(ws_bytes, dtype=torch.uint8, device=input.device)
    out = torch.empty(n, co, out_hw[0], out_hw[1], dtype=dt, device=input.device)
    _lib.call("b200_dcn_f16_ex", input.device, x.data_ptr(), wp.data_ptr(),
              bias_t.data_ptr() if bias_t is not None else None, offset.data_ptr(), mask.data_ptr(), out.data_ptr(),
              workspace.data_ptr(), n, c, h, w, co, kw, kh, stride[1], stride[0], padding[1], padding[0], dilation[1],
              dilation[0], 1, 1, flags)  # fmt: skip
    return out


def _backward(grad_out, input, offset, mask, weight, bias, stride, padding, dilation, groups, deform_groups, needs):
    """Gradients for (input, offset, mask, weight, bias), None where ``needs`` says not wanted. They are computed from
    the values the forward used (offset, mask, weight and bias cast to the input dtype) and returned in the dtype of
    the tensor the caller passed."""
    dt = input.dtype
    suffix, code = _lib.float_dtype(dt, "modulated_deformable_conv2d")
    (sh, sw), (ph, pw), (dh, dw) = _pair(stride), _pair(padding), _pair(dilation)
    x, off, msk, wt = (t.to(dt).contiguous() for t in (input, offset, mask, weight))
    go = grad_out.to(dt).contiguous()
    n, c, h, w = x.shape
    co, _, kh, kw = wt.shape
    lib = _lib.load()
    ws_bytes = lib.b200_dcn_backward_workspace_size(code, n, c, h, w, co, kw, kh, sw, sh, pw, ph, dw,
                                                    dh, groups, deform_groups)  # fmt: skip
    if ws_bytes == 0:
        raise _lib.B200OpsError("b200_dcn_backward_workspace_size", 2)
    workspace = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
    want = [needs[0], needs[3], needs[4] and bias is not None, needs[1], needs[2]]  # the C ABI's order
    like = [x, wt, go.new_empty(co), off, msk]
    grads = [torch.empty_like(t, memory_format=torch.contiguous_format) if k else None for k, t in zip(want, like)]
    ptr = [g.data_ptr() if g is not None else None for g in grads]
    flags = [0] if dt == torch.float16 else []  # the layout flags of the FP16 entry: plain NCHW, unpacked weights
    _lib.call(f"b200_dcn_backward_{suffix}", x.device, x.data_ptr(), wt.data_ptr(), off.data_ptr(), msk.data_ptr(), go.data_ptr(), *ptr,
              workspace.data_ptr(), n, c, h, w, co, kw, kh, sw, sh, pw, ph, dw, dh, groups, deform_groups, *flags)
    gi, gw, gb, go_, gm = grads
    cast = lambda g, t: g.to(t.dtype) if g is not None else None  # noqa: E731
    return cast(gi, input), cast(go_, offset), cast(gm, mask), cast(gw, weight), cast(gb, bias)


def _make(op_name):
    class _ModulatedDeformableConv2dFunction(Function):
        @staticmethod
        def symbolic(g, input, offset, mask, weight, bias, stride, padding, dilation, groups, deform_groups):
            inputs = [input, offset, mask, weight] + ([bias] if bias is not None else [])
            return g.op(op_name, *inputs, stride_i=_pair(stride), padding_i=_pair(padding), dilation_i=_pair(dilation),
                        groups_i=groups, deform_groups_i=deform_groups)  # fmt: skip

        @staticmethod
        def forward(ctx, input, offset, mask, weight, bias=None, stride=1, padding=0, dilation=1, groups=1,
                    deform_groups=1):  # fmt: skip
            if any(t is not None and t.requires_grad for t in (input, offset, mask, weight, bias)):
                ctx.save_for_backward(input, offset, mask, weight, bias)
                ctx.geometry = (stride, padding, dilation, groups, deform_groups)
            return _forward(input, offset, mask, weight, bias, stride, padding, dilation, groups, deform_groups)

        @staticmethod
        @once_differentiable
        def backward(ctx, grad_out):
            grads = _backward(grad_out, *ctx.saved_tensors, *ctx.geometry, ctx.needs_input_grad)
            return (*grads, None, None, None, None, None)

    return _ModulatedDeformableConv2dFunction


_ModulatedDeformableConv2dFunction = _make("ModulatedDeformableConv2dTRT")
_ModulatedDeformableConv2dFunction2 = _make("ModulatedDeformableConv2dTRT2")


def modulated_deformable_conv2d(input, offset, mask, weight, bias=None, stride=1, padding=0, dilation=1, groups=1,
                                deform_groups=1):
    """Plugin ModulatedDeformableConv2dTRT (FP32 / FP16 / BF16). Same contract as the reference wrapper (:208-248).
    Offset, mask, weight and bias are cast to the input's dtype; gradients come back in each argument's own dtype. BF16
    runs the generic kernel (csrc/dcn_generic.cu) for every shape."""
    return _ModulatedDeformableConv2dFunction.apply(input, offset, mask, weight, bias, stride, padding, dilation,
                                                    groups, deform_groups)  # fmt: skip


def modulated_deformable_conv2d2(input, offset, mask, weight, bias=None, stride=1, padding=0, dilation=1, groups=1,
                                 deform_groups=1):
    """Plugin ModulatedDeformableConv2dTRT2 (FP16 as half2). Same contract as the reference wrapper (:251-291)."""
    return _ModulatedDeformableConv2dFunction2.apply(input, offset, mask, weight, bias, stride, padding, dilation,
                                                     groups, deform_groups)  # fmt: skip


def modulated_deformable_conv2d_chw2(input_chw2, offset_chw2, mask, weight_chw2, bias, channels, stride=1, padding=0,
                                     dilation=1, groups=1, deform_groups=1):
    """FP16 in TensorRT's kCHW2 packets, the format table of the …TRT2 plugin (…Conv2dPlugin.cpp:222-250): ``input_chw2``
    [N, ceil(C/2), H, W, 2], ``offset_chw2`` [N, ceil(dg*2*kh*kw/2), Ho, Wo, 2], ``weight_chw2`` [Co, ceil(C/g/2), kh, kw, 2]
    (``functions.grid_sampler.pack_chw(x, 2)``); ``mask`` / ``bias`` plain FP16. Returns plain NCHW FP16."""
    assert input_chw2.is_cuda and input_chw2.dtype == torch.float16 and input_chw2.shape[-1] == 2
    (sh, sw), (ph, pw), (dh, dw) = _pair(stride), _pair(padding), _pair(dilation)
    n, _, h, w, _ = input_chw2.shape
    co, _, kh, kw, _ = weight_chw2.shape
    ho, wo = _out_extent(h, kh, sh, ph, dh), _out_extent(w, kw, sw, pw, dw)
    lib = _lib.load()
    ws_bytes = lib.b200_dcn_f16_chw2_workspace_size(n, channels, h, w, co, kw, kh, sw, sh, pw, ph, dw, dh, groups, deform_groups)
    workspace = torch.empty(ws_bytes, dtype=torch.uint8, device=input_chw2.device)
    out = torch.empty(n, co, ho, wo, dtype=torch.float16, device=input_chw2.device)
    x, off, msk, wt = (t.contiguous() for t in (input_chw2, offset_chw2, mask.half(), weight_chw2))
    bias_t = bias.half().contiguous() if bias is not None else None
    _lib.call("b200_dcn_f16_chw2", x.device, x.data_ptr(), wt.data_ptr(),
              bias_t.data_ptr() if bias_t is not None else None, off.data_ptr(), msk.data_ptr(), out.data_ptr(),
              workspace.data_ptr(), n, channels, h, w, co, kw, kh, sw, sh, pw, ph, dw, dh, groups, deform_groups,
              min(n, 32), None)  # fmt: skip
    return out


def modulated_deformable_conv2d_int8(input_chw4, scale_i, offset_q, scale_off, mask_q, scale_mask, weight_chw4, scale_w,
                                     bias, scale_o, channels, stride=1, padding=0, dilation=1, groups=1, deform_groups=1):
    """INT8 flavour of the plugin (…Conv2dPlugin.cpp:117-199 / launcher …Conv2dKernel.h:21-29): ``input_chw4`` int8
    [N, C/4, H, W, 4] and ``weight_chw4`` int8 [Co, C/4, kh, kw, 4] in TensorRT's kCHW4 layout
    (``functions.grid_sampler.pack_chw(x, 4)``), ``offset_q`` / ``mask_q`` int8 NCHW, per-tensor scales
    (real = q*scale), ``bias`` float32/float16 or None. Returns int8 [N, Co, Ho, Wo] at ``scale_o``. Backbone shapes
    run on the fused tensor-core kernel; other shapes (groups / deform_groups > 1, small channel counts) dequantise
    into the workspace and take the generic hand-written kernel (csrc/dcn_generic.cu)."""
    assert input_chw4.is_cuda and input_chw4.dtype == torch.int8 and input_chw4.shape[-1] == 4
    (sh, sw), (ph, pw), (dh, dw) = _pair(stride), _pair(padding), _pair(dilation)
    n, c4, h, w, _ = input_chw4.shape
    co, _, kh, kw, _ = weight_chw4.shape
    if c4 * 4 != channels or weight_chw4.shape[1] * 4 * groups != channels:
        raise ValueError("channels must be a multiple of 4 and match the packed tensors")
    ho, wo = _out_extent(h, kh, sh, ph, dh), _out_extent(w, kw, sw, pw, dw)
    if tuple(offset_q.shape) != (n, deform_groups * 2 * kh * kw, ho, wo) or \
            tuple(mask_q.shape) != (n, deform_groups * kh * kw, ho, wo):
        raise ValueError("offset / mask must be [N, deform_groups*2*kh*kw, Ho, Wo] / [N, deform_groups*kh*kw, Ho, Wo]")
    lib = _lib.load()
    ws_bytes = lib.b200_dcn_i8_workspace_size(n, channels, h, w, co, kw, kh, sw, sh, pw, ph, dw, dh, groups, deform_groups)
    workspace = torch.empty(ws_bytes, dtype=torch.uint8, device=input_chw4.device)
    out = torch.empty(n, co, ho, wo, dtype=torch.int8, device=input_chw4.device)
    x, wt, off, msk = (t.contiguous() for t in (input_chw4, weight_chw4, offset_q, mask_q))
    # the library reads kCHW4 packets as 32-bit words: a view at an unaligned storage offset goes through a fresh copy
    x, wt = (t.clone() if t.data_ptr() % 4 else t for t in (x, wt))
    bias_t = bias.contiguous() if bias is not None else None
    if bias_t is not None and bias_t.dtype not in (torch.float32, torch.float16):
        raise _lib.B200OpsError("modulated_deformable_conv2d_int8", 1)
    _lib.call("b200_dcn_i8", x.device, x.data_ptr(), float(scale_i), wt.data_ptr(), float(scale_w),
              bias_t.data_ptr() if bias_t is not None else None,
              int(bias_t is not None and bias_t.dtype == torch.float16), off.data_ptr(), float(scale_off), msk.data_ptr(),
              float(scale_mask), out.data_ptr(), float(scale_o), workspace.data_ptr(), n, channels, h, w, co, kw, kh, sw,
              sh, pw, ph, dw, dh, groups, deform_groups, min(n, 32), None)  # fmt: skip
    return out
