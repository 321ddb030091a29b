"""BEVPoolV2 — host-side mirror of the reference binding det2trt/models/functions/bev_pool_v2.py: ``bev_pool_v2`` and
its twin ``bev_pool_v2_2`` (plugins BEVPoolV2TRT / BEVPoolV2TRT2), with the same positional signature, defaults and ONNX
symbolics (``out_height_i``, ``out_width_i``). BEVDet calls it between the depth net and the BEV encoder.

    depth [N, D, H, W], feat [N, H, W, C] (channels last), ranks_depth / ranks_feat / ranks_bev [P],
    interval_starts / interval_lengths [I]  ->  out [1, out_height, out_width, C]
    out[ranks_bev[s_k], c] = sum_{i = s_k}^{s_k + len_k - 1} feat[ranks_feat[i], c] * depth[ranks_depth[i]]

Input contract (what ``voxel_pooling_prepare_v2`` produces, and what the reference assumes): points sorted by
``ranks_bev``, one interval per distinct cell, each depth element referenced by at most one point. Two intervals naming
the same cell, or a repeated ``ranks_depth``, are outside it. Every cell no interval names is +0. Unlike the reference,
every index is checked against the tensor it indexes: an interval whose cell is out of range is dropped, so is a point
whose ``ranks_depth`` or ``ranks_feat`` is out of range, and ``[start, start + length)`` is clipped to ``[0, P)``.

Index tensors go through ``.int()`` as in the reference (its TensorRT test feeds float ranks). Dtypes (depth, feat):

    depth     feat      out       depth grad   feat grad
    float32   float32   float32   float32      float32
    float16   float16   float16   float16      float16
    bfloat16  bfloat16  bfloat16  bfloat16     bfloat16
    float32   float16   float16   float32      float16     what torch.autocast hands the op: a softmax depth
    float32   bfloat16  bfloat16  float32      bfloat16    and conv features

Any other pair raises ``B200OpsError`` with status 1. The output has the features' dtype, as the plugin returns its
input's; the reference's eager path returns float32 because mmdet3d's ``QuickCumsumCuda`` upcasts. FP32 is the reference
kernel's FFMA chain bit for bit; every 2-byte element is widened to FP32 exactly, FP32 depth is used as loaded, the sum
is accumulated in FP32 and each 2-byte result rounded once, to nearest even. Both names run the same kernels.

Trainable: the backward returns each gradient in its argument's dtype, ``grad_out`` cast to the features' dtype (FP32
accumulation, no atomics, the same bits on every run and for every subset of gradients). ``bev_pool_v2_int8`` is the
INT8 inference form.
"""
import ctypes

import torch
from torch.autograd import Function

from .. import _lib


def _inputs(depth, feat, ranks):
    tensors = (depth, feat) + tuple(ranks)
    if not all(isinstance(t, torch.Tensor) and t.is_cuda for t in tensors):
        raise RuntimeError("bev_pool_v2: every input must be a CUDA tensor (no CPU fallback exists)")
    if feat.dim() < 1 or feat.shape[-1] == 0:
        raise RuntimeError("bev_pool_v2: feat must be [N, H, W, C] with C > 0")
    if any(t.device != feat.device for t in tensors):
        raise RuntimeError("bev_pool_v2: all inputs must be on one device")
    ranks = tuple(r.int().contiguous().reshape(-1) for r in ranks)
    if ranks[0].numel() != ranks[1].numel() or ranks[0].numel() != ranks[2].numel():
        raise RuntimeError("bev_pool_v2: ranks_depth, ranks_feat and ranks_bev must have the same length")
    if ranks[3].numel() != ranks[4].numel():
        raise RuntimeError("bev_pool_v2: interval_starts and interval_lengths must have the same length")
    return depth.contiguous(), feat.contiguous(), ranks


def _extents(depth, feat, ranks):
    C = feat.shape[-1]
    return [C, ranks[0].numel(), ranks[3].numel(), depth.numel(), feat.numel() // C]


# (depth dtype, feat dtype) -> (forward entry, backward entry, leading feat_dtype argument of the entries)
_ENTRIES = {
    (torch.float32, torch.float32): ("b200_bev_pool_f32", "b200_bev_pool_backward_f32", ()),
    (torch.float16, torch.float16): ("b200_bev_pool_f16", "b200_bev_pool_backward_f16", ()),
    (torch.bfloat16, torch.bfloat16): ("b200_bev_pool_bf16", "b200_bev_pool_backward_bf16", ()),
    (torch.float32, torch.float16): ("b200_bev_pool_f32_depth", "b200_bev_pool_backward_f32_depth", (1,)),
    (torch.float32, torch.bfloat16): ("b200_bev_pool_f32_depth", "b200_bev_pool_backward_f32_depth", (7,)),
}


def _entries(depth, feat):
    entries = _ENTRIES.get((depth.dtype, feat.dtype))
    if entries is None:
        raise _lib.B200OpsError("bev_pool_v2", 1)
    return entries


def _forward(depth, feat, ranks, out_height, out_width):
    depth, feat, ranks = _inputs(depth, feat, ranks)
    name, _, lead = _entries(depth, feat)
    out = torch.empty(1, int(out_height), int(out_width), feat.shape[-1], dtype=feat.dtype, device=feat.device)
    _lib.call(name, feat.device, *lead, depth.data_ptr(), feat.data_ptr(), *(r.data_ptr() for r in ranks),
              *_extents(depth, feat, ranks), int(out_height), int(out_width), out.data_ptr())  # fmt: skip
    return out


def _backward(ctx, grad_out):
    need_d, need_f = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
    none = (None,) * 7
    if not (need_d or need_f):
        return (None, None) + none
    depth, feat, *ranks = ctx.saved_tensors
    og = grad_out.to(feat.dtype).contiguous()
    P = ranks[0].numel()
    order = torch.sort(ranks[1], stable=True).indices.int() if need_f and P else None
    ws = torch.empty(max(P, 1), dtype=torch.int32, device=feat.device)
    dg = torch.empty_like(depth) if need_d else None
    fg = torch.empty_like(feat) if need_f else None
    _, name, lead = _entries(depth, feat)
    _lib.call(name, feat.device, *lead, og.data_ptr(), depth.data_ptr(), feat.data_ptr(), *(r.data_ptr() for r in ranks),
              order.data_ptr() if order is not None else None, *_extents(depth, feat, ranks), *ctx.out_hw,
              dg.data_ptr() if need_d else None, fg.data_ptr() if need_f else None, ws.data_ptr(),
              ws.numel() * 4)  # fmt: skip
    return (dg, fg) + none


def _make(op_name):
    class _BEVPoolV2(Function):
        @staticmethod
        def symbolic(g, depth, feat, ranks_depth, ranks_feat, ranks_bev, interval_starts, interval_lengths, out_height,
                     out_width):  # fmt: skip
            return g.op(op_name, depth, feat, ranks_depth, ranks_feat, ranks_bev, interval_starts, interval_lengths,
                        out_height_i=out_height, out_width_i=out_width)  # fmt: skip

        @staticmethod
        def forward(ctx, depth, feat, ranks_depth, ranks_feat, ranks_bev, interval_starts, interval_lengths, out_height,
                    out_width):  # fmt: skip
            ranks = (ranks_depth, ranks_feat, ranks_bev, interval_starts, interval_lengths)
            out = _forward(depth, feat, ranks, out_height, out_width)
            if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
                depth, feat, ranks = _inputs(depth, feat, ranks)
                ctx.save_for_backward(depth, feat, *ranks)
                ctx.out_hw = (int(out_height), int(out_width))
            return out

        backward = staticmethod(_backward)

    _BEVPoolV2.__name__ = "_" + op_name
    return _BEVPoolV2


_BEVPoolV2 = _make("BEVPoolV2TRT")
_BEVPoolV2_2 = _make("BEVPoolV2TRT2")


def bev_pool_v2(depth, feat, ranks_depth, ranks_feat, ranks_bev, interval_starts, interval_lengths, out_height=128,
                out_width=128):  # fmt: skip
    """Plugin BEVPoolV2TRT. Returns [1, out_height, out_width, C] in the features' dtype; (depth, feat) float32,
    float16 or bfloat16 pairs, or float32 depth with float16 / bfloat16 features (the module docstring's table)."""
    return _BEVPoolV2.apply(depth, feat, ranks_depth.int(), ranks_feat.int(), ranks_bev.int(), interval_starts.int(),
                            interval_lengths.int(), out_height, out_width)  # fmt: skip


def bev_pool_v2_2(depth, feat, ranks_depth, ranks_feat, ranks_bev, interval_starts, interval_lengths, out_height=128,
                  out_width=128):  # fmt: skip
    """Plugin BEVPoolV2TRT2: the same op and kernels as ``bev_pool_v2`` (the reference's variant picks a half2 kernel)."""
    return _BEVPoolV2_2.apply(depth, feat, ranks_depth.int(), ranks_feat.int(), ranks_bev.int(), interval_starts.int(),
                              interval_lengths.int(), out_height, out_width)  # fmt: skip


def bev_pool_v2_int8(depth_q, scale_d, feat_q, scale_f, ranks_depth, ranks_feat, ranks_bev, interval_starts,
                     interval_lengths, scale_o, out_height=128, out_width=128):  # fmt: skip
    """INT8 form of the plugin: int8 depth / feat with per-tensor scales, int8 output at ``scale_o``. The kernel sums
    ``feat_q * depth_q`` exactly in int32, multiplies once by ``scale_d * scale_f / scale_o`` (float32) and rounds half
    away from zero with saturation, as the reference's INT8 kernel does. Needs C % 4 == 0 (else status 1)."""
    ranks = (ranks_depth, ranks_feat, ranks_bev, interval_starts, interval_lengths)
    depth_q, feat_q, ranks = _inputs(depth_q, feat_q, ranks)
    if depth_q.dtype != torch.int8 or feat_q.dtype != torch.int8:
        raise _lib.B200OpsError("bev_pool_v2_int8", 1)
    out = torch.empty(1, int(out_height), int(out_width), feat_q.shape[-1], dtype=torch.int8, device=feat_q.device)
    f = ctypes.c_float
    _lib.call("b200_bev_pool_i8", feat_q.device, depth_q.data_ptr(), f(scale_d), feat_q.data_ptr(), f(scale_f),
              *(r.data_ptr() for r in ranks), *_extents(depth_q, feat_q, ranks), int(out_height), int(out_width),
              out.data_ptr(), f(scale_o))  # fmt: skip
    return out
