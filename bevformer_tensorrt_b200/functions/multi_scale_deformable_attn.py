"""Multi-scale deformable attention — host-side mirror of the reference binding
det2trt/models/functions/multi_scale_deformable_attn.py (:10-217): same module-level names, same positional
signature, same ONNX symbolic, so SpatialCrossAttentionTRTP / TemporalSelfAttentionTRTP / the decoder's
CustomMSDeformableAttentionTRTP call it unchanged (spatial_cross_attention.py:692,764-766;
temporal_self_attention.py:348,447-449; decoder.py:376,460-466).

The reference's forward() expands to sampling locations + softmax and calls mmcv's CUDA op; here forward() hands the
plugin-signature tensors straight to the fused sm_90a kernel behind the C ABI (include/b200_bev_ops.h). The reference's
Function defines no backward; this one does (csrc/msda_backward.cu: value, reference-point, sampling-offset and
pre-softmax logit gradients), so the attention modules train through the plugin-signature op. The fused forms
``…_sca``, ``…_sca_shared`` and (through ``…_sca``) ``…_queue_mean`` are differentiable too: they record a graph only
when grad mode is on and an input requires grad, so inference calls run exactly as before. ``…_sca`` with ``accum=``
given, and INT8, are inference-only.
"""
import os
from typing import NamedTuple

import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from .. import _lib

# Second-generation INT8 path (csrc/msda_v2.cu: pack pre-pass + 128-byte-run gather with dp2a) at channels == 32 and
# 16 <= levels*points <= 32 — every SpatialCrossAttention call of BEVFormer. Other shapes (TSA, decoder: 4 points) and the
# FP16 / FP32 ops run the round-1 kernel (csrc/msda.cu). B200_MSDA_V2=0 or set_msda_v2(False) forces the round-1 kernel.
_V2 = {"enabled": os.environ.get("B200_MSDA_V2", "1") != "0"}


def set_msda_v2(enabled: bool) -> bool:
    """Enables / disables the second-generation INT8 MSDA path; returns the previous setting."""
    prev, _V2["enabled"] = _V2["enabled"], bool(enabled)
    return prev


def set_msda_f16_path(resident: bool, resident_bytes: int = None):
    """Selects the kernel behind the FP16 plugin op: False (library default) = the gather kernel (csrc/msda.cu);
    True = the resident-tail kernel (csrc/msda_res.cu: coarse pyramid levels staged in shared memory by TMA) where its
    envelope holds — measured slower, opt-in. ``resident_bytes``: shared memory the resident kernel may use for the tail.
    Returns the previous (path, bytes-or-None)."""
    lib = _lib.load()
    prev = bool(lib.b200_msda_set_f16_path(int(bool(resident))))
    prev_bytes = None
    if resident_bytes is not None:
        prev_bytes = int(lib.b200_msda_set_resident_bytes(int(resident_bytes)))
    return prev, prev_bytes


def set_msda_batch_units(units: int, strided: bool = False):
    """Launch shape of the FP32 / FP16 plugin op (C entry b200_msda_set_batch_units): ``units`` = 1 is one block of
    items per CTA; 2 or 4 is the batched launch, where every warp first scans the visibility of that many item groups
    with all their loads in flight, writes zeros for the invisible ones and samples the rest. ``strided``: the units of
    a CTA lie a grid apart instead of side by side. Results are bit-identical for every setting.
    Returns the previous (units, strided)."""
    if units not in (1, 2, 4):
        raise ValueError("units must be 1, 2 or 4")
    prev = int(_lib.load().b200_msda_set_batch_units(int(units), int(bool(strided))))
    return prev & 0xFF, bool(prev >> 8)


def get_msda_batch_units():
    """Current (units, strided) of the FP32 / FP16 plugin-op launch."""
    prev = int(_lib.load().b200_msda_set_batch_units(0, 0))
    return prev & 0xFF, bool(prev >> 8)


def set_msda_gather_variant(variant: int) -> int:
    """Gather depth of the FP32 / FP16 plugin op (C entry b200_msda_set_gather_variant): 0 = default (24 warps per SM,
    one sampling point = 4 tap loads in flight per warp), 1 / 2 = 16 warps per SM with the 16 tap loads of a 4-point chunk
    in flight per warp (compiler-scheduled / written out), 3 = 20 warps per SM in 128-thread CTAs with 2 points = 8 loads
    issued together. Same bits for every variant. Returns the previous variant."""
    if variant not in (0, 1, 2, 3):
        raise ValueError("variant must be 0, 1, 2 or 3")
    return int(_lib.load().b200_msda_set_gather_variant(int(variant)))


def get_msda_gather_variant() -> int:
    return int(_lib.load().b200_msda_set_gather_variant(-1))


#: launch shapes autotune_msda tries: name -> (units per warp, grid-strided units, gather variant)
MSDA_LAUNCH_SHAPES = {
    "default": (1, False, 0),
    "batch2_strided": (2, True, 0),
    "deep_gather": (1, False, 1),
    "deep_gather_explicit": (1, False, 2),
    "mid_gather": (1, False, 3),
    "deep_batch2_strided": (2, True, 1),
    "deep_batch4_strided": (4, True, 1),
}


def autotune_msda(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights, iters=12, warmup=3,
                  min_gain=0.02):
    """Picks the launch shape of the FP32 / FP16 plugin op for THESE tensors the way a TensorRT builder picks a tactic:
    every shape in ``MSDA_LAUNCH_SHAPES`` is run on the given CUDA tensors, its output is compared bit for bit with the
    default shape's (a shape that differs is discarded, whatever its speed), and it is timed with CUDA events on the
    current stream (median of ``iters`` after ``warmup``). The fastest shape is made the process-wide setting if it beats
    the default by more than ``min_gain``; otherwise the default stays. Which shape wins depends on the input
    distribution (dense sampling is bound by the L1 line rate and wants warps; camera-ring inputs are latency-bound and
    want loads in flight), which the op cannot know from its arguments. Returns a report dict
    ``{"chosen": name, "ms": {name: median ms}, "rejected": [names]}``."""
    if not value.is_cuda or value.dtype not in (torch.float16, torch.bfloat16, torch.float32):
        raise ValueError("autotune_msda: FP32 / FP16 / BF16 CUDA tensors only (the INT8 op has a single launch shape)")
    args = (value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights)
    set_msda_launch_shape("default")
    base = multi_scale_deformable_attn(*args)
    return _timed_sweep(MSDA_LAUNCH_SHAPES, set_msda_launch_shape, lambda: multi_scale_deformable_attn(*args),
                        lambda: not torch.equal(multi_scale_deformable_attn(*args), base), iters, warmup, min_gain,
                        value.device)  # fmt: skip


def autotune_msda_fused(run, result, iters=10, warmup=2, tol=1e-4, min_gain=0.02):
    """Same idea for the fused spatial-cross-attention forms (``multi_scale_deformable_attn_sca`` /
    ``…_sca_shared``, and through them the sharded multi-GPU step), which have two launch shapes: the default and the
    2-CTAs-per-SM one (any non-zero gather variant). ``run()`` launches the caller's step on the current stream (e.g.
    zero the accumulator + fused op), ``result()`` returns the tensor it produced. The alternative is accepted only if
    its result agrees with the default's to ``tol`` x max|result| (the camera sum uses floating-point atomics, so the last
    bits depend on arrival order in either shape) and it is faster by more than ``min_gain``. Leaves the winner as the
    process-wide gather variant and returns ``{"chosen": "default" | "deep_gather", "ms": {...}, "rejected": [...]}``.
    Local launches only — safe to call per rank before a collective step."""
    variants = {"default": 0, "deep_gather": 1}
    set_msda_gather_variant(0)
    run()
    base = result().detach().float().clone()
    scale = max(1.0, float(base.abs().max()))

    def differs():
        run()
        return float((result().detach().float() - base).abs().max()) > tol * scale

    return _timed_sweep(variants, lambda name: set_msda_gather_variant(variants[name]), run, differs, iters, warmup,
                        min_gain)  # fmt: skip


def _timed_sweep(names, apply, run, differs, iters, warmup, min_gain, device=None):
    """The autotuners' sweep over the launch shapes ``names`` ("default" first), entered with the default applied and
    its result taken. ``apply(name)`` makes a shape the process-wide setting, ``run()`` launches the op once on the
    current stream, ``differs()`` launches it once more and tells whether its result disagrees with the default's (such
    a shape is rejected, whatever its speed). Leaves the chosen shape applied and returns the report."""
    report = {"chosen": "default", "ms": {}, "rejected": []}
    try:
        for _ in range(2 * warmup + 4):  # clocks and caches at their steady state before the first candidate is timed
            run()
        # the default shape is timed first AND last (its better median counts): a clock ramp or a neighbour's burst
        # during the sweep must not hand the win to whichever shape happened to run later
        for name in [*names, "default"]:
            if name in report["rejected"]:
                continue
            apply(name)
            if differs():
                report["rejected"].append(name)
                continue
            for _ in range(warmup):
                run()
            evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
            for a, b in evs:
                a.record()
                run()
                b.record()
            torch.cuda.synchronize(device)
            per = sorted(a.elapsed_time(b) for a, b in evs)
            report["ms"][name] = min(per[len(per) // 2], report["ms"].get(name, float("inf")))
    finally:
        apply("default")
    ms = report["ms"]
    if "default" in ms:
        best = min(ms, key=ms.get)
        if best != "default" and ms[best] < ms["default"] * (1.0 - min_gain):
            report["chosen"] = best
    apply(report["chosen"])
    return report


def set_msda_launch_shape(name: str):
    """Applies one of ``MSDA_LAUNCH_SHAPES`` by name (e.g. the ``chosen`` entry of an earlier ``autotune_msda`` report)."""
    units, strided, variant = MSDA_LAUNCH_SHAPES[name]
    set_msda_batch_units(units, strided)
    set_msda_gather_variant(variant)


class _Prepared(NamedTuple):
    """The tensors an MSDA entry reads — contiguous, int32 level shapes, reference points / offsets / logits in value's
    dtype (BF16: reference points in FP32; INT8: as given) — and the entry's eight dimension arguments
    (_lib._MSDA_DIMS)."""

    value: torch.Tensor
    shapes: torch.Tensor
    ref: torch.Tensor
    off: torch.Tensor
    w: torch.Tensor
    dims: tuple

    def ptrs(self):
        return self.value.data_ptr(), self.shapes.data_ptr(), self.ref.data_ptr(), self.off.data_ptr(), self.w.data_ptr()


def _prepare(name, value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights, dtype,
             bev_mask=None):
    """Checks the inputs of the op ``name`` and makes them what its C entry reads. ``dtype``: value's dtype, FP32, FP16
    or BF16, which offsets and logits are cast to, and reference points too except for BF16, whose entries read them in
    FP32; None (INT8) casts nothing. ``bev_mask`` is given by the
    camera-shared form only: its offsets and logits are ONE copy for all cameras and num_query is read from the mask.
    Otherwise they are ``bs`` copies and num_query is sampling_offsets.shape[1], the reference plugin's rule."""
    if not value.is_cuda:
        raise RuntimeError(f"{name}: value must be a CUDA tensor (no CPU fallback exists)")
    if value.dim() != 4:
        raise ValueError("value must be [bs, num_keys, num_heads, channels]")
    bs, num_keys, num_heads, channels = value.shape
    num_levels = value_spatial_shapes.shape[0]
    if reference_points.shape[-1] % 2 != 0:
        raise ValueError("reference_points last dim must hold (x, y) pairs")
    points_per_group = reference_points.shape[-1] // 2
    all_points = attention_weights.shape[-1]
    if all_points % num_levels != 0:
        raise ValueError("attention_weights last dim must be num_levels * num_points")
    if bev_mask is None:
        num_query, copies, lead = sampling_offsets.shape[1], bs, "bs"
    else:
        num_query, copies, lead = bev_mask.numel() // bs, 1, "1"
    if sampling_offsets.numel() != copies * num_query * num_heads * all_points * 2:
        raise ValueError(f"sampling_offsets does not match [{lead}, num_query, num_heads, num_levels*num_points*2]")
    if attention_weights.numel() != copies * num_query * num_heads * all_points:
        raise ValueError(f"attention_weights does not match [{lead}, num_query, num_heads, num_levels*num_points]")
    if reference_points.numel() != bs * num_query * points_per_group * 2:
        raise ValueError("reference_points does not match [bs, num_query, 1, 2*points_per_group]")
    if dtype is not None:
        _lib.float_dtype(dtype, name)
        # bf16 has 8 significant bits: a normalised reference point near 0.9 would move by up to 2^-9 of the level's
        # extent (0.4 px on a 200-wide BEV plane). A bf16 input is cast up, which is exact.
        reference_points = _cast(reference_points, torch.float32 if dtype == torch.bfloat16 else dtype)
        sampling_offsets = _cast(sampling_offsets, dtype)
        attention_weights = _cast(attention_weights, dtype)
    dims = (bs, num_keys, num_heads, channels, num_levels, num_query, all_points // num_levels, points_per_group)
    return _Prepared(value.contiguous(), _shapes_i32(value_spatial_shapes, value.device), reference_points.contiguous(),
                     sampling_offsets.contiguous(), attention_weights.contiguous(), dims)  # fmt: skip


def _cast(t, dtype):
    """``t.to(dtype)``, which returns ``t`` itself when the dtype already matches but still costs about a microsecond of
    host time to find that out."""
    return t if t.dtype == dtype else t.to(dtype)


def _shapes_i32(value_spatial_shapes, device):
    # PyTorch callers pass int64 (transformer.py:313); the plugin ABI is int32 (…Plugin.cpp:165-167)
    return value_spatial_shapes.to(device=device, dtype=torch.int32).contiguous()


def _per_camera(p):
    """The camera-shared form's inputs with offsets and logits repeated for the ``bs`` cameras, as the plugin op reads
    them."""
    bs, _, num_heads, _, num_levels, num_query, num_point, _ = p.dims
    n = num_levels * num_point
    return p._replace(off=p.off.reshape(1, num_query, num_heads, n * 2).expand(bs, -1, -1, -1).contiguous(),
                      w=p.w.reshape(1, num_query, num_heads, n).expand(bs, -1, -1, -1).contiguous())


def _v2_workspace(dims, device):
    """Workspace tensor for the INT8 v2 path, or None when the shape is outside its envelope (or v2 is switched off)."""
    if not _V2["enabled"]:
        return None
    bs, num_keys, num_heads, channels, num_levels, _, num_point, ppg = dims
    n = _lib.load().b200_msda_i8_workspace_size(bs, num_keys, num_heads, channels, num_levels, num_point, ppg)
    return torch.empty(n, dtype=torch.uint8, device=device) if n else None


def _launch_int8(p, scales, out, records=None):
    """Runs the INT8 plugin op on the prepared inputs ``p`` into ``out``: the packed kernel when ``_v2_workspace`` lends
    a workspace, the round-1 kernel otherwise or when the packed one declines the shape (status 1). ``records``: int32
    [bs, nq, heads, L*P, 4] for the kernel's own sampling-index records (trace entries), or None."""
    sv, so, sw, sout = (float(x) for x in scales)
    dev = p.value.device
    rec = None if records is None else records.data_ptr()
    args = (p.value.data_ptr(), sv, p.shapes.data_ptr(), p.ref.data_ptr(), int(p.ref.dtype == torch.float16),
            p.off.data_ptr(), so, p.w.data_ptr(), sw, *p.dims, out.data_ptr(), sout)  # fmt: skip
    ws = _v2_workspace(p.dims, dev)
    if ws is not None and _lib.call("b200_msda_i8_ws", dev, *args, ws.data_ptr(), ws.numel(), rec, accept=(0, 1)) == 0:
        return
    if records is None:
        _lib.call("b200_msda_i8", dev, *args)
    else:
        _lib.call("b200_msda_i8_trace", dev, *args, rec)


def _msda_forward(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights, use_h2, out=None):
    """The FP32 / FP16 / BF16 plugin op. Returns its output and the prepared inputs the kernel read (for the
    backward)."""
    dt = value.dtype
    p = _prepare("multi_scale_deformable_attn", value, value_spatial_shapes, reference_points, sampling_offsets,
                 attention_weights, dt)  # fmt: skip
    bs, _, num_heads, channels, _, num_query, _, _ = p.dims
    if out is None:
        out = torch.empty(bs, num_query, num_heads, channels, dtype=dt, device=value.device)
    elif out.dtype != dt or not out.is_contiguous() or out.numel() != bs * num_query * num_heads * channels:
        raise ValueError("out must be a contiguous [bs, num_query, num_heads, channels] tensor of value's dtype")
    if dt == torch.float16:
        name = "b200_msda_f16_h2" if use_h2 and channels % 2 == 0 else "b200_msda_f16"
    else:
        name = f"b200_msda_{_lib.float_dtype(dt, 'multi_scale_deformable_attn')[0]}"
    _lib.call(name, value.device, *p.ptrs(), *p.dims, out.data_ptr())
    return out, p


def _save(ctx, p, inputs, *extra):
    """Keeps for the backward the tensors the forward's kernel read (and ``extra``), its dimensions, and the dtype and
    shape of the differentiable ``inputs`` (value, reference points, offsets, logits), which their gradients take."""
    ctx.save_for_backward(p.value, p.shapes, p.ref, p.off, p.w, *extra)
    ctx.dims = p.dims
    ctx.like = [(t.dtype, t.shape) for t in inputs]


def _backward_launch(prefix, p, args, needs, accept=(0,)):
    """Runs the backward entry ``{prefix}_backward_{f32|f16|bf16}`` — b200_msda_, b200_msda_sca_ or b200_msda_sca_shared_ —
    on the forward's inputs ``p``. ``args``: the tensors the entry takes between the logits and the gradients (grad_out;
    bev_mask and grad_slots for the fused forms). ``needs``: the op's ``needs_input_grad``, which selects the value,
    reference-point, offset and logit gradients to compute. Returns them (None where not wanted), or None when the entry
    declined with a non-zero status in ``accept``."""
    dt, dev = p.value.dtype, p.value.device
    suffix, code = _lib.float_dtype(dt, prefix)
    ws_bytes = _lib.load().b200_msda_backward_workspace_size(code, *p.dims)
    if ws_bytes == 0:
        raise _lib.B200OpsError("b200_msda_backward_workspace_size", 2)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    grads = [torch.empty_like(t) if needs[i] else None for i, t in ((0, p.value), (2, p.ref), (3, p.off), (4, p.w))]
    name = f"{prefix}_backward_{suffix}"
    st = _lib.call(name, dev, *p.ptrs(), *[t.data_ptr() for t in args],
                   *[g.data_ptr() if g is not None else None for g in grads], ws.data_ptr(), *p.dims, accept=accept)
    return None if st else grads


def _grads_like(ctx, grads):
    """The op's gradients: value, reference points, offsets and logits in their inputs' dtypes and shapes."""
    gv, gr, go, gw = (_cast(g, d).reshape(shp) if g is not None else None for g, (d, shp) in zip(grads, ctx.like))
    return gv, None, gr, go, gw


def _msda_autograd_forward(ctx, value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights, use_h2):
    out, p = _msda_forward(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights, use_h2)
    if any(ctx.needs_input_grad):
        _save(ctx, p, (value, reference_points, sampling_offsets, attention_weights))
    return out


class _MultiScaleDeformableAttnFunction(Function):
    @staticmethod
    def symbolic(g, value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights):
        return g.op("MultiScaleDeformableAttnTRT", value, value_spatial_shapes, reference_points, sampling_offsets,
                    attention_weights)  # fmt: skip

    @staticmethod
    def forward(ctx, value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights):
        """value [bs, num_keys, num_heads, channels]; value_spatial_shapes [num_levels, 2] (h, w);
        reference_points [bs, num_queries, 1, 2*points_per_group]; sampling_offsets
        [bs, num_queries, num_heads, num_levels*num_points*2] in pixels, (x, y) innermost; attention_weights
        [bs, num_queries, num_heads, num_levels*num_points] pre-softmax. Returns [bs, num_queries, num_heads, channels].
        """
        return _msda_autograd_forward(ctx, value, value_spatial_shapes, reference_points, sampling_offsets,
                                      attention_weights, False)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        """(grad_value, None, grad_reference_points, grad_sampling_offsets, grad_attention_weights), each in its input's
        dtype and shape; ``None`` for inputs that do not require a gradient. The offset, logit and reference-point
        gradients are bit-reproducible; grad_value is summed with float atomics."""
        p = _Prepared(*ctx.saved_tensors, ctx.dims)
        go = _cast(grad_out, p.value.dtype).contiguous()
        return _grads_like(ctx, _backward_launch("b200_msda", p, (go,), ctx.needs_input_grad))


class _MultiScaleDeformableAttnFunction2(_MultiScaleDeformableAttnFunction):
    @staticmethod
    def symbolic(g, value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights):
        return g.op("MultiScaleDeformableAttnTRT2", value, value_spatial_shapes, reference_points, sampling_offsets,
                    attention_weights)  # fmt: skip

    @staticmethod
    def forward(ctx, value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights):
        return _msda_autograd_forward(ctx, value, value_spatial_shapes, reference_points, sampling_offsets,
                                      attention_weights, True)


def multi_scale_deformable_attn_out(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights,
                                    out):
    """The plugin op writing into a caller-owned ``out`` (no allocation on the call path; used by HostMSDA, whose
    device slots are fixed so that the stream-ordered allocator never has to synchronise)."""
    return _msda_forward(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights, False,
                         out)[0]  # fmt: skip


_multi_scale_deformable_attn_gpu = _MultiScaleDeformableAttnFunction.apply
_multi_scale_deformable_attn_gpu2 = _MultiScaleDeformableAttnFunction2.apply


def multi_scale_deformable_attn(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights):
    """Plugin MultiScaleDeformableAttnTRT (FP32 / FP16 / BF16). Same contract as the reference wrapper (:150-182).
    BF16 reads the reference points in FP32 (a bf16 tensor is cast up) and returns grad_reference_points in the
    dtype the caller passed."""
    assert value.is_cuda
    return _multi_scale_deformable_attn_gpu(value, value_spatial_shapes, reference_points, sampling_offsets,
                                            attention_weights)  # fmt: skip


def multi_scale_deformable_attn2(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights):
    """Plugin MultiScaleDeformableAttnTRT2 (FP32 / FP16 as half2 / BF16). Same contract as the reference wrapper
    (:185-217)."""
    assert value.is_cuda
    return _multi_scale_deformable_attn_gpu2(value, value_spatial_shapes, reference_points, sampling_offsets,
                                             attention_weights)  # fmt: skip


def multi_scale_deformable_attn_int8(value_q, scale_value, value_spatial_shapes, reference_points, offsets_q,
                                     scale_offset, weights_q, scale_weight, scale_out):
    """INT8 flavour of the plugin (…Plugin.cpp:118-134): int8 value / offsets / logits with per-tensor PTQ scales
    (real = q * scale), reference points FP16 or FP32, int8 output at ``scale_out``. In PyTorch the reference has no
    int8 entry (TensorRT supplies the scales through PluginTensorDesc); this mirrors the C launcher's argument list
    (…Kernel.h:29-38)."""
    assert value_q.is_cuda and value_q.dtype == torch.int8
    p = _prepare("multi_scale_deformable_attn_int8", value_q, value_spatial_shapes, reference_points, offsets_q,
                 weights_q, None)  # fmt: skip
    if reference_points.dtype not in (torch.float16, torch.float32):
        raise _lib.B200OpsError("multi_scale_deformable_attn_int8", 1)
    bs, _, num_heads, channels, _, num_query, _, _ = p.dims
    out = torch.empty(bs, num_query, num_heads, channels, dtype=torch.int8, device=value_q.device)
    _launch_int8(p, (scale_value, scale_offset, scale_weight, scale_out), out)
    return out


def _wants_grad(tensors, bev_mask, name):
    """True when the fused form has to record an autograd graph: grad mode is on and an input requires grad. bev_mask
    is a geometry constant; a gradient with respect to it is not computed, so asking for one is an error."""
    if not torch.is_grad_enabled():
        return False
    if isinstance(bev_mask, torch.Tensor) and bev_mask.requires_grad:
        raise ValueError(f"{name}: bev_mask requires grad, but no gradient with respect to bev_mask is computed; "
                         "pass bev_mask.detach()")  # fmt: skip
    return any(isinstance(t, torch.Tensor) and t.requires_grad for t in tensors)


def _sca_forward(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights, bev_mask, accum,
                 shared):
    """Both fused SCA forms: ``…_sca`` (``shared`` False; adds into ``accum``, allocated when None) and
    ``…_sca_shared``. Returns the result, the prepared inputs, the fp32 mask and whether the fused kernel ran (False:
    the plugin-op fallback)."""
    form = "sca_shared" if shared else "sca"
    dt = value.dtype
    p = _prepare(f"multi_scale_deformable_attn_{form}", value, value_spatial_shapes, reference_points, sampling_offsets,
                 attention_weights, dt, bev_mask if shared else None)  # fmt: skip
    bs, _, num_heads, channels, _, num_query, _, _ = p.dims
    mask = _cast(bev_mask.reshape(bs, num_query), torch.float32).contiguous()
    if shared:
        res = torch.empty(num_query, num_heads * channels, dtype=torch.float32, device=value.device)
    elif accum is None:
        res = torch.zeros(num_query, num_heads * channels, dtype=torch.float32, device=value.device)
    elif accum.dtype != torch.float32 or not accum.is_contiguous() or accum.numel() != num_query * num_heads * channels:
        raise ValueError("accum must be a contiguous float32 [num_query, heads*channels] tensor")
    else:
        res = accum
    name = f"b200_msda_{form}_{_lib.float_dtype(dt, form)[0]}"
    fused = _lib.call(name, value.device, *p.ptrs(), mask.data_ptr(), *p.dims, res.data_ptr(), accept=(0, 1)) == 0
    if not fused:
        # shapes the fused kernel does not take (e.g. channels != 32, more than 64 points, unaligned tensors): the plugin
        # op on bs copies of offsets / logits, then the masked camera sum
        q = _per_camera(p) if shared else p
        out, _ = _msda_forward(q.value, q.shapes, q.ref, q.off, q.w, False)
        total = (out.reshape(bs, num_query, -1).float() * mask.unsqueeze(-1)).sum(0)
        if shared:
            res = total
        else:
            res += total
    return res, p, mask, fused


class _MsdaScaFunction(Function):
    """Autograd of the fused SCA forms; ``shared`` selects the camera-shared one."""

    @staticmethod
    def forward(ctx, value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights, bev_mask,
                shared):  # fmt: skip
        out, p, mask, ctx.fused = _sca_forward(value, value_spatial_shapes, reference_points, sampling_offsets,
                                               attention_weights, bev_mask, None, shared)  # fmt: skip
        ctx.shared = shared
        _save(ctx, p, (value, reference_points, sampling_offsets, attention_weights), mask)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_slots):
        """The fused backward kernel when the forward ran the fused kernel; otherwise (the forward took the plugin-op
        fallback, or the backward kernel declines the shape) the plugin-op backward fed ``go = bev_mask * grad_slots``
        per camera, summed over the cameras for the shared offsets and logits."""
        *saved, mask = ctx.saved_tensors
        p = _Prepared(*saved, ctx.dims)
        bs, _, num_heads, channels, _, num_query, _, _ = p.dims
        gs = _cast(grad_slots, torch.float32).contiguous()
        if gs.data_ptr() % 16:
            gs = gs.clone()  # a fresh allocation is 16-byte aligned, as the fused kernel needs
        grads = None
        if ctx.fused:
            prefix = "b200_msda_sca_shared" if ctx.shared else "b200_msda_sca"
            grads = _backward_launch(prefix, p, (mask, gs), ctx.needs_input_grad, accept=(0, 1))
        if grads is None:
            go = _cast(mask.unsqueeze(-1) * gs, p.value.dtype).reshape(bs, num_query, num_heads, channels)
            grads = _backward_launch("b200_msda", _per_camera(p) if ctx.shared else p, (go,), ctx.needs_input_grad)
            if ctx.shared:
                grads[2:] = [g.float().sum(0) if g is not None else None for g in grads[2:]]
        return (*_grads_like(ctx, grads), None, None)


def multi_scale_deformable_attn_sca(value, value_spatial_shapes, reference_points, sampling_offsets,
                                    attention_weights, bev_mask, accum=None):
    """Fused SpatialCrossAttention sampling (SURVEY §8(f)-1): ``accum[q, :] += sum_b bev_mask[b, q] * MSDA(...)[b, q]``
    — what ``(queries * bev_mask).sum(0)`` computes from the plugin output (spatial_cross_attention.py:264-270) —
    without ever writing the per-camera output. ``bev_mask``: [bs, nq] or [bs, nq, 1]; ``accum``: float32
    [nq, heads*channels] (allocated and zeroed when None; accumulated into when given). Returns ``accum``.

    Differentiable when ``accum`` is None (csrc/msda_backward.cu, b200_msda_sca_backward_*): with grad mode on and an
    input requiring grad, the result carries a ``grad_fn`` that returns gradients for value, reference points, offsets
    and logits; a (camera, query) pair with ``bev_mask == 0`` gets exact zeros, whatever it samples. ``bev_mask`` gets
    no gradient (it must not require one). A call with ``accum`` given is inference-only: it records no graph."""
    assert value.is_cuda
    if accum is None and _wants_grad((value, reference_points, sampling_offsets, attention_weights), bev_mask,
                                     "multi_scale_deformable_attn_sca"):  # fmt: skip
        return _MsdaScaFunction.apply(value, value_spatial_shapes, reference_points, sampling_offsets,
                                      attention_weights, bev_mask, False)  # fmt: skip
    return _sca_forward(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights, bev_mask,
                        accum, False)[0]  # fmt: skip


def multi_scale_deformable_attn_queue_mean(value, value_spatial_shapes, reference_points, sampling_offsets,
                                           attention_weights):
    """TemporalSelfAttention's sampling with its BEV-queue mean folded in (SURVEY §8(f)-2): the reference calls the plugin
    on ``bs*num_bev_queue`` value stacks and then takes ``torch.mean(output, dim=0, keepdim=True)``
    (temporal_self_attention.py:447-453). Here the per-queue outputs are never written: the fused epilogue adds
    ``out[b] / num_bev_queue`` into one fp32 accumulator (two commutative adds per slot: deterministic). Same arguments
    as the plugin op; returns ``[1, num_query, heads*channels]`` in ``value.dtype``."""
    bs, num_query = value.shape[0], sampling_offsets.shape[1]
    mask = torch.full((bs, num_query), 1.0 / bs, dtype=torch.float32, device=value.device)
    acc = multi_scale_deformable_attn_sca(value, value_spatial_shapes, reference_points, sampling_offsets,
                                          attention_weights, mask)
    return acc.to(value.dtype).unsqueeze(0)


def multi_scale_deformable_attn_sca_shared(value, value_spatial_shapes, reference_points, sampling_offsets,
                                           attention_weights, bev_mask):
    """Camera-shared fused SCA sampling. SpatialCrossAttention repeats the BEV query per camera before its
    ``sampling_offsets`` / ``attention_weights`` Linear layers (spatial_cross_attention.py:254), so those two tensors
    are ``bs`` identical copies in the plugin call; here they are passed ONCE:

        value [bs, keys, heads, ch], reference_points [bs, nq, 1, 2G], bev_mask [bs, nq(, 1)]
        sampling_offsets [1 | -, nq, heads, L*P*2], attention_weights [1 | -, nq, heads, L*P]

    Returns slots float32 [nq, heads*ch] = sum_b bev_mask[b] * MSDA(value[b], ref[b], offsets, logits), every element
    written exactly once (one item per (query, head), cameras looped in registers, softmax evaluated once). Shapes the
    fused kernel does not take (more than two gather rounds, channels != 32, G not in {1, 2, 4}, P % 4 != 0, unaligned
    tensors) run the plugin op on ``bs`` copies of offsets / logits and sum the masked cameras, like
    ``multi_scale_deformable_attn_sca``.

    Differentiable like ``multi_scale_deformable_attn_sca`` (b200_msda_sca_shared_backward_*): the offset and logit
    gradients are summed over the cameras with ``bev_mask != 0`` inside the kernel and come back as the single copy;
    a query no camera sees gets zeros there."""
    if _wants_grad((value, reference_points, sampling_offsets, attention_weights), bev_mask,
                   "multi_scale_deformable_attn_sca_shared"):  # fmt: skip
        return _MsdaScaFunction.apply(value, value_spatial_shapes, reference_points, sampling_offsets,
                                      attention_weights, bev_mask, True)  # fmt: skip
    return _sca_forward(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights, bev_mask,
                        None, True)[0]  # fmt: skip


def msda_sampling_indices(value_spatial_shapes, reference_points, sampling_offsets, num_heads):
    """Diagnostic: int32 [bs, nq, heads, L*P, 4] records {in_range, h_low, w_low, tap_mask} from the device code."""
    assert reference_points.is_cuda and reference_points.dtype in (torch.float32, torch.float16)
    bs, nq = sampling_offsets.shape[:2]
    L = value_spatial_shapes.shape[0]
    G = reference_points.shape[-1] // 2
    NP = sampling_offsets.numel() // (bs * nq * num_heads * 2)
    shapes = _shapes_i32(value_spatial_shapes, reference_points.device)
    ref = reference_points.contiguous()
    off = sampling_offsets.to(ref.dtype).contiguous()
    rec = torch.empty(bs, nq, num_heads, NP, 4, dtype=torch.int32, device=ref.device)
    _lib.call("b200_msda_debug_indices", ref.device, int(ref.dtype == torch.float16), shapes.data_ptr(), ref.data_ptr(),
              off.data_ptr(), bs, num_heads, L, nq, NP // L, G, rec.data_ptr())  # fmt: skip
    return rec


def msda_trace(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights, scales=None):
    """The production MSDA kernel with its trace switch on. Returns ``(out, records)``: ``out`` as the plugin op computes
    it and int32 records [bs, nq, heads, L*P, 4] = {in_range, h_low, w_low, tap_mask} written by the gather kernel itself
    while it samples (C entries b200_msda_{f32,f16,bf16,i8}_trace). ``scales`` = (scale_value, scale_offset, scale_weight,
    scale_out) selects the INT8 kernel (int8 value / offsets / logits, float or half reference points)."""
    assert value.is_cuda
    dt = value.dtype
    p = _prepare("msda_trace", value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights,
                 None if dt == torch.int8 else dt)  # fmt: skip
    bs, _, num_heads, channels, num_levels, num_query, num_point, _ = p.dims
    out = torch.empty(bs, num_query, num_heads, channels, dtype=dt, device=value.device)
    rec = torch.empty(bs, num_query, num_heads, num_levels * num_point, 4, dtype=torch.int32, device=value.device)
    if dt == torch.int8:
        _launch_int8(p, scales, out, rec)
    else:
        name = f"b200_msda_{_lib.float_dtype(dt, 'msda_trace')[0]}_trace"
        _lib.call(name, value.device, *p.ptrs(), *p.dims, out.data_ptr(), rec.data_ptr())
    return out, rec
