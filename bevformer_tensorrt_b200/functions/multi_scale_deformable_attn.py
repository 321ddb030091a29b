"""Multi-scale deformable attention — host-side mirror of the reference binding
det2trt/models/functions/multi_scale_deformable_attn.py (:10-217): same module-level names, same positional
signature, same ONNX symbolic, so SpatialCrossAttentionTRTP / TemporalSelfAttentionTRTP / the decoder's
CustomMSDeformableAttentionTRTP call it unchanged (spatial_cross_attention.py:692,764-766;
temporal_self_attention.py:348,447-449; decoder.py:376,460-466).

The reference's forward() expands to sampling locations + softmax and calls mmcv's CUDA op; here forward() hands the
plugin-signature tensors straight to the fused sm_90a kernel behind the C ABI (include/b200_bev_ops.h). Inference
only, like the reference (its Function defines no backward).
"""
import ctypes
import os

import torch
from torch.autograd import Function

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
    if not value.is_cuda or value.dtype not in (torch.float16, torch.float32):
        raise ValueError("autotune_msda: FP16 / FP32 CUDA tensors only (the INT8 op has a single launch shape)")
    args = (value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights)
    report = {"chosen": "default", "ms": {}, "rejected": []}
    set_msda_batch_units(1)
    set_msda_gather_variant(0)
    try:
        base = multi_scale_deformable_attn(*args)
        for _ in range(2 * warmup + 4):  # clocks and caches at their steady state before the first candidate is timed
            multi_scale_deformable_attn(*args)
        # the default shape is timed first AND last (its better median counts): a clock ramp or a neighbour's burst
        # during the sweep must not hand the win to whichever shape happened to run later
        order = list(MSDA_LAUNCH_SHAPES.items()) + [("default", MSDA_LAUNCH_SHAPES["default"])]
        for name, (units, strided, variant) in order:
            if name in report["rejected"]:
                continue
            set_msda_batch_units(units, strided)
            set_msda_gather_variant(variant)
            out = multi_scale_deformable_attn(*args)
            if not torch.equal(out, base):
                report["rejected"].append(name)
                continue
            for _ in range(warmup):
                multi_scale_deformable_attn(*args)
            evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
            for a, b in evs:
                a.record()
                multi_scale_deformable_attn(*args)
                b.record()
            torch.cuda.synchronize(value.device)
            per = sorted(a.elapsed_time(b) for a, b in evs)
            report["ms"][name] = min(per[len(per) // 2], report["ms"].get(name, float("inf")))
    finally:
        set_msda_batch_units(1)
        set_msda_gather_variant(0)
    best = min(report["ms"], key=report["ms"].get)
    if best != "default" and report["ms"][best] < report["ms"]["default"] * (1.0 - min_gain):
        report["chosen"] = best
    units, strided, variant = MSDA_LAUNCH_SHAPES[report["chosen"]]
    set_msda_batch_units(units, strided)
    set_msda_gather_variant(variant)
    return report


def autotune_msda_fused(run, result, iters=10, warmup=2, tol=1e-4, min_gain=0.02):
    """Same idea for the fused spatial-cross-attention forms (``multi_scale_deformable_attn_sca`` /
    ``…_sca_shared``, and through them the sharded multi-GPU step), which have two launch shapes: the default and the
    2-CTAs-per-SM one (any non-zero gather variant). ``run()`` launches the caller's step on the current stream (e.g.
    zero the accumulator + fused op), ``result()`` returns the tensor it produced. The alternative is accepted only if
    its result agrees with the default's to ``tol`` x max|result| (the camera sum uses floating-point atomics, so the last
    bits depend on arrival order in either shape) and it is faster by more than ``min_gain``. Leaves the winner as the
    process-wide gather variant and returns ``{"chosen": "default" | "deep_gather", "ms": {...}, "rejected": [...]}``.
    Local launches only — safe to call per rank before a collective step."""
    report = {"chosen": "default", "ms": {}, "rejected": []}
    names = {"default": 0, "deep_gather": 1}
    set_msda_gather_variant(0)
    try:
        run()
        base = result().detach().float().clone()
        scale = max(1.0, float(base.abs().max()))
        for _ in range(2 * warmup + 4):
            run()
        for name, variant in list(names.items()) + [("default", 0)]:  # default first and last, better median counts
            if name in report["rejected"]:
                continue
            set_msda_gather_variant(variant)
            run()
            if float((result().detach().float() - base).abs().max()) > tol * scale:
                report["rejected"].append(name)
                continue
            for _ in range(warmup):
                run()
            evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
            for a, b in evs:
                a.record()
                run()
                b.record()
            torch.cuda.synchronize()
            per = sorted(a.elapsed_time(b) for a, b in evs)
            report["ms"][name] = min(per[len(per) // 2], report["ms"].get(name, float("inf")))
    finally:
        set_msda_gather_variant(0)
    ms = report["ms"]
    if "deep_gather" in ms and "default" in ms and ms["deep_gather"] < ms["default"] * (1.0 - min_gain):
        report["chosen"] = "deep_gather"
    set_msda_gather_variant(names[report["chosen"]])
    return report


def set_msda_launch_shape(name: str):
    """Applies one of ``MSDA_LAUNCH_SHAPES`` by name (e.g. the ``chosen`` entry of an earlier ``autotune_msda`` report)."""
    units, strided, variant = MSDA_LAUNCH_SHAPES[name]
    set_msda_batch_units(units, strided)
    set_msda_gather_variant(variant)


def _v2_workspace(lib, dims, device):
    """Workspace tensor for the INT8 v2 path, or None when the shape is outside its envelope (or v2 is switched off)."""
    if not _V2["enabled"]:
        return None
    bs, num_keys, num_heads, channels, num_levels, _, num_point, ppg = dims
    n = lib.b200_msda_i8_workspace_size(bs, num_keys, num_heads, channels, num_levels, num_point, ppg)
    return torch.empty(n, dtype=torch.uint8, device=device) if n else None


def _launch_int8(lib, dims, value_q, scales, shapes, ref, off, w, out, records=None):
    """Runs the INT8 plugin op into ``out``: the packed kernel when ``_v2_workspace`` lends a workspace, the round-1
    kernel otherwise or when the packed one declines the shape (status 1). ``records``: int32 [bs, nq, heads, L*P, 4]
    for the kernel's own sampling-index records (trace entries), or None."""
    sv, so, sw, sout = (float(x) for x in scales)
    half = int(ref.dtype == torch.float16)
    rec = None if records is None else records.data_ptr()
    with torch.cuda.device(value_q.device):
        ws = _v2_workspace(lib, dims, value_q.device)
        if ws is not None:
            st = lib.b200_msda_i8_ws(value_q.data_ptr(), sv, shapes.data_ptr(), ref.data_ptr(), half, off.data_ptr(), so,
                                     w.data_ptr(), sw, *dims, out.data_ptr(), sout, ws.data_ptr(), ws.numel(), rec,
                                     _lib.current_stream_ptr())  # fmt: skip
            if st != 1:
                _lib.check("b200_msda_i8_ws", st)
                return
        args = (value_q.data_ptr(), sv, shapes.data_ptr(), ref.data_ptr(), half, off.data_ptr(), so, w.data_ptr(), sw,
                *dims, out.data_ptr(), sout)  # fmt: skip
        if records is None:
            _lib.check("b200_msda_i8", lib.b200_msda_i8(*args, _lib.current_stream_ptr()))
        else:
            _lib.check("b200_msda_i8_trace", lib.b200_msda_i8_trace(*args, rec, _lib.current_stream_ptr()))


def _check_inputs(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights):
    if not value.is_cuda:
        raise RuntimeError("multi_scale_deformable_attn: value must be a CUDA tensor (no CPU fallback exists)")
    if value.dim() != 4:
        raise ValueError("value must be [bs, num_keys, num_heads, channels]")
    bs, num_keys, num_heads, channels = value.shape
    num_levels = value_spatial_shapes.shape[0]
    num_query = sampling_offsets.shape[1]
    if reference_points.shape[-1] % 2 != 0:
        raise ValueError("reference_points last dim must hold (x, y) pairs")
    points_per_group = reference_points.shape[-1] // 2
    all_points = attention_weights.shape[-1]
    if all_points % num_levels != 0:
        raise ValueError("attention_weights last dim must be num_levels * num_points")
    num_point = all_points // num_levels
    if sampling_offsets.numel() != bs * num_query * num_heads * all_points * 2:
        raise ValueError("sampling_offsets does not match [bs, num_query, num_heads, num_levels*num_points*2]")
    if attention_weights.numel() != bs * num_query * num_heads * all_points:
        raise ValueError("attention_weights does not match [bs, num_query, num_heads, num_levels*num_points]")
    if reference_points.numel() != bs * num_query * points_per_group * 2:
        raise ValueError("reference_points does not match [bs, num_query, 1, 2*points_per_group]")
    return bs, num_keys, num_heads, channels, num_levels, num_query, num_point, points_per_group


def _shapes_i32(value_spatial_shapes, device):
    # PyTorch callers pass int64 (transformer.py:313); the plugin ABI is int32 (…Plugin.cpp:165-167)
    return value_spatial_shapes.to(device=device, dtype=torch.int32).contiguous()


def _msda_forward(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights, use_h2, out=None):
    dims = _check_inputs(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights)
    bs, _, num_heads, channels, _, num_query, _, _ = dims
    lib = _lib.load()
    dt = value.dtype
    if dt not in (torch.float32, torch.float16):
        raise _lib.B200OpsError("multi_scale_deformable_attn", 1)
    value = value.contiguous()
    shapes = _shapes_i32(value_spatial_shapes, value.device)
    ref = reference_points.to(dt).contiguous()
    off = sampling_offsets.to(dt).contiguous()
    w = attention_weights.to(dt).contiguous()
    if out is None:
        out = torch.empty(bs, num_query, num_heads, channels, dtype=dt, device=value.device)
    elif out.dtype != dt or not out.is_contiguous() or out.numel() != bs * num_query * num_heads * channels:
        raise ValueError("out must be a contiguous [bs, num_query, num_heads, channels] tensor of value's dtype")
    if dt == torch.float32:
        name = "b200_msda_f32"
    else:
        name = "b200_msda_f16_h2" if use_h2 and channels % 2 == 0 else "b200_msda_f16"
    with torch.cuda.device(value.device):
        st = getattr(lib, name)(value.data_ptr(), shapes.data_ptr(), ref.data_ptr(), off.data_ptr(), w.data_ptr(),
                                *dims, out.data_ptr(), _lib.current_stream_ptr())  # fmt: skip
    _lib.check(name, st)
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
        return _msda_forward(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights, False)


class _MultiScaleDeformableAttnFunction2(_MultiScaleDeformableAttnFunction):
    @staticmethod
    def symbolic(g, value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights):
        return g.op("MultiScaleDeformableAttnTRT2", value, value_spatial_shapes, reference_points, sampling_offsets,
                    attention_weights)  # fmt: skip

    @staticmethod
    def forward(ctx, value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights):
        return _msda_forward(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights, True)


def multi_scale_deformable_attn_out(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights,
                                    out):
    """The plugin op writing into a caller-owned ``out`` (no allocation on the call path; used by HostMSDA, whose
    device slots are fixed so that the stream-ordered allocator never has to synchronise)."""
    return _msda_forward(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights, False, out)


_multi_scale_deformable_attn_gpu = _MultiScaleDeformableAttnFunction.apply
_multi_scale_deformable_attn_gpu2 = _MultiScaleDeformableAttnFunction2.apply


def multi_scale_deformable_attn(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights):
    """Plugin MultiScaleDeformableAttnTRT (FP32 / FP16). Same contract as the reference wrapper (:150-182)."""
    assert value.is_cuda
    return _multi_scale_deformable_attn_gpu(value, value_spatial_shapes, reference_points, sampling_offsets,
                                            attention_weights)  # fmt: skip


def multi_scale_deformable_attn2(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights):
    """Plugin MultiScaleDeformableAttnTRT2 (FP32 / FP16 as half2). Same contract as the reference wrapper (:185-217)."""
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
    dims = _check_inputs(value_q, value_spatial_shapes, reference_points, offsets_q, weights_q)
    bs, _, num_heads, channels, _, num_query, _, _ = dims
    if reference_points.dtype not in (torch.float16, torch.float32):
        raise _lib.B200OpsError("multi_scale_deformable_attn_int8", 1)
    lib = _lib.load()
    value_q = value_q.contiguous()
    shapes = _shapes_i32(value_spatial_shapes, value_q.device)
    ref = reference_points.contiguous()
    off = offsets_q.contiguous()
    w = weights_q.contiguous()
    out = torch.empty(bs, num_query, num_heads, channels, dtype=torch.int8, device=value_q.device)
    _launch_int8(lib, dims, value_q, (scale_value, scale_offset, scale_weight, scale_out), shapes, ref, off, w, out)
    return out


def multi_scale_deformable_attn_sca(value, value_spatial_shapes, reference_points, sampling_offsets,
                                    attention_weights, bev_mask, accum=None):
    """Fused SpatialCrossAttention sampling (SURVEY §8(f)-1): ``accum[q, :] += sum_b bev_mask[b, q] * MSDA(...)[b, q]``
    — what ``(queries * bev_mask).sum(0)`` computes from the plugin output (spatial_cross_attention.py:264-270) —
    without ever writing the per-camera output. ``bev_mask``: [bs, nq] or [bs, nq, 1]; ``accum``: float32
    [nq, heads*channels] (allocated and zeroed when None; accumulated into when given). Returns ``accum``."""
    assert value.is_cuda
    dims = _check_inputs(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights)
    bs, _, num_heads, channels, _, num_query, _, _ = dims
    dt = value.dtype
    if dt not in (torch.float32, torch.float16):
        raise _lib.B200OpsError("multi_scale_deformable_attn_sca", 1)
    lib = _lib.load()
    value = value.contiguous()
    shapes = _shapes_i32(value_spatial_shapes, value.device)
    ref = reference_points.to(dt).contiguous()
    off = sampling_offsets.to(dt).contiguous()
    w = attention_weights.to(dt).contiguous()
    mask = bev_mask.reshape(bs, num_query).to(torch.float32).contiguous()
    if accum is None:
        accum = torch.zeros(num_query, num_heads * channels, dtype=torch.float32, device=value.device)
    else:
        if accum.dtype != torch.float32 or not accum.is_contiguous() or accum.numel() != num_query * num_heads * channels:
            raise ValueError("accum must be a contiguous float32 [num_query, heads*channels] tensor")
    name = "b200_msda_sca_f32" if dt == torch.float32 else "b200_msda_sca_f16"
    with torch.cuda.device(value.device):
        st = getattr(lib, name)(value.data_ptr(), shapes.data_ptr(), ref.data_ptr(), off.data_ptr(), w.data_ptr(),
                                mask.data_ptr(), *dims, accum.data_ptr(), _lib.current_stream_ptr())  # fmt: skip
        if st == 1:
            # shapes neither fused kernel takes (channels != 32, more than 64 points): plugin op + masked camera sum
            out = _msda_forward(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights, False)
            accum += (out.reshape(bs, num_query, -1).float() * mask.unsqueeze(-1)).sum(0)
            return accum
    _lib.check(name, st)
    return accum


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
    ``multi_scale_deformable_attn_sca``."""
    if not value.is_cuda:
        raise RuntimeError("multi_scale_deformable_attn_sca_shared: value must be a CUDA tensor (no CPU fallback exists)")
    if value.dim() != 4:
        raise ValueError("value must be [bs, num_keys, num_heads, channels]")
    bs, num_keys, num_heads, channels = value.shape
    dt = value.dtype
    if dt not in (torch.float32, torch.float16):
        raise _lib.B200OpsError("multi_scale_deformable_attn_sca_shared", 1)
    num_levels = value_spatial_shapes.shape[0]
    all_points = attention_weights.shape[-1]
    if all_points % num_levels != 0:
        raise ValueError("attention_weights last dim must be num_levels * num_points")
    num_query = bev_mask.numel() // bs
    points_per_group = reference_points.shape[-1] // 2
    if sampling_offsets.numel() != num_query * num_heads * all_points * 2:
        raise ValueError("sampling_offsets must be ONE copy: [num_query, num_heads, num_levels*num_points*2]")
    if attention_weights.numel() != num_query * num_heads * all_points:
        raise ValueError("attention_weights must be ONE copy: [num_query, num_heads, num_levels*num_points]")
    if reference_points.numel() != bs * num_query * points_per_group * 2:
        raise ValueError("reference_points does not match [bs, num_query, 1, 2*points_per_group]")
    lib = _lib.load()
    value = value.contiguous()
    shapes = _shapes_i32(value_spatial_shapes, value.device)
    ref = reference_points.to(dt).contiguous()
    off = sampling_offsets.to(dt).contiguous()
    w = attention_weights.to(dt).contiguous()
    mask = bev_mask.reshape(bs, num_query).to(torch.float32).contiguous()
    slots = torch.empty(num_query, num_heads * channels, dtype=torch.float32, device=value.device)
    name = "b200_msda_sca_shared_f32" if dt == torch.float32 else "b200_msda_sca_shared_f16"
    with torch.cuda.device(value.device):
        st = getattr(lib, name)(value.data_ptr(), shapes.data_ptr(), ref.data_ptr(), off.data_ptr(), w.data_ptr(),
                                mask.data_ptr(), bs, num_keys, num_heads, channels, num_levels, num_query,
                                all_points // num_levels, points_per_group, slots.data_ptr(),
                                _lib.current_stream_ptr())  # fmt: skip
        if st == 1:
            # shapes the fused kernel does not take: plugin op on bs copies of offsets / logits + masked camera sum
            rep_off = off.reshape(1, num_query, num_heads, all_points * 2).expand(bs, -1, -1, -1)
            rep_w = w.reshape(1, num_query, num_heads, all_points).expand(bs, -1, -1, -1)
            out = _msda_forward(value, shapes, ref, rep_off, rep_w, False)
            return (out.reshape(bs, num_query, -1).float() * mask.unsqueeze(-1)).sum(0)
    _lib.check(name, st)
    return slots


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
    with torch.cuda.device(ref.device):
        st = _lib.load().b200_msda_debug_indices(int(ref.dtype == torch.float16), shapes.data_ptr(), ref.data_ptr(),
                                                 off.data_ptr(), bs, num_heads, L, nq, NP // L, G, rec.data_ptr(),
                                                 _lib.current_stream_ptr())  # fmt: skip
    _lib.check("b200_msda_debug_indices", st)
    return rec


def msda_trace(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights, scales=None):
    """The production MSDA kernel with its trace switch on. Returns ``(out, records)``: ``out`` as the plugin op computes
    it and int32 records [bs, nq, heads, L*P, 4] = {in_range, h_low, w_low, tap_mask} written by the gather kernel itself
    while it samples (C entries b200_msda_{f32,f16,i8}_trace). ``scales`` = (scale_value, scale_offset, scale_weight,
    scale_out) selects the INT8 kernel (int8 value / offsets / logits, float or half reference points)."""
    assert value.is_cuda
    dims = _check_inputs(value, value_spatial_shapes, reference_points, sampling_offsets, attention_weights)
    bs, _, num_heads, channels, num_levels, num_query, num_point, _ = dims
    lib = _lib.load()
    dt = value.dtype
    value = value.contiguous()
    shapes = _shapes_i32(value_spatial_shapes, value.device)
    out = torch.empty(bs, num_query, num_heads, channels, dtype=dt, device=value.device)
    rec = torch.empty(bs, num_query, num_heads, num_levels * num_point, 4, dtype=torch.int32, device=value.device)
    if dt == torch.int8:
        ref, off, w = reference_points.contiguous(), sampling_offsets.contiguous(), attention_weights.contiguous()
        _launch_int8(lib, dims, value, scales, shapes, ref, off, w, out, rec)
    elif dt in (torch.float32, torch.float16):
        ref, off, w = (t.to(dt).contiguous() for t in (reference_points, sampling_offsets, attention_weights))
        name = "b200_msda_f32_trace" if dt == torch.float32 else "b200_msda_f16_trace"
        with torch.cuda.device(value.device):
            st = getattr(lib, name)(value.data_ptr(), shapes.data_ptr(), ref.data_ptr(), off.data_ptr(), w.data_ptr(),
                                    *dims, out.data_ptr(), rec.data_ptr(), _lib.current_stream_ptr())  # fmt: skip
        _lib.check(name, st)
    else:
        raise _lib.B200OpsError("msda_trace", 1)
    return out, rec
