"""BF16 MSDA (every form, forward and backward) and BF16 DCNv2 (forward and five gradients) on the GPU.

The oracles evaluate float inputs as float32 values, so they are given the bf16-rounded tensors (reference points stay
fp32, as the BF16 entries read them). Everything between the loads and the stores is fp32 and each result is rounded to
bf16 once, so the bars follow the FP16 rule of test_msda_backward_gpu.py / test_dcn_backward_gpu.py with the BF16
spacing: half a bf16 spacing of max|want| plus the FP32 bar, and one full spacing for grad_value / grad_input, whose
float atomics are summed in fp32 in an order that varies and are then rounded."""
import math

import numpy as np
import pytest
import torch

import bevformer_tensorrt_b200 as bt
from bevformer_tensorrt_b200 import _lib
from bevformer_tensorrt_b200.functions.multi_scale_deformable_attn import (MSDA_LAUNCH_SHAPES, autotune_msda, msda_trace,
                                                                          set_msda_f16_path, set_msda_launch_shape)
from bevformer_tensorrt_b200.registry import TRT_FUNCTIONS
from bevformer_tensorrt_b200.workloads import CONFIGS, MSDAConfig, make_msda_inputs
from oracle import msda as omsda
from oracle.msda_backward import msda_backward_f64
from tests.helpers import DCN_CASES, make_dcn_inputs
from tests.test_dcn_backward_gpu import NAMES as DCN_NAMES
from tests.test_dcn_backward_gpu import _base_inputs, _BASE_KW, _oracle_grads
from tests.test_msda_backward_gpu import ENVELOPE
from tests.test_msda_fused_backward_gpu import ENVELOPE as FUSED_ENVELOPE
from tests.test_msda_fused_backward_gpu import _grad_slots, _mask
from tests.test_msda_gpu import EXTRA, SMALL, _want_records

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
FP32_TOL = 1e-5  # the FP32 forward bar of test_msda_gpu.py
MSDA_NAMES = ("value", "reference_points", "sampling_offsets", "attention_weights")


def bf16_spacing(m):
    """Distance between adjacent bf16 values at magnitude m (numpy has no bf16): 2^(floor(log2 m) - 7)."""
    return 2.0 ** (math.floor(math.log2(m)) - 7) if m > 0 else 0.0


def _fwd_bar(want):
    return 0.5 * bf16_spacing(float(np.abs(want).max())) + FP32_TOL


def _grad_bar(want, atomics=False):
    m = want.abs().max().item()
    return (1.0 if atomics else 0.5) * bf16_spacing(m) + 1e-4 * max(m, 1e-30)


def _cfg(name):
    return CONFIGS.get(name) or EXTRA[name]


def _bf16_inputs(cfg, dist, seed):
    """MSDA inputs built in fp32, value / offsets / logits rounded to bf16, reference points kept fp32."""
    value, shapes, ref, off, logits = make_msda_inputs(cfg, dist, seed, torch.float32)
    return value.to(BF), shapes, ref, off.to(BF), logits.to(BF)


def _oracle(inputs):
    return omsda.msda_f32(*(t.float().numpy() for t in inputs))


def _err(got, want):
    return float(np.abs(got.float().cpu().numpy().astype(np.float64) - want).max())


FWD_CASES = SMALL + [(n, "U", 20 + i) for i, n in enumerate(EXTRA)] + [("many_points", "edge", 40),
                                                                       ("one_pixel", "edge", 41), ("tiny_sca", "G", 42)]


# ---- 1. MSDA forward, every form, against the oracle ----------------------------------------------------------------------
@pytest.mark.parametrize("op", ["multi_scale_deformable_attn", "multi_scale_deformable_attn2"])
@pytest.mark.parametrize("name,dist,seed", FWD_CASES)
def test_plugin_op_matches_oracle(name, dist, seed, op):
    inputs = _bf16_inputs(_cfg(name), dist, seed)
    want = _oracle(inputs)
    got = getattr(bt, op)(*(t.cuda() for t in inputs))
    assert got.dtype == BF and got.shape == want.shape
    err, bar = _err(got, want), _fwd_bar(want)
    assert err <= bar, (name, dist, err, bar)


def _camera_sum(per_camera, mask):
    return (per_camera.astype(np.float64) * mask.numpy()[:, :, None, None].astype(np.float64)).sum(0)


FUSED_CASES = [("small_sca", "U", 61), ("small_sca", "edge", 62), ("tiny_sca", "G", 63), ("one_pixel", "edge", 64),
               ("many_points", "edge", 65), ("generic_c20", "edge", 66), ("g2", "U", 67)]  # fmt: skip


@pytest.mark.parametrize("mask_kind", ["ring", "ones"])
@pytest.mark.parametrize("name,dist,seed", FUSED_CASES)
def test_fused_sca_matches_oracle(name, dist, seed, mask_kind):
    """Camera-summed form; generic_c20 and many_points lie outside the fused kernel and take the plugin-op fallback,
    whose per-camera bf16 results are summed in fp32."""
    cfg = _cfg(name)
    inputs = _bf16_inputs(cfg, dist, seed)
    mask = _mask(cfg, "ring") if mask_kind == "ring" else torch.ones(cfg.batch, cfg.num_query)
    per = _oracle(inputs)
    want = _camera_sum(per, mask).reshape(cfg.num_query, -1)
    got = bt.multi_scale_deformable_attn_sca(*(t.cuda() for t in inputs), mask.cuda())
    assert got.dtype == torch.float32
    bar = (0.5 * bf16_spacing(float(np.abs(per).max())) + FP32_TOL) * float(mask.sum(0).max()) + FP32_TOL
    assert _err(got, want) <= bar, (name, _err(got, want), bar)


@pytest.mark.parametrize("name,dist,seed", FUSED_CASES)
def test_camera_shared_matches_oracle(name, dist, seed):
    cfg = _cfg(name)
    value, shapes, ref, off, logits = _bf16_inputs(cfg, dist, seed)
    off1, lg1 = off[:1], logits[:1]
    mask = _mask(cfg, "ring")
    per = _oracle((value, shapes, ref, off1.expand_as(off), lg1.expand_as(logits)))
    want = _camera_sum(per, mask).reshape(cfg.num_query, -1)
    got = bt.multi_scale_deformable_attn_sca_shared(*(t.cuda() for t in (value, shapes, ref, off1, lg1)), mask.cuda())
    bar = (0.5 * bf16_spacing(float(np.abs(per).max())) + FP32_TOL) * float(mask.sum(0).max()) + FP32_TOL
    assert got.dtype == torch.float32 and _err(got, want) <= bar


@pytest.mark.parametrize("name,dist,seed", [("tsa_like", "U", 71), ("small_sca", "edge", 72), ("generic_c20", "U", 73)])
def test_queue_mean_matches_oracle(name, dist, seed):
    cfg = _cfg(name)
    inputs = _bf16_inputs(cfg, dist, seed)
    want = _oracle(inputs).astype(np.float64).mean(0, keepdims=True).reshape(1, cfg.num_query, -1)
    got = bt.multi_scale_deformable_attn_queue_mean(*(t.cuda() for t in inputs))
    assert got.dtype == BF and _err(got, want) <= _fwd_bar(want) + FP32_TOL


@pytest.mark.parametrize("dist", ["G", "U"])
def test_base_sca_full_size_against_fp32_kernel(dist):
    """base_sca at full size (6 cameras, 40000 queries, 4 levels): every form against the FP32 kernel on the
    upcast inputs, which test_msda_gpu.py pins to the oracle and to the reference kernel."""
    cfg = CONFIGS["base_sca"]
    value, shapes, ref, off, logits = (t.cuda() for t in _bf16_inputs(cfg, dist, 3))
    want = bt.multi_scale_deformable_attn(value.float(), shapes, ref, off.float(), logits.float())
    got = bt.multi_scale_deformable_attn(value, shapes, ref, off, logits)
    m = want.abs().max().item()
    assert (got.float() - want).abs().max().item() <= 0.5 * bf16_spacing(m) + FP32_TOL
    mask = _mask(cfg, "ring").cuda()
    want_s = bt.multi_scale_deformable_attn_sca(value.float(), shapes, ref, off.float(), logits.float(), mask)
    got_s = bt.multi_scale_deformable_attn_sca(value, shapes, ref, off, logits, mask)
    assert (got_s - want_s).abs().max().item() <= 1e-4 * max(1.0, want_s.abs().max().item())
    want_c = bt.multi_scale_deformable_attn_sca_shared(value.float(), shapes, ref, off[:1].float(), logits[:1].float(), mask)
    got_c = bt.multi_scale_deformable_attn_sca_shared(value, shapes, ref, off[:1], logits[:1], mask)
    assert (got_c - want_c).abs().max().item() <= 1e-4 * max(1.0, want_c.abs().max().item())


def test_bf16_reference_points_are_read_as_fp32():
    """A bf16 reference-point tensor is cast up (exactly): the result equals the one from its fp32 copy."""
    value, shapes, ref, off, logits = (t.cuda() for t in _bf16_inputs(_cfg("small_sca"), "U", 5))
    ref16 = ref.to(BF)
    assert torch.equal(bt.multi_scale_deformable_attn(value, shapes, ref16, off, logits),
                       bt.multi_scale_deformable_attn(value, shapes, ref16.float(), off, logits))


# ---- 2. index records --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,dist,seed", [("small_sca", "edge", 51), ("small_sca", "U", 52), ("one_pixel", "edge", 53),
                                            ("tsa_like", "edge", 54), ("tiny_sca", "G", 55), ("many_points", "edge", 56),
                                            ("generic_c20", "edge", 57), ("ragged_tail", "edge", 58)])  # fmt: skip
def test_trace_records_are_the_fp32_oracle_records(name, dist, seed):
    """The positions come from the FP32 reference points: the bf16 kernel's own records equal the FP32 oracle's on the
    upcast inputs, bit for bit, and the traced launch computes the plain launch's bits."""
    cfg = _cfg(name)
    inputs = _bf16_inputs(cfg, dist, seed)
    _, shapes, ref, off, _ = inputs
    want = _want_records(shapes, ref.numpy(), off.float().numpy(), cfg)
    dev = [t.cuda() for t in inputs]
    out_t, rec = msda_trace(*dev)
    assert torch.equal(out_t, bt.multi_scale_deformable_attn(*dev))
    rec = rec.cpu().numpy()
    assert (rec == want).all(), f"{(rec != want).any(-1).sum()} of {want[..., 0].size} records differ"
    assert want[..., 0].any()


# ---- 3. launch shapes ----------------------------------------------------------------------------------------------------
@pytest.fixture
def restore_shape():
    yield
    set_msda_launch_shape("default")
    _lib.load().b200_msda_set_f16_mode(0)
    set_msda_f16_path(False)


@pytest.mark.parametrize("name,dist,seed", [("small_sca", "edge", 81), ("tiny_sca", "G", 83), ("tsa_like", "U", 84),
                                            ("ragged_tail", "edge", 85)])  # fmt: skip
def test_every_launch_shape_is_bit_identical(name, dist, seed, restore_shape):
    dev = [t.cuda() for t in _bf16_inputs(_cfg(name), dist, seed)]
    set_msda_launch_shape("default")
    base = bt.multi_scale_deformable_attn(*dev)
    for shape in MSDA_LAUNCH_SHAPES:
        set_msda_launch_shape(shape)
        assert torch.equal(bt.multi_scale_deformable_attn(*dev), base), shape
        assert torch.equal(msda_trace(*dev)[0], base), shape
    set_msda_launch_shape("default")
    _lib.load().b200_msda_set_f16_mode(1)
    set_msda_f16_path(True)
    assert torch.equal(bt.multi_scale_deformable_attn(*dev), base)


def test_autotune_accepts_bf16(restore_shape):
    dev = [t.cuda() for t in _bf16_inputs(_cfg("small_sca"), "U", 86)]
    report = autotune_msda(*dev, iters=3, warmup=1)
    assert report["chosen"] in MSDA_LAUNCH_SHAPES and not report["rejected"]


# ---- 4. MSDA backward ----------------------------------------------------------------------------------------------------
def _grads(inputs, go, op=None, requires=MSDA_NAMES, extra=()):
    value, shapes, ref, off, logits = inputs
    ts = [t.cuda().detach().requires_grad_(n in requires) for n, t in zip(MSDA_NAMES, (value, ref, off, logits))]
    out = (op or bt.multi_scale_deformable_attn)(ts[0], shapes.cuda(), ts[1], ts[2], ts[3], *extra)
    out.backward(go.cuda())
    return [t.grad for t in ts]


def _check_grads(got, want, tag):
    for n, g, w in zip(MSDA_NAMES, got, want):
        assert g.dtype == (torch.float32 if n == "reference_points" else BF), (tag, n, g.dtype)
        err, bar = (g.double().cpu() - w).abs().max().item(), _grad_bar(w, atomics=n == "value")
        assert err <= bar, (tag, n, err, bar)


@pytest.mark.parametrize("name", list(ENVELOPE))
def test_plugin_backward_matches_oracle(name):
    cfg = ENVELOPE[name][0]
    inputs = _bf16_inputs(cfg, "edge", 91)
    go = torch.randn(cfg.batch, cfg.num_query, cfg.num_heads, cfg.channels,
                     generator=torch.Generator().manual_seed(11)).to(BF)  # fmt: skip
    want = msda_backward_f64(*inputs, go)[1:]
    _check_grads(_grads(inputs, go), want, name)


def test_plugin_backward_base_sca_G():
    """Full size, against the FP32 backward on the upcast inputs (test_msda_backward_gpu.py pins it to the float64
    oracle; a float64 oracle of this size does not fit next to the op on one card)."""
    cfg = CONFIGS["base_sca"]
    inputs = _bf16_inputs(cfg, "G", 92)
    go = torch.randn(cfg.batch, cfg.num_query, cfg.num_heads, cfg.channels,
                     generator=torch.Generator().manual_seed(12)).to(BF)  # fmt: skip
    want = _grads([t.float() if t.dtype == BF else t for t in inputs], go.float())
    _check_grads(_grads(inputs, go), [w.double().cpu() for w in want], "base_sca")


@pytest.mark.parametrize("name", ["g2", "g4"])
def test_ordered_gradients_are_bit_stable_across_runs_and_subsets(name):
    cfg = ENVELOPE[name][0]
    inputs = _bf16_inputs(cfg, "edge", 93)
    go = torch.randn(cfg.batch, cfg.num_query, cfg.num_heads, cfg.channels).to(BF)
    full = _grads(inputs, go)
    again = _grads(inputs, go)
    for i in (1, 2, 3):
        assert torch.equal(full[i], again[i]), MSDA_NAMES[i]
        alone = _grads(inputs, go, requires=(MSDA_NAMES[i],))
        assert torch.equal(full[i], alone[i]), MSDA_NAMES[i]


@pytest.mark.parametrize("shared", [False, True])
@pytest.mark.parametrize("name", list(FUSED_ENVELOPE))
def test_fused_backward_matches_oracle(name, shared):
    """Oracle: the plugin-op backward fed go[b, q] = bev_mask[b, q] * grad_slots[q]; for the camera-shared form the
    offsets and logits are one copy, expanded for the oracle and their gradients summed over the cameras."""
    cfg = FUSED_ENVELOPE[name]
    value, shapes, ref, off, logits = _bf16_inputs(cfg, "edge", 94)
    if shared:
        off, logits = off[:1], logits[:1]
    mask, gs = _mask(cfg, "ring"), _grad_slots(cfg)
    go = (mask[:, :, None] * gs[None]).reshape(cfg.batch, cfg.num_query, cfg.num_heads, cfg.channels)
    if cfg.num_levels * cfg.num_points > 32:
        # more than two gather rounds: the forward took the plugin-op fallback, whose backward is the plugin-op
        # backward fed bev_mask * grad_slots in the op's dtype, bf16
        go = go.to(BF)
    oi = (value, shapes, ref, off.expand(cfg.batch, -1, -1, -1), logits.expand(cfg.batch, -1, -1, -1))
    want = list(msda_backward_f64(*oi, go)[1:])
    if shared:
        want[2], want[3] = want[2].sum(0, keepdim=True), want[3].sum(0, keepdim=True)
    op = bt.multi_scale_deformable_attn_sca_shared if shared else bt.multi_scale_deformable_attn_sca
    got = _grads((value, shapes, ref, off, logits), gs, op=op, extra=(mask.cuda(),))
    _check_grads(got, want, (name, shared))


# ---- 5. DCNv2 -------------------------------------------------------------------------------------------------------------
def _dcn_bf16(case):
    x, off, mask, w, b, kw = make_dcn_inputs(case)
    return [t.to(BF) for t in (x, off, mask, w, b)] + [kw]


def _dcn_ours(x, off, mask, w, b, go, kw):
    ts = [t.detach().cuda().requires_grad_(True) for t in (x, off, mask, w, b)]
    out = bt.modulated_deformable_conv2d(*ts, kw["stride"], kw["padding"], kw["dilation"], kw["groups"],
                                         kw["deform_groups"])  # fmt: skip
    out.backward(go.cuda())
    return out.detach(), [t.grad for t in ts]


def _dcn_check(out, got, want_out, want, tag):
    m = want_out.abs().max().item()
    assert out.dtype == BF
    assert (out.double().cpu() - want_out.cpu()).abs().max().item() <= 0.5 * bf16_spacing(m) + 1e-4 * max(1.0, m), tag
    for n, g, r in zip(DCN_NAMES, got, want):
        assert g.dtype == BF, (tag, n)
        err, bar = (g.double().cpu() - r.cpu()).abs().max().item(), _grad_bar(r, atomics=n == "input")
        assert err <= bar, (tag, n, err, bar)


@pytest.mark.parametrize("case", list(DCN_CASES))
def test_dcn_forward_and_grads_match_torchvision_float64(case):
    """Every DCN_CASES entry, groups and deformable groups > 1 included. The fused_* cases lie inside the FP16
    tensor-core envelope: a bf16 tensor read as FP16 bits there would be far off."""
    x, off, mask, w, b, kw = _dcn_bf16(case)
    n, co = x.shape[0], w.shape[0]
    go = torch.randn(n, co, off.shape[2], off.shape[3], generator=torch.Generator().manual_seed(11)).to(BF)
    want_out, want = _oracle_grads(x, off, mask, w, b, go, kw)
    out, got = _dcn_ours(x, off, mask, w, b, go, kw)
    _dcn_check(out, got, want_out, want, case)


def test_dcn_base_backbone_shape():
    """[6,256,58,100] 3x3, Co = 256 (inside the FP16 fused envelope), forward and five gradients on the GPU oracle."""
    x, off, mask, w, b, go = [t.to(BF) for t in _base_inputs()]
    want_out, want = _oracle_grads(x, off, mask, w, b, go, _BASE_KW, device="cuda")
    out, got = _dcn_ours(x, off, mask, w, b, go, _BASE_KW)
    _dcn_check(out, got, want_out, want, "base")


def test_dcn_gradients_in_the_callers_dtypes():
    """Under autocast the weight stays fp32: its gradient comes back in fp32, the others in bf16."""
    x, off, mask, w, b, kw = _dcn_bf16("k3_s1_p1_g2_dg2")
    ts = [t.cuda().requires_grad_(True) for t in (x, off, mask, w.float(), b.float())]
    out = bt.modulated_deformable_conv2d(*ts, kw["stride"], kw["padding"], kw["dilation"], kw["groups"], kw["deform_groups"])
    assert out.dtype == BF
    out.float().sum().backward()
    assert [t.grad.dtype for t in ts] == [BF, BF, BF, torch.float32, torch.float32]


# ---- 6. non-finite values ------------------------------------------------------------------------------------------------
def test_msda_poisoned_unread_pixel_leaves_bits_unchanged():
    cfg = MSDAConfig("sparse", 2, 2, 8, 32, ((20, 20),), 4, 1)  # 64 points per camera, at most 256 of 400 pixels read
    value, shapes, ref, off, logits = _bf16_inputs(cfg, "edge", 101)
    rec = _want_records(shapes, ref.numpy(), off.float().numpy(), cfg)  # [B, Q, M, L*P, 4]
    starts = np.concatenate([[0], np.cumsum([h * w for h, w in cfg.spatial_shapes])[:-1]])
    read = np.zeros((cfg.batch, cfg.spatial_size), bool)
    lvl = np.repeat(np.arange(cfg.num_levels), cfg.num_points)
    b_idx, _, _, k_idx = np.nonzero(rec[..., 0])
    r = rec[rec[..., 0] == 1]
    for (dh, dw), bit in (((0, 0), 1), ((0, 1), 2), ((1, 0), 4), ((1, 1), 8)):
        sel = (r[:, 3] & bit) != 0
        W = np.array([cfg.spatial_shapes[l][1] for l in lvl[k_idx[sel]]])
        read[b_idx[sel], starts[lvl[k_idx[sel]]] + (r[sel, 1] + dh) * W + r[sel, 2] + dw] = True
    b0 = 0
    free = np.nonzero(~read[b0])[0]
    assert free.size >= 2
    bad = value.clone()
    bad[b0, free[0]] = float("inf")
    bad[b0, free[1]] = float("nan")
    dev = [t.cuda() for t in (value, shapes, ref, off, logits)]
    clean = bt.multi_scale_deformable_attn(*dev)
    assert torch.equal(bt.multi_scale_deformable_attn(bad.cuda(), *dev[1:]), clean)
    mask = _mask(cfg, "ring").cuda()
    assert torch.equal(bt.multi_scale_deformable_attn_sca(bad.cuda(), *dev[1:], mask),
                       bt.multi_scale_deformable_attn_sca(*dev, mask))


def test_dcn_poisoned_unread_pixel_leaves_bits_unchanged():
    """Every sample lands in rows [0, 10) of a 24 x 24 image, so rows 12 and up are never read, by any corner."""
    g = torch.Generator().manual_seed(3)
    n, c, h, w, co = 2, 8, 24, 24, 16
    ho = wo = 22
    base_h = (torch.arange(ho)[:, None] + torch.arange(3).repeat_interleave(3)[:, None, None]).float()  # [9, ho, 1]
    oh = torch.rand(n, 9, ho, wo, generator=g) * 10 - base_h
    ow = torch.randn(n, 9, ho, wo, generator=g)
    off = torch.stack([oh, ow], 2).reshape(n, 18, ho, wo)
    x = torch.randn(n, c, h, w, generator=g)
    mask = torch.rand(n, 9, ho, wo, generator=g)
    wt = torch.randn(co, c, 3, 3, generator=g) / 8
    x, off, mask, wt = (t.to(BF).cuda() for t in (x, off, mask, wt))
    clean = bt.modulated_deformable_conv2d(x, off, mask, wt, None)
    bad = x.clone()
    bad[:, :, 15, 3] = float("inf")
    bad[:, :, 20, 17] = float("nan")
    assert torch.isfinite(clean).all()
    assert torch.equal(bt.modulated_deformable_conv2d(bad, off, mask, wt, None), clean)


def test_float64_still_raises_unsupported():
    inputs = [t.cuda().double() for t in make_msda_inputs(_cfg("small_sca"), "U", 1)]
    with pytest.raises(_lib.B200OpsError):
        bt.multi_scale_deformable_attn(inputs[0], inputs[1].int(), *inputs[2:])
    x, off, mask, w, b, _ = make_dcn_inputs("k3_s1_p1_g2_dg2")
    with pytest.raises(_lib.B200OpsError):
        bt.modulated_deformable_conv2d(*(t.cuda().double() for t in (x, off, mask, w, b)), 1, 1, 1, 2, 2)


# ---- 7. modules under autocast -------------------------------------------------------------------------------------------
# Per parameter-gradient tensor, max|bf16 autocast - reference| / max|reference|, where the reference is the same
# module whose op upcasts the bf16 inputs, runs the FP32 op and rounds the result to the bf16 op's output dtype. Both
# runs share every bf16 Linear / conv, so the difference is the op's own: bf16 gradients rounded once instead of fp32
# gradients rounded by the autocast cast-back.
# Measured on an H100: 1.3e-3 to 2.6e-3 for the SCA modes and TSA, 4.4e-3 for DCNv2P (a 64-channel 3x3 layer, whose
# 576-term weight-gradient sums see more bf16 inputs). The bar is about twice the largest.
MODULE_BAR = 1e-2


def _via_fp32(op, round_to_bf16):
    def run(value, shapes, ref, off, logits, *rest):
        out = op(value.float(), shapes, ref.float(), off.float(), logits.float(), *rest)
        return out.to(BF) if round_to_bf16 else out

    return run


def _sca_inputs():
    from tests.test_modules import _tiny_sca_inputs

    return _tiny_sca_inputs(torch.float32, "cuda")


def _train_step(module, run):
    module.zero_grad(set_to_none=True)
    with torch.autocast("cuda", dtype=BF):
        out = run()
    out.float().square().mean().backward()
    return {n: p.grad.detach().clone() for n, p in module.named_parameters() if p.grad is not None}


def _compare(module, run, reference_setup, reference_teardown):
    got = _train_step(module, run)
    reference_setup()
    try:
        want = _train_step(module, run)
    finally:
        reference_teardown()
    worst = 0.0
    for n, p in module.named_parameters():
        g, w = got[n], want[n]
        assert g.dtype == torch.float32 and torch.isfinite(g).all() and g.abs().max() > 0, n
        rel = ((g - w).abs().max() / w.abs().max()).item()
        worst = max(worst, rel)
        assert rel <= MODULE_BAR, (n, rel)
    print(f"worst per-tensor relative gradient difference {worst:.2e}")
    return worst


@pytest.mark.parametrize("mode", ["unfused", "fused", "camera_shared"])
def test_sca_module_trains_under_autocast(mode, monkeypatch):
    from bevformer_tensorrt_b200.modules.attention import SpatialCrossAttentionTRTP

    torch.manual_seed(0)
    sca = SpatialCrossAttentionTRTP(num_levels=1, num_points=8, fused=mode != "unfused",
                                    camera_shared=mode == "camera_shared").cuda()  # fmt: skip
    ins = _sca_inputs()
    attn = sca.deformable_attention
    name = {"unfused": None, "fused": "multi_scale_deformable_attn_sca",
            "camera_shared": "multi_scale_deformable_attn_sca_shared"}[mode]  # fmt: skip

    def setup():
        if name is None:
            attn.multi_scale_deformable_attn = _via_fp32(bt.multi_scale_deformable_attn, True)
        else:
            monkeypatch.setitem(TRT_FUNCTIONS.module_dict, name, _via_fp32(TRT_FUNCTIONS.get(name), False))

    def teardown():
        attn.multi_scale_deformable_attn = bt.multi_scale_deformable_attn
        monkeypatch.undo()

    _compare(sca, lambda: sca.forward_trt(*ins), setup, teardown)


def test_tsa_module_trains_under_autocast():
    from bevformer_tensorrt_b200.modules.attention import TemporalSelfAttentionTRTP

    torch.manual_seed(1)
    tsa = TemporalSelfAttentionTRTP().cuda()
    g = torch.Generator(device="cuda").manual_seed(2)
    q = torch.randn(1, 40 * 40, 256, device="cuda", generator=g)
    ref2d = torch.rand(2, 40 * 40, 1, 2, device="cuda", generator=g)
    shapes = torch.tensor([[40, 40]], device="cuda")

    def setup():
        tsa.multi_scale_deformable_attn = _via_fp32(bt.multi_scale_deformable_attn, True)

    def teardown():
        tsa.multi_scale_deformable_attn = bt.multi_scale_deformable_attn

    _compare(tsa, lambda: tsa.forward_trt(q, ref2d, shapes), setup, teardown)


def test_dcnv2p_trains_under_autocast():
    from bevformer_tensorrt_b200.modules.cnn.dcn import ModulatedDeformConv2dPackPlugin

    torch.manual_seed(3)
    m = ModulatedDeformConv2dPackPlugin(64, 64, 3, padding=1).cuda()
    torch.nn.init.normal_(m.conv_offset.weight, std=0.02)  # non-zero offsets, so the offset branch has gradients
    x = torch.randn(2, 64, 30, 40, device="cuda").to(BF)  # what a bf16 backbone conv hands the layer

    def via_fp32(inp, off, mask, w, b, *geo):
        return bt.modulated_deformable_conv2d(inp.float(), off.float(), mask.float(), w.float(), b.float(), *geo).to(BF)

    def setup():
        m._op = via_fp32

    def teardown():
        del m._op

    _compare(m, lambda: m(x), setup, teardown)
