"""Backward of the fused SCA forms (csrc/msda_backward.cu, EPI 1 / 2: b200_msda_sca_backward_* and
b200_msda_sca_shared_backward_*, and the autograd path of multi_scale_deformable_attn_sca / _sca_shared / _queue_mean).

Oracle: oracle.msda_backward.msda_backward_f64 fed go[b, q] = bev_mask[b, q] * grad_slots[q] (formed in fp32, as the
kernel forms it). For the camera-shared form the offsets and logits are expanded to B copies and their gradients summed
over the cameras. Tolerances are those of test_msda_backward_gpu.py (_bar)."""
import ctypes
import re

import numpy as np
import pytest
import torch

import bevformer_tensorrt_b200 as bt
from bevformer_tensorrt_b200 import _lib
from bevformer_tensorrt_b200.workloads import CONFIGS, MSDAConfig, make_msda_inputs
from oracle.msda_backward import msda_backward_f64
from tests.helpers import kernels_recorded

NAMES = ("value", "reference_points", "sampling_offsets", "attention_weights")
LEVELS3 = ((11, 13), (6, 7), (3, 4))
LEVELS4 = ((10, 12), (5, 6), (3, 3), (2, 2))
LEVELS16 = ((9, 11), (8, 3), (7, 1), (1, 7), (1, 1), (6, 6), (5, 4), (4, 5), (3, 3), (2, 6), (6, 2), (2, 2), (3, 1), (1, 3),
            (2, 1), (1, 2))  # fmt: skip
ENVELOPE = {
    "g1": MSDAConfig("g1", 2, 40, 8, 32, LEVELS4, 4, 1),
    "g2": MSDAConfig("g2", 3, 53, 8, 32, LEVELS3, 8, 2),
    "g4": MSDAConfig("g4", 2, 45, 8, 32, ((12, 20), (6, 10), (3, 5), (2, 3)), 8, 4),
    "l16": MSDAConfig("l16", 2, 30, 4, 32, LEVELS16, 4, 4),  # NP 64: the lane-group kernel's limit
}
# shapes the fused forward does not take: the autograd path composes the plugin-op backward
FALLBACK = {
    "c64": MSDAConfig("c64", 2, 20, 4, 64, ((7, 9), (4, 5)), 8, 4),
    "np36": MSDAConfig("np36", 2, 53, 8, 32, LEVELS3, 12, 2),  # FP16: more than two gather rounds
}


def _dims(cfg):
    return (cfg.batch, cfg.spatial_size, cfg.num_heads, cfg.channels, cfg.num_levels, cfg.num_query, cfg.num_points,
            cfg.points_per_group)  # fmt: skip


def _mask(cfg, kind, seed=5):
    B, Q = cfg.batch, cfg.num_query
    g = torch.Generator().manual_seed(seed)
    if kind == "zero":
        return torch.zeros(B, Q)
    if kind == "uniform":
        return torch.full((B, Q), 1.0 / 6.0)
    if kind == "binary":
        return (torch.rand(B, Q, generator=g) < 0.4).float()
    # "ring": fractional weights 1 / (cameras that see the query), as bev_reference_points_cam makes them; ~1/3 zeros
    seen = (torch.rand(B, Q, generator=g) < 0.5).float()
    return seen / seen.sum(0, keepdim=True).clamp(min=1e-4)


def _grad_slots(cfg, seed=11):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(cfg.num_query, cfg.num_heads * cfg.channels, generator=g)


def _shared_inputs(inputs):
    """Offsets and logits of camera 0 as the single shared copy [Q, M, ...]."""
    value, shapes, ref, off, logits = inputs
    return value, shapes, ref, off[0].contiguous(), logits[0].contiguous()


def _ours(inputs, mask, gs, shared=False, requires=NAMES, prepare=lambda t: t.cuda()):
    value, shapes, ref, off, logits = inputs
    ts = [prepare(t).detach().requires_grad_(n in requires) for n, t in zip(NAMES, (value, ref, off, logits))]
    op = bt.multi_scale_deformable_attn_sca_shared if shared else bt.multi_scale_deformable_attn_sca
    out = op(ts[0], shapes.cuda(), ts[1], ts[2], ts[3], mask.cuda())
    out.backward(prepare(gs))
    return out.detach(), [t.grad for t in ts]


def _oracle(inputs, mask, gs, shared=False, device="cpu", chunk=4096):
    value, shapes, ref, off, logits = inputs
    B, Q = mask.shape
    M, C = value.shape[2], value.shape[3]
    go = (mask.float().unsqueeze(-1) * gs.float().view(1, Q, M * C)).view(B, Q, M, C)
    if shared:
        off = off.reshape(1, *off.shape).expand(B, *off.shape)
        logits = logits.reshape(1, *logits.shape).expand(B, *logits.shape)
    _, gv, gr, goff, glog = msda_backward_f64(value, shapes, ref, off, logits, go, device=device, chunk=chunk)
    if shared:
        goff, glog = goff.sum(0), glog.sum(0)
    return gv, gr, goff, glog


def _max_err(got, want):
    return (got.double().cpu() - want.double().cpu()).abs().max().item()


def _bar(want, dtype, atomics=False):
    m = want.abs().max().item()
    if dtype == torch.float32:
        return 1e-4 * max(m, 1e-30)
    return (1.0 if atomics else 0.5) * float(np.spacing(np.float16(m))) + 1e-4 * max(m, 1e-30)


def _check_all(got, want, dtype, what=""):
    errs = {}
    for n, g, w in zip(NAMES, got, want):
        assert g.dtype == dtype and g.shape == w.shape, (what, n, g.shape, w.shape)
        assert torch.isfinite(g).all(), (what, n)
        errs[n] = (_max_err(g, w), _bar(w, dtype, atomics=n == "value"))
    assert all(e <= b for e, b in errs.values()), (what, errs)
    return errs


# ---- CPU: the C ABI without a GPU ------------------------------------------------------------------------------------
ENTRIES = ("b200_msda_sca_backward_f32", "b200_msda_sca_backward_f16", "b200_msda_sca_shared_backward_f32",
           "b200_msda_sca_shared_backward_f16")  # fmt: skip


def test_fused_backward_symbols_are_declared_bound_and_exported():
    from tests.test_host_logic import _header_symbols

    syms = _header_symbols()
    for s in ENTRIES:
        assert s in syms and s in _lib.SIGNATURES and hasattr(ctypes.CDLL(_lib.LIB_PATH), s)


_A = 1 << 20
_PTRS = [_A * (i + 1) for i in range(11)]  # value, shapes, ref, off, logits, mask, grad_slots, 4 gradients
_WS = _A * 64
_DIMS = [2, 300, 8, 32, 2, 50, 4, 2]


def _call(name, ptrs=_PTRS, ws=_WS, dims=_DIMS):
    return getattr(_lib.load(), name)(*ptrs, ws, *dims, None)


@pytest.mark.parametrize("which", range(8))
def test_null_required_pointer_is_bad_param(which):
    for name in ENTRIES:
        if which == 7:
            assert _call(name, ws=None) == 2
        else:
            ptrs = list(_PTRS)
            ptrs[which] = None
            assert _call(name, ptrs) == 2, name


@pytest.mark.parametrize("which", [0, 2, 3, 4, 5, 6, 7, 8, 9, 10])
def test_pointer_not_aligned_to_its_element_is_bad_param(which):
    for name in ENTRIES:
        ptrs = list(_PTRS)
        ptrs[which] += 1
        assert _call(name, ptrs) == 2, name
        if which in (5, 6) or name.endswith("f32"):  # float tensors: half aligned is not enough
            ptrs[which] += 1
            assert _call(name, ptrs) == 2, name
    assert all(_call(name, ws=_WS + 16) == 2 for name in ENTRIES)


def test_outside_the_lane_group_envelope_is_unsupported_before_any_launch():
    for name in ENTRIES:
        for idx, val in ((3, 64), (3, 16), (6, 6), (7, 3)):  # channels, points % 4, groups
            dims = list(_DIMS)
            dims[idx] = val
            assert _call(name, dims=dims) == 1, (name, idx, val)
        many = list(_DIMS)
        many[4], many[6] = 5, 16  # 80 points
        assert _call(name, dims=many) == 1
        ptrs = list(_PTRS)
        ptrs[6] += 4  # grad_slots float aligned, not 16-byte aligned
        assert _call(name, ptrs) == 1
        assert _call(name, dims=[2, 300, 8, 32, 17, 50, 4, 2]) == 1


def test_nothing_requested_returns_ok():
    ptrs = list(_PTRS[:7]) + [None] * 4
    assert all(_call(name, ptrs) == 0 for name in ENTRIES)


@pytest.mark.gpu
def test_mask_requiring_grad_raises():
    cfg = ENVELOPE["g4"]
    value, shapes, ref, off, logits = (t.cuda() for t in make_msda_inputs(cfg, "U", 1))
    mask = _mask(cfg, "ring").cuda().requires_grad_(True)
    for op in (bt.multi_scale_deformable_attn_sca, bt.multi_scale_deformable_attn_sca_shared):
        with pytest.raises(ValueError, match="bev_mask"):
            op(value.requires_grad_(True), shapes, ref, off, logits, mask)


# ---- GPU: gradients against the oracle -------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("shared", [False, True], ids=["sca", "shared"])
@pytest.mark.parametrize("dist", ["U", "edge"])
@pytest.mark.parametrize("mask_kind", ["ring", "binary", "zero", "uniform"])
def test_small_sca_matches_the_oracle(mask_kind, dist, shared, dtype):
    cfg = CONFIGS["small_sca"]
    inputs = make_msda_inputs(cfg, dist, 21, dtype)
    if shared:
        inputs = _shared_inputs(inputs)
    mask, gs = _mask(cfg, mask_kind), _grad_slots(cfg)
    _, got = _ours(inputs, mask, gs, shared)
    want = _oracle(inputs, mask, gs, shared)
    if mask_kind == "zero":
        assert all((g == 0).all() for g in got)
    else:
        _check_all(got, want, dtype, (mask_kind, dist))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("shared", [False, True], ids=["sca", "shared"])
@pytest.mark.parametrize("name", ENVELOPE)
@pytest.mark.parametrize("mask_kind", ["ring", "binary"])
def test_envelope_configs_match_the_oracle(mask_kind, name, shared, dtype):
    cfg = ENVELOPE[name]
    inputs = make_msda_inputs(cfg, "edge", 31, dtype)
    if shared:
        inputs = _shared_inputs(inputs)
    mask, gs = _mask(cfg, mask_kind), _grad_slots(cfg)
    (_, got), names = kernels_recorded(lambda: _ours(inputs, mask, gs, shared),
                                       lambda names: any("msda_bw_c32_kernel" in n for n in names))  # fmt: skip
    ran = [n for n in names if "msda_bw_" in n and "kernel<" in n]
    epi = [re.search(r"msda_bw_c32_kernel<[^,]+, (\d)>", n) for n in ran if "msda_bw_c32_kernel" in n]
    # the fused forward takes at most two gather rounds (FP16: 32 points); beyond, autograd composes the plugin backward
    fused = dtype == torch.float32 or cfg.num_levels * cfg.num_points <= 32
    assert epi and all(e and e.group(1) == (("2" if shared else "1") if fused else "0") for e in epi), ran
    assert not any("generic" in n for n in ran), ran
    want = _oracle(inputs, mask, gs, shared)
    _check_all(got, want, dtype, (name, mask_kind))
    # the fused entry itself, whichever path autograd took
    entry = f"b200_msda_sca{'_shared' if shared else ''}_backward_{'f32' if dtype == torch.float32 else 'f16'}"
    _check_all(_raw(entry, inputs, mask, gs), want, dtype, (name, mask_kind, "entry"))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("shared", [False, True], ids=["sca", "shared"])
@pytest.mark.parametrize("dist", ["G", "U"])
def test_base_sca_every_element_matches_the_oracle(dist, shared, dtype):
    """G with the camera-ring bev_mask of the same geometry; U with a uniform 1/6 mask."""
    from bevformer_tensorrt_b200.workloads import bev_reference_points_cam, camera_ring_lidar2img

    cfg = CONFIGS["base_sca"]
    inputs = make_msda_inputs(cfg, dist, 0, dtype)
    if dist == "G":
        _, m = bev_reference_points_cam(cfg.bev_hw, camera_ring_lidar2img(cfg.batch), pillars=cfg.points_per_group)
        mask = m.reshape(cfg.batch, cfg.num_query).float()
    else:
        mask = _mask(cfg, "uniform")
    if shared:
        inputs = _shared_inputs(inputs)
    gs = _grad_slots(cfg)
    _, got = _ours(inputs, mask, gs, shared)
    errs = _check_all(got, _oracle(inputs, mask, gs, shared, device="cuda", chunk=2048), dtype, dist)
    print(f"base_sca {dist} {'shared' if shared else 'sca'} {dtype}: "
          + ", ".join(f"{n} err {e:.3e} (bar {b:.3e})" for n, (e, b) in errs.items()))  # fmt: skip


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("shared", [False, True], ids=["sca", "shared"])
@pytest.mark.parametrize("name", FALLBACK)
def test_shapes_the_fused_forward_falls_back_on(name, shared, dtype):
    cfg = FALLBACK[name]
    inputs = make_msda_inputs(cfg, "edge", 35, dtype)
    if shared:
        inputs = _shared_inputs(inputs)
    mask, gs = _mask(cfg, "ring"), _grad_slots(cfg)
    _, got = _ours(inputs, mask, gs, shared)
    want = _oracle(inputs, mask, gs, shared)
    if dtype == torch.float32:
        _check_all(got, want, dtype, name)
    else:
        # the composition rounds go = mask * grad_slots to FP16 and, for the shared form, each camera's offset / logit
        # gradient before the camera sum: two more roundings than the fused kernel, so twice the bar
        for n, g, w in zip(NAMES, got, want):
            assert g.dtype == dtype and g.shape == w.shape and torch.isfinite(g).all(), n
            assert _max_err(g, w) <= 2 * _bar(w, dtype, atomics=True), (name, n)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_queue_mean_trains_like_the_mean_over_the_plugin_op(dtype):
    cfg = CONFIGS["base_tsa"]
    value, shapes, ref, off, logits = (t.cuda() for t in make_msda_inputs(cfg, "U", 3, dtype))
    w = torch.randn(1, cfg.num_query, cfg.num_heads * cfg.channels, generator=torch.Generator().manual_seed(2)).cuda()

    def grads(fused):
        ts = [t.detach().requires_grad_(True) for t in (value, ref, off, logits)]
        if fused:
            out = bt.multi_scale_deformable_attn_queue_mean(ts[0], shapes, *ts[1:])
        else:
            out = torch.mean(bt.multi_scale_deformable_attn(ts[0], shapes, *ts[1:]).flatten(2), dim=0, keepdim=True)
        (out.float() * w).sum().backward()
        return [t.grad for t in ts]

    got, want = grads(True), grads(False)
    for n, g, r in zip(NAMES, got, want):
        assert g.dtype == dtype and g.shape == r.shape
        # both sides round to FP16 once; the fused side forms go = grad / 2 in fp32 instead of rounding it to FP16
        assert _max_err(g, r) <= 2 * _bar(r.float(), dtype, atomics=True), n


# ---- GPU: exactness, isolation, determinism ----------------------------------------------------------------------------
def _raw(fn_name, inputs, mask, gs, asked=(0, 1, 2, 3), go=None):
    """Direct C call; returns the four gradient buffers (None where not asked). ``go``: plugin-op backward instead."""
    lib = _lib.load()
    value, shapes, ref, off, logits = (t.cuda() for t in inputs)
    dt = value.dtype
    B, S, M, C = value.shape
    L, Q = shapes.shape[0], mask.shape[1]
    NP = logits.shape[-1]
    dims = (B, S, M, C, L, Q, NP // L, ref.shape[-1] // 2)
    ws = torch.empty(lib.b200_msda_backward_workspace_size(int(dt == torch.float16), *dims), dtype=torch.uint8,
                     device="cuda")  # fmt: skip
    bufs = [torch.full_like(t, float("nan")) if i in asked else None  # requested buffers must be overwritten
            for i, t in enumerate((value, ref, off, logits))]  # fmt: skip
    ptrs = [b.data_ptr() if b is not None else None for b in bufs]
    mask, gs = mask.cuda().contiguous(), gs.cuda().contiguous()  # alive until the launch has run
    if go is None:
        st = getattr(lib, fn_name)(value.data_ptr(), shapes.data_ptr(), ref.data_ptr(), off.data_ptr(),
                                   logits.data_ptr(), mask.data_ptr(), gs.data_ptr(), *ptrs, ws.data_ptr(), *dims,
                                   _lib.current_stream_ptr())  # fmt: skip
    else:
        go = go.cuda().to(dt).contiguous()
        st = getattr(lib, fn_name)(value.data_ptr(), shapes.data_ptr(), ref.data_ptr(), off.data_ptr(),
                                   logits.data_ptr(), go.data_ptr(), *ptrs, ws.data_ptr(), *dims,
                                   _lib.current_stream_ptr())  # fmt: skip
    assert st == 0
    torch.cuda.synchronize()
    return bufs


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["g4", "g1"])
def test_fp32_sca_gradients_are_the_plugin_backward_bit_for_bit(name):
    """The deterministic gradients of pairs with mask != 0 are those of b200_msda_backward_f32 fed mask * grad_slots,
    bit for bit; pairs with mask == 0 get exact zeros."""
    cfg = ENVELOPE[name]
    inputs = make_msda_inputs(cfg, "edge", 37)
    mask, gs = _mask(cfg, "ring"), _grad_slots(cfg)
    fused = _raw("b200_msda_sca_backward_f32", inputs, mask, gs)
    go = (mask.unsqueeze(-1) * gs.unsqueeze(0)).view(cfg.batch, cfg.num_query, cfg.num_heads, cfg.channels)
    plain = _raw("b200_msda_backward_f32", inputs, mask, gs, go=go)
    on = (mask != 0).cuda()
    assert on.any() and (~on).any()
    for i in (1, 2, 3):
        assert torch.equal(fused[i][on], plain[i][on]), NAMES[i]
        assert (fused[i][~on] == 0).all(), NAMES[i]
    assert _max_err(fused[0], plain[0]) <= 1e-6 * plain[0].abs().max().item()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("poison", [float("nan"), float("inf")])
def test_nonfinite_inputs_of_masked_pairs_change_nothing(poison, dtype):
    """camera-summed form: value pixels, offsets and logits that only mask-0 pairs touch."""
    cfg = ENVELOPE["g4"]
    value, shapes, ref, off, logits = make_msda_inputs(cfg, "U", 39, dtype)
    mask, gs = _mask(cfg, "binary"), _grad_slots(cfg)
    mask[1] = 0.0  # camera 1 sees nothing: all of its value pixels are touched by mask-0 pairs only
    clean_out, clean = _ours((value, shapes, ref, off, logits), mask, gs)
    off_m = (mask == 0).view(cfg.batch, cfg.num_query, 1, 1)
    bad = (torch.where(torch.arange(cfg.batch).view(-1, 1, 1, 1) == 1, torch.full_like(value, poison), value),
           shapes, torch.where(off_m, torch.full_like(ref, poison), ref), torch.where(off_m, torch.full_like(off, poison), off),
           torch.where(off_m, torch.full_like(logits, poison), logits))  # fmt: skip
    out, got = _ours(bad, mask, gs)
    assert _max_err(out, clean_out) <= 1e-6 * clean_out.abs().max().item()  # the camera sum is a float atomic
    for i in (1, 2, 3):
        assert torch.isfinite(got[i]).all() and torch.equal(got[i], clean[i]), NAMES[i]
    assert torch.isfinite(got[0]).all() and (got[0][1] == 0).all()
    assert _max_err(got[0], clean[0]) <= _bar(clean[0].float(), dtype, True)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_shared_form_isolates_masked_cameras_and_unseen_queries(dtype):
    cfg = ENVELOPE["g4"]
    value, shapes, ref, off, logits = _shared_inputs(make_msda_inputs(cfg, "U", 41, dtype))
    mask, gs = _mask(cfg, "binary"), _grad_slots(cfg)
    mask[:, 5] = 0.0  # query 5: no camera
    mask[1] = 0.0  # camera 1: no query, so none of its value pixels is read
    clean_out, clean = _ours((value, shapes, ref, off, logits), mask, gs, shared=True)
    bad_v, bad_r, bad_o, bad_l = value.clone(), ref.clone(), off.clone(), logits.clone()
    bad_v[1] = float("inf")
    for b in range(cfg.batch):  # reference points of the mask-0 (camera, query) pairs
        bad_r[b, mask[b] == 0] = float("nan")
    bad_o[5] = float("nan")
    bad_l[5] = float("nan")
    out, got = _ours((bad_v, shapes, bad_r, bad_o, bad_l), mask, gs, shared=True)
    assert torch.equal(out, clean_out)  # one plain store per slot: deterministic
    assert (got[0][1] == 0).all() and torch.isfinite(got[0]).all()
    assert _max_err(got[0], clean[0]) <= _bar(clean[0].float(), dtype, True)
    for i in (1, 2, 3):
        assert torch.isfinite(got[i]).all() and torch.equal(got[i], clean[i]), NAMES[i]
    assert (got[2][5] == 0).all() and (got[3][5] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("shared", [False, True], ids=["sca", "shared"])
def test_determinism_subsets_and_overwrite(shared, dtype):
    cfg = ENVELOPE["g4"]
    inputs = make_msda_inputs(cfg, "edge", 45, dtype)
    if shared:
        inputs = _shared_inputs(inputs)
    mask, gs = _mask(cfg, "ring"), _grad_slots(cfg)
    name = f"b200_msda_sca{'_shared' if shared else ''}_backward_{'f32' if dtype == torch.float32 else 'f16'}"
    first = _raw(name, inputs, mask, gs)
    again = _raw(name, inputs, mask, gs)
    for i in (1, 2, 3):
        assert torch.equal(first[i], again[i]), NAMES[i]
    for asked in ((1,), (2,), (3,), (0, 2), (1, 3), (2, 3), (0, 1, 2)):
        got = _raw(name, inputs, mask, gs, asked)
        for i in range(4):
            if i not in asked:
                assert got[i] is None
            elif i == 0:
                assert torch.isfinite(got[0]).all() and _max_err(got[0], first[0]) <= _bar(first[0].float(), dtype, True)
            else:
                assert torch.equal(got[i], first[i]), (asked, NAMES[i])


@pytest.mark.gpu
@pytest.mark.parametrize("shared", [False, True], ids=["sca", "shared"])
def test_forward_bits_do_not_depend_on_requires_grad_and_accum_stays_inference_only(shared):
    cfg = CONFIGS["small_sca"]
    for dtype in (torch.float32, torch.float16):
        inputs = make_msda_inputs(cfg, "edge", 55, dtype)
        if shared:
            inputs = _shared_inputs(inputs)
        mask, gs = _mask(cfg, "ring"), _grad_slots(cfg)
        out, _ = _ours(inputs, mask, gs, shared)
        op = bt.multi_scale_deformable_attn_sca_shared if shared else bt.multi_scale_deformable_attn_sca
        plain = op(*(t.cuda() for t in inputs), mask.cuda())
        assert plain.grad_fn is None and torch.equal(out, plain)
        with torch.no_grad():
            ng = op(*(t.cuda().requires_grad_(t.is_floating_point()) for t in inputs), mask.cuda())
        assert ng.grad_fn is None and torch.equal(ng, plain)
    if not shared:
        value, shapes, ref, off, logits = (t.cuda() for t in make_msda_inputs(cfg, "U", 56))
        acc = torch.zeros(cfg.num_query, cfg.num_heads * cfg.channels, device="cuda")
        res = bt.multi_scale_deformable_attn_sca(value.requires_grad_(True), shapes, ref, off, logits,
                                                 _mask(cfg, "ring").cuda(), accum=acc)  # fmt: skip
        assert res is acc and res.grad_fn is None
        assert torch.allclose(acc, bt.multi_scale_deformable_attn_sca(value.detach(), shapes, ref, off, logits,
                                                                     _mask(cfg, "ring").cuda()), atol=1e-5)  # fmt: skip


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("shared", [False, True], ids=["sca", "shared"])
def test_forward_and_backward_replay_from_a_cuda_graph(shared, dtype):
    cfg = CONFIGS["small_sca"]
    first = make_msda_inputs(cfg, "edge", 57, dtype)
    second = make_msda_inputs(cfg, "U", 58, dtype)
    if shared:
        first, second = _shared_inputs(first), _shared_inputs(second)
    mask, gs = _mask(cfg, "ring").cuda(), _grad_slots(cfg).cuda()
    op = bt.multi_scale_deformable_attn_sca_shared if shared else bt.multi_scale_deformable_attn_sca
    static = [t.cuda().requires_grad_(t.is_floating_point()) for t in first]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            op(*static, mask).backward(gs)
    torch.cuda.current_stream().wait_stream(side)
    for t in static:
        t.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = op(*static, mask)
        out.backward(gs)
    with torch.no_grad():
        for t, src in zip(static, second):
            t.copy_(src)
    graph.replay()
    torch.cuda.synchronize()
    want_out, want = _ours(second, mask.cpu(), gs.cpu(), shared)
    assert _max_err(out.detach(), want_out) <= 1e-5 * max(1.0, want_out.abs().max().item())
    grads = [static[0].grad, static[2].grad, static[3].grad, static[4].grad]
    for i in (1, 2, 3):
        assert torch.equal(grads[i], want[i]), NAMES[i]
    assert _max_err(grads[0], want[0]) <= _bar(want[0].float(), dtype, True)


@pytest.mark.gpu
def test_sca_module_trains_the_same_in_every_mode():
    """SpatialCrossAttentionTRTP unfused, fused and fused camera-shared from one state_dict: every parameter gradient
    and the query / value gradients agree within 1e-4 x max|g|."""
    from bevformer_tensorrt_b200.modules import SpatialCrossAttentionTRTP
    from bevformer_tensorrt_b200.workloads import bev_reference_points_cam, camera_ring_lidar2img

    torch.manual_seed(0)
    g = torch.Generator().manual_seed(0)
    nq, cams = 2500, 6
    query = torch.randn(1, nq, 256, generator=g).cuda()
    value = torch.randn(cams, 375, 256, generator=g).cuda()
    uv, mask = bev_reference_points_cam((50, 50), camera_ring_lidar2img(cams))
    ref_cam = uv.view(cams, 1, nq, 4, 2).clamp(-60000, 60000).cuda()
    shapes = torch.tensor([[15, 25]], device="cuda")
    weight = torch.randn(1, nq, 256, generator=g).cuda()
    base = SpatialCrossAttentionTRTP(num_levels=1, num_points=8).cuda()
    with torch.no_grad():
        base.deformable_attention.sampling_offsets.weight.mul_(20.0)
    state = base.state_dict()
    results = []
    for kw in ({}, {"fused": True}, {"fused": True, "camera_shared": True}):
        m = SpatialCrossAttentionTRTP(num_levels=1, num_points=8, **kw).cuda()
        m.load_state_dict(state)
        q, v = query.clone().requires_grad_(True), value.clone().requires_grad_(True)
        (m.forward_trt(q, v, ref_cam, mask.cuda(), shapes) * weight).sum().backward()
        gr = {n: p.grad for n, p in m.named_parameters()}
        gr["query"], gr["value"] = q.grad, v.grad
        assert all(t is not None for t in gr.values()), kw
        results.append(gr)
    for other in results[1:]:
        for n, want in results[0].items():
            scale = want.abs().max().item()
            assert scale > 0 and (other[n] - want).abs().max().item() <= 1e-4 * scale, n
