"""MSDA backward (csrc/msda_backward.cu, b200_msda_backward_f32 / _f16, and the autograd backward of
multi_scale_deformable_attn[2]). Oracle: oracle/msda_backward.py, a float64 autograd gather pinned to the bit-exact
sampling-index records of the FP32 oracle; it is itself pinned here, on the CPU, against float64 autograd through the
reference's grid_sample algorithm and against finite differences.

Tolerances, per gradient tensor g:
  FP32: 1e-4 x max|g| (fp32 summation order, fp32 expf, the fp32 rounding of the sampling position).
  FP16: the oracle runs on the FP16-rounded inputs; everything between the loads and the stores is fp32 and each gradient
        is rounded once, so the bar is half an FP16 spacing of max|g| plus the FP32 bar. grad_value is summed with float
        atomics, whose order can move the rounded result by one more half spacing.
grad_sampling_offsets, grad_attention_weights and grad_reference_points are ordered sums and are checked bitwise for
run-to-run and requested-subset stability; grad_value is not."""
import ctypes

import numpy as np
import pytest
import torch

import bevformer_tensorrt_b200 as bt
from bevformer_tensorrt_b200 import _lib
from bevformer_tensorrt_b200.workloads import CONFIGS, MSDAConfig, make_msda_inputs
from oracle import msda as omsda
from oracle.msda_backward import msda_backward_f64
from tests.helpers import kernels_recorded

NAMES = ("value", "reference_points", "sampling_offsets", "attention_weights")

LEVELS3 = ((11, 13), (6, 7), (3, 4))
LEVELS4 = ((10, 12), (5, 6), (3, 3), (2, 2))
LEVELS16 = ((9, 11), (8, 3), (7, 1), (1, 7), (1, 1), (6, 6), (5, 4), (4, 5), (3, 3), (2, 6), (6, 2), (2, 2), (3, 1), (1, 3),
            (2, 1), (1, 2))  # fmt: skip
# shapes on both sides of every clause of the kernel selection rule: (config, kernel both dtypes run)
ENVELOPE = {
    "g1": (MSDAConfig("g1", 2, 40, 8, 32, LEVELS4, 4, 1), "c32"),
    "g2": (MSDAConfig("g2", 1, 53, 8, 32, LEVELS3, 12, 2), "c32"),  # NP 36
    "g4": (MSDAConfig("g4", 2, 45, 8, 32, ((12, 20), (6, 10), (3, 5), (2, 3)), 8, 4), "c32"),
    "l16": (MSDAConfig("l16", 1, 30, 4, 32, LEVELS16, 4, 4), "c32"),  # NP 64: the lane-group kernel's limit
    "np80": (MSDAConfig("np80", 1, 40, 8, 32, LEVELS4, 20, 4), "generic"),  # more points than the kernel parks
    "g8": (MSDAConfig("g8", 2, 30, 4, 32, ((8, 9), (4, 5)), 8, 8), "generic"),
    "c64": (MSDAConfig("c64", 2, 20, 4, 64, ((7, 9), (4, 5)), 8, 4), "generic"),
    "c16": (MSDAConfig("c16", 1, 25, 4, 16, ((7, 9), (4, 5)), 4, 2), "generic"),
    "c5": (MSDAConfig("c5", 1, 25, 3, 5, ((6, 7), (3, 4)), 4, 2), "generic"),
    "p2": (MSDAConfig("p2", 1, 30, 4, 32, ((8, 9), (4, 5)), 2, 2), "generic"),
}


def _dims(cfg):
    return (cfg.batch, cfg.spatial_size, cfg.num_heads, cfg.channels, cfg.num_levels, cfg.num_query, cfg.num_points,
            cfg.points_per_group)  # fmt: skip


def _grad_out(cfg, dtype, seed=11):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(cfg.batch, cfg.num_query, cfg.num_heads, cfg.channels, generator=g).to(dtype)


def _ours(inputs, go, requires=NAMES, op=None, prepare=lambda t: t.cuda()):
    """(out, [grad per NAMES entry or None]) through the autograd Function."""
    value, shapes, ref, off, logits = inputs
    ts = [prepare(t).detach().requires_grad_(n in requires) for n, t in zip(NAMES, (value, ref, off, logits))]
    out = (op or bt.multi_scale_deformable_attn)(ts[0], shapes.cuda(), ts[1], ts[2], ts[3])
    out.backward(prepare(go))
    return out.detach(), [t.grad for t in ts]


def _oracle(inputs, go, device="cpu", chunk=4096):
    value, shapes, ref, off, logits = inputs
    return msda_backward_f64(value, shapes, ref, off, logits, go, device=device, chunk=chunk)


def _max_err(got, want):
    return (got.double().cpu() - want.double().cpu()).abs().max().item()


def _bar(want, dtype, atomics=False):
    m = want.abs().max().item()
    if dtype == torch.float32:
        return 1e-4 * max(m, 1e-30)
    return (1.0 if atomics else 0.5) * float(np.spacing(np.float16(m))) + 1e-4 * max(m, 1e-30)


def _check_all(got, want, dtype, what=""):
    errs = {}
    for n, g, w in zip(NAMES, got, want[1:]):
        assert g.dtype == dtype and g.shape == w.shape, (what, n)
        errs[n] = (_max_err(g, w), _bar(w, dtype, atomics=n == "value"))
        assert torch.isfinite(g).all(), (what, n)
    assert all(e <= b for e, b in errs.values()), (what, errs)
    return errs


# ---- CPU: the C ABI without a GPU ------------------------------------------------------------------------------------
def test_backward_symbols_are_declared_and_bound():
    from tests.test_host_logic import _header_symbols

    syms = _header_symbols()
    for s in ("b200_msda_backward_workspace_size", "b200_msda_backward_f32", "b200_msda_backward_f16"):
        assert s in syms and s in _lib.SIGNATURES and hasattr(ctypes.CDLL(_lib.LIB_PATH), s)


# fake device addresses: every check below must return before anything touches them
_A = 1 << 20
_PTRS = [_A * (i + 1) for i in range(10)]  # value, shapes, ref, off, logits, grad_out, 4 gradients
_WS = _A * 64
_DIMS = [2, 300, 8, 32, 2, 50, 4, 2]  # batch, spatial_size, heads, channels, levels, queries, points, points per group


def _f32(ptrs=_PTRS, ws=_WS, dims=_DIMS):
    return _lib.load().b200_msda_backward_f32(*ptrs, ws, *dims, None)


def _f16(ptrs=_PTRS, ws=_WS, dims=_DIMS):
    return _lib.load().b200_msda_backward_f16(*ptrs, ws, *dims, None)


@pytest.mark.parametrize("which", range(6))
def test_null_required_pointer_is_bad_param(which):
    ptrs = list(_PTRS)
    ptrs[which] = None
    assert _f32(ptrs) == 2 and _f16(ptrs) == 2
    assert _f32(ws=None) == 2 and _f16(ws=None) == 2


@pytest.mark.parametrize("idx", range(8))
@pytest.mark.parametrize("val", [0, -3])
def test_non_positive_dimension_is_bad_param(idx, val):
    dims = list(_DIMS)
    dims[idx] = val
    assert _f32(dims=dims) == 2 and _f16(dims=dims) == 2
    assert all(_lib.load().b200_msda_backward_workspace_size(dt, *dims) == 0 for dt in (0, 1))


def test_seventeen_levels_and_the_forward_size_limit():
    lib = _lib.load()
    l17 = list(_DIMS)
    l17[4] = 17
    assert _f32(dims=l17) == 1 and _f16(dims=l17) == 1
    l16 = list(_DIMS)
    l16[4] = 16
    big = list(_DIMS)
    big[1] = (1 << 31) // (8 * 32 * 4)  # (S + 1) * M * C * 4 >= 2^31
    assert _f32(dims=big) == 2 and _f16(dims=big) == 2
    for dt in (0, 1):
        assert lib.b200_msda_backward_workspace_size(dt, *l17) == 0 and lib.b200_msda_backward_workspace_size(dt, *big) == 0
        assert lib.b200_msda_backward_workspace_size(dt, *l16) > 0
    assert lib.b200_msda_backward_workspace_size(2, *_DIMS) == 0  # no INT8 backward


@pytest.mark.parametrize("which", [0, 2, 3, 4, 5, 6, 7, 8, 9])
def test_pointer_not_aligned_to_its_element_is_bad_param(which):
    ptrs = list(_PTRS)
    ptrs[which] += 1
    assert _f16(ptrs) == 2 and _f32(ptrs) == 2
    ptrs[which] += 1  # half aligned, not float aligned
    assert _f32(ptrs) == 2
    assert _f16(ws=_WS + 16) == 2 and _f32(ws=_WS + 16) == 2  # workspace: 256 bytes


def test_workspace_size_formula():
    lib = _lib.load()

    def up(n):
        return (n + 255) // 256 * 256

    for dims in (_DIMS, list(_dims(CONFIGS["base_sca"])), list(_dims(ENVELOPE["c5"][0]))):
        B, S, M, C, L, Q, P, G = dims
        ref_part = up(B * Q * M * G * 2 * 4)
        assert lib.b200_msda_backward_workspace_size(0, *dims) == ref_part
        assert lib.b200_msda_backward_workspace_size(1, *dims) == up(B * S * M * C * 4) + ref_part


def test_nothing_requested_returns_ok_without_launch():
    ptrs = list(_PTRS[:6]) + [None] * 4
    assert _f32(ptrs) == 0 and _f16(ptrs) == 0


# ---- CPU: the oracle -------------------------------------------------------------------------------------------------
def _off_integers(inputs, eps=1e-3):
    """The same inputs with every sampling position at least ``eps`` pixels away from an integer (where the bilinear
    derivative jumps and two correct implementations may differ)."""
    value, shapes, ref, off, logits = inputs
    B, Q, M, _ = off.shape
    L, G = shapes.shape[0], ref.shape[-1] // 2
    P = logits.shape[-1] // L
    o = off.double().reshape(B, Q, M, L, P // G, G, 2).clone()
    wh = torch.stack([shapes[:, 1], shapes[:, 0]], -1).double().view(1, 1, 1, L, 1, 1, 2)
    pos = ref.double().reshape(B, Q, 1, 1, 1, G, 2) * wh + o - 0.5
    near = (pos - pos.round()).abs() < eps
    o = torch.where(near, o + 0.25, o)
    return value, shapes, ref, o.reshape(off.shape).float(), logits


ORACLE_CASES = {
    "cpu_plumbing": (CONFIGS["cpu_plumbing"], "edge"),
    "small_sca": (CONFIGS["small_sca"], "edge"),
    "odd": (MSDAConfig("odd", 2, 17, 3, 5, ((6, 7), (3, 4)), 2, 1), "edge"),
}


@pytest.mark.parametrize("name", ORACLE_CASES)
def test_oracle_forward_is_the_fp32_oracle_and_gradients_are_grid_sample_autograd(name):
    cfg, dist = ORACLE_CASES[name]
    inputs = _off_integers(make_msda_inputs(cfg, dist, 5))
    go = _grad_out(cfg, torch.float32)
    out, *grads = _oracle(inputs, go)
    want_out = omsda.msda_f32(*(t.float().numpy() for t in inputs))
    assert np.abs(out.numpy() - want_out).max() < 1e-5
    value, shapes, ref, off, logits = inputs
    ts = [t.double().requires_grad_(True) for t in (value, ref, off, logits)]
    port = omsda.msda_torch_port(ts[0], shapes, ts[1], ts[2], ts[3])
    port.backward(go.double())
    assert (port.detach() - out).abs().max().item() < 1e-4  # fp32 position rounding moves the oracle's fractions
    for n, t, g in zip(NAMES, ts, grads):
        assert g.shape == t.shape
        assert (t.grad - g).abs().max().item() <= 1e-4 * t.grad.abs().max().item() + 1e-12, n


def test_oracle_against_finite_differences():
    cfg = MSDAConfig("fd", 1, 3, 2, 3, ((4, 5), (2, 3)), 2, 2)
    inputs = _off_integers(make_msda_inputs(cfg, "U", 9), eps=0.05)
    go = _grad_out(cfg, torch.float32)
    _, *grads = _oracle(inputs, go)
    value, shapes, ref, off, logits = inputs

    def f(v, r, o, w):  # the reference algorithm in float64: an independent function to difference
        return (omsda.msda_torch_port(v, shapes, r, o, w) * go.double()).sum().item()

    base = [t.double() for t in (value, ref, off, logits)]
    h = 1e-6
    gen = torch.Generator().manual_seed(0)
    for i, (n, g) in enumerate(zip(NAMES, grads)):
        for _ in range(12):
            j = int(torch.randint(base[i].numel(), (1,), generator=gen))
            hi, lo = [t.clone() for t in base], [t.clone() for t in base]
            hi[i].view(-1)[j] += h
            lo[i].view(-1)[j] -= h
            fd = (f(*hi) - f(*lo)) / (2 * h)
            assert abs(fd - g.reshape(-1)[j].item()) < 1e-5 * max(1.0, abs(fd)), (n, j)


# ---- GPU -------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("name,dist", [("cpu_plumbing", "U"), ("cpu_plumbing", "edge"), ("tiny_sca", "G"), ("tiny_sca", "edge"),
                                       ("small_sca", "U"), ("small_sca", "edge"), ("base_decoder", "U"),
                                       ("base_decoder", "edge")])  # fmt: skip
def test_gradients_match_the_oracle(name, dist, dtype):
    cfg = CONFIGS[name]
    inputs = make_msda_inputs(cfg, dist, 21, dtype)
    go = _grad_out(cfg, dtype)
    _, got = _ours(inputs, go)
    _check_all(got, _oracle(inputs, go), dtype, (name, dist))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("name,dist", [("base_tsa", "U"), ("base_sca", "G")])
def test_base_shapes_match_the_oracle(name, dist, dtype):
    """The headline shapes, every element of every gradient; the float64 oracle runs on the GPU in query chunks."""
    cfg = CONFIGS[name]
    inputs = make_msda_inputs(cfg, dist, 0, dtype)
    go = _grad_out(cfg, dtype)
    _, got = _ours(inputs, go)
    want = _oracle(inputs, go, device="cuda", chunk=2048)
    errs = _check_all(got, want, dtype, name)
    print(f"{name} {dist} {dtype}: " + ", ".join(f"{n} err {e:.3e} (bar {b:.3e})" for n, (e, b) in errs.items()))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("name", ENVELOPE)
@pytest.mark.parametrize("dist", ["edge", "U"])
def test_both_kernels_across_the_selection_rule(name, dist, dtype):
    cfg, kernel = ENVELOPE[name]
    inputs = make_msda_inputs(cfg, dist, 31, dtype)
    go = _grad_out(cfg, dtype)
    took = lambda names: any(f"msda_bw_{kernel}_kernel" in n for n in names)  # noqa: E731
    (_, got), names = kernels_recorded(lambda: _ours(inputs, go), took)
    ran = {n for n in names if "msda_bw_" in n}
    assert took(ran), ran
    assert not any(f"msda_bw_{'generic' if kernel == 'c32' else 'c32'}_kernel" in n for n in ran), ran
    _check_all(got, _oracle(inputs, go), dtype, (name, dist))


def _misaligned(t):
    """The same values in a contiguous device view whose data pointer is one element past 16-byte alignment."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device="cuda")
    view = buf[1:].view(t.shape)
    view.copy_(t)
    assert view.is_contiguous() and view.data_ptr() % 16 != 0
    return view


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_tensors_one_element_off_alignment(dtype):
    cfg = ENVELOPE["g4"][0]
    inputs = make_msda_inputs(cfg, "edge", 33, dtype)
    go = _grad_out(cfg, dtype)
    _, got = _ours(inputs, go, prepare=_misaligned)
    _check_all(got, _oracle(inputs, go), dtype)


def _probe(C, dtype):
    """Dyadic values and grad_out, one 4x6 level, reference points 0 (position = offset - 0.5), uniform logits over four
    points: every product and sum of the backward is exact in fp32. Positions: every pair from the list below."""
    H, W = 4, 6
    ys = [-1.0, -0.5, 0.0, 1.5, H - 1.0, H - 0.5, float(H)]
    xs = [-1.0, -0.5, 0.0, 2.25, W - 1.0, W - 0.5, float(W)]
    pairs = [(y, x) for y in ys for x in xs] + [(1.0, 1.0), (2.5, 3.5), (0.25, 4.75)]  # 52 = 13 queries x 4 points
    Q, M, NP = 13, 2, 4
    g = torch.Generator().manual_seed(3)
    value = torch.randint(-8, 9, (1, H * W, M, C), generator=g).float() / 4
    go = torch.randint(-4, 5, (1, Q, M, C), generator=g).float() / 2
    pos = torch.tensor(pairs).view(Q, 1, NP, 2).expand(Q, M, NP, 2)
    off = torch.stack([pos[..., 1], pos[..., 0]], -1) + 0.5  # (x, y) innermost
    off = off.reshape(1, Q, M, NP * 2).contiguous()
    ref = torch.zeros(1, Q, 1, 2)
    logits = torch.zeros(1, Q, M, NP)
    shapes = torch.tensor([[H, W]], dtype=torch.int32)
    inputs = [t.to(dtype) if t.is_floating_point() else t for t in (value, shapes, ref, off, logits)]
    return inputs, go.to(dtype), pos


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("C", [32, 8])
def test_exact_probe_on_integer_and_border_positions(C, dtype):
    inputs, go, pos = _probe(C, dtype)
    _, got = _ours(inputs, go)
    want = _oracle(inputs, go)[1:]
    for n, g, w in zip(NAMES, got, want):
        w = w if dtype == torch.float32 else w.to(torch.float16)  # exact in fp32, so FP16 is one rounding of the truth
        assert torch.equal(g.double().cpu(), w.double()), (n, _max_err(g, w))
    # a position at exactly -1 or H (W) is outside the range gate: no offset gradient, whatever its neighbours hold
    y, x = pos[..., 0], pos[..., 1]
    out = (y <= -1) | (x <= -1) | (y >= 4) | (x >= 6)
    goff = got[2].float().cpu().view(13, 2, 4, 2)
    assert out.any() and (goff[out] == 0).all() and (goff[~out] != 0).any()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_items_with_no_point_in_range(dtype):
    """All points of some items out of range (mixed into visible warps), and a camera that sees nothing (whole warps
    leave early): zero offset / reference-point / value gradients, logits gradients exactly 0."""
    cfg = CONFIGS["small_sca"]
    value, shapes, ref, off, logits = make_msda_inputs(cfg, "U", 41, dtype)
    ref = ref.clone()
    ref[1] = 30.0  # camera 1 sees nothing
    ref[0, ::3] = -20.0  # every third query of camera 0 is invisible
    go = _grad_out(cfg, dtype)
    _, got = _ours((value, shapes, ref, off, logits), go)
    gv, gref, goff, glog = got
    for g in (gv[1], gref[1], goff[1], glog[1], gref[0, ::3], goff[0, ::3], glog[0, ::3]):
        assert (g == 0).all()
    assert (gv[0] != 0).any() and (glog[0, 1::3] != 0).any()
    _check_all(got, _oracle((value, shapes, ref, off, logits), go), dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["g4", "c5"])
def test_grad_value_touches_only_the_pixels_the_index_records_name(name):
    cfg = ENVELOPE[name][0]
    inputs = make_msda_inputs(cfg, "edge", 43)
    value, shapes, ref, off, logits = inputs
    _, idx = omsda.msda_f32(*(t.numpy() for t in inputs), return_index=True)
    b, q, m = cfg.batch - 1, 7, 1
    go = torch.zeros(cfg.batch, cfg.num_query, cfg.num_heads, cfg.channels)
    go[b, q, m] = 1.0
    allowed = torch.zeros(cfg.spatial_size, dtype=torch.bool)
    start = 0
    for lvl, (H, W) in enumerate(cfg.spatial_shapes):
        for p in range(cfg.num_points):
            r = idx[b, q, m, lvl * cfg.num_points + p]
            for t, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
                if r["in_range"] and (r["tap_mask"] >> t) & 1:
                    allowed[start + (r["h_low"] + dy) * W + r["w_low"] + dx] = True
        start += H * W
    assert allowed.any()
    gv = _ours(inputs, go)[1][0].cpu()
    touched = (gv != 0).any(-1)  # [B, S, M]
    assert touched[b, :, m][allowed].any() and not touched[b, :, m][~allowed].any()
    touched[b, :, m] = False
    assert not touched.any()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("name", ["g4", "g8"])
def test_determinism_and_requested_subsets(name, dtype):
    cfg = ENVELOPE[name][0]
    inputs = make_msda_inputs(cfg, "edge", 45, dtype)
    go = _grad_out(cfg, dtype)
    _, first = _ours(inputs, go)
    _, again = _ours(inputs, go)
    for i in (1, 2, 3):
        assert torch.equal(first[i], again[i]), NAMES[i]
    scale = first[0].float().abs().max().item()
    assert _max_err(first[0], again[0]) <= (1e-6 * scale if dtype == torch.float32 else float(np.spacing(np.float16(scale))))
    for subset in ([1], [2], [3], [1, 2], [2, 3], [0, 3], [0, 1], [1, 2, 3]):
        _, got = _ours(inputs, go, requires=[NAMES[i] for i in subset])
        for i in range(4):
            if i not in subset:
                assert got[i] is None
            elif i > 0:
                assert torch.equal(got[i], first[i]), (subset, NAMES[i])


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("name", ["g4", "c16"])
def test_requested_gradients_are_overwritten_and_others_untouched(name, dtype):
    cfg = ENVELOPE[name][0]
    lib = _lib.load()
    inputs = make_msda_inputs(cfg, "edge", 47, dtype)
    go = _grad_out(cfg, dtype).cuda()
    value, shapes, ref, off, logits = (t.cuda() for t in inputs)
    ws = torch.empty(lib.b200_msda_backward_workspace_size(int(dtype == torch.float16), *_dims(cfg)), dtype=torch.uint8,
                     device="cuda")  # fmt: skip
    fn = lib.b200_msda_backward_f32 if dtype == torch.float32 else lib.b200_msda_backward_f16
    _, want = _ours(inputs, go.cpu())
    for asked in ((0, 1, 2, 3), (0, 2), (1, 3), (3,)):
        bufs = [torch.full_like(t, float("nan")) for t in (value, ref, off, logits)]
        ptrs = [b.data_ptr() if i in asked else None for i, b in enumerate(bufs)]
        st = fn(value.data_ptr(), shapes.data_ptr(), ref.data_ptr(), off.data_ptr(), logits.data_ptr(), go.data_ptr(),
                *ptrs, ws.data_ptr(), *_dims(cfg), _lib.current_stream_ptr())
        assert st == 0
        for i, b in enumerate(bufs):
            if i not in asked:
                assert torch.isnan(b).all(), NAMES[i]
            elif i == 0:
                assert torch.isfinite(b).all() and _max_err(b, want[0]) <= _bar(want[0].float(), dtype, True)
            else:
                assert torch.equal(b, want[i]), NAMES[i]


@pytest.mark.gpu
def test_gradient_dtype_is_the_input_dtype():
    """The modules pass FP16 value with FP32 reference points: each gradient comes back in its input's dtype and shape."""
    cfg = CONFIGS["small_sca"]
    value, shapes, ref, off, logits = make_msda_inputs(cfg, "U", 49, torch.float16)
    go = _grad_out(cfg, torch.float16)
    ts = [value.cuda().requires_grad_(), ref.float().cuda().requires_grad_(),
          off.float().view(cfg.batch, cfg.num_query, cfg.num_heads, -1, 2).cuda().requires_grad_(),
          logits.cuda().requires_grad_()]  # fmt: skip
    out = bt.multi_scale_deformable_attn(ts[0], shapes.cuda(), ts[1], ts[2], ts[3])
    out.backward(go.cuda())
    for t in ts:
        assert t.grad.dtype == t.dtype and t.grad.shape == t.shape
    _, want = _ours((value, shapes, ref, off, logits), go)
    assert torch.equal(ts[1].grad, want[1].float()) and torch.equal(ts[2].grad.view(want[2].shape), want[2].float())


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("poison", [float("nan"), float("inf")])
def test_poisoned_pixel_no_tap_reads_changes_nothing(dtype, poison):
    cfg = CONFIGS["cpu_plumbing"]
    inputs = make_msda_inputs(cfg, "edge", 51, dtype)
    value, shapes, ref, off, logits = inputs
    _, idx = omsda.msda_f32(*(t.float().numpy() for t in inputs), return_index=True)
    H, W = cfg.spatial_shapes[0]
    read = np.zeros((cfg.num_heads, H * W), bool)
    for t, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        ok = (idx["in_range"] != 0) & (((idx["tap_mask"] >> t) & 1) != 0)  # [B, Q, M, NP]
        pix = (idx["h_low"] + dy) * W + idx["w_low"] + dx
        for m in range(cfg.num_heads):
            read[m, pix[0, :, m][ok[0, :, m]]] = True
    m = 2
    free = np.flatnonzero(~read[m])
    assert free.size > 0
    bad = value.clone()
    bad[0, int(free[0]), m, :] = poison
    go = _grad_out(cfg, dtype)
    _, clean = _ours(inputs, go)
    _, got = _ours((bad, shapes, ref, off, logits), go)
    for i in (1, 2, 3):
        assert torch.equal(clean[i], got[i]), NAMES[i]
    assert torch.isfinite(got[0]).all() and (got[0][0, int(free[0]), m] == 0).all()
    assert _max_err(got[0], clean[0]) <= _bar(clean[0].float(), dtype, True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["g4", "c16"])
def test_nan_offset_is_an_out_of_range_point(name):
    cfg = ENVELOPE[name][0]
    inputs = make_msda_inputs(cfg, "U", 53)
    value, shapes, ref, off, logits = inputs
    go = _grad_out(cfg, torch.float32)
    far = off.clone()
    far[0, 3, 1, 4] = 1e6  # x of point 2: far outside
    nan = off.clone()
    nan[0, 3, 1, 4] = float("nan")
    _, want = _ours((value, shapes, ref, far, logits), go)
    _, got = _ours((value, shapes, ref, nan, logits), go)
    for i in (1, 2, 3):
        assert torch.isfinite(got[i]).all() and torch.equal(got[i], want[i]), NAMES[i]
    assert (got[2][0, 3, 1, 4:6] == 0).all() and torch.isfinite(got[0]).all()


@pytest.mark.gpu
def test_h2_entry_gives_the_same_gradients_and_forward_bits_do_not_depend_on_requires_grad():
    cfg = CONFIGS["small_sca"]
    for dtype in (torch.float32, torch.float16):
        inputs = make_msda_inputs(cfg, "edge", 55, dtype)
        go = _grad_out(cfg, dtype)
        out1, g1 = _ours(inputs, go)
        out2, g2 = _ours(inputs, go, op=bt.multi_scale_deformable_attn2)
        with torch.no_grad():
            plain = bt.multi_scale_deformable_attn(*(t.cuda() for t in inputs))
        assert torch.equal(out1, plain) and torch.equal(out2, plain)
        for i in (1, 2, 3):
            assert torch.equal(g1[i], g2[i])
        assert _max_err(g1[0], g2[0]) <= _bar(g1[0].float(), dtype, True)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_forward_and_backward_replay_from_a_cuda_graph(dtype):
    cfg = CONFIGS["small_sca"]
    first = make_msda_inputs(cfg, "edge", 57, dtype)
    second = make_msda_inputs(cfg, "U", 58, dtype)
    go = _grad_out(cfg, dtype).cuda()
    static = [t.cuda().requires_grad_(t.is_floating_point()) for t in first]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            bt.multi_scale_deformable_attn(*static).backward(go)
    torch.cuda.current_stream().wait_stream(side)
    for t in static:
        t.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = bt.multi_scale_deformable_attn(*static)
        out.backward(go)
    with torch.no_grad():
        for t, src in zip(static, second):
            t.copy_(src)
    graph.replay()
    torch.cuda.synchronize()
    want_out, want = _ours(second, go.cpu())
    assert torch.equal(out.detach(), want_out)
    grads = [static[0].grad, static[2].grad, static[3].grad, static[4].grad]
    for i in (1, 2, 3):
        assert torch.equal(grads[i], want[i]), NAMES[i]
    assert _max_err(grads[0], want[0]) <= _bar(want[0].float(), dtype, True)


def _port_op(value, shapes, ref, off, logits):
    return omsda.msda_torch_port(value, shapes, ref.to(value.dtype), off, logits)


def _param_grads(module, run):
    module.zero_grad()
    run().backward()
    return {n: p.grad.clone() for n, p in module.named_parameters()}


@pytest.mark.gpu
def test_sca_and_tsa_modules_train_through_the_op():
    """loss.backward() through the unfused SpatialCrossAttentionTRTP and TemporalSelfAttentionTRTP fills every parameter's
    gradient, and one SGD step moves the parameters where torch autograd through the reference algorithm moves them."""
    from bevformer_tensorrt_b200.modules import SpatialCrossAttentionTRTP, TemporalSelfAttentionTRTP
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
    sca = SpatialCrossAttentionTRTP(num_levels=1, num_points=8).cuda()
    # the default initialisation gives offsets of a fraction of a pixel: spread them so that taps differ
    with torch.no_grad():
        sca.deformable_attention.sampling_offsets.weight.mul_(20.0)
    tsa = TemporalSelfAttentionTRTP().cuda()
    with torch.no_grad():
        tsa.sampling_offsets.weight.mul_(20.0)
    q2 = torch.randn(1, 40 * 40, 256, generator=g).cuda()
    ref2d = torch.rand(2, 40 * 40, 1, 2, generator=g).cuda()
    shapes2 = torch.tensor([[40, 40]], device="cuda")
    w2 = torch.randn(1, 40 * 40, 256, generator=g).cuda()

    cases = [(sca, sca.deformable_attention, lambda: (sca.forward_trt(query, value, ref_cam, mask.cuda(), shapes) * weight).sum()),
             (tsa, tsa, lambda: (tsa.forward_trt(q2, ref2d, shapes2) * w2).sum())]  # fmt: skip
    for module, holder, run in cases:
        assert holder.multi_scale_deformable_attn is bt.multi_scale_deformable_attn
        ours = _param_grads(module, run)
        holder.multi_scale_deformable_attn = _port_op
        want = _param_grads(module, run)
        holder.multi_scale_deformable_attn = bt.multi_scale_deformable_attn
        assert ours.keys() == want.keys()
        for n in ours:
            scale = want[n].abs().max().item()
            assert scale > 0 and (ours[n] - want[n]).abs().max().item() <= 1e-4 * scale, n
        before = {n: p.detach().clone() for n, p in module.named_parameters()}
        opt = torch.optim.SGD(module.parameters(), lr=0.1)
        module.zero_grad()
        run().backward()
        opt.step()
        for n, p in module.named_parameters():
            assert not torch.equal(p.detach(), before[n]), n
