"""Every kernel-selection branch of the MSDA ops against the CPU oracle (pytest -m gpu).

The selection lives in csrc/msda.cu (``validate`` / ``dispatch`` / ``dispatch_rounds`` / ``msda_*_op``), in the declines
of csrc/msda_v2.cu (packed INT8) and csrc/msda_res.cu (FP16 resident tail), and in the Python fallbacks of the fused
spatial-cross-attention forms. tests/test_msda_gpu.py holds the main path to its bars (C = 32, G in {1, 2, 4}, at most
4 levels, freshly allocated tensors, at most 2 gather rounds); this file runs what lies around it: the ROUNDS = 4
template with a full and a partial last round, the generic kernel (more than 4 rounds, C != 32, G not in {1, 2, 4},
P % 4 != 0, unaligned pointers) in FP32, FP16 and INT8, 16 and 17 levels, the edges of the packed INT8 and resident-tail
envelopes, and the fused forms outside their envelope.

Which kernel ran is read from a CUPTI activity trace (``torch.profiler``, CUDA activity only: kernel names, no hardware
counters). If the trace records no kernels, only the kernel-identity assertions are skipped
(``test_kernel_trace_names_the_launched_kernel`` says so); the value checks run regardless.

Bars are those of tests/test_msda_gpu.py: FP32 1e-5, FP16 1e-3 exact / 1.6e-3 mixed, INT8 2e-2 after x scale_out and at
most 1 LSB on < 2 % of the elements against the oracle's requantisation.
"""
import ctypes
import dataclasses
import importlib
import re

import numpy as np
import pytest
import torch

import bevformer_tensorrt_b200 as bt
from bevformer_tensorrt_b200 import _lib
from bevformer_tensorrt_b200.functions.multi_scale_deformable_attn import (msda_trace, multi_scale_deformable_attn_out,
                                                                            set_msda_v2)  # fmt: skip
from bevformer_tensorrt_b200.workloads import MSDAConfig, make_msda_inputs, quantize_per_tensor
from oracle import msda as omsda

# the module itself (the package re-exports a function of the same name)
msda_mod = importlib.import_module("bevformer_tensorrt_b200.functions.multi_scale_deformable_attn")

pytestmark = pytest.mark.gpu

FP32_TOL = 1e-5
FP16_TOL = 1e-3
FP16_MIXED_TOL = 1.6e-3
INT8_TOL = 2e-2

LEVELS4 = ((10, 12), (5, 6), (3, 3), (2, 2))
LEVELS8 = ((9, 10), (7, 8), (5, 6), (4, 5), (3, 4), (2, 3), (2, 2), (1, 1))
LEVELS16 = ((9, 11), (8, 3), (7, 1), (1, 7), (1, 1), (6, 6), (5, 4), (4, 5), (3, 3), (2, 6), (6, 2), (2, 2), (3, 1), (1, 3),
            (2, 1), (1, 2))  # fmt: skip
LEVELS3 = ((11, 13), (6, 7), (3, 4))

# name: (B, Q, M, C, levels, P, G[, bev_hw])
CASES = {
    "base": MSDAConfig("base", 2, 45, 8, 32, ((12, 20), (6, 10), (3, 5), (2, 3)), 8, 4),  # NP 32: the BEVFormer SCA shape
    "r3": MSDAConfig("r3", 1, 53, 8, 32, LEVELS3, 12, 2),  # NP 36
    "r3g": MSDAConfig("r3g", 6, 56, 8, 32, LEVELS3, 12, 4, (7, 8)),  # NP 36 on camera-ring reference points
    "r4_f32": MSDAConfig("r4_f32", 1, 40, 8, 32, LEVELS4, 20, 4),  # NP 80
    "np128": MSDAConfig("np128", 1, 24, 8, 32, LEVELS8, 16, 4),
    "np132": MSDAConfig("np132", 1, 24, 4, 32, LEVELS3, 44, 4),
    "l16": MSDAConfig("l16", 1, 30, 4, 32, LEVELS16, 4, 4),  # NP 64, one lane per level in the level table
    "g8": MSDAConfig("g8", 2, 30, 4, 32, ((8, 9), (4, 5)), 8, 8),
    "c64": MSDAConfig("c64", 2, 20, 4, 64, ((7, 9), (4, 5)), 8, 4),
    "c16": MSDAConfig("c16", 1, 25, 4, 16, ((7, 9), (4, 5)), 4, 2),
    "c8": MSDAConfig("c8", 1, 25, 8, 8, ((6, 7), (3, 4)), 8, 1),
    "c5": MSDAConfig("c5", 1, 25, 3, 5, ((6, 7), (3, 4)), 4, 2),
    "p2": MSDAConfig("p2", 1, 30, 4, 32, ((8, 9), (4, 5)), 2, 2),
    "v2_np12": MSDAConfig("v2_np12", 1, 40, 8, 32, ((9, 10), (5, 6), (3, 3)), 4, 4),
    "v2_np16": MSDAConfig("v2_np16", 1, 40, 8, 32, LEVELS4, 4, 4),
    "v2_l8": MSDAConfig("v2_l8", 1, 30, 8, 32, LEVELS8, 4, 4),  # NP 32 at the packed kernel's 8-level limit
}
SEED = {name: 3000 + 10 * i for i, name in enumerate(CASES)}

# The kernel each op runs, derived from the selection code. gatherR = msda_gather_kernel<..., ROUNDS = R, ...>;
# fused = msda_gather_kernel with the camera-sum epilogue (EPI 1 / 2); fallback = plugin op + masked sum in Python;
# v2 = msda_pack_kernel + msda_i8p_kernel; status1 = refused (B200OpsError), nothing launched.
#   FP32 (8 lanes per item): gather iff C = 32, P % 4 = 0, G in {1, 2, 4}, aligned, NP <= 32 / 64 / 128 (R = 1 / 2 / 4)
#   FP16 (4 lanes per item): the same with NP <= 16 / 32 / 64
#   INT8: C % 4 or P % 4 != 0 -> status1; v2 iff C = 32, L <= 8, P % 4 = 0, 16 <= NP <= 32, G in {1, 2, 4}, aligned;
#         else the FP16 rules
#   fused forms: gather at <= 2 rounds (FP32 NP <= 64, FP16 NP <= 32) plus the C / G / P / alignment rules
PATHS = {  # name: (fp32, fp16, int8, fused fp32, fused fp16)
    "base": ("gather1", "gather2", "v2", "fused", "fused"),
    "r3": ("gather2", "gather4", "gather4", "fused", "fallback"),
    "r3g": ("gather2", "gather4", "gather4", "fused", "fallback"),
    "r4_f32": ("gather4", "generic", "generic", "fallback", "fallback"),
    "np128": ("gather4", "generic", "generic", "fallback", "fallback"),
    "np132": ("generic", "generic", "generic", "fallback", "fallback"),
    "l16": ("gather2", "gather4", "gather4", "fused", "fallback"),
    "g8": ("generic", "generic", "generic", "fallback", "fallback"),
    "c64": ("generic", "generic", "generic", "fallback", "fallback"),
    "c16": ("generic", "generic", "generic", "fallback", "fallback"),
    "c8": ("generic", "generic", "generic", "fallback", "fallback"),
    "c5": ("generic", "generic", "status1", "fallback", "fallback"),
    "p2": ("generic", "generic", "status1", "fallback", "fallback"),
    "v2_np12": ("gather1", "gather1", "gather1", "fused", "fused"),
    "v2_np16": ("gather1", "gather1", "v2", "fused", "fused"),
    "v2_l8": ("gather1", "gather2", "v2", "fused", "fused"),
}
assert PATHS.keys() == CASES.keys()


def _dists(name):
    return ["G"] if CASES[name].bev_hw != (0, 0) else ["edge", "U"]


CASE_DISTS = [(n, d) for n in CASES for d in _dists(n)]


# ---------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------
_FAMILIES = ("msda_gather_kernel", "msda_generic_kernel", "msda_res_kernel", "msda_pack_kernel", "msda_i8p_kernel")
_GATHER_ARGS = re.compile(r"msda_gather_kernel<\s*[\w: ]+,\s*[\w: ]+,\s*(\d+),\s*(\d+),\s*(\d+),\s*(\d+)")


def kernels_run(fn):
    """Runs ``fn()`` under a CUPTI activity trace; returns (its result, names of the MSDA kernels it launched)."""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        result = fn()
        torch.cuda.synchronize()
    try:
        names = [e.name() for e in prof.profiler.kineto_results.events()]
    except (AttributeError, RuntimeError):
        names = []
    if not names:
        names = [e.name for e in prof.events()]
    return result, [n for n in names if any(f in n for f in _FAMILIES)]


def path_of(names):
    """The selection-table label of a list of launched MSDA kernel names (see PATHS)."""
    if not names:
        return None
    if len(names) == 2 and any("msda_pack_kernel" in n for n in names) and any("msda_i8p_kernel" in n for n in names):
        return "v2"
    if len(names) != 1:
        return tuple(names)
    n = names[0]
    if "msda_generic_kernel" in n:
        return "generic"
    if "msda_res_kernel" in n:
        return "res"
    if "msda_gather_kernel" in n:
        m = _GATHER_ARGS.search(n)
        if m is None:  # template arguments not in the recorded name: the family is all that can be told
            return "gather?"
        rounds, epi = int(m.group(2)), int(m.group(4))
        return "fused" if epi != 0 else f"gather{rounds}"
    return tuple(names)


def run_expecting(path, fn):
    """``fn()``, asserting that it launched the kernel(s) of ``path``. An empty trace leaves the identity unchecked."""
    result, names = kernels_run(fn)
    got = path_of(names)
    if got is not None:
        if got == "gather?":
            assert path.startswith("gather") or path == "fused", (path, names)
        else:
            assert got == path, (path, names)
    return result


def misaligned(t):
    """The same values in a contiguous device view whose data pointer is NOT 16-byte aligned (one element in)."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device="cuda")
    view = buf[1:].view(t.shape)
    view.copy_(t)
    assert view.is_contiguous() and view.data_ptr() % 16 != 0
    return view


def _cuda(ts):
    return [t.cuda() for t in ts]


def _oracle_f32(inputs):
    return omsda.msda_f32(*(t.float().numpy() for t in inputs))


def _want_records(shapes, ref, off, cfg):
    """The oracle's sampling-index records {in_range, h_low, w_low, tap_mask} as int32 [B, Q, M, L*P, 4]."""
    B, Q, M, C = cfg.batch, cfg.num_query, cfg.num_heads, cfg.channels
    NP = cfg.num_levels * cfg.num_points
    dummy_v = np.zeros((B, cfg.spatial_size, M, C), np.float32)
    dummy_w = np.zeros((B, Q, M, NP), np.float32)
    _, idx = omsda.msda_f32(dummy_v, shapes.numpy(), ref, off, dummy_w, return_index=True)
    return np.stack([idx["in_range"], idx["h_low"], idx["w_low"], idx["tap_mask"]], -1)


def _quantised(cfg, dist, seed, ref_dtype):
    value, shapes, ref, off, logits = make_msda_inputs(cfg, dist, seed, torch.float32)
    vq, sv = quantize_per_tensor(value)
    oq, so = quantize_per_tensor(off)
    wq, sw = quantize_per_tensor(logits)
    ref = ref.to(ref_dtype)
    real = omsda.msda_f32(vq.float().numpy() * sv, shapes.numpy(), ref.float().numpy(), oq.float().numpy() * so,
                          wq.float().numpy() * sw)  # fmt: skip
    sout = float(np.abs(real).max()) / 127.0
    return (vq, sv, shapes, ref, oq, so, wq, sw, sout), real


def _int8_args(q):
    vq, sv, shapes, ref, oq, so, wq, sw, sout = q
    return (vq.cuda(), sv, shapes.cuda(), ref.cuda(), oq.cuda(), so, wq.cuda(), sw, sout)


def _check_int8(got, q, real):
    vq, sv, shapes, ref, oq, so, wq, sw, sout = q
    got = got.cpu().numpy()
    assert np.abs(got.astype(np.float32) * sout - real).max() < INT8_TOL
    want_q = omsda.msda_i8_dequant(vq.numpy(), sv, shapes.numpy(), ref.float().numpy(), oq.numpy(), so, wq.numpy(), sw,
                                   sout)  # fmt: skip
    diff = np.abs(got.astype(np.int32) - want_q.astype(np.int32))
    assert diff.max() <= 1 and (diff != 0).mean() < 0.02, (diff.max(), (diff != 0).mean())
    assert np.abs(got).max() >= 100  # the output scale is used: a lost factor cannot hide in the rounding


@pytest.fixture(autouse=True)
def default_switches():
    """Every test starts from the library defaults and leaves every process-wide switch as it found it."""
    lib = _lib.load()
    units, variant = bt.get_msda_batch_units(), bt.get_msda_gather_variant()
    path, mode, v2 = bt.set_msda_f16_path(False)[0], lib.b200_msda_set_f16_mode(0), set_msda_v2(True)
    bt.set_msda_batch_units(1)
    bt.set_msda_gather_variant(0)
    yield
    bt.set_msda_batch_units(*units)
    bt.set_msda_gather_variant(variant)
    bt.set_msda_f16_path(path)
    lib.b200_msda_set_f16_mode(mode)
    set_msda_v2(v2)


def test_kernel_trace_names_the_launched_kernel():
    """The CUPTI trace behind every kernel-identity assertion in this file records the kernels the op launched."""
    inputs = _cuda(make_msda_inputs(CASES["base"], "U", 1, torch.float32))
    _, names = kernels_run(lambda: bt.multi_scale_deformable_attn(*inputs))
    if not names:
        pytest.skip("the profiler trace recorded no kernels here: kernel-identity assertions are skipped, values are "
                    "still checked")  # fmt: skip
    assert len(names) == 1 and "msda_gather_kernel" in names[0], names
    assert path_of(names) == "gather1", names  # the template arguments are readable from the recorded name


# ---------------------------------------------------------------------------------------------------------------
# plugin ops: expected kernel, values, index records of the kernel that ran
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,dist", CASE_DISTS)
def test_fp32_selection_and_values(name, dist):
    cfg = CASES[name]
    inputs = make_msda_inputs(cfg, dist, SEED[name], torch.float32)
    want = _oracle_f32(inputs)
    dev = _cuda(inputs)
    for fn in (bt.multi_scale_deformable_attn, bt.multi_scale_deformable_attn2):
        got = run_expecting(PATHS[name][0], lambda: fn(*dev))
        err = np.abs(got.cpu().numpy() - want).max()
        assert err < FP32_TOL, (name, dist, err)
    out_t, rec = run_expecting(PATHS[name][0], lambda: msda_trace(*dev))
    assert torch.equal(out_t, got)
    wrec = _want_records(inputs[1], inputs[2].numpy(), inputs[3].numpy(), cfg)
    assert (rec.cpu().numpy() == wrec).all(), f"{(rec.cpu().numpy() != wrec).any(-1).sum()} records differ"


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("name,dist", CASE_DISTS)
def test_fp16_selection_and_values(name, dist, mode):
    cfg = CASES[name]
    inputs = make_msda_inputs(cfg, dist, SEED[name] + 1, torch.float16)
    want = _oracle_f32(inputs)  # fp32 formulas on the fp16-rounded inputs
    dev = _cuda(inputs)
    _lib.load().b200_msda_set_f16_mode(mode)
    for fn in (bt.multi_scale_deformable_attn, bt.multi_scale_deformable_attn2):  # …2 takes b200_msda_f16 for odd C
        got = run_expecting(PATHS[name][1], lambda: fn(*dev))
        assert got.dtype == torch.float16
        err = np.abs(got.float().cpu().numpy() - want).max()
        assert err < (FP16_TOL if mode == 0 else FP16_MIXED_TOL), (name, dist, mode, err)
    if mode == 0:  # a traced FP16 launch is exact
        out_t, rec = run_expecting(PATHS[name][1], lambda: msda_trace(*dev))
        assert torch.equal(out_t, got)
        wrec = _want_records(inputs[1], inputs[2].float().numpy(), inputs[3].float().numpy(), cfg)
        assert (rec.cpu().numpy() == wrec).all(), f"{(rec.cpu().numpy() != wrec).any(-1).sum()} records differ"


@pytest.mark.parametrize("name,dist", CASE_DISTS)
def test_int8_selection_and_values(name, dist):
    cfg = CASES[name]
    ref_dtype = torch.float16 if dist == "edge" else torch.float32
    q, real = _quantised(cfg, dist, SEED[name] + 2, ref_dtype)
    args = _int8_args(q)
    path = PATHS[name][2]
    if path == "status1":  # C % 4 or P % 4 != 0: refused before anything is launched
        n0 = _lib.launch_count()
        with pytest.raises(_lib.B200OpsError) as e:
            bt.multi_scale_deformable_attn_int8(*args)
        assert e.value.status == 1 and _lib.launch_count() == n0
        return
    n0 = _lib.launch_count()
    got = run_expecting(path, lambda: bt.multi_scale_deformable_attn_int8(*args))
    assert _lib.launch_count() - n0 == (2 if path == "v2" else 1)
    assert got.dtype == torch.int8
    _check_int8(got, q, real)
    vq, sv, shapes, ref, oq, so, wq, sw, sout = q
    out_t, rec = run_expecting(path, lambda: msda_trace(args[0], args[2], args[3], args[4], args[6],
                                                        scales=(sv, so, sw, sout)))  # fmt: skip
    assert torch.equal(out_t, got)
    off_real = oq.numpy().astype(np.float32) * np.float32(so)
    assert (rec.cpu().numpy() == _want_records(shapes, ref.float().numpy(), off_real, cfg)).all()


@pytest.mark.parametrize("channels", [32, 20])
def test_seventeen_levels_refused_by_every_entry(channels):
    """kMaxLevels = 16 (one lane per level in the level table): L = 17 is status 1 from every entry — the gather and
    the generic kernels (C = 20) alike, the fused forms through their fallback — and nothing is launched."""
    cfg = MSDAConfig("l17", 2, 12, 2, channels, tuple((1 + i % 3, 2 + i % 2) for i in range(17)), 4, 2)
    inputs = make_msda_inputs(cfg, "U", 17, torch.float32)
    d32 = _cuda(inputs)
    d16 = [t.half() if t.is_floating_point() else t for t in d32]
    q, _ = _quantised(cfg, "U", 18, torch.float16)
    i8 = _int8_args(q)
    mask = torch.ones(cfg.batch, cfg.num_query, device="cuda")
    out = torch.empty(cfg.batch, cfg.num_query, cfg.num_heads, channels, device="cuda")
    calls = [
        lambda: bt.multi_scale_deformable_attn(*d32),
        lambda: bt.multi_scale_deformable_attn(*d16),
        lambda: bt.multi_scale_deformable_attn2(*d16),
        lambda: multi_scale_deformable_attn_out(*d32, out),
        lambda: msda_trace(*d32),
        lambda: msda_trace(*d16),
        lambda: bt.multi_scale_deformable_attn_int8(*i8),
        lambda: msda_trace(i8[0], i8[2], i8[3], i8[4], i8[6], scales=(i8[1], i8[5], i8[7], i8[8])),
        lambda: bt.multi_scale_deformable_attn_sca(*d32, mask),
        lambda: bt.multi_scale_deformable_attn_sca(*d16, mask),
        lambda: bt.multi_scale_deformable_attn_sca_shared(*d32[:3], d32[3][:1], d32[4][:1], mask),
        lambda: bt.multi_scale_deformable_attn_queue_mean(*d16),
    ]
    n0 = _lib.launch_count()
    for i, call in enumerate(calls):
        with pytest.raises(_lib.B200OpsError) as e:
            call()
        assert e.value.status == 1, i
    assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------------------------
# unaligned tensors: the plugin op takes the generic kernel (the packed INT8 and resident-tail kernels decline first)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["value", "offsets", "logits", "reference_points", "out"])
@pytest.mark.parametrize("name", ["base", "l16"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_misaligned_float_runs_generic_kernel(dtype, name, which):
    """One tensor at a time one element off 16-byte alignment: the generic kernel runs and agrees with the oracle and
    with the aligned run (the gather kernel) on the same data — two independent kernels."""
    cfg = CASES[name]
    inputs = make_msda_inputs(cfg, "edge", SEED[name] + 3, dtype)
    want = _oracle_f32(inputs)
    dev = _cuda(inputs)
    tol = FP32_TOL if dtype == torch.float32 else FP16_TOL
    aligned = run_expecting(PATHS[name][0 if dtype == torch.float32 else 1],
                            lambda: bt.multi_scale_deformable_attn(*dev))  # fmt: skip
    args = list(dev)
    out = None
    if which == "out":
        out = misaligned(torch.zeros(cfg.batch, cfg.num_query, cfg.num_heads, cfg.channels, dtype=dtype, device="cuda"))
    else:
        i = {"value": 0, "reference_points": 2, "offsets": 3, "logits": 4}[which]
        args[i] = misaligned(args[i])
    if out is None:
        got = run_expecting("generic", lambda: bt.multi_scale_deformable_attn(*args))
    else:
        got = run_expecting("generic", lambda: multi_scale_deformable_attn_out(*args, out))
        assert got.data_ptr() == out.data_ptr()
    assert np.abs(got.float().cpu().numpy() - want).max() < tol
    assert (got.float() - aligned.float()).abs().max().item() < tol
    if which != "out":
        out_t, rec = run_expecting("generic", lambda: msda_trace(*args))
        assert torch.equal(out_t, got)
        wrec = _want_records(inputs[1], inputs[2].float().numpy(), inputs[3].float().numpy(), cfg)
        assert (rec.cpu().numpy() == wrec).all()


@pytest.mark.parametrize("which", ["value", "offsets", "logits", "reference_points"])
@pytest.mark.parametrize("name", ["base", "l16"])
def test_misaligned_int8_runs_generic_kernel(name, which):
    """INT8: the packed kernel (base) and the round-1 gather kernel (l16) both decline an unaligned tensor; the generic
    kernel's requantisation meets the INT8 bars and lies within 1 LSB of the aligned run on a few elements."""
    cfg = CASES[name]
    q, real = _quantised(cfg, "edge", SEED[name] + 4, torch.float32)
    args = list(_int8_args(q))
    aligned = run_expecting(PATHS[name][2], lambda: bt.multi_scale_deformable_attn_int8(*args))
    i = {"value": 0, "reference_points": 3, "offsets": 4, "logits": 6}[which]
    args[i] = misaligned(args[i])
    got = run_expecting("generic", lambda: bt.multi_scale_deformable_attn_int8(*args))
    _check_int8(got, q, real)
    d = (got.int() - aligned.int()).abs()
    assert d.max().item() <= 1 and (d != 0).float().mean().item() < 0.03


# ---------------------------------------------------------------------------------------------------------------
# launch-shape and resident-tail switches where they do not apply
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,dtype", [("r4_f32", torch.float32), ("np128", torch.float32), ("np132", torch.float32),
                                        ("g8", torch.float32), ("r3", torch.float16), ("l16", torch.float16),
                                        ("c64", torch.float16), ("c5", torch.float16)])  # fmt: skip
def test_switches_leave_other_kernels_bit_identical(name, dtype):
    """The batched launch and the gather-depth variants exist for <= 2 rounds only, the resident-tail kernel for
    NP <= 32 and C = 32: on the ROUNDS = 4 template and the generic kernel every setting gives the default's bytes and
    leaves the kernel choice alone."""
    cfg = CASES[name]
    dev = _cuda(make_msda_inputs(cfg, "edge", SEED[name] + 5, dtype))
    path = PATHS[name][0 if dtype == torch.float32 else 1]
    assert path in ("gather4", "generic")
    base = bt.multi_scale_deformable_attn(*dev)
    for shape in bt.MSDA_LAUNCH_SHAPES:
        bt.set_msda_launch_shape(shape)
        got = run_expecting(path, lambda: bt.multi_scale_deformable_attn(*dev))
        assert torch.equal(got, base), shape
    bt.set_msda_launch_shape("default")
    if dtype == torch.float16:
        bt.set_msda_f16_path(True)
        got = run_expecting(path, lambda: bt.multi_scale_deformable_attn(*dev))
        assert torch.equal(got, base)


@pytest.mark.parametrize("name,misalign,path", [("base", False, "res"), ("v2_l8", False, "res"), ("r3", False, "gather4"),
                                                ("l16", False, "gather4"), ("base", True, "generic")])  # fmt: skip
def test_resident_tail_envelope(name, misalign, path):
    """With the resident-tail kernel selected: it runs up to NP = 32 (4 and 8 levels), the gather kernel beyond, the
    generic kernel on an unaligned value tensor. Values against the oracle, records traced out of the kernel that ran."""
    cfg = CASES[name]
    inputs = make_msda_inputs(cfg, "edge", SEED[name] + 6, torch.float16)
    want = _oracle_f32(inputs)
    dev = _cuda(inputs)
    if misalign:
        dev[0] = misaligned(dev[0])
    bt.set_msda_f16_path(True)
    got = run_expecting(path, lambda: bt.multi_scale_deformable_attn(*dev))
    assert np.abs(got.float().cpu().numpy() - want).max() < FP16_TOL
    out_t, rec = run_expecting(path, lambda: msda_trace(*dev))
    assert torch.equal(out_t, got)
    wrec = _want_records(inputs[1], inputs[2].float().numpy(), inputs[3].float().numpy(), cfg)
    assert (rec.cpu().numpy() == wrec).all()


# ---------------------------------------------------------------------------------------------------------------
# INT8 through the plugin enqueue outside the packed kernel's envelope
# ---------------------------------------------------------------------------------------------------------------
def _desc(t, ttype, scale=1.0):
    d = _lib.TensorDesc()
    d.dims.nbDims = t.dim()
    for i, s in enumerate(t.shape):
        d.dims.d[i] = s
    d.type, d.format, d.scale = ttype, 0, scale
    return d


@pytest.mark.parametrize("name", ["r3", "c16", "g8"])
def test_int8_enqueue_outside_packed_envelope(name):
    """getWorkspaceSize asks for 0 bytes outside the packed kernel's envelope, and enqueue — with no workspace or with
    one lent anyway — writes the Python op's bytes."""
    cfg = CASES[name]
    q, real = _quantised(cfg, "edge", SEED[name] + 7, torch.float16)
    vq, sv, shapes, ref, oq, so, wq, sw, sout = q
    qt = [vq.cuda(), shapes.cuda(), ref.cuda(), oq.cuda(), wq.cuda()]
    want = bt.multi_scale_deformable_attn_int8(qt[0], sv, qt[1], qt[2], qt[3], so, qt[4], sw, sout)
    _check_int8(want, q, real)
    lib = _lib.load()
    d8 = (_lib.TensorDesc * 5)(_desc(qt[0], 2, sv), _desc(qt[1], 3), _desc(qt[2], 1), _desc(qt[3], 2, so),
                               _desc(qt[4], 2, sw))  # fmt: skip
    assert lib.b200_msda_enqueue_workspace_size(d8) == 0
    spare = torch.empty(4096, dtype=torch.uint8, device="cuda")
    for ws in (None, spare.data_ptr()):
        out = torch.full_like(want, 77)
        o8 = (_lib.TensorDesc * 1)(_desc(out, 2, sout))
        p8 = (ctypes.c_void_p * 5)(*[t.data_ptr() for t in qt])
        q8 = (ctypes.c_void_p * 1)(out.data_ptr())
        assert lib.b200_msda_enqueue(d8, o8, p8, q8, ws, _lib.current_stream_ptr(), 0) == 0
        torch.cuda.synchronize()
        assert torch.equal(out, want), ws


# ---------------------------------------------------------------------------------------------------------------
# fused spatial-cross-attention forms: fused kernel inside the envelope, plugin op + masked sum outside
# ---------------------------------------------------------------------------------------------------------------
def _fused_inputs(name, dtype, seed, cams=3):
    """Plugin-signature inputs with ``cams`` cameras whose offsets / logits are identical copies (what
    SpatialCrossAttention feeds the plugin), the single copy, and a bev_mask normalised over the cameras that see a query
    (0 for the first 5 queries: nobody sees them)."""
    cfg = dataclasses.replace(CASES[name], batch=cams)
    value, shapes, ref, off, logits = make_msda_inputs(cfg, "edge", seed, dtype)
    off1, lg1 = off[:1].contiguous(), logits[:1].contiguous()
    rep = (value, shapes, ref, off1.expand_as(off).contiguous(), lg1.expand_as(logits).contiguous())
    seen = (torch.rand(cams, cfg.num_query, 1, generator=torch.Generator().manual_seed(seed)) > 0.4).float()
    seen[:, :5] = 0
    mask = seen / seen.sum(0, keepdim=True).clamp(min=1.0)
    return cfg, rep, (off1, lg1), mask


class _Spy:
    """Counts the calls of the module's plugin-op entry (the fused forms' fallback) and passes them through."""

    def __init__(self, monkeypatch):
        self.calls = 0
        real = msda_mod._msda_forward

        def spy(*a, **k):
            self.calls += 1
            return real(*a, **k)

        monkeypatch.setattr(msda_mod, "_msda_forward", spy)


FUSED_CASES = [  # (name, dtype, misaligned tensor)
    ("r3", torch.float16, None),
    ("r3", torch.float32, None),
    ("r4_f32", torch.float32, None),
    ("l16", torch.float16, None),
    ("c64", torch.float32, None),
    ("c64", torch.float16, None),
    ("g8", torch.float32, None),
    ("g8", torch.float16, None),
    ("p2", torch.float16, None),
    ("base", torch.float32, "offsets"),
    ("base", torch.float16, "offsets"),
    ("base", torch.float32, "accum"),
    ("base", torch.float32, None),
    ("base", torch.float16, None),
    ("l16", torch.float32, None),
    ("v2_np12", torch.float16, None),
]


@pytest.mark.parametrize("name,dtype,mis", FUSED_CASES)
def test_fused_forms_against_oracle(name, dtype, mis, monkeypatch):
    """``…_sca`` (+= into a caller's accumulator), ``…_sca_shared`` (offsets / logits once, with or without the leading
    1) and ``…_queue_mean`` against the masked camera sum / queue mean of the oracle. Inside the envelope each is one
    fused launch and the Python fallback never runs; outside it each takes the fallback exactly once."""
    cfg, rep, (off1, lg1), mask = _fused_inputs(name, dtype, SEED[name] + 8)
    in_envelope = PATHS[name][3 if dtype == torch.float32 else 4] == "fused"
    fused = in_envelope and mis != "offsets"  # an unaligned accumulator only concerns the call that is given it
    tol = 2e-5 if dtype == torch.float32 else FP16_TOL
    B, Q = cfg.batch, cfg.num_query
    per_cam = torch.from_numpy(_oracle_f32(rep)).reshape(B, Q, -1)
    want = (per_cam * mask).sum(0)
    dev, dmask = _cuda(rep), mask.cuda()
    off1, lg1 = off1.cuda(), lg1.cuda()
    if mis == "offsets":
        dev[3], off1 = misaligned(dev[3]), misaligned(off1)
    spy = _Spy(monkeypatch)

    def expect(fn, one_kernel=fused):
        n0, c0 = _lib.launch_count(), spy.calls
        out, names = kernels_run(fn)
        assert spy.calls - c0 == (0 if one_kernel else 1)
        if one_kernel:
            assert _lib.launch_count() - n0 == 1
            assert path_of(names) in (None, "fused", "gather?"), names
        else:
            assert not any(path_of([n]) == "fused" for n in names), names
        return out

    # per-camera fused form, += semantics
    acc0 = torch.full((Q, cfg.num_heads * cfg.channels), 0.5, device="cuda")
    acc = misaligned(acc0) if mis == "accum" else acc0.clone()
    got = expect(lambda: bt.multi_scale_deformable_attn_sca(*dev, dmask, acc), fused and mis is None)
    assert got.data_ptr() == acc.data_ptr() and got.dtype == torch.float32
    assert (got.cpu() - 0.5 - want).abs().max().item() < tol
    fresh = expect(lambda: bt.multi_scale_deformable_attn_sca(*dev, dmask))
    assert (fresh.cpu() - want).abs().max().item() < tol
    assert (got - 0.5 - fresh).abs().max().item() < 1e-6
    # camera-shared form
    shared = expect(lambda: bt.multi_scale_deformable_attn_sca_shared(*dev[:3], off1, lg1, dmask))
    assert shared.dtype == torch.float32 and shared.shape == want.shape
    assert (shared.cpu() - want).abs().max().item() < tol
    unseen = mask.sum(0)[:, 0] == 0
    assert unseen.any() and torch.equal(shared.cpu()[unseen], torch.zeros_like(shared.cpu()[unseen]))
    if not in_envelope:  # both forms run the same plugin op on the same tensors
        assert torch.equal(shared, fresh)
    elif fused:  # two fused kernels, fp32 camera sums in either
        assert (shared - fresh).abs().max().item() < (2e-6 if dtype == torch.float32 else 2e-4)
    else:  # an unaligned copy of the offsets: the generic kernel behind one form, the gather kernel behind the other
        assert (shared - fresh).abs().max().item() < tol
    shared2 = bt.multi_scale_deformable_attn_sca_shared(*dev[:3], off1[0], lg1[0], dmask)
    assert torch.equal(shared2, shared)
    # BEV-queue mean (TemporalSelfAttention)
    qm = expect(lambda: bt.multi_scale_deformable_attn_queue_mean(*dev))
    assert qm.shape == (1, Q, cfg.num_heads * cfg.channels) and qm.dtype == dtype
    want_mean = per_cam.mean(0, keepdim=True)
    assert (qm.float().cpu() - want_mean).abs().max().item() < (1e-5 if dtype == torch.float32 else FP16_TOL)
