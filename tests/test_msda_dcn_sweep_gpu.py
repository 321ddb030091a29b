"""MSDA and DCNv2, forward and backward, over seeded random geometries in FP32, FP16 and BF16, checked element by element
against the float64 references of oracle/f64.py.

Every element e of every output and gradient must satisfy

    |got_e - r_e| <= 1/2 ulp_dtype(|r_e| + E_e) + E_e,
    E_e = (8 + n_e) * u_acc * mag_e + 2^-24 * pmag_e + u_low * lmag_e + s_low * lcnt_e

with r_e the float64 value, mag_e the sum of |terms| behind it, n_e the length of its longest chain of sums (softmax
included), pmag_e the MSDA position term, and lmag_e / lcnt_e the values a path rounds to FP16 / BF16 on the way, times
the fixed number of roundings each goes through (oracle/f64.py defines them all). The constants, once for every case
and dtype:

* 1/2 ulp of the output dtype: the one rounding of the result to its storage type, taken at |r_e| + E_e because the
  value rounded is the computed one, which may sit in the next binade up.
* (8 + n_e) * u_acc * mag_e: a float sum of n terms is within (n - 1) u sum|terms| of the exact sum in any order,
  atomics included, and a sum of sums within (n_inner + n_outer) u; the 8 covers the few products and conversions
  around the sums. u_acc = 2^-24 for the fp32 sums of every kernel (csrc/msda.cu:157, 204, 215-216, 771-798, 885-889;
  csrc/msda_backward.cu:26, 458-464; csrc/dcn_generic.cu:19, 144; the DCN backward), and 2^-23 for the wgmma
  accumulation of the fused DCN kernel, since tensor-core fp32 accumulation is not specified to round to nearest.
* u_low * lmag_e + s_low * lcnt_e: an FP16 / BF16 rounding of v errs by at most u_low |v| (2^-11 / 2^-8), or by
  s_low (half the smallest subnormal: 2^-25 / 2^-134) in the subnormal range. Paths and their counts:
    - the fused DCN kernel's FP16 columns: four weights and four blend operations, five roundings
      (csrc/dcn_fused.cu:337-354), counted as 6;
    - the MSDA fused forms' fallback (functions/multi_scale_deformable_attn.py:462-471, 503-507): each camera's output
      once; each grad_out element once; for the shared form each camera's offset and logit gradient once more;
    - every other path: none (u_low = s_low = 0). The FP16 h2 entry is the FP16 op (csrc/msda.cu:1121-1128).
* 2^-24 * pmag_e: MSDA forms x = ref * W + off - 0.5 in fp32; pmag_e carries the factor 3 of its three roundings.
  DCN's reference uses the fp32 position sums themselves, so its pmag is 0.

Every tensor also keeps the per-tensor bar the rest of the suite uses: FP32 1e-4 max|r|; FP16 / BF16 half a spacing at
max|r| plus 1e-4 max|r|; on the fallback forms that bar plus the largest intermediate rounding u_low max(lmag); on the
fused DCN FP16 output tests.helpers.fp16_tol, whose 1e-3 is taken at the mask's scale, max(1, max|mask|): the FP16
blend's error grows with |mask|, and with masks up to 1.5 the unscaled bar is exceeded by a correct kernel (seed 490:
2.2e-3 against 2.0e-3).

The kernel trace now and then loses a record (tests/helpers.kernels_recorded); a call whose trace holds no kernel of
the op at all leaves the identity unchecked (its values are still checked), as in tests/test_msda_envelope_gpu.py.

The geometries are drawn by numpy.random.default_rng(seed) over the envelope of the C entries (levels, heads, channels,
points, groups, level shapes down to 1 x 1, offsets in range, out of range and on integer and border positions, zero
bev_mask entries, unaligned views; DCN groups and deformable groups 1-4, kernels up to 75 taps, per-axis stride, padding
and dilation, fused-eligible layers with H or W of 1). A Python restatement of each kernel-selection rule predicts the
kernel each case runs; the CPU tests check that the seed list reaches every branch, and the GPU tests that the predicted
kernel ran. B200_SWEEP_SEEDS=<k> adds k seeds beyond the default list (a longer soak over new geometries).
"""
import math
import os
import re

import numpy as np
import pytest
import torch

import bevformer_tensorrt_b200 as bt
from oracle import dcn as odcn
from oracle import msda as omsda
from oracle.f64 import dcn_f64, msda_f64, msda_sca_f64
from tests.helpers import U32, check, kernels_recorded, ulp
from tests.test_dcn_backward_edges_gpu import _plan, _ragged, _ws_query

U_WGMMA = 2.0**-23
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
DT_IDS = ["fp32", "fp16", "bf16"]

# chosen so that together they reach every selection branch and every edge the CPU coverage tests list
MSDA_SEEDS = [1, 2, 5, 10, 11, 17, 18, 19, 25, 33, 47, 65, 113, 127, 152, 227, 371, 486]
DCN_SEEDS = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 13, 26, 66, 490, 651, 940]
_EXTRA = int(os.environ.get("B200_SWEEP_SEEDS", "0") or 0)
MSDA_SEEDS += [100_000 + i for i in range(_EXTRA)]
DCN_SEEDS += [100_000 + i for i in range(_EXTRA)]


# ---- MSDA geometries ---------------------------------------------------------------------------------------------------
_C_CHOICES = [32] * 6 + [1, 5, 16, 40, 64]
_G_CHOICES = [1, 1, 2, 2, 4, 4, 3, 8]
_MSDA_WORK = 600_000  # B * Q * M * L*P * C cap: Q shrinks to fit


def msda_geometry(seed):
    """One drawn MSDA call: a dict of B, Q, M, C, shapes ((H, W) per level), P, G, the offset distribution and whether
    value is passed as a view one element off alignment."""
    rng = np.random.default_rng([0x5EED, seed])
    B = int(rng.integers(1, 7))
    M = int(rng.integers(1, 10))
    L = 1 + int(15 * rng.random() ** 2)
    shapes = []
    for _ in range(L):
        kind = rng.random()
        h, w = (int(v) for v in rng.integers(1, 25, 2))
        if kind < 0.15:
            h = 1
        elif kind < 0.3:
            w = 1
        shapes.append((h, w))
    C = int(rng.choice(_C_CHOICES))
    P = int(rng.choice([4, 8, 12, 16, 20])) if rng.random() < 0.6 else int(rng.integers(1, 21))
    G = int(rng.choice(_G_CHOICES))
    Q = int(rng.integers(1, 301))
    Q = max(1, min(Q, _MSDA_WORK // (B * M * L * P * C)))
    dist = str(rng.choice(["normal", "out", "dyadic"]))
    misaligned = bool(rng.random() < 0.15)
    return dict(B=B, Q=Q, M=M, C=C, shapes=tuple(shapes), P=P, G=G, dist=dist, misaligned=misaligned)


def msda_inputs(geo, seed):
    """float32 CPU tensors value, shapes (int64), ref, off, logits, bev_mask [B, Q], grad_out [B,Q,M,C]."""
    rng = np.random.default_rng([0xDA7A, seed])
    B, Q, M, C, P, G = (geo[k] for k in ("B", "Q", "M", "C", "P", "G"))
    shapes = np.array(geo["shapes"], np.int64)
    L = len(shapes)
    S = int((shapes[:, 0] * shapes[:, 1]).sum())
    value = rng.standard_normal((B, S, M, C))
    logits = rng.standard_normal((B, Q, M, L * P))
    Wl = np.repeat(shapes[:, 1], P).reshape(1, 1, 1, L * P).astype(np.float64)
    Hl = np.repeat(shapes[:, 0], P).reshape(1, 1, 1, L * P).astype(np.float64)
    gk = np.arange(L * P) % P % G
    if geo["dist"] == "dyadic":  # positions on integers, half-integers, -1, 0, H-1, H and beyond
        ref = rng.integers(0, 65, (B, Q, 1, 2 * G)) / 64.0
        rx, ry = ref[..., 0::2][..., gk], ref[..., 1::2][..., gk]
        tx = rng.integers(-4, 2 * Wl.astype(np.int64) + 4, (B, Q, M, L * P)) / 2.0 - 1.0
        ty = rng.integers(-4, 2 * Hl.astype(np.int64) + 4, (B, Q, M, L * P)) / 2.0 - 1.0
        off = np.stack([tx + 0.5 - rx * Wl, ty + 0.5 - ry * Hl], -1)
    else:
        lo, hi, scale = (0.0, 1.0, 2.0) if geo["dist"] == "normal" else (-0.5, 1.5, 8.0)
        ref = rng.uniform(lo, hi, (B, Q, 1, 2 * G))
        off = rng.standard_normal((B, Q, M, L * P, 2)) * scale
    mask = np.where(rng.random((B, Q)) < 0.3, 0.0, rng.uniform(0.0, 2.0, (B, Q)))
    go = rng.standard_normal((B, Q, M, C))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).float()  # noqa: E731
    return (t(value), torch.from_numpy(shapes), t(ref), t(off.reshape(B, Q, M, L * P * 2)), t(logits), t(mask), t(go))


# The kernel-selection rules, restated.
#   Forward (csrc/msda.cu:990-997 dispatch, :979-988 dispatch_rounds, msda_geometry.cuh:35-37 msda_lane_group_shape):
#   the lane-group gather when every tensor is 16-byte aligned, C == 32, P % 4 == 0, G in {1, 2, 4} and L*P <= 256
#   (kMaxChunks * 4), at ceil(L*P/4 / LPI) <= 4 rounds (LPI = 8 lanes per item in FP32, 4 in FP16 / BF16:
#   Io<T>::kVec = 4 / 8); the plugin op runs the generic kernel otherwise. The fused SCA epilogues take the gather at
#   <= 2 rounds only; otherwise the entry declines and the Python fallback runs the plugin op (functions/
#   multi_scale_deformable_attn.py:461-471).
#   Backward (csrc/msda_backward.cu:482-485 msda_bw_takes_c32, :516-531): the c32 kernel for the lane-group shape with
#   L*P <= 64 (kBwC32MaxPoints) and aligned tensors, the generic kernel otherwise; the fused forms' backward entry takes
#   the c32 kernel only, and when the forward ran the fallback, or the entry declines, the plugin backward runs
#   (multi_scale_deformable_attn.py:500-507).
def _lane_group_shape(geo):
    return geo["C"] == 32 and geo["P"] % 4 == 0 and geo["G"] in (1, 2, 4) and not geo["misaligned"]


def _rounds(geo, dtype):
    lpi = 8 if dtype == torch.float32 else 4
    return -(-(len(geo["shapes"]) * geo["P"] // 4) // lpi)


def msda_forward_path(geo, dtype):
    NP = len(geo["shapes"]) * geo["P"]
    return "gather" if _lane_group_shape(geo) and NP <= 256 and _rounds(geo, dtype) <= 4 else "generic"


def msda_fused_path(geo, dtype):
    return "fused" if _lane_group_shape(geo) and _rounds(geo, dtype) <= 2 else "fallback"


def msda_backward_path(geo):
    return "c32" if _lane_group_shape(geo) and len(geo["shapes"]) * geo["P"] <= 64 else "generic"


def _msda_dims_ok(geo):
    """msda_check_dims (csrc/msda_geometry.cuh:25-31): every dimension positive, L <= 16, (S + 1) * M * C * 4 < 2^31."""
    S = sum(h * w for h, w in geo["shapes"])
    return all(geo[k] > 0 for k in ("B", "Q", "M", "C", "P", "G")) and 1 <= len(geo["shapes"]) <= 16 and \
        (S + 1) * geo["M"] * geo["C"] * 4 < 2**31


# ---- DCN geometries ----------------------------------------------------------------------------------------------------
_DCN_WORK = 1_500_000  # N * C * kh*kw * Ho*Wo cap


def _out_extent(size, k, s, p, d):
    return (size + 2 * p - (d * (k - 1) + 1)) // s + 1


def dcn_geometry(seed):
    """One drawn DCNv2 layer: (N, C, H, W, Co, kh, kw, (sh, sw), (ph, pw), (dh, dw), groups, deform_groups) plus
    whether it has a bias and whether the input is passed channels-last."""
    rng = np.random.default_rng([0xDC2, seed])
    while True:
        N = int(rng.integers(1, 4))
        fused_shape = rng.random() < 0.35
        if fused_shape:
            g = dg = 1
            C, Co = int(rng.choice([64, 128])), int(rng.choice([128, 256, 512]))
            kh, kw = (int(v) for v in rng.integers(1, 4, 2))
        else:
            g, dg = (int(v) for v in rng.choice([1, 2, 3, 4], 2))
            C = math.lcm(g, dg) * int(rng.integers(1, max(2, 48 // math.lcm(g, dg)) + 1))
            Co = g * int(rng.integers(1, 25))
            kh, kw = (int(v) for v in rng.integers(1, 10, 2))
        if kh * kw > 75:
            continue
        s = tuple(int(v) for v in rng.integers(1, 4, 2))
        p = tuple(int(v) for v in rng.integers(0, 4, 2))
        d = tuple(int(v) for v in rng.integers(1, 4, 2))
        H, W = (int(v) for v in rng.integers(1, 41, 2))
        edge = rng.random()
        if edge < 0.12:
            H = 1
        elif edge < 0.24:
            W = 1
        Ho, Wo = _out_extent(H, kh, s[0], p[0], d[0]), _out_extent(W, kw, s[1], p[1], d[1])
        if Ho < 1 or Wo < 1 or N * C * kh * kw * Ho * Wo > _DCN_WORK:
            continue
        geo = (N, C, H, W, Co, kh, kw, s, p, d, g, dg)
        return dict(geo=geo, bias=bool(rng.random() < 0.7), channels_last=bool(fused_shape and rng.random() < 0.5))


def dcn_inputs(layer, seed):
    """float32 CPU tensors x, offset, mask, weight, bias (or None), grad_out."""
    N, C, H, W, Co, kh, kw, s, p, d, g, dg = layer["geo"]
    rng = np.random.default_rng([0xDC3, seed])
    kk = kh * kw
    Ho, Wo = _out_extent(H, kh, s[0], p[0], d[0]), _out_extent(W, kw, s[1], p[1], d[1])
    x = rng.standard_normal((N, C, H, W))
    kind = rng.random((N, dg * 2 * kk, Ho, Wo))
    off = np.where(kind < 0.5, rng.standard_normal(kind.shape) * 1.5,  # ordinary
                   np.where(kind < 0.8, rng.integers(-6, 7, kind.shape) / 2.0,  # integer / half-integer positions
                            rng.choice([-1.0, 1.0], kind.shape) * (max(H, W) + rng.uniform(0, 4, kind.shape))))  # outside
    mk = rng.random((N, dg * kk, Ho, Wo))
    mask = np.where(mk < 0.1, 0.0, np.where(mk < 0.3, rng.uniform(-1.5, 1.5, mk.shape),
                                             1 / (1 + np.exp(-rng.standard_normal(mk.shape)))))  # fmt: skip
    w = rng.standard_normal((Co, C // g, kh, kw)) / math.sqrt(C // g * kk)
    b = rng.standard_normal(Co) if layer["bias"] else None
    go = rng.standard_normal((N, Co, Ho, Wo))
    t = lambda a: torch.from_numpy(a).float() if a is not None else None  # noqa: E731
    return t(x), t(off), t(mask), t(w), t(b), t(go)


def dcn_forward_path(layer, dtype):
    """functions/modulated_deformable_conv2d.py:43-46: the fused wgmma kernel for FP16 with groups = deform_groups = 1,
    C % 64 == 0, Co in {128, 256, 512} and kh*kw <= 9; the generic kernel otherwise."""
    N, C, H, W, Co, kh, kw, s, p, d, g, dg = layer["geo"]
    fused = dtype == torch.float16 and g == 1 and dg == 1 and C % 64 == 0 and Co in (128, 256, 512) and kh * kw <= 9
    return "fused" if fused else "generic"


def _dcn_kw(geo):
    *_, s, p, d, g, dg = geo
    return dict(stride=s, padding=p, dilation=d, groups=g, deform_groups=dg)


# ---- CPU: the generators, the mirrors and the bound --------------------------------------------------------------------
def test_msda_geometries_are_accepted_and_reach_every_branch():
    geos = [msda_geometry(s) for s in MSDA_SEEDS]
    assert all(_msda_dims_ok(g) for g in geos)
    assert len({repr(g) for g in geos}) == len(geos)  # no case repeats
    fwd = {msda_forward_path(g, dt) for g in geos for dt in DTYPES}
    fused = {msda_fused_path(g, dt) for g in geos for dt in DTYPES}
    bwd = {msda_backward_path(g) for g in geos}
    assert fwd == {"gather", "generic"} and fused == {"fused", "fallback"} and bwd == {"c32", "generic"}
    # the lane-group shape just below and just above the backward's 64-point limit, and the forward's round limits
    nps = {len(g["shapes"]) * g["P"] for g in geos if _lane_group_shape(g)}
    assert any(n <= 64 for n in nps) and any(n > 64 for n in nps), nps
    assert {_rounds(g, dt) for g in geos if _lane_group_shape(g) for dt in DTYPES} >= {1, 2, 3}
    assert any(_lane_group_shape(g) and _rounds(g, torch.float16) > 4 for g in geos)  # FP16 gather -> generic
    # the edges of every dimension
    assert {1} <= {g["M"] for g in geos} and {1} <= {g["C"] for g in geos} and {1} <= {g["Q"] for g in geos}
    assert {1, 5, 16, 32, 40, 64} <= {g["C"] for g in geos}
    assert {1, 2, 3, 4, 8} <= {g["G"] for g in geos}
    assert any((1, 1) in g["shapes"] for g in geos)
    assert any(h == 1 and w > 1 for g in geos for h, w in g["shapes"])
    assert any(w == 1 and h > 1 for g in geos for h, w in g["shapes"])
    assert any(len(g["shapes"]) == 1 for g in geos) and max(len(g["shapes"]) for g in geos) >= 12
    assert {"normal", "out", "dyadic"} == {g["dist"] for g in geos}
    assert any(g["misaligned"] and g["C"] == 32 and g["P"] % 4 == 0 and g["G"] in (1, 2, 4) for g in geos)


def test_dcn_geometries_are_accepted_and_reach_every_branch():
    layers = [dcn_geometry(s) for s in DCN_SEEDS]
    assert len({repr(x) for x in layers}) == len(layers)
    for lay in layers:
        geo = lay["geo"]
        assert geo[5] * geo[6] <= 75
        for f16 in (False, True):
            assert _ws_query(geo, f16) == _plan(geo, f16)["total"] > 0, geo
    assert {dcn_forward_path(x, torch.float16) for x in layers} == {"fused", "generic"}
    fused = [x["geo"] for x in layers if dcn_forward_path(x, torch.float16) == "fused"]
    assert any(geo[2] == 1 or geo[3] == 1 for geo in fused)  # a fused-eligible layer with H or W of 1
    assert any(x["channels_last"] for x in layers)
    geos = [x["geo"] for x in layers]
    assert {3} <= {geo[10] for geo in geos} and {3} <= {geo[11] for geo in geos}
    assert {1, 2, 3, 4} <= {geo[10] for geo in geos} | {geo[11] for geo in geos}
    assert {True, False} == {x["bias"] for x in layers}
    plans = [_plan(geo, f16) for geo in geos for f16 in (False, True)]  # FP32 / BF16 and FP16 workspace layouts
    assert {pl["KC"] for pl in plans} == {16, 8, 4, 2, 1}
    assert {pl["npass"] for pl in plans} == {1, 2}
    assert any(_ragged(pl["nch"], pl["nsplit"]) for pl in plans)
    assert any(_ragged(pl["items"], pl["wsplit"]) for pl in plans)
    assert any(pl["nsplit"] == 1 for pl in plans) and any(pl["wsplit"] == 1 for pl in plans)


@pytest.mark.parametrize("seed", MSDA_SEEDS)
def test_fp32_msda_oracle_meets_the_element_bound(seed):
    """The FP32 C oracle (the kernels' arithmetic restated) against the float64 reference: validates the bound on the
    CPU, on every swept geometry."""
    geo = msda_geometry(seed)
    value, shapes, ref, off, logits, _, _ = msda_inputs(geo, seed)
    got = omsda.msda_f32(value.numpy(), shapes.numpy(), ref.numpy(), off.numpy(), logits.numpy())
    want = msda_f64(value, shapes, ref, off, logits)
    check(f"msda oracle seed {seed} {geo}", "out", torch.from_numpy(got), want["out"], U32)


@pytest.mark.parametrize("seed", DCN_SEEDS)
def test_fp32_dcn_oracle_meets_the_element_bound(seed):
    lay = dcn_geometry(seed)
    x, off, mask, w, b, _ = dcn_inputs(lay, seed)
    kw = _dcn_kw(lay["geo"])
    got = odcn.modulated_deformable_conv2d(x.numpy(), off.numpy(), mask.numpy(), w.numpy(),
                                           None if b is None else b.numpy(), **kw)  # fmt: skip
    want = dcn_f64(x, off, mask, w, b, **kw)
    check(f"dcn oracle seed {seed} {lay}", "out", torch.from_numpy(got), want["out"], U32)


def test_float64_gradients_match_the_autograd_references():
    """The gradient formulas of oracle/f64.py against the independent float64 autograd references the suite already
    has (oracle.msda_backward.msda_backward_f64; torchvision with mmcv's rule, tests/test_dcn_backward_gpu._oracle_grads),
    and every magnitude at least |r|."""
    from oracle.msda_backward import msda_backward_f64
    from tests.test_dcn_backward_gpu import _oracle_grads

    for seed in MSDA_SEEDS[:8]:
        geo = msda_geometry(seed)
        value, shapes, ref, off, logits, mask, go = msda_inputs(geo, seed)
        ours = msda_f64(value, shapes, ref, off, logits, go)
        theirs = msda_backward_f64(value, shapes, ref, off, logits, go)
        for name, t in zip(("out", "grad_value", "grad_ref", "grad_off", "grad_logits"), theirs):
            e = ours[name]
            assert float((e["r"] - t).abs().max()) <= 1e-12 * max(1.0, float(t.abs().max())), (seed, name)
            assert bool((e["mag"] >= e["r"].abs() * (1 - 1e-12)).all()), (seed, name)
    for seed in DCN_SEEDS[:8]:
        lay = dcn_geometry(seed)
        x, off, mask, w, b, go = dcn_inputs(lay, seed)
        kw = _dcn_kw(lay["geo"])
        ours = dcn_f64(x, off, mask, w, b, **kw, grad_out=go)
        out, theirs = _oracle_grads(x, off, mask, w, b, go, kw)
        for name, t in zip(("out",) + tuple(_DCN_KEYS.values()), [out] + theirs):
            if t is None:
                assert name not in ours, (seed, name)
                continue
            e = ours[name]
            assert float((e["r"] - t).abs().max()) <= 1e-12 * max(1.0, float(t.abs().max())), (seed, name)
            assert bool((e["mag"] >= e["r"].abs() * (1 - 1e-12)).all()), (seed, name)


# ---- GPU: kernel identity ----------------------------------------------------------------------------------------------
_GATHER_EPI = re.compile(r"msda_gather_kernel<\s*[\w: ]+,\s*[\w: ]+,\s*\d+,\s*\d+,\s*\d+,\s*(\d+)")
_BW_EPI = re.compile(r"msda_bw_c32_kernel<[^,]+,\s*(\d)")


_MSDA_FWD = ("msda_gather_kernel", "msda_generic_kernel")
_MSDA_BW = ("msda_bw_c32_kernel", "msda_bw_generic_kernel")


def _traced(names, families):
    """Whether the trace holds a kernel of ``families`` (False: the records were lost, the identity is unchecked)."""
    return any(f in n for n in names for f in families)


def _msda_fwd_family(names, fused_form):
    """'gather' / 'generic' for a plugin-op call; for a fused form 'fused' when a gather kernel with a camera-sum
    epilogue ran, 'fallback' otherwise."""
    gathers = [_GATHER_EPI.search(n) for n in names if "msda_gather_kernel" in n]
    if fused_form:
        return "fused" if any(m is not None and m.group(1) != "0" for m in gathers) else "fallback"
    fams = {"gather" if "msda_gather_kernel" in n else "generic" for n in names
            if "msda_gather_kernel" in n or "msda_generic_kernel" in n}  # fmt: skip
    return fams.pop() if len(fams) == 1 else tuple(sorted(fams))


def _msda_bw_family(names, fused_form):
    c32 = [_BW_EPI.search(n) for n in names if "msda_bw_c32_kernel" in n]
    if fused_form and any(m is not None and m.group(1) != "0" for m in c32):
        return "fused"
    fams = {"c32" if "msda_bw_c32_kernel" in n else "generic" for n in names
            if "msda_bw_c32_kernel" in n or "msda_bw_generic_kernel" in n}  # fmt: skip
    return fams.pop() if len(fams) == 1 else tuple(sorted(fams))


# ---- GPU: MSDA ---------------------------------------------------------------------------------------------------------
_MSDA_NAMES = ("value", "ref", "off", "logits")
_GRAD_KEYS = {"value": "grad_value", "ref": "grad_ref", "off": "grad_off", "logits": "grad_logits"}


def _requested(rng, names):
    want = [n for n in names if rng.random() < 0.6]
    return want or [names[int(rng.integers(len(names)))]]


def _device_inputs(geo, seed, dtype, shared=False):
    """The op's inputs on the GPU in ``dtype`` (BF16: reference points in FP32, as the op reads them); value one element
    off alignment for a misaligned geometry; offsets and logits one copy for the camera-shared form."""
    value, shapes, ref, off, logits, mask, go = msda_inputs(geo, seed)
    if shared:
        off, logits = off[:1], logits[:1]
    ref_dt = torch.float32 if dtype == torch.bfloat16 else dtype
    dev = [value.to(dtype), shapes, ref.to(ref_dt), off.to(dtype), logits.to(dtype)]
    dev = [t.cuda() for t in dev]
    if geo["misaligned"]:
        buf = torch.empty(dev[0].numel() + 1, dtype=dtype, device="cuda")
        view = buf[1:].view(dev[0].shape)
        view.copy_(dev[0])
        dev[0] = view
    return dev, mask.cuda(), go.cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("seed", MSDA_SEEDS)
def test_msda_plugin_op_meets_the_element_bound(seed, dtype):
    """multi_scale_deformable_attn and its …2 twin (FP16: the h2 entry when C is even), forward and backward of a random
    subset of the inputs."""
    geo = msda_geometry(seed)
    dev, _, go = _device_inputs(geo, seed, dtype)
    go = go.to(dtype)
    want = msda_f64(*dev, grad_out=go, device="cuda")
    rng = np.random.default_rng([0x6AD, seed])
    wanted = _requested(rng, _MSDA_NAMES)
    fwd, bwd = msda_forward_path(geo, dtype), msda_backward_path(geo)
    for op in (bt.multi_scale_deformable_attn, bt.multi_scale_deformable_attn2):
        tag = f"seed {seed} {DT_IDS[DTYPES.index(dtype)]} {op.__name__} {geo} grads {wanted}"

        def run():
            leaves = [t.detach().requires_grad_(n in wanted) if i != 1 else t
                      for i, (n, t) in enumerate(zip(("value", "shapes", "ref", "off", "logits"), dev))]  # fmt: skip
            out = op(*leaves)
            out.backward(go)
            return out.detach(), {n: leaves[i].grad for i, n in ((0, "value"), (2, "ref"), (3, "off"), (4, "logits"))}

        (out, grads), names = kernels_recorded(run, lambda ns: _msda_fwd_family(ns, False) == fwd and
                                               _msda_bw_family(ns, False) == bwd)  # fmt: skip
        assert _msda_fwd_family(names, False) == fwd or not _traced(names, _MSDA_FWD), (tag, fwd, names)
        assert _msda_bw_family(names, False) == bwd or not _traced(names, _MSDA_BW), (tag, bwd, names)
        check(tag, "out", out, want["out"], U32)
        for n in _MSDA_NAMES:
            if n not in wanted:
                assert grads[n] is None, (tag, n)
                continue
            check(tag, _GRAD_KEYS[n], grads[n], want[_GRAD_KEYS[n]], U32)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("seed", MSDA_SEEDS)
def test_msda_fused_forms_meet_the_element_bound(seed, dtype):
    """multi_scale_deformable_attn_sca, …_sca_shared and …_queue_mean, forward and backward, with zeros in bev_mask."""
    geo = msda_geometry(seed)
    path = msda_fused_path(geo, dtype)
    bwd_plain = msda_backward_path(geo)
    rng = np.random.default_rng([0xF05, seed])
    wanted = _requested(rng, _MSDA_NAMES)
    B, Q, M, C = geo["B"], geo["Q"], geo["M"], geo["C"]
    gs = torch.from_numpy(rng.standard_normal((Q, M * C))).float().cuda()
    for form in ("sca", "sca_shared", "queue_mean"):
        shared = form == "sca_shared"
        dev, mask, _ = _device_inputs(geo, seed, dtype, shared=shared)
        if form == "queue_mean":
            mask = torch.full((B, Q), 1.0 / B, dtype=torch.float32, device="cuda")
            g_in = gs.to(dtype).reshape(1, Q, M * C)
            g_slots = g_in.float().reshape(Q, M * C)
        else:
            g_in = g_slots = gs
        want = msda_sca_f64(*dev, mask, grad_slots=g_slots, shared=shared, device="cuda")
        tag = f"seed {seed} {DT_IDS[DTYPES.index(dtype)]} {form} {geo} grads {wanted}"

        def run():
            leaves = [t.detach().requires_grad_(n in wanted) if i != 1 else t
                      for i, (n, t) in enumerate(zip(("value", "shapes", "ref", "off", "logits"), dev))]  # fmt: skip
            if form == "sca":
                out = bt.multi_scale_deformable_attn_sca(*leaves, mask)
            elif form == "sca_shared":
                out = bt.multi_scale_deformable_attn_sca_shared(*leaves, mask)
            else:
                out = bt.multi_scale_deformable_attn_queue_mean(*leaves)
            out.backward(g_in)
            return out.detach(), {n: leaves[i].grad for i, n in ((0, "value"), (2, "ref"), (3, "off"), (4, "logits"))}

        bwd = "fused" if path == "fused" and bwd_plain == "c32" else bwd_plain
        (out, grads), names = kernels_recorded(run, lambda ns: _msda_fwd_family(ns, True) == path and
                                               _msda_bw_family(ns, True) == bwd)  # fmt: skip
        assert _msda_fwd_family(names, True) == path or not _traced(names, _MSDA_FWD), (tag, path, names)
        assert _msda_bw_family(names, True) == bwd or not _traced(names, _MSDA_BW), (tag, bwd, names)
        ent = want["out"]
        if form == "queue_mean":
            ent = {k: (v.reshape(1, Q, M * C) if torch.is_tensor(v) and v.dim() == 2 else v) for k, v in ent.items()}
        check(tag, "out", out, ent, U32, low=None if path == "fused" else dtype)
        for n in _MSDA_NAMES:
            if n not in wanted:
                assert grads[n] is None, (tag, n)
                continue
            check(tag, _GRAD_KEYS[n], grads[n], want[_GRAD_KEYS[n]], U32, low=None if bwd == "fused" else dtype)


# ---- GPU: DCN ----------------------------------------------------------------------------------------------------------
_DCN_NAMES = ("input", "offset", "mask", "weight", "bias")
_DCN_KEYS = {"input": "grad_input", "offset": "grad_offset", "mask": "grad_mask", "weight": "grad_weight",
             "bias": "grad_bias"}  # fmt: skip


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("seed", DCN_SEEDS)
def test_dcn_meets_the_element_bound(seed, dtype):
    """modulated_deformable_conv2d forward and the backward of a random subset of its inputs."""
    lay = dcn_geometry(seed)
    geo = lay["geo"]
    kw = _dcn_kw(geo)
    x, off, mask, w, b, go = (t.to(dtype).cuda() if t is not None else None for t in dcn_inputs(lay, seed))
    if lay["channels_last"]:
        x = x.contiguous(memory_format=torch.channels_last)
    want = dcn_f64(x, off, mask, w, b, **kw, grad_out=go, device="cuda")
    rng = np.random.default_rng([0xDC4, seed])
    names = [n for n in _DCN_NAMES if n != "bias" or b is not None]
    wanted = _requested(rng, names)
    path = dcn_forward_path(lay, dtype)
    tag = f"seed {seed} {DT_IDS[DTYPES.index(dtype)]} {lay} {path} grads {wanted}"

    def run():
        leaves = [t.detach().requires_grad_(n in wanted) if t is not None else None
                  for n, t in zip(_DCN_NAMES, (x, off, mask, w, b))]  # fmt: skip
        out = bt.modulated_deformable_conv2d(*leaves, kw["stride"], kw["padding"], kw["dilation"], kw["groups"],
                                             kw["deform_groups"])  # fmt: skip
        out.backward(go)
        return out.detach(), {n: t.grad if t is not None else None for n, t in zip(_DCN_NAMES, leaves)}

    kernel = {"fused": "dcn_fused_kernel", "generic": "dcn_generic_kernel"}
    (out, grads), ran = kernels_recorded(run, lambda ns: any(kernel[path] in n for n in ns))
    assert any(kernel[path] in n for n in ran) or not _traced(ran, tuple(kernel.values())), (tag, ran)
    assert not any(k in n for n in ran for p_, k in kernel.items() if p_ != path), (tag, ran)
    # the backward's data kernel runs for input / offset / mask gradients, its weight kernel for the weight gradient
    # (csrc/dcn_backward.cu); channels per K block, tap passes and splits are launch arguments the trace does not show
    if _traced(ran, ("dcn_bw_",)):
        assert any("dcn_bw_data_kernel" in n for n in ran) == bool({"input", "offset", "mask"} & set(wanted)), (tag, ran)
        assert any("dcn_bw_weight_kernel" in n for n in ran) == ("weight" in wanted), (tag, ran)
    if path == "fused":
        r = want["out"]["r"]
        fp16_tol = 0.5 * float(ulp(r.abs().max().reshape(1), torch.float16)) + 1e-3 * max(1.0, float(mask.abs().max()))
        check(tag, "out", out, want["out"], U_WGMMA, low=torch.float16, bar=fp16_tol)
    else:
        check(tag, "out", out, want["out"], U32)
    for n in _DCN_NAMES:
        if n not in wanted:
            assert grads[n] is None, (tag, n)
            continue
        check(tag, _DCN_KEYS[n], grads[n], want[_DCN_KEYS[n]], U32)
