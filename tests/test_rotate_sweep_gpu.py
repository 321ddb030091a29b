"""Rotate (RotateTRT / RotateTRT2, csrc/rotate.cu) over seeded random geometries in every entry and layout, checked
element by element against the float64 reference oracle.f64.rotate_f64.

Each case is one image [C, H, W], one angle and one centre, run through every entry that accepts them: ``rotate`` and
``rotate2`` in FP32, ``rotate`` and ``rotate_chw2`` (kCHW2) in FP16, ``rotate_int8`` (kCHW4) with an FP32 and with an
FP16 angle and centre, and the channels-last kernel in FP32 and FP16 where C is a whole number of 16-byte vectors, both
interpolations. The FP16 entries read the angle and centre as FP16; a case whose angle or centre has no finite FP16
value (a rotation near 1e5 degrees, a centre near 1e10) runs the FP32-angle entries only. So ``rot_safe``
(csrc/rotate.cu:64-67), which needs an index beyond the int range, is reached by the FP32-angle entries only: with a
finite FP16 centre (|c| <= 65504) an index stays within 3 * 65504 plus twice the image's extent, far below 2^31.

**Indices.** ``b200_rotate_debug_indices`` gives the source index (ix, iy) of every output pixel (FP16 angles and
centres are passed as their exact fp32 widening, the matrix the FP16 entries build). They must equal the C oracle's
(oracle/rotate_oracle.c) given the device's cos / sin bit for bit, and lie within

    |i - i*| <= K_IDX * 2^-24 * (|cx| + |cy| + |x| + |y| + |i*| + S),   K_IDX = 12,

of the float64 position i* (S = W for ix, H for iy; x, y the pixel's centred coordinates; cx, cy the centre minus half
the image). i* takes the angle rounded once to fp32 (csrc/rotate.cu:55) and exact cos / sin. In units of 2^-24, the
error of ix is at most: the roundings of cx, cy (:57-58) moving nx by 2|cx| + |cy|; cosf / sinf, 2 ulp each in CUDA's
documented bounds, at most 4 units absolute for a value of magnitude <= 1, times |x - cx| + |y - cy|; the three
roundings of m2 (:60), 3|cx| + 3|cy|; the three of nx (:72), 2|x| + 2|y| + |ix| + W; the division, the + 1 and the fma
(:74, :77), |ix| + W each at most. Together 9|cx| + 8|cy| + 6|x| + 6|y| + 4|ix| + 3W, and iy likewise: K_IDX = 12
leaves room for the second-order terms. Where i* is clearly beyond the int range the index must be -100 (rot_safe).

**Values.** rotate_f64 takes the device's indices, so the index arithmetic and the blend are separate questions. Every
element must satisfy the bound of tests/test_msda_dcn_sweep_gpu.py (tests.helpers.element_bound),

    |got - r| <= 1/2 ulp_dtype(|r| + E) + E,   E = (8 + n) * 2^-24 * mag,

with n = 4 for bilinear. The kernel's bilinear weight is one product of two differences (:95-99); a difference is
exact by Sterbenz where |i| >= 1 and rounds once otherwise, so each weight is within 3 * 2^-24 of its value, relative;
the blend is a chain of one product and three fmaf (:149, :237), four roundings of partial sums at most mag. That is
7 * 2^-24 * mag, within (8 + 4) * 2^-24 * mag. The values read are exact (FP16 widened; INT8's q * scale_i is the value
the oracle is given). Then one rounding to the output dtype, FP16 subnormals included. Nearest copies a pixel: it is
bit-exact in every float entry. rotate2 equals rotate, kCHW2 the FP16 linear entry, and the channels-last kernel the
planar one, bit for bit.

**INT8** is checked in output steps. Nearest is bit-exact against the float32 restatement
``t2int8(fl32(fl32(q * si) * fl32(1 / so)))`` (csrc/packets.cuh:74-85, csrc/common.cuh:103-107: the ``a + 0.5f`` of the
rounding included). Bilinear: ``|q - clip(r / so, -128, 127)| <= 1/2 + delta`` with
``delta = (E + 2.0001 * 2^-24 |r|) / so * (1 + 2^-21) + 2^-17``: the blend's error E; the rounding of 1 / so and of the
product v * (1 / so), 2^-24 relative each; and the rounding of a +- 0.5 for |a| <= 128, half an ulp at most 2^-17.
Where r / so is beyond the range by more than delta, q is exactly 127 or -128.

**Launch plans.** A thread owns a run of ``cps`` channel packets of one pixel (plan_slices, csrc/common.cuh:36-42,
restated below with rotate.cu:284's arguments), and channels-last lanes share a pixel in groups of ``lp``
(rotate.cu:300). The CPU coverage test checks that the default seeds reach, for packet widths 1, 2 and 4, the
single-slice plan, one packet per slice, several packets per slice dividing CP and a ragged last slice; every lp and a
vector count that lp does not divide; and for every entry H = 1, W = 1, 1 x 1, a multiple of 90 degrees, a case with
every source outside the image and (FP32-angle entries) a rot_safe case. B200_SWEEP_SEEDS=<k> adds k seeds beyond the
default list.

``bt.rotate`` handed a permuted channels-last view must run rotate_hwc_kernel and return a view of a channels-last
output, and the same view an element off 16-byte alignment rotate_planar_kernel (tests.helpers.kernels_recorded, one
trace per call). The kernel trace now and then loses a record; a call whose trace holds no rotate kernel at all leaves
the kernel's name unchecked (its bits and the output's layout are still checked), as in
tests/test_msda_dcn_sweep_gpu.py.

When the reference project's kernels are built (oracle.REF_LIB), the FP32 cases are also run through them: nearest
picks the same pixels and bilinear meets the same bound.
"""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

import bevformer_tensorrt_b200 as bt
from bevformer_tensorrt_b200 import _lib
from bevformer_tensorrt_b200.functions.grid_sampler import pack_chw, unpack_chw
from oracle import REF_LIB
from oracle import rotate as orot
from oracle.f64 import rotate_f64
from tests.helpers import U32, check, kernels_recorded
from tests.test_rotate_gpu import device_trig

K_IDX = 12
MIN_THREADS = 132 * 2048 * 4  # rotate.cu:284: plan_slices' min_threads and max_cps
MAX_CPS = 16
INTERPS = ((0, "bilinear"), (1, "nearest"))

# chosen so that together they reach every plan and edge the CPU coverage test lists
SEEDS = [0, 1, 2, 3, 4, 5, 6, 7, 9, 11, 12, 14, 16, 17, 19, 37, 137, 143, 164, 196, 209, 255, 270, 294, 298, 359, 387]
_EXTRA = int(os.environ.get("B200_SWEEP_SEEDS", "0") or 0)
SEEDS += [100_000 + i for i in range(_EXTRA)]


# ---- the launch plans, restated ----------------------------------------------------------------------------------------
def plan_slices(pixels, packets):
    """common.cuh:36-42 with rotate.cu:284's arguments: (slices, cps)."""
    n = 1
    while n < packets and (pixels * n < MIN_THREADS or -(-packets // n) > MAX_CPS):
        n <<= 1
    cps = -(-packets // n)
    return -(-packets // cps), cps


def hwc_lanes(nvec):
    """rotate.cu:300: lanes per pixel of the channels-last kernel."""
    return 8 if nvec >= 8 else 4 if nvec >= 4 else 2 if nvec >= 2 else 1


# ---- geometries --------------------------------------------------------------------------------------------------------
_ELEMS = 7_000_000  # C * H * W cap


def _shape(rng, pixels):
    """(H, W) of about ``pixels`` pixels: a line either way, or a rectangle of odd or random width."""
    k = rng.random()
    if k < 0.15:
        return 1, pixels
    if k < 0.3:
        return pixels, 1
    W = int(rng.integers(100, 2000)) | (1 if rng.random() < 0.5 else 0)
    return -(-pixels // W), W


def rotate_geometry(seed):
    """One drawn case: C, H, W, the angle (degrees) and centre (x, y) as float32 values, their kinds, and the value
    scales: ``k32`` (FP32 image x 2^k), ``k16`` (FP16 image x 2^k, down to subnormal outputs), ``si`` / ``so`` (INT8
    input and output scales)."""
    rng = np.random.default_rng([0x2074, seed])
    kind = str(rng.choice(["small"] * 5 + ["line", "mid", "big"]))
    if kind == "small":
        H, W = (int(v) for v in rng.integers(1, 65, 2))
        e = rng.random()
        if e < 0.12:
            H = 1
        elif e < 0.24:
            W = 1
        elif e < 0.3:
            H = W = 1
        C = int(rng.integers(1, 33)) if rng.random() < 0.6 else int(rng.integers(33, 400))
    elif kind == "line":
        n = int(rng.integers(2, 5000))
        H, W = (1, n) if rng.random() < 0.5 else (n, 1)
        C = int(rng.integers(1, 65))
    elif kind == "mid":  # several packets per slice: CP4 just above the slice count n the plan stops at
        n = int(rng.choice([2, 4, 8, 16, 32]))
        H, W = _shape(rng, int(MIN_THREADS / n * rng.uniform(1.0, 1.1)))
        cp4 = int(rng.integers(n + 1, n + n // 2 + 2))
        C = 4 * cp4 - int(rng.integers(0, 4))
    else:  # one slice: a plane of at least MIN_THREADS pixels
        H, W = _shape(rng, int(MIN_THREADS * rng.uniform(1.0, 1.05)))
        C = int(rng.integers(5, 7))
    C = max(1, min(C, _ELEMS // (H * W)))

    akind = str(rng.choice(["zero", "right", "right", "tiny", "random", "random", "huge"]))
    if akind == "zero":
        ang = 0.0
    elif akind == "right":
        ang = 90.0 * int(rng.integers(-8, 9))
    elif akind == "tiny":
        ang = float(rng.choice([-1.0, 1.0]) * 10.0 ** rng.uniform(-7, -2))
    elif akind == "random":
        ang = float(rng.uniform(-720, 720))
    else:
        ang = float(rng.choice([-1.0, 1.0]) * rng.uniform(3e4, 1.2e5))
    ckind = str(rng.choice(["centre", "corner", "edge", "frac", "frac", "neg", "outside", "far"]))
    if ckind == "centre":
        ctr = (W / 2, H / 2)
    elif ckind == "corner":
        ctr = (float(rng.choice([0, W])), float(rng.choice([0, H])))
    elif ckind == "edge":
        ctr = (float(rng.choice([0, W])), float(rng.uniform(0, H))) if rng.random() < 0.5 else \
            (float(rng.uniform(0, W)), float(rng.choice([0, H])))
    elif ckind == "frac":
        ctr = (float(rng.uniform(-0.5, 1.5) * W), float(rng.uniform(-0.5, 1.5) * H))
    elif ckind == "neg":
        ctr = (-float(rng.uniform(0, W)), -float(rng.uniform(0, H)))
    elif ckind == "outside":
        k = rng.integers(2, 7, 2) * rng.choice([-1, 1], 2)
        ctr = (float(k[0] * W + rng.uniform(0, W)), float(k[1] * H + rng.uniform(0, H)))
    else:
        ctr = tuple(float(v) for v in rng.choice([-1.0, 1.0], 2) * rng.uniform(1e10, 3e10, 2))
    ang, ctr = float(np.float32(ang)), tuple(float(np.float32(v)) for v in ctr)
    si = float(np.float32(2.0 ** int(rng.integers(-12, 5)) if rng.random() < 0.5 else 10.0 ** rng.uniform(-4, 1)))
    so = float(np.float32(si * 128 / 127 * 10.0 ** rng.uniform(-0.6, 0.2)))  # below si * 128 / 127: some saturate
    return dict(kind=kind, C=C, H=H, W=W, akind=akind, ang=ang, ckind=ckind, ctr=ctr, k32=int(rng.integers(-60, 61)),
                k16=int(rng.integers(-22, 13)), si=si, so=so)  # fmt: skip


def half_ok(geo):
    """Whether the angle and centre have finite FP16 values (the FP16 entries read them as FP16)."""
    with np.errstate(over="ignore"):
        return bool(np.isfinite(np.float16([geo["ang"], *geo["ctr"]])).all())


def half_scalars(geo):
    """The angle and centre the FP16 entries see, as float32 values (exact)."""
    h = np.float16([geo["ang"], *geo["ctr"]]).astype(np.float32)
    return float(h[0]), (float(h[1]), float(h[2]))


def entries(geo):
    """The entries a case runs."""
    C = geo["C"]
    e = ["rotate_f32", "rotate2_f32", "int8_f32_angle"] + (["hwc_f32"] if C % 4 == 0 else [])
    if half_ok(geo):
        e += ["rotate_f16", "chw2", "int8_f16_angle"] + (["hwc_f16"] if C % 8 == 0 else [])
    return e


def rotate_inputs(geo, seed):
    """float32 CPU tensors: the FP32 image, the FP16 image (as float16), the INT8 image (as int8)."""
    rng = np.random.default_rng([0x2075, seed])
    C, H, W = geo["C"], geo["H"], geo["W"]
    x = rng.standard_normal((C, H, W), dtype=np.float32)
    img32 = torch.from_numpy(np.ldexp(x, geo["k32"]).astype(np.float32))
    img16 = torch.from_numpy(np.ldexp(x, geo["k16"])).half()
    q = torch.from_numpy(rng.integers(-128, 128, (C, H, W), dtype=np.int8))
    return img32, img16, q


# ---- index checks ------------------------------------------------------------------------------------------------------
def ideal_indices(ang, ctr, H, W):
    """float64 (ix*, iy*) [H, W] and their bounds: the angle rounded once to fp32 (rotate.cu:55), exact cos / sin."""
    a = float(np.float32(np.float64(-np.float32(ang)) * math.pi / 180.0))
    c, s = math.cos(a), math.sin(a)
    cx, cy = float(ctr[0]) - 0.5 * W, float(ctr[1]) - 0.5 * H
    x = (np.arange(W, dtype=np.float64) + 0.5 - 0.5 * W)[None, :]
    y = (np.arange(H, dtype=np.float64) + 0.5 - 0.5 * H)[:, None]
    ix = c * (x - cx) + s * (y - cy) + cx + 0.5 * (W - 1)
    iy = c * (y - cy) - s * (x - cx) + cy + 0.5 * (H - 1)
    common = abs(cx) + abs(cy) + np.abs(x) + np.abs(y)
    return ix, iy, K_IDX * U32 * (common + np.abs(ix) + W), K_IDX * U32 * (common + np.abs(iy) + H)


def assert_indices_near_ideal(tag, got, ang, ctr):
    """got [H, W, 2] float32 source indices: within the bound of the float64 position, or -100 where it is beyond the
    int range."""
    H, W = got.shape[:2]
    ix, iy, bx, by = ideal_indices(ang, ctr, H, W)
    lim = 2.0**31
    for name, g, i, b in (("ix", got[..., 0], ix, bx), ("iy", got[..., 1], iy, by)):
        g = g.astype(np.float64)
        beyond = (i - b > lim) | (i + b < -lim)  # rot_safe replaces this axis' index only
        in_range = (i + b < lim - 2) & (i - b > -lim)
        assert (g[beyond] == -100.0).all(), (tag, name, "rot_safe")
        err = np.abs(g - i)
        bad = in_range & ~(err <= b)
        if bad.any():
            h, w = np.argwhere(bad)[0]
            raise AssertionError(f"{tag} {name}: {int(bad.sum())} of {bad.size} indices off the float64 position; "
                                 f"at ({h}, {w}) got {g[h, w]!r} ideal {i[h, w]!r} bound {b[h, w]:.3e}")  # fmt: skip


# ---- CPU: the generator, the restated plans and the bounds -------------------------------------------------------------
def _reach(geo):
    """(every source is outside the image, some index is rot_safe's -100), from the C oracle's indices."""
    xy = orot.source_indices(geo["ang"], geo["ctr"], geo["H"], geo["W"])
    ix, iy = xy[..., 0], xy[..., 1]
    return bool(((ix <= -1) | (ix >= geo["W"]) | (iy <= -1) | (iy >= geo["H"])).all()), bool((xy == -100).any())


def test_geometries_reach_every_plan_and_edge():
    geos = [rotate_geometry(s) for s in SEEDS]
    assert all(g["C"] * g["H"] * g["W"] <= _ELEMS and g["H"] * g["W"] < 2**31 for g in geos)
    for width in (1, 2, 4):
        plans = [(-(-g["C"] // width), *plan_slices(g["H"] * g["W"], -(-g["C"] // width))) for g in geos]
        assert any(sl == 1 and cp > 1 for cp, sl, cps in plans), width
        assert any(cps == 1 and sl > 1 for cp, sl, cps in plans), width
        assert any(cps > 1 and cp % cps == 0 and sl > 1 for cp, sl, cps in plans), width
        assert any(cps > 1 and cp % cps != 0 for cp, sl, cps in plans), width
    for vec, ent in ((4, "hwc_f32"), (8, "hwc_f16")):
        nvecs = [g["C"] // vec for g in geos if ent in entries(g)]
        assert {hwc_lanes(n) for n in nvecs} == {1, 2, 4, 8}, ent
        assert all(any(hwc_lanes(n) == lp and n % lp for n in nvecs) for lp in (2, 4, 8)), ent
    reach = {s: _reach(g) for s, g in zip(SEEDS, geos)}
    for ent in ("rotate_f32", "rotate2_f32", "int8_f32_angle", "hwc_f32", "rotate_f16", "chw2", "int8_f16_angle",
                "hwc_f16"):  # fmt: skip
        mine = [(s, g) for s, g in zip(SEEDS, geos) if ent in entries(g)]
        assert any(g["H"] == 1 and g["W"] > 1 for _, g in mine), ent
        assert any(g["W"] == 1 and g["H"] > 1 for _, g in mine), ent
        assert any(g["W"] == 1 and g["H"] == 1 for _, g in mine), ent
        assert any(g["ang"] != 0 and g["ang"] % 90 == 0 for _, g in mine), ent
        assert any(reach[s][0] for s, _ in mine), ent
        if ent in ("rotate_f32", "rotate2_f32", "int8_f32_angle", "hwc_f32"):  # module docstring: FP32 angles only
            assert any(reach[s][1] for s, _ in mine), ent
    assert {"zero", "right", "tiny", "random", "huge"} == {g["akind"] for g in geos}
    assert {"centre", "corner", "edge", "frac", "neg", "outside", "far"} == {g["ckind"] for g in geos}
    assert {1, 2, 3} <= {g["C"] % 4 for g in geos} and max(g["C"] for g in geos) >= 300
    assert any(g["kind"] in ("mid", "big") and (g["H"] == 1 or g["W"] == 1) for g in geos)


def test_no_case_repeats():
    geos = [repr(rotate_geometry(s)) for s in SEEDS]
    assert len(set(geos)) == len(geos)


@pytest.mark.parametrize("seed", SEEDS)
def test_fp32_oracle_meets_the_element_bound(seed):
    """The C oracle (the kernel's arithmetic restated, libm trig) against rotate_f64 fed the oracle's own indices, and
    those indices against the float64 position: validates both bounds on the CPU."""
    geo = rotate_geometry(seed)
    img32, _, _ = rotate_inputs(geo, seed)
    tag = f"seed {seed} {geo}"
    for interp, _ in INTERPS:
        got, xy = orot.rotate(img32.numpy(), geo["ang"], geo["ctr"], interp, return_index=True)
        want = rotate_f64(img32, torch.from_numpy(xy[..., 0]), torch.from_numpy(xy[..., 1]), interp)
        if interp == 1:
            assert torch.equal(torch.from_numpy(got), want["r"].float()), tag
        else:
            check(tag, "oracle out", torch.from_numpy(got), want, U32)
        assert_indices_near_ideal(tag, xy, geo["ang"], geo["ctr"])


# ---- GPU ---------------------------------------------------------------------------------------------------------------
def device_indices(ang, ctr, H, W):
    """b200_rotate_debug_indices for an fp32 angle and centre: [H, W, 2] float32 on the GPU."""
    out = torch.empty(H, W, 2, dtype=torch.float32, device="cuda")
    a, c = torch.tensor([ang], device="cuda"), torch.tensor(list(ctr), device="cuda")
    st = _lib.load().b200_rotate_debug_indices(a.data_ptr(), c.data_ptr(), (ctypes.c_int * 3)(1, H, W), out.data_ptr(),
                                               _lib.current_stream_ptr())  # fmt: skip
    _lib.check("b200_rotate_debug_indices", st)
    return out


def checked_indices(tag, ang, ctr, H, W):
    """The device's indices, checked against the C oracle (bit for bit, device trig) and the float64 position."""
    idx = device_indices(ang, ctr, H, W)
    got = idx.cpu().numpy()
    want = orot.source_indices(ang, ctr, H, W, trig=device_trig(ang))
    same = (got == want) | (np.isnan(got) & np.isnan(want))
    assert same.all(), (tag, "indices differ from the C oracle", int((~same).sum()), np.argwhere(~same)[0])
    assert_indices_near_ideal(tag, got, ang, ctr)


def _hwc_views(img):
    """[C, H, W] views of a dense [H, W, C] copy of ``img`` (as ``.view(H, W, C).permute(2, 0, 1)`` gives them, strides
    (1, W * C, C) even on a size-1 axis): one 16-byte aligned, one an element off alignment."""
    C, H, W = img.shape
    hwc = torch.empty(H, W, C, dtype=img.dtype, device=img.device)
    hwc.copy_(img.permute(1, 2, 0))
    buf = torch.empty(hwc.numel() + 1, dtype=img.dtype, device=img.device)
    off = buf[1:].view(H, W, C)
    off.copy_(hwc)
    return hwc.permute(2, 0, 1), off.permute(2, 0, 1)


def _runs(fn, kernel):
    """fn()'s result, checking from the kernel trace that the rotate kernel it ran is ``kernel``. The trace now and then
    loses a record: a trace that holds no rotate kernel at all leaves the identity unchecked."""
    out, names = kernels_recorded(fn, lambda ns: any(kernel in n for n in ns))
    ran = [n for n in names if "b200::rotate_" in n]
    assert not ran or any(kernel in n for n in ran), (kernel, ran)
    return out


def check_channels_last(tag, img, a, c, mode, planar):
    """``bt.rotate`` on a permuted channels-last view runs rotate_hwc_kernel and returns a view of a channels-last
    output; the same view an element off alignment runs rotate_planar_kernel; both return the planar entry's bits."""
    C, H, W = img.shape
    aligned, unaligned = _hwc_views(img)
    assert aligned.data_ptr() % 16 == 0 and unaligned.data_ptr() % 16 != 0
    o1 = _runs(lambda: bt.rotate(aligned, a, c, mode), "rotate_hwc_kernel")
    o2 = _runs(lambda: bt.rotate(unaligned, a, c, mode), "rotate_planar_kernel")
    assert o1.stride() == (1, W * C, C) and o2.is_contiguous(), (tag, o1.stride(), o2.stride())
    assert torch.equal(o1, planar), (tag, "channels-last kernel differs from the planar entry")
    assert torch.equal(o2, planar), (tag, "unaligned channels-last view differs from the planar entry")


def check_int8(tag, got_q, ent, interp, so):
    """got_q [C, H, W] int8 against the float64 entry ``ent`` in output steps (module docstring)."""
    q = got_q.to(torch.float64)
    r = ent["r"]
    if interp == 1:
        v = r.float().cpu().numpy()  # a copied fp32 product q * si, or 0
        want = orot.t2int8(v * (np.float32(1.0) / np.float32(so)))
        assert np.array_equal(got_q.cpu().numpy(), want), (tag, "int8 nearest", int((got_q.cpu().numpy() != want).sum()))
        return
    E = (8 + ent["n"]) * U32 * ent["mag"]
    t = r / so
    delta = (E + 2.0001 * U32 * r.abs()) / so * (1 + 2.0**-21) + 2.0**-17
    err = (q - t.clamp(-128, 127)).abs()
    bad = ~(err <= 0.5 + delta)
    if bool(bad.any()):
        i = int(bad.reshape(-1).nonzero()[0])
        raise AssertionError(f"{tag} int8: {int(bad.sum())} of {r.numel()} outside the bound; first at "
                             f"{np.unravel_index(i, tuple(r.shape))}: got {q.reshape(-1)[i].item()} want "
                             f"{t.reshape(-1)[i].item()!r} +- {0.5 + delta.reshape(-1)[i].item():.6f}")  # fmt: skip
    assert bool((q[t > 127 + delta] == 127).all()) and bool((q[t < -128 - delta] == -128).all()), (tag, "saturation")


def _case(seed, angle="f32"):
    """The drawn case on the GPU: geo, the three images, the angle and centre as the entries take them (``angle``:
    "f32" or "f16") and the device's source indices for them."""
    geo = rotate_geometry(seed)
    if angle == "f16" and not half_ok(geo):
        pytest.skip("the angle or centre has no finite FP16 value")
    ang, ctr = (geo["ang"], geo["ctr"]) if angle == "f32" else half_scalars(geo)
    dt = torch.float32 if angle == "f32" else torch.float16
    a, c = torch.tensor([ang], device="cuda").to(dt), torch.tensor(list(ctr), device="cuda").to(dt)
    idx = device_indices(ang, ctr, geo["H"], geo["W"])
    imgs = tuple(t.cuda() for t in rotate_inputs(geo, seed))
    return geo, imgs, a, c, idx[..., 0], idx[..., 1], f"seed {seed} {angle}-angle {geo}"


@pytest.mark.gpu
@pytest.mark.parametrize("angle", ["f32", "f16"])
@pytest.mark.parametrize("seed", SEEDS)
def test_source_indices(seed, angle):
    geo = rotate_geometry(seed)
    if angle == "f16" and not half_ok(geo):
        pytest.skip("the angle or centre has no finite FP16 value")
    ang, ctr = (geo["ang"], geo["ctr"]) if angle == "f32" else half_scalars(geo)
    checked_indices(f"seed {seed} {angle}-angle {geo}", ang, ctr, geo["H"], geo["W"])


@pytest.mark.gpu
@pytest.mark.parametrize("seed", SEEDS)
def test_fp32_rotate_and_rotate2(seed):
    geo, (img32, _, _), a, c, ix, iy, tag = _case(seed)
    for interp, mode in INTERPS:
        t = f"{tag} {mode}"
        want = rotate_f64(img32, ix, iy, interp)
        got = bt.rotate(img32, a, c, mode)
        if interp == 1:
            assert torch.equal(got, want["r"].float()), (t, "fp32 nearest")
        else:
            check(t, "fp32", got, want, U32)
        assert torch.equal(bt.rotate2(img32, a, c, mode), got), (t, "rotate2")
        if os.path.exists(REF_LIB):
            ref = orot.RefRotate().rotate(img32, a, c, interp)
            if interp == 1:
                assert torch.equal(ref, got), (t, "the reference kernel picks other pixels")
            else:
                check(t, "reference kernel", ref, want, U32)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", SEEDS)
def test_fp16_rotate_and_chw2(seed):
    geo, (_, img16, _), a, c, ix, iy, tag = _case(seed, "f16")
    C = geo["C"]
    h2 = pack_chw(img16[None], 2)[0]
    for interp, mode in INTERPS:
        t = f"{tag} {mode}"
        want = rotate_f64(img16, ix, iy, interp)
        got = bt.rotate(img16, a, c, mode)
        assert got.dtype == torch.float16
        if interp == 1:
            assert torch.equal(got, want["r"].half()), (t, "fp16 nearest")
        else:
            check(t, "fp16", got, want, U32)
        out2 = unpack_chw(bt.rotate_chw2(h2, C, a, c, mode)[None], C)[0]
        assert torch.equal(out2.view(torch.int16), got.view(torch.int16)), (t, "kCHW2")


@pytest.mark.gpu
@pytest.mark.parametrize("angle", ["f32", "f16"])
@pytest.mark.parametrize("seed", SEEDS)
def test_int8_chw4(seed, angle):
    geo, (_, _, q), a, c, ix, iy, tag = _case(seed, angle)
    C, si, so = geo["C"], geo["si"], geo["so"]
    real = q.float() * np.float32(si)  # the values the kernel blends
    q4 = pack_chw(q[None], 4)[0]
    for interp, mode in INTERPS:
        out4 = bt.rotate_int8(q4, si, C, a, c, so, mode)
        assert out4.dtype == torch.int8
        check_int8(f"{tag} {mode}", unpack_chw(out4[None], C)[0], rotate_f64(real, ix, iy, interp), interp, so)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["f32", "f16"])
@pytest.mark.parametrize("seed", SEEDS)
def test_channels_last(seed, dtype):
    geo = rotate_geometry(seed)
    if f"hwc_{dtype}" not in entries(geo):
        pytest.skip("C is not a whole number of 16-byte vectors, or the angle has no finite FP16 value")
    geo, (img32, img16, _), a, c, _, _, tag = _case(seed, dtype)
    img = img32 if dtype == "f32" else img16
    for _, mode in INTERPS:
        check_channels_last(f"{tag} {mode}", img, a, c, mode, bt.rotate(img, a, c, mode))
