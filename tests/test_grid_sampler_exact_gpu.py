"""The grid sampler (csrc/grid_sampler.cu) pinned bit for bit on exact probes, in every mode, format and dimension, and
at the launch geometry where a thread's channel slice is partial and where the grid-stride loop takes a second pass.

Checker: ``oracle.grid_sampler.grid_sample_np``, a numpy restatement of the kernel's semantics (channel-first grid over
[-10, 10], unnormalise, clip, reflect, safe, bilinear / trilinear, nearest rounding half away from zero, bicubic with
A = -0.75 and get_value_bounded) evaluated in float64. The CPU tests pin it against ATen in float64 (the reference
binding's own forward), against the float32 C oracle, and check that every probe is exact.

The exact probe: image values are small integers; grid values are multiples of 1/8 (of the int8 grid scale for INT8);
image sizes make size/10 (align_corners=False) or (size-1)/10 (align_corners=True) a power of two, or are 1. Every
grid value is kept only if its source coordinate is the same in float32 and float64 and lies on a 1/16 lattice (1/4
for bicubic, so the cubic coefficients are multiples of 2^-8). Then every float32 operation of the kernel is exact,
and any correct implementation produces the same bits in any operation order; a difference is a wrong tap, weight or
padding rule, not rounding. The float32 evaluation equalling the float64 one on every probe (test_probe_is_exact) is
what makes the GPU comparisons bit-exact; a probe that fails it is a wrong probe, not a reason to loosen a GPU test.

The probe grids hold, per axis: -10, 0 and +10; every integer source position (pixel centres with align_corners=False)
and every .5 tie from two pixels outside the image to two inside; points 1/16, 1/8 and 1/4 either side of -1, -0.5,
0, size-1, size-0.5 and size (the zeros-padding bounds of bilinear and nearest); values up to several image widths
out, so reflection flips many times; and seeded random lattice points."""
import ctypes
import functools
import itertools
import os

import numpy as np
import pytest
import torch

import bevformer_tensorrt_b200 as bt
from bevformer_tensorrt_b200.functions.grid_sampler import pack_chw, unpack_chw
from oracle import REF_LIB
from oracle import grid_sampler as ogs
from tests.helpers import make_grid_sampler_inputs

MODES = list(itertools.product(["bilinear", "nearest", "bicubic"], ["zeros", "border", "reflection"], [False, True]))
MODES_3D = [m for m in MODES if m[0] != "bicubic"]
IM = {"bilinear": 0, "nearest": 1, "bicubic": 2}
PM = {"zeros": 0, "border": 1, "reflection": 2}

# exact-probe image sizes (Hi, Wi) / (Di, Hi, Wi): size/10 resp. (size-1)/10 a power of two, and size-1 axes
SHAPES_2D = {False: [(10, 20), (40, 1), (1, 10)], True: [(11, 21), (41, 1), (1, 11)]}
SHAPES_3D = {False: [(10, 1, 20), (1, 20, 10)], True: [(11, 21, 1), (1, 11, 41)]}
TILE_SHAPE = (10, 40)  # Wi * 4 and Wi * 2 bytes are multiples of 16: the tile kernel's copies are legal in every format

# INT8 probe scales: powers of two, so dequantisation and v * (1 / so) are exact; so = si / 2 puts the +127 and -128
# pixels at +254 and -256 output steps (saturation) and makes odd half-sums land on .5 steps (requantisation ties)
SI, SO = 2.0**-3, 2.0**-4
SG = 2.0**-2  # int8 grid: multiples of 1/4 in [-32, 31.75]


# ---- probes ----------------------------------------------------------------------------------------------------------
def _axis_values(size, align, lattice, quantum=0.125, lim=64.0, dense=True, seed=0):
    """Sorted grid values for one axis: multiples of `quantum` with |g| <= lim whose source coordinate is equal in
    float32 and float64 and a multiple of 1/lattice (see the module docstring for what they hold). dense=False keeps
    integer positions and ties near the two edges only (3-D probes are outer products of three axes)."""
    S = size
    near = range(-2, S + 2) if dense else [k for k in range(-2, S + 2) if k <= 2 or k >= S - 3]
    xs = [float(k) for k in near] + [k + 0.5 for k in near if k <= S]
    ds = (-0.25, -0.125, -0.0625, 0.0625, 0.125, 0.25) if dense else (-0.0625, 0.0625)
    xs += [e + d for e in (-1, -0.5, 0, S - 1, S - 0.5, S) for d in ds]
    xs += [-3 * S - 0.25, -2 * S - 0.75, -7.25, 2 * S + 0.5, 3 * S + 0.5, 4 * S + 0.25]
    xs = np.array(xs)
    if align:
        gs = xs * 20 / (S - 1) - 10 if S > 1 else np.zeros(0)
    else:
        gs = (xs + 0.5) * 20 / S - 10
    rng = np.random.default_rng(seed + 97 * S + int(align))
    extra = [-10, 0, 10, -10 - quantum, -10 + quantum, 10 - quantum, 10 + quantum, -30, 30, -lim, lim]
    gs = np.concatenate([gs, extra, rng.integers(-lim / quantum, lim / quantum + 1, 24 if dense else 6) * quantum])
    gs = np.round(gs / quantum) * quantum
    gs = np.unique(gs[np.abs(gs) <= lim])
    x64 = ogs.unnormalize(gs, S, align, np.float64)
    x32 = ogs.unnormalize(gs.astype(np.float32), S, align, np.float32)
    keep = (x32.astype(np.float64) == x64) & (x64 * lattice == np.round(x64 * lattice))
    return gs[keep]


def _lattice(interp):
    return 4 if interp == "bicubic" else 16


def _image(shape, C, seed, lo=-15, hi=15):
    return np.random.default_rng(seed).integers(lo, hi + 1, (2, C, *shape)).astype(np.float64)


def _outer_grid(axes):
    """[2, len(axes), len(a_last)..., ] channel-first grid over the outer product of per-axis values (x, y[, z]) for
    two images: the second image's grid is the first one's reversed along every output axis."""
    mesh = np.meshgrid(*axes[::-1], indexing="ij")[::-1]  # output axes (Do,) Ho, Wo carry z, y, x
    g = np.stack(mesh, 0)[None]
    flip = tuple(range(2, g.ndim))
    return np.concatenate([g, np.flip(g, flip)], 0).copy()


@functools.lru_cache(maxsize=None)
def probe_2d(shape, align, interp, C=3, quantum=0.125, lim=64.0):
    """(image [2, C, Hi, Wi], grid [2, 2, Ho, Wo]) float64 with small-integer pixels and an outer-product grid."""
    H, W = shape
    lat = _lattice(interp)
    axes = [_axis_values(W, align, lat, quantum, lim), _axis_values(H, align, lat, quantum, lim, seed=1)]
    return _image(shape, C, seed=H * 100 + W), _outer_grid(axes)


@functools.lru_cache(maxsize=None)
def probe_3d(shape, align):
    D, H, W = shape
    axes = [_axis_values(s, align, 16, dense=False, seed=i) for i, s in enumerate((W, H, D))]
    return _image(shape, 2, seed=D * 10000 + H * 100 + W), _outer_grid(axes)


@functools.lru_cache(maxsize=None)
def probe_int8(shape, align, interp):
    """(quantised image [2, 6, Hi, Wi] in int8 range, grid in units of SG): pixels mostly in [-40, 40] with +127 and
    -128 pixels so that outputs saturate at both ends."""
    q, grid = probe_2d(shape, align, interp, C=6, quantum=SG, lim=127 * SG)
    q = np.random.default_rng(5).integers(-40, 41, q.shape).astype(np.float64)
    flat = q.reshape(-1)
    pick = np.random.default_rng(6).permutation(flat.size)
    flat[pick[: max(2, flat.size // 16)]] = 127.0
    flat[pick[flat.size // 16 : flat.size // 8 + 1]] = -128.0
    return q, grid / SG


@functools.lru_cache(maxsize=None)
def probe_tile():
    """The smooth grid the tile kernel stages in shared memory (a quarter-pixel x step and a 5/8-pixel y step from
    1.5 pixels left of / 1.25 above the image to past its far edges), on TILE_SHAPE with align_corners=False; the
    second image's grid is shifted by (3/4, 5/16) pixels. Multiples of 1/8, so the INT8 grid uses a 1/8 scale."""
    H, W = TILE_SHAPE
    x = -1.5 + 0.25 * np.arange(180)
    y = -1.25 + 0.625 * np.arange(20)
    g = []
    for dx, dy in ((0.0, 0.0), (0.75, 0.3125)):
        gx, gy = (x + dx + 0.5) * 20 / W - 10, (y + dy + 0.5) * 20 / H - 10
        g.append(np.stack(np.meshgrid(gx, gy, indexing="xy"), 0))
    return _image(TILE_SHAPE, 37, seed=77), np.stack(g, 0)


def _requant(real, so):
    """T2int8 of the reference: saturate to [-128, 127], round half away from zero."""
    return ogs.round_half_away(np.clip(real / so, -128, 127)).astype(np.int8)


def _expect(inp, grid, interp, pad, align):
    return ogs.grid_sample_np(inp, grid, IM[interp], PM[pad], align)


# ---- 1. the float64 restatement, pinned on the CPU -------------------------------------------------------------------
def _near_tie(grid, sizes, align, px=1e-9):
    """Mask of output points whose float64 source coordinate on any axis is within px of a .5 tie: there ATen's
    nearest (nearbyint, half to even) and the reference's (::round, half away from zero) may differ. Padding maps a
    coordinate by reflections about integers or half-integers, or clips it to an integer, so a tie after padding is a
    tie before it."""
    near = np.zeros(grid[:, 0].shape, bool)
    for axis, size in enumerate(sizes):  # grid planes x, y[, z] against Wi, Hi[, Di]
        x = ogs.unnormalize(grid[:, axis], size, align, np.float64)
        near |= np.abs(x - np.floor(x) - 0.5) < px
    return near


@pytest.mark.parametrize("interp,pad,align", MODES + [("3d_" + i, p, a) for i, p, a in MODES_3D])
def test_restatement_matches_aten_float64(interp, pad, align):
    """Against aten.grid_sampler in float64 on grid / 10 (the reference binding's forward), on random images and on
    random grids as well as on the exact probes, at sizes with 1 on every axis. Nearest is compared away from .5
    ties only: the kernel rounds half away from zero like the reference's ::round, ATen half to even (a deliberate,
    documented difference: at x = -0.5, grid value -10 with align_corners=False, the kernel samples nothing under
    zeros padding where ATen samples pixel 0)."""
    three = interp.startswith("3d_")
    interp = interp[3:] if three else interp
    rng = np.random.default_rng(11)
    if three:
        shapes = [(1, 4, 5), (3, 1, 5), (3, 4, 1), (1, 1, 1)]
        cases = [(rng.standard_normal((2, 3, *s)), rng.uniform(-25, 25, (2, 3, 3, 4, 5))) for s in shapes]
        cases += [probe_3d(s, align) for s in SHAPES_3D[align]]
    else:
        shapes = [(1, 7), (6, 1), (1, 1), (6, 9)]
        cases = [(rng.standard_normal((2, 3, *s)), rng.uniform(-25, 25, (2, 2, 8, 9))) for s in shapes]
        cases += [probe_2d(s, align, interp) for s in SHAPES_2D[align]]
    for inp, grid in cases:
        want = ogs.grid_sampler_torch_port(torch.from_numpy(inp), torch.from_numpy(grid), IM[interp], PM[pad],
                                           align).numpy()  # fmt: skip
        d = np.abs(_expect(inp, grid, interp, pad, align) - want)
        if interp == "nearest":
            d = d[~np.broadcast_to(_near_tie(grid, inp.shape[:1:-1], align)[:, None], d.shape)]
        assert d.max() < 1e-9, (inp.shape, d.max())


@pytest.mark.parametrize("interp,pad,align", MODES)
def test_restatement_matches_c_oracle(interp, pad, align):
    """Against the float32 C oracle on the random sweep inputs of tests/test_grid_sampler_gpu.py: float64 within 1e-5;
    the float32 evaluation (same formulas, same roundings) within 1e-5 with identical nearest taps."""
    inp, grid = make_grid_sampler_inputs(2, 7, 11, 13, 23, 19, seed=5)
    inp, grid = inp.numpy(), grid.numpy()
    want = ogs.grid_sample_2d(inp, grid, IM[interp], PM[pad], align)
    assert np.abs(_expect(inp, grid, interp, pad, align) - want).max() < 1e-5
    f32 = ogs.grid_sample_np(inp, grid, IM[interp], PM[pad], align, np.float32)
    assert np.abs(f32 - want).max() < 1e-5
    if interp == "nearest":
        assert np.array_equal(f32, want)


def _assert_exact_in_f32(inp, grid, interp, pad, align):
    f64 = _expect(inp, grid, interp, pad, align)
    f32 = ogs.grid_sample_np(inp, grid, IM[interp], PM[pad], align, np.float32)
    bad = f32.astype(np.float64) != f64
    assert not bad.any(), (inp.shape, grid.shape, int(bad.sum()))
    return f64


@pytest.mark.parametrize("interp,pad,align", MODES)
def test_probe_is_exact(interp, pad, align):
    """Every probe the GPU tests use: the float32 evaluation equals the float64 one exactly, so the float64 result is
    what a correct kernel produces in any operation order. Also checks that the probes hold what they claim: the
    grid values -10, 0 and +10, the zeros-padding bounds, ties, size-1 axes, and for INT8 saturation at both ends and
    requantisation ties of both signs."""
    ties = set()
    for shape in SHAPES_2D[align]:
        inp, grid = probe_2d(shape, align, interp)
        _assert_exact_in_f32(inp, grid, interp, pad, align)
        assert {-10.0, 0.0, 10.0} <= set(grid[0, 0, 0]) and {-10.0, 0.0, 10.0} <= set(grid[0, 1, :, 0])
        for axis, size in enumerate(shape[::-1]):
            x = set(ogs.unnormalize(grid[0, axis], size, align, np.float64).reshape(-1))
            if size > 1 or not align:
                edges = {-1.0, 0.0, size - 1.0, float(size)} | ({-0.5, size - 0.5} if interp != "bicubic" else set())
                assert edges <= x, (shape, axis, sorted(edges - x))
                assert any(v % 1 == 0.5 for v in x) and min(x) < -size and max(x) > 2 * size
        q, g = probe_int8(shape, align, interp)
        real = _assert_exact_in_f32(q * SI, g * SG, interp, pad, align)
        assert np.abs(g).max() <= 128 and np.abs(q).max() <= 128
        steps = real / SO
        assert (steps > 127).any() and (steps < -128).any(), (shape, steps.max(), steps.min())
        half = np.abs(steps - np.trunc(steps)) == 0.5
        ties |= set(np.sign(steps[half]))
    assert interp == "nearest" or ties == {1.0, -1.0}  # nearest outputs are 2 q: whole steps
    if interp != "bicubic":
        for shape in SHAPES_3D[align]:
            _assert_exact_in_f32(*probe_3d(shape, align), interp, pad, align)
    if interp == "bilinear" and not align:
        inp, grid = probe_tile()
        _assert_exact_in_f32(inp, grid, interp, pad, align)
        assert (np.abs(grid) * 8 % 1 == 0).all() and np.abs(grid).max() < 16
        _assert_exact_in_f32(*probe_2d(TILE_SHAPE, False, "bilinear", C=37), interp, pad, align)
        _assert_exact_in_f32(*probe_2d((10, 20), False, "bilinear", C=1), interp, pad, align)


# ---- the launch plan, restated (launch_gs) ---------------------------------------------------------------------------
_MAX_BLOCKS, _BLOCK = 1 << 22, 256


def _slice_plan(pixels, cp, cap=64):
    """(slices, packets per slice) that launch_gs picks: double the slices until about two waves of 132 SMs x 1024
    threads are busy and no thread handles more than `cap` packets."""
    slices = 1
    while slices < cp and (pixels * slices < 132 * 1024 * 2 or -(-cp // slices) > cap):
        slices <<= 1
    cps = -(-cp // slices)
    return -(-cp // cps), cps


SLICE_PIXELS = (3, 300, 302)  # N, Ho, Wo: 271800 output pixels, more than two waves on their own
SLICE_CASES = {"fp32": 130, "fp16": 130, "chw2": 259, "int8_c517": 517, "int8_c518": 518, "int8_c519": 519}
STRIDE_SHAPE = (32769, 32768)  # Ho, Wo: 2^30 + 2^15 pixels, N = C = 1


def test_launch_plan_reaches_partial_slices_and_a_second_pass():
    """The slicing shapes make the 64-packet cap bind (without it one slice would do) and leave a partial last slice
    of 31 packets; the grid-stride shape needs more threads than the 2^22-block cap launches in one pass."""
    n, ho, wo = SLICE_PIXELS
    for name, c in SLICE_CASES.items():
        cp = -(-c // {"chw2": 2}.get(name, 4 if name.startswith("int8") else 1))
        assert cp == 130
        slices, cps = _slice_plan(n * ho * wo, cp)
        assert (slices, cps, cp - (slices - 1) * cps) == (4, 33, 31)
        assert _slice_plan(n * ho * wo, cp, cap=1 << 30) == (1, 130)
    pixels = STRIDE_SHAPE[0] * STRIDE_SHAPE[1]
    slices, _ = _slice_plan(pixels, 1)
    total = pixels * slices
    blocks = min(total // _BLOCK + 1, _MAX_BLOCKS)
    assert blocks * _BLOCK == 1 << 30 < total < 1 << 31


# ---- 2. exact probes on the GPU --------------------------------------------------------------------------------------
def _same_bits(got, want):
    got = got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else got
    assert got.shape == want.shape and got.dtype == want.dtype, (got.shape, want.shape, got.dtype, want.dtype)
    bits = {1: np.uint8, 2: np.uint16, 4: np.uint32}[got.dtype.itemsize]
    bad = got.view(bits) != want.view(bits)
    if bad.any():
        i = tuple(int(v[0]) for v in np.nonzero(bad))
        raise AssertionError(f"{int(bad.sum())} of {bad.size} differ; first at {i}: got {got[i]}, want {want[i]}")


def _grid_shapes(grid):
    """The probe grid as given and with every point on one output row (Ho = 1) or one column (Wo = 1)."""
    n, k = grid.shape[0], grid[0, 0].size
    return [grid, grid.reshape(n, 2, 1, k), grid.reshape(n, 2, k, 1)]


def _ref_lib():
    if not os.path.exists(REF_LIB):
        return None
    lib = ctypes.CDLL(REF_LIB)
    ip = ctypes.POINTER(ctypes.c_int)
    vp = ctypes.c_void_p
    lib.ref_grid_sample.argtypes = [ctypes.c_int] + [vp] * 3 + [ip] * 3 + [ctypes.c_int] * 4 + [vp]
    lib.ref_grid_sample.restype = None
    return lib


def _ref_grid_sample_f32(lib, inp, grid, interp, pad, align):
    out = torch.empty(inp.shape[0], inp.shape[1], *grid.shape[2:], device="cuda")
    dims = lambda t: (ctypes.c_int * 4)(*t.shape)  # noqa: E731
    lib.ref_grid_sample(0, out.data_ptr(), inp.data_ptr(), grid.data_ptr(), dims(out), dims(inp), dims(grid), 4,
                        IM[interp], PM[pad], int(align), torch.cuda.current_stream().cuda_stream)  # fmt: skip
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("interp,pad,align", MODES)
def test_fp32_probe_bit_exact(interp, pad, align):
    """grid_sampler and grid_sampler2 (FP32) equal the float64 result as float32, on every probe shape and with one
    output row or column; so does the reference's own grid_sample<float> kernel where oracle/_ref was built."""
    ref = _ref_lib()
    for shape in SHAPES_2D[align]:
        inp, grid = probe_2d(shape, align, interp)
        want = _expect(inp, grid, interp, pad, align).astype(np.float32)
        x = torch.from_numpy(inp).float().cuda()
        for g in _grid_shapes(grid):
            gd = torch.from_numpy(g).float().cuda()
            w = want.reshape(want.shape[:2] + g.shape[2:])
            for fn in (bt.grid_sampler, bt.grid_sampler2):
                _same_bits(fn(x, gd, interp, pad, align), w)
            if ref is not None:
                _same_bits(_ref_grid_sample_f32(ref, x, gd, interp, pad, align), w)


@pytest.mark.gpu
@pytest.mark.parametrize("interp,pad,align", MODES)
def test_fp16_probe_bit_exact(interp, pad, align):
    """FP16 kLINEAR (grid_sampler) and kCHW2 (grid_sampler_chw2, 3 channels: a half-empty last packet) equal the
    float64 result rounded once to half: the probe's fp32 accumulation is exact, so the output rounding is the only
    one."""
    for shape in SHAPES_2D[align]:
        inp, grid = probe_2d(shape, align, interp)
        want = _expect(inp, grid, interp, pad, align).astype(np.float16)
        x = torch.from_numpy(inp).half()
        x2 = pack_chw(x, 2).cuda()
        for g in _grid_shapes(grid):
            gh = torch.from_numpy(g).half()
            w = want.reshape(want.shape[:2] + g.shape[2:])
            _same_bits(bt.grid_sampler(x.cuda(), gh.cuda(), interp, pad, align), w)
            g2 = gh.permute(0, 2, 3, 1).unsqueeze(1).contiguous().cuda()
            out2 = bt.grid_sampler_chw2(x2, g2, inp.shape[1], interp, pad, align)
            _same_bits(unpack_chw(out2.cpu(), inp.shape[1]), w)


def _grid_chw4(gq):
    g4 = torch.zeros(gq.shape[0], 1, gq.shape[2], gq.shape[3], 4, dtype=torch.int8)
    g4[:, 0, :, :, 0], g4[:, 0, :, :, 1] = gq[:, 0], gq[:, 1]
    return g4


@pytest.mark.gpu
@pytest.mark.parametrize("interp,pad,align", MODES)
def test_int8_probe_bit_exact(interp, pad, align):
    """INT8 kCHW4 (grid_sampler_int8, 6 channels: a half-empty last packet) equals round_half_away(clamp(real / so,
    -128, 127)) of the float64 result on the dequantised tensors, with outputs saturating at +127 and -128 and
    landing on .5 steps (test_probe_is_exact checks that they do)."""
    for shape in SHAPES_2D[align]:
        q, g = probe_int8(shape, align, interp)
        want = _requant(_expect(q * SI, g * SG, interp, pad, align), SO)
        x4 = pack_chw(torch.from_numpy(q).to(torch.int8), 4).cuda()
        for gs in _grid_shapes(g):
            g4 = _grid_chw4(torch.from_numpy(gs).to(torch.int8)).cuda()
            out = bt.grid_sampler_int8(x4, SI, g4, SG, SO, q.shape[1], interp, pad, align)
            _same_bits(unpack_chw(out.cpu(), q.shape[1]), want.reshape(want.shape[:2] + gs.shape[2:]))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["fp32", "fp16"])
@pytest.mark.parametrize("interp,pad,align", MODES_3D)
def test_3d_probe_bit_exact(interp, pad, align, dtype):
    """GridSampler3D (trilinear and nearest, FP32 and FP16 kLINEAR) on outer-product probes over depth, height and
    width, with a size-1 axis in every shape."""
    tt, nt = (torch.float32, np.float32) if dtype == "fp32" else (torch.float16, np.float16)
    for shape in SHAPES_3D[align]:
        inp, grid = probe_3d(shape, align)
        want = _expect(inp, grid, interp, pad, align).astype(nt)
        got = bt.grid_sampler(torch.from_numpy(inp).to(tt).cuda(), torch.from_numpy(grid).to(tt).cuda(), interp, pad,
                              align)  # fmt: skip
        _same_bits(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("pad", ["zeros", "border", "reflection"])
@pytest.mark.parametrize("mode", [1, 2])
def test_tile_path_probe_bit_exact(mode, pad):
    """2-D bilinear through the opt-in tile kernel (b200_grid_sample_set_tile_path: 1 = bulk copy per row, 2 = one
    tensor copy per channel packet) in every format, on a smooth grid whose source windows fit in shared memory and
    on the outer-product probe whose windows do not (the per-tile fallback). 37 channels leave a partial channel
    block; the previous tile mode is restored afterwards."""
    lib = bt._lib.load()
    prev = lib.b200_grid_sample_set_tile_path(mode)
    try:
        for inp, grid in (probe_tile(), probe_2d(TILE_SHAPE, False, "bilinear", C=37)):
            want = _expect(inp, grid, "bilinear", pad, False)
            C = inp.shape[1]
            x, gd = torch.from_numpy(inp), torch.from_numpy(grid)
            _same_bits(bt.grid_sampler(x.float().cuda(), gd.float().cuda(), "bilinear", pad, False),
                       want.astype(np.float32))  # fmt: skip
            _same_bits(bt.grid_sampler(x.half().cuda(), gd.half().cuda(), "bilinear", pad, False),
                       want.astype(np.float16))  # fmt: skip
            g2 = gd.half().permute(0, 2, 3, 1).unsqueeze(1).contiguous().cuda()
            out2 = bt.grid_sampler_chw2(pack_chw(x.half(), 2).cuda(), g2, C, "bilinear", pad, False)
            _same_bits(unpack_chw(out2.cpu(), C), want.astype(np.float16))
            if np.abs(grid).max() < 16:  # int8 grid at a 1/8 scale
                sg = 0.125
                real = _expect(inp * SI, grid, "bilinear", pad, False)
                g4 = _grid_chw4(torch.from_numpy(grid / sg).to(torch.int8)).cuda()
                x4 = pack_chw(x.to(torch.int8), 4).cuda()
                out4 = bt.grid_sampler_int8(x4, SI, g4, sg, SO, C, "bilinear", pad, False)
                _same_bits(unpack_chw(out4.cpu(), C), _requant(real, SO))
    finally:
        lib.b200_grid_sample_set_tile_path(prev)


# ---- 3. launch geometry ----------------------------------------------------------------------------------------------
def _subset(n_images, ho, wo, k, seed):
    """A fixed random set of k output pixels per image, as (row, column) index arrays [n_images, k]."""
    rng = np.random.default_rng(seed)
    flat = np.stack([rng.choice(ho * wo, k, replace=False) for _ in range(n_images)])
    return flat // wo, flat % wo


def _oracle_at(inp, grid, rows, cols, interp=0, pad=0, align=False):
    """The C oracle at the chosen pixels only: an output depends on its own grid point alone, so image n is sampled at
    grid[n, :, rows[n], cols[n]] laid out as one output row. Returns [N, C, k]."""
    outs = []
    for n in range(inp.shape[0]):
        g = np.ascontiguousarray(grid[n][:, rows[n], cols[n]][None, :, None, :])
        outs.append(ogs.grid_sample_2d(inp[n : n + 1], g, interp, pad, align)[0, :, 0])
    return np.stack(outs)


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(SLICE_CASES))
def test_partial_channel_slice(case):
    """130 channel packets over 271800 output pixels: the 64-packet cap splits each pixel into 4 slices of 33 packets,
    the last holding 31. Three images with different grids; kCHW2 with an odd channel count and kCHW4 with 1, 2 and 3
    channels in the last packet. Every channel at 4096 fixed pixels per image against the C oracle at the tolerances of
    tests/test_grid_sampler_gpu.py."""
    C = SLICE_CASES[case]
    N, Ho, Wo = SLICE_PIXELS
    inp, grid = make_grid_sampler_inputs(N, C, 23, 29, Ho, Wo, seed=41, span=12.0)
    grid[1] = grid[1].flip(1, 2)
    grid[2] = grid[2] * 0.5 + 1.5
    rows, cols = _subset(N, Ho, Wo, 4096, seed=42)
    pick = lambda out: np.stack([out[n][:, rows[n], cols[n]] for n in range(N)])  # noqa: E731
    if case == "fp32":
        want = _oracle_at(inp.numpy(), grid.numpy(), rows, cols)
        got = pick(bt.grid_sampler(inp.cuda(), grid.cuda(), "bilinear", "zeros", False).cpu().numpy())
        assert np.abs(got - want).max() < 1e-5
    elif case in ("fp16", "chw2"):
        ih, gh = inp.half(), grid.half()
        want = _oracle_at(ih.float().numpy(), gh.float().numpy(), rows, cols)
        if case == "fp16":
            out = bt.grid_sampler(ih.cuda(), gh.cuda(), "bilinear", "zeros", False).cpu()
        else:
            g2 = gh.permute(0, 2, 3, 1).unsqueeze(1).contiguous().cuda()
            out = unpack_chw(bt.grid_sampler_chw2(pack_chw(ih, 2).cuda(), g2, C, "bilinear", "zeros", False).cpu(), C)
        got = pick(out.float().numpy())
        assert np.abs(got - want).max() < 1e-3 + np.abs(want).max() * 2.0**-11
    else:
        iq = torch.randint(-128, 128, inp.shape, generator=torch.Generator().manual_seed(43), dtype=torch.int8)
        si, sg = 0.03, 12.0 / 127
        gq = torch.round(grid / sg).clamp(-128, 127).to(torch.int8)
        real = _oracle_at(iq.float().numpy() * si, gq.float().numpy() * sg, rows, cols)
        so = 128 * si / 127  # a bilinear sample is a convex combination of pixels: nothing saturates
        out = bt.grid_sampler_int8(pack_chw(iq, 4).cuda(), si, _grid_chw4(gq).cuda(), sg, so, C, "bilinear", "zeros",
                                   False)  # fmt: skip
        got = pick(unpack_chw(out.cpu(), C).float().numpy()) * so
        assert np.abs(got - real).max() <= 0.5 * so + 1e-6


@pytest.mark.gpu
def test_grid_stride_second_pass():
    """FP16 bilinear over 2^30 + 2^15 output pixels (N = C = 1), more than the 2^22 blocks x 256 threads of one pass:
    the last output row is written by the grid-stride loop's second pass. The grid repeats the exact probe values of a
    (10, 20) image along x and y; 2048 fixed pixels from the first pass and 2048 from the second equal the float64
    result rounded to half."""
    Ho, Wo = STRIDE_SHAPE
    need = 2 * 2 * Ho * Wo + 2 * Ho * Wo + (256 << 20)  # fp16 grid and output, plus slack
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free")
    inp, _ = probe_2d((10, 20), False, "bilinear", C=1)
    inp = inp[:1]
    xs = _axis_values(20, False, 16)
    ys = _axis_values(10, False, 16, seed=1)
    gx = xs[np.random.default_rng(1).integers(0, xs.size, Wo)]
    gy = ys[np.random.default_rng(2).integers(0, ys.size, Ho)]
    grid = out = None
    try:
        grid = torch.empty(1, 2, Ho, Wo, dtype=torch.float16, device="cuda")
        grid[0, 0].copy_(torch.from_numpy(gx).half().cuda().expand(Ho, Wo))
        grid[0, 1].copy_(torch.from_numpy(gy).half().cuda()[:, None].expand(Ho, Wo))
        out = bt.grid_sampler(torch.from_numpy(inp).half().cuda(), grid, "bilinear", "zeros", False)
        rng = np.random.default_rng(3)
        one_pass = _MAX_BLOCKS * _BLOCK
        first = rng.choice(one_pass, 2048, replace=False)
        second = one_pass + rng.choice(Ho * Wo - one_pass, 2048, replace=False)
        flat = np.concatenate([first, second])
        r, c = flat // Wo, flat % Wo
        got = out[0, 0].reshape(-1)[torch.from_numpy(flat).cuda()].cpu().numpy()
    finally:
        del grid, out
        torch.cuda.empty_cache()
    sub = np.stack([gx[c], gy[r]], 0)[None, :, None, :]
    want = _expect(inp, sub, "bilinear", "zeros", False).astype(np.float16)[0, 0, 0]
    _same_bits(got, want)
