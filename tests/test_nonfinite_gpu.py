"""Non-finite inputs to the sampling kernels (pytest -m gpu): grid sampler, rotate, MSDA, DCN.

Every forward sampler keeps its inner loop branch-free by giving a bilinear tap that falls outside the image a clamped,
in-image address (a sample that is out of range altogether used to read element 0 of the plane / head slice) and
weight 0. 0 * Inf and 0 * NaN are NaN, and the reference kernels never load such a tap, so a drop-in must not let one
overflowed FP16 activation at the aliased address reach every output that has an out-of-range tap. The contract held
here: a tap outside the image contributes an exact 0 whatever the tensor holds, and a non-finite coordinate is an
out-of-range sample.

Group A (value containment). One element of the sampled tensor is replaced by +Inf, -Inf or NaN (one kind per run).
The CPU oracle is run three times on the same tensors — clean, poisoned, and "bumped" (the element replaced by a
different finite value) — and every output element falls into one of three sets:
  MUST  clean != bumped: a tap with non-zero weight reads the element -> the device output must be non-finite;
  MAY   the oracle's poisoned output is non-finite without being in MUST: only in-image taps of weight exactly 0 touch
        the element, where the reference itself computes 0 * Inf -> either result is accepted;
  rest  -> the device output must be bit-identical to the device's own output on the clean tensor.
Inf versus NaN is not asserted: on an element that is poisoned anyway the aliased dummy loads may turn the reference's
Inf into NaN. Expected sets never come from the device.

Group B (non-finite coordinate, finite values). NaN, +Inf, -Inf and a huge finite value are planted in the sampling
grid, the MSDA reference points / offsets, the DCN offsets / mask and the rotate angle / centre. The affected outputs
are compared with the reference's CUDA semantics written out below (for the grid sampler: the finite coordinate the
reference's clip / safe_downgrade_to_int_range rules turn the planted one into, evaluated by the oracle; the C oracles
themselves are not trusted with a NaN -> int cast); everything else must be bit-identical to the clean run.
"""
import itertools

import numpy as np
import pytest
import torch

import bevformer_tensorrt_b200 as bt
from bevformer_tensorrt_b200 import _lib
from bevformer_tensorrt_b200.functions.grid_sampler import pack_chw, unpack_chw
from bevformer_tensorrt_b200.functions.modulated_deformable_conv2d import modulated_deformable_conv2d_chw2
from bevformer_tensorrt_b200.workloads import CONFIGS, MSDAConfig, make_msda_inputs
from oracle import dcn as odcn
from oracle import grid_sampler as ogs
from oracle import msda as omsda
from oracle import rotate as orot
from tests.helpers import make_dcn_inputs, make_grid_sampler_inputs
from tests.test_grid_sampler_gpu import _tile_grid
from tests.test_rotate_gpu import device_trig

pytestmark = pytest.mark.gpu

POISON = {"+inf": np.inf, "-inf": -np.inf, "nan": np.nan}
BUMP = 37.0
IM = {"bilinear": 0, "nearest": 1, "bicubic": 2}
PM = {"zeros": 0, "border": 1, "reflection": 2}


def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.float16 else torch.int32).numpy()


def check_containment(oracle, device, x, idx, oob=None, untouched=None, may_be_unread=False):
    """``oracle(x) -> ndarray`` and ``device(x) -> CPU tensor`` of the same shape, ``x`` a float32 ndarray already
    rounded to the storage type, ``idx`` the element(s) to poison. ``oob``: outputs known to have an out-of-range tap
    (the rest set must contain some, or the case proves nothing); ``untouched``: outputs no poisoned element can reach
    at all (other heads), which must be in the rest set; ``may_be_unread``: the sampling pattern is fixed by the path under
    test and need not reach the element (then only dummy taps can, and nothing may change)."""
    clean = oracle(x)
    bumped = x.copy()
    bumped[idx] += BUMP
    must = clean != oracle(bumped)
    assert must.any() or may_be_unread, "no output reads the poisoned element with a non-zero weight"
    dev_clean = device(x)
    assert torch.isfinite(dev_clean).all()
    for kind, v in POISON.items():
        xp = x.copy()
        xp[idx] = v
        with np.errstate(invalid="ignore", over="ignore"):
            bad = ~np.isfinite(oracle(xp))
        assert bad[must].all(), kind
        rest = ~(must | bad)
        assert rest.any(), kind
        if oob is not None:
            assert (rest & oob).any(), "no unaffected output has an out-of-range tap"
        if untouched is not None:
            assert rest[untouched].all()
        got = device(xp)
        assert got.shape == dev_clean.shape == clean.shape
        nonfinite = ~torch.isfinite(got).numpy()
        assert nonfinite[must].all(), (kind, int((~nonfinite & must).sum()))
        same = _bits(got) == _bits(dev_clean)
        assert same[rest].all(), (kind, int((~same & rest).sum()), int(rest.sum()))


def check_planted(want, dev_clean, got, affected, tol):
    """Group B: ``want`` (ndarray, NaN where the reference gives NaN) on the affected outputs, clean bits elsewhere."""
    assert got.shape == dev_clean.shape == want.shape and affected.any() and not affected.all()
    same = _bits(got) == _bits(dev_clean)
    assert same[~affected].all(), int((~same & ~affected).sum())
    g, w = got.float().numpy()[affected], want[affected]
    assert (np.isnan(g) == np.isnan(w)).all(), (int(np.isnan(g).sum()), int(np.isnan(w).sum()))
    ok = ~np.isnan(w)
    assert np.isfinite(g[ok]).all()
    if ok.any():
        assert np.abs(g[ok] - w[ok]).max() < tol, np.abs(g[ok] - w[ok]).max()


# ---------------------------------------------------------------------------------------------------------------
# grid sampler
# ---------------------------------------------------------------------------------------------------------------
GS_SHAPE = (2, 7, 11, 13, 23, 19)  # N, C (odd: the last channel sits alone in a kCHW2 packet), Hi, Wi, Ho, Wo


def _gs_inputs(fmt, seed, shape=GS_SHAPE, depth=None):
    """The reference test's sweep 1.5x beyond the image plus jitter (out-of-range samples and samples straddling every
    border), and a few samples at exact coordinates: grid 0 is an integer source index for odd sizes (in-image taps of
    weight exactly 0), +-10 the image edge."""
    inp, grid = make_grid_sampler_inputs(*shape, seed=seed, depth=depth)
    sp = grid.shape[2:]
    grid[(slice(None), slice(None)) + tuple(s // 2 for s in sp)] = 0.0
    grid[(slice(None), slice(None)) + tuple(s // 3 for s in sp)] = 0.0
    grid[(slice(None), 0) + tuple(s // 4 for s in sp)] = -10.0
    grid[(slice(None), 1) + tuple(s // 5 for s in sp)] = 10.0
    if fmt != "f32":
        inp, grid = inp.half().float(), grid.half().float()
    return inp.numpy(), grid


def _gs_device(fmt, grid, interp, pad, align):
    if fmt == "f32":
        g = grid.cuda()
        return lambda x: bt.grid_sampler(torch.from_numpy(x).cuda(), g, interp, pad, align).cpu()
    if fmt == "f16":
        g = grid.half().cuda()
        return lambda x: bt.grid_sampler(torch.from_numpy(x).half().cuda(), g, interp, pad, align).cpu()
    g2 = grid.half().permute(0, 2, 3, 1).unsqueeze(1).contiguous().cuda()  # kCHW2: [N, 1, Ho, Wo, 2] = (x, y)

    def run(x):
        c = x.shape[1]
        out = bt.grid_sampler_chw2(pack_chw(torch.from_numpy(x).half(), 2).cuda(), g2, c, interp, pad, align)
        return unpack_chw(out.cpu(), c)

    return run


def _gs_oracle(grid, interp, pad, align):
    if grid.dim() == 4:
        g = grid.numpy()
        return lambda x: ogs.grid_sample_2d(x, g, IM[interp], PM[pad], align)
    # 3-D: ATen's CPU kernel (what the reference binding calls), which loads a corner only if it is inside the volume
    return lambda x: ogs.grid_sampler_torch_port(torch.from_numpy(x), grid, IM[interp], PM[pad], align).numpy()


def _plane_positions(shape):
    """(a) flat element 0 of a plane, the address a dummy tap uses; (b) its last element, the far clamped corner;
    (c) an interior element next to the exact-coordinate samples (their zero-weight in-image tap)."""
    last = tuple(s - 1 for s in shape)
    mid = tuple(s // 2 for s in shape[:-1]) + (shape[-1] // 2 + 1,)
    return {"first": tuple(0 for _ in shape), "last": last, "interior": mid}


def _gs_containment(fmt, interp, pad, align, pos, seed, shape=GS_SHAPE, depth=None, grid=None, may_be_unread=False):
    x, g = _gs_inputs(fmt, seed, shape, depth)
    g = g if grid is None else (grid if fmt == "f32" else grid.half().float())
    oracle, device = _gs_oracle(g, interp, pad, align), _gs_device(fmt, g, interp, pad, align)
    oob = None
    if pad == "zeros" and interp == "bilinear":
        oob = np.broadcast_to(oracle(np.ones_like(x))[:, -1:] < 0.999, oracle(x).shape)
    idx = (slice(None), x.shape[1] - 1) + _plane_positions(x.shape[2:])[pos]
    check_containment(oracle, device, x, idx, oob, may_be_unread=may_be_unread)


@pytest.mark.parametrize("pos", ["first", "last", "interior"])
@pytest.mark.parametrize("pad,align", list(itertools.product(["zeros", "border", "reflection"], [False, True])))
@pytest.mark.parametrize("fmt", ["f32", "f16", "chw2"])
def test_grid_sampler_2d_bilinear_contains_a_poisoned_pixel(fmt, pad, align, pos):
    _gs_containment(fmt, "bilinear", pad, align, pos, seed=41)


@pytest.mark.parametrize("pos", ["first", "last", "interior"])
@pytest.mark.parametrize("interp", ["nearest", "bicubic"])
def test_grid_sampler_2d_nearest_and_bicubic_contain_a_poisoned_pixel(interp, pos):
    """Controls: these paths select by validity before use."""
    _gs_containment("f32", interp, "zeros", False, pos, seed=42)


@pytest.mark.parametrize("pos", ["first", "last", "interior"])
@pytest.mark.parametrize("pad", ["zeros", "border"])
@pytest.mark.parametrize("kind", ["rot", "wild"])
@pytest.mark.parametrize("fmt", ["f32", "f16"])
@pytest.mark.parametrize("mode", [1, 2])
def test_grid_sampler_tile_path_contains_a_poisoned_pixel(mode, fmt, kind, pad, pos):
    """The shared-memory tile kernel at a TMA-legal layout: "rot" grids take the staged window (bulk copies per row in
    mode 1, one tensor copy per packet in mode 2), "wild" grids its per-tile global-load fallback."""
    shape = (2, 37, 26, 40, 19, 45)
    lib = _lib.load()
    prev = lib.b200_grid_sample_set_tile_path(mode)
    try:
        # the small rotation never samples the image corners under zeros padding: only dummy taps read them
        _gs_containment(fmt, "bilinear", pad, False, pos, seed=43, shape=shape, grid=_tile_grid(kind, 2, 19, 45, 12),
                        may_be_unread=kind == "rot")
    finally:
        lib.b200_grid_sample_set_tile_path(prev)


@pytest.mark.parametrize("pos", ["first", "last", "interior"])
@pytest.mark.parametrize("fmt,interp,pad,align", [("f32", "bilinear", "zeros", False), ("f32", "bilinear", "zeros", True),
                                                   ("f32", "bilinear", "border", False), ("f32", "bilinear", "reflection", True),
                                                   ("f16", "bilinear", "zeros", False), ("f16", "bilinear", "border", True),
                                                   ("f32", "nearest", "zeros", False)])  # fmt: skip
def test_grid_sampler_3d_contains_a_poisoned_voxel(fmt, interp, pad, align, pos):
    # 280 nearest samples, most of them outside the volume, need not hit a given corner voxel
    _gs_containment(fmt, interp, pad, align, pos, seed=44, shape=(1, 3, 5, 7, 7, 8), depth=(5, 6),
                    may_be_unread=interp == "nearest")


def _coordinate_kinds(fmt):
    return {"nan": np.nan, "+inf": np.inf, "-inf": -np.inf, "huge": 1e30 if fmt == "f32" else 65504.0}


def _gs_substitute(kind, pad):
    """The finite grid coordinate the reference's rules turn a planted one into (gridSamplerKernel.cu:82-126): zeros:
    safe_downgrade_to_int_range sends a non-finite or > INT_MAX index to -100, a huge finite one is simply outside ->
    the tap contributes 0 (any coordinate far outside does the same: -1000); border: clip = fmin(size - 1, fmax(x, 0))
    and fmax(NaN, 0) = 0 -> first pixel for NaN / -Inf (-10), last for +Inf / huge (+10); reflection: fmod(Inf, span) and
    every operation on NaN give NaN, which the final clip sends to 0 (-10). A huge finite value under reflection is
    left out: the flip parity of an index beyond 2^24 is arbitrary in the reference too."""
    if pad == "zeros":
        return -1000.0
    if pad == "border":
        return 10.0 if kind in ("+inf", "huge") else -10.0
    return -10.0


def _gs_planted(fmt, interp, pad, align, seed, shape=GS_SHAPE, depth=None):
    x, g = _gs_inputs(fmt, seed, shape, depth)
    sp = g.shape[2:]
    spots = [(0, 0) + tuple(s // 2 - 1 for s in sp), (0, 1) + tuple(1 for _ in sp),
             (g.shape[0] - 1, g.shape[1] - 1) + tuple(s - 2 for s in sp), (g.shape[0] - 1, 0) + tuple(0 for _ in sp)]  # fmt: skip
    affected = np.zeros((g.shape[0],) + tuple(sp), bool)
    for s in spots:
        affected[(s[0],) + s[2:]] = True
    dev_clean = _gs_device(fmt, g, interp, pad, align)(x)
    affected = np.broadcast_to(affected[:, None], dev_clean.shape)
    tol = 3e-5 if fmt == "f32" else 1e-3 + 4.0 * 2.0**-11
    for kind, v in _coordinate_kinds(fmt).items():
        if kind == "huge" and (pad == "reflection" or (interp == "bicubic" and pad != "zeros")):
            continue
        planted, finite = g.clone(), g.clone()
        for s in spots:
            planted[s], finite[s] = v, _gs_substitute(kind, pad)
        want = _gs_oracle(finite, interp, pad, align)(x)
        if interp == "bicubic" and kind != "huge":
            # the fractional part of a NaN / Inf index is NaN, and so is every cubic coefficient (:757-792)
            want = np.where(affected, np.float32(np.nan), want)
        check_planted(want, dev_clean, _gs_device(fmt, planted, interp, pad, align)(x), affected, tol)


# kCHW2 shares the kernel with the linear layouts: one alignment of its bilinear path is enough
@pytest.mark.parametrize("fmt,pad,align,interp", [
    c for c in itertools.product(["f32", "f16", "chw2"], ["zeros", "border", "reflection"], [False, True],
                                 ["bilinear", "nearest", "bicubic"]) if c[0] != "chw2" or (c[3] == "bilinear" and not c[2])])  # fmt: skip
def test_grid_sampler_2d_non_finite_coordinate_is_an_out_of_range_sample(fmt, pad, align, interp):
    _gs_planted(fmt, interp, pad, align, seed=45)


@pytest.mark.parametrize("interp", ["bilinear", "nearest"])
@pytest.mark.parametrize("pad,align", list(itertools.product(["zeros", "border", "reflection"], [False, True])))
@pytest.mark.parametrize("fmt", ["f32", "f16"])
def test_grid_sampler_3d_non_finite_coordinate_is_an_out_of_range_sample(fmt, pad, align, interp):
    _gs_planted(fmt, interp, pad, align, seed=46, shape=(1, 3, 5, 7, 7, 8), depth=(5, 6))


# ---------------------------------------------------------------------------------------------------------------
# rotate
# ---------------------------------------------------------------------------------------------------------------
ROT_HW = (21, 23)
ROT_CENTER = (11.0, 10.0)  # exact in FP16, like the angles below


def _rot_device(fmt, angle, center, interp):
    a, c = torch.tensor([angle]), torch.tensor(list(center))
    if fmt == "f32":
        return lambda x: bt.rotate(torch.from_numpy(x).cuda(), a.cuda(), c.cuda(), interp).cpu()
    if fmt == "f16":
        return lambda x: bt.rotate(torch.from_numpy(x).half().cuda(), a.half().cuda(), c.half().cuda(), interp).cpu()
    if fmt == "chw2":
        def run(x):
            out = bt.rotate_chw2(pack_chw(torch.from_numpy(x).half()[None], 2)[0].cuda(), x.shape[0], a.half().cuda(),
                                 c.half().cuda(), interp)  # fmt: skip
            return unpack_chw(out.cpu()[None], x.shape[0])[0]

        return run
    dt = torch.float32 if fmt == "hwc_f32" else torch.float16

    def run_hwc(x):
        img = torch.from_numpy(x).to(dt).permute(1, 2, 0).contiguous().cuda()
        return bt.rotate_hwc(img, a.to(dt).cuda(), c.to(dt).cuda(), interp).permute(2, 0, 1).contiguous().cpu()

    return run_hwc


def _rot_image(fmt, seed):
    c = 8 if fmt.startswith("hwc") else 7  # channels-last wants whole 16-byte vectors; 7 leaves half a kCHW2 packet
    x = torch.randn(c, *ROT_HW, generator=torch.Generator().manual_seed(seed))
    return (x if fmt in ("f32", "hwc_f32") else x.half().float()).numpy()


ROT_FORMATS = ["f32", "f16", "chw2", "hwc_f32", "hwc_f16"]


@pytest.mark.parametrize("pos", ["first", "last", "interior"])
@pytest.mark.parametrize("angle", [33.25, 90.0])  # corners outside the image; 90 degrees lands on integer / x.5 indices
@pytest.mark.parametrize("interp", ["bilinear", "nearest"])
@pytest.mark.parametrize("fmt", ROT_FORMATS)
def test_rotate_contains_a_poisoned_pixel(fmt, interp, angle, pos):
    x = _rot_image(fmt, 51)
    mode, trig = 0 if interp == "bilinear" else 1, device_trig(angle)  # the oracle with CUDA's cosf / sinf, not libm's

    def oracle(a):
        return orot.rotate(a, angle, ROT_CENTER, mode, trig=trig)

    oob = np.broadcast_to(oracle(np.ones_like(x))[-1:] < 0.999, x.shape)
    idx = (x.shape[0] - 1,) + _plane_positions(ROT_HW)[pos]
    # a rotation about the middle moves the image corners out of the output: nothing samples them but dummy taps
    check_containment(oracle, _rot_device(fmt, angle, ROT_CENTER, interp), x, idx, oob, may_be_unread=pos != "interior")


@pytest.mark.parametrize("what", ["angle", "center_x", "center_y"])
@pytest.mark.parametrize("interp", ["bilinear", "nearest"])
@pytest.mark.parametrize("fmt", ROT_FORMATS)
def test_rotate_non_finite_angle_or_centre_gives_zeros(fmt, interp, what):
    """cos / sin of a non-finite angle are NaN, a non-finite centre makes the translation column Inf or NaN: every
    source index is non-finite, safe_downgrade_to_int_range (rotateKernel.cu:73-78) maps it to -100, and every output
    pixel is zero padding."""
    x = _rot_image(fmt, 52)
    for v in (np.nan, np.inf, -np.inf):
        angle, center = 33.25, list(ROT_CENTER)
        if what == "angle":
            angle = v
        else:
            center[0 if what == "center_x" else 1] = v
        out = _rot_device(fmt, angle, center, interp)(x)
        assert torch.equal(out, torch.zeros_like(out)), (v, int((out != 0).sum()))


# ---------------------------------------------------------------------------------------------------------------
# MSDA
# ---------------------------------------------------------------------------------------------------------------
MSDA_CASES = {
    "small_sca": CONFIGS["small_sca"],
    "tiny_sca": CONFIGS["tiny_sca"],
    "g2": MSDAConfig("g2", 2, 129, 8, 32, ((9, 11), (5, 6)), 8, 2),
}
HEAD, CHANNEL = 3, 5  # the poisoned head slice; every other head must not notice


@pytest.fixture
def restore_msda_switches():
    lib = _lib.load()
    units, variant, path = bt.get_msda_batch_units(), bt.get_msda_gather_variant(), bt.set_msda_f16_path(False)
    bt.set_msda_f16_path(path[0], path[1])
    mode = lib.b200_msda_set_f16_mode(0)
    lib.b200_msda_set_f16_mode(mode)
    yield
    bt.set_msda_batch_units(*units)
    bt.set_msda_gather_variant(variant)
    bt.set_msda_f16_path(path[0], path[1])
    lib.b200_msda_set_f16_mode(mode)


def _sca_mask(cfg):
    mask = (torch.rand(cfg.batch, cfg.num_query, 1, generator=torch.Generator().manual_seed(3)) > 0.4).float()
    mask[:, :5] = 0
    return mask * 0.5


def _msda_op(op, cfg, dt, shapes, ref, off, logits):
    """(oracle, device) of one entry point as functions of (value, ref, off) float32 ndarrays -> [.., M, C] outputs."""
    B, Q, M, C = cfg.batch, cfg.num_query, cfg.num_heads, cfg.channels
    lg = logits.float().numpy()
    mask = _sca_mask(cfg) if op in ("sca", "sca_shared") else torch.full((B, Q, 1), 1.0 / B)

    def oracle(v, r=None, o=None):
        r = ref.float().numpy() if r is None else r
        o = off.float().numpy() if o is None else o
        per_cam = omsda.msda_f32(v, shapes.numpy(), r, o, lg)
        if op == "plugin":
            return per_cam
        m = mask.numpy().reshape(B, Q, 1, 1)
        with np.errstate(invalid="ignore"):  # a camera the mask excludes is not sampled at all
            return np.where(m != 0, per_cam * m, np.float32(0)).sum(0, dtype=np.float32)

    def device(v, r=None, o=None):
        vd = torch.from_numpy(v).to(dt).cuda()
        rd = (ref if r is None else torch.from_numpy(r)).to(dt).cuda()
        od = (off if o is None else torch.from_numpy(o)).to(dt).cuda()
        ld, sd = logits.to(dt).cuda(), shapes.cuda()
        if op == "plugin":
            return bt.multi_scale_deformable_attn(vd, sd, rd, od, ld).cpu()
        if op == "sca":
            out = bt.multi_scale_deformable_attn_sca(vd, sd, rd, od, ld, mask.cuda())
        elif op == "sca_shared":
            out = bt.multi_scale_deformable_attn_sca_shared(vd, sd, rd, od[:1].contiguous(), ld[:1].contiguous(), mask.cuda())
        else:
            out = bt.multi_scale_deformable_attn_queue_mean(vd, sd, rd, od, ld)
        return out.reshape(Q, M, C).cpu()

    return oracle, device


def _msda_inputs(name, op, dt, seed):
    cfg = MSDA_CASES[name]
    value, shapes, ref, off, logits = make_msda_inputs(cfg, "edge", seed, dt)
    if op == "sca_shared":  # one copy of offsets / logits for all cameras; the oracle sees the repeated tensors
        off, logits = off[:1].expand_as(off).contiguous(), logits[:1].expand_as(logits).contiguous()
    return cfg, value.float().numpy(), shapes, ref, off, logits


def _msda_pixels(cfg, pos):
    """(a) the first pixel of every level: element 0 of the head slice, the address of an out-of-range point in the
    gather kernel, and the level starts the resident-tail kernel aliases; (b) the last pixel of every level; (c) an
    interior pixel of level 0."""
    starts = np.cumsum([0] + [h * w for h, w in cfg.spatial_shapes])
    if pos == "first":
        return list(starts[:-1])
    if pos == "last":
        return list(starts[1:] - 1)
    h, w = cfg.spatial_shapes[0]
    return [(h // 2) * w + w // 2]


def _msda_containment(name, op, dt, pos, seed):
    cfg, value, shapes, ref, off, logits = _msda_inputs(name, op, dt, seed)
    oracle, device = _msda_op(op, cfg, dt, shapes, ref, off, logits)
    # coverage of the plugin op on an all-ones value: below 1 where some point or tap is outside its image
    covered = omsda.msda_f32(np.ones_like(value), shapes.numpy(), ref.float().numpy(), off.float().numpy(),
                             logits.float().numpy())  # fmt: skip
    oob = covered < 0.999 if op == "plugin" else (covered < 0.999).any(0)
    idx = (slice(None), _msda_pixels(cfg, pos), HEAD, CHANNEL)
    untouched = np.ones(oob.shape, bool)
    untouched[..., HEAD, :] = False
    check_containment(oracle, device, value, idx, oob, untouched)


MSDA_POS = ["first", "last", "interior"]


@pytest.mark.parametrize("pos", MSDA_POS)
@pytest.mark.parametrize("name", list(MSDA_CASES))
@pytest.mark.parametrize("dt,f16_mode", [(torch.float32, 0), (torch.float16, 0), (torch.float16, 1)])
def test_msda_plugin_op_contains_a_poisoned_feature(dt, f16_mode, name, pos, restore_msda_switches):
    """FP32 and both FP16 arithmetic modes (exact, and fp16 tap weights) of the gather kernel at the default launch."""
    bt.set_msda_launch_shape("default")
    bt.set_msda_f16_path(False)
    _lib.load().b200_msda_set_f16_mode(f16_mode)
    _msda_containment(name, "plugin", dt, pos, seed=61)


@pytest.mark.parametrize("pos", ["first", "interior"])
@pytest.mark.parametrize("dt", [torch.float32, torch.float16])
@pytest.mark.parametrize("shape", [s for s in bt.MSDA_LAUNCH_SHAPES if s != "default"])
def test_msda_launch_shapes_contain_a_poisoned_feature(shape, dt, pos, restore_msda_switches):
    """Every launch shape the autotuner may pick: batched visibility scan, deeper gathers, 128-thread CTAs."""
    bt.set_msda_f16_path(False)
    bt.set_msda_launch_shape(shape)
    _msda_containment("small_sca", "plugin", dt, pos, seed=62)


@pytest.mark.parametrize("pos", ["first", "interior"])
@pytest.mark.parametrize("dt", [torch.float32, torch.float16])
@pytest.mark.parametrize("units,strided", [(2, False), (4, False), (4, True)])
def test_msda_batched_launch_contains_a_poisoned_feature(units, strided, dt, pos, restore_msda_switches):
    bt.set_msda_f16_path(False)
    bt.set_msda_gather_variant(0)
    bt.set_msda_batch_units(units, strided)
    _msda_containment("g2", "plugin", dt, pos, seed=63)


@pytest.mark.parametrize("pos", MSDA_POS)
@pytest.mark.parametrize("name", list(MSDA_CASES))
@pytest.mark.parametrize("cap", [8192, 131072])
def test_msda_resident_tail_kernel_contains_a_poisoned_feature(cap, name, pos, restore_msda_switches):
    """FP16 resident-tail kernel: coarse levels in shared memory (all of a small pyramid at 128 KB, the coarsest only at
    8 KB), the rest gathered from global memory."""
    bt.set_msda_f16_path(True, cap)
    _msda_containment(name, "plugin", torch.float16, pos, seed=64)


@pytest.mark.parametrize("pos", MSDA_POS)
@pytest.mark.parametrize("dt", [torch.float32, torch.float16])
@pytest.mark.parametrize("op,name", [("sca", "small_sca"), ("sca", "g2"), ("sca_shared", "small_sca"), ("sca_shared", "tiny_sca"),
                                     ("sca_shared", "g2"), ("queue_mean", "small_sca"), ("queue_mean", "g2")])  # fmt: skip
def test_msda_fused_epilogues_contain_a_poisoned_feature(op, name, dt, pos, restore_msda_switches):
    """Fused SCA (two cameras: the two float adds per slot commute, so runs are bit-reproducible), camera-shared SCA and
    the queue-mean epilogue."""
    bt.set_msda_launch_shape("default")
    _msda_containment(name, op, dt, pos, seed=65)


def _msda_planted(name, op, dt, seed):
    """One x or y of a reference point (every point of that query's group goes out of range, in every head) and single
    sampling offsets (one point of one head) are replaced; the oracle's range test is a comparison, which a NaN fails
    and an Inf falls outside of, before any conversion to int."""
    cfg, value, shapes, ref, off, logits = _msda_inputs(name, op, dt, seed)
    oracle, device = _msda_op(op, cfg, dt, shapes, ref, off, logits)
    B, Q, M = cfg.batch, cfg.num_query, cfg.num_heads
    G, NP = cfg.points_per_group, cfg.num_levels * cfg.num_points
    ref_spots = [(0, 7, 0, 0), (B - 1, Q - 1, 0, 2 * G - 1)]
    off_spots = [(0, 20, 1, 0), (0, 21, 2, 2 * NP - 1), (B - 1, 40, M - 1, NP + 1), (B - 1, 41, 0, 3)]
    dev_clean = device(value)
    hit = np.zeros((B, Q, M), bool)
    for b, q, _, _ in ref_spots:
        hit[b, q] = True
    for b, q, m, _ in off_spots:
        hit[(slice(None) if op == "sca_shared" else b), q, m] = True
    hit = hit if op == "plugin" else hit.any(0)
    affected = np.broadcast_to(hit[..., None], dev_clean.shape)
    tol = 2e-5 if dt == torch.float32 else 1e-3
    for kind, v in _coordinate_kinds("f32" if dt == torch.float32 else "f16").items():
        r, o = ref.float().numpy().copy(), off.float().numpy().copy()
        for s in ref_spots:
            r[s] = v
        for b, q, m, k in off_spots:
            o[(slice(None) if op == "sca_shared" else b), q, m, k] = v
        check_planted(oracle(value, r, o), dev_clean, device(value, r, o), affected, tol)


# not the fused SCA on six cameras: they add into a slot in arbitrary order, so no clean run is bit-reproducible
@pytest.mark.parametrize("dt", [torch.float32, torch.float16])
@pytest.mark.parametrize("op,name", [c for c in itertools.product(["plugin", "sca", "sca_shared", "queue_mean"], list(MSDA_CASES))
                                     if c != ("sca", "tiny_sca")])  # fmt: skip
def test_msda_non_finite_coordinate_is_an_out_of_range_point(op, name, dt, restore_msda_switches):
    bt.set_msda_launch_shape("default")
    bt.set_msda_f16_path(False)
    _msda_planted(name, op, dt, seed=66)


@pytest.mark.parametrize("dt", [torch.float32, torch.float16])
def test_msda_non_finite_coordinate_in_every_launch_shape_and_the_resident_kernel(dt, restore_msda_switches):
    bt.set_msda_f16_path(False)
    for shape in bt.MSDA_LAUNCH_SHAPES:
        bt.set_msda_launch_shape(shape)
        _msda_planted("small_sca", "plugin", dt, seed=67)
    bt.set_msda_gather_variant(0)
    for units, strided in [(2, False), (4, False)]:
        bt.set_msda_batch_units(units, strided)
        _msda_planted("g2", "plugin", dt, seed=68)
    if dt == torch.float16:
        bt.set_msda_launch_shape("default")
        for cap in (8192, 131072):
            bt.set_msda_f16_path(True, cap)
            _msda_planted("small_sca", "plugin", dt, seed=69)


# ---------------------------------------------------------------------------------------------------------------
# DCN
# ---------------------------------------------------------------------------------------------------------------
def _dcn_inputs(case, dt, seed=0):
    """Seeded inputs with a fifth of the offsets rounded: samples at exact integer positions, whose missing-neighbour
    taps have weight exactly 0."""
    x, off, mask, w, b, kw = make_dcn_inputs(case, seed=seed, dtype=dt)
    pick = torch.rand(off.shape, generator=torch.Generator().manual_seed(seed + 1)) < 0.2
    off = torch.where(pick, off.float().round(), off.float()).to(dt)
    return x.float().numpy(), off, mask, w, b, kw


def _dcn_ops(path, dt, off, mask, w, b, kw):
    args = (kw["stride"], kw["padding"], kw["dilation"], kw["groups"], kw["deform_groups"])
    wf, bf = w.float().numpy(), b.float().numpy()

    def oracle(x, o=None, m=None):
        o = off.float().numpy() if o is None else o
        m = mask.float().numpy() if m is None else m
        with np.errstate(invalid="ignore", over="ignore"):
            return odcn.modulated_deformable_conv2d(x, o, m, wf, bf, **kw)

    def device(x, o=None, m=None):
        xd = torch.from_numpy(x).to(dt)
        od = off if o is None else torch.from_numpy(o).to(dt)
        md = mask if m is None else torch.from_numpy(m).to(dt)
        if path == "chw2":
            return modulated_deformable_conv2d_chw2(pack_chw(xd, 2).cuda(), pack_chw(od, 2).cuda(), md.cuda(),
                                                    pack_chw(w, 2).cuda(), b.cuda(), xd.shape[1], *args).cpu()  # fmt: skip
        return bt.modulated_deformable_conv2d(xd.cuda(), od.cuda(), md.cuda(), w.cuda(), b.cuda(), *args).cpu()

    return oracle, device


DCN_PATHS = [
    # (path, case): padding 0 / 1 / 2 on every kernel
    ("f32", "k3_s1_p1_g2_dg2"), ("f32", "k1_s1_p0_g1_dg1"), ("f32", "k3_s1_p2_d2_g1_dg4"), ("f32", "gen_asym_g2_dg4"),
    ("f16_generic", "fused_co128"), ("f16_generic", "fused_p0"), ("f16_generic", "k3_s1_p2_d2_g1_dg4"),
    ("f16_fused", "fused_co128"), ("f16_fused", "fused_co256_ragged"), ("f16_fused", "fused_d2"), ("f16_fused", "fused_p0"),
    ("f16_fused", "fused_p2"),
    ("chw2", "k3_s1_p1_g2_dg2"), ("chw2", "fused_co128"),
]  # fmt: skip


@pytest.fixture
def dcn_path(request):
    lib = _lib.load()
    prev = lib.b200_dcn_set_fused(0 if request.param == "f16_generic" else 1)
    yield request.param
    lib.b200_dcn_set_fused(prev)


def _dcn_dtype(path):
    return torch.float32 if path == "f32" else torch.float16


@pytest.mark.parametrize("pos", ["first", "last", "interior"])
@pytest.mark.parametrize("dcn_path,case", DCN_PATHS, indirect=["dcn_path"])
def test_dcn_forward_contains_a_poisoned_pixel(dcn_path, case, pos):
    dt = _dcn_dtype(dcn_path)
    x, off, mask, w, b, kw = _dcn_inputs(case, dt)
    oracle, device = _dcn_ops(dcn_path, dt, off, mask, w, b, kw)
    kh, kw_ = w.shape[2:]
    geo = {k: kw[k] for k in ("stride", "padding", "dilation")}
    col, _ = odcn.im2col(np.ones_like(x), off.float().numpy(), np.ones(mask.shape, np.float32), kh, kw_,
                         deform_groups=kw["deform_groups"], **geo)  # fmt: skip
    out_shape = oracle(x).shape
    oob = np.broadcast_to((col < 0.999).any(1).reshape(out_shape[0], 1, *out_shape[2:]), out_shape)
    idx = (slice(None), 1) + _plane_positions(x.shape[2:])[pos]
    check_containment(oracle, device, x, idx, oob)


@pytest.mark.parametrize("dcn_path,case", [("f32", "k3_s1_p1_g2_dg2"), ("f32", "k3_s1_p2_d2_g1_dg4"), ("f16_generic", "fused_co128"),
                                           ("f16_fused", "fused_co128"), ("f16_fused", "fused_co256_ragged"),
                                           ("f16_fused", "fused_d2"), ("chw2", "k3_s1_p1_g2_dg2")], indirect=["dcn_path"])  # fmt: skip
def test_dcn_non_finite_offset_is_an_out_of_range_tap_and_nan_mask_follows_the_reference(dcn_path, case):
    """A non-finite or huge offset fails the range test (comparisons, before any conversion), so the tap contributes
    0 * mask = 0. The column value is val * mask in the reference (…Conv2dKernel.cu:259-318), also when val is the 0 of
    an out-of-range tap: a NaN mask gives NaN for the output channels that read it at that pixel, inside the image or not."""
    dt = _dcn_dtype(dcn_path)
    x, off, mask, w, b, kw = _dcn_inputs(case, dt, seed=3)
    oracle, device = _dcn_ops(dcn_path, dt, off, mask, w, b, kw)
    dev_clean = device(x)
    n, _, ho, wo = off.shape
    spots = [(0, 0, 0, 0), (0, 1, ho // 2, wo // 2), (n - 1, off.shape[1] - 1, ho - 1, wo - 1), (n - 1, 2, 1, wo - 2)]
    affected = np.zeros(dev_clean.shape, bool)
    for s in spots:
        affected[s[0], :, s[2], s[3]] = True
    want_clean = oracle(x)
    tol = 1e-4 if dt == torch.float32 else 0.5 * float(np.spacing(np.float16(np.abs(want_clean).max()))) + 1e-3
    for kind, v in _coordinate_kinds("f32" if dt == torch.float32 else "f16").items():
        o = off.float().numpy().copy()
        for s in spots:
            o[s] = v
        check_planted(oracle(x, o=o), dev_clean, device(x, o=o), affected, tol)
    # NaN mask: once on a tap far outside the image (its offset pushed out as well), once wherever the seeded tap lies
    o, m = off.float().numpy().copy(), mask.float().numpy().copy()
    tap = 2
    o[0, 2 * tap, 0, 0] = -50.0
    mspots = [(0, tap, 0, 0), (n - 1, 0, ho // 2, wo // 2), (n - 1, mask.shape[1] - 1, ho - 1, 0)]
    affected = np.zeros(dev_clean.shape, bool)
    for s in mspots:
        m[s] = np.nan
        affected[s[0], :, s[2], s[3]] = True
    want = oracle(x, o=o, m=m)
    # every output channel of the convolution group(s) that read the masked deformable group, at those pixels only
    assert np.isnan(want[affected]).any() and not np.isnan(want[~affected]).any()
    for s in mspots:
        assert np.isnan(want[s[0], :, s[2], s[3]]).any()
    o_clean = off.float().numpy().copy()
    o_clean[0, 2 * tap, 0, 0] = -50.0
    check_planted(want, device(x, o=o_clean), device(x, o=o, m=m), affected, tol)


@pytest.mark.parametrize("pos", ["first", "interior"])
@pytest.mark.parametrize("dt", [torch.float32, torch.float16])
def test_dcn_backward_contains_a_poisoned_pixel(dt, pos):
    """Control: the backward kernels select by validity flags before use. grad_offset, grad_mask and grad_weight read
    x; the oracle is torchvision's CPU autograd of the same DCNv2 definition."""
    import torchvision

    case = "k3_s1_p1_g2_dg2"
    x, off, mask, w, b, kw = make_dcn_inputs(case, seed=5, dtype=dt)
    go = torch.randn(x.shape[0], w.shape[0], off.shape[2], off.shape[3], generator=torch.Generator().manual_seed(6)).to(dt)
    x = x.float().numpy()

    def oracle(a):
        ts = [t.float().clone().requires_grad_(True) for t in (off, mask, w)]
        out = torchvision.ops.deform_conv2d(torch.from_numpy(a), ts[0], ts[2], b.float(), stride=kw["stride"],
                                            padding=kw["padding"], dilation=kw["dilation"], mask=ts[1])  # fmt: skip
        out.backward(go.float())
        return torch.cat([t.grad.reshape(-1) for t in ts]).numpy()

    def device(a):
        ts = [t.cuda().requires_grad_(True) for t in (off, mask, w)]
        out = bt.modulated_deformable_conv2d(torch.from_numpy(a).to(dt).cuda(), ts[0], ts[1], ts[2], b.cuda(), kw["stride"],
                                             kw["padding"], kw["dilation"], kw["groups"], kw["deform_groups"])  # fmt: skip
        out.backward(go.cuda())
        return torch.cat([t.grad.reshape(-1) for t in ts]).cpu()

    idx = (slice(None), 1) + _plane_positions(x.shape[2:])[pos]
    check_containment(oracle, device, x, idx)
