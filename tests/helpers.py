"""Shared test helpers (tests may use oracle/; the product package may not)."""
import glob
import hashlib
import os

import numpy as np
import torch

from bevformer_tensorrt_b200.workloads import MSDAConfig, make_msda_inputs

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
REF_KERNELS_GOLDEN = os.path.join(GOLDEN, "ref_kernels.npz")
GOLDEN_SAMPLE = 4096  # elements kept of a larger reference-kernel output


def golden_index(numel):
    """Flat positions of an output of `numel` elements kept in tests/golden/ref_kernels.npz: all of them for small outputs,
    else GOLDEN_SAMPLE positions from a generator seeded by the size (the same positions on every run)."""
    if numel <= GOLDEN_SAMPLE:
        return np.arange(numel)
    return np.sort(np.random.default_rng(numel).choice(numel, GOLDEN_SAMPLE, replace=False))


def golden_sample(t):
    """The kept elements of a tensor / array, flattened, as float32 (int8 outputs are exact in float32)."""
    a = t.detach().float().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t, np.float32)
    flat = a.reshape(-1)
    return flat[golden_index(flat.size)].astype(np.float32)


def ref_kernels_golden():
    """Outputs of the reference project's own CUDA kernels (tests/golden/make_golden_ref_kernels.py), by case key."""
    return np.load(REF_KERNELS_GOLDEN)


def input_digest(*tensors):
    h = hashlib.sha256()
    for t in tensors:
        h.update(t.contiguous().numpy().tobytes())
    return h.hexdigest()


def golden_msda_cases():
    return sorted(glob.glob(os.path.join(GOLDEN, "msda_*.npz")))


def load_golden_msda(path):
    """Returns (cfg, (value, shapes, ref, off, logits) float32 CPU tensors, expected out ndarray)."""
    z = np.load(path)
    B, Q, M, C, L, P, G, seed = (int(x) for x in z["meta"])
    shapes = tuple((int(h), int(w)) for h, w in z["shapes"])
    cfg = MSDAConfig(os.path.basename(path), B, Q, M, C, shapes, P, G)
    inputs = make_msda_inputs(cfg, str(z["dist"]), seed, torch.float32)
    if input_digest(*inputs) != str(z["digest"]):
        if "value" in z.files:  # self-contained fixture
            inputs = (torch.from_numpy(z["value"]), inputs[1], torch.from_numpy(z["ref"]),
                      torch.from_numpy(z["off"]), torch.from_numpy(z["logits"]))  # fmt: skip
        else:
            raise RuntimeError(f"{path}: seeded CPU generator no longer reproduces the golden inputs")
    return cfg, inputs, z["out"]


def kernels_recorded(fn, found, tries=3):
    """Runs ``fn()`` under a CUDA activity trace until ``found(names)`` holds, at most ``tries`` times. Returns (the last
    result, the kernel names recorded over every try). The trace now and then loses a kernel record: on an H100, about
    one MSDA backward call in 300 came back without its gather kernel, once without any of its kernels. Since the
    names of every try are kept, a kernel that should never run is checked against every call made."""
    from torch.profiler import ProfilerActivity, profile

    names = []
    for _ in range(tries):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            result = fn()
            torch.cuda.synchronize()
        names += [e.name for e in prof.events()]
        if found(names):
            break
    return result, names


def make_grid_sampler_inputs(N, C, Hi, Wi, Ho, Wo, seed=0, depth=None, span=15.0):
    """input ~ N(0,1); grid = a regular sweep over [-span, span] (1.5x beyond the image, as the reference test's
    linspace(-15, 15), test_grid_sampler.py:29-36) plus N(0, 0.5) jitter, channel-first [N, 2|3, ...]."""
    g = torch.Generator().manual_seed(seed)
    if depth is None:
        inp = torch.randn(N, C, Hi, Wi, generator=g)
        ys, xs = torch.meshgrid(torch.linspace(-span, span, Ho), torch.linspace(-span, span, Wo), indexing="ij")
        grid = torch.stack([xs, ys], 0)[None].repeat(N, 1, 1, 1)
    else:
        Di, Do = depth
        inp = torch.randn(N, C, Di, Hi, Wi, generator=g)
        zs, ys, xs = torch.meshgrid(torch.linspace(-span, span, Do), torch.linspace(-span, span, Ho),
                                    torch.linspace(-span, span, Wo), indexing="ij")  # fmt: skip
        grid = torch.stack([xs, ys, zs], 0)[None].repeat(N, 1, 1, 1, 1)
    grid = grid + 0.5 * torch.randn(grid.shape, generator=g)
    return inp, grid.contiguous()


def make_rotation_grid(H, W, angle_deg, shift=(0.0, 0.0)):
    """The prev-BEV warp grid of BASELINE configs[3]: output pixel centres rotated by ``angle_deg`` about the image
    centre (plus a translation in pixels), normalised to [-1, 1] and scaled x10 — the plugin's [-10, 10] convention
    (SURVEY.md Appendix B; onnx_ops.py:226-232 builds the same grid x10). Returns float32 [1, 2, H, W] (x plane, y)."""
    import math

    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    cx, cy = (W - 1) / 2.0, (H - 1) / 2.0
    c, s_ = math.cos(math.radians(angle_deg)), math.sin(math.radians(angle_deg))
    sx = c * (xs - cx) - s_ * (ys - cy) + cx + shift[0]
    sy = s_ * (xs - cx) + c * (ys - cy) + cy + shift[1]
    gx = ((sx + 0.5) / W * 2 - 1) * 10
    gy = ((sy + 0.5) / H * 2 - 1) * 10
    return torch.stack([gx, gy], 0)[None].contiguous()


ROTATE_CASES = {
    # name: (C, H, W, angle_deg, (center_x, center_y))
    "bev_small": (8, 50, 50, 1.7, (25.0, 25.0)),        # prev_bev alignment: a few degrees about the BEV centre
    "bev_neg": (6, 40, 48, -4.25, (24.0, 20.0)),
    "big_angle": (5, 33, 47, 127.3, (20.5, 13.25)),     # reference test: angle ~ N(0,1)*360 (test_rotate.py:21-25)
    "off_center": (4, 31, 29, -61.0, (40.0, 38.0)),     # centre outside the image (test_rotate.py: center = 500, 500)
    "zero": (3, 17, 19, 0.0, (9.5, 8.5)),
    "right_angle": (3, 16, 16, 90.0, (8.0, 8.0)),       # lands on x.5 / integer source indices
    "odd_c": (7, 21, 23, 33.3, (11.0, 10.0)),           # C not a multiple of the kCHW2 / kCHW4 packet
}


def make_rotate_inputs(case, seed=0):
    """img ~ N(0,1) [C,H,W], angle [1] (degrees), center [2] as float32 tensors (test_rotate.py:19-26)."""
    C, H, W, ang, ctr = ROTATE_CASES[case]
    g = torch.Generator().manual_seed(seed)
    return torch.randn(C, H, W, generator=g), torch.tensor([ang]), torch.tensor(list(ctr))


_PC_RANGE = (-51.2, -51.2, -5.0, 51.2, 51.2, 3.0)  # BEVFormer nuScenes configs (point_cloud_range)
POINT_SAMPLING_CASES = {
    # name: (bev_h, bev_w, num_points_in_pillar, image (h, w), pc_range)
    "ring_small": (50, 50, 4, (928, 1600), _PC_RANGE),     # BEVFormer-tiny BEV size
    "ring_rect": (30, 44, 4, (480, 800), _PC_RANGE),       # non-square BEV, small images (BEVFormer-small-like)
    "ring_d8": (20, 20, 8, (928, 1600), (-40.0, -40.0, -1.0, 40.0, 40.0, 5.4)),
    "ring_d1": (16, 24, 1, (928, 1600), _PC_RANGE),
}


def make_point_sampling_inputs(case):
    """lidar2img [6, 4, 4] float32 of the synthetic camera ring (bevformer_tensorrt_b200.workloads)."""
    from bevformer_tensorrt_b200.workloads import camera_ring_lidar2img

    return camera_ring_lidar2img(6, img_hw=POINT_SAMPLING_CASES[case][3])


DCN_CASES = {
    # name: (N, Ci, H, W, Co, kh, kw, stride, padding, dilation, groups, deform_groups); stride, padding and dilation are
    # an int or an (h, w) pair
    "k3_s1_p1_g2_dg2": (2, 16, 13, 17, 12, 3, 3, 1, 1, 1, 2, 2),  # the reference op test's structure, reduced
    "k3_s2_p1_g1_dg1": (2, 8, 14, 15, 6, 3, 3, 2, 1, 1, 1, 1),
    "k3_s1_p2_d2_g1_dg4": (1, 16, 12, 12, 8, 3, 3, 1, 2, 2, 1, 4),
    "k1_s1_p0_g1_dg1": (2, 8, 9, 9, 8, 1, 1, 1, 0, 1, 1, 1),
    "k3x5_s1_p1_g1_dg1": (1, 4, 11, 13, 4, 3, 5, 1, 1, 1, 1, 1),
    "backbone_like": (2, 64, 29, 50, 64, 3, 3, 1, 1, 1, 1, 1),  # BEVFormer R101 stage shapes, channels reduced
    # generic kernel: every geometry pair asymmetric, so an h/w swap anywhere changes the output
    "gen_asym_g2_dg4": (2, 16, 15, 19, 12, 3, 3, (2, 1), (1, 2), (1, 2), 2, 4),
    "gen_co100": (2, 32, 14, 15, 100, 3, 3, 1, 1, 1, 1, 1),  # Co = 100: a partial 64-row output tile
    "gen_k7": (1, 8, 17, 19, 16, 7, 7, 1, 3, 1, 1, 1),  # kh*kw = 49 > 48: one input channel per K block
    # shapes the fused wgmma path takes in FP16 (groups = dg = 1, C % 64 == 0, Co in {128, 256, 512})
    "fused_co128": (2, 64, 20, 24, 128, 3, 3, 1, 1, 1, 1, 1),
    "fused_co256_ragged": (3, 128, 29, 50, 256, 3, 3, 1, 1, 1, 1, 1),  # 1450 pixels: partial last tile, unaligned rows
    "fused_co512_s2": (1, 64, 31, 33, 512, 3, 3, 2, 1, 1, 1, 1),
    "fused_k1": (2, 128, 16, 16, 128, 1, 1, 1, 0, 1, 1, 1),
    "fused_d2": (2, 64, 21, 23, 128, 3, 3, 1, 2, 2, 1, 1),
    "fused_p0": (1, 64, 18, 20, 256, 3, 3, 1, 0, 1, 1, 1),
    "fused_p2": (1, 64, 15, 17, 512, 3, 3, 1, 2, 1, 1, 1),
    "fused_s2x1": (2, 64, 24, 19, 128, 3, 3, (2, 1), 1, 1, 1, 1),
    "fused_k1x3": (1, 64, 14, 17, 256, 1, 3, 1, (0, 1), 1, 1, 1),
    "fused_k3x1": (1, 64, 17, 14, 128, 3, 1, 1, (1, 0), 1, 1, 1),
    "fused_k3x2_d1x2": (2, 64, 13, 16, 512, 3, 2, 1, (1, 0), (1, 2), 1, 1),  # kh*kw = 6
    "fused_k1x9": (1, 64, 12, 30, 128, 1, 9, 1, (0, 4), 1, 1, 1),
    "fused_c192": (2, 192, 15, 18, 256, 3, 3, 1, 1, 1, 1, 1),  # three 64-channel chunks
}


def _hw(v):
    return (v, v) if isinstance(v, int) else tuple(v)


def make_dcn_inputs(case, seed=0, dtype=torch.float32):
    N, Ci, H, W, Co, kh, kw, s, p, d, g, dg = DCN_CASES[case]
    (sh, sw), (ph, pw), (dh, dw) = _hw(s), _hw(p), _hw(d)
    gen = torch.Generator().manual_seed(seed)
    Ho = (H + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1
    Wo = (W + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1
    x = torch.randn(N, Ci, H, W, generator=gen)
    off = torch.randn(N, dg * 2 * kh * kw, Ho, Wo, generator=gen) * 1.5
    mask = torch.sigmoid(torch.randn(N, dg * kh * kw, Ho, Wo, generator=gen))  # dcn.py:74
    w = torch.randn(Co, Ci // g, kh, kw, generator=gen) / (Ci // g * kh * kw) ** 0.5
    b = torch.randn(Co, generator=gen)
    kwargs = dict(stride=s, padding=p, dilation=d, groups=g, deform_groups=dg)
    return x.to(dtype), off.to(dtype), mask.to(dtype), w.to(dtype), b.to(dtype), kwargs


def fp16_tol(want):
    """FP16-output error budget: 0.5 * spacing_fp16(max|want|) + 1e-3 (see tests/test_dcn_gpu.py)."""
    return 0.5 * float(np.spacing(np.float16(np.abs(want).max()))) + 1e-3


# ---- the per-element bound against the float64 references of oracle/f64.py (tests/test_msda_dcn_sweep_gpu.py derives
# it; tests/test_rotate_sweep_gpu.py applies it to rotate) -------------------------------------------------------------
U32 = 2.0**-24
U_DTYPE = {torch.float32: 2.0**-24, torch.float16: 2.0**-11, torch.bfloat16: 2.0**-8}
S_DTYPE = {torch.float32: 2.0**-150, torch.float16: 2.0**-25, torch.bfloat16: 2.0**-134}  # half the least subnormal
_MANT = {torch.float32: (23, -126), torch.float16: (10, -14), torch.bfloat16: (7, -126)}


def ulp(a, dtype):
    """Spacing of ``dtype`` at the float64 magnitudes ``a`` (subnormal spacing below the smallest normal)."""
    mant, emin = _MANT[dtype]
    _, e = torch.frexp(a)
    return torch.ldexp(torch.ones_like(a), torch.clamp(e - 1, min=emin) - mant)


def element_bound(ent, u_acc, dtype, low=None):
    """|got - r| <= 1/2 ulp_dtype(|r| + E) + E, E = (8 + n) u_acc mag + 2^-24 pmag (+ the low-precision terms).
    ``low``: the dtype the path rounds intermediates to, or None."""
    E = (8 + ent["n"]) * u_acc * ent["mag"] + U32 * ent["pmag"]
    if low is not None:
        E = E + U_DTYPE[low] * ent["lmag"] + S_DTYPE[low] * ent["lcnt"]
    return 0.5 * ulp(ent["r"].abs() + E, dtype) + E


def tensor_bar(r, dtype):
    m = float(r.abs().max()) if r.numel() else 0.0
    if dtype == torch.float32:
        return 1e-4 * m
    return 0.5 * float(ulp(torch.tensor([m], dtype=torch.float64), dtype)) + 1e-4 * m


def check(tag, name, got, ent, u_acc, low=None, bar=None):
    """Asserts the per-element bound on every element of ``got`` (and the per-tensor bar); reports the worst element."""
    assert got is not None, f"{tag}: {name} was requested but is None"
    r = ent["r"]
    assert tuple(got.shape) == tuple(r.shape), (tag, name, tuple(got.shape), tuple(r.shape))
    g = got.detach().to(r.device, torch.float64)
    bound = element_bound(ent, u_acc, got.dtype, low)
    err = (g - r).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        ratio = torch.where(bad, err / bound.clamp(min=1e-300), torch.zeros_like(err))
        i = int(ratio.reshape(-1).argmax())
        idx = np.unravel_index(i, tuple(r.shape))
        raise AssertionError(f"{tag} {name}: {int(bad.sum())} of {r.numel()} elements outside the bound; worst at "
                             f"{tuple(int(v) for v in idx)}: got {g.reshape(-1)[i].item()!r} ref {r.reshape(-1)[i].item()!r} "
                             f"bound {bound.reshape(-1)[i].item():.3e} (mag {ent['mag'].reshape(-1)[i].item():.3e})")  # fmt: skip
    if not r.numel():
        return
    b = tensor_bar(r, got.dtype) if bar is None else bar
    if low is not None and bar is None:  # the largest intermediate rounding on top of the per-tensor bar
        b += U_DTYPE[low] * float(ent["lmag"].max()) + S_DTYPE[low] * float(ent["lcnt"].max())
    assert float(err.max()) <= b, (tag, name, float(err.max()), b)


def rounding_bound(want, scale, n, dtype):
    """Per-element bound on a float32-accumulated chain of ``n`` products stored in ``dtype``: half a ulp of ``dtype``
    at the float64 result ``want``, plus (n + 1) * 2^-24 * ``scale``, where ``scale`` is the same op in float64 on the
    inputs' magnitudes (it bounds every partial sum of the chain)."""
    ulp = np.spacing(np.abs(np.asarray(want)).astype(dtype)).astype(np.float64)
    return 0.5 * ulp + (np.asarray(n, np.float64) + 1.0) * 2.0**-24 * np.asarray(scale, np.float64)
