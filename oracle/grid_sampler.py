"""oracle/grid_sampler.py — TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

ctypes driver for oracle/grid_sampler_oracle.c (the reference GridSampler2DTRT FP32 kernel restated), a torch
restatement of the reference binding's forward (det2trt/models/functions/grid_sampler.py:28-32) and ``grid_sample_np``,
a vectorised numpy restatement of the kernel's semantics in 2-D and 3-D evaluated in float64 or float32."""
import ctypes

import numpy as np

from . import lib

_f32p = ctypes.POINTER(ctypes.c_float)
INDEX_DTYPE = np.dtype([("ix", "<i4"), ("iy", "<i4")])


def grid_sample_2d(inp, grid, interp, padding, align, return_index=False):
    """inp [N,C,Hi,Wi], grid [N,2,Ho,Wo] in [-10,10]; interp 0/1/2 = bilinear/nearest/bicubic; padding 0/1/2 =
    zeros/border/reflection. float32 evaluation of the kernel's formulas."""
    inp = np.ascontiguousarray(inp, np.float32)
    grid = np.ascontiguousarray(grid, np.float32)
    N, C, Hi, Wi = inp.shape
    _, two, Ho, Wo = grid.shape
    assert two == 2 and grid.shape[0] == N
    out = np.empty((N, C, Ho, Wo), np.float32)
    idx = np.empty((N, Ho, Wo), INDEX_DTYPE) if return_index else None
    lib().oracle_grid_sample_2d_f32(inp.ctypes.data_as(_f32p), grid.ctypes.data_as(_f32p), out.ctypes.data_as(_f32p),
                                    N, C, Hi, Wi, Ho, Wo, int(interp), int(padding), int(bool(align)),
                                    idx.ctypes.data_as(ctypes.c_void_p) if return_index else None)  # fmt: skip
    return (out, idx) if return_index else out


def grid_sampler_torch_port(inp, grid, interp, padding, align):
    """The reference binding's forward: aten.grid_sampler(input, grid.permute(0,2,3,1)/10, mode, pad, align) for 4-D,
    permute(0,2,3,4,1) for 5-D (grid_sampler.py:28-32, :84-88)."""
    import torch

    perm = (0, 2, 3, 1) if grid.dim() == 4 else (0, 2, 3, 4, 1)
    return torch.ops.aten.grid_sampler(inp, grid.permute(*perm) / 10, interp, padding, bool(align))


# ---- grid_sample_np: the kernel's semantics in numpy -----------------------------------------------------------------
# gridSamplerKernel.cu :82-92 unnormalise from the channel-first [-10, 10] grid, :157-162 clip, :226-247 reflect,
# :342-351 safe_downgrade_to_int_range, :372-393 compute_coordinates, :457-533 cubic convolution (A = -0.75) and
# :615-629 get_value_bounded; 3-D as :1271-1923 (trilinear / nearest). Every operation is one numpy operation in the
# evaluation dtype, so float32 evaluation rounds where the kernel's fp32 does and float64 evaluation is the same
# formulas carried (almost) without rounding.
_INT_RANGE = 2.0**31  # (float)(INT_MAX - 1) and -(float)INT_MIN


def unnormalize(g, size, align, dt):
    half = (g + dt(10)) * dt(0.5)
    if align:
        return half * (dt(size - 1) / dt(10))
    return half * (dt(size) / dt(10)) - dt(0.5)


def _clip(x, size, dt):
    return np.fmin(dt(size - 1), np.fmax(x, dt(0)))  # fminf / fmaxf: a NaN operand yields the other one


def _reflect(x, twice_low, twice_high, dt):
    if twice_low == twice_high:
        return np.zeros_like(x)
    mn, span = dt(twice_low) * dt(0.5), dt(twice_high - twice_low) * dt(0.5)
    x = np.abs(x - mn)
    extra = np.fmod(x, span)
    with np.errstate(invalid="ignore"):
        even = np.floor(x / span) % 2 == 0
    return np.where(even, extra + mn, (span - extra) + mn)


def _safe(x, dt):
    with np.errstate(invalid="ignore"):
        bad = (x > _INT_RANGE) | (x < -_INT_RANGE) | ~np.isfinite(x)
    return np.where(bad, dt(-100), x)


def _coordinates(x, size, padding, align, dt):
    if padding == 1:
        x = _clip(x, size, dt)
    elif padding == 2:
        x = _reflect(x, 0, 2 * (size - 1), dt) if align else _reflect(x, -1, 2 * size - 1, dt)
        x = _clip(x, size, dt)
    return _safe(x, dt)


def round_half_away(x):
    """::round / roundf: half away from zero (ATen's nearest mode uses nearbyint, half to even)."""
    a = np.abs(x)
    r = np.floor(a)
    return np.copysign(r + (a - r >= 0.5), x)


def _cubic_coeffs(t, dt):
    A = dt(-0.75)

    def c1(x):
        return ((A + dt(2)) * x - (A + dt(3))) * x * x + dt(1)

    def c2(x):
        return ((A * x - dt(5) * A) * x + dt(8) * A) * x - dt(4) * A

    x2 = dt(1) - t
    return [c2(t + dt(1)), c1(t), c1(x2), c2(x2 + dt(1))]


def _gather(flat, idx, sizes):
    """flat [N, C, prod(sizes)]; idx = integer-valued coordinate arrays [N, P] (x, y[, z]) against sizes (W, H[, D]).
    Returns the tapped values [N, C, P], out-of-range taps replaced by 0 (dropped, never multiplied), and validity."""
    ok = np.ones(idx[0].shape, bool)
    lin = np.zeros(idx[0].shape, np.int64)
    stride = 1
    for i, s in zip(idx, sizes):
        with np.errstate(invalid="ignore"):
            ok &= (i >= 0) & (i < s)
        lin += np.clip(np.nan_to_num(i), 0, s - 1).astype(np.int64) * stride
        stride *= s
    v = np.take_along_axis(flat, lin[:, None, :], axis=2)
    return np.where(ok[:, None, :], v, 0), ok


def grid_sample_np(inp, grid, interp, padding, align, dtype=np.float64):
    """inp [N, C, (Di,) Hi, Wi], grid [N, 2|3, (Do,) Ho, Wo] (x, y[, z] planes) in [-10, 10]; interp 0/1/2 =
    bilinear (trilinear in 3-D) / nearest / bicubic (2-D only); padding 0/1/2 = zeros / border / reflection. Evaluated
    in `dtype` (np.float64 or np.float32); returns [N, C, (Do,) Ho, Wo] in that dtype."""
    dt = np.dtype(dtype).type
    inp = np.asarray(inp).astype(dt)
    grid = np.asarray(grid).astype(dt)
    nd = grid.shape[1]
    assert nd in (2, 3) and inp.ndim == grid.ndim == nd + 2 and inp.shape[0] == grid.shape[0]
    assert not (nd == 3 and interp == 2), "bicubic is 2-D only"
    N, C = inp.shape[:2]
    sizes = inp.shape[2:][::-1]  # (Wi, Hi[, Di]) against the grid planes (x, y[, z])
    out_sp = grid.shape[2:]
    flat = inp.reshape(N, C, -1)
    g = [grid[:, a].reshape(N, -1) for a in range(nd)]
    out = np.zeros((N, C, g[0].shape[1]), dt)
    if interp == 2:
        ix = [unnormalize(g[a], sizes[a], align, dt) for a in range(2)]
        lo = [np.floor(c) for c in ix]
        cx, cy = (_cubic_coeffs(c - f, dt) for c, f in zip(ix, lo))
        col = [np.trunc(_coordinates(lo[0] + dt(q - 1), sizes[0], padding, align, dt)) for q in range(4)]
        for r in range(4):
            yi = np.trunc(_coordinates(lo[1] + dt(r - 1), sizes[1], padding, align, dt))
            row = np.zeros_like(out)
            for q in range(4):
                row = row + _gather(flat, (col[q], yi), sizes)[0] * cx[q][:, None, :]
            out = out + row * cy[r][:, None, :]
    else:
        ix = [_coordinates(unnormalize(g[a], sizes[a], align, dt), sizes[a], padding, align, dt) for a in range(nd)]
        if interp == 1:
            out = _gather(flat, [round_half_away(c) for c in ix], sizes)[0]
        else:
            lo = [np.floor(c) for c in ix]
            for t in range(1 << nd):  # corner t: bit a set = high side on axis a (x, y, z); the kernel's tap order
                hi = [(t >> a) & 1 for a in range(nd)]
                w = None
                for a in range(nd):
                    wa = ix[a] - lo[a] if hi[a] else (lo[a] + dt(1)) - ix[a]
                    w = wa if w is None else w * wa
                v, ok = _gather(flat, [lo[a] + dt(hi[a]) for a in range(nd)], sizes)
                out = out + v * np.where(ok, w, dt(0))[:, None, :]
    return out.reshape(N, C, *out_sp)
