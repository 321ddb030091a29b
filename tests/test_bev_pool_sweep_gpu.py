"""BEVPoolV2 at every launch shape its kernels take, bit for bit against the C oracle.

The kernels pick a vector width VEC (the widest that divides C and keeps every pointer the kernel touches aligned), a
lane group of G = pow2(ceil(C / VEC)) <= 32 lanes, and, for the forward and the feature gradient, one channel tile of
G * VEC channels per blockIdx.y. Each case below reaches one (VEC, G, tiles) through C and through contiguous views at an
element offset (the binding keeps a view's data_ptr), and the kernel names in a torch.profiler trace, taken in a child
process, confirm which <T, VEC> instantiation ran. Every output is compared bit for bit with the oracle's restatement of the kernel's
arithmetic (fmaf chains in point order; the depth gradient's lane partials and xor butterfly), and element by element
with float64 within half an output ulp plus (n + 1) roundings of the magnitude sum. The backward also keeps non-finite
values where float64 puts them, and the depth gradient's bits do not depend on the feature gradient's buffer."""
import ctypes
import json
import os
import re
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

import bevformer_tensorrt_b200 as bt
from bevformer_tensorrt_b200 import _lib
from oracle import bev_pool as obev
from tests.helpers import kernels_recorded, rounding_bound

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

VECS = {torch.float32: (4, 2, 1), torch.float16: (8, 4, 2, 1), torch.int8: (16, 8, 4, 2, 1)}
TYPE_NAMES = {torch.float32: "float", torch.float16: "__half", torch.int8: "signed char"}
NP_TYPES = {torch.float32: np.float32, torch.float16: np.float16}
BITS = {torch.float32: np.uint32, torch.float16: np.uint16}


def pick_vec(dtype, C, ptrs):
    """bev_pool.cu's pick_vec: the widest vector (elements) that divides C and keeps every pointer aligned."""
    size = torch.empty(0, dtype=dtype).element_size()
    for v in VECS[dtype][:-1]:
        if C % v == 0 and all(p % (v * size) == 0 for p in ptrs):
            return v
    return 1


def group_size(C, vec):
    lanes, G = -(-C // vec), 1
    while G < lanes and G < 32:
        G *= 2
    return G


# (dtype, C, feat offset, out_grad offset): offsets in elements from a 512-byte aligned allocation
CASES = [
    (torch.float32, 1, 0, 0),  # VEC 1, G 1
    (torch.float32, 2, 0, 0),  # VEC 2, G 1
    (torch.float32, 3, 0, 0),  # VEC 1, G 4 with an idle lane
    (torch.float32, 8, 0, 0),  # VEC 4, G 2
    (torch.float32, 12, 0, 2),  # VEC 4, G 4 with an idle lane forward; VEC 2, G 8 with idle lanes backward
    (torch.float32, 16, 2, 0),  # VEC 2 forward / depth, G 8; VEC 4 feature gradient
    (torch.float32, 33, 0, 0),  # VEC 1, G 32, two tiles (the last one channel); depth loop of two strides
    (torch.float32, 64, 0, 0),  # VEC 4, G 16
    (torch.float32, 64, 0, 1),  # VEC 4, G 16 forward; VEC 1, G 32 backward (two feature-gradient tiles)
    (torch.float32, 80, 1, 0),  # VEC 1, G 32, three tiles (the last half full); VEC 4, G 32 (20 lanes) feature gradient
    (torch.float32, 130, 0, 0),  # VEC 2, G 32, three tiles (the last 2 channels)
    (torch.float32, 132, 0, 0),  # VEC 4, G 32, two tiles (the last 4 channels)
    (torch.float16, 1, 0, 0),  # VEC 1, G 1
    (torch.float16, 4, 0, 0),  # VEC 4, G 1
    (torch.float16, 6, 0, 0),  # VEC 2, G 4 with an idle lane
    (torch.float16, 8, 0, 0),  # VEC 8, G 1
    (torch.float16, 16, 0, 0),  # VEC 8, G 2
    (torch.float16, 17, 0, 0),  # VEC 1, G 32
    (torch.float16, 24, 0, 0),  # VEC 8, G 4 with an idle lane
    (torch.float16, 40, 4, 0),  # VEC 4 forward / depth, G 16; VEC 8 feature gradient, G 8 with idle lanes
    (torch.float16, 40, 0, 2),  # VEC 8, G 8 with idle lanes forward; VEC 2, G 32 with idle lanes backward
    (torch.float16, 64, 0, 0),  # VEC 8, G 8
    (torch.float16, 64, 0, 3),  # VEC 8, G 8 forward; VEC 1, G 32 backward (two feature-gradient tiles)
    (torch.float16, 128, 2, 0),  # VEC 2, G 32, two tiles forward and depth; VEC 8, G 16 feature gradient
    (torch.float16, 260, 0, 0),  # VEC 4, G 32, three tiles (the last 4 channels)
    (torch.float16, 264, 0, 0),  # VEC 8, G 32, two tiles (the last 8 channels)
    (torch.int8, 4, 0, 0),  # VEC 4, G 1
    (torch.int8, 8, 0, 0),  # VEC 8, G 1
    (torch.int8, 16, 0, 0),  # VEC 16, G 1
    (torch.int8, 20, 0, 0),  # VEC 4, G 8 with idle lanes
    (torch.int8, 24, 0, 0),  # VEC 8, G 4 with an idle lane
    (torch.int8, 32, 0, 0),  # VEC 16, G 2
    (torch.int8, 48, 0, 0),  # VEC 16, G 4 with an idle lane
    (torch.int8, 64, 1, 0),  # VEC 1, G 32, two tiles
    (torch.int8, 64, 2, 0),  # VEC 2, G 32
    (torch.int8, 64, 4, 0),  # VEC 4, G 16
    (torch.int8, 260, 0, 0),  # VEC 4, G 32, three tiles (the last 4 channels)
    (torch.int8, 528, 0, 0),  # VEC 16, G 32, two tiles (the last 16 channels)
]


def _id(case):
    dtype, C, fo, go = case
    return f"{TYPE_NAMES[dtype].replace(' ', '_')}-C{C}-f{fo}-g{go}"


def shapes_of(dtype, C, feat_off, gout_off):
    """{kernel: (VEC, G, tiles)} for the kernels a case launches, from offsets off a 512-byte aligned base (the
    binding allocates the output and the feature gradient itself, aligned)."""
    size = torch.empty(0, dtype=dtype).element_size()
    f, g = feat_off * size, gout_off * size
    vecs = {"bev_pool_kernel": pick_vec(dtype, C, [f, 0])}
    if dtype != torch.int8:
        vecs["bev_pool_depth_grad_kernel"] = pick_vec(dtype, C, [g, f])
        vecs["bev_pool_feat_grad_kernel"] = pick_vec(dtype, C, [g, 0])
    out = {}
    for k, v in vecs.items():
        G = group_size(C, v)
        out[k] = (v, G, 1 if k == "bev_pool_depth_grad_kernel" else -(-C // (G * v)))
    return out


def test_cases_cover_every_launch_shape():
    """Every VEC per dtype and kernel, every G from 1 to 32, idle lanes, more than one channel tile and a partial last
    tile in FP32 and FP16 (forward and feature gradient), and a depth-gradient loop of more than one stride."""
    seen = {}
    for dtype, C, fo, go in CASES:
        for k, (v, G, tiles) in shapes_of(dtype, C, fo, go).items():
            s = seen.setdefault((dtype, k), {"vec": set(), "G": set(), "idle": False, "tiles": False, "partial": False,
                                             "strides": False})  # fmt: skip
            s["vec"].add(v)
            s["G"].add(G)
            s["idle"] |= -(-C // v) < G
            s["tiles"] |= tiles > 1
            s["partial"] |= tiles > 1 and C % (G * v) != 0
            s["strides"] |= C > G * v
    kernels = {torch.float32: 3, torch.float16: 3, torch.int8: 1}
    assert len(seen) == sum(kernels.values())
    for (dtype, k), s in seen.items():
        assert s["vec"] == set(VECS[dtype]), (dtype, k, s)
        assert s["G"] == {1, 2, 4, 8, 16, 32}, (dtype, k, s)
        assert s["idle"], (dtype, k)
        if k == "bev_pool_depth_grad_kernel":
            assert s["strides"], (dtype, k)
        elif dtype != torch.int8:
            assert s["tiles"] and s["partial"], (dtype, k)


def _geometry(seed=0):
    """Ranks for one pooled frame with interval lengths around the 4-point unroll and every group size (1, 3, 4, 5,
    G - 1, G, G + 1, 4G + 3 for G = 1 .. 32, 5000 and random ones), points between intervals, two dropped intervals
    (cell out of range), a first interval starting before 0 and a last one running past P (both clipped), points
    with out-of-range ranks_depth / ranks_feat, and feature rows referenced 1 to 400 times plus one 3000 times.
    Returns (ranks as int32 numpy arrays, depth_size, feat_rows, (out_h, out_w))."""
    rng = np.random.default_rng(seed)
    lengths = {1, 3, 4, 5, 5000}
    for G in (1, 2, 4, 8, 16, 32):
        lengths |= {max(G - 1, 1), G, G + 1, 4 * G + 3}
    lengths = list(lengths) + list(rng.integers(1, 70, 150))
    rng.shuffle(lengths)
    out_hw = (23, 29)
    cells = np.sort(rng.choice(out_hw[0] * out_hw[1], len(lengths), replace=False))
    rb, starts, p = [], [], 0
    for n, cell in zip(lengths, cells):
        gap = int(rng.integers(1, 4)) if rng.random() < 0.2 else 0  # points no interval names
        rb += [cell] * gap
        p += gap
        starts.append(p)
        rb += [cell] * n
        p += n
    rb, st, ln = np.array(rb, np.int32), np.array(starts, np.int32), np.array(lengths, np.int32)
    P, I = rb.size, st.size
    for k in (7, 40):  # dropped: the cell the interval names lies outside the output
        rb[st[k]:st[k] + ln[k]] = out_hw[0] * out_hw[1] + k if k == 7 else -1
    st[0] -= 2
    ln[0] += 2
    ln[I - 1] += 9
    runs = [3000, 400, 300, 257, 256, 255, 129, 128, 127, 65, 64, 63, 33, 32, 31, 17, 16, 15, 9, 8, 5, 4, 3, 2]
    fixed = np.repeat(np.arange(len(runs)), runs)
    rows = 3 * P // 4
    rf = np.concatenate([fixed, rng.integers(len(runs), rows - 50, P - fixed.size)])  # the last 50 rows unused
    rf = rng.permutation(rf).astype(np.int32)
    depth_size = P + 1000
    rd = rng.permutation(depth_size)[:P].astype(np.int32)
    bad = rng.choice(P, 60, replace=False)
    rd[bad[:15]], rd[bad[15:30]] = -1, depth_size + np.arange(15)
    rf[bad[30:45]], rf[bad[45:]] = -3, rows + np.arange(15)
    return (rd, rf, rb, st, ln), depth_size, rows, out_hw


GEOMETRY = _geometry()


def at_offset(a, off, dtype):
    """A contiguous CUDA copy of ``a`` (in ``dtype``) whose data starts ``off`` elements into a fresh allocation."""
    t = torch.as_tensor(np.ascontiguousarray(a)).to(dtype)
    buf = torch.empty(t.numel() + off, dtype=dtype, device="cuda")
    assert buf.data_ptr() % 512 == 0
    view = buf[off:].view(t.shape)
    view.copy_(t)
    return view


def _inputs(dtype, C, seed):
    ranks, depth_size, rows, hw = GEOMETRY
    g = torch.Generator().manual_seed(seed)
    depth = torch.rand(depth_size, generator=g) + 0.01
    feat = torch.randn(rows, C, generator=g)
    gout = torch.randn(1, hw[0], hw[1], C, generator=g)
    if dtype == torch.float16:  # the inputs the half kernels see, exactly
        depth, feat, gout = depth.half().float(), feat.half().float(), gout.half().float()
    return depth.numpy(), feat.numpy(), gout.numpy()


_KERNEL = re.compile(r"(bev_pool(?:_depth_grad|_feat_grad)?_kernel)<\s*([\w ]+?)\s*,\s*(?:\(int\))?\s*(\d+)\s*>")
_TYPE_ALIASES = {"half": "__half", "char": "signed char", "int8_t": "signed char"}


def _names(names):
    """{kernel: [VEC, ...]} from recorded kernel names such as bev_pool_kernel<float, 4>."""
    out = {}
    for n in names:
        m = _KERNEL.search(n)
        if m:
            out.setdefault(m.group(1), []).append((_TYPE_ALIASES.get(m.group(2), m.group(2)), int(m.group(3))))
    return out


def _bits(a, dtype):
    return np.ascontiguousarray(a).view(BITS[dtype])


_INT8_SCALES = (1 / 127, 1 / 40, 0.02)  # depth, feat, out


def _int8(depth, feat):
    return np.clip(np.round(depth * 127), -127, 127).astype(np.int8), np.clip(np.round(feat * 40), -127, 127).astype(np.int8)


def _run_case(case):
    """Runs a case on the device: the INT8 forward, or the FP32 / FP16 forward and its backward through autograd, with
    feat and out_grad at the case's element offsets. Returns (the outputs, {kernel: pointers its VEC depends on})."""
    dtype, C, feat_off, gout_off = case
    ranks, depth_size, rows, hw = GEOMETRY
    depth, feat, gout = _inputs(dtype, C, C)
    rk = [torch.from_numpy(r).cuda() for r in ranks]
    if dtype == torch.int8:
        dq, fq = _int8(depth, feat)
        d, f = at_offset(dq, 0, dtype), at_offset(fq, feat_off, dtype)
        sd, sf, so = _INT8_SCALES
        return bt.bev_pool_v2_int8(d, sd, f, sf, *rk, so, *hw), {"bev_pool_kernel": [f.data_ptr()]}
    d = at_offset(depth, 0, dtype).requires_grad_(True)
    f = at_offset(feat, feat_off, dtype).requires_grad_(True)
    g = at_offset(gout.reshape(1, hw[0], hw[1], C), gout_off, dtype)
    out = bt.bev_pool_v2(d, f, *rk, *hw)
    out.backward(g)
    ptrs = {"bev_pool_kernel": [f.data_ptr()], "bev_pool_depth_grad_kernel": [g.data_ptr(), f.data_ptr()],
            "bev_pool_feat_grad_kernel": [g.data_ptr()]}  # fmt: skip
    return (out.detach(), d.grad, f.grad), ptrs


def record_kernels():
    """{case id: {kernel: [[type, VEC], ...]}}: every case run once under a CUDA activity trace."""
    out = {}
    for case in CASES:
        want = len(shapes_of(*case))
        _, names = kernels_recorded(lambda: _run_case(case), lambda ns: len(_names(ns)) == want)
        out[_id(case)] = {k: sorted(set(v)) for k, v in _names(names).items()}
    return out


@pytest.fixture(scope="module")
def recorded():
    """record_kernels() in a child process. The traces run there, not in the test process: in one process, this
    file's CUDA activity traces followed by those of tests/test_msda_backward_gpu.py left the next trace (in
    tests/test_msda_envelope_gpu.py) without any kernel record."""
    code = f"import json, sys; sys.path.insert(0, {ROOT!r}); from tests.test_bev_pool_sweep_gpu import record_kernels; " \
           "print(json.dumps(record_kernels()))"
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=_id)
def test_launch_shape_bit_for_bit(case, recorded):
    dtype, C, feat_off, gout_off = case
    ranks, depth_size, rows, hw = GEOMETRY
    depth, feat, gout = _inputs(dtype, C, C)
    want_shapes = shapes_of(*case)
    ran = {k: [tuple(x) for x in v] for k, v in recorded[_id(case)].items()}
    assert ran == {k: [(TYPE_NAMES[dtype], vec)] for k, (vec, _, _) in want_shapes.items()}, ran
    got, ptrs = _run_case(case)
    for k, p in ptrs.items():  # the offsets reach the widths shapes_of expects
        assert pick_vec(dtype, C, p) == want_shapes[k][0], k
    if dtype == torch.int8:
        dq, fq = _int8(depth, feat)
        sd, sf, so = _INT8_SCALES
        want = obev.bev_pool_i8(dq, sd, fq, sf, ranks, so, hw)
        assert np.array_equal(got.cpu().numpy(), want)
        assert 0 < np.count_nonzero(np.abs(want.astype(np.int32)) == 127) < np.count_nonzero(want) // 2
        return
    out, dg, fg = got

    # bit for bit: the forward's fmaf chain in point order, rounded once to the output type
    want = obev.bev_pool_f32_fma(depth, feat, ranks, hw).astype(NP_TYPES[dtype])
    assert np.array_equal(_bits(out.cpu().numpy(), dtype), _bits(want, dtype))
    vd, Gd, _ = want_shapes["bev_pool_depth_grad_kernel"]
    vf, Gf, _ = want_shapes["bev_pool_feat_grad_kernel"]
    wd, _ = obev.bev_pool_backward_f32_lanes(gout, depth, feat, ranks, hw, Gd, vd, feat_grad=False)
    _, wf = obev.bev_pool_backward_f32_lanes(gout, depth, feat, ranks, hw, Gf, vf, depth_grad=False)
    assert np.array_equal(_bits(dg.cpu().numpy(), dtype), _bits(wd.astype(NP_TYPES[dtype]), dtype))
    assert np.array_equal(_bits(fg.cpu().numpy(), dtype), _bits(wf.astype(NP_TYPES[dtype]), dtype))

    # element by element against float64: half an output ulp plus (n + 1) roundings of the magnitude sum
    rd, rf, rb, st, ln = ranks
    lo, hi = np.maximum(st, 0), np.minimum(st.astype(np.int64) + ln, rd.size)
    n_cell = np.zeros(hw[0] * hw[1])
    ok = (rb[lo] >= 0) & (rb[lo] < n_cell.size)
    n_cell[rb[lo][ok]] = (hi - lo)[ok]
    n_row = np.bincount(rf[(rf >= 0) & (rf < rows)], minlength=rows)
    w64 = obev.bev_pool_f64(depth, feat, ranks, hw)
    s64 = obev.bev_pool_f64(np.abs(depth), np.abs(feat), ranks, hw)
    wd64, wf64 = obev.bev_pool_backward_f64(gout, depth, feat, ranks, hw)
    sd64, sf64 = obev.bev_pool_backward_f64(np.abs(gout), depth, np.abs(feat), ranks, hw)
    npt = NP_TYPES[dtype]
    for got, w, s, n in ((out, w64, s64, n_cell.reshape(1, hw[0], hw[1], 1)), (dg, wd64, sd64, C),
                         (fg, wf64, sf64, n_row[:, None])):  # fmt: skip
        err = np.abs(got.double().cpu().numpy() - w)
        assert np.all(err <= rounding_bound(w, s, n, npt)), float((err - rounding_bound(w, s, n, npt)).max())
    assert np.count_nonzero(wd) > 0.9 * rd.size and np.count_nonzero(wf) > 0.5 * wf.size


NONFINITE_CASES = [(torch.float32, 33, 0), (torch.float32, 64, 0), (torch.float16, 24, 0), (torch.float16, 64, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,C,gout_off", NONFINITE_CASES, ids=lambda v: str(v).replace("torch.", ""))
@pytest.mark.parametrize("value", [float("nan"), float("inf")])
def test_backward_non_finite_stays_where_float64_puts_it(dtype, C, gout_off, value):
    """One non-finite value in out_grad (one cell, one channel), in one feat row and in one depth element: the set of
    non-finite gradient elements is float64's, and every other element keeps the clean run's bits."""
    ranks, depth_size, rows, hw = GEOMETRY
    rd, rf, rb, st, ln = ranks
    depth, feat, gout = _inputs(dtype, C, 11)
    rk = [torch.from_numpy(r).cuda() for r in ranks]

    def grads(depth, feat, gout):
        d = at_offset(depth, 0, dtype).requires_grad_(True)
        f = at_offset(feat, 0, dtype).requires_grad_(True)
        bt.bev_pool_v2(d, f, *rk, *hw).backward(at_offset(gout, gout_off, dtype))
        return d.grad.cpu().numpy(), f.grad.cpu().numpy()

    clean = grads(depth, feat, gout)
    kept = np.flatnonzero((rd >= 0) & (rd < depth_size) & (rf >= 0) & (rf < rows))
    i_cell, i_row, i_depth = (kept[np.searchsorted(kept, st[k])] for k in (3, 8, 12))  # in kept intervals
    depth2, feat2, gout2 = depth.copy(), feat.copy(), gout.copy()
    gout2.reshape(-1, C)[rb[i_cell], C // 2] = value
    feat2[rf[i_row], C - 1] = value
    depth2[rd[i_depth]] = value
    got = grads(depth2, feat2, gout2)
    with np.errstate(invalid="ignore"):
        want = obev.bev_pool_backward_f64(gout2, depth2, feat2, ranks, hw)
    for g, c, w in zip(got, clean, want):
        bad = ~np.isfinite(w)
        assert 0 < bad.sum() < bad.size
        assert np.array_equal(~np.isfinite(g.astype(np.float64)), bad)
        assert np.array_equal(_bits(g[~bad], dtype), _bits(c[~bad], dtype))


def _abi_backward(dtype, gout, depth, feat, ranks, hw, order, depth_grad, feat_grad, ws):
    name = "b200_bev_pool_backward_f32" if dtype == torch.float32 else "b200_bev_pool_backward_f16"
    C = feat.shape[-1]
    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    st = getattr(_lib.load(), name)(gout.data_ptr(), depth.data_ptr(), feat.data_ptr(), *(r.data_ptr() for r in ranks),
                                    ptr(order), C, ranks[0].numel(), ranks[3].numel(), depth.numel(), feat.numel() // C,
                                    hw[0], hw[1], ptr(depth_grad), ptr(feat_grad), ws.data_ptr(), ws.numel() * 4,
                                    ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))  # fmt: skip
    assert st == 0, st


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_depth_grad_bits_do_not_depend_on_the_feat_grad_buffer(dtype):
    """The C ABI's depth gradient alone (feat_grad NULL), and with a feat_grad buffer one element off 16 bytes: the
    same bits, each kernel's vector width taken from the tensors it touches."""
    ranks, depth_size, rows, hw = GEOMETRY
    C = 64
    depth, feat, gout = _inputs(dtype, C, 21)
    rk = [torch.from_numpy(r).cuda() for r in ranks]
    d, f, g = at_offset(depth, 0, dtype), at_offset(feat, 0, dtype), at_offset(gout, 0, dtype)
    order = torch.sort(rk[1], stable=True).indices.int()
    ws = torch.empty(rk[0].numel(), dtype=torch.int32, device="cuda")
    dg_alone = torch.full_like(d, float("nan"))
    _abi_backward(dtype, g, d, f, rk, hw, None, dg_alone, None, ws)
    dg = torch.full_like(d, float("nan"))
    fg = at_offset(np.full(feat.shape, np.nan, np.float32), 1, dtype)
    _abi_backward(dtype, g, d, f, rk, hw, order, dg, fg, ws)
    torch.cuda.synchronize()
    assert torch.equal(dg, dg_alone)
    vec = VECS[dtype][0]
    wd, _ = obev.bev_pool_backward_f32_lanes(gout, depth, feat, ranks, hw, group_size(C, vec), vec, feat_grad=False)
    _, wf = obev.bev_pool_backward_f32_lanes(gout, depth, feat, ranks, hw, 32, 1, depth_grad=False)
    assert np.array_equal(_bits(dg.cpu().numpy(), dtype), _bits(wd.astype(NP_TYPES[dtype]), dtype))
    assert np.array_equal(_bits(fg.cpu().numpy(), dtype), _bits(wf.astype(NP_TYPES[dtype]), dtype))


@pytest.mark.gpu
def test_feat_grad_runs_past_two_to_the_27_points():
    """P = 2^27 + 3000 points at C = 17 (VEC 1, G = 32): the feature-gradient launch has P * 32 > 2^32 threads, so a
    32-bit thread index would wrap and leave the runs that start past point 2^27 at zero. ranks_feat is non-decreasing:
    1024-point runs up to 2^27, then one row per point; 1000 intervals of about 134,000 points. About 3 GB of device
    memory and 5 GB of host memory; the test took 7 to 12 s on an H100 (80 GB), most of it the oracle on the host."""
    C, P, I = 17, 2**27 + 3000, 1000
    t0 = time.time()
    if torch.cuda.get_device_properties(0).total_memory < 16 * 2**30:
        pytest.skip("needs about 3 GB of free device memory")
    head = 2**27 // 1024
    rows = head + (P - 2**27)
    idx = np.arange(P, dtype=np.int32)
    rf = np.where(idx < 2**27, idx // 1024, head + (idx - 2**27)).astype(np.int32)
    per = P // I
    st = (np.arange(I) * per).astype(np.int32)
    ln = np.full(I, per, np.int32)
    ln[-1] = P - st[-1]
    rb = np.minimum(idx // per, I - 1).astype(np.int32)
    ranks = (idx, rf, rb, st, ln)  # ranks_depth = the point index
    hw = (25, 40)
    g = torch.Generator().manual_seed(0)
    depth = (torch.rand(P, generator=g) + 0.5).numpy()
    feat = torch.randn(rows, C, generator=g).numpy()
    gout = torch.randn(I, C, generator=g).numpy()
    rk = [torch.from_numpy(r).cuda() for r in ranks]
    d, f, og = (torch.from_numpy(a).cuda() for a in (depth, feat, gout))
    fg = torch.full_like(f, float("nan"))
    ws = torch.empty(P, dtype=torch.int32, device="cuda")
    _abi_backward(torch.float32, og, d, f, rk, hw, rk[0], None, fg, ws)  # order = the identity: rf is sorted
    got = fg.cpu().numpy()
    del rk, d, f, og, fg, ws
    _, want = obev.bev_pool_backward_f32_lanes(gout, depth, feat, ranks, hw, 32, 1, depth_grad=False)
    late = want[head:]
    assert np.count_nonzero(late) == late.size  # every run past 2^27 has a gradient
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), int((got[head:] == 0).all(axis=1).sum())
    print(f"P = {P}: {time.time() - t0:.1f} s")
