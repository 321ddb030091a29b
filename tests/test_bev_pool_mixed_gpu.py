"""BEVPoolV2 in BF16 and with FP32 depth and FP16 / BF16 features (what torch.autocast hands the op: a softmax depth and
conv features), forward and both gradients.

Every 2-byte element is widened to FP32 exactly and FP32 depth is used as loaded, so every output equals an existing
oracle bit for bit: ``out`` is oracle/bev_pool.py's bev_pool_f32_fma of the widened inputs rounded once to the features'
dtype, and the gradients are bev_pool_backward_f32_lanes at the lane group (G, VEC) the 2-byte tensors give, rounded
once where the gradient is 2 bytes (an FP32 depth gradient is not rounded). CPU torch conversion is the
round-to-nearest-even reference (numpy has no bf16). The cases reach every (VEC, G, tiles) of the FP16 sweep through C
and element offsets of feat / out_grad, and kernel names in a torch.profiler trace, taken in a child process, confirm
which instantiation ran. Every element is also within tests.helpers.element_bound of float64, here and on the full
bevdet_r50 workload."""
import json
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
from torch import nn

import bevformer_tensorrt_b200 as bt
from bevformer_tensorrt_b200 import _lib
from bevformer_tensorrt_b200.functions.bev_pool_v2 import _entries
from bevformer_tensorrt_b200.workloads import BEV_POOL_CONFIGS, bev_pool_ranks, make_bev_pool_inputs
from oracle import bev_pool as obev
from tests.helpers import U32, U_DTYPE, check, kernels_recorded
from tests.test_bev_pool_sweep_gpu import CASES as SWEEP_CASES
from tests.test_bev_pool_sweep_gpu import GEOMETRY, ROOT, at_offset, group_size, pick_vec

F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16
PAIRS = {"bf16": (BF16, BF16), "f32_f16": (F32, F16), "f32_bf16": (F32, BF16)}  # name: (depth dtype, feat dtype)
BITS = {F32: torch.int32, F16: torch.int16, BF16: torch.int16}
TYPE_TAG = {F16: "f16", BF16: "bf16"}

# the FP16 sweep's (C, feat offset, out_grad offset) cases, which reach every launch shape of a 2-byte feature type,
# for each new dtype pair
CASES = [(pair, C, fo, go) for pair in PAIRS for dt, C, fo, go in SWEEP_CASES if dt == F16]


def _id(case):
    pair, C, fo, go = case
    return f"{pair}-C{C}-f{fo}-g{go}"


def kernel_names(pair):
    """{kernel base: recorded name} of a pair: the same-dtype kernels for bf16, the FP32-depth wrappers otherwise."""
    suffix = "" if PAIRS[pair][0] == PAIRS[pair][1] else "_f32_depth"
    return {k: f"{k}{suffix}_kernel" for k in ("bev_pool", "bev_pool_depth_grad", "bev_pool_feat_grad")}


def shapes_of(pair, C, feat_off, gout_off):
    """{kernel base: (VEC, G, tiles)}. The width comes from the 2-byte feat / out / out_grad / feat_grad pointers alone
    (the output and feature gradient are allocated aligned), so the vector table is FP16's whatever the depth type."""
    f, g = feat_off * 2, gout_off * 2
    vecs = {"bev_pool": pick_vec(F16, C, [f, 0]), "bev_pool_depth_grad": pick_vec(F16, C, [g, f]),
            "bev_pool_feat_grad": pick_vec(F16, C, [g, 0])}  # fmt: skip
    out = {}
    for k, v in vecs.items():
        G = group_size(C, v)
        out[k] = (v, G, 1 if k == "bev_pool_depth_grad" else -(-C // (G * v)))
    return out


def test_cases_cover_every_launch_shape():
    """Per pair and kernel: VEC 8, 4, 2 and 1, every G from 1 to 32, idle lanes, more than one channel tile and a
    partial last tile (forward and feature gradient), and a depth-gradient loop of more than one stride."""
    seen = {}
    for pair, C, fo, go in CASES:
        for k, (v, G, tiles) in shapes_of(pair, C, fo, go).items():
            s = seen.setdefault((pair, k), {"vec": set(), "G": set(), "idle": False, "tiles": False, "partial": False,
                                            "strides": False})  # fmt: skip
            s["vec"].add(v)
            s["G"].add(G)
            s["idle"] |= -(-C // v) < G
            s["tiles"] |= tiles > 1
            s["partial"] |= tiles > 1 and C % (G * v) != 0
            s["strides"] |= C > G * v
    assert len(seen) == 3 * len(PAIRS)
    for (pair, k), s in seen.items():
        assert s["vec"] == {8, 4, 2, 1} and s["G"] == {1, 2, 4, 8, 16, 32} and s["idle"], (pair, k, s)
        assert s["strides"] if k == "bev_pool_depth_grad" else s["tiles"] and s["partial"], (pair, k, s)


def _inputs(pair, C, seed):
    """float32 numpy (depth, feat, out_grad) of the sweep geometry, each exactly representable in its dtype."""
    dd, fd = PAIRS[pair]
    _, depth_size, rows, hw = GEOMETRY
    g = torch.Generator().manual_seed(seed)
    depth = torch.rand(depth_size, generator=g) + 0.01
    feat = torch.randn(rows, C, generator=g)
    gout = torch.randn(1, hw[0], hw[1], C, generator=g)
    return depth.to(dd).float().numpy(), feat.to(fd).float().numpy(), gout.to(fd).float().numpy()


def _run_case(case):
    """The forward and its backward through autograd, feat and out_grad at the case's element offsets. Returns (out,
    depth_grad, feat_grad) and {kernel base: the pointers its VEC depends on}."""
    pair, C, feat_off, gout_off = case
    dd, fd = PAIRS[pair]
    ranks, _, _, hw = GEOMETRY
    depth, feat, gout = _inputs(pair, C, C)
    rk = [torch.from_numpy(r).cuda() for r in ranks]
    d = at_offset(depth, 0, dd).requires_grad_(True)
    f = at_offset(feat, feat_off, fd).requires_grad_(True)
    g = at_offset(gout, gout_off, fd)
    out = bt.bev_pool_v2(d, f, *rk, *hw)
    out.backward(g)
    ptrs = {"bev_pool": [f.data_ptr()], "bev_pool_depth_grad": [g.data_ptr(), f.data_ptr()],
            "bev_pool_feat_grad": [g.data_ptr()]}  # fmt: skip
    return (out.detach(), d.grad, f.grad), ptrs


_KERNEL = re.compile(r"(bev_pool(?:_depth_grad|_feat_grad)?(?:_f32_depth)?_kernel)<\s*([\w ]+?)\s*,\s*(?:\(int\))?\s*(\d+)\s*>")


def _type_tag(t):
    return "bf16" if "bfloat16" in t else "f16" if "half" in t else "f32" if "float" in t else t


def _names(names):
    """{kernel: [(type tag, VEC), ...]} from recorded kernel names such as bev_pool_f32_depth_kernel<__half, 8>."""
    out = {}
    for n in names:
        m = _KERNEL.search(n)
        if m:
            out.setdefault(m.group(1), []).append((_type_tag(m.group(2)), int(m.group(3))))
    return out


def record_kernels():
    """{case id: {kernel: [[type tag, VEC], ...]}}: every case run once under a CUDA activity trace."""
    out = {}
    for case in CASES:
        _, names = kernels_recorded(lambda: _run_case(case), lambda ns: len(_names(ns)) == 3)
        out[_id(case)] = {k: sorted(set(v)) for k, v in _names(names).items()}
    return out


@pytest.fixture(scope="module")
def recorded():
    """record_kernels() in a child process, for the reason tests/test_bev_pool_sweep_gpu.py's fixture gives: CUDA
    activity traces taken in the test process can leave a later test's trace without kernel records."""
    code = f"import json, sys; sys.path.insert(0, {ROOT!r}); from tests.test_bev_pool_mixed_gpu import record_kernels; " \
           "print(json.dumps(record_kernels()))"
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def _rounded(a, dtype):
    """float32 numpy -> a CPU tensor of ``dtype`` (round to nearest even; float32 as is)."""
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dtype)


def assert_bits(tag, got, want):
    assert got.dtype == want.dtype, (tag, got.dtype, want.dtype)
    g, w = got.detach().cpu().reshape(want.shape), want
    same = g.view(BITS[g.dtype]) == w.view(BITS[w.dtype])
    assert bool(same.all()), f"{tag}: {int((~same).sum())} of {same.numel()} elements differ in their bits"


def oracle_bits(pair, depth, feat, gout, ranks, hw, vd, Gd, vf, Gf):
    """(out, depth_grad, feat_grad) as the kernels compute them, each in its dtype."""
    dd, fd = PAIRS[pair]
    out = _rounded(obev.bev_pool_f32_fma(depth, feat, ranks, hw), fd)
    wd, _ = obev.bev_pool_backward_f32_lanes(gout, depth, feat, ranks, hw, Gd, vd, feat_grad=False)
    _, wf = obev.bev_pool_backward_f32_lanes(gout, depth, feat, ranks, hw, Gf, vf, depth_grad=False)
    return out, _rounded(wd, dd), _rounded(wf, fd)


def float64_entries(depth, feat, gout, ranks, hw):
    """{name: element_bound entry} of out, depth_grad and feat_grad: the float64 result, the same op on magnitudes and
    the chain length (a cell's points, C, a feature row's points)."""
    rd, rf, rb, st, ln = ranks
    C, rows = feat.shape[-1], feat.size // feat.shape[-1]
    lo, hi = np.maximum(st, 0), np.minimum(st.astype(np.int64) + ln, rd.size)
    n_cell = np.zeros(hw[0] * hw[1])
    ok = (lo < hi) & (rb[np.minimum(lo, rd.size - 1)] >= 0) & (rb[np.minimum(lo, rd.size - 1)] < n_cell.size)
    n_cell[rb[lo[ok]]] = (hi - lo)[ok]
    n_row = np.bincount(rf[(rf >= 0) & (rf < rows)], minlength=rows)
    w64 = obev.bev_pool_f64(depth, feat, ranks, hw)
    s64 = obev.bev_pool_f64(np.abs(depth), np.abs(feat), ranks, hw)
    wd64, wf64 = obev.bev_pool_backward_f64(gout, depth, feat, ranks, hw)
    sd64, sf64 = obev.bev_pool_backward_f64(np.abs(gout), depth, np.abs(feat), ranks, hw)
    t = torch.from_numpy
    return {"out": {"r": t(w64), "mag": t(s64), "n": t(n_cell.reshape(1, hw[0], hw[1], 1)), "pmag": 0.0},
            "depth_grad": {"r": t(wd64), "mag": t(sd64), "n": C, "pmag": 0.0},
            "feat_grad": {"r": t(wf64), "mag": t(sf64), "n": t(n_row.reshape(feat.shape[:-1] + (1,)).astype(np.float64)), "pmag": 0.0}}


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=_id)
def test_launch_shape_bit_for_bit_and_within_float64_bound(case, recorded):
    pair, C, feat_off, gout_off = case
    ranks, _, _, hw = GEOMETRY
    depth, feat, gout = _inputs(pair, C, C)
    want_shapes = shapes_of(*case)
    names = kernel_names(pair)
    tag = TYPE_TAG[PAIRS[pair][1]]
    ran = {k: [tuple(x) for x in v] for k, v in recorded[_id(case)].items()}
    assert ran == {names[k]: [(tag, vec)] for k, (vec, _, _) in want_shapes.items()}, ran
    got, ptrs = _run_case(case)
    for k, p in ptrs.items():  # the offsets reach the widths shapes_of expects
        assert pick_vec(F16, C, p) == want_shapes[k][0], k
    (vd, Gd, _), (vf, Gf, _) = want_shapes["bev_pool_depth_grad"], want_shapes["bev_pool_feat_grad"]
    for name, g, w in zip(("out", "depth_grad", "feat_grad"), got,
                          oracle_bits(pair, depth, feat, gout, ranks, hw, vd, Gd, vf, Gf)):  # fmt: skip
        assert_bits(f"{_id(case)} {name}", g, w)
    for (name, ent), g in zip(float64_entries(depth, feat, gout, ranks, hw).items(), got):
        check(_id(case), name, g, ent, U32)
    assert np.count_nonzero(got[1].float().cpu().numpy()) > 0.9 * ranks[0].size


def _workload(pair, name="bevdet_r50", seed=5):
    """CUDA (depth, feat, out_grad) of a workload in the pair's dtypes, the ranks and the output size."""
    dd, fd = PAIRS[pair]
    depth, feat, ranks, hw = make_bev_pool_inputs(name, seed)
    gout = torch.randn(1, hw[0], hw[1], feat.shape[-1], generator=torch.Generator().manual_seed(seed + 1))
    return depth.to(dd).cuda(), feat.to(fd).cuda(), gout.to(fd).cuda(), [r.cuda() for r in ranks], hw


def _grads(depth, feat, gout, rk, hw, need=(True, True), fn=bt.bev_pool_v2):
    d = depth.detach().clone().requires_grad_(need[0])
    f = feat.detach().clone().requires_grad_(need[1])
    out = fn(d, f, *rk, *hw)
    out.backward(gout)
    return out.detach(), d.grad, f.grad


@pytest.mark.gpu
@pytest.mark.parametrize("pair", PAIRS)
def test_bevdet_r50_bit_for_bit_and_within_float64_bound(pair):
    depth, feat, gout, rk, hw = _workload(pair)
    got = _grads(depth, feat, gout, rk, hw)
    np_ = lambda t: t.float().cpu().numpy()  # noqa: E731
    ranks = [r.cpu().numpy() for r in rk]
    C = feat.shape[-1]
    v = 8  # C = 64, every tensor aligned: 8 two-byte elements per lane
    want = oracle_bits(pair, np_(depth), np_(feat), np_(gout), ranks, hw, v, group_size(C, v), v, group_size(C, v))
    for name, g, w in zip(("out", "depth_grad", "feat_grad"), got, want):
        assert_bits(f"{pair} {name}", g, w)
    for (name, ent), g in zip(float64_entries(np_(depth), np_(feat), np_(gout), ranks, hw).items(), got):
        check(pair, name, g, ent, U32)


NONFINITE_CASES = [(pair, C, go) for pair in PAIRS for C, go in ((24, 0), (64, 3))]


@pytest.mark.gpu
@pytest.mark.parametrize("pair,C,gout_off", NONFINITE_CASES, ids=lambda v: str(v))
@pytest.mark.parametrize("value", [float("nan"), float("inf")])
def test_non_finite_stays_where_float64_puts_it(pair, C, gout_off, value):
    """One non-finite value in depth, in one feat row and in out_grad (one cell, one channel): the non-finite elements of
    the output and of both gradients are exactly float64's, and every other element keeps the clean run's bits."""
    dd, fd = PAIRS[pair]
    ranks, depth_size, rows, hw = GEOMETRY
    rd, rf, rb, st, ln = ranks
    depth, feat, gout = _inputs(pair, C, 11)
    rk = [torch.from_numpy(r).cuda() for r in ranks]

    def run(depth, feat, gout):
        d = at_offset(depth, 0, dd).requires_grad_(True)
        f = at_offset(feat, 0, fd).requires_grad_(True)
        out = bt.bev_pool_v2(d, f, *rk, *hw)
        out.backward(at_offset(gout, gout_off, fd))
        return [t.detach().float().cpu().numpy().reshape(-1) for t in (out, d.grad, f.grad)]

    clean = run(depth, feat, gout)
    kept = np.flatnonzero((rd >= 0) & (rd < depth_size) & (rf >= 0) & (rf < rows))
    i_cell, i_row, i_depth = (kept[np.searchsorted(kept, st[k])] for k in (3, 8, 12))  # in kept intervals
    depth2, feat2, gout2 = depth.copy(), feat.copy(), gout.copy()
    gout2.reshape(-1, C)[rb[i_cell], C // 2] = value
    feat2[rf[i_row], C - 1] = value
    depth2[rd[i_depth]] = value
    got = run(depth2, feat2, gout2)
    with np.errstate(invalid="ignore"):
        want = [obev.bev_pool_f64(depth2, feat2, ranks, hw)]
        want += list(obev.bev_pool_backward_f64(gout2, depth2, feat2, ranks, hw))
    for name, g, c, w in zip(("out", "depth_grad", "feat_grad"), got, clean, want):
        bad = ~np.isfinite(w.reshape(-1))
        assert 0 < bad.sum() < bad.size, name
        assert np.array_equal(~np.isfinite(g), bad), name
        assert np.array_equal(g[~bad].view(np.uint32), c[~bad].view(np.uint32)), name


def _abi_forward(pair, depth, feat, ranks, hw, out):
    """The pair's forward entry into a caller-owned output buffer."""
    name, _, lead = _entries(depth, feat)
    C = feat.shape[-1]
    st = getattr(_lib.load(), name)(*lead, depth.data_ptr(), feat.data_ptr(), *(r.data_ptr() for r in ranks), C,
                                    ranks[0].numel(), ranks[3].numel(), depth.numel(), feat.numel() // C, hw[0], hw[1],
                                    out.data_ptr(), _lib.current_stream_ptr())  # fmt: skip
    assert st == 0, st


@pytest.mark.gpu
@pytest.mark.parametrize("pair", PAIRS)
def test_out_of_range_indices_are_dropped(pair):
    """tests/test_bev_pool_gpu.py's case: ranks past either end of depth and feat, intervals naming cells outside the
    output, a start before 0, a length past P and an interval wholly past the points. No write lands outside the
    output; the output and both gradients equal the oracles bit for bit."""
    dd, fd = PAIRS[pair]
    depth, feat, ranks, hw = make_bev_pool_inputs("tiny", 3)
    depth, feat = depth.to(dd), feat.to(fd)
    rd, rf, rb, st, ln = (r.clone() for r in ranks)
    P, I = rd.numel(), st.numel()
    g = torch.Generator().manual_seed(9)
    pick = torch.randperm(P, generator=g)
    rd[pick[:40]] = depth.numel() + torch.arange(40, dtype=torch.int32)  # past the end
    rd[pick[40:60]] = -1
    rf[pick[60:100]] = feat.numel() // feat.shape[-1]
    rf[pick[100:110]] = -7
    rb[st[5].long()] = hw[0] * hw[1]  # interval 5 names a cell past the output
    rb[st[6].long()] = -1
    st[7] = -3  # clipped at 0
    ln[I - 1] += 1000  # clipped at P
    st[8], ln[8] = P + 10, 4  # entirely past the points
    ranks = (rd, rf, rb, st, ln)
    C = feat.shape[-1]
    cells = hw[0] * hw[1] * C
    buf = torch.full((cells + 2 * 4096,), 12345.0, dtype=fd, device="cuda")
    out = buf[4096:4096 + cells].view(1, hw[0], hw[1], C)
    rk = [r.cuda() for r in ranks]
    _abi_forward(pair, depth.cuda(), feat.cuda(), rk, hw, out)
    torch.cuda.synchronize()
    assert torch.all(buf[:4096] == 12345.0) and torch.all(buf[4096 + cells:] == 12345.0)
    gout = torch.randn(1, hw[0], hw[1], C, generator=torch.Generator().manual_seed(2)).to(fd)
    got = _grads(depth.cuda(), feat.cuda(), gout.cuda(), rk, hw)
    assert torch.equal(got[0], out)
    np_ = lambda t: t.float().cpu().numpy()  # noqa: E731
    v = 8  # C = 16
    want = oracle_bits(pair, np_(depth), np_(feat), np_(gout), [r.numpy() for r in ranks], hw, v, group_size(C, v), v,
                       group_size(C, v))  # fmt: skip
    for name, g_, w in zip(("out", "depth_grad", "feat_grad"), got, want):
        assert_bits(f"{pair} {name}", g_, w)


@pytest.mark.gpu
@pytest.mark.parametrize("pair", PAIRS)
def test_same_bits_on_every_run_and_for_every_gradient_subset(pair):
    depth, feat, gout, rk, hw = _workload(pair, seed=8)
    out, dg, fg = _grads(depth, feat, gout, rk, hw)
    out2, dg2, fg2 = _grads(depth, feat, gout, rk, hw)
    assert torch.equal(out, out2) and torch.equal(dg, dg2) and torch.equal(fg, fg2)
    assert torch.equal(_grads(depth, feat, gout, rk, hw, (True, False))[1], dg)
    assert torch.equal(_grads(depth, feat, gout, rk, hw, (False, True))[2], fg)
    assert torch.equal(_grads(depth, feat, gout, rk, hw, fn=bt.bev_pool_v2_2)[1], dg)


DTYPE_ROWS = [((F32, F32), F32, F32, F32), ((F16, F16), F16, F16, F16), ((BF16, BF16), BF16, BF16, BF16),
              ((F32, F16), F16, F32, F16), ((F32, BF16), BF16, F32, BF16)]  # (depth, feat), out, depth_grad, feat_grad


@pytest.mark.gpu
@pytest.mark.parametrize("row", DTYPE_ROWS, ids=lambda r: f"{r[0][0]}-{r[0][1]}".replace("torch.", ""))
@pytest.mark.parametrize("fn", [bt.bev_pool_v2, bt.bev_pool_v2_2], ids=["bev_pool_v2", "bev_pool_v2_2"])
def test_output_and_gradient_dtypes(row, fn):
    (dd, fd), od, dgd, fgd = row
    depth, feat, ranks, hw = make_bev_pool_inputs("tiny", 1)
    d = depth.to(dd).cuda().requires_grad_(True)
    f = feat.to(fd).cuda().requires_grad_(True)
    out = fn(d, f, *[r.cuda() for r in ranks], *hw)
    assert out.dtype == od and out.shape == (1, hw[0], hw[1], feat.shape[-1])
    out.float().sum().backward()
    assert d.grad.dtype == dgd and f.grad.dtype == fgd
    assert d.grad.shape == depth.shape and f.grad.shape == feat.shape


@pytest.mark.gpu
@pytest.mark.parametrize("pair", [(F16, BF16), (BF16, F16), (F16, F32), (BF16, F32), (torch.float64, torch.float64),
                                  (F32, torch.float64), (torch.float64, F32)], ids=str)  # fmt: skip
@pytest.mark.parametrize("fn", [bt.bev_pool_v2, bt.bev_pool_v2_2], ids=["bev_pool_v2", "bev_pool_v2_2"])
def test_every_other_dtype_pair_is_unsupported(pair, fn):
    depth, feat, ranks, hw = make_bev_pool_inputs("tiny", 1)
    with pytest.raises(_lib.B200OpsError) as e:
        fn(depth.to(pair[0]).cuda(), feat.to(pair[1]).cuda(), *[r.cuda() for r in ranks], *hw)
    assert e.value.status == 1


# ---- autocast, end to end ------------------------------------------------------------------------------------------------
class _LSS(nn.Module):
    """A lift-splat view transformer in small: a Conv2d depth net whose first D channels are softmaxed into depth and
    whose other C channels are the features (channels last), BEV pooling, and a Conv2d on the BEV plane."""

    def __init__(self, c_in, D, C, c_out, ranks, hw, pool):
        super().__init__()
        self.depth_net = nn.Conv2d(c_in, D + C, 3, padding=1)
        self.bev = nn.Conv2d(C, c_out, 3, padding=1)
        self.D, self.ranks, self.hw, self.pool = D, ranks, hw, pool

    def forward(self, x):
        y = self.depth_net(x)
        depth = y[:, :self.D].softmax(dim=1)
        feat = y[:, self.D:].permute(0, 2, 3, 1)
        bev = self.pool(depth, feat, *self.ranks, *self.hw)
        return self.bev(bev.permute(0, 3, 1, 2))


@pytest.mark.gpu
@pytest.mark.parametrize("low", [F16, BF16], ids=["fp16", "bf16"])
def test_autocast_lss_step(low):
    """Under torch.autocast the op receives FP32 depth (softmax) and low-precision features (conv) and returns
    low-precision output. The parameter gradients are compared with the same module whose op is fed ``.float()``
    inputs. The two differ by at most one rounding of the op's output and one of its feature gradient to ``low``,
    each a relative change of at most u = U_DTYPE[low], which to first order moves a parameter gradient by at most
    u times its magnitude: the bar is 2 u max|g| per parameter tensor."""
    cfg = BEV_POOL_CONFIGS["tiny"]
    ranks = [r.cuda() for r in bev_pool_ranks(cfg)]
    seen = []

    def pool(depth, feat, *args):
        seen.append((depth.dtype, feat.dtype))
        return bt.bev_pool_v2(depth, feat, *args)

    def pool_f32(depth, feat, *args):
        return bt.bev_pool_v2(depth.float(), feat.float(), *args)

    torch.manual_seed(0)
    fh, fw = cfg.feat_hw
    x = torch.randn(cfg.cams, 8, fh, fw, device="cuda")
    w = torch.randn(1, 8, *cfg.out_hw, device="cuda")
    grads = []
    for fn in (pool, pool_f32):
        torch.manual_seed(1)
        m = _LSS(8, cfg.num_depth, cfg.channels, 8, ranks, cfg.out_hw, fn).cuda()
        with torch.autocast("cuda", dtype=low):
            out = m(x)
            loss = (out.float() * w).sum()
        loss.backward()
        grads.append({k: p.grad.detach().clone() for k, p in m.named_parameters()})
    assert seen == [(F32, low)], seen
    u = U_DTYPE[low]
    for k, ref in grads[1].items():
        err = float((grads[0][k] - ref).abs().max())
        bar = 2 * u * float(ref.abs().max())
        print(f"{low} {k}: max |diff| {err:.3e}, bar {bar:.3e}, ratio {err / bar:.3f}")
        assert float(ref.abs().max()) > 0, k
        assert err <= bar, (k, err, bar)
