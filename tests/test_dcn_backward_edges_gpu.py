"""DCNv2 backward (csrc/dcn_backward.cu) at the inputs where a bilinear backward goes wrong and random offsets never land:
sample positions on integers (where the offset derivative jumps: mmcv's rule takes the forward difference), exactly on
-1, 0, H-1 and H (where the range rule changes), the zero-offset state every DCNv2 training run starts from, FP16 for
every geometry, and 25 to 75 taps. Oracle: tests/test_dcn_backward_gpu.py's float64 torchvision autograd with mmcv's
rule at -1.

The exact probe picks inputs on which every term of every accumulator is a short dyadic rational (integer pixels,
weights in multiples of 1/8, integer grad_output, masks in multiples of 1/4, integer or half-integer sample positions,
so every corner weight is a multiple of 1/4). Every term then lies on the 2^-7 grid, and when every accumulator's
sum of |term| stays below 2^24 grid units every partial sum is exact in fp32, in any order, atomics included. So the
FP32 results must equal the float64 oracle bit for bit, and the FP16 results the oracle rounded once to FP16.

A Python restatement of the backward's launch plan (bw_plan) checks the workspace query and shows which branches of the
plan (channels per K block, tap passes, ragged splits) the GPU cases reach; each GPU case's id names them."""
import numpy as np
import pytest
import torch
from torch.nn.modules.utils import _pair

import bevformer_tensorrt_b200 as bt
from bevformer_tensorrt_b200 import _lib
from tests.helpers import DCN_CASES, fp16_tol, make_dcn_inputs
from tests.test_dcn_backward_gpu import NAMES, _fp16_bar, _grad_out, _input_bar, _max_err, _oracle_grads, _our_grads

# ---- the launch plan, restated ---------------------------------------------------------------------------------------
# pixels per tile, K block rows, data-kernel M step, CTA target, sizeof(BwTap)
_BT, _RB, _MC, _TARGET, _TAP_BYTES = 64, 48, 32, 512, 20


def _cdiv(a, b):
    return -(-a // b)


def _out_hw(geo):
    n, c, h, w, co, kh, kw, s, p, d, g, dg = geo
    (sh, sw), (ph, pw), (dh, dw) = _pair(s), _pair(p), _pair(d)
    return (h + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1, (w + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1


def _plan(geo, f16):
    """bw_plan: channels per K block (KC), tap passes, data / weight splits, workspace sections and the data kernel's
    dynamic shared memory; total 0 where the library returns UNSUPPORTED."""
    n, c, h, w, co, kh, kw, *_, g, dg = geo
    ho, wo = _out_hw(geo)
    P, kk, cg, cpd, mg = ho * wo, kh * kw, c // g, c // dg, co // g
    kc = 16
    while kc > 1 and (kc * kk > _RB or cg % kc or cpd % kc):
        kc //= 2
    npass = 1 if kc > 1 else _cdiv(kk, _RB)
    ptiles, nch = _cdiv(P, _BT), cpd // kc
    nsplit = min(nch, max(1, _cdiv(_TARGET, dg * ptiles)))
    wbase = _cdiv(mg, 64) * g * (cg // kc) * npass
    items = n * ptiles
    wsplit = min(items, max(1, _cdiv(4 * _TARGET, wbase)))
    a256 = lambda b: _cdiv(b, 256) * 256  # noqa: E731
    sections = (a256(n * c * h * w * 4) if f16 else 0, a256(n * dg * nsplit * 3 * kk * P * 4),
                a256(wsplit * co * cg * kk * 4))  # fmt: skip
    smem = (_MC * _BT + _MC * _RB + 3 * _RB * _BT + 3 * kk * _BT) * 4 + kk * _BT * _TAP_BYTES
    ok = wbase <= 65535 and smem <= 200 * 1024
    return dict(KC=kc, npass=npass, nch=nch, nsplit=nsplit, items=items, wsplit=wsplit, sections=sections, smem=smem,
                total=sum(sections) if ok else 0)  # fmt: skip


def _ragged(n, splits):
    return splits > 1 and n % splits != 0


def _branch_id(name, geo):
    pl = _plan(geo, False)
    ns = f"ns{pl['nsplit']}" + ("r" if _ragged(pl["nch"], pl["nsplit"]) else "")
    ws = f"ws{pl['wsplit']}" + ("r" if _ragged(pl["items"], pl["wsplit"]) else "")
    return f"{name}-KC{pl['KC']}-np{pl['npass']}-{ns}-{ws}"


def _kw(geo):
    *_, s, p, d, g, dg = geo
    return dict(stride=s, padding=p, dilation=d, groups=g, deform_groups=dg)


# geometry: (N, Ci, H, W, Co, kh, kw, stride, padding, dilation, groups, deform_groups), as tests/helpers.DCN_CASES
EXACT_CASES = {
    "k1_co100_dg2": (2, 32, 11, 13, 100, 1, 1, 1, 0, 1, 1, 2),  # KC 16, one chunk per deformable group: nsplit 1
    "k2x3_g2_dg2_co12": (2, 16, 12, 15, 12, 2, 3, 1, 1, 1, 2, 2),  # KC 8, 48-row K blocks, Mg = 6
    "asym_g2_dg4": (2, 16, 15, 19, 12, 3, 3, (2, 1), (1, 2), (1, 2), 2, 4),  # KC 4, every geometry pair asymmetric
    "k3x5": (1, 8, 11, 13, 8, 3, 5, 1, (1, 2), 1, 1, 1),  # KC 2
    "k5_ragged": (4, 24, 40, 40, 16, 5, 5, 1, 2, 1, 1, 1),  # KC 1, one pass; ragged data and weight splits
    "k7_g2_dg2_1tile": (1, 8, 8, 8, 12, 7, 7, 1, 3, 1, 2, 2),  # two tap passes, one pixel tile: wsplit 1
    "fused_co128": (1, 64, 12, 14, 128, 3, 3, 1, 1, 1, 1, 1),  # the FP16 forward takes the wgmma kernel
}
TAP_CASES = {
    "k5x5": (2, 8, 14, 15, 8, 5, 5, 1, 2, 1, 2, 2),  # 25 taps, KC 1, one pass
    "k6x8": (1, 8, 13, 16, 12, 6, 8, 1, (2, 3), 1, 1, 2),  # 48 taps: one full K block
    "k7x7": (1, 4, 15, 16, 8, 7, 7, 1, 3, 1, 2, 1),  # 49 taps: two passes
    "k8x9": (1, 4, 16, 18, 6, 8, 9, 1, 4, 1, 1, 2),  # 72 taps
    "k5x15": (1, 4, 12, 24, 8, 5, 15, 1, (2, 7), 1, 2, 2),  # 75 taps: 200 KB of data-kernel shared memory
    "k15x5": (1, 4, 24, 12, 8, 15, 5, 1, (7, 2), 1, 1, 4),
}
INIT_CASES = {  # zero-offset state: border taps on -1 / -2 and H / H+1
    "p1": (2, 16, 13, 17, 12, 3, 3, 1, 1, 1, 2, 2),
    "p2_d2": (1, 16, 12, 12, 8, 3, 3, 1, 2, 2, 1, 4),
    "p2_k5": (1, 8, 11, 14, 8, 5, 5, 1, 2, 1, 1, 1),
}
# the shapes tests/test_dcn_backward_gpu.py runs outside DCN_CASES: the base backbone layer and the DCNv2P module test
_OTHER_GEOMETRIES = [(6, 256, 58, 100, 256, 3, 3, 1, 1, 1, 1, 1), (2, 32, 23, 31, 64, 3, 3, 1, 1, 1, 1, 2)]
_MODULE_GEO = (2, 16, 13, 15, 24, 3, 3, 1, 1, 1, 2, 2)


def _ws_query(geo, f16):
    n, c, h, w, co, kh, kw, s, p, d, g, dg = geo
    (sh, sw), (ph, pw), (dh, dw) = _pair(s), _pair(p), _pair(d)
    return _lib.load().b200_dcn_backward_workspace_size(int(f16), n, c, h, w, co, kw, kh, sw, sh, pw, ph, dw, dh, g, dg)


# ---- CPU: the plan mirror --------------------------------------------------------------------------------------------
def test_plan_mirror_matches_the_workspace_query():
    geos = (list(DCN_CASES.values()) + list(EXACT_CASES.values()) + list(TAP_CASES.values()) + list(INIT_CASES.values())
            + _OTHER_GEOMETRIES + [_MODULE_GEO])  # fmt: skip
    for geo in geos:
        for f16 in (False, True):
            pl = _plan(geo, f16)
            assert pl["total"] > 0 and _ws_query(geo, f16) == pl["total"], (geo, f16, pl)
    for kh, kw in ((5, 15), (15, 5), (8, 9)):  # supported up to exactly the 200 KB data-kernel cap
        assert _plan(TAP_CASES[f"k{kh}x{kw}"], False)["smem"] <= 200 * 1024
    assert _plan(TAP_CASES["k5x15"], False)["smem"] == 200 * 1024
    for kh, kw in ((4, 19), (9, 9), (1, 76)):  # 76 and 81 taps: UNSUPPORTED, in the mirror and the library
        geo = (1, 8, 24, 80, 8, kh, kw, 1, (kh // 2, kw // 2), 1, 1, 1)
        assert _plan(geo, False)["total"] == 0 and _ws_query(geo, False) == 0 and _ws_query(geo, True) == 0


def test_gpu_cases_reach_every_branch_of_the_plan():
    plans = {name: _plan(geo, False) for cases in (EXACT_CASES, TAP_CASES) for name, geo in cases.items()}
    assert {pl["KC"] for pl in plans.values()} == {16, 8, 4, 2, 1}
    assert {pl["npass"] for pl in plans.values()} == {1, 2}
    assert any(pl["nsplit"] == 1 for pl in plans.values())
    assert any(_ragged(pl["nch"], pl["nsplit"]) for pl in plans.values())
    assert any(pl["wsplit"] == 1 for pl in plans.values())
    assert any(_ragged(pl["items"], pl["wsplit"]) for pl in plans.values())
    # an exact-probe case whose partial sums cross ragged split boundaries on both reductions
    assert any(_ragged(plans[n]["nch"], plans[n]["nsplit"]) and _ragged(plans[n]["items"], plans[n]["wsplit"])
               for n in EXACT_CASES)  # fmt: skip
    # exact-probe coverage of the rest of the geometry: Mg not a multiple of 32, groups 2, deformable groups 2 and 4
    geos = EXACT_CASES.values()
    assert {geo[4] // geo[10] % 32 != 0 for geo in geos} == {True, False}
    assert {2} <= {geo[10] for geo in geos} and {2, 4} <= {geo[11] for geo in geos}
    assert any(not isinstance(geo[7], int) and not isinstance(geo[8], int) and not isinstance(geo[9], int) for geo in geos)


def test_exact_probe_inputs_meet_their_precondition():
    """The bitwise bar of the exact probe rests on the float64 oracle being exactly representable in fp32 and every
    accumulator staying exact; checked here on the CPU for every probe geometry (the GPU test checks it again)."""
    for name, geo in EXACT_CASES.items():
        x, off, mask, w, b, go = _exact_inputs(geo, seed=len(name))
        want_out, want = _oracle_grads(x, off, mask, w, b, go, _kw(geo))
        _assert_exact_precondition(x, off, mask, w, b, go, _kw(geo), want_out, want)


# ---- the exact probe -------------------------------------------------------------------------------------------------
def _exact_inputs(geo, seed):
    """float64 CPU tensors x, offset, mask, weight, bias, grad_out on the grids named in the module docstring. Sample
    positions: a quarter from an edge set (far outside, -1.5, -1, -0.5, 0, 0.5 and the same about H-1 / H), the rest
    half-integers from -1.5 to H + 0.5; offset = position - base."""
    n, c, h, w, co, kh, kw, s, p, d, g, dg = geo
    (sh, sw), (ph, pw), (dh, dw) = _pair(s), _pair(p), _pair(d)
    ho, wo = _out_hw(geo)
    kk = kh * kw
    rng = np.random.default_rng(seed)

    def positions(size):
        edges = np.array([-40.0, -1.5, -1.0, -0.5, 0.0, 0.5, size - 1.5, size - 1.0, size - 0.5, size, size + 0.5, size + 37])
        inside = rng.integers(-3, 2 * size + 2, (n, dg, kk, ho, wo)) / 2.0
        return np.where(rng.random(inside.shape) < 0.25, rng.choice(edges, inside.shape), inside)

    t = np.arange(kk)
    base_h = (np.arange(ho) * sh - ph)[None, :, None] + (t // kw * dh)[:, None, None]  # [kk, Ho, 1]
    base_w = (np.arange(wo) * sw - pw)[None, None, :] + (t % kw * dw)[:, None, None]  # [kk, 1, Wo]
    off = np.stack([positions(h) - base_h, positions(w) - base_w], 3).reshape(n, dg * 2 * kk, ho, wo)
    x = rng.integers(-4, 5, (n, c, h, w)).astype(np.float64)
    mask = rng.choice([0.0, 0.25, 0.5, 0.75, 1.0, 1.25, -0.5], (n, dg * kk, ho, wo))
    wt = rng.integers(-8, 9, (co, c // g, kh, kw)) / 8.0
    bias = rng.integers(-16, 17, co) / 8.0
    go = rng.integers(-2, 3, (n, co, ho, wo)).astype(np.float64)
    return [torch.from_numpy(a) for a in (x, off, mask, wt, bias, go)]


_GRID = 2.0**-7  # every term of every accumulator is a multiple of this


def _assert_exact_precondition(x, off, mask, w, b, go, kw, want_out, want):
    for name, r in zip(("out",) + NAMES, [want_out] + want):
        assert torch.equal(r, r.float().double()), f"oracle {name} is not fp32-representable"
    # the inputs are on their grids: x integer, 8 w, 8 b, 4 mask, 2 offset and grad_out integer
    for t, k in ((x, 1), (w, 8), (b, 8), (mask, 4), (off, 2), (go, 1)):
        assert torch.equal(t * k, (t * k).round())
    # sum of |term| of every accumulator. gc[(c, t), p] = sum_m W g: A = |W|^T |grad_out| per group bounds |gc|. With |x|,
    # |mask|, |W|, |bias|, |grad_out| the oracle's out, grad_input, grad_mask, grad_weight and grad_bias are those sums
    # (corner weights are >= 0); an offset term is |gc| |mask| times a coordinate-weight difference <= 2 max|x|.
    n, c = x.shape[:2]
    co, cg, kh, kw_ = w.shape
    g, dg, kk = c // cg, kw["deform_groups"], kh * kw_
    P = go.shape[2] * go.shape[3]
    wa = w.abs().reshape(g, co // g, cg * kk)
    ga = go.abs().reshape(n, g, co // g, P)
    A = torch.einsum("gmk,ngmp->ngkp", wa, ga).reshape(n, dg, c // dg, kk, P)
    sums = [A.max(), 2 * x.abs().max() * mask.abs().max() * A.sum(2).max()]
    out_abs, abs_grads = _oracle_grads(x.abs(), off, mask.abs(), w.abs(), b.abs(), go.abs(), kw)
    sums += [out_abs.max()] + [abs_grads[i].max() for i in (0, 2, 3, 4)]
    assert max(float(v) for v in sums) < 2.0**24 * _GRID, sums


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16], ids=["fp32", "fp16"])
@pytest.mark.parametrize("name", list(EXACT_CASES), ids=[_branch_id(n, g) for n, g in EXACT_CASES.items()])
def test_exact_probe_is_bitwise_equal_to_the_float64_oracle(name, dtype):
    geo = EXACT_CASES[name]
    kw = _kw(geo)
    x, off, mask, w, b, go = _exact_inputs(geo, seed=len(name))
    want_out, want = _oracle_grads(x, off, mask, w, b, go, kw)
    _assert_exact_precondition(x, off, mask, w, b, go, kw, want_out, want)
    out, got = _our_grads(*(t.to(dtype) for t in (x, off, mask, w, b, go)), kw)
    for gname, gt, r in zip(("out",) + NAMES, [out] + got, [want_out] + want):
        assert gt.dtype == dtype, gname
        r = r.to(dtype)
        gt = gt.cpu()
        assert torch.equal(gt, r), (gname, _max_err(gt, r), int((gt != r).sum()), r.numel())


# ---- the zero-offset initial state -----------------------------------------------------------------------------------
def _rand_inputs(geo, seed, dtype=torch.float32, offsets="randn"):
    """x, offset, mask, weight, bias, grad_out. offsets: 'randn' (x 1.5, sigmoid mask, as tests/helpers), 'zero' or 'int'
    (integers in [-2, 2]); the last two with mask exactly 0.5, as DCNv2P after init_weights."""
    n, c, h, w, co, kh, kw, *_, g, dg = geo
    ho, wo = _out_hw(geo)
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(n, c, h, w, generator=gen)
    oshape, mshape = (n, dg * 2 * kh * kw, ho, wo), (n, dg * kh * kw, ho, wo)
    if offsets == "randn":
        off, mask = torch.randn(oshape, generator=gen) * 1.5, torch.sigmoid(torch.randn(mshape, generator=gen))
    else:
        off = torch.zeros(oshape) if offsets == "zero" else torch.randint(-2, 3, oshape, generator=gen).float()
        mask = torch.full(mshape, 0.5)
    wt = torch.randn(co, c // g, kh, kw, generator=gen) / (c // g * kh * kw) ** 0.5
    b = torch.randn(co, generator=gen)
    go = torch.randn(n, co, ho, wo, generator=gen)
    return [t.to(dtype) for t in (x, off, mask, wt, b, go)]


def _check_against_oracle(geo, inputs, tag, op=None):
    """Forward output and all five gradients against the float64 oracle: FP32 at 1e-4 x max|g|, FP16 at _fp16_bar.
    `op` replaces modulated_deformable_conv2d (the …2 twin)."""
    x, off, mask, w, b, go = inputs
    kw = _kw(geo)
    want_out, want = _oracle_grads(x, off, mask, w, b, go, kw)
    if op is None:
        out, got = _our_grads(x, off, mask, w, b, go, kw)
    else:
        ts = [t.detach().cuda().requires_grad_(True) if t is not None else None for t in (x, off, mask, w, b)]
        out = op(*ts, kw["stride"], kw["padding"], kw["dilation"], kw["groups"], kw["deform_groups"])
        out.backward(go.cuda())
        out, got = out.detach(), [t.grad if t is not None else None for t in ts]
    f16 = x.dtype == torch.float16
    lines = []
    for name, gt, r in zip(("out",) + NAMES, [out] + got, [want_out] + want):
        if r is None:
            assert gt is None, name
            continue
        assert gt.dtype == x.dtype and gt.shape == r.shape, name
        err = _max_err(gt, r)
        if not f16:
            bar = 1e-4 * max(r.abs().max().item(), 1e-30)
        elif name == "out":  # the forward's FP16 budget (tests/test_dcn_gpu.py): the wgmma path rounds its columns to FP16
            bar = fp16_tol(r.numpy())
        else:
            bar = _fp16_bar(r)
        lines.append(f"{name} max {r.abs().max().item():.3g} err {err:.2e} bar {bar:.2e}")
        assert err <= bar, (tag, name, err, bar)
    print(f"[{tag}] " + "; ".join(lines))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16], ids=["fp32", "fp16"])
@pytest.mark.parametrize("offsets", ["zero", "int"])
@pytest.mark.parametrize("name", list(INIT_CASES))
def test_integer_sample_positions_with_mask_one_half(name, offsets, dtype):
    """Every sample on an integer position, where the offset derivative takes the forward difference, and the border
    taps exactly on -1 / -2 and H / H+1 (padding 1 and 2, dilation 2)."""
    geo = INIT_CASES[name]
    _check_against_oracle(geo, _rand_inputs(geo, seed=5, dtype=dtype, offsets=offsets), f"dcn bwd init {name} {offsets}")


class _MaskedOracle(torch.autograd.Function):
    """float64 torchvision forward; backward = _oracle_grads (mmcv's rule: no offset gradient for a sample exactly on
    h or w = -1, where plain torchvision differentiates the one corner inside the image)."""

    @staticmethod
    def forward(ctx, x, offset, mask, weight, bias, kw):
        import torchvision

        ctx.save_for_backward(x, offset, mask, weight, bias)
        ctx.kw = kw
        return torchvision.ops.deform_conv2d(x, offset, weight, bias, kw["stride"], kw["padding"], kw["dilation"], mask)

    @staticmethod
    def backward(ctx, grad_out):
        with torch.enable_grad():
            _, grads = _oracle_grads(*ctx.saved_tensors, grad_out, ctx.kw, device=grad_out.device)
        return (*grads, None)


@pytest.mark.gpu
@pytest.mark.parametrize("layer", ["DCNv2P", "DCNv2P2"])
def test_dcnv2p_from_init_weights_matches_float64_module_over_one_step(layer):
    """DCNv2P straight from init_weights (zero conv_offset: every offset 0, every mask 0.5, the padding-1 border taps on
    -1 and H) with a non-zero bias, against a float64 module on the masked oracle: parameter gradients at step 0, then
    after one SGD step (small non-integer offsets) at step 1."""
    from bevformer_tensorrt_b200.modules.cnn.dcn import CONV_LAYERS

    cls = CONV_LAYERS[layer]
    n, c, h, w, co, k, _, s, p, d, g, dg = _MODULE_GEO
    torch.manual_seed(4)
    ours = cls(c, co, k, stride=s, padding=p, dilation=d, groups=g, deform_groups=dg).cuda()
    with torch.no_grad():
        ours.bias.normal_()

    class Ref(cls):
        _op = staticmethod(lambda x, o, m, wt, b, s_, p_, d_, g_, dg_: _MaskedOracle.apply(
            x, o, m, wt, b, dict(stride=s_, padding=p_, dilation=d_)))  # fmt: skip

    ref = Ref(c, co, k, stride=s, padding=p, dilation=d, groups=g, deform_groups=dg).cuda().double()
    x = torch.randn(n, c, h, w, device="cuda")
    target = torch.randn(n, co, *_out_hw(_MODULE_GEO), device="cuda")
    opt = torch.optim.SGD(ours.parameters(), lr=2.0)
    # conv_offset is a plain FP32 convolution: no TF32, so its own rounding stays far below the bar
    with torch.backends.cudnn.flags(enabled=True, benchmark=False, deterministic=True, allow_tf32=False):
        for step in range(2):
            ref.load_state_dict({k_: v.double() for k_, v in ours.state_dict().items()})
            for mod, xin, tgt in ((ours, x, target), (ref, x.double(), target.double())):
                mod.zero_grad()
                torch.nn.functional.mse_loss(mod(xin), tgt).backward()
            for (pname, pa), (_, q) in zip(ours.named_parameters(), ref.named_parameters()):
                err, bar = _max_err(pa.grad, q.grad), 1e-4 * q.grad.abs().max().item()
                print(f"[dcn bwd {layer} step {step}] {pname} max {q.grad.abs().max().item():.3g} err {err:.2e} bar {bar:.2e}")
                assert q.grad.abs().max().item() > 0 and err <= bar, (step, pname, err, bar)
            if step == 0:
                assert not ours.conv_offset.weight.abs().any()
                opt.step()
        offs = ours.conv_offset(x).detach()
        assert offs.abs().max().item() < 1 and (offs != offs.round()).float().mean().item() > 0.9


# ---- FP16 for every DCN_CASES geometry -------------------------------------------------------------------------------
_TWIN_CASES = ("k3_s1_p1_g2_dg2", "gen_asym_g2_dg4", "fused_co128")


def _case_inputs(case, dtype):
    x, off, mask, w, b, _ = make_dcn_inputs(case, dtype=dtype)
    return [x, off, mask, w, b, _grad_out(case, dtype)]


@pytest.mark.gpu
@pytest.mark.parametrize("with_bias", [True, False], ids=["bias", "nobias"])
@pytest.mark.parametrize("case", list(DCN_CASES))
def test_fp16_grads_match_float64_oracle_for_every_case(case, with_bias):
    inputs = _case_inputs(case, torch.float16)
    if not with_bias:
        inputs[4] = None
    _check_against_oracle(DCN_CASES[case], inputs, f"dcn bwd fp16 {case} {'bias' if with_bias else 'nobias'}")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16], ids=["fp32", "fp16"])
@pytest.mark.parametrize("case", _TWIN_CASES)
def test_twin_op_shares_the_backward(case, dtype):
    """modulated_deformable_conv2d2 (plugin …TRT2) against the oracle, and bit for bit against modulated_deformable_conv2d
    (grad_input within _input_bar)."""
    inputs = _case_inputs(case, dtype)
    geo = DCN_CASES[case]
    _check_against_oracle(geo, inputs, f"dcn bwd twin {case}", op=bt.modulated_deformable_conv2d2)
    x, off, mask, w, b, go = inputs
    outs = []
    for op in (bt.modulated_deformable_conv2d, bt.modulated_deformable_conv2d2):
        ts = [t.cuda().requires_grad_(True) for t in (x, off, mask, w, b)]
        out = op(*ts, *(_kw(geo)[k] for k in ("stride", "padding", "dilation", "groups", "deform_groups")))
        out.backward(go.cuda())
        outs.append([out.detach()] + [t.grad for t in ts])
    for name, a, e in zip(("out",) + NAMES, *outs):
        if name == "input":
            assert _max_err(a, e) <= _input_bar(e)
        else:
            assert torch.equal(a, e), name


# ---- 25 to 75 taps ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16], ids=["fp32", "fp16"])
@pytest.mark.parametrize("name", list(TAP_CASES), ids=[_branch_id(n, g) for n, g in TAP_CASES.items()])
def test_large_kernels_match_float64_oracle(name, dtype):
    geo = TAP_CASES[name]
    _check_against_oracle(geo, _rand_inputs(geo, seed=9, dtype=dtype), f"dcn bwd {name} {str(dtype)[6:]}")


# ---- autograd plumbing -----------------------------------------------------------------------------------------------
def _grads_of(backward, x, off, mask, w, b, geo):
    """All five gradients of modulated_deformable_conv2d, with `backward(out)` driving autograd; also the strides of
    the gradient the op's backward received."""
    ts = [t.detach().cuda().requires_grad_(True) for t in (x, off, mask, w, b)]
    kw = _kw(geo)
    out = bt.modulated_deformable_conv2d(*ts, kw["stride"], kw["padding"], kw["dilation"], kw["groups"], kw["deform_groups"])
    seen = []
    out.register_hook(lambda g: seen.append(g.stride()))
    backward(out)
    return [t.grad for t in ts], seen[0]


def _assert_same(got, ref):
    for name, a, e in zip(NAMES, got, ref):
        if name == "input":
            assert _max_err(a, e) <= _input_bar(e), name
        else:
            assert torch.equal(a, e), name


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["gen_asym_g2_dg4", "fused_co128"])
def test_non_contiguous_grad_out(case):
    """out.sum() hands backward a stride-0 expansion; a channels-last consumer hands it an NHWC-strided gradient. Both
    give the gradients of the same values passed contiguous."""
    geo = DCN_CASES[case]
    x, off, mask, w, b, go = _case_inputs(case, torch.float32)
    ones, _ = _grads_of(lambda o: o.backward(torch.ones_like(o)), x, off, mask, w, b, geo)
    summed, st = _grads_of(lambda o: o.sum().backward(), x, off, mask, w, b, geo)
    assert st == (0, 0, 0, 0)
    _assert_same(summed, ones)
    go_c = go.cuda()
    plain, _ = _grads_of(lambda o: o.backward(go_c), x, off, mask, w, b, geo)
    go_cl = go_c.contiguous(memory_format=torch.channels_last)
    cl, st = _grads_of(lambda o: (o.contiguous(memory_format=torch.channels_last) * go_cl).sum().backward(),
                       x, off, mask, w, b, geo)  # fmt: skip
    assert st == go_cl.stride() != go_c.stride()
    _assert_same(cl, plain)


@pytest.mark.gpu
def test_fp32_channels_last_input():
    geo = DCN_CASES["gen_co100"]
    x, off, mask, w, b, go = _case_inputs("gen_co100", torch.float32)
    go_c = go.cuda()
    plain, _ = _grads_of(lambda o: o.backward(go_c), x, off, mask, w, b, geo)
    x_cl = x.cuda().contiguous(memory_format=torch.channels_last)
    cl, _ = _grads_of(lambda o: o.backward(go_c), x_cl, off, mask, w, b, geo)
    _assert_same(cl, plain)


@pytest.mark.gpu
def test_frozen_weights_request_only_offset_and_mask_gradients():
    """A DCNv2P with frozen weight / bias and an input that needs no gradient: the op is asked for the offset and mask
    gradients alone, and conv_offset's gradients are those of the full request, bit for bit."""
    from bevformer_tensorrt_b200.modules.cnn.dcn import ModulatedDeformConv2dPackPlugin

    torch.manual_seed(6)
    mod = ModulatedDeformConv2dPackPlugin(16, 32, 3, padding=1, deform_groups=2).cuda()
    with torch.no_grad():
        mod.conv_offset.weight.normal_(0, 0.05)
        mod.conv_offset.bias.normal_(0, 0.5)
    x = torch.randn(2, 16, 17, 19, device="cuda")
    target = torch.randn(2, 32, 17, 19, device="cuda")
    captured = []
    real_op = type(mod)._op

    def spy(*args):
        captured.append(args[1:3])
        for t in args[1:3]:
            t.retain_grad()
        return real_op(*args)

    mod._op = spy
    grads = []
    with torch.backends.cudnn.flags(enabled=True, benchmark=False, deterministic=True, allow_tf32=False):
        for frozen in (False, True):
            mod.weight.requires_grad_(not frozen)
            mod.bias.requires_grad_(not frozen)
            mod.zero_grad(set_to_none=True)
            torch.nn.functional.mse_loss(mod(x), target).backward()
            off, msk = captured[-1]
            grads.append((off.grad, msk.grad, mod.conv_offset.weight.grad, mod.conv_offset.bias.grad, mod.weight.grad))
    assert grads[1][4] is None and grads[0][4] is not None
    for name, a, e in zip(("offset", "mask", "conv_offset.weight", "conv_offset.bias"), grads[1][:4], grads[0][:4]):
        assert torch.equal(a, e), name
