"""BEVPoolV2 on the GPU: FP32 and INT8 bit for bit against the reference kernels' stored outputs and the C oracle, FP16
within budget and no worse than the reference's FP16 / half2 kernels, channel counts, interval shapes, the zero fill,
index safety, non-finite containment, and the backward against the float64 oracle."""
import ctypes
import os

import numpy as np
import pytest
import torch

import bevformer_tensorrt_b200 as bt
from bevformer_tensorrt_b200 import _lib
from bevformer_tensorrt_b200.workloads import make_bev_pool_inputs, quantize_per_tensor
from oracle import bev_pool as obev
from tests.helpers import GOLDEN, fp16_tol, golden_index, input_digest

pytestmark = pytest.mark.gpu
WORKLOADS = ("tiny", "bevdet_r50", "ref_test")


def _kept(name, a):
    flat = np.asarray(a).reshape(-1)
    return flat if name == "tiny" else flat[golden_index(flat.size)]


def _np(ranks):
    return [r.cpu().numpy() for r in ranks]


def _cuda(ranks):
    return [r.cuda() for r in ranks]


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "ref_bev_pool.npz"))


@pytest.mark.parametrize("name", WORKLOADS)
def test_fp32_and_int8_bit_identical_to_reference(golden, name):
    depth, feat, ranks, hw = make_bev_pool_inputs(name, 0)
    assert input_digest(depth, feat, *ranks) == str(golden[f"{name}_digest"])
    got = bt.bev_pool_v2(depth.cuda(), feat.cuda(), *_cuda(ranks), *hw)
    assert got.shape == (1, hw[0], hw[1], feat.shape[-1]) and got.dtype == torch.float32
    assert np.array_equal(_kept(name, got.cpu().numpy()).view(np.uint32), golden[f"{name}_f32"].view(np.uint32))
    want = obev.bev_pool_f32_fma(depth.numpy(), feat.numpy(), _np(ranks), hw)  # the whole output
    assert np.array_equal(got.cpu().numpy().view(np.uint32), want.view(np.uint32))
    dq, sd = quantize_per_tensor(depth)
    fq, sf = quantize_per_tensor(feat)
    so = float(golden[f"{name}_i8_scales"][2])
    got8 = bt.bev_pool_v2_int8(dq.cuda(), sd, fq.cuda(), sf, *_cuda(ranks), so, *hw)
    assert np.array_equal(_kept(name, got8.cpu().numpy()).astype(np.float32), golden[f"{name}_i8"])
    assert np.array_equal(got8.cpu().numpy(), obev.bev_pool_i8(dq.numpy(), sd, fq.numpy(), sf, _np(ranks), so, hw))


@pytest.mark.parametrize("name", WORKLOADS)
def test_fp16_within_budget_and_not_worse_than_reference(golden, name):
    depth, feat, ranks, hw = make_bev_pool_inputs(name, 0)
    dh, fh = depth.half(), feat.half()
    want = obev.bev_pool_f64(dh.double().numpy(), fh.double().numpy(), _np(ranks), hw)
    for fn in (bt.bev_pool_v2, bt.bev_pool_v2_2):
        got = fn(dh.cuda(), fh.cuda(), *_cuda(ranks), *hw)
        assert got.dtype == torch.float16
        err = float(np.abs(got.double().cpu().numpy() - want).max())
        assert err <= fp16_tol(want), (err, fp16_tol(want))
        ours = np.abs(_kept(name, got.double().cpu().numpy()) - _kept(name, want)).max()
        for ref in ("f16", "h2"):
            theirs = np.abs(golden[f"{name}_{ref}"].astype(np.float64) - _kept(name, want)).max()
            assert ours <= theirs, (ref, ours, theirs)


def _channel_case(C, seed=0):
    depth, feat, ranks, hw = make_bev_pool_inputs("tiny", seed)
    g = torch.Generator().manual_seed(seed + 100)
    return depth, torch.randn(*feat.shape[:-1], C, generator=g), ranks, hw


@pytest.mark.parametrize("C", [1, 3, 64, 80, 128, 256])
def test_channel_counts(C):
    depth, feat, ranks, hw = _channel_case(C)
    got = bt.bev_pool_v2(depth.cuda(), feat.cuda(), *_cuda(ranks), *hw)
    want = obev.bev_pool_f32_fma(depth.numpy(), feat.numpy(), _np(ranks), hw)
    assert np.array_equal(got.cpu().numpy().view(np.uint32), want.view(np.uint32))
    got16 = bt.bev_pool_v2(depth.half().cuda(), feat.half().cuda(), *_cuda(ranks), *hw)
    want64 = obev.bev_pool_f64(depth.half().double().numpy(), feat.half().double().numpy(), _np(ranks), hw)
    assert np.abs(got16.double().cpu().numpy() - want64).max() <= fp16_tol(want64)


@pytest.mark.parametrize("C", [4, 8, 12, 20, 64, 80, 256])
def test_int8_channel_counts(C):
    depth, feat, ranks, hw = _channel_case(C, 1)
    dq, sd = quantize_per_tensor(depth)
    fq, sf = quantize_per_tensor(feat)
    so = 0.05
    got = bt.bev_pool_v2_int8(dq.cuda(), sd, fq.cuda(), sf, *_cuda(ranks), so, *hw)
    assert np.array_equal(got.cpu().numpy(), obev.bev_pool_i8(dq.numpy(), sd, fq.numpy(), sf, _np(ranks), so, hw))
    if C % 8 == 4:
        with pytest.raises(_lib.B200OpsError):
            bt.bev_pool_v2_int8(dq.cuda(), sd, fq[..., :-2].contiguous().cuda(), sf, *_cuda(ranks), so, *hw)


def _intervals(cells):
    """ranks_bev = cells (sorted), one interval per distinct cell."""
    cells = torch.as_tensor(cells, dtype=torch.int64)
    first = torch.ones(cells.numel(), dtype=torch.bool)
    first[1:] = cells[1:] != cells[:-1]
    starts = torch.nonzero(first).flatten()
    lengths = torch.diff(starts, append=torch.tensor([cells.numel()]))
    return cells.int(), starts.int(), lengths.int()


@pytest.mark.parametrize("shape", ["no_intervals", "length_one", "one_long", "wide"])
def test_interval_shapes(shape):
    g = torch.Generator().manual_seed(5)
    N, D, H, W, C = 2, 40, 8, 12, 24
    hw = (7, 19)
    depth, feat = torch.rand(N, D, H, W, generator=g), torch.randn(N, H, W, C, generator=g)
    if shape == "no_intervals":
        P = 50
        rb, st, ln = torch.zeros(P, dtype=torch.int32), torch.zeros(0, dtype=torch.int32), torch.zeros(0, dtype=torch.int32)
    elif shape == "length_one":
        P = 100
        rb, st, ln = _intervals(torch.sort(torch.randperm(hw[0] * hw[1], generator=g)[:P]).values)
    elif shape == "one_long":  # several thousand points pooled into one cell
        P = 6000
        rb, st, ln = _intervals(torch.full((P,), 77))
    else:  # every cell, uneven lengths
        P = 3000
        rb, st, ln = _intervals(torch.sort(torch.randint(0, hw[0] * hw[1], (P,), generator=g)).values)
    rd = torch.randperm(depth.numel(), generator=g)[:P].int()
    rf = torch.randint(0, N * H * W, (P,), generator=g).int()
    ranks = (rd, rf, rb, st, ln)
    got = bt.bev_pool_v2(depth.cuda(), feat.cuda(), *_cuda(ranks), *hw)
    want = obev.bev_pool_f32_fma(depth.numpy(), feat.numpy(), _np(ranks), hw)
    assert np.array_equal(got.cpu().numpy().view(np.uint32), want.view(np.uint32))
    if shape == "no_intervals":
        assert not got.any()


def _abi_forward(depth, feat, ranks, hw, out, stream):
    """b200_bev_pool_f32 / _f16 into a caller-owned output buffer."""
    name = "b200_bev_pool_f32" if feat.dtype == torch.float32 else "b200_bev_pool_f16"
    C = feat.shape[-1]
    st = getattr(_lib.load(), name)(depth.data_ptr(), feat.data_ptr(), *(r.data_ptr() for r in ranks), C,
                                    ranks[0].numel(), ranks[3].numel(), depth.numel(), feat.numel() // C, hw[0], hw[1],
                                    out.data_ptr(), ctypes.c_void_p(stream.cuda_stream))  # fmt: skip
    assert st == 0


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_garbage_output_buffer_on_a_side_stream_ends_zero_where_uncovered(dtype):
    depth, feat, ranks, hw = make_bev_pool_inputs("tiny", 2, dtype)
    d, f, rk = depth.cuda(), feat.cuda(), _cuda(ranks)
    out = torch.full((1, hw[0], hw[1], feat.shape[-1]), float("nan"), dtype=dtype, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _abi_forward(d, f, rk, hw, out, s)
    s.synchronize()
    want = bt.bev_pool_v2(d, f, *rk, *hw)
    assert torch.equal(out, want)
    covered = torch.zeros(hw[0] * hw[1], dtype=torch.bool)
    covered[ranks[2][ranks[3].long()].long()] = True
    assert not out.view(-1, feat.shape[-1])[~covered.cuda()].any()
    assert covered.sum() < covered.numel()  # the case has uncovered cells


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_out_of_range_indices_are_dropped(dtype):
    depth, feat, ranks, hw = make_bev_pool_inputs("tiny", 3, dtype)
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
    buf = torch.full((cells + 2 * 4096,), 12345.0, dtype=dtype, device="cuda")
    out = buf[4096:4096 + cells].view(1, hw[0], hw[1], C)
    _abi_forward(depth.cuda(), feat.cuda(), _cuda(ranks), hw, out, torch.cuda.current_stream())
    torch.cuda.synchronize()
    assert torch.all(buf[:4096] == 12345.0) and torch.all(buf[4096 + cells:] == 12345.0)
    if dtype == torch.float32:
        want = obev.bev_pool_f32_fma(depth.numpy(), feat.numpy(), _np(ranks), hw)
        assert np.array_equal(out.cpu().numpy().view(np.uint32), want.view(np.uint32))
    else:
        want = obev.bev_pool_f64(depth.double().numpy(), feat.double().numpy(), _np(ranks), hw)
        assert np.abs(out.double().cpu().numpy() - want).max() <= fp16_tol(want)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_non_finite_values_reach_only_their_intervals(dtype):
    depth, feat, ranks, hw = make_bev_pool_inputs("tiny", 4, dtype)
    clean = bt.bev_pool_v2(depth.cuda(), feat.cuda(), *_cuda(ranks), *hw)
    rd, rf, rb, st, ln = ranks
    bad_row = int(rf[len(rf) // 2])
    bad_depth = int(rd[len(rd) // 3])
    feat2, depth2 = feat.clone(), depth.clone()
    feat2.view(-1, feat.shape[-1])[bad_row, ::3] = float("inf")
    feat2.view(-1, feat.shape[-1])[bad_row, 1::3] = float("nan")
    depth2.view(-1)[bad_depth] = float("nan")
    got = bt.bev_pool_v2(depth2.cuda(), feat2.cuda(), *_cuda(ranks), *hw)
    hit = torch.zeros(hw[0] * hw[1], dtype=torch.bool)
    for k in range(st.numel()):
        s, n = int(st[k]), int(ln[k])
        if (rf[s:s + n] == bad_row).any() or (rd[s:s + n] == bad_depth).any():
            hit[int(rb[s])] = True
    g2, c2 = got.view(hw[0] * hw[1], -1).cpu(), clean.view(hw[0] * hw[1], -1).cpu()
    assert torch.equal(g2[~hit], c2[~hit])
    assert not torch.isfinite(g2[hit]).all(dim=1).any()


def _backward(dtype, depth, feat, ranks, hw, gout, need=(True, True)):
    d = depth.cuda().requires_grad_(need[0])
    f = feat.cuda().requires_grad_(need[1])
    out = bt.bev_pool_v2(d, f, *_cuda(ranks), *hw)
    out.backward(gout.cuda())
    return d.grad, f.grad


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("name", ["tiny", "bevdet_r50"])
def test_backward_against_float64_oracle(dtype, name):
    depth, feat, ranks, hw = make_bev_pool_inputs(name, 5, dtype)
    gout = torch.randn(1, hw[0], hw[1], feat.shape[-1], generator=torch.Generator().manual_seed(6)).to(dtype)
    dg, fg = _backward(dtype, depth, feat, ranks, hw, gout)
    assert dg.dtype == dtype and fg.dtype == dtype
    wd, wf = obev.bev_pool_backward_f64(gout.double().numpy(), depth.double().numpy(), feat.double().numpy(),
                                        _np(ranks), hw)  # fmt: skip
    tol = 2e-6 if dtype == torch.float32 else 2e-3
    for got, want in ((dg, wd), (fg, wf)):
        err = float(np.abs(got.double().cpu().numpy() - want).max() / np.abs(want).max())
        assert err < tol, err
    # zero where no pooled point refers
    used_d = torch.zeros(depth.numel(), dtype=torch.bool)
    used_d[ranks[0].long()] = True
    used_f = torch.zeros(feat.numel() // feat.shape[-1], dtype=torch.bool)
    used_f[ranks[1].long()] = True
    assert not dg.view(-1)[~used_d.cuda()].any() and not fg.view(-1, feat.shape[-1])[~used_f.cuda()].any()
    assert (~used_d).any()
    # the same bits on a second run and for each single gradient
    dg2, fg2 = _backward(dtype, depth, feat, ranks, hw, gout)
    assert torch.equal(dg, dg2) and torch.equal(fg, fg2)
    assert torch.equal(_backward(dtype, depth, feat, ranks, hw, gout, (True, False))[0], dg)
    assert torch.equal(_backward(dtype, depth, feat, ranks, hw, gout, (False, True))[1], fg)


def test_backward_fp32_close_to_reference_kernel(golden):
    depth, feat, ranks, hw = make_bev_pool_inputs("tiny", 0)
    gout = torch.randn(1, hw[0], hw[1], feat.shape[-1], generator=torch.Generator().manual_seed(1))
    dg, fg = _backward(torch.float32, depth, feat, ranks, hw, gout)
    np.testing.assert_allclose(dg.cpu().numpy().reshape(-1), golden["tiny_dgrad"], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(fg.cpu().numpy().reshape(-1), golden["tiny_fgrad"], rtol=1e-5, atol=1e-6)


def test_backward_with_out_of_range_indices_matches_oracle():
    depth, feat, ranks, hw = make_bev_pool_inputs("tiny", 7)
    rd, rf, rb, st, ln = (r.clone() for r in ranks)
    rd[::50] = -2
    rf[3::70] = 10**6
    rb[st[4].long()] = 10**6
    ranks = (rd, rf, rb, st, ln)
    gout = torch.randn(1, hw[0], hw[1], feat.shape[-1], generator=torch.Generator().manual_seed(2))
    dg, fg = _backward(torch.float32, depth, feat, ranks, hw, gout)
    wd, wf = obev.bev_pool_backward_f64(gout.double().numpy(), depth.double().numpy(), feat.double().numpy(),
                                        _np(ranks), hw)  # fmt: skip
    assert np.abs(dg.double().cpu().numpy() - wd).max() / np.abs(wd).max() < 2e-6
    assert np.abs(fg.double().cpu().numpy() - wf).max() / np.abs(wf).max() < 2e-6
