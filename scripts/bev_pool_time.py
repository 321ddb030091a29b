"""Times BEVPoolV2 on the GPU: the forward in FP32 / FP16 / INT8 and the backward in FP32 / FP16, on the BEVDet-R50 and
reference-test workloads, against the reference's own kernels (oracle/_ref/libref_bev_pool.so, when built) and a torch
eager index_select / index_add_ baseline. CUDA events, a warm-up, then the median / min / max of three windows of
per-call times. Prints the card and its power limit, the workload statistics, the bytes each call moves (computed from
shapes: HBM-unique bytes and feat bytes gathered from L2, separately), one line per leg and one JSON line at the end.

The BF16 and FP32-depth legs (bf16 / bf16, fp32 depth + fp16 feat, fp32 depth + bf16 feat, forward and backward) are
timed against FP16 in the same call with their windows alternating (`*_alt` legs, seven windows each), so that the
comparison does not straddle a change in clocks or in other work on the card.

    python scripts/bev_pool_time.py [--iters 200]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bevformer_tensorrt_b200 as bt  # noqa: E402
from bevformer_tensorrt_b200 import _lib  # noqa: E402
from bevformer_tensorrt_b200.workloads import bev_pool_stats, make_bev_pool_inputs, quantize_per_tensor  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)  # fmt: skip
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, iters, windows=3):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    per = []
    for _ in range(windows):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        per.append(a.elapsed_time(b) * 1e3 / iters)
    per.sort()
    return {"median_us": round(per[len(per) // 2], 2), "min_us": round(per[0], 2), "max_us": round(per[-1], 2)}


def traffic(depth, feat, ranks, hw, elem):
    """HBM-unique bytes (depth and feat read once, index streams, the output zero-filled and written) and the feat rows
    gathered per point (mostly L2 hits: feat is small and every row is read by every depth bin that lands in the grid)."""
    C, P, I = feat.shape[-1], ranks[0].numel(), ranks[3].numel()
    out = hw[0] * hw[1] * C * elem
    hbm = depth.numel() * elem + feat.numel() * elem + 3 * P * 4 + 2 * I * 4 + 2 * out
    return {"hbm_unique_MB": round(hbm / 1e6, 1), "l2_gathered_MB": round(P * C * elem / 1e6, 1)}


def timed_alternating(legs, iters, windows=7):
    """{leg: median / min / max per-call µs}, each window of every leg timed in turn, after a warm-up of every leg."""
    for fn in legs.values():
        for _ in range(10):
            fn()
    torch.cuda.synchronize()
    per = {k: [] for k in legs}
    for _ in range(windows):
        for k, fn in legs.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                fn()
            b.record()
            b.synchronize()
            per[k].append(a.elapsed_time(b) * 1e3 / iters)
    out = {}
    for k, v in per.items():
        v.sort()
        out[k] = {"median_us": round(v[len(v) // 2], 2), "min_us": round(v[0], 2), "max_us": round(v[-1], 2)}
    return out


# the FP16 baseline and the pairs torch.autocast hands the op: (depth dtype, feat dtype), C entries, leading feat_dtype
PAIR_LEGS = {"f16_alt": (torch.float16, torch.float16, "b200_bev_pool_f16", "b200_bev_pool_backward_f16", ()),
             "bf16": (torch.bfloat16, torch.bfloat16, "b200_bev_pool_bf16", "b200_bev_pool_backward_bf16", ()),
             "f32d_f16": (torch.float32, torch.float16, "b200_bev_pool_f32_depth", "b200_bev_pool_backward_f32_depth",
                          (1,)),
             "f32d_bf16": (torch.float32, torch.bfloat16, "b200_bev_pool_f32_depth", "b200_bev_pool_backward_f32_depth",
                           (7,))}  # fmt: skip


def pair_legs(depth, feat, rk, hw):
    """{leg: call} of the forward and the backward (both gradients) of every PAIR_LEGS pair, through the C ABI: at
    bevdet_r50 a forward through the autograd binding costs about as much host time as the kernel takes."""
    legs = {}
    C = feat.shape[-1]
    order = torch.sort(rk[1], stable=True).indices.int()
    ws = torch.empty(rk[0].numel(), dtype=torch.int32, device="cuda")
    out = torch.empty(1, hw[0], hw[1], C, dtype=torch.float32, device="cuda")  # room for every pair's output
    for name, (dd, fd, fwd, bwd, lead) in PAIR_LEGS.items():
        d, f = depth.to(dd).cuda(), feat.to(fd).cuda()
        gout = torch.randn(1, hw[0], hw[1], C, device="cuda").to(fd)
        dg, fg = torch.empty_like(d), torch.empty_like(f)
        legs[f"fwd_{name}"] = lambda d=d, f=f, fwd=fwd, lead=lead: _lib.call(
            fwd, f.device, *lead, d.data_ptr(), f.data_ptr(), *(r.data_ptr() for r in rk), C, rk[0].numel(),
            rk[3].numel(), d.numel(), f.numel() // C, hw[0], hw[1], out.data_ptr())  # fmt: skip
        legs[f"bwd_{name}"] = lambda d=d, f=f, gout=gout, dg=dg, fg=fg, bwd=bwd, lead=lead: _lib.call(
            bwd, f.device, *lead, gout.data_ptr(), d.data_ptr(), f.data_ptr(), *(r.data_ptr() for r in rk),
            order.data_ptr(), C, rk[0].numel(), rk[3].numel(), d.numel(), f.numel() // C, hw[0], hw[1], dg.data_ptr(),
            fg.data_ptr(), ws.data_ptr(), ws.numel() * 4)  # fmt: skip
    return legs


def eager(depth, feat, ranks, hw):
    rd, rf, rb, st, _ = ranks
    C = feat.shape[-1]
    cell = rb.long()
    out = torch.zeros(hw[0] * hw[1], C, dtype=feat.dtype, device=feat.device)
    out.index_add_(0, cell, feat.view(-1, C).index_select(0, rf.long()) * depth.view(-1).index_select(0, rd.long())[:, None])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bev_pool_time.py measures on a GPU"
    gpu = card()
    print("card:", gpu, flush=True)
    try:
        from oracle.bev_pool import RefBevPool

        ref = RefBevPool()
    except (FileNotFoundError, OSError) as e:
        print("reference kernels not available:", e)
        ref = None
    results = {}
    for name in ("bevdet_r50", "ref_test"):
        depth, feat, ranks, hw = make_bev_pool_inputs(name, 0)
        stats = bev_pool_stats(ranks)
        rk = [r.cuda() for r in ranks]
        res = {"stats": stats, "bytes_f32": traffic(depth, feat, ranks, hw, 4), "bytes_f16": traffic(depth, feat, ranks, hw, 2),
               "bytes_i8": traffic(depth, feat, ranks, hw, 1)}  # fmt: skip
        print(name, stats, res["bytes_f16"], flush=True)
        for prec, dt in (("f32", torch.float32), ("f16", torch.float16)):
            d, f = depth.to(dt).cuda(), feat.to(dt).cuda()
            res[f"fwd_{prec}"] = timed(lambda: bt.bev_pool_v2(d, f, *rk, *hw), args.iters)
            res[f"fwd_{prec}_eager"] = timed(lambda: eager(d, f, rk, hw), args.iters)
            if ref is not None:
                res[f"fwd_{prec}_ref"] = timed(lambda: ref.forward(d, f, rk, hw, prec), args.iters)
                if prec == "f16":
                    res["fwd_f16_ref_h2"] = timed(lambda: ref.forward(d, f, rk, hw, "f16_h2"), args.iters)
            # backward: the gradient kernels through the C ABI (regrouping order precomputed)
            gout = torch.randn(1, hw[0], hw[1], feat.shape[-1], device="cuda").to(dt)
            order = torch.sort(rk[1], stable=True).indices.int()
            ws = torch.empty(rk[0].numel(), dtype=torch.int32, device="cuda")
            dg, fg = torch.empty_like(d), torch.empty_like(f)
            fn = "b200_bev_pool_backward_f32" if prec == "f32" else "b200_bev_pool_backward_f16"
            C = f.shape[-1]
            res[f"bwd_{prec}"] = timed(lambda: _lib.call(fn, f.device, gout.data_ptr(), d.data_ptr(), f.data_ptr(),
                                                         *(r.data_ptr() for r in rk), order.data_ptr(), C,
                                                         rk[0].numel(), rk[3].numel(), d.numel(), f.numel() // C,
                                                         hw[0], hw[1], dg.data_ptr(), fg.data_ptr(), ws.data_ptr(),
                                                         ws.numel() * 4), args.iters)  # fmt: skip
            if ref is not None and prec == "f32":
                res["bwd_f32_ref"] = timed(lambda: ref.backward_f32(gout, d, f, rk), max(args.iters // 10, 5))
        dq, sd = quantize_per_tensor(depth)
        fq, sf = quantize_per_tensor(feat)
        dq, fq = dq.cuda(), fq.cuda()
        res["fwd_i8"] = timed(lambda: bt.bev_pool_v2_int8(dq, sd, fq, sf, *rk, 0.02, *hw), args.iters)
        if ref is not None:
            res["fwd_i8_ref"] = timed(lambda: ref.forward_int8(dq, sd, fq, sf, rk, 0.02, hw), args.iters)
        res.update(timed_alternating(pair_legs(depth, feat, rk, hw), args.iters))
        for k, v in res.items():
            if k.startswith(("fwd", "bwd")):
                print(f"  {name:11s} {k:16s} median {v['median_us']:9.2f} us  (min {v['min_us']}, max {v['max_us']})")
        results[name] = res
    print(json.dumps({"card": gpu, "results": results}))


if __name__ == "__main__":
    main()
