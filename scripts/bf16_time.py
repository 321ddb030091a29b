"""BF16 against FP16 on the same seeded inputs: MSDA plugin op forward and backward (with and without grad_value) at
base_sca G / U and base_tsa, the camera-shared fused SCA forward and backward at base_sca G, and the DCNv2 layer
(BF16 generic kernel against the FP16 fused kernel) forward and backward at the base backbone shape [6,256,58,100] 3x3.

Each number is the per-call time of a 50-call window timed with CUDA events; three windows, median / min / max.
Prints the card name and power limit from the same run, then one JSON line per measurement.

    python scripts/bf16_time.py [--windows 3] [--steps 50]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bevformer_tensorrt_b200 as bt  # noqa: E402
from bevformer_tensorrt_b200.workloads import CONFIGS, make_msda_inputs  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)  # fmt: skip
    return r.stdout.strip().splitlines()[torch.cuda.current_device()] if r.returncode == 0 else torch.cuda.get_device_name()


def timed(fn, steps, windows):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    per = []
    for _ in range(windows):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(steps):
            fn()
        b.record()
        torch.cuda.synchronize()
        per.append(a.elapsed_time(b) * 1e3 / steps)
    per.sort()
    return {"us_median": round(per[len(per) // 2], 2), "us_min": round(per[0], 2), "us_max": round(per[-1], 2)}


def msda_inputs(cfg_name, dist, dtype):
    value, shapes, ref, off, logits = make_msda_inputs(CONFIGS[cfg_name], dist, 0, torch.float32)
    return [value.to(dtype).cuda(), shapes.cuda(), ref.cuda(), off.to(dtype).cuda(), logits.to(dtype).cuda()]


def msda_cases(steps, windows):
    for cfg_name, dist in (("base_sca", "G"), ("base_sca", "U"), ("base_tsa", "U")):
        for dtype in (torch.float16, torch.bfloat16):
            value, shapes, ref, off, logits = msda_inputs(cfg_name, dist, dtype)
            tag = {"config": cfg_name, "dist": dist, "dtype": str(dtype)[6:]}
            yield {"op": "msda_forward", **tag, **timed(lambda: bt.multi_scale_deformable_attn(value, shapes, ref, off,
                                                                                               logits), steps, windows)}
            for with_value in (True, False):
                ts = [t.detach().requires_grad_(with_value or i > 0) for i, t in enumerate((value, ref, off, logits))]
                out = bt.multi_scale_deformable_attn(ts[0], shapes, *ts[1:])
                go = torch.randn_like(out)
                want = [t for t in ts if t.requires_grad]
                fn = lambda: torch.autograd.grad(out, want, go, retain_graph=True)  # noqa: E731
                yield {"op": "msda_backward" + ("" if with_value else "_no_grad_value"), **tag, **timed(fn, steps, windows)}


def shared_cases(steps, windows):
    cfg = CONFIGS["base_sca"]
    g = torch.Generator().manual_seed(5)
    seen = (torch.rand(cfg.batch, cfg.num_query, generator=g) < 0.3).float()
    mask = (seen / seen.sum(0, keepdim=True).clamp(min=1e-4)).cuda()
    for dtype in (torch.float16, torch.bfloat16):
        value, shapes, ref, off, logits = msda_inputs("base_sca", "G", dtype)
        off, logits = off[:1].contiguous(), logits[:1].contiguous()
        tag = {"config": "base_sca", "dist": "G", "dtype": str(dtype)[6:]}
        fwd = lambda: bt.multi_scale_deformable_attn_sca_shared(value, shapes, ref, off, logits, mask)  # noqa: E731
        yield {"op": "sca_shared_forward", **tag, **timed(fwd, steps, windows)}
        ts = [t.detach().requires_grad_(True) for t in (value, ref, off, logits)]
        out = bt.multi_scale_deformable_attn_sca_shared(ts[0], shapes, ts[1], ts[2], ts[3], mask)
        go = torch.randn_like(out)
        yield {"op": "sca_shared_backward", **tag,
               **timed(lambda: torch.autograd.grad(out, ts, go, retain_graph=True), steps, windows)}


def dcn_cases(steps, windows):
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(6, 256, 58, 100, device="cuda", generator=g)
    off = torch.randn(6, 18, 58, 100, device="cuda", generator=g) * 2
    mask = torch.sigmoid(torch.randn(6, 9, 58, 100, device="cuda", generator=g))
    w = torch.randn(256, 256, 3, 3, device="cuda", generator=g) / 48.0
    b = torch.randn(256, device="cuda", generator=g)
    for dtype in (torch.float16, torch.bfloat16):
        ts = [t.to(dtype) for t in (x, off, mask, w, b)]
        tag = {"shape": "[6,256,58,100] 3x3 Co 256", "dtype": str(dtype)[6:],
               "kernel": "fused wgmma" if dtype == torch.float16 else "generic"}  # fmt: skip
        fwd = lambda: bt.modulated_deformable_conv2d(*ts, 1, 1, 1, 1, 1)  # noqa: E731
        yield {"op": "dcn_forward", **tag, **timed(fwd, steps, windows)}
        rg = [t.detach().requires_grad_(True) for t in ts]
        out = bt.modulated_deformable_conv2d(*rg, 1, 1, 1, 1, 1)
        go = torch.randn_like(out)
        yield {"op": "dcn_backward", **{k: v for k, v in tag.items() if k != "kernel"},
               **timed(lambda: torch.autograd.grad(out, rg, go, retain_graph=True), steps, windows)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--windows", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bf16_time.py measures on a CUDA device; none is present")
    print(json.dumps({"card": card(), "torch": torch.__version__}))
    for gen in (msda_cases, shared_cases, dcn_cases):
        for rec in gen(a.steps, a.windows):
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
