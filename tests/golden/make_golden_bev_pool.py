"""Generates tests/golden/ref_bev_pool.npz: outputs of the REFERENCE's own BEVPoolV2 CUDA kernels, compiled unmodified
into oracle/_ref/libref_bev_pool.so (oracle/bev_pool.mk), run once on an H100:

    f32, f16, h2   bev_pool_v2<float>, bev_pool_v2<__half>, bev_pool_v2_h2 (TensorRT/plugin/bev_pool_v2/bevPoolKernel.cu)
    i8             bev_pool_v2_int8 on per-tensor quantised depth / feat, output scale max|float64 result| / 127
    dgrad, fgrad   mmdet3d's bev_pool_grad_kernel (third_party/bev_mmdet3d/ops/bev_pool_v2/src/bev_pool_cuda.cu) with the
                   point regrouping of QuickCumsumCuda.backward, for out_grad ~ N(0, 1) from seed 1

Inputs are regenerated from seeds (bevformer_tensorrt_b200.workloads.make_bev_pool_inputs) and pinned by digest. "tiny"
is stored in full; the larger workloads keep the tests.helpers.golden_sample positions.

    python tests/golden/make_golden_bev_pool.py [output.npz]
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from bevformer_tensorrt_b200.workloads import make_bev_pool_inputs, quantize_per_tensor  # noqa: E402
from oracle import bev_pool as obev  # noqa: E402
from tests.helpers import golden_sample, input_digest  # noqa: E402

WORKLOADS = ("tiny", "bevdet_r50", "ref_test")
SEED = 0


def keep(name, t):
    return t.detach().float().cpu().numpy().reshape(-1) if name == "tiny" else golden_sample(t)


def main(path):
    ref = obev.RefBevPool()
    out = {}
    for name in WORKLOADS:
        depth, feat, ranks, hw = make_bev_pool_inputs(name, SEED)
        out[f"{name}_digest"] = np.array(input_digest(depth, feat, *ranks))
        rk = [r.cuda() for r in ranks]
        d, f = depth.cuda(), feat.cuda()
        out[f"{name}_f32"] = keep(name, ref.forward(d, f, rk, hw, "f32"))
        out[f"{name}_f16"] = keep(name, ref.forward(d.half(), f.half(), rk, hw, "f16"))
        out[f"{name}_h2"] = keep(name, ref.forward(d.half(), f.half(), rk, hw, "f16_h2"))
        dq, sd = quantize_per_tensor(depth)
        fq, sf = quantize_per_tensor(feat)
        real = obev.bev_pool_f64(dq.double().numpy() * sd, fq.double().numpy() * sf, [r.numpy() for r in ranks], hw)
        so = float(np.abs(real).max()) / 127.0
        out[f"{name}_i8_scales"] = np.array([sd, sf, so], np.float64)
        out[f"{name}_i8"] = keep(name, ref.forward_int8(dq.cuda(), sd, fq.cuda(), sf, rk, so, hw))
        gout = torch.randn(1, hw[0], hw[1], feat.shape[-1], generator=torch.Generator().manual_seed(1))
        dg, fg = ref.backward_f32(gout.cuda(), d, f, rk)
        out[f"{name}_dgrad"], out[f"{name}_fgrad"] = keep(name, dg), keep(name, fg)
        torch.cuda.synchronize()
        print(name, "done", flush=True)
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "ref_bev_pool.npz"))
