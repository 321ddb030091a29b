"""oracle/bev_pool.py — TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

ctypes driver for oracle/bev_pool_cpu.c (BEVPoolV2 restated in C: float64 forward / backward, the FP32 forward as an
fmaf chain, the INT8 forward, the FP32 backward in the kernels' lane partition) and ``RefBevPool``, which calls the reference's own BEVPoolV2 kernels
(oracle/ref_bev_pool_shim.cu, built into oracle/_ref/libref_bev_pool.so by oracle/bev_pool.mk) on torch CUDA tensors.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_LIB = os.path.join(_HERE, "_build", "libbev_pool_oracle.so")
REF_LIB = os.path.join(_HERE, "_ref", "libref_bev_pool.so")
_SRC = os.path.join(_HERE, "bev_pool_cpu.c")


def build(ref: bool = True) -> None:
    """Compile libbev_pool_oracle.so (gcc) and, where the reference sources are present, _ref/libref_bev_pool.so."""
    subprocess.run(["make", "-s", "-C", _HERE, "-f", "bev_pool.mk", "oracle"], check=True)
    if ref:
        subprocess.run(["make", "-s", "-C", _HERE, "-f", "bev_pool.mk", "ref"], check=True)


_lib = None


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(ORACLE_LIB) or os.path.getmtime(_SRC) > os.path.getmtime(ORACLE_LIB):
            build(ref=False)
        _lib = ctypes.CDLL(ORACLE_LIB)
    return _lib


def _i32(a):
    return np.ascontiguousarray(np.asarray(a), np.int32)


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _common(ranks, depth_size, feat_rows, C, out_hw):
    rd, rf, rb, st, ln = (_i32(r) for r in ranks)
    return [_ptr(rd), _ptr(rf), _ptr(rb), _ptr(st), _ptr(ln), ctypes.c_int(C), ctypes.c_int(rd.size),
            ctypes.c_int(st.size), ctypes.c_longlong(depth_size), ctypes.c_longlong(feat_rows),
            ctypes.c_longlong(out_hw[0] * out_hw[1])], (rd, rf, rb, st, ln)  # fmt: skip


def _shape(feat):
    C = feat.shape[-1]
    return C, feat.size // C


def bev_pool_f64(depth, feat, ranks, out_hw):
    """ranks = (ranks_depth, ranks_feat, ranks_bev, interval_starts, interval_lengths). Returns [1, h, w, C] float64."""
    depth, feat = np.ascontiguousarray(depth, np.float64), np.ascontiguousarray(feat, np.float64)
    C, rows = _shape(feat)
    args, keep = _common(ranks, depth.size, rows, C, out_hw)
    out = np.empty((1, out_hw[0], out_hw[1], C), np.float64)
    lib().bev_pool_f64(_ptr(depth), _ptr(feat), *args, _ptr(out))
    return out


def bev_pool_f32_fma(depth, feat, ranks, out_hw):
    depth, feat = np.ascontiguousarray(depth, np.float32), np.ascontiguousarray(feat, np.float32)
    C, rows = _shape(feat)
    args, keep = _common(ranks, depth.size, rows, C, out_hw)
    out = np.empty((1, out_hw[0], out_hw[1], C), np.float32)
    lib().bev_pool_f32_fma(_ptr(depth), _ptr(feat), *args, _ptr(out))
    return out


def bev_pool_i8(depth_q, scale_d, feat_q, scale_f, ranks, scale_o, out_hw):
    depth_q, feat_q = np.ascontiguousarray(depth_q, np.int8), np.ascontiguousarray(feat_q, np.int8)
    C, rows = _shape(feat_q)
    args, keep = _common(ranks, depth_q.size, rows, C, out_hw)
    out = np.empty((1, out_hw[0], out_hw[1], C), np.int8)
    f = ctypes.c_float
    lib().bev_pool_i8(_ptr(depth_q), _ptr(feat_q), *args, f(scale_d), f(scale_f), f(scale_o), _ptr(out))
    return out


def bev_pool_backward_f64(out_grad, depth, feat, ranks, out_hw):
    """Returns (depth_grad shaped like depth, feat_grad shaped like feat), float64."""
    og = np.ascontiguousarray(out_grad, np.float64)
    depth, feat = np.ascontiguousarray(depth, np.float64), np.ascontiguousarray(feat, np.float64)
    C, rows = _shape(feat)
    args, keep = _common(ranks, depth.size, rows, C, out_hw)
    dg, fg = np.empty_like(depth), np.empty_like(feat)
    lib().bev_pool_backward_f64(_ptr(og), _ptr(depth), _ptr(feat), *args, _ptr(dg), _ptr(fg))
    return dg, fg


def bev_pool_backward_f32_lanes(out_grad, depth, feat, ranks, out_hw, G, vec, depth_grad=True, feat_grad=True):
    """The float32 depth / feature gradients as the device kernels compute them for a lane group of ``G`` lanes of
    ``vec`` channels each (see bev_pool_cpu.c). Returns (depth_grad shaped like depth or None, feat_grad shaped like feat
    or None), float32. For FP16, pass the widened halves and round the result once with ``np.float16``."""
    og = np.ascontiguousarray(out_grad, np.float32)
    depth, feat = np.ascontiguousarray(depth, np.float32), np.ascontiguousarray(feat, np.float32)
    C, rows = _shape(feat)
    assert G in (1, 2, 4, 8, 16, 32) and C % vec == 0, (G, vec, C)
    args, keep = _common(ranks, depth.size, rows, C, out_hw)
    dg = np.empty_like(depth) if depth_grad else None
    fg = np.empty_like(feat) if feat_grad else None
    scratch = np.empty(keep[0].size, np.int64)
    lib().bev_pool_backward_f32_lanes(_ptr(og), _ptr(depth), _ptr(feat), *args, ctypes.c_int(G), ctypes.c_int(vec),
                                      None if dg is None else _ptr(dg), None if fg is None else _ptr(fg), _ptr(scratch))
    return dg, fg


class RefBevPool:
    """The reference's own BEVPoolV2 kernels on torch CUDA tensors (index tensors int32, contiguous)."""

    def __init__(self):
        if not os.path.exists(REF_LIB):
            raise FileNotFoundError(f"{REF_LIB} missing: run `make -C oracle -f bev_pool.mk ref` where the reference exists")
        self.lib = ctypes.CDLL(REF_LIB)

    @staticmethod
    def _p(t):
        return ctypes.c_void_p(t.data_ptr())

    def forward(self, depth, feat, ranks, out_hw, variant="f32"):
        """variant f32 / f16 / f16_h2 (BEVPoolV2TRT2's half2 kernel, C even). Returns [1, h, w, C]."""
        import torch

        C = feat.shape[-1]
        out = torch.empty(1, out_hw[0], out_hw[1], C, dtype=feat.dtype, device=feat.device)
        dt = {"f32": 0, "f16": 1, "f16_h2": 2}[variant]
        self.lib.ref_bev_pool(dt, C, ranks[3].numel(), out.numel(), self._p(depth), self._p(feat),
                              *(self._p(r) for r in ranks), self._p(out),
                              ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))  # fmt: skip
        return out

    def forward_int8(self, depth_q, scale_d, feat_q, scale_f, ranks, scale_o, out_hw):
        import torch

        C = feat_q.shape[-1]
        out = torch.empty(1, out_hw[0], out_hw[1], C, dtype=torch.int8, device=feat_q.device)
        f = ctypes.c_float
        self.lib.ref_bev_pool_int8(C, ranks[3].numel(), out.numel(), self._p(depth_q), f(scale_d), self._p(feat_q),
                                   f(scale_f), *(self._p(r) for r in ranks), self._p(out), f(scale_o),
                                   ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))  # fmt: skip
        return out

    def backward_f32(self, out_grad, depth, feat, ranks):
        """QuickCumsumCuda.backward (bev_pool.py): regroup the points by ranks_feat, then bev_pool_grad_kernel."""
        import torch

        rd, rf, rb = ranks[0], ranks[1], ranks[2]
        order = torch.sort(rf, stable=True).indices
        rf, rd, rb = rf[order].contiguous(), rd[order].contiguous(), rb[order].contiguous()
        kept = torch.ones(rb.shape[0], device=rb.device, dtype=torch.bool)
        kept[1:] = rf[1:] != rf[:-1]
        starts = torch.where(kept)[0].int()
        lengths = torch.zeros_like(starts)
        lengths[:-1] = starts[1:] - starts[:-1]
        lengths[-1] = rb.shape[0] - starts[-1]
        dg, fg = torch.zeros_like(depth), torch.zeros_like(feat)
        torch.cuda.synchronize()
        self.lib.ref_bev_pool_backward_f32(feat.shape[-1], starts.numel(), self._p(out_grad.contiguous()),
                                           self._p(depth), self._p(feat), self._p(rd), self._p(rf), self._p(rb),
                                           self._p(starts), self._p(lengths), self._p(dg), self._p(fg))  # fmt: skip
        return dg, fg
