"""BEVPoolV2TRT / BEVPoolV2TRT2 through the TensorRT plugin shells on device data: tests/mock_trt/bev_pool_capi.cpp
drives create -> serialise -> deserialise -> output dimensions -> enqueue for both names and every precision, and the
result must equal the Python binding's (the same kernels)."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import bevformer_tensorrt_b200 as bt
from bevformer_tensorrt_b200 import _lib
from bevformer_tensorrt_b200.workloads import make_bev_pool_inputs, quantize_per_tensor

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def shell_capi(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    lib_dir = os.path.dirname(_lib.LIB_PATH)
    so = str(tmp_path_factory.mktemp("bev_shell_capi") / "libbev_capi.so")
    cmd = ["g++", "-std=c++17", "-Wall", "-shared", "-fPIC", "-I", os.path.join(ROOT, "tests", "mock_trt"), "-I",
           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "mock_trt", "bev_pool_capi.cpp"), "-L", lib_dir,
           "-lb200_bev_ops", f"-Wl,-rpath,{lib_dir}", "-o", so]  # fmt: skip
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    lib = ctypes.CDLL(so)
    vp = ctypes.c_void_p
    lib.bcapi_create.restype = vp
    lib.bcapi_create.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.POINTER(ctypes.c_char_p),
                                 ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int32)]  # fmt: skip
    lib.bcapi_deserialize.restype = vp
    lib.bcapi_deserialize.argtypes = [ctypes.c_char_p, vp, ctypes.c_size_t]
    lib.bcapi_plugin_type.restype = ctypes.c_char_p
    lib.bcapi_plugin_type.argtypes = [vp]
    lib.bcapi_serialization_size.restype = ctypes.c_size_t
    lib.bcapi_serialization_size.argtypes = [vp]
    lib.bcapi_serialize.argtypes = [vp, vp]
    lib.bcapi_output_dims.argtypes = [vp, ctypes.c_int32, ctypes.POINTER(ctypes.c_int32)]
    lib.bcapi_supports.argtypes = [vp, ctypes.c_int, ctypes.POINTER(_lib.TensorDesc), ctypes.c_int, ctypes.c_int]
    lib.bcapi_enqueue.argtypes = [vp, ctypes.POINTER(_lib.TensorDesc), ctypes.POINTER(_lib.TensorDesc),
                                  ctypes.POINTER(vp), ctypes.POINTER(vp), vp]  # fmt: skip
    lib.bcapi_destroy.argtypes = [vp]
    return lib


def _desc(t, type_, scale=1.0):
    d = _lib.TensorDesc()
    d.dims.nbDims = t.dim()
    for i, v in enumerate(t.shape):
        d.dims.d[i] = v
    d.type, d.format, d.scale = type_, 0, scale
    return d


def _reloaded(lib, name, hw):
    names = (ctypes.c_char_p * 2)(b"out_height", b"out_width")
    p = lib.bcapi_create(name.encode(), 2, names, (ctypes.c_int32 * 2)(*hw), (ctypes.c_int32 * 2)(1, 1))
    assert p
    n = lib.bcapi_serialization_size(p)
    blob = ctypes.create_string_buffer(n)
    lib.bcapi_serialize(p, blob)
    q = lib.bcapi_deserialize(name.encode(), blob, n)
    lib.bcapi_destroy(p)
    assert q and lib.bcapi_plugin_type(q) == name.encode()
    return q


@pytest.mark.parametrize("name", ["BEVPoolV2TRT", "BEVPoolV2TRT2"])
@pytest.mark.parametrize("precision", ["f32", "f16", "i8"])
def test_plugin_enqueue_matches_the_binding(shell_capi, name, precision):
    lib = shell_capi
    depth, feat, ranks, hw = make_bev_pool_inputs("bevdet_r50", 1)
    C = feat.shape[-1]
    plugin = _reloaded(lib, name, hw)
    dims = (ctypes.c_int32 * 4)()
    assert lib.bcapi_output_dims(plugin, C, dims) == 4 and list(dims) == [1, hw[0], hw[1], C]
    rk = [r.cuda() for r in ranks]
    if precision == "i8":
        dq, sd = quantize_per_tensor(depth)
        fq, sf = quantize_per_tensor(feat)
        so = 0.02
        d, f, type_ = dq.cuda(), fq.cuda(), 2
        scales = (sd, sf, so)
        want = bt.bev_pool_v2_int8(d, sd, f, sf, *rk, so, *hw)
    else:
        dt = torch.float32 if precision == "f32" else torch.float16
        d, f, type_ = depth.to(dt).cuda(), feat.to(dt).cuda(), 0 if precision == "f32" else 1
        scales = (1.0, 1.0, 1.0)
        want = bt.bev_pool_v2(d, f, *rk, *hw)
    out = torch.full_like(want, 7)
    ins = (_lib.TensorDesc * 7)(_desc(d, type_, scales[0]), _desc(f, type_, scales[1]), *(_desc(r, 3) for r in rk))
    outs = (_lib.TensorDesc * 1)(_desc(out, type_, scales[2]))
    io = (_lib.TensorDesc * 8)(*ins, *outs)
    assert all(lib.bcapi_supports(plugin, pos, io, 7, 1) for pos in range(8))
    ptrs = (ctypes.c_void_p * 7)(d.data_ptr(), f.data_ptr(), *(r.data_ptr() for r in rk))
    optr = (ctypes.c_void_p * 1)(out.data_ptr())
    st = lib.bcapi_enqueue(plugin, ins, outs, ptrs, optr, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    lib.bcapi_destroy(plugin)
    assert st == 0
    assert np.array_equal(out.cpu().numpy().view(np.uint8), want.cpu().numpy().view(np.uint8))
