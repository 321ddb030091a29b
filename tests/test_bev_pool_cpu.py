"""BEVPoolV2 without a GPU: the C oracle against the reference kernels' stored outputs, the Python binding's symbolics,
registry entries and input checks, the C ABI's argument validation, and the TensorRT shells (tests/mock_trt)."""
import ctypes
import ctypes.util
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import bevformer_tensorrt_b200 as bt
from bevformer_tensorrt_b200 import _lib
from bevformer_tensorrt_b200.workloads import make_bev_pool_inputs, quantize_per_tensor
from oracle import bev_pool as obev
from tests.helpers import GOLDEN, golden_index, input_digest, rounding_bound

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKLOADS = ("tiny", "bevdet_r50", "ref_test")


def _golden():
    return np.load(os.path.join(GOLDEN, "ref_bev_pool.npz"))


def _kept(name, a):
    flat = np.asarray(a).reshape(-1)
    return flat if name == "tiny" else flat[golden_index(flat.size)]


@pytest.mark.parametrize("name", WORKLOADS)
def test_oracle_reproduces_reference_kernels_fp32_and_int8(name):
    z = _golden()
    depth, feat, ranks, hw = make_bev_pool_inputs(name, 0)
    assert input_digest(depth, feat, *ranks) == str(z[f"{name}_digest"]), "seeded generator changed"
    rk = [r.numpy() for r in ranks]
    got = obev.bev_pool_f32_fma(depth.numpy(), feat.numpy(), rk, hw)
    assert np.array_equal(_kept(name, got).view(np.uint32), z[f"{name}_f32"].view(np.uint32))
    dq, sd = quantize_per_tensor(depth)
    fq, sf = quantize_per_tensor(feat)
    _, _, so = (float(x) for x in z[f"{name}_i8_scales"])
    assert (sd, sf) == tuple(float(x) for x in z[f"{name}_i8_scales"][:2])
    got8 = obev.bev_pool_i8(dq.numpy(), sd, fq.numpy(), sf, rk, so, hw)
    assert np.array_equal(_kept(name, got8).astype(np.float32), z[f"{name}_i8"])


def test_oracle_backward_matches_reference_kernel_on_tiny():
    z = _golden()
    depth, feat, ranks, hw = make_bev_pool_inputs("tiny", 0)
    gout = torch.randn(1, hw[0], hw[1], feat.shape[-1], generator=torch.Generator().manual_seed(1))
    dg, fg = obev.bev_pool_backward_f64(gout.numpy(), depth.numpy(), feat.numpy(), [r.numpy() for r in ranks], hw)
    np.testing.assert_allclose(dg.reshape(-1), z["tiny_dgrad"], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(fg.reshape(-1), z["tiny_fgrad"], rtol=1e-5, atol=1e-6)



def _lane_case(C, seed):
    depth, feat, ranks, hw = make_bev_pool_inputs("tiny", seed)
    g = torch.Generator().manual_seed(seed + 50)
    feat = torch.randn(*feat.shape[:-1], C, generator=g)
    gout = torch.randn(1, hw[0], hw[1], C, generator=g)
    return gout.numpy(), depth.numpy(), feat.numpy(), [r.numpy() for r in ranks], hw


@pytest.mark.parametrize("C,G,vec", [(1, 1, 1), (3, 4, 1), (16, 4, 4), (33, 32, 1), (64, 8, 8), (130, 32, 2),
                                     (132, 32, 4), (256, 32, 8), (17, 2, 1)])  # fmt: skip
def test_lane_oracle_within_per_element_bound_of_float64(C, G, vec):
    """The kernels' lane partition restated in float32 is the backward op: within half a float32 ulp plus (n + 1)
    roundings of the magnitude sum of float64, element by element (n = C for the depth gradient, the row's point count
    for the feature gradient). G = 2 at C = 17 is a partition no launch uses: each lane chains many chunks."""
    og, depth, feat, ranks, hw = _lane_case(C, C)
    dg, fg = obev.bev_pool_backward_f32_lanes(og, depth, feat, ranks, hw, G, vec)
    wd, wf = obev.bev_pool_backward_f64(og, depth, feat, ranks, hw)
    sd, sf = obev.bev_pool_backward_f64(np.abs(og), np.abs(depth), np.abs(feat), ranks, hw)
    runs = np.bincount(ranks[1], minlength=feat.size // C)
    assert np.all(np.abs(dg - wd) <= rounding_bound(wd, sd, C, np.float32))
    assert np.all(np.abs(fg - wf) <= rounding_bound(wf, sf, runs.reshape(feat.shape[:-1] + (1,)), np.float32))
    assert np.count_nonzero(dg) > 0.9 * ranks[0].size and np.count_nonzero(fg) > 0


def _libm_fmaf():
    f = ctypes.CDLL(ctypes.util.find_library("m")).fmaf
    f.restype, f.argtypes = ctypes.c_float, [ctypes.c_float] * 3
    return f


def test_lane_oracle_at_one_lane_is_a_plain_fmaf_chain():
    """G = VEC = 1: the depth gradient is one fmaf chain over c (no butterfly), and the feature gradient one fmaf chain
    over a row's points in point order, here restated with the C library's fmaf element by element. With one lane the
    vector width does not reorder anything, so VEC = 2 and 4 give the same bits."""
    fmaf = _libm_fmaf()
    C = 12
    og, depth, feat, ranks, hw = _lane_case(C, 3)
    rd, rf, rb, st, ln = ranks
    dg, fg = obev.bev_pool_backward_f32_lanes(og, depth, feat, ranks, hw, 1, 1)
    ogf, ff, df = og.reshape(-1, C), feat.reshape(-1, C), depth.reshape(-1)
    want_d, want_f = np.zeros_like(df), np.zeros_like(ff)
    for k in range(st.size):
        cell = rb[st[k]]
        for i in range(st[k], st[k] + ln[k]):
            acc = 0.0
            for c in range(C):
                acc = fmaf(ogf[cell, c], ff[rf[i], c], acc)
            want_d[rd[i]] = acc
    for i in np.argsort(rf, kind="stable"):  # the points of each row in point order
        cell = rb[i]
        for c in range(C):
            want_f[rf[i], c] = fmaf(ogf[cell, c], df[rd[i]], want_f[rf[i], c])
    assert np.array_equal(dg.reshape(-1).view(np.uint32), want_d.view(np.uint32))
    assert np.array_equal(fg.reshape(-1, C).view(np.uint32), want_f.view(np.uint32))
    for vec in (2, 4):
        dv, fv = obev.bev_pool_backward_f32_lanes(og, depth, feat, ranks, hw, 1, vec)
        assert np.array_equal(dv.view(np.uint32), dg.view(np.uint32)) and np.array_equal(fv.view(np.uint32), fg.view(np.uint32))
    dv, _ = obev.bev_pool_backward_f32_lanes(og, depth, feat, ranks, hw, 4, 1)
    assert not np.array_equal(dv.view(np.uint32), dg.view(np.uint32))  # four lanes sum in another order

class _Graph:
    def __init__(self):
        self.ops = []

    def op(self, name, *args, **attrs):
        self.ops.append((name, len(args), attrs))
        return name


def test_symbolics_emit_the_reference_plugin_names_and_attributes():
    from bevformer_tensorrt_b200.functions.bev_pool_v2 import _BEVPoolV2, _BEVPoolV2_2

    for cls, name in ((_BEVPoolV2, "BEVPoolV2TRT"), (_BEVPoolV2_2, "BEVPoolV2TRT2")):
        g = _Graph()
        cls.symbolic(g, *range(7), 200, 100)
        assert g.ops == [(name, 7, {"out_height_i": 200, "out_width_i": 100})]


def test_registry_and_package_exports():
    for name in ("bev_pool_v2", "bev_pool_v2_2", "bev_pool_v2_int8"):
        assert bt.TRT_FUNCTIONS.get(name) is getattr(bt, name)
        assert name in bt.__all__
    import inspect

    for fn in (bt.bev_pool_v2, bt.bev_pool_v2_2):
        params = inspect.signature(fn).parameters
        assert list(params)[:7] == ["depth", "feat", "ranks_depth", "ranks_feat", "ranks_bev", "interval_starts",
                                    "interval_lengths"]  # fmt: skip
        assert params["out_height"].default == 128 and params["out_width"].default == 128


def test_cpu_tensors_are_refused():
    depth, feat, ranks, hw = make_bev_pool_inputs("tiny", 0)
    for call in (lambda: bt.bev_pool_v2(depth, feat, *ranks, *hw),
                 lambda: bt.bev_pool_v2_2(depth, feat, *ranks, *hw),
                 lambda: bt.bev_pool_v2_int8(depth.to(torch.int8), 1.0, feat.to(torch.int8), 1.0, *ranks, 1.0, *hw)):  # fmt: skip
        with pytest.raises(RuntimeError, match="CUDA tensor"):
            call()


def _fake(n=7):
    """Non-null pointers that no call below dereferences: validation fails before any CUDA call."""
    return [ctypes.c_void_p(0x1000 * (i + 1)) for i in range(n)]


def test_abi_validates_arguments_before_any_cuda_call():
    lib = _lib.load()
    p = _fake()
    ok_dims = [16, 10, 3, 100, 50, 8, 8]  # C, P, I, depth_size, feat_rows, out h, out w
    nulls = [None] * 7
    assert lib.b200_bev_pool_f32(*nulls, *ok_dims, None, None) == 2
    for i in range(7):  # one null pointer at a time, everything else plausible
        args = list(p)
        args[i] = None
        assert lib.b200_bev_pool_f32(*args, *ok_dims, p[0], None) == 2, i
        assert lib.b200_bev_pool_f16(*args, *ok_dims, p[0], None) == 2, i
    assert lib.b200_bev_pool_f32(*p, *ok_dims, None, None) == 2  # output
    for i, bad in ((0, 0), (0, -4), (1, -1), (2, -1), (3, -1), (4, -1), (5, 0), (6, -2)):
        dims = list(ok_dims)
        dims[i] = bad
        assert lib.b200_bev_pool_f32(*p, *dims, p[0], None) == 2, (i, bad)
        assert lib.b200_bev_pool_i8(p[0], 1.0, p[1], 1.0, *p[2:], *dims, p[0], 1.0, None) == 2, (i, bad)
    # zero-length index arrays may be NULL; an INT8 channel count that is not a multiple of 4 is unsupported
    dims = list(ok_dims)
    dims[0] = 6
    assert lib.b200_bev_pool_i8(p[0], 1.0, p[1], 1.0, *p[2:], *dims, p[0], 1.0, None) == 1
    assert lib.b200_bev_pool_backward_workspace_size(1000) == 4000
    assert lib.b200_bev_pool_backward_workspace_size(0) == 0
    bwd = [p[0]] * 3 + list(p[2:]) + [p[1]]
    assert lib.b200_bev_pool_backward_f32(*bwd, *ok_dims, None, None, p[0], 40, None) == 2  # no gradient asked for
    assert lib.b200_bev_pool_backward_f32(*bwd, *ok_dims, p[0], p[1], p[0], 39, None) == 2  # workspace too small
    assert lib.b200_bev_pool_backward_f32(*bwd, *ok_dims, p[0], p[1], None, 40, None) == 2  # no workspace
    nb = list(bwd)
    nb[8] = None  # feat_order, needed for feat_grad
    assert lib.b200_bev_pool_backward_f16(*nb, *ok_dims, p[0], p[1], p[0], 40, None) == 2



def test_abi_rejects_element_misaligned_pointers_before_any_cuda_call():
    """A float, half or int32 pointer that is not aligned to its element is B200_ERR_BAD_PARAM, one pointer at a time,
    in every entry (int8 data needs no alignment; an int8 call fails only on its int32 arrays)."""
    lib = _lib.load()
    dims = [16, 10, 3, 100, 50, 8, 8]  # C, P, I, depth_size, feat_rows, out h, out w

    def fake(miss, nbytes):
        return [ctypes.c_void_p(0x1000 * (i + 1) + (nbytes if i == miss else 0)) for i in range(12)]

    for i in range(7):  # depth, feat, 5 int32 arrays
        for elem, name in ((2, "b200_bev_pool_f32"), (1, "b200_bev_pool_f16")):
            p = fake(i, elem if i < 2 else 2)
            assert getattr(lib, name)(*p[:7], *dims, p[7], None) == 2, (name, i)
        if i >= 2:
            p = fake(i, 2)
            assert lib.b200_bev_pool_i8(p[0], 1.0, p[1], 1.0, *p[2:7], *dims, p[7], 1.0, None) == 2, i
    for elem, name in ((2, "b200_bev_pool_f32"), (1, "b200_bev_pool_f16")):
        p = fake(7, elem)  # out
        assert getattr(lib, name)(*p[:7], *dims, p[7], None) == 2, name
    for name, elem in (("b200_bev_pool_backward_f32", 2), ("b200_bev_pool_backward_f16", 1)):
        # out_grad, depth, feat, 5 int32 arrays, feat_order, then depth_grad, feat_grad, workspace
        for i in range(12):
            p = fake(i, 2 if 3 <= i <= 8 or i == 11 else elem)
            assert getattr(lib, name)(*p[:9], *dims, p[9], p[10], p[11], 40, None) == 2, (name, i)

def _desc(dims, type_, fmt=0, scale=1.0):
    d = _lib.TensorDesc()
    d.dims.nbDims = len(dims)
    for i, v in enumerate(dims):
        d.dims.d[i] = v
    d.type, d.format, d.scale = type_, fmt, scale
    return d


def bev_descs(type_, C=16, P=100, I=10, hw=(8, 6), N=2, D=5, H=4, W=5):
    ins = (_lib.TensorDesc * 7)(_desc([N, D, H, W], type_), _desc([N, H, W, C], type_), _desc([P], 3), _desc([P], 3),
                                _desc([P], 3), _desc([I], 3), _desc([I], 3))  # fmt: skip
    out = (_lib.TensorDesc * 1)(_desc([1, hw[0], hw[1], C], type_))
    return ins, out


def test_enqueue_checks_descriptors_against_attributes():
    lib = _lib.load()
    ptrs = (ctypes.c_void_p * 7)(*[0x1000 * (i + 1) for i in range(7)])
    outs = (ctypes.c_void_p * 1)(0x9000)
    ins, out = bev_descs(0)
    assert lib.b200_bev_pool_enqueue(ins, out, ptrs, outs, None, None, 7, 6) == 2  # out dims say 8 x 6
    ins, out = bev_descs(0)
    ins[3].dims.d[0] = 99  # ranks_feat shorter than ranks_depth
    assert lib.b200_bev_pool_enqueue(ins, out, ptrs, outs, None, None, 8, 6) == 2
    ins, out = bev_descs(0)
    ins[6].dims.d[0] = 11
    assert lib.b200_bev_pool_enqueue(ins, out, ptrs, outs, None, None, 8, 6) == 2
    ins, out = bev_descs(0)
    out[0].dims.d[3] = 8  # output channels differ from feat's
    assert lib.b200_bev_pool_enqueue(ins, out, ptrs, outs, None, None, 8, 6) == 2
    ins, out = bev_descs(2, C=6)
    assert lib.b200_bev_pool_enqueue(ins, out, ptrs, outs, None, None, 8, 6) == 1
    ins, out = bev_descs(3)
    assert lib.b200_bev_pool_enqueue(ins, out, ptrs, outs, None, None, 8, 6) == 1
    assert lib.b200_bev_pool_enqueue(None, out, ptrs, outs, None, None, 8, 6) == 2


def test_supports_format_table():
    lib = _lib.load()
    for t in (0, 1, 2):
        io = (_lib.TensorDesc * 8)(*bev_descs(t)[0], *bev_descs(t)[1])
        assert all(lib.b200_bev_pool_supports_format(pos, io, 7, 1) for pos in range(8)), t
        io[2].type = 0  # an index tensor that is not int32
        assert not lib.b200_bev_pool_supports_format(2, io, 7, 1)
        io[1].format = 1  # feat not linear
        assert not lib.b200_bev_pool_supports_format(1, io, 7, 1)
    io = (_lib.TensorDesc * 8)(*bev_descs(0)[0], *bev_descs(0)[1])
    io[7].type = 1  # output type differs from depth's
    assert not lib.b200_bev_pool_supports_format(7, io, 7, 1)
    io = (_lib.TensorDesc * 8)(*bev_descs(2, C=6)[0], *bev_descs(2, C=6)[1])
    assert not lib.b200_bev_pool_supports_format(0, io, 7, 1)  # INT8 needs C % 4 == 0
    io = (_lib.TensorDesc * 8)(*bev_descs(0)[0], *bev_descs(0)[1])
    assert not lib.b200_bev_pool_supports_format(0, io, 6, 1) and not lib.b200_bev_pool_supports_format(8, io, 7, 1)


def test_plugin_shell_compiles_against_the_mock_api_with_both_names():
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    src = os.path.join(ROOT, "bevformer_tensorrt_b200", "csrc", "trt_plugin", "b200_trt_plugins.cpp")
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-I", os.path.join(ROOT, "tests", "mock_trt"),
                        "-I", os.path.join(ROOT, "include"), src], capture_output=True, text=True)  # fmt: skip
    assert r.returncode == 0, r.stderr
    text = open(src).read()
    assert '"BEVPoolV2TRT"' in text and '"BEVPoolV2TRT2"' in text


@pytest.fixture(scope="module")
def bev_capi(tmp_path_factory):
    """tests/mock_trt/bev_pool_capi.cpp (the shells + the mock plugin API + libb200_bev_ops.so) as a shared library."""
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    lib_dir = os.path.dirname(_lib.LIB_PATH)
    so = str(tmp_path_factory.mktemp("bev_capi") / "libbev_capi.so")
    cmd = ["g++", "-std=c++17", "-Wall", "-shared", "-fPIC", "-I", os.path.join(ROOT, "tests", "mock_trt"), "-I",
           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "mock_trt", "bev_pool_capi.cpp"), "-L", lib_dir,
           "-lb200_bev_ops", f"-Wl,-rpath,{lib_dir}", "-o", so]  # fmt: skip
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    lib = ctypes.CDLL(so)
    for fn in ("bcapi_create", "bcapi_deserialize"):
        getattr(lib, fn).restype = ctypes.c_void_p
    lib.bcapi_create.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.POINTER(ctypes.c_char_p),
                                 ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int32)]  # fmt: skip
    lib.bcapi_deserialize.argtypes = [ctypes.c_char_p, ctypes.c_void_p, ctypes.c_size_t]
    for fn in ("bcapi_plugin_type", "bcapi_plugin_version"):
        getattr(lib, fn).restype = ctypes.c_char_p
        getattr(lib, fn).argtypes = [ctypes.c_void_p]
    lib.bcapi_serialization_size.restype = ctypes.c_size_t
    lib.bcapi_serialization_size.argtypes = [ctypes.c_void_p]
    lib.bcapi_serialize.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    lib.bcapi_output_dims.argtypes = [ctypes.c_void_p, ctypes.c_int32, ctypes.POINTER(ctypes.c_int32)]
    lib.bcapi_destroy.argtypes = [ctypes.c_void_p]
    return lib


def create(lib, name, fields):
    names = (ctypes.c_char_p * max(len(fields), 1))(*[k.encode() for k in fields])
    vals = [v for vs in fields.values() for v in vs]
    values = (ctypes.c_int32 * max(len(vals), 1))(*vals)
    lengths = (ctypes.c_int32 * max(len(fields), 1))(*[len(v) for v in fields.values()])
    p = lib.bcapi_create(name.encode(), len(fields), names, values, lengths)
    assert p, name
    return p


def test_plugin_creators_fields_dims_and_serialisation(bev_capi):
    lib = bev_capi
    buf = ctypes.create_string_buffer(256)
    for name in ("BEVPoolV2TRT", "BEVPoolV2TRT2"):
        lib.bcapi_field_names(name.encode(), buf, 256)
        assert buf.value == b"out_height,out_width"
        p = create(lib, name, {"out_height": [200], "out_width": [100]})
        assert lib.bcapi_plugin_type(p) == name.encode() and lib.bcapi_plugin_version(p) == b"1"
        dims = (ctypes.c_int32 * 4)()
        assert lib.bcapi_output_dims(p, 80, dims) == 4 and list(dims) == [1, 200, 100, 80]
        assert lib.bcapi_serialization_size(p) == 8
        blob = ctypes.create_string_buffer(8)
        lib.bcapi_serialize(p, blob)
        assert np.frombuffer(blob.raw, np.int32).tolist() == [100, 200]  # out_width, then out_height
        q = lib.bcapi_deserialize(name.encode(), blob, 8)
        assert lib.bcapi_plugin_type(q) == name.encode()
        assert lib.bcapi_output_dims(q, 3, dims) == 4 and list(dims) == [1, 200, 100, 3]
        lib.bcapi_destroy(p)
        lib.bcapi_destroy(q)
    # the other plugins' blobs keep their size: Attrs (11 int32) + the input count
    r = create(lib, "RotateTRT", {"interpolation": [1]})
    assert lib.bcapi_serialization_size(r) == 48
    lib.bcapi_destroy(r)


def test_workload_generator_is_deterministic():
    for name in WORKLOADS:
        a = make_bev_pool_inputs(name, 3)
        b = make_bev_pool_inputs(name, 3)
        assert input_digest(a[0], a[1], *a[2]) == input_digest(b[0], b[1], *b[2]) and a[3] == b[3]
        assert input_digest(a[0], a[1]) != input_digest(*make_bev_pool_inputs(name, 4)[:2])
        rd, rf, rb, st, ln = a[2]
        assert torch.all(rb[1:] >= rb[:-1]) and int(ln.sum()) == rd.numel() and torch.all(ln > 0)
        assert torch.unique(rd).numel() == rd.numel()  # each depth element referenced once
        assert torch.equal(st[1:], torch.cumsum(ln, 0)[:-1].int())
