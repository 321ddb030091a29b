"""BF16 entries of the C ABI without a GPU: every symbol is declared, bound and exported; the workspace queries take
dtype 7 (nvinfer1::DataType::kBF16; 2 is kINT8); argument errors return B200_ERR_BAD_PARAM before anything is launched (fake device addresses, launch counter
unchanged)."""
import ctypes

import pytest
import torch

from bevformer_tensorrt_b200 import _lib
from tests.test_host_logic import _header_symbols

BF16_ENTRIES = ("b200_msda_bf16", "b200_msda_bf16_trace", "b200_msda_sca_bf16", "b200_msda_sca_shared_bf16",
                "b200_msda_backward_bf16", "b200_msda_sca_backward_bf16", "b200_msda_sca_shared_backward_bf16",
                "b200_dcn_bf16", "b200_dcn_backward_bf16")  # fmt: skip


def test_symbols_are_declared_bound_and_exported():
    syms = _header_symbols()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for s in BF16_ENTRIES:
        assert s in syms, s
        assert s in _lib.SIGNATURES, s
        assert hasattr(lib, s), s
    _lib.load()  # binds every signature


def test_bf16_entries_mirror_their_fp16_siblings():
    """Same argument list as the FP16 sibling; the DCN backward has the FP32 entry's (no flags)."""
    for s in BF16_ENTRIES:
        sib = s.replace("bf16", "f32" if s == "b200_dcn_backward_bf16" else "f16")
        assert _lib.SIGNATURES[s] == _lib.SIGNATURES[sib], s


def test_float_dtype_codes():
    assert _lib.float_dtype(torch.float32, "x") == ("f32", 0)
    assert _lib.float_dtype(torch.float16, "x") == ("f16", 1)
    assert _lib.float_dtype(torch.bfloat16, "x") == ("bf16", 7)
    for dt in (torch.float64, torch.int8, torch.int32):
        with pytest.raises(_lib.B200OpsError) as e:
            _lib.float_dtype(dt, "x")
        assert e.value.status == 1


# ---- workspace queries ---------------------------------------------------------------------------------------------------
MSDA_DIMS = [(6, 30825, 8, 32, 4, 2500, 8, 4), (2, 1000, 8, 32, 1, 900, 4, 1), (1, 61, 3, 20, 2, 17, 3, 1)]


@pytest.mark.parametrize("dims", MSDA_DIMS)
def test_msda_backward_workspace_bf16_is_the_fp16_formula(dims):
    """FP16 and BF16 both accumulate grad_value in fp32 in the workspace, then keep the reference-point partials."""
    lib = _lib.load()
    b, s, m, c, _, q, _, g = dims
    f16 = lib.b200_msda_backward_workspace_size(1, *dims)
    assert lib.b200_msda_backward_workspace_size(7, *dims) == f16
    a256 = lambda n: (n + 255) // 256 * 256  # noqa: E731
    assert f16 == a256(b * s * m * c * 4) + a256(b * q * m * g * 2 * 4)
    assert lib.b200_msda_backward_workspace_size(2, *dims) == 0  # kINT8: no backward
    assert lib.b200_msda_backward_workspace_size(7, *dims[:2], 0, *dims[3:]) == 0


DCN_GEO = [(6, 256, 58, 100, 256, 3, 3, 1, 1, 1, 1, 1, 1, 1, 1), (2, 16, 13, 17, 12, 3, 3, 1, 1, 1, 1, 1, 1, 2, 2)]


@pytest.mark.parametrize("geo", DCN_GEO)
def test_dcn_workspace_bf16(geo):
    """Backward: the FP16 size (fp32 grad_input accumulator). Forward: BF16 runs the generic kernel, which needs no
    scratch, so its size is FP32's (the FP16 size adds the fused kernel's NHWC copy)."""
    lib = _lib.load()
    assert lib.b200_dcn_backward_workspace_size(7, *geo) == lib.b200_dcn_backward_workspace_size(1, *geo)
    assert lib.b200_dcn_backward_workspace_size(7, *geo) > lib.b200_dcn_backward_workspace_size(0, *geo)
    n, c, h, w, _, kw, kh, sw, sh, pw, ph, dw, dh, _, _ = geo
    fwd = (n, c, h, w, kw, kh, sw, sh, pw, ph, dw, dh)
    assert lib.b200_dcn_workspace_size(7, *fwd) == lib.b200_dcn_workspace_size(0, *fwd) == 256


# ---- argument errors before any launch -----------------------------------------------------------------------------------
_A = 1 << 20
_P = [_A * (i + 1) for i in range(12)]  # fake 16-byte-aligned device addresses, never touched
_D = [2, 100, 8, 32, 2, 40, 4, 2]  # batch, spatial_size, heads, channels, levels, queries, points, points_per_group


def _launches_unchanged(fn):
    before = _lib.launch_count()
    st = fn()
    assert _lib.launch_count() == before
    return st


def _fwd(name, ptrs, dims, extra=0):
    lib = _lib.load()
    records = [_P[10]] if name.endswith("_trace") else []
    return _launches_unchanged(lambda: getattr(lib, name)(*ptrs[: 5 + extra], *dims, _P[11], *records, None))


FWD = [("b200_msda_bf16", 0), ("b200_msda_bf16_trace", 0), ("b200_msda_sca_bf16", 1), ("b200_msda_sca_shared_bf16", 1)]


@pytest.mark.parametrize("name,extra", FWD)
@pytest.mark.parametrize("which", range(5))
def test_msda_forward_null_pointer_is_bad_param(name, extra, which):
    ptrs = list(_P)
    ptrs[which] = None
    assert _fwd(name, ptrs, _D, extra) == 2


@pytest.mark.parametrize("name,extra", FWD)
@pytest.mark.parametrize("idx", range(8))
def test_msda_forward_non_positive_dimension_is_bad_param(name, extra, idx):
    for v in (0, -3):
        dims = list(_D)
        dims[idx] = v
        assert _fwd(name, _P, dims, extra) == 2


def test_msda_trace_without_records_is_bad_param():
    lib = _lib.load()
    assert _launches_unchanged(lambda: lib.b200_msda_bf16_trace(*_P[:5], *_D, _P[11], None, None)) == 2


BWD = [("b200_msda_backward_bf16", 1), ("b200_msda_sca_backward_bf16", 2), ("b200_msda_sca_shared_backward_bf16", 2)]


def _bwd(name, n_in, ptrs, dims):
    lib = _lib.load()
    # 0 value, 1 shapes, 2 ref, 3 off, 4 logits, 5 grad_out | bev_mask, (6 grad_slots), 7-10 the four gradients
    args = ptrs[: 5 + n_in] + ptrs[7:11] + [_A * 64]
    return _launches_unchanged(lambda: getattr(lib, name)(*args, *dims, None))


@pytest.mark.parametrize("name,n_in", BWD)
@pytest.mark.parametrize("which", [0, 1, 2, 3, 4, 5, 6])
def test_msda_backward_null_required_pointer_is_bad_param(name, n_in, which):
    if which >= 5 + n_in:
        pytest.skip("the plugin-op backward has no sixth input")
    ptrs = list(_P)
    ptrs[which] = None
    assert _bwd(name, n_in, ptrs, _D) == 2


@pytest.mark.parametrize("name,n_in", BWD)
@pytest.mark.parametrize("idx", range(8))
def test_msda_backward_non_positive_dimension_is_bad_param(name, n_in, idx):
    dims = list(_D)
    dims[idx] = 0
    assert _bwd(name, n_in, _P, dims) == 2


@pytest.mark.parametrize("name,n_in", BWD)
@pytest.mark.parametrize("which,shift", [(0, 1), (3, 1), (4, 1), (7, 1), (9, 1), (10, 1), (2, 2), (8, 2)])
def test_msda_backward_misaligned_pointer_is_bad_param(name, n_in, which, shift):
    """bf16 tensors must be 2-byte aligned, the fp32 reference points (2) and their gradient (8) 4-byte aligned: a
    2-byte shift that a bf16 tensor would accept is rejected for them."""
    ptrs = list(_P)
    ptrs[which] += shift
    assert _bwd(name, n_in, ptrs, _D) == 2


# DCN: input, weight, bias, offset, mask, output (forward); input, weight, offset, mask, grad_output, 5 grads (backward)
_GEO = [2, 64, 20, 24, 128, 3, 3, 1, 1, 1, 1, 1, 1, 1, 1]


def _dcn_fwd(ptrs, geo=_GEO):
    lib = _lib.load()
    return _launches_unchanged(lambda: lib.b200_dcn_bf16(*ptrs[:6], _A * 64, *geo, 1, None, None))


def _dcn_bwd(ptrs, geo=_GEO, ws=_A * 64):
    lib = _lib.load()
    return _launches_unchanged(lambda: lib.b200_dcn_backward_bf16(*ptrs[:10], ws, *geo, None))


@pytest.mark.parametrize("which", [0, 1, 3, 4, 5])
def test_dcn_forward_null_required_pointer_is_bad_param(which):
    ptrs = list(_P)
    ptrs[which] = None
    assert _dcn_fwd(ptrs) == 2


@pytest.mark.parametrize("idx", [i for i in range(15) if i not in (9, 10)])  # padding may be 0
def test_dcn_non_positive_dimension_is_bad_param(idx):
    geo = list(_GEO)
    geo[idx] = 0
    assert _dcn_fwd(_P, geo) == 2
    assert _dcn_bwd(_P, geo) == 2


@pytest.mark.parametrize("which", range(5))
def test_dcn_backward_null_required_pointer_is_bad_param(which):
    ptrs = list(_P)
    ptrs[which] = None
    assert _dcn_bwd(ptrs) == 2
    assert _dcn_bwd(_P, ws=None) == 2


@pytest.mark.parametrize("which", range(10))
def test_dcn_backward_misaligned_pointer_is_bad_param(which):
    ptrs = list(_P)
    ptrs[which] += 1
    assert _dcn_bwd(ptrs) == 2
