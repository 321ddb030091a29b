"""BEVPoolV2's BF16 and FP32-depth entries without a GPU: the four entries are declared, bound and exported with their
FP16 siblings' arguments (the FP32-depth ones led by feat_dtype), the binding's (depth, feat) dtype table, and every
argument error returns its status before anything is launched (fake device addresses, launch counter unchanged)."""
import ctypes

import pytest
import torch

from bevformer_tensorrt_b200 import _lib
from bevformer_tensorrt_b200.functions.bev_pool_v2 import _entries
from tests.test_host_logic import _header_symbols

ENTRIES = ("b200_bev_pool_bf16", "b200_bev_pool_backward_bf16", "b200_bev_pool_f32_depth",
           "b200_bev_pool_backward_f32_depth")  # fmt: skip


def test_symbols_are_declared_bound_and_exported():
    syms = _header_symbols()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for s in ENTRIES:
        assert s in syms, s
        assert s in _lib.SIGNATURES, s
        assert hasattr(lib, s), s
    _lib.load()  # binds every signature


def test_entries_mirror_their_fp16_siblings():
    """bf16: the FP16 entry's arguments; f32_depth: an int feat_dtype, then the FP16 entry's arguments."""
    for s in ENTRIES:
        sib = s.replace("bf16", "f16").replace("f32_depth", "f16")
        res, args = _lib.SIGNATURES[sib]
        want = (res, args) if "bf16" in s else (res, [ctypes.c_int] + args)
        assert _lib.SIGNATURES[s] == want, s


F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16


@pytest.mark.parametrize("pair,want", [
    ((F32, F32), ("b200_bev_pool_f32", "b200_bev_pool_backward_f32", ())),
    ((F16, F16), ("b200_bev_pool_f16", "b200_bev_pool_backward_f16", ())),
    ((BF16, BF16), ("b200_bev_pool_bf16", "b200_bev_pool_backward_bf16", ())),
    ((F32, F16), ("b200_bev_pool_f32_depth", "b200_bev_pool_backward_f32_depth", (1,))),
    ((F32, BF16), ("b200_bev_pool_f32_depth", "b200_bev_pool_backward_f32_depth", (7,))),
])  # fmt: skip
def test_binding_picks_the_entry_from_the_dtype_pair(pair, want):
    assert _entries(torch.empty(0, dtype=pair[0]), torch.empty(0, dtype=pair[1])) == want


@pytest.mark.parametrize("pair", [(F16, BF16), (BF16, F16), (F16, F32), (BF16, F32), (torch.float64, torch.float64),
                                  (F32, torch.float64), (torch.float64, F16), (torch.int8, torch.int8)])  # fmt: skip
def test_binding_rejects_every_other_pair_with_status_1(pair):
    with pytest.raises(_lib.B200OpsError) as e:
        _entries(torch.empty(0, dtype=pair[0]), torch.empty(0, dtype=pair[1]))
    assert e.value.status == 1


# ---- argument errors before any launch -----------------------------------------------------------------------------------
_A = 1 << 20
_DIMS = [16, 10, 3, 100, 50, 8, 8]  # C, P, I, depth_size, feat_rows, out h, out w


def _ptrs(n, shift=None, by=0):
    """n fake 16-byte-aligned device addresses, never touched; the one at ``shift`` moved by ``by`` bytes."""
    return [ctypes.c_void_p(_A * (i + 1) + (by if i == shift else 0)) for i in range(n)]


def _status(name, lead, shift=None, by=0):
    """The entry's status on fake pointers: forward (depth, feat, 5 int32 arrays, out) or backward (out_grad, depth,
    feat, 5 int32 arrays, feat_order, depth_grad, feat_grad, workspace). The launch counter must not move."""
    lib = _lib.load()
    before = _lib.launch_count()
    if "backward" in name:
        p = _ptrs(12, shift, by)
        st = getattr(lib, name)(*lead, *p[:9], *_DIMS, p[9], p[10], p[11], 40, None)
    else:
        p = _ptrs(8, shift, by)
        st = getattr(lib, name)(*lead, *p[:7], *_DIMS, p[7], None)
    assert _lib.launch_count() == before
    return st


F32_DEPTH = ("b200_bev_pool_f32_depth", "b200_bev_pool_backward_f32_depth")


@pytest.mark.parametrize("name", F32_DEPTH)
@pytest.mark.parametrize("feat_dtype", [0, 2, 3, 5, 6, 8, -1])
def test_f32_depth_feat_dtype_outside_fp16_bf16_is_unsupported(name, feat_dtype):
    assert _status(name, [feat_dtype]) == 1


@pytest.mark.parametrize("name", F32_DEPTH)
def test_f32_depth_unsupported_feat_dtype_is_reported_before_argument_errors(name):
    assert _status(name, [0], shift=1, by=1) == 1
    assert _status(name, [1], shift=1, by=1) == 2


# (forward index, backward index) of depth, feat, out / out_grad, and the backward's depth_grad, feat_grad
_FWD = {"depth": 0, "feat": 1, "out": 7}
_BWD = {"out_grad": 0, "depth": 1, "feat": 2, "depth_grad": 9, "feat_grad": 10}


@pytest.mark.parametrize("feat_dtype", [1, 7])
@pytest.mark.parametrize("tensor", ["depth", "depth_grad"])
def test_f32_depth_tensors_two_bytes_off_are_bad_param(feat_dtype, tensor):
    """FP32 depth and its gradient must be 4-byte aligned: a 2-byte shift that a 2-byte tensor would accept is
    rejected for them."""
    if tensor in _FWD:
        assert _status("b200_bev_pool_f32_depth", [feat_dtype], _FWD[tensor], 2) == 2
    assert _status("b200_bev_pool_backward_f32_depth", [feat_dtype], _BWD[tensor], 2) == 2


@pytest.mark.parametrize("feat_dtype", [1, 7])
@pytest.mark.parametrize("tensor", ["feat", "out", "out_grad", "feat_grad"])
def test_f32_depth_feature_tensors_one_byte_off_are_bad_param(feat_dtype, tensor):
    if tensor in _FWD:
        assert _status("b200_bev_pool_f32_depth", [feat_dtype], _FWD[tensor], 1) == 2
    if tensor in _BWD:
        assert _status("b200_bev_pool_backward_f32_depth", [feat_dtype], _BWD[tensor], 1) == 2


@pytest.mark.parametrize("tensor", ["depth", "feat", "out", "out_grad", "depth_grad", "feat_grad"])
def test_bf16_tensors_one_byte_off_are_bad_param(tensor):
    if tensor in _FWD:
        assert _status("b200_bev_pool_bf16", [], _FWD[tensor], 1) == 2
    if tensor in _BWD:
        assert _status("b200_bev_pool_backward_bf16", [], _BWD[tensor], 1) == 2


@pytest.mark.parametrize("name,lead", [("b200_bev_pool_bf16", []), ("b200_bev_pool_backward_bf16", []),
                                       ("b200_bev_pool_f32_depth", [1]), ("b200_bev_pool_f32_depth", [7]),
                                       ("b200_bev_pool_backward_f32_depth", [1]),
                                       ("b200_bev_pool_backward_f32_depth", [7])])  # fmt: skip
@pytest.mark.parametrize("which", range(3, 8))
def test_int32_arrays_two_bytes_off_are_bad_param(name, lead, which):
    """The five index arrays (and the backward's feat_order) stay int32-aligned in every new entry."""
    idx = which if "backward" in name else which - 1  # the backward's arrays follow out_grad
    assert _status(name, lead, idx, 2) == 2
    if "backward" in name and which == 7:
        assert _status(name, lead, 8, 2) == 2  # feat_order
