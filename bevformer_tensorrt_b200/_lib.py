"""ctypes binding of libb200_bev_ops.so (C ABI declared in include/b200_bev_ops.h).

There is no CPU fallback and no PyTorch fallback: if the shared library is missing the import of any operator fails
loudly with the build command, and if no CUDA device is present the operators raise.
"""
import ctypes
import os

_PKG = os.path.dirname(os.path.abspath(__file__))
# B200_BEV_OPS_LIB lets A/B experiments load an alternative build of the same ABI (scripts/ab_build.sh)
LIB_PATH = os.environ.get("B200_BEV_OPS_LIB") or os.path.join(_PKG, "lib", "libb200_bev_ops.so")

B200_OK = 0
STATUS = {0: "ok", 1: "unsupported dtype/format/shape", 2: "bad parameter", 3: "CUDA launch error"}

_vp, _i, _f = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
_ip = ctypes.POINTER(ctypes.c_int)


class B200OpsError(RuntimeError):
    def __init__(self, fn, status):
        super().__init__(f"{fn} failed: status {status} ({STATUS.get(status, 'unknown')})")
        self.status = status


class Dims(ctypes.Structure):
    _fields_ = [("nbDims", ctypes.c_int32), ("d", ctypes.c_int32 * 8)]


class TensorDesc(ctypes.Structure):
    """POD mirror of nvinfer1::PluginTensorDesc (b200_tensor_desc)."""

    _fields_ = [("dims", Dims), ("type", ctypes.c_int32), ("format", ctypes.c_int32), ("scale", ctypes.c_float)]


#: storage dtype of a float entry -> (entry-name suffix, dtype code of the workspace-size queries). The codes are
#: nvinfer1::DataType's (b200_tensor_desc.type): kFLOAT 0, kHALF 1, kBF16 7.
DTYPE_CODES = {"float32": ("f32", 0), "float16": ("f16", 1), "bfloat16": ("bf16", 7)}

_MSDA_DIMS = [_i] * 8  # batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group
_BEV_POOL_DIMS = [_i, _i, _i, ctypes.c_longlong, ctypes.c_longlong, _i, _i]  # C, P, I, depth_size, feat_rows, out h, w

SIGNATURES = {
    # name: (restype, argtypes)
    "b200_bev_ops_version": (ctypes.c_char_p, []),
    "b200_status_string": (ctypes.c_char_p, [_i]),
    "b200_launch_count": (ctypes.c_ulonglong, []),
    "b200_msda_f32": (_i, [_vp] * 5 + _MSDA_DIMS + [_vp, _vp]),
    "b200_msda_f16": (_i, [_vp] * 5 + _MSDA_DIMS + [_vp, _vp]),
    "b200_msda_f16_h2": (_i, [_vp] * 5 + _MSDA_DIMS + [_vp, _vp]),
    "b200_msda_bf16": (_i, [_vp] * 5 + _MSDA_DIMS + [_vp, _vp]),
    "b200_msda_i8": (_i, [_vp, _f, _vp, _vp, _i, _vp, _f, _vp, _f] + _MSDA_DIMS + [_vp, _f, _vp]),
    "b200_msda_sca_f32": (_i, [_vp] * 6 + _MSDA_DIMS + [_vp, _vp]),
    "b200_msda_sca_f16": (_i, [_vp] * 6 + _MSDA_DIMS + [_vp, _vp]),
    "b200_msda_sca_bf16": (_i, [_vp] * 6 + _MSDA_DIMS + [_vp, _vp]),
    "b200_msda_sca_shared_f32": (_i, [_vp] * 6 + _MSDA_DIMS + [_vp, _vp]),
    "b200_msda_sca_shared_f16": (_i, [_vp] * 6 + _MSDA_DIMS + [_vp, _vp]),
    "b200_msda_sca_shared_bf16": (_i, [_vp] * 6 + _MSDA_DIMS + [_vp, _vp]),
    "b200_msda_i8_workspace_size": (ctypes.c_size_t, [_i] * 7),
    "b200_msda_i8_ws": (_i, [_vp, _f, _vp, _vp, _i, _vp, _f, _vp, _f] + _MSDA_DIMS + [_vp, _f, _vp, ctypes.c_size_t, _vp, _vp]),
    "b200_sca_peer_reduce": (_i, [ctypes.POINTER(_vp), ctypes.POINTER(_vp), _i, _i, ctypes.c_uint, ctypes.c_longlong,
                                  ctypes.c_longlong, _vp, _i, _vp, ctypes.c_longlong, _vp]),
    "b200_sca_peer_reduce_auto": (_i, [ctypes.POINTER(_vp), ctypes.POINTER(_vp), ctypes.POINTER(_vp), _i, _i, ctypes.c_longlong,
                                       ctypes.c_longlong, _vp, _i, ctypes.c_longlong, _vp]),
    "b200_sca_peer_pull_auto": (_i, [ctypes.POINTER(_vp), ctypes.POINTER(_vp), ctypes.POINTER(_vp), _i, _i, ctypes.c_longlong,
                                     ctypes.c_longlong, _vp, _vp]),
    "b200_sca_peer_add_auto": (_i, [_vp, _vp, _vp, _i, ctypes.c_longlong, ctypes.c_longlong, _vp, _vp, _i,
                                    ctypes.c_longlong, _vp]),
    "b200_msda_f32_trace": (_i, [_vp] * 5 + _MSDA_DIMS + [_vp, _vp, _vp]),
    "b200_msda_f16_trace": (_i, [_vp] * 5 + _MSDA_DIMS + [_vp, _vp, _vp]),
    "b200_msda_bf16_trace": (_i, [_vp] * 5 + _MSDA_DIMS + [_vp, _vp, _vp]),
    "b200_msda_i8_trace": (_i, [_vp, _f, _vp, _vp, _i, _vp, _f, _vp, _f] + _MSDA_DIMS + [_vp, _f, _vp, _vp]),
    "b200_msda_debug_indices": (_i, [_i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "b200_msda_backward_workspace_size": (ctypes.c_size_t, [_i] + _MSDA_DIMS),
    "b200_msda_backward_f32": (_i, [_vp] * 11 + _MSDA_DIMS + [_vp]),
    "b200_msda_backward_f16": (_i, [_vp] * 11 + _MSDA_DIMS + [_vp]),
    "b200_msda_backward_bf16": (_i, [_vp] * 11 + _MSDA_DIMS + [_vp]),
    "b200_msda_sca_backward_f32": (_i, [_vp] * 12 + _MSDA_DIMS + [_vp]),
    "b200_msda_sca_backward_f16": (_i, [_vp] * 12 + _MSDA_DIMS + [_vp]),
    "b200_msda_sca_backward_bf16": (_i, [_vp] * 12 + _MSDA_DIMS + [_vp]),
    "b200_msda_sca_shared_backward_f32": (_i, [_vp] * 12 + _MSDA_DIMS + [_vp]),
    "b200_msda_sca_shared_backward_f16": (_i, [_vp] * 12 + _MSDA_DIMS + [_vp]),
    "b200_msda_sca_shared_backward_bf16": (_i, [_vp] * 12 + _MSDA_DIMS + [_vp]),
    "b200_msda_set_f16_mode": (_i, [_i]),
    "b200_msda_set_f16_path": (_i, [_i]),
    "b200_msda_set_batch_units": (_i, [_i, _i]),
    "b200_msda_set_gather_variant": (_i, [_i]),
    "b200_msda_set_resident_bytes": (_i, [_i]),
    "b200_msda_set_i8_resident_bytes": (_i, [_i]),
    "b200_msda_enqueue": (_i, [ctypes.POINTER(TensorDesc), ctypes.POINTER(TensorDesc), ctypes.POINTER(_vp),
                               ctypes.POINTER(_vp), _vp, _vp, _i]),
    "b200_msda_enqueue_workspace_size": (ctypes.c_size_t, [ctypes.POINTER(TensorDesc)]),
    "b200_msda_supports_format": (_i, [_i, ctypes.POINTER(TensorDesc), _i, _i]),
    "b200_grid_sampler_enqueue": (_i, [ctypes.POINTER(TensorDesc), ctypes.POINTER(TensorDesc), ctypes.POINTER(_vp),
                                       ctypes.POINTER(_vp), _vp, _vp, _i, _i, _i]),
    "b200_grid_sampler_supports_format": (_i, [_i, ctypes.POINTER(TensorDesc), _i, _i, _i]),
    "b200_rotate_enqueue": (_i, [ctypes.POINTER(TensorDesc), ctypes.POINTER(TensorDesc), ctypes.POINTER(_vp),
                                 ctypes.POINTER(_vp), _vp, _vp, _i, _i]),
    "b200_rotate_supports_format": (_i, [_i, ctypes.POINTER(TensorDesc), _i, _i, _i]),
    "b200_dcn_supports_format": (_i, [_i, ctypes.POINTER(TensorDesc), _i, _i, _i, _i]),
    "b200_dcn_enqueue_workspace_size": (ctypes.c_size_t, [ctypes.POINTER(TensorDesc), _ip, _ip, _ip, _i, _i]),
    "b200_dcn_enqueue": (_i, [ctypes.POINTER(TensorDesc), ctypes.POINTER(TensorDesc), ctypes.POINTER(_vp),
                              ctypes.POINTER(_vp), _vp, _vp, _i, _ip, _ip, _ip, _i, _i]),
    "b200_dcn_workspace_size": (ctypes.c_size_t, [_i] * 13),
    "b200_dcn_i8_workspace_size": (ctypes.c_size_t, [_i] * 15),
    "b200_dcn_set_fused": (_i, [_i]),
    "b200_dcn_pack_weights_f16": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "b200_dcn_f16_ex": (_i, [_vp] * 7 + [_i] * 16 + [_vp]),
    "b200_dcn_i8": (_i, [_vp, _f, _vp, _f, _vp, _i, _vp, _f, _vp, _f, _vp, _f, _vp] + [_i] * 16 + [_vp, _vp]),
    "b200_dcn_f32": (_i, [_vp] * 7 + [_i] * 16 + [_vp, _vp]),
    "b200_dcn_f16": (_i, [_vp] * 7 + [_i] * 16 + [_vp, _vp]),
    "b200_dcn_bf16": (_i, [_vp] * 7 + [_i] * 16 + [_vp, _vp]),
    "b200_dcn_f16_chw2": (_i, [_vp] * 7 + [_i] * 16 + [_vp, _vp]),
    "b200_dcn_f16_chw2_workspace_size": (ctypes.c_size_t, [_i] * 15),
    "b200_dcn_backward_workspace_size": (ctypes.c_size_t, [_i] * 16),
    "b200_dcn_backward_f32": (_i, [_vp] * 11 + [_i] * 15 + [_vp]),
    "b200_dcn_backward_f16": (_i, [_vp] * 11 + [_i] * 16 + [_vp]),
    "b200_dcn_backward_bf16": (_i, [_vp] * 11 + [_i] * 15 + [_vp]),
    "b200_grid_sample_set_tile_path": (_i, [_i]),
    "b200_grid_sample_f32": (_i, [_vp, _vp, _vp, _ip, _ip, _ip, _i, _i, _i, _i, _vp]),
    "b200_grid_sample_f16": (_i, [_vp, _vp, _vp, _ip, _ip, _ip, _i, _i, _i, _i, _vp]),
    "b200_grid_sample_f16_chw2": (_i, [_vp, _vp, _vp, _ip, _ip, _ip, _i, _i, _i, _i, _vp]),
    "b200_grid_sample_i8_chw4": (_i, [_vp, _f, _vp, _f, _vp, _f, _ip, _ip, _ip, _i, _i, _i, _i, _vp]),
    "b200_rotate_f32": (_i, [_vp, _vp, _vp, _vp, _ip, _i, _vp]),
    "b200_rotate_f16": (_i, [_vp, _vp, _vp, _vp, _ip, _i, _vp]),
    "b200_rotate_f16_h2": (_i, [_vp, _vp, _vp, _vp, _ip, _i, _vp]),
    "b200_rotate_i8": (_i, [_vp, _f, _vp, _f, _vp, _vp, _i, _ip, _i, _vp]),
    "b200_rotate_hwc": (_i, [_vp, _vp, _vp, _vp, _i, _ip, _i, _vp]),
    "b200_rotate_debug_indices": (_i, [_vp, _vp, _ip, _vp, _vp]),
    "b200_bev_point_sampling": (_i, [_vp, ctypes.POINTER(ctypes.c_double), _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "b200_bev_point_sampling_pillar_heights": (_i, [ctypes.POINTER(ctypes.c_double), _i, ctypes.POINTER(_f)]),
    # depth, feat, ranks_depth, ranks_feat, ranks_bev, interval_starts, interval_lengths, channels, num_points,
    # num_intervals, depth_size, feat_rows, out_height, out_width, out, stream
    "b200_bev_pool_f32": (_i, [_vp] * 7 + _BEV_POOL_DIMS + [_vp, _vp]),
    "b200_bev_pool_f16": (_i, [_vp] * 7 + _BEV_POOL_DIMS + [_vp, _vp]),
    "b200_bev_pool_bf16": (_i, [_vp] * 7 + _BEV_POOL_DIMS + [_vp, _vp]),
    "b200_bev_pool_f32_depth": (_i, [_i] + [_vp] * 7 + _BEV_POOL_DIMS + [_vp, _vp]),  # feat_dtype first
    "b200_bev_pool_i8": (_i, [_vp, _f, _vp, _f] + [_vp] * 5 + _BEV_POOL_DIMS + [_vp, _f, _vp]),
    "b200_bev_pool_backward_workspace_size": (ctypes.c_size_t, [_i]),
    "b200_bev_pool_backward_f32": (_i, [_vp] * 9 + _BEV_POOL_DIMS + [_vp, _vp, _vp, ctypes.c_size_t, _vp]),
    "b200_bev_pool_backward_f16": (_i, [_vp] * 9 + _BEV_POOL_DIMS + [_vp, _vp, _vp, ctypes.c_size_t, _vp]),
    "b200_bev_pool_backward_bf16": (_i, [_vp] * 9 + _BEV_POOL_DIMS + [_vp, _vp, _vp, ctypes.c_size_t, _vp]),
    "b200_bev_pool_backward_f32_depth": (_i, [_i] + [_vp] * 9 + _BEV_POOL_DIMS + [_vp, _vp, _vp, ctypes.c_size_t, _vp]),
    "b200_bev_pool_enqueue": (_i, [ctypes.POINTER(TensorDesc), ctypes.POINTER(TensorDesc), ctypes.POINTER(_vp),
                                   ctypes.POINTER(_vp), _vp, _vp, _i, _i]),
    "b200_bev_pool_supports_format": (_i, [_i, ctypes.POINTER(TensorDesc), _i, _i]),
}  # fmt: skip

_lib = None


def load() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: the CUDA extension is not built. Run "
                "`python -m bevformer_tensorrt_b200.build` (nvcc, sm_90a). There is no CPU/PyTorch fallback."
            )
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            try:
                fn = getattr(lib, name)
            except AttributeError as e:  # header/library mismatch: the .so is older than the sources
                raise ImportError(f"{LIB_PATH} lacks `{name}`: stale build, rerun "
                                  "`python -m bevformer_tensorrt_b200.build --force`") from e
            fn.restype, fn.argtypes = res, args
        _lib = lib
    return _lib


def check(fn_name: str, status: int) -> None:
    if status != B200_OK:
        raise B200OpsError(fn_name, status)


def call(fn_name: str, device, *args, accept=(B200_OK,)) -> int:
    """Calls the C entry ``fn_name`` with ``args`` followed by the current stream of ``device``, with ``device`` made
    the current device, and returns its status. A status outside ``accept`` raises B200OpsError; callers that fall back
    on B200_ERR_UNSUPPORTED pass ``accept=(0, 1)``."""
    import torch

    with torch.cuda.device(device):
        status = getattr(load(), fn_name)(*args, current_stream_ptr())
    if status not in accept:
        raise B200OpsError(fn_name, status)
    return status


def float_dtype(dtype, fn_name: str):
    """(entry-name suffix, workspace-query dtype code) of a float storage dtype: ("f32", 0), ("f16", 1) or ("bf16", 7).
    Any other dtype raises B200OpsError(fn_name, 1), the status of an unsupported dtype."""
    code = DTYPE_CODES.get(str(dtype).rpartition(".")[2])
    if code is None:
        raise B200OpsError(fn_name, 1)
    return code


def launch_count() -> int:
    return int(load().b200_launch_count())


def current_stream_ptr():
    import torch

    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
