"""bevformer_tensorrt_b200 — BEVFormer's attention-sampling hot path (multi-scale deformable attention, grid sampler,
modulated deformable conv) as hand-written sm_90a CUDA behind the operator interface of DerryHub/BEVFormer_tensorrt.

Importing the package loads lib/libb200_bev_ops.so (built in-tree by ``python -m bevformer_tensorrt_b200.build``) and
fails loudly if it is missing — there is no CPU or PyTorch fallback on this path.
"""
import os as _os
import sys as _sys

from . import _lib

# Eager load: a missing or stale library is an ImportError at `import bevformer_tensorrt_b200`, not a late surprise.
# The only exemption is the build step itself (python -m bevformer_tensorrt_b200.build / __graft_entry__.build()),
# which has to import this package's build module before the library exists.
_building = _os.environ.get("B200_BEV_OPS_BUILDING") == "1" or any(
    a == "bevformer_tensorrt_b200.build" for a in getattr(_sys, "orig_argv", [])
)
if not _building:
    _lib.load()

from .functions import (  # noqa: E402
    TRT_FUNCTIONS,
    bev_point_sampling,
    bev_pool_v2,
    bev_pool_v2_2,
    bev_pool_v2_int8,
    get_reference_points_3d,
    grid_sampler,
    grid_sampler2,
    grid_sampler_chw2,
    grid_sampler_int8,
    modulated_deformable_conv2d,
    modulated_deformable_conv2d2,
    modulated_deformable_conv2d_int8,
    multi_scale_deformable_attn,
    multi_scale_deformable_attn2,
    multi_scale_deformable_attn_int8,
    multi_scale_deformable_attn_sca,
    multi_scale_deformable_attn_sca_shared,
    multi_scale_deformable_attn_queue_mean,
    point_sampling_trt,
    rotate,
    rotate2,
    rotate_chw2,
    rotate_hwc,
    rotate_int8,
    set_msda_v2,
    set_msda_f16_path,
    set_msda_batch_units,
    get_msda_batch_units,
    set_msda_gather_variant,
    get_msda_gather_variant,
    autotune_msda,
    autotune_msda_fused,
    set_msda_launch_shape,
    MSDA_LAUNCH_SHAPES,
)

from .host_pipeline import HostMSDA, empty_pinned  # noqa: E402

__all__ = [
    "HostMSDA",
    "empty_pinned",
    "TRT_FUNCTIONS",
    "bev_point_sampling",
    "bev_pool_v2",
    "bev_pool_v2_2",
    "bev_pool_v2_int8",
    "get_reference_points_3d",
    "grid_sampler",
    "grid_sampler2",
    "grid_sampler_chw2",
    "grid_sampler_int8",
    "modulated_deformable_conv2d",
    "modulated_deformable_conv2d2",
    "modulated_deformable_conv2d_int8",
    "multi_scale_deformable_attn",
    "multi_scale_deformable_attn2",
    "multi_scale_deformable_attn_int8",
    "multi_scale_deformable_attn_sca",
    "multi_scale_deformable_attn_sca_shared",
    "multi_scale_deformable_attn_queue_mean",
    "point_sampling_trt",
    "rotate",
    "rotate2",
    "rotate_chw2",
    "rotate_hwc",
    "rotate_int8",
    "set_msda_v2",
    "set_msda_f16_path",
    "set_msda_batch_units",
    "get_msda_batch_units",
    "set_msda_gather_variant",
    "get_msda_gather_variant",
    "autotune_msda",
    "autotune_msda_fused",
    "set_msda_launch_shape",
    "MSDA_LAUNCH_SHAPES",
]
__version__ = "0.1.2"
