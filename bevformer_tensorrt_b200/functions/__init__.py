"""Operator bindings with the reference's names (det2trt/models/functions/__init__.py:1-35) and its function
registry (det2trt/models/utils/register.py:9-69,86): ``TRT_FUNCTIONS.get("multi_scale_deformable_attn")`` etc."""
from ..registry import TRT_FUNCTIONS
from .bev_pool_v2 import bev_pool_v2, bev_pool_v2_2, bev_pool_v2_int8
from .grid_sampler import grid_sampler, grid_sampler2, grid_sampler_chw2, grid_sampler_int8
from .modulated_deformable_conv2d import (
    modulated_deformable_conv2d,
    modulated_deformable_conv2d2,
    modulated_deformable_conv2d_int8,
)
from .multi_scale_deformable_attn import (
    multi_scale_deformable_attn,
    multi_scale_deformable_attn2,
    multi_scale_deformable_attn_int8,
    multi_scale_deformable_attn_sca,
    multi_scale_deformable_attn_sca_shared,
    multi_scale_deformable_attn_queue_mean,
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
from .point_sampling import bev_point_sampling, get_reference_points_3d, point_sampling_trt
from .rotate import rotate, rotate2, rotate_chw2, rotate_hwc, rotate_int8

TRT_FUNCTIONS.register_module(module=grid_sampler)
TRT_FUNCTIONS.register_module(module=grid_sampler2)
TRT_FUNCTIONS.register_module(module=grid_sampler_chw2)
TRT_FUNCTIONS.register_module(module=grid_sampler_int8)

TRT_FUNCTIONS.register_module(module=modulated_deformable_conv2d)
TRT_FUNCTIONS.register_module(module=modulated_deformable_conv2d2)
TRT_FUNCTIONS.register_module(module=modulated_deformable_conv2d_int8)

TRT_FUNCTIONS.register_module(module=multi_scale_deformable_attn)
TRT_FUNCTIONS.register_module(module=multi_scale_deformable_attn2)
TRT_FUNCTIONS.register_module(module=multi_scale_deformable_attn_int8)
TRT_FUNCTIONS.register_module(module=multi_scale_deformable_attn_sca)
TRT_FUNCTIONS.register_module(module=multi_scale_deformable_attn_sca_shared)
TRT_FUNCTIONS.register_module(module=multi_scale_deformable_attn_queue_mean)

TRT_FUNCTIONS.register_module(module=rotate)
TRT_FUNCTIONS.register_module(module=rotate2)
TRT_FUNCTIONS.register_module(module=rotate_chw2)
TRT_FUNCTIONS.register_module(module=rotate_hwc)
TRT_FUNCTIONS.register_module(module=rotate_int8)

TRT_FUNCTIONS.register_module(module=get_reference_points_3d)
TRT_FUNCTIONS.register_module(module=point_sampling_trt)
TRT_FUNCTIONS.register_module(module=bev_point_sampling)

TRT_FUNCTIONS.register_module(module=bev_pool_v2)
TRT_FUNCTIONS.register_module(module=bev_pool_v2_2)
TRT_FUNCTIONS.register_module(module=bev_pool_v2_int8)
