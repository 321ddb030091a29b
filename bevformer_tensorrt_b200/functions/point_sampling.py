"""BEV pillar points -> per-camera reference points + visibility weights — host-side mirror of the encoder prologue
``BEVFormerEncoderTRTP.get_reference_points_3d`` / ``point_sampling_trt`` (det2trt/models/modules/encoder.py:168-259).

The reference evaluates this in eager PyTorch (about thirty small launches: linspace / repeat / stack, a broadcast
4x4 matmul, where / max / prod / clamp); ``point_sampling_trt`` here is one sm_90a kernel through the C ABI
(``b200_bev_point_sampling``) with the same arguments and return values:

    reference_points_cam  [num_cams, 1, Q, D, 2]   (the reference returns a permuted view of the same logical shape)
    bev_mask              [num_cams, Q, 1]

``bev_point_sampling`` is the fused form that also generates the pillar grid in registers (no ``ref_3d`` tensor).
"""
import ctypes

import torch

from .. import _lib


def get_reference_points_3d(H, W, Z=8, num_points_in_pillar=4, bs=1, device="cuda", dtype=torch.float):
    """Same signature and result as encoder.py:168-194: [1, num_points_in_pillar, H*W, 3] in [0, 1]. Plain tensor
    construction (it also yields ref_2d for temporal self-attention, encoder.py:290); not on the hot path."""
    D = num_points_in_pillar
    zs = torch.linspace(0.5, Z - 0.5, D, dtype=dtype, device=device).view(-1, 1, 1).expand(D, H, W) / Z
    xs = torch.linspace(0.5, W - 0.5, W, dtype=dtype, device=device).view(1, 1, W).expand(D, H, W) / W
    ys = torch.linspace(0.5, H - 0.5, H, dtype=dtype, device=device).view(1, H, 1).expand(D, H, W) / H
    return torch.stack((xs, ys, zs), -1).view(1, D, -1, 3)


def _launch(ref3d, pc_range, lidar2img, image_shape, bev_h, bev_w, D, dtype, device):
    if len(pc_range) != 6:
        raise ValueError("pc_range must be (x0, y0, z0, x1, y1, z1)")
    if dtype not in (torch.float32, torch.float16):
        raise _lib.B200OpsError("point_sampling_trt", 1)
    lidar2img = lidar2img.reshape(-1, 4, 4).to(device=device, dtype=torch.float32).contiguous()
    cams, Q = lidar2img.shape[0], bev_h * bev_w
    ref_cam = torch.empty(cams, 1, Q, D, 2, dtype=dtype, device=device)
    bev_mask = torch.empty(cams, Q, 1, dtype=dtype, device=device)
    pcr = (ctypes.c_double * 6)(*[float(v) for v in pc_range])
    _lib.call("b200_bev_point_sampling", device, ref3d.data_ptr() if ref3d is not None else None, pcr,
              lidar2img.data_ptr(), cams, int(image_shape[0]), int(image_shape[1]), bev_h, bev_w, D,
              int(dtype == torch.float16), ref_cam.data_ptr(), bev_mask.data_ptr())  # fmt: skip
    return ref_cam, bev_mask


def point_sampling_trt(reference_points, pc_range, lidar2img, image_shape):
    """encoder.py:196-259 with the same arguments: reference_points [1, D, Q, 3] (from get_reference_points_3d),
    pc_range 6 numbers, lidar2img [.., num_cams, 4, 4], image_shape (h, w). Returns (reference_points_cam, bev_mask)."""
    if not reference_points.is_cuda:
        raise RuntimeError("point_sampling_trt: reference_points must be a CUDA tensor (no CPU fallback exists)")
    if reference_points.dim() != 4 or reference_points.shape[0] != 1 or reference_points.shape[-1] != 3:
        raise ValueError("reference_points must be [1, num_points_in_pillar, num_query, 3]")
    ref = reference_points.contiguous()
    return _launch(ref, pc_range, lidar2img, image_shape, 1, ref.shape[2], ref.shape[1], ref.dtype, ref.device)


def bev_point_sampling(bev_h, bev_w, pc_range, lidar2img, image_shape, num_points_in_pillar=4, dtype=torch.float32):
    """get_reference_points_3d(bev_h, bev_w, pc_range[5]-pc_range[2], D) + point_sampling_trt in one launch (the
    encoder's call sequence, encoder.py:281-295), the pillar grid generated in registers."""
    if not lidar2img.is_cuda:
        raise RuntimeError("bev_point_sampling: lidar2img must be a CUDA tensor (no CPU fallback exists)")
    return _launch(None, pc_range, lidar2img, image_shape, int(bev_h), int(bev_w), int(num_points_in_pillar), dtype,
                   lidar2img.device)  # fmt: skip
