"""Synthetic NuScenes-shaped inputs for the attention-sampling path (host logic, CPU-generated, seeded).

Shapes follow SURVEY.md §8(a)/Appendix D (reference: configs/bevformer/bevformer_base.py:30-35,84-101,
configs/bevformer/bevformer_tiny.py:44-58 and det2trt/models/utils/test_trt_ops/test_multi_scale_deformable_attn.py:7-33).
Two input distributions for the MSDA op (SURVEY.md §8(d) config 3):

* ``"U"`` — the reference unit test's: value/offsets/logits ~ N(0,1), reference points ~ U[0,1)
  (test_multi_scale_deformable_attn.py:25-33). Every sampling point lands inside the image: worst case for the gather.
* ``"G"`` — geometry-realistic: reference points are the BEV pillar grid of ``get_reference_points_3d`` projected
  through a synthetic 6-camera ring with the formulas of ``point_sampling_trt``
  (det2trt/models/modules/encoder.py:170-259), so only about one camera in six sees a given BEV query; offsets ~ N(0, 2 px).

Everything is generated on the CPU with a seeded ``torch.Generator`` so vectors are reproducible anywhere.
"""
import math
from dataclasses import dataclass, field
from typing import List, Tuple

import torch


@dataclass(frozen=True)
class MSDAConfig:
    name: str
    batch: int  # cameras for SCA, bev-queue length for TSA, 1 for the decoder
    num_query: int
    num_heads: int
    channels: int  # per head
    spatial_shapes: Tuple[Tuple[int, int], ...]  # (h, w) per level
    num_points: int  # per level
    points_per_group: int  # Z anchors (4 in SCA, 1 in TSA / decoder)
    bev_hw: Tuple[int, int] = field(default=(0, 0))

    @property
    def num_levels(self):
        return len(self.spatial_shapes)

    @property
    def spatial_size(self):
        return sum(h * w for h, w in self.spatial_shapes)

    def algorithmic_bytes(self, elem_bytes: int, ref_bytes: int = None) -> int:
        """Each input read once, output written once (SURVEY.md §8(d)); no credit for gather re-reads."""
        ref_bytes = elem_bytes if ref_bytes is None else ref_bytes
        B, Q, M, C = self.batch, self.num_query, self.num_heads, self.channels
        NP = self.num_levels * self.num_points
        value = B * self.spatial_size * M * C * elem_bytes
        ref = B * Q * self.points_per_group * 2 * ref_bytes
        off = B * Q * M * NP * 2 * elem_bytes
        logit = B * Q * M * NP * elem_bytes
        out = B * Q * M * C * elem_bytes
        return value + ref + off + logit + out + self.num_levels * 2 * 4


BASE_LEVELS = ((116, 200), (58, 100), (29, 50), (15, 25))

CONFIGS = {
    # BASELINE.json configs[0]: the reference's own CPU-runnable plumbing case
    "cpu_plumbing": MSDAConfig("cpu_plumbing", 1, 100, 8, 32, ((64, 64),), 4, 1),
    # configs[1]: BEVFormer-tiny SCA op shapes (50x50 BEV, 6 cams, 1 level 15x25, 8 points)
    "tiny_sca": MSDAConfig("tiny_sca", 6, 2500, 8, 32, ((15, 25),), 8, 4, (50, 50)),
    # configs[2]: BEVFormer-base SCA op shapes — the headline (200x200 BEV, 6 cams, 4 levels, 4x8 points)
    "base_sca": MSDAConfig("base_sca", 6, 40000, 8, 32, BASE_LEVELS, 8, 4, (200, 200)),
    # the other MSDA call sites of BEVFormer-base (SURVEY §8(f) rank 2)
    "base_tsa": MSDAConfig("base_tsa", 2, 40000, 8, 32, ((200, 200),), 4, 1, (200, 200)),
    "base_decoder": MSDAConfig("base_decoder", 1, 900, 8, 32, ((200, 200),), 4, 1, (200, 200)),
    # small multi-level case for oracle-speed parity tests
    "small_sca": MSDAConfig("small_sca", 2, 333, 8, 32, ((12, 20), (6, 10), (3, 5), (2, 3)), 8, 4, (0, 0)),
}


def camera_ring_lidar2img(num_cams=6, img_hw=(928, 1600), focal=1260.0, radius=1.0, cam_height=1.5):
    """A synthetic NuScenes-like rig: ``num_cams`` pinhole cameras looking outward at 360/num_cams degree yaw spacing.
    Returns lidar2img [num_cams,4,4] (float64 -> float32) such that  (u*d, v*d, d, 1) = lidar2img @ (x, y, z, 1)."""
    H, W = img_hw
    K = torch.tensor([[focal, 0, W / 2, 0], [0, focal, H / 2, 0], [0, 0, 1, 0], [0, 0, 0, 1]], dtype=torch.float64)
    mats = []
    for i in range(num_cams):
        yaw = 2 * math.pi * i / num_cams
        fwd = torch.tensor([math.cos(yaw), math.sin(yaw), 0.0], dtype=torch.float64)
        up = torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64)
        right = torch.linalg.cross(fwd, up)  # camera x axis (image right)
        down = -up  # camera y axis (image down)
        R = torch.stack([right, down, fwd])  # world -> camera rotation
        c = radius * fwd + torch.tensor([0.0, 0.0, cam_height], dtype=torch.float64)
        E = torch.eye(4, dtype=torch.float64)
        E[:3, :3] = R
        E[:3, 3] = -R @ c
        mats.append(K @ E)
    return torch.stack(mats).float()


def bev_reference_points_cam(bev_hw, lidar2img, img_hw=(928, 1600), Z=8.0, pillars=4,
                             pc_range=(-51.2, -51.2, -5.0, 51.2, 51.2, 3.0)):  # fmt: skip
    """encoder.py:170-259 restated: pillar grid -> per-camera normalised image coordinates + visibility weights.
    Returns (reference_points_cam [cams, nq, pillars, 2], bev_mask [cams, nq, 1])."""
    H, W = bev_hw
    dev = lidar2img.device
    zs = (torch.linspace(0.5, Z - 0.5, pillars, device=dev) / Z).view(pillars, 1, 1).expand(pillars, H, W)
    xs = (torch.linspace(0.5, W - 0.5, W, device=dev) / W).view(1, 1, W).expand(pillars, H, W)
    ys = (torch.linspace(0.5, H - 0.5, H, device=dev) / H).view(1, H, 1).expand(pillars, H, W)
    ref3d = torch.stack((xs, ys, zs), -1).reshape(pillars, H * W, 3)
    lo = torch.tensor(pc_range[:3], device=dev)
    ext = torch.tensor(pc_range[3:], device=dev) - lo
    pts = torch.cat((ref3d * ext + lo, torch.ones(pillars, H * W, 1, device=dev)), -1)  # [pillars, nq, 4]
    cam = torch.einsum("cij,pqj->cqpi", lidar2img, pts)  # [cams, nq, pillars, 4]
    eps = 1e-5
    depth = cam[..., 2:3]
    vis = (depth > eps).float()
    uv = cam[..., 0:2] / torch.clamp(depth, min=eps)
    uv = uv / torch.tensor([img_hw[1], img_hw[0]], dtype=uv.dtype, device=dev)
    vis = vis * ((uv[..., 0:1] > 0) & (uv[..., 0:1] < 1) & (uv[..., 1:2] > 0) & (uv[..., 1:2] < 1)).float()
    seen = 1 - (1 - vis).prod(2)  # [cams, nq, 1]: any pillar visible
    bev_mask = seen / torch.clamp(seen.sum(0, keepdim=True), min=1e-4)
    return uv, bev_mask


def make_msda_inputs(cfg: MSDAConfig, dist: str = "U", seed: int = 0, dtype=torch.float32):
    """Returns CPU tensors (value[B,S,M,C], spatial_shapes int32[L,2], reference_points[B,Q,1,2G],
    sampling_offsets[B,Q,M,L*P*2], attention logits[B,Q,M,L*P]) in ``dtype`` (float32 or float16)."""
    g = torch.Generator().manual_seed(seed)
    B, Q, M, C = cfg.batch, cfg.num_query, cfg.num_heads, cfg.channels
    L, P, G = cfg.num_levels, cfg.num_points, cfg.points_per_group
    value = torch.randn(B, cfg.spatial_size, M, C, generator=g)
    logits = torch.randn(B, Q, M, L * P, generator=g)
    if dist == "U":
        ref = torch.rand(B, Q, 1, 2 * G, generator=g)
        off = torch.randn(B, Q, M, L * P * 2, generator=g)
    elif dist == "G":
        assert cfg.bev_hw[0] * cfg.bev_hw[1] == Q and G == 4, "distribution G needs an SCA-shaped config"
        uv, _ = bev_reference_points_cam(cfg.bev_hw, camera_ring_lidar2img(B), pillars=G)
        ref = uv.reshape(B, Q, 1, 2 * G).clone()
        # keep fp16 finite: points behind the camera divide by eps and overflow; any value far outside [0,1] is
        # equivalent for the op (every sample is out of range), so clamp like a calibrated fp16 engine would.
        ref = ref.clamp(-60000.0, 60000.0)
        off = 2.0 * torch.randn(B, Q, M, L * P * 2, generator=g)
    elif dist == "edge":
        # stress the range gate and the per-tap validity rules: refs on/over the borders, large offsets
        ref = torch.rand(B, Q, 1, 2 * G, generator=g) * 1.4 - 0.2
        snap = torch.rand(B, Q, 1, 2 * G, generator=g)
        ref = torch.where(snap < 0.15, torch.zeros_like(ref), ref)
        ref = torch.where(snap > 0.85, torch.ones_like(ref), ref)
        off = torch.randn(B, Q, M, L * P * 2, generator=g) * 3.0
        half = torch.rand(B, Q, M, L * P * 2, generator=g) < 0.3
        off = torch.where(half, torch.round(off) + 0.5, off)  # lands exactly on pixel centres / edges
    else:
        raise ValueError(dist)
    shapes = torch.tensor(cfg.spatial_shapes, dtype=torch.int32)
    return value.to(dtype), shapes, ref.to(dtype), off.to(dtype), logits.to(dtype)


def quantize_per_tensor(x: torch.Tensor):
    """MinMax PTQ convention of the reference's op tests (det2trt/models/utils/test_trt_ops/utils.py:18-50):
    scale = amax/127, q = clamp(round(x/scale), -128, 127), real = q*scale."""
    scale = float(x.abs().max()) / 127.0
    scale = scale if scale > 0 else 1.0
    q = torch.clamp(torch.round(x.float() / scale), -128, 127).to(torch.int8)
    return q, scale


@dataclass(frozen=True)
class BevPoolConfig:
    """One BEVPoolV2 call site: cameras, image size and feature stride, depth bins, channels and the BEV grid."""

    name: str
    cams: int
    image_hw: Tuple[int, int]
    stride: int
    depth_bins: Tuple[float, float, float]  # (start, stop, step): the frustum's depths, as grid_config["depth"]
    channels: int
    grid_lower: Tuple[float, float, float]
    grid_interval: Tuple[float, float, float]
    grid_size: Tuple[int, int, int]  # (x, y, z) cells

    @property
    def feat_hw(self):
        return self.image_hw[0] // self.stride, self.image_hw[1] // self.stride

    @property
    def num_depth(self):
        start, stop, step = self.depth_bins
        return int(round((stop - start) / step))

    @property
    def out_hw(self):  # (out_height, out_width) = (y cells, x cells): ranks_bev = y * size_x + x
        return self.grid_size[1], self.grid_size[0]


BEV_POOL_CONFIGS = {
    # BEVDet-R50 (configs/bevdet/bevdet-r50-cbgs.py): 256x704 input / 16 -> 16x44 features, depth 1..60 m (59 bins),
    # numC_Trans = 64, a 128x128 grid of 0.8 m cells over +-51.2 m with one z bin over [-5, 3)
    "bevdet_r50": BevPoolConfig("bevdet_r50", 6, (256, 704), 16, (1.0, 60.0, 1.0), 64, (-51.2, -51.2, -5.0),
                                (0.8, 0.8, 8.0), (128, 128, 1)),  # fmt: skip
    # the reference's own op test (det2trt/models/utils/test_trt_ops/test_bev_pool_v2.py): depth [6, 160, 32, 88],
    # feat [6, 32, 88, 128], a 200x200 grid of 1 m cells over +-100 m
    "ref_test": BevPoolConfig("ref_test", 6, (512, 1408), 16, (1.0, 161.0, 1.0), 128, (-100.0, -100.0, -5.0),
                              (1.0, 1.0, 8.0), (200, 200, 1)),  # fmt: skip
    # a small non-square case that golden fixtures store in full
    "tiny": BevPoolConfig("tiny", 2, (128, 352), 16, (1.0, 17.0, 1.0), 16, (-12.0, -16.0, -5.0), (1.0, 1.0, 8.0),
                          (32, 24, 1)),  # fmt: skip
}


def bev_pool_ranks(cfg: BevPoolConfig):
    """The LSS rank preparation (BEVDet's voxel_pooling_prepare_v2) for a synthetic camera ring, in float64 on the CPU:
    the frustum (u, v, d) of every feature pixel and depth bin is lifted to the ego frame through the inverse of
    ``camera_ring_lidar2img``, truncated to voxel coordinates, kept inside the grid, sorted by BEV cell, and cut into one
    interval per cell. Returns int32 (ranks_depth, ranks_feat, ranks_bev, interval_starts, interval_lengths)."""
    N, (fh, fw), D = cfg.cams, cfg.feat_hw, cfg.num_depth
    H_in, W_in = cfg.image_hw
    start, _, step = cfg.depth_bins
    d = (start + step * torch.arange(D, dtype=torch.float64)).view(D, 1, 1).expand(D, fh, fw)
    u = torch.linspace(0, W_in - 1, fw, dtype=torch.float64).view(1, 1, fw).expand(D, fh, fw)
    v = torch.linspace(0, H_in - 1, fh, dtype=torch.float64).view(1, fh, 1).expand(D, fh, fw)
    img = torch.stack((u * d, v * d, d, torch.ones_like(d)), -1)  # [D, fh, fw, 4]
    l2i = camera_ring_lidar2img(N, img_hw=cfg.image_hw, focal=1260.0 * W_in / 1600.0).double()
    ego = torch.einsum("nij,dhwj->ndhwi", torch.linalg.inv(l2i), img)[..., :3]  # [N, D, fh, fw, 3]
    coor = ((ego - torch.tensor(cfg.grid_lower, dtype=torch.float64)) /
            torch.tensor(cfg.grid_interval, dtype=torch.float64)).long().reshape(-1, 3)  # fmt: skip
    P_all = N * D * fh * fw
    ranks_depth = torch.arange(P_all, dtype=torch.int64)
    ranks_feat = torch.arange(N * fh * fw, dtype=torch.int64).view(N, 1, fh, fw).expand(N, D, fh, fw).reshape(-1)
    sx, sy, sz = cfg.grid_size
    kept = ((coor[:, 0] >= 0) & (coor[:, 0] < sx) & (coor[:, 1] >= 0) & (coor[:, 1] < sy) & (coor[:, 2] >= 0) &
            (coor[:, 2] < sz))  # fmt: skip
    coor, ranks_depth, ranks_feat = coor[kept], ranks_depth[kept], ranks_feat[kept]
    ranks_bev = coor[:, 2] * sx * sy + coor[:, 1] * sx + coor[:, 0]
    order = torch.sort(ranks_bev, stable=True).indices
    ranks_bev, ranks_depth, ranks_feat = ranks_bev[order], ranks_depth[order], ranks_feat[order]
    first = torch.ones(ranks_bev.numel(), dtype=torch.bool)
    first[1:] = ranks_bev[1:] != ranks_bev[:-1]
    starts = torch.nonzero(first).flatten()
    lengths = torch.diff(starts, append=torch.tensor([ranks_bev.numel()]))
    return tuple(t.to(torch.int32).contiguous() for t in (ranks_depth, ranks_feat, ranks_bev, starts, lengths))


def make_bev_pool_inputs(name: str, seed: int = 0, dtype=torch.float32):
    """Returns CPU tensors (depth [N, D, fh, fw], feat [N, fh, fw, C], ranks) and (out_height, out_width) for the
    BEVPoolV2 workload ``name``. depth is a softmax over the depth bins of N(0, 2) logits (what the depth net emits),
    feat ~ N(0, 1); ranks (bev_pool_ranks) do not depend on the seed."""
    cfg = BEV_POOL_CONFIGS[name]
    g = torch.Generator().manual_seed(seed)
    N, (fh, fw), D, C = cfg.cams, cfg.feat_hw, cfg.num_depth, cfg.channels
    depth = torch.softmax(2.0 * torch.randn(N, D, fh, fw, generator=g), dim=1)
    feat = torch.randn(N, fh, fw, C, generator=g)
    return depth.to(dtype), feat.to(dtype), bev_pool_ranks(cfg), cfg.out_hw


def bev_pool_stats(ranks):
    """Points kept, intervals and the longest interval of a rank set."""
    lengths = ranks[4]
    return {"points": int(ranks[0].numel()), "intervals": int(lengths.numel()),
            "max_interval": int(lengths.max()) if lengths.numel() else 0}  # fmt: skip
