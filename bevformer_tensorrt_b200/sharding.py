"""Per-camera sharding of spatial cross-attention's sampling step across GPUs (SURVEY.md §8(e)).

The SCA output is a sum over cameras of per-camera MSDA outputs weighted by ``bev_mask[cam, q]``
(reference: det2trt/models/modules/spatial_cross_attention.py:254-270 — ``slots = (queries * bev_mask).sum(0)``), and
each camera's MSDA touches only that camera's value stack, so the work splits into independent (camera, query-tile)
units. Every rank runs the sm_90a MSDA kernel on its units, folds them into a local BEV accumulator ``[nq, heads*ch]``
and ONE collective (all-reduce, NCCL over NVLink on GPUs / gloo in the CPU tests) produces the summed accumulator.
6 cameras do not divide 4 or 8 ranks, hence query tiles: the unit count is lcm-friendly (12 units for 4 ranks,
24 for 8) so every rank gets the same amount of work.
"""
import ctypes
import math
from dataclasses import dataclass
from typing import Callable, List, Sequence

import torch


@dataclass(frozen=True)
class Unit:
    cam: int
    q0: int
    q1: int


def plan_units(num_cams: int, num_query: int, world_size: int, align: int = 8) -> List[List[Unit]]:
    """Round-robin assignment of (camera, query-tile) units: returns per-rank unit lists, equal counts per rank.
    Tiles per camera = world_size / gcd(num_cams, world_size); tile edges are multiples of ``align`` queries."""
    if world_size < 1 or num_cams < 1 or num_query < 1:
        raise ValueError("world_size, num_cams and num_query must be positive")
    tiles = world_size // math.gcd(num_cams, world_size)
    edges = [min(num_query, ((num_query * t // tiles + align - 1) // align) * align) for t in range(tiles)] + [num_query]
    units = [Unit(c, edges[t], edges[t + 1]) for c in range(num_cams) for t in range(tiles) if edges[t + 1] > edges[t]]
    per_rank: List[List[Unit]] = [[] for _ in range(world_size)]
    # camera-major order keeps one camera's tiles on as few ranks as possible: rank r takes a contiguous run
    n = len(units)
    for r in range(world_size):
        per_rank[r] = units[n * r // world_size : n * (r + 1) // world_size]
    return per_rank


def plan_chunked(num_cams: int, num_query: int, world_size: int, chunks: int, align: int = 8) -> List[List[List[Unit]]]:
    """Splits the query range into ``chunks`` pieces and plans each piece like ``plan_units``: result[chunk][rank] is
    that rank's unit list for that query chunk. Every rank has the same amount of work in every chunk, so the
    all-reduce of chunk k can overlap the kernels of chunk k+1 without stragglers."""
    chunks = max(1, min(chunks, num_query // align if num_query >= align else 1))
    edges = [min(num_query, ((num_query * c // chunks + align - 1) // align) * align) for c in range(chunks)] + [num_query]
    out = []
    for c in range(chunks):
        q0, q1 = edges[c], edges[c + 1]
        if q1 <= q0:
            continue
        per_rank = plan_units(num_cams, q1 - q0, world_size, align)
        out.append([[Unit(u.cam, u.q0 + q0, u.q1 + q0) for u in units] for units in per_rank])
    return out


def plan_chunk_bounds(plan) -> List[tuple]:
    """(q_lo, q_hi) of every chunk of a ``plan_chunked`` result, over all ranks."""
    return [(min(u.q0 for units in chunk for u in units), max(u.q1 for units in chunk for u in units)) for chunk in plan]


def merge_units(units: Sequence[Unit]) -> List[Unit]:
    """Coalesces adjacent query tiles of the same camera (fewer, larger kernel launches)."""
    out: List[Unit] = []
    for u in sorted(units, key=lambda x: (x.cam, x.q0)):
        if out and out[-1].cam == u.cam and out[-1].q1 == u.q0:
            out[-1] = Unit(u.cam, out[-1].q0, u.q1)
        else:
            out.append(u)
    return out


def group_cameras(units: Sequence[Unit]):
    """Batches consecutive cameras that cover the same query range into one launch: (cam0, cam1, q0, q1) tuples."""
    groups = []
    for u in merge_units(units):
        if groups and groups[-1][1] == u.cam and groups[-1][2:] == (u.q0, u.q1):
            groups[-1] = (groups[-1][0], u.cam + 1, u.q0, u.q1)
        else:
            groups.append((u.cam, u.cam + 1, u.q0, u.q1))
    return groups


class ShardedSCASampler:
    """Holds one rank's slice of the SCA sampling inputs and produces the all-reduced BEV accumulator.

    ``units`` is either one unit list (single collective at the end) or a list of per-chunk unit lists from
    ``plan_chunked`` (the all-reduce of query chunk k is issued asynchronously right after chunk k's kernels and runs
    on the communication stream while chunk k+1 computes). ``msda`` is the operator to run per launch group (the
    product passes ``multi_scale_deformable_attn``; the CPU tests pass a checker so the host-side plumbing — planning,
    slicing, masking, the collective — is covered without a GPU). ``fused_sca`` (optional,
    ``multi_scale_deformable_attn_sca``) folds MSDA + bev_mask camera-sum into one kernel writing the accumulator.
    """

    def __init__(self, units, num_query: int, msda: Callable, group=None, accum_dtype: torch.dtype = torch.float32,
                 fused_sca: Callable = None, chunk_bounds=None, wire_dtype: torch.dtype = None):  # fmt: skip
        chunked = len(units) > 0 and isinstance(units[0], (list, tuple))
        self.chunk_units = [merge_units(u) for u in units] if chunked else [merge_units(units)]
        self.num_query = num_query
        self.msda = msda
        self.group = group
        self.accum_dtype = accum_dtype
        self.fused_sca = fused_sca if accum_dtype == torch.float32 else None
        # dtype on the wire: every rank accumulates in accum_dtype (fp32); with wire_dtype=float16 the partial sums are
        # rounded once to fp16 for the collective (half the NVLink bytes) and the reduced result is widened back
        self.wire_dtype = wire_dtype if wire_dtype not in (None, accum_dtype) else None
        self._wire = None
        # the accumulator slice every rank reduces for chunk k — must be identical on all ranks (plan_chunk_bounds)
        self.chunk_bounds = list(chunk_bounds) if chunk_bounds is not None else None
        if chunked and self.chunk_bounds is None:
            raise ValueError("chunked unit lists need chunk_bounds (use plan_chunk_bounds on the full plan)")
        self.chunks = []  # per chunk: (q_lo, q_hi, [(cam0, cam1, q0, q1)], [(value, ref, off, logits, mask)])
        self.shapes = None
        self.accum = None
        self._graph = None

    def load(self, value, shapes, ref, off, logits, bev_mask, device):
        """Copies this rank's units out of full-size host tensors (a real model produces them in place)."""
        self.shapes = shapes.to(device)
        self.chunks = []
        cams = {}
        for units in self.chunk_units:
            groups = group_cameras(units)  # (cam0, cam1, q0, q1): consecutive cameras sharing a query range
            local = []
            for c0, c1, q0, q1 in groups:
                sl = slice(q0, q1)
                if (c0, c1) not in cams:  # one device copy of a camera's value stack, shared by its query tiles
                    cams[(c0, c1)] = value[c0:c1].to(device).contiguous()
                local.append((cams[(c0, c1)],) + tuple(
                    t.to(device).contiguous() for t in (ref[c0:c1, sl], off[c0:c1, sl], logits[c0:c1, sl],
                                                        bev_mask[c0:c1, sl])))  # fmt: skip
            lo, hi = self.chunk_bounds[len(self.chunks)] if self.chunk_bounds is not None else (0, self.num_query)
            self.chunks.append((lo, hi, groups, local))
        M, C = value.shape[2], value.shape[3]
        self.accum = torch.zeros(self.num_query, M * C, dtype=self.accum_dtype, device=device)
        if self.wire_dtype is not None:
            self._wire = torch.empty(self.num_query, M * C, dtype=self.wire_dtype, device=device)
        return self

    def _compute(self, groups, local):
        for (c0, c1, q0, q1), (v, r, o, w, mask) in zip(groups, local):
            if self.fused_sca is not None:
                self.fused_sca(v, self.shapes, r, o, w, mask, self.accum[q0:q1])
                continue
            out = self.msda(v, self.shapes, r, o, w)  # [cams, q, M, C]
            weighted = out.reshape(c1 - c0, q1 - q0, -1).to(self.accum_dtype) * mask.to(self.accum_dtype)
            self.accum[q0:q1] += weighted.sum(0)

    def capture(self, warmup: int = 3):
        """Captures one full step (accumulator memset, this rank's kernels, wire conversion, the NCCL all-reduce) into a
        CUDA graph; ``step()`` then replays it. The step is 0.2-0.7 ms of device work issued as five to ten small
        launches plus a collective, so the host launch path and the inter-stream hand-offs around the collective are
        a visible share of it; the replay removes them. Every rank must call this (it runs collectives)."""
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):
                self._step_eager(True)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            self._step_eager(True)
        self._graph = graph
        return self

    def step(self, reduce: bool = True):
        """One SCA sampling step on this rank: kernels for the local units, masked camera-sum, all-reduce (one
        collective, or one per query chunk overlapped with the next chunk's kernels). Replays the captured graph when
        ``capture()`` has been called."""
        if reduce and self._graph is not None:
            self._graph.replay()
            return self.accum
        return self._step_eager(reduce)

    def _step_eager(self, reduce: bool = True):
        import torch.distributed as dist

        do_reduce = reduce and dist.is_available() and dist.is_initialized() and dist.get_world_size(self.group) > 1
        self.accum.zero_()
        works = []
        for lo, hi, groups, local in self.chunks:
            self._compute(groups, local)
            if do_reduce and hi > lo:
                buf = self.accum[lo:hi]
                if self._wire is not None:
                    buf = self._wire[lo:hi]
                    buf.copy_(self.accum[lo:hi])
                works.append(dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=self.group,
                                             async_op=len(self.chunks) > 1))  # fmt: skip
        for w in works:
            if w is not None:
                w.wait()
        if do_reduce and self._wire is not None:
            self.accum.copy_(self._wire)
        return self.accum


# ---------------------------------------------------------------------------------------------------------------------
# Round 2: camera-group x query-tile grid with an owner-sliced reduce-scatter (the step's only inter-GPU traffic)
# ---------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class GridShard:
    """One rank's place in the (camera group, query tile) grid.

    ``world = A * T``: the cameras are split into ``A`` groups (A divides the camera count), the queries into ``T``
    tiles; rank ``r`` = (group ``r // T``, tile ``r % T``) samples cameras ``[cam0, cam1)`` for queries ``[q0, q1)``
    into a partial accumulator ``[q1 - q0, heads*ch]``. The ``A`` ranks that share a tile (``peers``, ordered by camera
    group) reduce-scatter their partials: this rank ends up owning the final sum of rows ``[own0, own1)`` (a slice of its
    tile). Every BEV query is owned by exactly one rank; the consumer (``output_proj``, spatial_cross_attention.py:273) is
    query-parallel, so no all-gather follows."""

    rank: int
    world: int
    groups: int  # A
    tiles: int  # T
    cam0: int
    cam1: int
    q0: int  # rows [q0, q1) of the TILED query order (see tiled_query_order); = BEV query ids when block == 0
    q1: int
    peers: tuple  # global ranks sharing this tile, index = camera group
    own0: int
    own1: int
    block: int = 0  # > 0: tile t holds the query blocks t, t+T, t+2T, ... of `block` consecutive BEV queries
    num_query: int = 0

    @property
    def my_index(self):
        return self.peers.index(self.rank)

    def tile_queries(self):
        """BEV query ids of this rank's tile rows, LongTensor [q1 - q0]."""
        return tiled_query_order(self.num_query, self.tiles, self.block)[self.q0 : self.q1]

    def own_queries(self):
        """BEV query ids of the rows this rank owns after the exchange, LongTensor [own1 - own0]."""
        return tiled_query_order(self.num_query, self.tiles, self.block)[self.own0 : self.own1]


def tiled_query_order(num_query: int, tiles: int, block: int):
    """Permutation of the BEV queries in which tile t is a CONTIGUOUS run: block == 0 -> identity (tile = a contiguous
    query range); block > 0 -> tile t = the blocks t, t+T, ... of `block` consecutive queries (interleaved). A camera
    sees a compact wedge of the BEV, so contiguous ranges give the ranks of one camera group very different numbers of
    visible (camera, query) pairs (measured max/mean 1.7 at 4 ranks, 2.0 at 8 on the camera ring); interleaved blocks
    balance them to within 0.2 %."""
    idx = torch.arange(num_query)
    if block <= 0 or tiles <= 1:
        return idx
    nb = (num_query + block - 1) // block
    pad = torch.full((nb * block,), -1, dtype=torch.long)
    pad[:num_query] = idx
    blocks = pad.view(nb, block)
    order = torch.cat([blocks[t::tiles].reshape(-1) for t in range(tiles)])
    return order[order >= 0]


def _tile_edges(num_query: int, tiles: int, block: int, align: int):
    if block <= 0 or tiles <= 1:
        return _edges(num_query, tiles, align)
    nb = (num_query + block - 1) // block
    sizes = []
    for t in range(tiles):
        n_blocks = len(range(t, nb, tiles))
        size = n_blocks * block
        if n_blocks and (nb - 1) % tiles == t:  # the (possibly short) last block lives in this tile
            size -= nb * block - num_query
        sizes.append(size)
    edges = [0]
    for sz in sizes:
        edges.append(edges[-1] + sz)
    return edges


def _edges(n: int, parts: int, align: int, lo: int = 0):
    return [lo + min(n, ((n * t // parts + align - 1) // align) * align) for t in range(parts)] + [lo + n]


def choose_camera_groups(num_cams: int, world: int) -> int:
    """Smallest A > 1 dividing both the camera count and the world size (least inter-GPU traffic: a rank sends
    (A-1)/A of its tile), A = 1 (pure query split, no exchange at all) when world == 1 or nothing divides."""
    for a in range(2, num_cams + 1):
        if num_cams % a == 0 and world % a == 0:
            return a
    return 1


def plan_grid(num_cams: int, num_query: int, world: int, align: int = 8, groups: int = None,
              block: int = 8) -> List[GridShard]:
    """``block``: query-tile interleave granularity (see tiled_query_order); 0 = contiguous query ranges."""
    if world < 1 or num_cams < 1 or num_query < 1:
        raise ValueError("world_size, num_cams and num_query must be positive")
    A = choose_camera_groups(num_cams, world) if groups is None else groups
    if num_cams % A or world % A:
        raise ValueError(f"{A} camera groups do not divide {num_cams} cameras / {world} ranks")
    T = world // A
    if T <= 1:
        block = 0
    qe = _tile_edges(num_query, T, block, align)
    per = num_cams // A
    shards = []
    for r in range(world):
        g, t = divmod(r, T)
        q0, q1 = qe[t], qe[t + 1]
        oe = _edges(q1 - q0, A, align if align % 4 == 0 else 4, q0)
        shards.append(GridShard(r, world, A, T, g * per, (g + 1) * per, q0, q1, tuple(gg * T + t for gg in range(A)),
                                oe[g], oe[g + 1], block, num_query))
    return shards


class GroupedSCASampler:
    """One rank of the camera-group x query-tile grid: local fused sampling into a partial accumulator, then the
    reduce-scatter inside the camera group. ``step()`` returns this rank's OWNED rows ``[own1 - own0, heads*ch]``.

    exchange = "peer"  : ``b200_sca_peer_reduce`` — our kernel pulls the peers' partials over NVLink peer memory (torch
                         symmetric memory supplies the mapped pointers); no NCCL call in the step.
             = "nccl"  : ``reduce_scatter_tensor`` on the camera group's communicator (all-reduce + slice on gloo, which
                         has no reduce-scatter) — the library baseline and the CPU-test path.
    ``fused_sca(value, shapes, ref, off, logits, mask, accum)`` is the product kernel; the CPU tests inject a checker."""

    def __init__(self, shard: GridShard, width: int, fused_sca: Callable, exchange: str = "nccl", out_dtype=torch.float32,
                 overlap: bool = False):
        self.shard, self.width, self.fused_sca, self.exchange = shard, width, fused_sca, exchange
        # overlap: sample the peers' rows first and pull their results while sampling the own rows (two sampling launches,
        # pull on a side stream, a separate add pass). The extra pass over the accumulator and the second launch can cost
        # more than the NVLink traffic they hide, so it is opt-in.
        self.overlap = overlap and exchange == "peer"
        self.out_dtype = out_dtype
        self.rows = shard.q1 - shard.q0
        self.local = None
        self.partial = None  # [2][rows_max, width] fp32 (peer) or [rows, width] (nccl)
        self.out = None
        self.group = None
        self.epoch = 0
        self._peer = None

    # -- setup ---------------------------------------------------------------------------------------------------
    def load(self, value, shapes, ref, off, logits, bev_mask, device):
        s = self.shard
        cs = slice(s.cam0, s.cam1)
        if s.block > 0:  # interleaved tile: gather its query blocks once (upstream layers produce them in place)
            qi = s.tile_queries()
            take = lambda t: t[cs].index_select(1, qi)  # noqa: E731
        else:
            take = lambda t: t[cs, s.q0 : s.q1]  # noqa: E731
        self.shapes = shapes.to(device)
        # bev_mask as the fused kernel reads it (fp32 [cams, rows]): no per-step conversion launch
        mask32 = take(bev_mask).reshape(s.cam1 - s.cam0, -1).to(torch.float32)
        full = (take(ref), take(off), take(logits), mask32)
        val = value[cs].to(device).contiguous()
        # Row parts of the tile for the overlapped step: the rows the PEERS own are sampled first (so that the peers can pull
        # them while this rank samples its own rows). Only when those rows are one contiguous range (always for 2 groups).
        lo, hi, rows = s.own0 - s.q0, s.own1 - s.q0, s.q1 - s.q0
        self.parts = None
        if s.groups > 1 and self.overlap and (lo == 0 or hi == rows) and 0 < hi - lo < rows:
            others = (hi, rows) if lo == 0 else (0, lo)
            self.parts = []
            for r0, r1 in (others, (lo, hi)):
                self.parts.append((r0, r1, tuple(t[:, r0:r1].to(device).contiguous() for t in full)))
            self.local = (val,) + self.parts[0][2] + self.parts[1][2]
        else:
            self.local = (val,) + tuple(t.to(device).contiguous() for t in full)
        self.out = torch.empty(s.own1 - s.own0, self.width, dtype=self.out_dtype, device=device)
        return self

    def connect(self, all_shards: Sequence[GridShard], device):
        """Collective: every rank calls it with the full plan. Builds the camera-group communicators ("nccl") or the
        symmetric-memory window ("peer")."""
        import torch.distributed as dist

        s = self.shard
        if s.groups == 1 or not (dist.is_available() and dist.is_initialized()):
            self.exchange = "none"
            self.partial = torch.zeros(self.rows, self.width, dtype=torch.float32, device=device)
            return self
        if self.exchange == "peer":
            import torch.distributed._symmetric_memory as symm_mem

            rows_max = max(x.q1 - x.q0 for x in all_shards)
            n = 2 * rows_max * self.width + 64  # two partial buffers + the flag row (uint32[10] viewed as float bits)
            buf = symm_mem.empty(n, dtype=torch.float32, device=device)
            buf.zero_()
            hdl = symm_mem.rendezvous(buf, dist.group.WORLD)
            torch.cuda.synchronize(device)
            dist.barrier()
            self._attach_peer_window(buf, [int(hdl.buffer_ptrs[r]) for r in s.peers], rows_max)
            self._peer["hdl"] = hdl
        else:
            tiles = sorted({x.peers for x in all_shards})
            for peers in tiles:  # every rank creates every group, in the same order
                g = dist.new_group(list(peers))
                if peers == s.peers:
                    self.group = g
            self.partial = torch.zeros(self.rows, self.width, dtype=torch.float32, device=device)
        return self

    def _attach_peer_window(self, buf, base_ptrs, rows_max):
        """Lays out the peer exchange over one window per rank of ``2 * rows_max * width + 64`` floats: the partial of
        even steps, the partial of odd steps, then the flag row. ``buf`` is this rank's window (zeroed),
        ``base_ptrs[i]`` the device address of the window of ``shard.peers[i]`` as this rank maps it."""
        stride = rows_max * self.width * 4
        self._peer = {"buf": buf, "rows_max": rows_max,
                      "part": [[b + k * stride for b in base_ptrs] for k in (0, 1)],
                      "flags": [b + 2 * stride for b in base_ptrs]}
        self.partial = [buf[k * rows_max * self.width:(k + 1) * rows_max * self.width][: self.rows * self.width]
                        .view(self.rows, self.width) for k in (0, 1)]  # fmt: skip

    # -- one step ------------------------------------------------------------------------------------------------
    def compute(self, accum):
        if self.parts is None:
            v, r, o, w, m = self.local
            self.fused_sca(v, self.shapes, r, o, w, m, accum)
        else:
            for i in (0, 1):
                self._compute_part(i, accum)

    def _compute_part(self, i, accum):
        r0, r1, (r, o, w, m) = self.parts[i]
        self.fused_sca(self.local[0], self.shapes, r, o, w, m, accum[r0:r1])

    def step(self):
        s = self.shard
        if self.exchange == "peer":
            return self._step_peer()
        self.partial.zero_()
        self.compute(self.partial)
        lo, hi = s.own0 - s.q0, s.own1 - s.q0
        if self.exchange == "none":
            self.out.copy_(self.partial[lo:hi])
            return self.out
        import torch.distributed as dist

        equal = (s.own1 - s.own0) * s.groups == self.rows  # reduce_scatter_tensor needs equal slices
        if dist.get_backend(self.group) == "nccl" and equal and self.out_dtype == torch.float32:
            dist.reduce_scatter_tensor(self.out, self.partial, op=dist.ReduceOp.SUM, group=self.group)
        else:
            dist.all_reduce(self.partial, op=dist.ReduceOp.SUM, group=self.group)
            self.out.copy_(self.partial[lo:hi])
        return self.out

    def exchange_only(self):
        """The exchange without the sampling launch (bench.py's breakdown). Collective: every rank calls it equally often."""
        s = self.shard
        if self.exchange == "peer":
            return self._step_peer(compute=False)
        if self.exchange == "none":
            return self.out
        import torch.distributed as dist

        if dist.get_backend(self.group) == "nccl" and (s.own1 - s.own0) * s.groups == self.rows and \
                self.out_dtype == torch.float32:
            dist.reduce_scatter_tensor(self.out, self.partial, op=dist.ReduceOp.SUM, group=self.group)
        else:
            dist.all_reduce(self.partial, op=dist.ReduceOp.SUM, group=self.group)
        return self.out

    def _step_peer(self, compute=True):
        from . import _lib

        s, p = self.shard, self._peer
        if compute and self.parts is not None and self.exchange == "peer":
            return self._step_overlapped()
        k = self.epoch & 1  # the device counts the steps itself (flag row slot 8): same parity by construction
        self.epoch += 1
        if compute:
            self.compute(self.partial[k])
        if "args" not in p:
            n = len(s.peers)
            p["args"] = ((ctypes.c_void_p * n)(*p["part"][0]), (ctypes.c_void_p * n)(*p["part"][1]),
                         (ctypes.c_void_p * n)(*p["flags"]), n, s.my_index, (s.own0 - s.q0) * self.width,
                         (s.own1 - s.own0) * self.width, self.out.data_ptr(), int(self.out_dtype == torch.float16),
                         self.rows * self.width)  # fmt: skip
        _lib.call("b200_sca_peer_reduce_auto", self.out.device, *p["args"])
        return self.out

    def _step_overlapped(self):
        """Launch 1: the rows the peers own -> side stream: publish + pull the peers' launch-1 rows of MY slice into a staging
        buffer (NVLink traffic under launch 2) -> launch 2: my own rows -> out = own partial + staging."""
        from . import _lib

        s, p = self.shard, self._peer
        lib = _lib.load()
        k = self.epoch & 1
        self.epoch += 1
        dev = self.out.device
        if "ov" not in p:
            n = len(s.peers)
            loc = [p["part"][kk][s.my_index] for kk in (0, 1)]
            p["ov"] = {
                "side": torch.cuda.Stream(device=dev, priority=-1), "e1": torch.cuda.Event(), "e2": torch.cuda.Event(),
                "staging": torch.empty((s.own1 - s.own0) * self.width, dtype=torch.float32, device=dev),
                "pull": ((ctypes.c_void_p * n)(*p["part"][0]), (ctypes.c_void_p * n)(*p["part"][1]),
                         (ctypes.c_void_p * n)(*p["flags"]), n, s.my_index, (s.own0 - s.q0) * self.width,
                         (s.own1 - s.own0) * self.width),
                "add": (loc[0], loc[1], p["flags"][s.my_index], s.my_index, (s.own0 - s.q0) * self.width,
                        (s.own1 - s.own0) * self.width),
            }
        ov = p["ov"]
        main = torch.cuda.current_stream(dev)
        with torch.cuda.device(dev):
            self._compute_part(0, self.partial[k])
            ov["e1"].record(main)
            ov["side"].wait_event(ov["e1"])
            st = lib.b200_sca_peer_pull_auto(*ov["pull"], ov["staging"].data_ptr(), ctypes.c_void_p(ov["side"].cuda_stream))
            _lib.check("b200_sca_peer_pull_auto", st)
            ov["e2"].record(ov["side"])
            self._compute_part(1, self.partial[k])
            main.wait_event(ov["e2"])
            st = lib.b200_sca_peer_add_auto(*ov["add"], ov["staging"].data_ptr(), self.out.data_ptr(),
                                            int(self.out_dtype == torch.float16), self.rows * self.width,
                                            ctypes.c_void_p(main.cuda_stream))
            _lib.check("b200_sca_peer_add_auto", st)
        return self.out

    # -- CUDA graph of the step (peer exchange only: no library collective inside) -----------------------------------
    def capture_pair(self):
        """Captures TWO consecutive steps (the partial buffers alternate with the step parity; the exchange kernel keeps
        the step number on the device, so its launch parameters never change) into one CUDA graph. ``step_pair()``
        replays it: two full steps per call, the host launch path reduced to one graph launch."""
        if self.exchange != "peer":
            raise RuntimeError("capture_pair needs the peer-memory exchange")
        if self.epoch & 1:
            self.step()  # align to an even step count: the captured pair is (even buffer, odd buffer)
        torch.cuda.synchronize(self.out.device)
        g = torch.cuda.CUDAGraph()
        e0 = self.epoch
        with torch.cuda.graph(g):
            self._step_peer()
            self._step_peer()
        self.epoch = e0  # capture does not execute
        self._graph = g
        return self

    def step_pair(self):
        if self.epoch & 1:  # the captured pair starts on the even buffer: realign after an odd number of eager steps
            self._step_peer()
        self._graph.replay()
        self.epoch += 2
        return self.out
