"""Multi-GPU plumbing of the data-parallel path (SURVEY.md §8e): one process per GPU, scenes are the
independent units, no collective on the data path.  Collectives (NCCL over NVLink on the box, gloo in the
CPU tests): one flat gradient all-reduce per optimiser step (the reference's DDP, scripts/train.py:213-216)
and the packed SyncBatchNorm statistics (unet3d_sparse_v2.py:172-175 + Trainer(sync_batchnorm=True))."""
from __future__ import annotations

from typing import Iterable, List, Optional, Sequence

import torch
import torch.distributed as dist


def scene_seeds(rank: int, world: int, n: int) -> List[int]:
    """Disjoint synthetic-scene seeds per rank (weak scaling: every rank gets n scenes)."""
    return [1000 * rank + i for i in range(n)]


def allreduce_gradients(params: Sequence[torch.nn.Parameter], group=None, bucket: Optional[torch.Tensor] = None):
    """Average gradients over the group with ONE flat all-reduce (parameters without a gradient contribute
    zeros = DDP's find_unused_parameters=True).  Returns the flat bucket so it can be reused next step."""
    world = dist.get_world_size(group)
    if world == 1:
        return bucket
    total = sum(p.numel() for p in params)
    ref = next(p for p in params)
    if bucket is None or bucket.numel() != total or bucket.device != ref.device:
        bucket = torch.empty(total, dtype=torch.float32, device=ref.device)
    off = 0
    for p in params:
        n = p.numel()
        if p.grad is None:
            bucket[off:off + n].zero_()
        else:
            bucket[off:off + n].copy_(p.grad.reshape(-1))
        off += n
    dist.all_reduce(bucket, group=group)
    bucket /= world
    off = 0
    for p in params:
        n = p.numel()
        g = bucket[off:off + n].view_as(p)
        if p.grad is None:
            p.grad = g.clone()
        else:
            p.grad.copy_(g)
        off += n
    return bucket


class GradReducer:
    """Bucketed gradient averaging overlapped with the backward pass — what the reference gets from DDP
    (scripts/train.py:213-216), without DDP's module wrapper.

    * every parameter's `.grad` is a VIEW into one flat fp32 buffer (laid out in reverse registration order ≈ the order
      in which the backward pass produces gradients), so a bucket is a contiguous slice and nothing is copied in or out
      (round 1 copied all 130 M gradients into a staging buffer and back around one 520 MB all-reduce after backward);
    * a post-accumulate hook per parameter counts its bucket down; a complete bucket is all-reduced immediately with
      async_op=True (NCCL runs it on its own stream, behind an event on the compute stream) while the backward pass
      continues; `finish()` launches the buckets that hold unused parameters (their slices are zero: DDP's
      find_unused_parameters=True) and waits for all of them;
    * averaging uses ReduceOp.AVG on NCCL (no extra pass), SUM + one scaling pass elsewhere (gloo in the CPU tests)."""

    def __init__(self, params: Sequence[torch.nn.Parameter], group=None, bucket_mb: float = 64.0):
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.params = [p for p in params if p.requires_grad][::-1]
        dev = self.params[0].device
        total = sum(p.numel() for p in self.params)
        self.flat = torch.zeros(total, dtype=torch.float32, device=dev)
        cap = max(1, int(bucket_mb * (1 << 20) / 4))
        self.buckets: List[List[int]] = []          # [start, end, n_params]
        self._bucket_of = {}
        off, start, count = 0, 0, 0
        for p in self.params:
            n = p.numel()
            p.grad = self.flat[off:off + n].view_as(p)
            self._bucket_of[id(p)] = len(self.buckets)
            off += n
            count += 1
            if off - start >= cap:
                self.buckets.append([start, off, count])
                start, count = off, 0
        if count:
            self.buckets.append([start, off, count])
        self._pending = [b[2] for b in self.buckets]
        self._launched = [False] * len(self.buckets)
        self._works = []
        self.sync = True            # False while accumulating micro-steps (--accum): hooks only count, nothing is reduced
        self._avg = dist.is_initialized() and dist.get_backend(group) == "nccl"
        self._handles = [p.register_post_accumulate_grad_hook(self._hook) for p in self.params] if self.world > 1 else []

    def zero_grad(self) -> None:
        """One memset of the flat buffer (the gradients stay views into it: never set them to None)."""
        self.flat.zero_()
        self.sync = True
        self._pending = [b[2] for b in self.buckets]
        self._launched = [False] * len(self.buckets)
        self._works = []

    def _launch(self, b: int) -> None:
        self._launched[b] = True
        s, e, _ = self.buckets[b]
        op = dist.ReduceOp.AVG if self._avg else dist.ReduceOp.SUM
        self._works.append(dist.all_reduce(self.flat[s:e], op=op, group=self.group, async_op=True))

    def rearm(self, sync: bool) -> None:
        """Before the backward pass of a further micro-step of the same optimiser step (gradients keep accumulating
        in the flat buffer); sync=True on the last one: its hooks launch the bucket all-reduces."""
        self.sync = sync
        self._pending = [b[2] for b in self.buckets]

    def _hook(self, p) -> None:
        if not self.sync:
            return
        b = self._bucket_of[id(p)]
        self._pending[b] -= 1
        if self._pending[b] == 0 and not self._launched[b]:
            self._launch(b)

    def finish(self) -> None:
        """After loss.backward(): reduce what is left, wait, and (non-NCCL) scale to the mean."""
        if self.world == 1:
            return
        for b in range(len(self.buckets)):
            if not self._launched[b]:
                self._launch(b)
        for w in self._works:
            w.wait()
        self._works = []
        if not self._avg:
            self.flat /= self.world

    def detach(self) -> None:
        for h in self._handles:
            h.remove()
        self._handles = []


def all_gather_rows(t: torch.Tensor, group=None) -> List[torch.Tensor]:
    """All-gather of row sets with different row counts (the sparse logits of the MIMO subnets: [K1_i, 100] mask logits,
    [K1_i, 4] coordinates, ...): one small all-gather of the counts, one all-gather of the rows padded to the longest.
    Returns the per-rank tensors in rank order."""
    world = dist.get_world_size(group)
    n = torch.tensor([t.shape[0]], dtype=torch.int64, device=t.device)
    counts = [torch.zeros_like(n) for _ in range(world)]
    dist.all_gather(counts, n, group=group)
    counts = [int(c.item()) for c in counts]
    mx = max(counts)
    pad = torch.zeros((mx,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    pad[: t.shape[0]] = t
    out = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(out, pad, group=group)
    return [o[:c] for o, c in zip(out, counts)]


def sharded_mimo_forward(net, scene, group=None, test=True):
    """MIMO head sharding (BASELINE configs[3]): the M subnets of one MIMO group are spread one per rank.  Every rank runs
    the SHARED trunk (voxeliser → merge → encoder → dense bottleneck → decoder stages with all M completion heads: the
    trunk is one network, 4.4 of the ~5.2 TFLOP), rank r then runs only subnet r's panoptic heads (voxel_feats +
    mask transformer, 0.86 TFLOP each), and the sparse results are all-gathered over NCCL: mask logits [K1_r, 100],
    their coordinates [K1_r, 4], query logits [1, 100, K+1] and the pruned semantic logits.  Returns the same dict as
    PascoNet.forward with panop_predictions / sem_logits_pruneds of ALL subnets (as (features, coordinates) pairs), ready
    for pasco_b200.ensemble.  Amdahl: at most 1.3x over running the three heads on one GPU (SURVEY.md §8e)."""
    from . import me as ME
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    M = net.n_infers
    mine = [m for m in range(M) if m % world == rank]
    out = net(scene["in_feats"], scene["in_coords"], scene["global_min_Cs"], scene["global_max_Cs"], scene["min_Cs"],
              scene["max_Cs"], predict_panop=True, test=test, subnets=mine)
    preds = [None] * M
    pruned = [None] * M
    dev = scene["in_feats"][0].device
    for j in range((M + world - 1) // world):                 # round j: rank r contributes subnet j*world + r (or nothing)
        m = j * world + rank
        have = m < M
        p = out["panop_predictions"][j] if have else None
        Q = net.transformer_predictor.num_queries
        vl = p["voxel_logits"].F.detach() if have else torch.zeros(0, Q, device=dev)
        vc = p["voxel_logits"].C if have else torch.zeros(0, 4, dtype=torch.int32, device=dev)
        ql = p["query_logits"].detach() if have else torch.zeros(0, Q, 21, device=dev)
        sl = out["sem_logits_pruneds"][j] if have else None
        sf = sl.F.detach() if have else torch.zeros(0, net.n_classes, device=dev)
        sc = sl.C if have else torch.zeros(0, 4, dtype=torch.int32, device=dev)
        g_vl, g_vc, g_ql = all_gather_rows(vl, group), all_gather_rows(vc, group), all_gather_rows(ql, group)
        g_sf, g_sc = all_gather_rows(sf, group), all_gather_rows(sc, group)
        for r in range(world):
            mm = j * world + r
            if mm < M:
                preds[mm] = {"voxel_logits": (g_vl[r], g_vc[r]), "query_logits": g_ql[r]}
                pruned[mm] = (g_sf[r], g_sc[r])
    return {"sem_logits_at_scales": out["sem_logits_at_scales"], "panop_predictions": preds, "sem_logits_pruneds": pruned}


def sync_bn_statistics(stats: torch.Tensor, count: float, group=None):
    """Packed SyncBatchNorm reduction: stats float64 [2,C] (Σx, Σx²) and the local row count travel in one
    [2C+1] all-reduce; returns (global stats, global count)."""
    packed = torch.cat([stats.reshape(-1), torch.full((1,), float(count), dtype=stats.dtype, device=stats.device)])
    dist.all_reduce(packed, group=group)
    return packed[:-1].view_as(stats), float(packed[-1].item())


def enable_sync_batchnorm(model: torch.nn.Module, group=None) -> int:
    """Switch every MinkowskiBatchNorm of the model to MinkowskiSyncBatchNorm over `group` (None: the default group), in
    place and with the same parameters and buffers.  Returns the number of layers switched."""
    from .me import MinkowskiBatchNorm, MinkowskiSyncBatchNorm
    n = sum(type(m) is MinkowskiBatchNorm for m in model.modules())
    MinkowskiSyncBatchNorm.convert_sync_batchnorm(model, group)
    return n


def max_over_ranks(ms: float, device) -> float:
    t = torch.tensor([ms], dtype=torch.float64, device=device)
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())
