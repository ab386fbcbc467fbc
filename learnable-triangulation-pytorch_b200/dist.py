"""View-sharded multi-GPU execution of the volumetric path (one process per GPU, torch.distributed plumbing).

The reference has no view sharding (its only parallelism is batch DDP, train.py:452-453).  Views are independent
until the aggregation inside the unprojection (op.py:150-162), so rank r of a G-rank *view group* owns views
{v : v mod G == r} of every sample of the group's batch, runs the backbone + unprojection on them and produces a
partial voxel aggregate; ONE collective over NVLink completes it; the V2V + soft-argmax then run batch-sharded.

softmax aggregation is not a plain sum:  out = sum_v s_v e^{s_v} / sum_v e^{s_v}.  Each rank therefore emits the
packed pair (numerator, denominator) [B][2][nvox][C] (lt_unproject_partial_fwd) and the collective is a SUM:
  collective="all_reduce"      one NCCL all-reduce of the packed buffer (the contract of BASELINE.json north_star)
  collective="reduce_scatter"  same bytes in, but each rank receives only the samples it will run V2V on
then lt_unproject_finalize_fwd divides and converts to the conv operand format.

With W ranks and V views: view-group size G = gcd-compatible min(W, V); the W/G groups are plain data-parallel
replicas over different samples (no communication between groups).
"""
import math
from dataclasses import dataclass

import torch


@dataclass
class ShardPlan:
    world: int
    rank: int
    n_views: int
    group_size: int      # G: ranks that share one batch and split its views
    n_groups: int        # data-parallel replicas
    group_index: int
    view_rank: int       # rank inside the view group

    @property
    def views(self):
        """View indices this rank owns."""
        return list(range(self.view_rank, self.n_views, self.group_size))

    def owned_samples(self, batch):
        """Samples (indices into the group's batch) this rank runs V2V / soft-argmax on: a contiguous block."""
        assert batch % self.group_size == 0, "group batch must be divisible by the view-group size"
        per = batch // self.group_size
        return list(range(self.view_rank * per, (self.view_rank + 1) * per))

    @property
    def group_ranks(self):
        return list(range(self.group_index * self.group_size, (self.group_index + 1) * self.group_size))


def make_plan(world, rank, n_views):
    g = math.gcd(world, n_views)     # largest group size that divides both the world and the view count
    return ShardPlan(world, rank, n_views, g, world // g, rank // g, rank % g)


def new_view_groups(plan):
    """Create every view group (collective call: all ranks must call it) and return this rank's group."""
    import torch.distributed as dist
    mine = None
    for gi in range(plan.n_groups):
        ranks = list(range(gi * plan.group_size, (gi + 1) * plan.group_size))
        pg = dist.new_group(ranks)
        if gi == plan.group_index:
            mine = pg
    return mine


def complete_partials(partial, plan, pg, collective="all_reduce", reduce_op="sum", out=None, max_bytes=1 << 29):
    """partial: [B][P][nvox][C] float32 on every rank of the group -> the block of fully reduced samples this rank owns.

    Returns a tensor [B/G][P][nvox][C].  `reduce_op` is "sum" (softmax num/den, sum, conf) or "max".
    """
    import torch.distributed as dist
    if plan.group_size == 1:
        return partial
    op = dist.ReduceOp.SUM if reduce_op == "sum" else dist.ReduceOp.MAX
    B = partial.shape[0]
    per = B // plan.group_size
    if collective == "reduce_scatter":
        if partial.numel() * partial.element_size() >= (1 << 31):
            # see below: a single 2 GiB collective on this buffer gave wrong sums on a 4-GPU node; the all-reduce is sliced, the
            # reduce-scatter (one output block per rank) is not
            raise NotImplementedError("reduce_scatter of a packed buffer >= 2 GiB is not validated; use collective='all_reduce' or 'features'")
        if out is None:
            out = torch.empty((per,) + tuple(partial.shape[1:]), dtype=partial.dtype, device=partial.device)
        dist.reduce_scatter_tensor(out, partial.contiguous(), op=op, group=pg)
        return out
    # Issued in slices of at most 512 MiB (whole samples).  Measured on the kernels' first 4- and 8-GPU target: with the
    # 2 GiB buffer of a 32-sample group as ONE call the key points came out wrong by a run-dependent 2-84 mm, while the 1 GiB buffer
    # of a 16-sample group (N = 2) and every smaller case agree with the single-GPU forward to 0.02-0.07 mm.
    per_sample = partial[0].numel() * partial.element_size()
    step = max(1, max_bytes // per_sample)
    for s0 in range(0, B, step):
        dist.all_reduce(partial[s0:s0 + step], op=op, group=pg)
    return partial[plan.view_rank * per:(plan.view_rank + 1) * per]


class PeerExchange:
    """Per-rank reduction buffers of a view group mapped into every member (torch symmetric memory = CUDA IPC /
    fabric handles over NVLink): the fused unprojection kernel stores its partials straight into the owner's buffer
    (`lt_unproject_push_fwd`), a group barrier orders the stores, the owner reduces its slots (`lt_unproject_reduce_
    finalize_fwd`).  No NCCL collective on the data path.
    """

    def __init__(self, plan, pg, batch, planes, nvox, channels, device):
        import torch.distributed._symmetric_memory as symm_mem
        if plan.n_groups > 1:
            # measured on 8 GPUs (2 groups x 4): the symmetric-memory exchanges give wrong key points as soon as two view groups
            # rendezvous side by side, while one group of 2 / 4 / 8 ranks is exact
            raise NotImplementedError("the peer-memory exchange is validated for ONE view group spanning all ranks; "
                                      "use collective='all_reduce' / 'reduce_scatter' / 'features' with several groups")
        self.plan, self.pg = plan, pg
        per = batch // plan.group_size
        self.shape = (plan.group_size, per, planes, nvox, channels)
        self.buf = symm_mem.empty(self.shape, dtype=torch.float32, device=device)
        self.handle = symm_mem.rendezvous(self.buf, pg.group_name if hasattr(pg, "group_name") else pg)
        self.peer_ptrs = [int(p) for p in self.handle.buffer_ptrs]

    def barrier(self):
        self.handle.barrier()


class FeatureExchange:
    """Exchange the 32-channel FEATURE maps instead of voxel partials (SURVEY 8e alternative (i)): 1.18 MB per
    (sample, view) instead of 67 MB per sample, and the owner then unprojects all views locally with exactly the
    single-GPU arithmetic.  Each rank writes its views of sample b into the owner's buffer over NVLink peer memory.
    """

    def __init__(self, plan, pg, batch, n_views, h, w, channels, device):
        self.plan, self.pg = plan, pg
        self.per = batch // plan.group_size
        self.shape = (self.per, n_views, h, w, channels)
        self.n_views = n_views
        # One view group spanning all ranks: symmetric memory + our own store kernel.  Several groups side by side (world 8, 4 views):
        # the symmetric-memory path returned wrong key points on an 8-GPU node (2 groups x 4 ranks; one group of 2 / 4 ranks is exact), so the groups then exchange the same maps with one NCCL all-gather each and assemble locally.
        self.nccl = plan.n_groups > 1
        if self.nccl:
            self.buf = torch.empty(self.shape, dtype=torch.float32, device=device)
            self.gathered = None
            return
        import torch.distributed._symmetric_memory as symm_mem
        self.buf = symm_mem.empty(self.shape, dtype=torch.float32, device=device)
        self.handle = symm_mem.rendezvous(self.buf, pg.group_name if hasattr(pg, "group_name") else pg)
        self.peer_ptrs = [int(p) for p in self.handle.buffer_ptrs]

    def scatter(self, feats_local):
        """feats_local: (B, V_local, h, w, C) -> rows of the owners' buffers: one launch of our own copy kernel whose float4
        stores go straight into peer memory over NVLink (lt_feature_scatter_fwd); NCCL variant: all-gather + local assembly."""
        if self.nccl:
            import torch.distributed as dist
            G = self.plan.group_size
            B, Vl = feats_local.shape[:2]
            if self.gathered is None or self.gathered.shape[1:] != feats_local.shape:
                self.gathered = torch.empty((G,) + tuple(feats_local.shape), dtype=torch.float32, device=feats_local.device)
            dist.all_gather([self.gathered[r] for r in range(G)], feats_local.contiguous(), group=self.pg)
            lo = self.plan.view_rank * self.per
            # global view v = j * G + r is local view j of group rank r:  buf[bl, j, r] = gathered[r, lo + bl, j]
            self.buf.view(self.per, Vl, G, *self.shape[2:]).copy_(self.gathered[:, lo:lo + self.per].permute(1, 2, 0, 3, 4, 5))
            return
        from . import capi
        capi.feature_scatter(feats_local, self.peer_ptrs, self.plan.view_rank, self.n_views)

    def barrier(self):
        if not self.nccl:
            self.handle.barrier()


def gather_keypoints(kp_local, plan, pg):
    """[B/G][J][3] on each rank -> [B][J][3] on every rank of the group."""
    import torch.distributed as dist
    if plan.group_size == 1:
        return kp_local
    outs = [torch.empty_like(kp_local) for _ in range(plan.group_size)]
    dist.all_gather(outs, kp_local.contiguous(), group=pg)
    return torch.cat(outs, dim=0)
