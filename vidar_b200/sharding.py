"""Work partitioning of the hot path over ranks (one process per GPU).

SURVEY.md 8(e): the MSDA stage shards the (camera, query) rows of SpatialCrossAttention --
cameras are independent until the scatter-add into the BEV slots
(spatial_cross_attention.py:164-171) -- and exchanges the per-row outputs ONCE (all-gather of
the BEV rows); the ray stages shard rays and all-reduce the small grad_sigma volume.  The
reference has no counterpart (replica DDP only, apis/mmdet_train.py:72-81).
Pure host logic: usable with any torch.distributed backend (tests run it over gloo on CPU).
"""
import torch
import torch.distributed as dist


def shard_range(n, rank, world):
    """Contiguous, balanced [lo, hi) share of n items."""
    return rank * n // world, (rank + 1) * n // world


def shard_rows(rank, world, cams, Q):
    """Contiguous share of the cams*Q (camera, query) rows -> [(cam, q0, q1), ...]."""
    lo, hi = shard_range(cams * Q, rank, world)
    segs = []
    for c in range(cams):
        a, b = max(lo, c * Q), min(hi, (c + 1) * Q)
        if a < b:
            segs.append((c, a - c * Q, b - c * Q))
    return segs


def cameras_of(rank, world, cams, Q):
    return sorted({c for c, _, _ in shard_rows(rank, world, cams, Q)})


def shard_layouts(group, world):
    """Global ranks of the `world` ranks of every rank's shard group -> (every distinct layout, sorted; this rank's).
    group None or WORLD: the one layout 0 .. world - 1.  Otherwise one all-gather over the world, so EVERY rank must
    call this, each with its own shard group: sub-groups made from these layouts are then made by every rank in the
    same order (new_group is collective over the whole world and takes global ranks)."""
    if group is None or group is dist.group.WORLD:
        mine = tuple(range(world))
        return [mine], mine
    mine = tuple(dist.get_global_rank(group, r) for r in range(world))
    every = [None] * dist.get_world_size()
    dist.all_gather_object(every, mine)
    return sorted(set(every)), mine


def camera_groups(world, cams, Q, rank, group=None):
    """Process groups for cameras whose rows are split over several ranks (their partial
    grad_value must be summed).  EVERY rank must call this (new_group is collective).
    `world` / `rank`: size of and rank in the shard group `group` (None: the whole world); every shard group's camera
    groups are made on every rank, from global ranks.  -> {cam: group} for the cameras this rank shares."""
    layouts, mine = shard_layouts(group, world)
    groups = {}
    for ranks in layouts:
        for c in range(cams):
            members = [r for r in range(world) if c in cameras_of(r, world, cams, Q)]
            if len(members) > 1:
                g = dist.new_group([ranks[m] for m in members])
                if ranks == mine and rank in members:
                    groups[c] = g
    return groups


# ------------------------------------------------------------------------------------------------
# Data-parallel replicas of the sharded step: a (replica x shard) process grid.
#
# The world splits into R = world / S replicas of S contiguous ranks; each replica trains on its own sample and shards
# it over its shard group exactly as a single-replica run shards over the world.  After backward a parameter's
# gradient on a rank is either PARTIAL (tagged `vidar_partial_grad`: the shard group's sum is the replica's gradient)
# or REPLICATED (every shard rank of the replica holds the whole, identical gradient).  One all-reduce (SUM) over the
# world of the bucket
#     partial:     grad * 1/R                        on every rank
#     replicated:  grad * 1/R on shard rank 0,  * 0  on the other shard ranks
# leaves on every rank the mean over replicas of the shard sums, and the mean over replicas of the replicated
# gradients -- taken once per replica, so it never becomes (x + x + x) / 3 with its extra rounding.
# ------------------------------------------------------------------------------------------------
class Grid:
    """This rank's place in the (replica x shard) grid (`make_grid`).
      group        its shard group (S contiguous global ranks; the world itself when R == 1)
      replica      replica index, 0 .. replicas - 1 (rank // S)
      shard_rank   rank in the shard group (rank % S)
      replicas, shard_size   R and S
      world_group  the group of the gradient all-reduce (every rank)"""

    def __init__(self, group, replica, shard_rank, replicas, shard_size, world_group):
        self.group, self.replica, self.shard_rank = group, replica, shard_rank
        self.replicas, self.shard_size, self.world_group = replicas, shard_size, world_group

    def __repr__(self):
        return (f"Grid({self.replicas} x {self.shard_size}: replica {self.replica}, shard rank {self.shard_rank})")


def make_grid(shard_size):
    """Split the world into world / shard_size replicas of `shard_size` contiguous ranks.  EVERY rank must call this
    (each shard group is made by every rank, in the same order).  -> this rank's `Grid`."""
    world, rank = dist.get_world_size(), dist.get_rank()
    if not isinstance(shard_size, int) or shard_size < 1 or world % shard_size:
        raise ValueError(f"shard_size must be a positive divisor of the world size {world}, got {shard_size!r}")
    replicas = world // shard_size
    if replicas == 1:
        group = dist.group.WORLD
    else:
        group = None
        for r in range(replicas):
            g = dist.new_group(list(range(r * shard_size, (r + 1) * shard_size)))
            if r == rank // shard_size:
                group = g
    return Grid(group, rank // shard_size, rank % shard_size, replicas, shard_size, dist.group.WORLD)


def grid_grad_scales(params, grid):
    """The bucket scale of every parameter (see the comment above `Grid`)."""
    inv = 1.0 / grid.replicas
    return [inv if getattr(p, "vidar_partial_grad", False) or grid.shard_rank == 0 else 0.0 for p in params]


def allreduce_grid_grads(module, grid):
    """Every trainable parameter's gradient -> the replica mean (partial ones: of the shard sums), identical on
    every rank: pack into one fp32 bucket (`grad_bucket.pack`, gradients that are None pack as zeros), ONE all-reduce
    over the world, unpack into `.grad` (allocated where None).  -> bucket elements."""
    from . import grad_bucket
    ps = [p for p in module.parameters() if p.requires_grad]
    if not ps:
        return 0
    bucket = grad_bucket.pack(ps, grid_grad_scales(ps, grid))
    if grid.replicas * grid.shard_size > 1:
        dist.all_reduce(bucket, group=grid.world_group)
    grad_bucket.unpack(bucket, ps)
    return bucket.numel()


def gather_rows(local_rows, world, total_rows, group=None):
    """all-gather of per-rank row blocks [n_r, C] (balanced contiguous shards) -> [total_rows, C]."""
    if world == 1:
        return local_rows
    if total_rows % world == 0:
        full = local_rows.new_empty(total_rows, local_rows.shape[1])
        dist.all_gather_into_tensor(full.view(-1), local_rows.contiguous().view(-1), group=group)
        return full
    max_rows = -(-total_rows // world)
    pad = local_rows.new_zeros(max_rows, local_rows.shape[1])
    pad[: local_rows.shape[0]] = local_rows
    flat = local_rows.new_empty(world * max_rows, local_rows.shape[1])
    dist.all_gather_into_tensor(flat.view(-1), pad.view(-1), group=group)
    buf = flat.view(world, max_rows, local_rows.shape[1])
    parts = []
    for r in range(world):
        lo, hi = shard_range(total_rows, r, world)
        parts.append(buf[r, : hi - lo])
    return torch.cat(parts, 0)


# ------------------------------------------------------------------------------------------------
# Replicated <-> row-sharded conversions with autograd (the BEV-grid exchange of SURVEY.md 8e).
#
# Convention: tensors outside a sharded region are REPLICATED (every rank holds the same value and runs
# the same downstream computation, so every rank also holds the same gradient).  Inside a region each
# rank holds either a partial sum of the full tensor (camera-sharded SpatialCrossAttention slots) or a
# contiguous block of its rows.
#   reduce_scatter_rows : partial sums [R, C] on every rank  ->  this rank's rows of the total
#                         (backward: all-gather of the row gradients -- d total / d partial_r = I)
#   all_gather_rows     : this rank's rows  ->  the full replicated tensor  (the ONE all-gather of the BEV
#                         grid; backward: the local slice of the replicated gradient, no communication -- or,
#                         with grad="sum", the reduce-scatter of per-rank partial gradients when the consumers
#                         of the gathered grid are themselves sharded)
# Parameters used on sharded data (value_proj on a rank's cameras, output_proj / FFN on a rank's rows)
# end up with PARTIAL gradients; they are tagged with `mark_partial` and summed over the group once per
# step by `allreduce_partial_grads` (one bucketed all-reduce, like DDP's).
# ------------------------------------------------------------------------------------------------
def _rows_padded(n, world):
    return -(-n // world)


def _reduce_scatter_block(partial, group):
    """[R, ...] partial sums -> (this rank's block of the sum, rows per block)."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    R = partial.shape[0]
    per = _rows_padded(R, world)
    x = partial.contiguous()
    if per * world != R:
        pad = x.new_zeros((per * world,) + tuple(x.shape[1:]))
        pad[:R] = x
        x = pad
    lo = rank * per
    if dist.get_backend(group) == "gloo":          # CPU tests: gloo has no reduce_scatter
        x = x.clone()
        dist.all_reduce(x, group=group)
        out = x[lo: lo + per]
    else:
        out = x.new_empty((per,) + tuple(x.shape[1:]))
        dist.reduce_scatter_tensor(out, x, group=group)
    return out[: max(0, min(R, lo + per) - lo)], per


def _all_gather_blocks(rows, R, group):
    """This rank's block (possibly short) -> the full [R, ...] tensor."""
    world = dist.get_world_size(group)
    per = _rows_padded(R, world)
    x = rows.contiguous()
    if x.shape[0] != per:
        pad = x.new_zeros((per,) + tuple(x.shape[1:]))
        pad[: x.shape[0]] = x
        x = pad
    full = x.new_empty((per * world,) + tuple(x.shape[1:]))
    dist.all_gather_into_tensor(full, x, group=group)
    return full[:R]


class _ReduceScatterRows(torch.autograd.Function):
    @staticmethod
    def forward(ctx, partial, group):
        ctx.meta = (group, partial.shape[0])
        return _reduce_scatter_block(partial, group)[0]

    @staticmethod
    def backward(ctx, grad_rows):
        group, R = ctx.meta
        return _all_gather_blocks(grad_rows, R, group), None


class _AllGatherRows(torch.autograd.Function):
    """Consumers downstream are REPLICATED: every rank holds the same full gradient, its block is a slice."""

    @staticmethod
    def forward(ctx, rows, R, group):
        ctx.meta = row_range(R, dist.get_rank(group), dist.get_world_size(group))
        return _all_gather_blocks(rows, R, group)

    @staticmethod
    def backward(ctx, grad_full):
        lo, hi = ctx.meta
        return grad_full[lo:hi], None, None


class _AllGatherRowsSumGrad(torch.autograd.Function):
    """Consumers downstream are SHARDED (each rank uses the gathered tensor for its own rows / cameras only): the
    per-rank gradients are partial sums, the block's gradient is their reduce-scatter."""

    @staticmethod
    def forward(ctx, rows, R, group):
        ctx.group = group
        return _all_gather_blocks(rows, R, group)

    @staticmethod
    def backward(ctx, grad_full):
        return _reduce_scatter_block(grad_full, ctx.group)[0], None, None


def row_range(R, rank, world):
    """[lo, hi) of the rows `reduce_scatter_rows` / `all_gather_rows` give to `rank` (equal blocks of
    ceil(R / world) rows, the last ones possibly short or empty)."""
    per = _rows_padded(R, world)
    lo = min(R, rank * per)
    return lo, min(R, lo + per)


def reduce_scatter_rows(partial, group):
    """[R, ...] partial sums on every rank -> this rank's block of rows of the sum."""
    return _ReduceScatterRows.apply(partial, group)


def all_gather_rows(rows, R, group, grad="slice"):
    """This rank's block of rows -> the full [R, ...] tensor on every rank.
    grad="slice": what follows is replicated computation (identical gradients on every rank; backward takes the
    block, no communication).  grad="sum": what follows is sharded computation (row-sharded encoder layers, camera-
    sharded sampling) whose per-rank gradients are partial sums; backward reduce-scatters them."""
    if grad not in ("slice", "sum"):
        raise ValueError(f"grad must be 'slice' or 'sum', got {grad!r}")
    return (_AllGatherRows if grad == "slice" else _AllGatherRowsSumGrad).apply(rows, R, group)


def local_rows(full, group):
    """The block of a replicated [R, ...] tensor that belongs to this rank (no communication)."""
    lo, hi = row_range(full.shape[0], dist.get_rank(group), dist.get_world_size(group))
    return full[lo:hi]


def mark_partial(module):
    """Tag a module's parameters: inside a sharded region their gradients are per-rank partial sums."""
    for p in module.parameters():
        p.vidar_partial_grad = True
    return module


def allreduce_partial_grads(module, group):
    """Sum the gradients of every tagged parameter over `group` in ONE all-reduce."""
    # every rank must contribute the SAME bucket: a rank that owns no camera never touches the backbone and has no
    # gradient for it (None) -- it sends zeros and receives the sum
    ps = [p for p in module.parameters() if getattr(p, "vidar_partial_grad", False) and p.requires_grad]
    if not ps or dist.get_world_size(group) == 1:
        return 0
    flat = torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1) for p in ps])
    dist.all_reduce(flat, group=group)
    off = 0
    for p in ps:
        n = p.numel()
        if p.grad is None:
            p.grad = flat[off: off + n].view_as(p).clone()
        else:
            p.grad.copy_(flat[off: off + n].view_as(p.grad))
        off += n
    return flat.numel()


class _SumGrad(torch.autograd.Function):
    """Identity whose backward sums the gradient over the group: for a REPLICATED tensor that every rank
    consumes in a sharded computation (each rank's gradient is then a partial sum)."""

    @staticmethod
    def forward(ctx, x, group):
        ctx.group = group
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous().clone()
        dist.all_reduce(g, group=ctx.group)
        return g, None


def sum_grad(x, group):
    return _SumGrad.apply(x, group)


class _ScaleGrad(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, scale):
        ctx.scale = scale
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return g * ctx.scale, None


def replicated_view(x, group):
    """View of a tensor gathered with `all_gather_rows(..., grad="sum")` for a REPLICATED consumer (one that every
    rank runs identically): its gradient is the same on every rank, so each rank contributes 1/world of it to the
    reduce-scatter.  Lets one gathered tensor feed sharded and replicated consumers at once."""
    return _ScaleGrad.apply(x, 1.0 / dist.get_world_size(group))
