"""Multi-GPU rendering: poses (or, for small batches, detector rows) shard across ranks, the volume is replicated,
ONE gather of the image stack.

The reference has no distributed code (SURVEY.md 2a).  Every ray is independent given the volume, so the only
exchange step of the path is assembling the image stack: `all_gather_into_tensor` over NCCL (NVLink/NVSwitch),
whose backward is the local slice of the incoming gradient (pose gradients never leave their rank).
One process per GPU (`torchrun`), `torch.distributed` for the plumbing.

Trilinear caveat (quirk Q3): the sampling range alphamin/alphamax is global over all rays of the call, so sharded
ranks must agree on it -- `global_alpha_range` all-reduces the two scalars (MIN/MAX) and the result is passed
explicitly through the reference's own `alphamin=`, `alphamax=` keywords (renderers.py:214-215).
"""
from __future__ import annotations

import torch
import torch.distributed as dist


class PeerGather:
    """All-gather of equally sized per-rank shards that uses NO SM: every rank owns a symmetric-memory buffer (CUDA VMM
    mapped into all peers of the node), a rank PUSHES its shard into every peer's buffer with plain device copies
    (copy engines over NVLink / NVSwitch) on a side stream, and a symmetric-memory barrier (signal pads) closes the
    exchange.  The NCCL all-gather it replaces runs as a kernel that shares the SMs with the next step's walk and slows it.

    `slots` independent buffers allow the gather of step k to overlap the walk of step k+1 (double buffering).
    Raises if symmetric memory is unavailable (single node with P2P access is required); callers may then fall back to
    `dist.all_gather_into_tensor`."""

    def __init__(self, shard_shape, dtype, device, group=None, slots: int = 2):
        import torch.distributed._symmetric_memory as symm_mem

        group = group if group is not None else dist.group.WORLD
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.shard_shape, self.slots = tuple(shard_shape), slots
        self.full_shape = (self.world * self.shard_shape[0],) + self.shard_shape[1:]
        self.buf = symm_mem.empty((slots,) + self.full_shape, dtype=dtype, device=device)
        self.hdl = symm_mem.rendezvous(self.buf, group)
        self.peers = [self.hdl.get_buffer(p, (slots,) + self.full_shape, dtype) for p in range(self.world)]
        self.stream = torch.cuda.Stream(device=device)
        self.done = [None] * slots
        self.n = self.shard_shape[0]

    def push(self, local: torch.Tensor, slot: int = 0) -> None:
        """Start gathering `local` (this rank's shard) into slot `slot` of every rank's buffer; returns immediately."""
        ready = torch.cuda.Event()
        ready.record(torch.cuda.current_stream())
        lo, hi = self.rank * self.n, (self.rank + 1) * self.n
        with torch.cuda.stream(self.stream):
            self.stream.wait_event(ready)
            # start with the right-hand neighbour so the 8 ranks do not all write to the same peer at once
            for k in range(self.world):
                p = (self.rank + k) % self.world
                self.peers[p][slot, lo:hi].copy_(local, non_blocking=True)
            self.hdl.barrier(channel=slot)   # every rank's pushes into MY buffer are complete once this returns
            ev = torch.cuda.Event()
            ev.record(self.stream)
        self.done[slot] = ev

    def wait(self, slot: int = 0) -> torch.Tensor:
        """Make the current stream wait for the gather of `slot`; returns the gathered (world*B, ...) tensor."""
        if self.done[slot] is not None:
            torch.cuda.current_stream().wait_event(self.done[slot])
            self.done[slot] = None
        return self.buf[slot]


def shard_bounds(n_items: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous, balanced [lo, hi) slice of `n_items` for `rank` (first n_items % world ranks get one more)."""
    if world <= 0 or not 0 <= rank < world:
        raise ValueError(f"bad rank/world {rank}/{world}")
    base, extra = divmod(n_items, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def balanced_pose_assignment(costs, world: int) -> list[list[int]]:
    """Split len(costs) poses into `world` groups of EQUAL size whose summed costs are as even as a greedy pass gets them
    (longest-processing-time first, each group capped at n / world members).  The walk's time is data dependent (voxels
    visited per pose, `siddon_visits`), and a step ends when the slowest rank does: with contiguous slices the slowest of
    8 ranks carried 2.5 % more visits than the mean in the bench's pose set."""
    n = len(costs)
    if world <= 0 or n % world:
        raise ValueError("the number of poses must be a multiple of the number of ranks")
    cap = n // world
    order = sorted(range(n), key=lambda i: -float(costs[i]))
    groups, loads = [[] for _ in range(world)], [0.0] * world
    for i in order:
        r = min((g for g in range(world) if len(groups[g]) < cap), key=lambda g: loads[g])
        groups[r].append(i)
        loads[r] += float(costs[i])
    return [sorted(g) for g in groups]


class _AllGatherBatch(torch.autograd.Function):
    """Concatenate equally-sized per-rank batches along dim 0; backward keeps this rank's slice of the gradient."""

    @staticmethod
    def forward(ctx, local, group):
        world = dist.get_world_size(group)
        ctx.rank = dist.get_rank(group)
        ctx.n = local.shape[0]
        out = local.new_empty((world * local.shape[0],) + tuple(local.shape[1:]))
        dist.all_gather_into_tensor(out, local.contiguous(), group=group)
        return out

    @staticmethod
    def backward(ctx, grad):
        return grad[ctx.rank * ctx.n:(ctx.rank + 1) * ctx.n], None


def all_gather_images(local: torch.Tensor, batch: int | None = None, group=None) -> torch.Tensor:
    """(B_local, C, H, W) on every rank -> (B, C, H, W) on every rank (differentiable).  Ragged shards are padded."""
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return local
    world = dist.get_world_size(group)
    if batch is None or batch % world == 0:
        return _AllGatherBatch.apply(local, group)
    per = -(-batch // world)  # ceil: pad every shard to the same size, gather, drop the padding
    pad = per - local.shape[0]
    padded = torch.cat([local, local.new_zeros((pad,) + tuple(local.shape[1:]))]) if pad else local
    full = _AllGatherBatch.apply(padded, group)
    keep = []
    for r in range(world):
        lo, hi = shard_bounds(batch, r, world)
        keep.append(full[r * per:r * per + (hi - lo)])
    return torch.cat(keep)


class _GlobalExtremum(torch.autograd.Function):
    """min (or max) of one scalar per rank.  Backward: the upstream gradients of ALL ranks are summed (every rank's
    rays march the shared range) and handed to the rank(s) that own the extremum -- the distributed form of the
    arg-min / arg-max branch of reference renderers.py:221-223."""

    @staticmethod
    def forward(ctx, local, is_min, group):
        out = local.detach().clone()
        dist.all_reduce(out, op=dist.ReduceOp.MIN if is_min else dist.ReduceOp.MAX, group=group)
        ctx.owner = bool(local.detach() == out)
        ctx.group = group
        return out

    @staticmethod
    def backward(ctx, grad):
        total = grad.contiguous().clone()
        dist.all_reduce(total, op=dist.ReduceOp.SUM, group=ctx.group)
        return (total if ctx.owner else torch.zeros_like(total)), None, None


def global_alpha_range(alphamin: torch.Tensor, alphamax: torch.Tensor, group=None):
    """Trilinear sampling range shared by all ranks (MIN / MAX of the per-rank ranges), differentiable."""
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        return _GlobalExtremum.apply(alphamin, True, group), _GlobalExtremum.apply(alphamax, False, group)
    return alphamin, alphamax


class _SumGradAcrossRanks(torch.autograd.Function):
    """Identity whose backward all-reduces (SUM) the gradient: pose parameters are replicated on every rank while each
    rank differentiates only its own rays, so the true gradient is the sum of the per-rank partials."""

    @staticmethod
    def forward(ctx, x, group):
        ctx.group = group
        return x.view_as(x)

    @staticmethod
    def backward(ctx, grad):
        total = grad.contiguous().clone()
        dist.all_reduce(total, op=dist.ReduceOp.SUM, group=ctx.group)
        return total, None


class _AllGatherRows(torch.autograd.Function):
    """(B, C, h_local, W) row blocks (balanced contiguous split of H, shard_bounds) -> (B, C, H, W) on every rank;
    backward keeps this rank's rows of the gradient."""

    @staticmethod
    def forward(ctx, local, height, group):
        rank, world = dist.get_rank(group), dist.get_world_size(group)
        B, C, h, W = local.shape
        per = -(-height // world)
        padded = local if h == per else torch.cat([local, local.new_zeros(B, C, per - h, W)], dim=2)
        flat = local.new_empty(world * B, C, per, W)  # rank-major concatenation along dim 0
        dist.all_gather_into_tensor(flat, padded.contiguous(), group=group)
        out = flat.view(world, B, C, per, W)
        blocks = []
        for r in range(world):
            lo, hi = shard_bounds(height, r, world)
            blocks.append(out[r, :, :, :hi - lo])
        ctx.span = shard_bounds(height, rank, world)
        return torch.cat(blocks, dim=2)

    @staticmethod
    def backward(ctx, grad):
        return grad[:, :, ctx.span[0]:ctx.span[1]].contiguous(), None, None


def render_ray_sharded(drr, *pose_args, group=None, gather: bool = True, **kwargs):
    """`drr(*pose_args, **kwargs)` with the DETECTOR ROWS sharded over the ranks (SURVEY.md 8e: the partitioning for
    batches smaller than the GPU count, e.g. the B = 1 registration loop).  Every rank holds the full pose batch, renders
    a contiguous block of rows of every pose and (gather=True) returns the full (B, C, H, W) stack.  Pose gradients are
    summed over the ranks in backward, so after `loss.backward()` every rank holds the full gradient, exactly as on
    one GPU.  Trilinear's batch-global alpha range is computed from the full ray set on every rank (no collective)."""
    from .pose import RigidTransform, convert
    from .renderers import Trilinear, _dims_tensor, _get_alpha_minmax

    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return drr(*pose_args, **kwargs)
    det = drr.detector
    if det.n_subsample is not None or drr.patch_size is not None or not drr.reshape:
        raise NotImplementedError("ray sharding needs the full, reshaped detector grid (no p_subsample / patch_size)")
    kwargs = dict(kwargs)
    parameterization, convention = kwargs.pop("parameterization", None), kwargs.pop("convention", None)
    degrees, calibration = kwargs.pop("degrees", False), kwargs.pop("calibration", None)
    mask_to_channels = kwargs.pop("mask_to_channels", False)
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    if parameterization is None:
        pose = RigidTransform(_SumGradAcrossRanks.apply(pose_args[0].matrix, group))
    else:
        pose = convert(*(_SumGradAcrossRanks.apply(a, group) for a in pose_args), parameterization=parameterization,
                       convention=convention, degrees=degrees)
    H, W, B = det.height, det.width, len(pose)
    h0, h1 = shard_bounds(H, rank, world)
    if drr._pose_in_ok(mask_to_channels, kwargs):
        img = drr._render_pose_in(pose, calibration, rows=(h0, h1))
    else:
        source, target = det(pose, calibration)
        if isinstance(drr.renderer, Trilinear) and kwargs.get("alphamin") is None:
            s_v, t_v = drr.affine_inverse(source), drr.affine_inverse(target)
            amin, amax = _get_alpha_minmax(s_v, t_v, _dims_tensor(drr.density.shape, s_v.device, s_v.dtype),
                                           drr.renderer.voxel_shift, drr.renderer.eps)
            kwargs.update(alphamin=amin.min(), alphamax=amax.max())  # quirk Q3: the range of ALL rays of the call
        img = drr.render(drr.density, source, target[:, h0 * W:h1 * W].contiguous(), mask_to_channels,
                         grid_shape=(h1 - h0, W), **kwargs)
    img = img.view(B, -1, h1 - h0, W)
    return _AllGatherRows.apply(img, H, group) if gather else img


def render_sharded(drr, *pose_args, group=None, gather: bool = True, shard: str = "auto", **kwargs):
    """`drr(*pose_args, **kwargs)` sharded over the ranks of `group`.

    shard="poses": every rank passes the FULL pose batch (rotation, translation tensors or a RigidTransform), renders only
    its contiguous slice of poses and, with gather=True, returns the full (B, C, H, W) stack; gradients flow to the local
    slice.  shard="rays": `render_ray_sharded` (detector rows split, pose gradients summed over ranks).
    shard="auto": poses when the batch has at least one pose per rank, rays otherwise.
    """
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return drr(*pose_args, **kwargs)
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    batch = len(pose_args[0])
    if shard not in ("auto", "poses", "rays"):
        raise ValueError("shard must be 'auto', 'poses' or 'rays'")
    if shard == "rays" or (shard == "auto" and batch < world):
        return render_ray_sharded(drr, *pose_args, group=group, gather=gather, **kwargs)
    lo, hi = shard_bounds(batch, rank, world)
    local_args = tuple(a[lo:hi] for a in pose_args)
    from .renderers import Trilinear, _get_alpha_minmax

    if isinstance(drr.renderer, Trilinear) and kwargs.get("alphamin") is None:
        # the range must come from ALL rays of the call, not only this rank's (quirk Q3)
        from .pose import convert

        pose = local_args[0] if kwargs.get("parameterization") is None else convert(
            *local_args, parameterization=kwargs["parameterization"], convention=kwargs.get("convention"),
            degrees=kwargs.get("degrees", False))
        src, tgt = drr.detector(pose, kwargs.get("calibration"))
        src, tgt = drr.affine_inverse(src), drr.affine_inverse(tgt)
        dims = torch.tensor(drr.density.shape, device=src.device, dtype=src.dtype)
        amin, amax = _get_alpha_minmax(src, tgt, dims, drr.renderer.voxel_shift, drr.renderer.eps)
        amin, amax = global_alpha_range(amin.min(), amax.max(), group)  # differentiable: owner rank keeps the branch
        kwargs = dict(kwargs, alphamin=amin, alphamax=amax)
    img = drr(*local_args, **kwargs)
    return all_gather_images(img, batch, group) if gather else img
