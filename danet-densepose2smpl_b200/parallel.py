"""Image-parallel sharding of the hot path over the GPUs of one node (SURVEY section 8e).

The path has no cross-image state at inference (BatchNorm in eval mode), so each rank runs the
whole pipeline on a contiguous slice of the batch with replicated weights; the only collective is
one all_gather of the outputs the caller consumes (para: 916 B / image)."""
import torch
import torch.distributed as dist


def shard_bounds(n, world, rank):
    """Contiguous slice [lo, hi) of n items for `rank`; remainder goes to the low ranks."""
    base, rem = divmod(n, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard(t, world=None, rank=None):
    world = dist.get_world_size() if world is None else world
    rank = dist.get_rank() if rank is None else rank
    lo, hi = shard_bounds(t.shape[0], world, rank)
    return t[lo:hi]


def gather_outputs(local, n_total, group=None):
    """All-gather variable-length shards (padded to the largest shard) back into [n_total, ...]."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return local
    world = dist.get_world_size(group)
    per = (n_total + world - 1) // world
    pad = torch.zeros((per,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[:local.shape[0]] = local
    out = torch.empty((world * per,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, pad, group=group)
    pieces = []
    for r in range(world):
        lo, hi = shard_bounds(n_total, world, r)
        pieces.append(out[r * per:r * per + (hi - lo)])
    return torch.cat(pieces, 0)


def infer_sharded(model, images, group=None, infer=None):
    """Every rank passes the same [N,3,224,224] batch (or its own view of it); returns para [N,229]
    on every rank.  `infer` (images -> para) defaults to model.infer_net; an empty shard contributes an empty
    tensor on the MODEL's device (the collective needs one device type on every rank)."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    lo, hi = shard_bounds(images.shape[0], world, rank)
    local = images[lo:hi]
    if infer is None:
        infer = lambda x: model.infer_net(x)["para"]
    if hi > lo:
        para = infer(local)
    else:
        dev = next(model.parameters()).device if model is not None else images.device
        para = torch.zeros(0, 229, device=dev)
    return gather_outputs(para, images.shape[0], group)


def all_reduce_gradients(tensors, group=None, bucket_bytes=64 << 20, average=True):
    """Data-parallel gradient exchange of the training step (SURVEY section 8e/8f-2: the reference trains on one process
    and has none; BASELINE configs[4] is 16 images x 8 GPUs).  `tensors`: parameters (their .grad is reduced in place;
    parameters without a gradient are skipped) or plain gradient tensors.  Gradients of one dtype are packed into
    flat buckets of <= bucket_bytes so that ~100 M parameters are a handful of collectives sized for NVLink bandwidth,
    not 2476 launch-latency-bound ones; SUM over ranks, then / world (average=True).  Every rank must pass the same
    tensors in the same order.  Returns the number of collectives issued (0 without a process group / with one rank)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return 0
    world = dist.get_world_size(group)
    grads = []
    for t in tensors:
        g = t.grad if isinstance(t, torch.nn.Parameter) or getattr(t, "grad", None) is not None else t
        if g is not None:
            grads.append(g)
    buckets, cur, cur_bytes = [], [], 0
    for g in grads:
        nb = g.numel() * g.element_size()
        if cur and (cur[0].dtype != g.dtype or cur[0].device != g.device or cur_bytes + nb > bucket_bytes):
            buckets.append(cur)
            cur, cur_bytes = [], 0
        cur.append(g)
        cur_bytes += nb
    if cur:
        buckets.append(cur)
    for b in buckets:
        flat = torch.cat([g.reshape(-1) for g in b]) if len(b) > 1 else b[0].reshape(-1).clone()
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
        if average:
            flat /= world
        off = 0
        for g in b:
            n = g.numel()
            g.copy_(flat[off:off + n].view_as(g))
            off += n
    return len(buckets)


def broadcast_buffers(tensors, group=None, src=0, bucket_bytes=64 << 20):
    """Rank `src` (a rank of `group`)'s copy of `tensors` on every rank, in place: DistributedDataParallel's default
    broadcast_buffers, which the training step uses for the BatchNorm running statistics and counters (each rank's
    training-mode forward updates them from its own shard).  Tensors of one dtype and device are packed into flat
    buckets of <= bucket_bytes (one tensor larger than that is a bucket of its own), as all_reduce_gradients packs
    gradients.  Every rank must pass the same tensors in the
    same order.  Returns the number of collectives issued (0 without a process group / with one rank)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return 0
    root = dist.get_global_rank(group, src) if group is not None else src
    kinds = {}                                   # BatchNorm interleaves fp32 statistics and int64 counters
    for t in tensors:
        kinds.setdefault((t.dtype, t.device), []).append(t)
    buckets = []
    for ts in kinds.values():
        cur, cur_bytes = [], 0
        for t in ts:
            nb = t.numel() * t.element_size()
            if cur and cur_bytes + nb > bucket_bytes:
                buckets.append(cur)
                cur, cur_bytes = [], 0
            cur.append(t)
            cur_bytes += nb
        if cur:
            buckets.append(cur)
    for b in buckets:
        flat = torch.cat([t.reshape(-1) for t in b])
        dist.broadcast(flat, src=root, group=group)
        off = 0
        for t in b:
            n = t.numel()
            t.copy_(flat[off:off + n].view_as(t))
            off += n
    return len(buckets)
