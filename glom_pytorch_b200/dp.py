"""Data-parallel training plumbing: the only collective the GLOM path ever needs.

The forward shards along the batch with no exchange step (``sharding.py``).  When a loss is attached
(README.md:58-90), each rank's backward (``glom_b200_backward``) produces gradients of the replicated parameters for
its own images; they are averaged over the ranks with a bucketed all-reduce (NCCL over NVLink / NVSwitch between
GPUs, gloo in the CPU tests).

Why this is a plain collective and not a kernel fused with the backward: the engine's backward walks the T
iterations in reverse and ACCUMULATES every weight gradient over all of them (the MLP weights are shared by all
iterations), so no parameter's gradient is final before the last kernel of the reverse pass has run -- there is no
tile of the result that could be sent while later tiles are still being computed.  The transfer is 23.5 M fp32
values (94 MB) per step: ~0.3 ms at the measured 725 GB/s all-reduce bus bandwidth against a ~19 ms backward.
"""
import torch
import torch.distributed as dist

BUCKET_BYTES = 32 << 20     # launch-latency-sized buckets; NVSwitch bandwidth is per GPU, not per link


def _buckets(tensors, bucket_bytes):
    cur, size = [], 0
    for t in tensors:
        nb = t.numel() * t.element_size()
        if cur and size + nb > bucket_bytes:
            yield cur
            cur, size = [], 0
        cur.append(t)
        size += nb
    if cur:
        yield cur


def allreduce_gradients(module, group=None, bucket_bytes=BUCKET_BYTES, average=True):
    """Average ``p.grad`` of every parameter of ``module`` over the ranks of ``group`` (in place).

    Parameters without a gradient on this rank (e.g. ``init_levels`` when ``levels`` was passed) contribute zeros so
    that every rank issues the same collectives.  Returns the number of all-reduce calls issued."""
    if not dist.is_available() or not dist.is_initialized():
        return 0
    world = dist.get_world_size(group)
    if world == 1:
        return 0
    grads = []
    for p in module.parameters():
        if not p.requires_grad:
            continue
        if p.grad is None:
            p.grad = torch.zeros_like(p)
        grads.append(p.grad)
    calls = 0
    works = []
    for bucket in _buckets(grads, bucket_bytes):
        flat = torch.cat([g.reshape(-1) for g in bucket]) if len(bucket) > 1 else bucket[0].reshape(-1)
        works.append((dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group, async_op=True), flat, bucket))
        calls += 1
    for work, flat, bucket in works:          # buckets are in flight together; unpack as each completes
        work.wait()
        if average:
            flat.div_(world)
        if len(bucket) > 1:
            off = 0
            for g in bucket:
                g.copy_(flat[off:off + g.numel()].view_as(g))
                off += g.numel()
    return calls


def broadcast_parameters(module, src=0, group=None):
    """Replicate rank ``src``'s parameters and buffers (setup-time only)."""
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return
    for t in list(module.parameters()) + list(module.buffers()):
        dist.broadcast(t.data, src=src, group=group)
    if hasattr(module, "invalidate_packed"):
        module.invalidate_packed()
