"""Batch-axis partitioning of the column update across ranks: every term of the
update is per-image, so rank r owns a contiguous slice of images and no collective is needed."""


def shard_range(batch, rank, world):
    """[start, stop) of the images rank `rank` of `world` owns; remainders go to the low ranks."""
    if world < 1 or not (0 <= rank < world):
        raise ValueError(f"bad rank/world {rank}/{world}")
    base, rem = divmod(batch, world)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


def shard(t, rank, world, dim=0):
    s, e = shard_range(t.shape[dim], rank, world)
    return t.narrow(dim, s, e - s)
