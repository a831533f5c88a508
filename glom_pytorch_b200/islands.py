"""Island analytics on the column states.

The reference's README (README.md:34-36) names the use: ``return_all=True`` "gives you access to all the level data
across iterations for clustering, from which one can inspect for the theorized islands in the paper" -- islands of
(near-)identical vectors at a level across neighbouring image locations.  The reference ships no code for it; this is
the downstream consumer of the ``(T+1, B, n, L, d)`` slab, run on the GPU by ``glom_b200_islands``
(include/glom_b200.h; kernels in csrc/islands.cu, HBM-bound: every state vector is read once).
"""
from collections import namedtuple
from math import isqrt

import torch

from . import _native

Islands = namedtuple("Islands", "cos_right cos_down agreement labels num_islands")


def islands(states, *, grid=None, threshold=0.9):
    """states: (..., n, L, d) fp32 CUDA tensor (e.g. ``model(img, return_all=True)``: (T+1, B, n, L, d)).
    grid: (side_h, side_w) with side_h * side_w == n (default: square).  Returns ``Islands`` of tensors shaped
    (..., L, n) -- ``cos_right``, ``cos_down``, ``agreement`` fp32, ``labels`` int32 (island id = smallest patch index
    of the 4-connected component of neighbour pairs with cosine similarity >= threshold) -- and ``num_islands`` (..., L)."""
    if not states.is_cuda:
        raise RuntimeError("glom_pytorch_b200.islands runs on CUDA sm_90a (H100) only (no CPU fallback)")
    if states.dim() < 3:
        raise RuntimeError("states must be (..., n, L, d)")
    *lead, n, L, d = states.shape
    if grid is None:
        s = isqrt(n)
        if s * s != n:
            raise RuntimeError(f"n = {n} is not a square: pass grid=(side_h, side_w)")
        grid = (s, s)
    side_h, side_w = grid
    if side_h * side_w != n:
        raise RuntimeError(f"grid {grid} does not tile n = {n}")
    if torch.compiler.is_compiling():      # torch.compile / torch.export: the custom op (ops.py), no gradient
        return Islands(*torch.ops.glom_b200.islands(states.detach(), side_h, side_w, float(threshold)))
    x = states.detach().to(torch.float32).contiguous()
    if x.data_ptr() % 16:                 # a contiguous view starting mid-row: the kernels load float4
        x = x.clone()
    slabs = 1
    for v in lead:
        slabs *= v
    dev = x.device
    shape = (*lead, L, n)
    out = [torch.empty(shape, dtype=torch.float32, device=dev) for _ in range(3)]
    labels = torch.empty(shape, dtype=torch.int32, device=dev)
    num = torch.empty((*lead, L), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _native.islands(x.data_ptr(), slabs, side_h, side_w, L, d, float(threshold), out[0].data_ptr(), out[1].data_ptr(),
                        out[2].data_ptr(), labels.data_ptr(), num.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
    return Islands(out[0], out[1], out[2], labels, num)
