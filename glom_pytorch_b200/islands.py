"""Island analytics on the column states.

The reference's README (README.md:34-36) names the use: ``return_all=True`` "gives you access to all the level data
across iterations for clustering, from which one can inspect for the theorized islands in the paper" -- islands of
(near-)identical vectors at a level across neighbouring image locations.  The reference ships no code for it; this is
the downstream consumer of the ``(T+1, B, n, L, d)`` slab, run on the GPU by ``glom_b200_islands``
(include/glom_b200.h; kernels in csrc/islands.cu, HBM-bound: every state vector is read once).  ``parse_tree`` relates
each level's islands to the level above -- the part-whole tree the paper is about -- by ``glom_b200_island_tree``
(include/glom_b200_tree.h; kernels in csrc/island_tree.cu).
"""
from collections import namedtuple
from math import isqrt

import torch

from . import _native
from .glom import _f32

Islands = namedtuple("Islands", "cos_right cos_down agreement labels num_islands")
ParseTree = namedtuple("ParseTree", "labels num_islands size parent containment nested embedding member_cos coherence")


def _geometry(states, grid):
    """-> (lead, n, L, d, side_h, side_w) of (..., n, L, d) CUDA states on a side_h x side_w patch grid."""
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
    return lead, n, L, d, side_h, side_w


def islands(states, *, grid=None, threshold=0.9):
    """states: (..., n, L, d) fp32 CUDA tensor (e.g. ``model(img, return_all=True)``: (T+1, B, n, L, d)).
    grid: (side_h, side_w) with side_h * side_w == n (default: square).  Returns ``Islands`` of tensors shaped
    (..., L, n) -- ``cos_right``, ``cos_down``, ``agreement`` fp32, ``labels`` int32 (island id = smallest patch index
    of the 4-connected component of neighbour pairs with cosine similarity >= threshold) -- and ``num_islands`` (..., L)."""
    lead, n, L, d, side_h, side_w = _geometry(states, grid)
    if torch.compiler.is_compiling():      # torch.compile / torch.export: the custom op (ops.py), no gradient
        return Islands(*torch.ops.glom_b200.islands(states.detach(), side_h, side_w, float(threshold)))
    x = _f32(states)                       # the kernels load float4
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


def parse_tree(states, *, grid=None, threshold=0.9, embeddings=False):
    """The part-whole tree of the islands of ``islands(states, grid=grid, threshold=threshold)``: each level's islands
    nested in the level above (include/glom_b200_tree.h, kernels in csrc/island_tree.cu).  Returns ``ParseTree``:

    - ``labels``, ``num_islands``: those of ``islands`` (same call, same bits);
    - ``size`` (..., L, n) int32: at a root j (``labels[..., l, j] == j``) its patch count, 0 elsewhere;
    - ``parent`` (..., L, n) int32: at a root of level l < L-1 the level-(l+1) island holding most of its patches (ties
      to the smaller label), -1 elsewhere and at level L-1;
    - ``containment`` (..., L, n) fp32: that overlap / size where ``parent >= 0``, else 0;
    - ``nested`` (..., L-1) fp32: share of patches whose level-l island lies wholly inside one level-(l+1) island;
    - with ``embeddings=True``, else None: ``embedding`` (..., L, n, d) fp32, at a root the mean of its members'
      level-l vectors (a patch's island vector is ``embedding[..., l, labels[..., l, i], :]``), 0 elsewhere;
      ``member_cos`` (..., L, n) each patch's cosine with its island's embedding; ``coherence`` (..., L, n) at a root
      the mean of its members' ``member_cos``, 0 elsewhere.

    Every output is bit-reproducible.  Nothing is read back to the host, so the call can be captured in a CUDA graph;
    under torch.compile it is the ``glom_b200::parse_tree`` op.  No gradient flows through it."""
    lead, n, L, d, side_h, side_w = _geometry(states, grid)
    if torch.compiler.is_compiling():
        out = torch.ops.glom_b200.parse_tree(states.detach(), side_h, side_w, float(threshold), bool(embeddings))
        return ParseTree(*out[:6], *(out[6:] if embeddings else (None,) * 3))
    x = _f32(states)                       # the kernels load float4
    isl = islands(x, grid=(side_h, side_w), threshold=threshold)
    slabs = 1
    for v in lead:
        slabs *= v
    dev = x.device
    shape = (*lead, L, n)
    size = torch.empty(shape, dtype=torch.int32, device=dev)
    parent = torch.empty(shape, dtype=torch.int32, device=dev)
    containment = torch.empty(shape, dtype=torch.float32, device=dev)
    nested = torch.empty((*lead, L - 1), dtype=torch.float32, device=dev)
    emb = member_cos = coherence = None
    if embeddings:
        emb = torch.empty((*lead, L, n, d), dtype=torch.float32, device=dev)
        member_cos = torch.empty(shape, dtype=torch.float32, device=dev)
        coherence = torch.empty(shape, dtype=torch.float32, device=dev)

    def ptr(t):
        return t.data_ptr() if t is not None and t.numel() else None
    with torch.cuda.device(dev):
        _native.island_tree(isl.labels.data_ptr(), x.data_ptr() if embeddings else None, slabs, n, L, d, ptr(size),
                            ptr(parent), ptr(containment), ptr(nested), ptr(emb), ptr(member_cos), ptr(coherence),
                            torch.cuda.current_stream(dev).cuda_stream)
    return ParseTree(isl.labels, isl.num_islands, size, parent, containment, nested, emb, member_cos, coherence)
