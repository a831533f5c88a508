"""CPU oracle for the GLOM column update  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline /
``--impl reference`` legs may import this module.  The product path
(``glom_pytorch_b200``) never imports it and fails loudly without its CUDA library.

What it restates (all citations relative to the reference checkout,
``glom_pytorch/glom_pytorch.py``):

* ``grouped_ff``      <- GroupedFeedForward (:23-36): per-level 2-layer MLP, the
                         grouped 1x1 Conv1d (:29, :31) written as per-group matmuls;
                         nn.GELU() (:30) is the exact erf form.
* ``consensus``       <- ConsensusAttention.forward (:56-73): F.normalize eps=1e-12
                         (:58), scale d**-0.5 (:60), diagonal fill -5e-4 (:11, :62-65)
                         applied BEFORE the radius mask (:67-69), softmax (:71), P.V (:72).
* ``radius_mask``     <- ConsensusAttention.__init__ (:44-54): meshgrid 'ij', (h w) order.
* ``tokenize``        <- image_to_tokens (:94-97): 'b c (h p1) (w p2) -> b (h w) (p1 p2 c)'.
* ``glom_forward``    <- Glom.forward (:110-150): S_0 (:123-124), contributions 4..4,3
                         (:128-129), the Jacobi loop (:131-145), return_all (:147-148).

Parity pinning: the reference ships NO tests or golden vectors, so
this oracle is pinned against outputs of the live reference itself: the fixtures in
``tests/golden/*.npz`` were produced by ``tests/golden/make_golden.py`` importing
``/root/reference`` in the build container; ``tests/test_oracle_golden.py`` checks
this file against every one of them (fp64 oracle vs fp32 reference <= 2e-5 max-abs).

Arithmetic is numpy; ``dtype`` selects float32/float64.  ``emulate='bf16'`` rounds the
tensor-core operands to bfloat16 (round-to-nearest-even) exactly where the bf16 engine
does, to give a tight prediction of the engine's own output for diagnostics.
"""
from __future__ import annotations

import math
import numpy as np

try:  # scipy is in the image; fall back to math.erf (slow) if it ever is not
    from scipy.special import erf as _erf
except Exception:  # pragma: no cover
    _erf = np.vectorize(math.erf, otypes=[np.float64])

TOKEN_ATTEND_SELF_VALUE = -5e-4  # glom_pytorch.py:11


# ----------------------------------------------------------------------------- helpers
def bf16_round(x: np.ndarray) -> np.ndarray:
    """Round float32 values to the nearest bfloat16 (ties to even); returns float32."""
    a = np.ascontiguousarray(x, dtype=np.float32)
    u = a.view(np.uint32).astype(np.uint64)
    lsb = (u >> 16) & 1
    u = (u + 0x7FFF + lsb) & 0xFFFF0000
    out = u.astype(np.uint32).view(np.float32).reshape(a.shape)
    # NaN stays NaN (not produced by these paths); inf stays inf.
    return out


_POOL = None


def _gelu_block(x):
    return (0.5 * x * (1.0 + _erf(x * x.dtype.type(1.0 / math.sqrt(2.0))))).astype(x.dtype)


def gelu_erf(x: np.ndarray) -> np.ndarray:
    """nn.GELU() default = 0.5 x (1 + erf(x / sqrt 2))   (glom_pytorch.py:30).
    Large inputs are split over a thread pool (the erf ufunc releases the GIL) so that the CPU port
    used as bench.py's baseline is not single-threaded in its second-largest cost."""
    global _POOL
    if x.ndim != 2 or x.shape[0] < 512:
        return _gelu_block(x)
    import os
    from concurrent.futures import ThreadPoolExecutor
    nthreads = min(32, os.cpu_count() or 1)
    if _POOL is None:
        _POOL = ThreadPoolExecutor(max_workers=nthreads)
    out = np.empty_like(x)
    step = -(-x.shape[0] // nthreads)

    def work(i):
        out[i:i + step] = _gelu_block(x[i:i + step])
    list(_POOL.map(work, range(0, x.shape[0], step)))
    return out


def synth_params(dim, levels, image_size, patch_size, seed=0, dtype=np.float32):
    """Deterministic synthetic parameters with the reference's shapes and default-init
    scales (SURVEY.md 3.4), keyed exactly like ``Glom.state_dict()``.
    Uses numpy's PCG64 so fixtures do not depend on torch's RNG stream."""
    rng = np.random.default_rng(seed)
    L, d = levels, dim
    side = image_size // patch_size
    N = side * side
    pdim = 3 * patch_size * patch_size

    def unif(shape, fan_in):
        b = 1.0 / math.sqrt(fan_in)
        return rng.uniform(-b, b, size=shape).astype(dtype)

    p = {
        "init_levels": rng.standard_normal((L, d)).astype(dtype),
        "image_to_tokens.1.weight": unif((d, pdim), pdim),
        "image_to_tokens.1.bias": unif((d,), pdim),
        "pos_emb.weight": rng.standard_normal((N, d)).astype(dtype),
        "bottom_up.net.1.weight": unif((L * 4 * d, d, 1), d),
        "bottom_up.net.1.bias": unif((L * 4 * d,), d),
        "bottom_up.net.3.weight": unif((L * d, 4 * d, 1), 4 * d),
        "bottom_up.net.3.bias": unif((L * d,), 4 * d),
    }
    if L > 1:
        p.update({
            "top_down.net.1.weight": unif(((L - 1) * 4 * d, d, 1), d),
            "top_down.net.1.bias": unif(((L - 1) * 4 * d,), d),
            "top_down.net.3.weight": unif(((L - 1) * d, 4 * d, 1), 4 * d),
            "top_down.net.3.bias": unif(((L - 1) * d,), 4 * d),
        })
    return p


# ----------------------------------------------------------------------------- operators
def tokenize(img: np.ndarray, w: np.ndarray, b: np.ndarray, patch_size: int, emulate=None) -> np.ndarray:
    """image_to_tokens (:94-97, call :114). img (B,3,H,W) -> (B, n, d).
    emulate='bf16': operands rounded to bf16 as the engine's tensor-core tokeniser (and autocast) does."""
    B, C, H, W = img.shape
    p = patch_size
    h, wd = H // p, W // p
    x = img.reshape(B, C, h, p, wd, p)            # b c h p1 w p2
    x = x.transpose(0, 2, 4, 3, 5, 1)             # b h w p1 p2 c
    x = x.reshape(B, h * wd, p * p * C)
    if emulate == "bf16":
        return (bf16_round(x) @ bf16_round(w).T + b.astype(np.float32)).astype(img.dtype)
    return x @ w.T + b


def grouped_ff(x: np.ndarray, w1, b1, w2, b2, emulate=None) -> np.ndarray:
    """GroupedFeedForward.forward (:35) on x (B, n, G, d) -> (B, n, G, d).
    Conv1d(groups=G, k=1) weights (G*4d, d, 1)/(G*d, 4d, 1): group g owns output rows
    [g*4d, (g+1)*4d) of w1 and [g*d, (g+1)*d) of w2 (:29, :31)."""
    B, n, G, d = x.shape
    h = 4 * d
    w1 = w1.reshape(G, h, d)
    w2 = w2.reshape(G, d, h)
    b1 = b1.reshape(G, h)
    b2 = b2.reshape(G, d)
    out = np.empty_like(x)
    for g in range(G):
        a = x[:, :, g, :].reshape(B * n, d)
        W1, W2 = w1[g], w2[g]
        if emulate == "bf16":
            a, W1, W2 = bf16_round(a), bf16_round(W1), bf16_round(W2)
        hid = gelu_erf((a @ W1.T + b1[g]).astype(x.dtype))
        if emulate == "bf16":
            hid = bf16_round(hid)
        out[:, :, g, :] = (hid @ W2.T + b2[g]).reshape(B, n, d)
    return out


def radius_mask(side: int, radius: float) -> np.ndarray:
    """non_local_mask (:44-54): True where the Euclidean grid distance exceeds radius.
    Patch index i = h*side + w ('ij' meshgrid, '(h w) c')."""
    hh, ww = np.meshgrid(np.arange(side), np.arange(side), indexing="ij")
    co = np.stack([hh.reshape(-1), ww.reshape(-1)], -1).astype(np.float32)
    d2 = ((co[:, None, :] - co[None, :, :]) ** 2).sum(-1)
    dist = np.sqrt(d2.astype(np.float32))          # cdist in fp32 (:51)
    return dist > np.float32(radius)


def consensus(levels: np.ndarray, attend_self: bool, mask, emulate=None) -> np.ndarray:
    """ConsensusAttention.forward (:56-73). levels (B, n, L, d) -> (B, n, L, d)."""
    B, n, L, d = levels.shape
    dt = levels.dtype
    q = levels
    norm = np.sqrt((levels.astype(np.float64) ** 2).sum(-1, keepdims=True))
    k = (levels / np.maximum(norm, 1e-12)).astype(dt)        # F.normalize (:58)
    v = levels
    if emulate == "bf16":
        # engine: Gram of the bf16 state, column-scaled by the fp32 reciprocal norm
        qb = bf16_round(q)
        qt = qb.transpose(0, 2, 1, 3)
        g = qt @ qt.transpose(0, 1, 3, 2)
        rinv = (1.0 / np.maximum(norm, 1e-12))[..., 0]       # (B, n, L)
        sim = g * rinv.transpose(0, 2, 1)[:, :, None, :] * (d ** -0.5)
        v = qb
    else:
        sim = (q.transpose(0, 2, 1, 3) @ k.transpose(0, 2, 3, 1)) * (d ** -0.5)   # (:60) 'b i l d, b j l d -> b l i j'
    sim = sim.astype(dt)
    if not attend_self:                                       # (:62-65)
        idx = np.arange(n)
        sim[:, :, idx, idx] = TOKEN_ATTEND_SELF_VALUE
    if mask is not None:                                      # (:67-69)
        sim = np.where(mask[None, None], -np.finfo(dt).max, sim)
    sim = sim - sim.max(-1, keepdims=True)
    e = np.exp(sim)
    if emulate == "bf16":
        # engine: unnormalised bf16 probabilities, fp32 row sum of the unrounded ones
        out = (bf16_round(e) @ v.transpose(0, 2, 1, 3)).transpose(0, 2, 1, 3) / \
            e.sum(-1).transpose(0, 2, 1)[..., None]
        return bf16_round(out.astype(np.float32)).astype(dt)
    attn = e / e.sum(-1, keepdims=True)                       # (:71)
    return (attn @ v.transpose(0, 2, 1, 3)).transpose(0, 2, 1, 3).astype(dt)  # (:72) 'b l i j, b j l d -> b i l d'


# ----------------------------------------------------------------------------- the path
def glom_forward(params, img, *, patch_size, iters=None, levels=None, return_all=False,
                 consensus_self=False, local_consensus_radius=0, image_size=None,
                 dtype=np.float64, emulate=None, tokens=None):
    """Glom.forward (:110-150).  ``params`` uses the reference state_dict keys.

    Returns S_T (B, n, L, d) or stack(S_0..S_T) (T+1, B, n, L, d) when ``return_all``.
    ``tokens`` may be given instead of ``img`` to start after image_to_tokens.
    """
    P = {k: np.asarray(v, dtype=dtype) for k, v in params.items()
         if k != "attention.non_local_mask"}
    L, d = P["init_levels"].shape
    if tokens is None:
        tokens = tokenize(np.asarray(img, dtype=dtype), P["image_to_tokens.1.weight"],
                          P["image_to_tokens.1.bias"], patch_size, emulate)   # (:114)
    else:
        tokens = np.asarray(tokens, dtype=dtype)
    B, n, _ = tokens.shape
    iters = 2 * L if iters is None else iters                            # (:112)
    pos = P["pos_emb.weight"][:n][None, :, None, :]                      # (:117-118)
    bottom = tokens[:, :, None, :]                                       # (:121)
    if levels is None:
        levels = np.broadcast_to(P["init_levels"], (B, n, L, d)).copy()  # (:123-124)
    else:
        levels = np.asarray(levels, dtype=dtype).copy()
    mask = None
    if local_consensus_radius > 0:
        side = int(round(math.sqrt(P["pos_emb.weight"].shape[0]))) if image_size is None \
            else image_size // patch_size
        mask = radius_mask(side, local_consensus_radius)
    hiddens = [levels]
    contrib = np.full((L,), 4.0, dtype=dtype)                            # (:128)
    contrib[-1] = 3.0                                                    # (:129)
    for _ in range(iters):                                               # (:131)
        lwi = np.concatenate([bottom, levels], axis=-2)                  # (:132)
        bu = grouped_ff(lwi[..., :-1, :], P["bottom_up.net.1.weight"],
                        P["bottom_up.net.1.bias"], P["bottom_up.net.3.weight"],
                        P["bottom_up.net.3.bias"], emulate)              # (:134)
        td = np.zeros_like(levels)                                       # (:137) zero top
        if L > 1:
            td_in = lwi[..., 2:, :] + pos                                # (:136)
            td[..., :-1, :] = grouped_ff(td_in, P["top_down.net.1.weight"],
                                         P["top_down.net.1.bias"],
                                         P["top_down.net.3.weight"],
                                         P["top_down.net.3.bias"], emulate)
        cons = consensus(levels, consensus_self, mask, emulate)          # (:139)
        levels = (levels + bu + td + cons) / contrib[None, None, :, None]  # (:141-142)
        hiddens.append(levels)                                           # (:145)
    if return_all:
        return np.stack(hiddens)                                         # (:147-148)
    return levels                                                        # (:150)
