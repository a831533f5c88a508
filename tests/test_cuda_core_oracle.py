"""The CUDA-core path against float64 at dims, patch sizes and depths off the tensor-core grid.

precision="fp32" runs the column update on CUDA cores (simt_kernels.cu: `sgemm_kernel` for FF1, FF2 and the tokeniser,
`attn_f32_kernel` for the consensus) and the whole backward in bwd_kernels.cu, which the bf16 engine also takes when
dim % 256 != 0.  The engine accepts any dim % 4 == 0, levels >= 2 and patch size that divides the image, and every dim
off the 64-grid runs on this path alone.  Each quantity is compared with a float64 reference fed the engine's own
tokens and states, so rounding carried in from earlier steps drops out:
  forward   S_{t+1} vs `column_step`, H (workspace buffer 0, fp32 (R, G, 4d)) vs `hidden_activations`, C (buffer 1,
            fp32 (B, n, L, d)) vs `_consensus`, one step and chains of 3 (with and without return_all, carried state and
            init_levels), iters = 0;
  backward  every gradient vs `grads_at_states` + `token_grads`, one step and chains of 3, with and without
            torch.use_deterministic_algorithms (then three runs must be bit-identical);
  tokeniser fp32 (MODE_TOK) and tensor-core forward vs float64 `patchify(img) W^T + b`; its backward through
            `_Tokenize.apply` with each subset of (image, weight, bias) vs `token_grads`.

Metric (`errors`): each tensor is cut into the blocks of the CUDA-core launches -- S_{t+1} per (64-row, level, 64-column)
FF2 tile, H per (group, 64-row, 64-column) FF1 tile, C per (image, level, 16-query) attention block, tokens per 64 x 64
tile; weight gradients per (group, 64 x 64 gemm_f32 tile), biases per (group, 32-column colsum strip), d_levels per
(image, level), d_pos per 64-row block (rows >= n exactly zero), d_init per level, d_img per (image, channel) -- and each
block's rel-Frobenius error is taken against max(|ref block|, FLOOR * rms block norm of the tensor).  `rel` is the worst
block, `abs` the worst max-abs error over the tensor's max |ref|.

Bounds (rel, abs), over all the GPU tests of the path on one H100 80GB HBM3 (700 W power limit); observed maxima in
brackets:
  simt      fp32 S_{t+1} vs column_step: test_forward_oracle's bound      (8e-7, 1.2e-6)   [rel 4.5e-7, abs 8.3e-7,
                                                                                            both d132_L2, p = 1]
  simt_H    fp32 H vs hidden_activations, about 3x the maximum            (1e-6, 2.2e-6)   [rel 3.1e-7, abs 7.2e-7]
  simt_C    fp32 C vs _consensus, about 3x the maximum                    (8e-7, 1.1e-6)   [rel 2.6e-7, abs 3.7e-7]
  tok32     fp32 tokens vs patchify W^T + b, about 3x the maximum         (1.6e-6, 3.2e-6) [rel 5.4e-7, abs 1.05e-6,
                                                                                            both at p = 16, K = 768]
  tok       tensor-core tokens vs the bf16-operand tokeniser: test_forward_oracle's bound
                                                                          (1.5e-6, 3e-6)   [rel 6.9e-7, abs 8.4e-7]
  bwd       CUDA-core backward and the tokeniser backward vs float64: test_backward_oracle's simt bound
                                                                          (3e-6, 6e-6)     [rel 7.0e-7, abs 1.24e-6]
  emu, tc   the two bf16 rows' forward: test_forward_oracle's bounds      [S_1 vs column_step rel 1.1e-3; abs 4.1e-3
                                                                           vs step_forward_bf16, both at G = 23]
  tc_bwd    the G = 23 row's tensor-core backward: test_backward_oracle's tc bound
                                                                          (2e-2, 3.5e-2)   [rel 5.7e-3, abs 4.6e-3]
One finding: the fp32 consensus summed P.V in one running fp32 sum over all n keys.  From init_levels every key of a
level is equal, the rounding errors of that sum add up coherently, and the error of S_1 grew linearly with n: rel 2.7e-6
at n = 729 and 1.4e-5 at n = 3600 (simt bound 8e-7).  attn_f32_kernel now sums blocks of 32 keys into a compensated
total; both shapes are within the simt bound.  The faults of test_bounds_catch_faults miss the bounds their GPU tests
assert by 3x at least (the margins are printed, all above 10^4 x).
"""
import ctypes
import math

import pytest
import torch

from oracle import glom_oracle as O
from oracle import glom_oracle_torch as OT

import test_backward_oracle as BO
import test_deterministic_backward as TD
import test_forward_oracle as FO

DEV = "cuda:0"
FLOOR = 0.1
TOL = {"simt": FO.TOL["simt"], "simt_H": (1e-6, 2.2e-6), "simt_C": (8e-7, 1.1e-6), "tok32": (1.6e-6, 3.2e-6),
       "tok": FO.TOL["tok"], "emu": FO.TOL["emu"], "tc": FO.TOL["tc"], "bwd": BO.TOL["simt"], "tc_bwd": BO.TOL["tc"]}
FWD_TOL = {"state": TOL["simt"], "H": TOL["simt_H"], "C": TOL["simt_C"]}
ATTN_F32_MAX_DIM_PLUS_N = 3632        # 227 KB of shared memory / (16 queries x 4 bytes)


# ----------------------------------------------------------------------------- metric
def _tiles(x, rows, cols):
    """64 x 64 (rows x cols) tiles of the last two dims of a 2-D x."""
    return [x[r:r + rows, c:c + cols] for r in range(0, x.shape[0], rows) for c in range(0, x.shape[1], cols)]


def _blocks(key, x, meta):
    """-> list of blocks of x (float64 CPU) along the CUDA-core launches; meta = (B, n, L, d)."""
    B, n, L, d = meta
    if key == "state":                                                       # FF2 tiles
        x = x.reshape(B * n, L, d)
        return [b for l in range(L) for b in _tiles(x[:, l], 64, 64)]
    if key == "H":                                                           # FF1 tiles
        return [b for g in range(x.shape[0]) for b in _tiles(x[g], 64, 64)]
    if key == "C":                                                           # attention blocks
        return [x[b, i:i + 16, l] for b in range(B) for l in range(L) for i in range(0, n, 16)]
    if key == "tokens":                                                      # MODE_TOK tiles
        return _tiles(x.reshape(-1, x.shape[-1]), 64, 64)
    if key == "d_levels":                                                    # per (image, level)
        return [x[b, :, l] for b in range(x.shape[0]) for l in range(L)]
    if key == "init_levels":                                                 # per level
        return list(x)
    if key == "d_img":                                                       # per (image, channel)
        return [x[b, c] for b in range(x.shape[0]) for c in range(x.shape[1])]
    if key == "pos_emb.weight":
        return [x[r:min(r + 64, n)] for r in range(0, n, 64)]
    if key == "image_to_tokens.1.bias":
        return [x[c:c + 32] for c in range(0, x.shape[0], 32)]
    if key == "image_to_tokens.1.weight":
        return _tiles(x, 64, 64)
    G = L if key.startswith("bottom_up") else L - 1
    if key.endswith("bias"):                                                 # per (group, 32-column strip)
        x = x.reshape(G, -1)
        return [x[g, c:c + 32] for g in range(G) for c in range(0, x.shape[1], 32)]
    w = x.reshape(G, x.shape[0] // G, x.shape[1])                            # per (group, gemm_f32 tile)
    return [b for g in range(G) for b in _tiles(w[g], 64, 64)]


def errors(got, ref, meta):
    """-> {key: (worst block rel-Frobenius, max-abs / max |ref|)} for the keys of `ref`."""
    n = meta[1]
    out = {}
    for k, r in ref.items():
        g = torch.as_tensor(got[k]).detach().to("cpu", torch.float64)
        r = torch.as_tensor(r).to("cpu", torch.float64)
        assert g.shape == r.shape, (k, tuple(g.shape), tuple(r.shape))
        assert torch.isfinite(g).all(), k
        if k == "pos_emb.weight":
            assert not g[n:].any(), "d_pos rows >= n must be exactly zero"
        gb, rb = _blocks(k, g, meta), _blocks(k, r, meta)
        rms = float(torch.linalg.norm(r)) / math.sqrt(len(rb))
        rel = max(float(torch.linalg.norm(a - b)) / max(float(torch.linalg.norm(b)), FLOOR * rms, 1e-300)
                  for a, b in zip(gb, rb))
        ab = float((g - r).abs().max()) / max(float(r.abs().max()), 1e-300)
        out[k] = (rel, ab)
    return out


def check(errs, tol, what):
    """tol: one (rel, abs) pair, or {key: (rel, abs)}."""
    bad = {k: e for k, e in errs.items()
           if e[0] > (tol[k] if isinstance(tol, dict) else tol)[0] or e[1] > (tol[k] if isinstance(tol, dict) else tol)[1]}
    assert not bad, (what, tol, bad)


def _report(name, what, errs):
    print(f"[cuda-core-oracle] {name} {what}: " + " ".join(f"{k}=({e[0]:.2e},{e[1]:.2e})" for k, e in errs.items()))


# ----------------------------------------------------------------------------- shapes
# name: dim, levels, (H, W), patch, batch, Glom kwargs, precision, backward tested.  Each row's comment names what it
# reaches (R = B n rows; k3 = 3 p^2, the tokeniser's K).
SHAPES = {
    # d < 32 (most lanes of attn_f32 / normalize_rows hold zeros through the shuffles), one partial k-block of FF1 (K = 4),
    # d / 4 = 1 in scale_by_contrib, R = 27 < 32 (colsum, init_grad), L d = 8
    "d4_L2_12x12_p4_B3": (4, 2, (12, 12), 4, 3, {}, "fp32", True),
    # FF1 K tail 12 (< 16), k3 = 27, a non-square image (5 x 7 patches, n = 35 of 49 pos rows), d / 4 = 3
    "d12_L3_15x21_p3_B2": (12, 3, (15, 21), 3, 2, {}, "fp32", True),
    # d % 16 = 4 (FF1 k tail), 4d = 144 (a partial FF1 N tile), d = 36 < 64 (partial N tiles of FF2 and gemm_f32),
    # k3 = 75, d / 4 = 9, radius mask with attend_self, L = 5
    "d36_L5_40x40_p5_r2.5_self": (36, 5, (40, 40), 5, 2, dict(local_consensus_radius=2.5, consensus_self=True), "fp32",
                                  True),
    # attention opts in to 64 (100 + 729) = 53 KB of shared memory, n % 16 = 9 (a partial last query tile), R = 729
    # (R mod 32 = 25, R mod 64 = 25), softmax rows of 729 keys
    "d100_L3_54x54_p2_B1": (100, 3, (54, 54), 2, 1, {}, "fp32", True),
    # p = 1 (k3 = 3), R = 585 rows, d = 132 (FF2 N tiles 64 + 64 + 4, 4d = 528), n = 117 of 169 pos rows, d / 4 = 33
    "d132_L2_9x13_p1_B5": (132, 2, (9, 13), 1, 5, {}, "fp32", True),
    # G = 31 groups on the fp32 engine (L = 16)
    "d12_L16_16x16_p4_B2": (12, 16, (16, 16), 4, 2, {}, "fp32", True),
    # d + n = 3632: the fp32 consensus limit exactly, 227 KB of shared memory (forward only)
    "d32_L2_240x240_p4_B1": (32, 2, (240, 240), 4, 1, {}, "fp32", False),
    # G = 23 on the tensor-core K1 / K2 / attention and the BW_* backward (dim % 256 == 0, n % 8 == 0)
    "d256_L12_32x32_p4_bf16": (256, 12, (32, 32), 4, 2, {}, "bf16", True),
    # smallest bf16 dim: tensor-core forward, wholly CUDA-core backward (dim % 256 != 0), n = 49 (n % 8 != 0)
    "d64_L3_28x28_p4_bf16": (64, 3, (28, 28), 4, 2, {}, "bf16", True),
}
FP32_SHAPES = [k for k, v in SHAPES.items() if v[6] == "fp32"]
BF16_SHAPES = [k for k, v in SHAPES.items() if v[6] == "bf16"]
BWD_SHAPES = [k for k, v in SHAPES.items() if v[7]]


def _model(name, seed=0):
    dim, L, hw, p, B, kw, precision, _ = SHAPES[name]
    import glom_pytorch_b200 as G
    isz = max(hw)
    params = O.synth_params(dim, L, isz, p, seed=seed)
    m = G.Glom(dim=dim, levels=L, image_size=isz, patch_size=p, precision=precision, **kw)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=False)
    m = m.to(DEV)
    n = (hw[0] // p) * (hw[1] // p)
    g = torch.Generator().manual_seed(seed + 41)
    img = torch.randn((B, 3) + hw, generator=g)
    S = torch.randn(B, n, L, dim, generator=g)
    return m, img, S, n, g


def _f32_engine(m, img, S, iters):
    """forward(iters) of the fp32 engine from S (None: init_levels) -> (S_iters, H (G, R, 4d), C (B, n, L, d)), H and C of
    the last step read from workspace buffers 0 and 1 (row-major fp32)."""
    from glom_pytorch_b200 import _native
    with torch.no_grad():
        out = m(img.to(DEV), iters=iters, levels=None if S is None else S.to(DEV))
    torch.cuda.synchronize()
    B, n, L, d = out.shape
    cfg, ws = m.engine_cfg(n), m._workspace

    def buf(which):
        off, nb = _native.workspace_offset(cfg, B, iters, False, which)
        return ws[off:off + nb].view(torch.float32)
    H = buf(0).reshape(B * n, 2 * L - 1, 4 * d).permute(1, 0, 2).cpu()
    C = buf(1).reshape(B, n, L, d).cpu()
    return out.cpu(), H, C


def _f32_refs(m, tok, P, pos, mask, S):
    S = OT._f64(S)
    return {"state": FO._exact(m, tok, P, pos, mask, S), "H": OT.hidden_activations(P, tok, pos, S),
            "C": OT._consensus(S, m.attention.attend_self, mask)}


# ----------------------------------------------------------------------------- CPU: the references
def _small(d, L, isz, p, B, seed=1):
    P = {k: torch.from_numpy(v).double() for k, v in O.synth_params(d, L, isz, p, seed=seed).items()}
    n = (isz // p) ** 2
    g = torch.Generator().manual_seed(seed)
    tok = torch.randn(B, n, d, generator=g, dtype=torch.float64)
    S = torch.randn(B, n, L, d, generator=g, dtype=torch.float64)
    return P, tok, P["pos_emb.weight"][:n].clone(), S, g


@pytest.mark.parametrize("d,L", [(4, 2), (12, 3), (36, 5), (12, 16)])
def test_hidden_activations_give_column_step(d, L):
    """hidden_activations in the engine's group order, through the second layers, plus the consensus, is column_step."""
    P, tok, pos, S, _ = _small(d, L, 16, 4, 2)
    H = OT.hidden_activations(P, tok, pos, S)
    B, n = S.shape[:2]
    w2bu = P["bottom_up.net.3.weight"].reshape(L, d, 4 * d)
    w2td = P["top_down.net.3.weight"].reshape(L - 1, d, 4 * d)
    b2 = P["bottom_up.net.3.bias"].reshape(L, d).clone()
    b2[:-1] += P["top_down.net.3.bias"].reshape(L - 1, d)
    contrib = torch.full((L,), 4.0, dtype=torch.float64)
    contrib[-1] = 3.0
    got = OT._fwd_k2(S, H, OT._consensus(S, False, None), w2bu, w2td, b2, contrib)
    want = OT.column_step(S, tok, pos, P, None, False)
    assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max())


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_blocks_partition_every_tensor(name):
    """Every element of every compared tensor lies in exactly one block of the metric (no tile escapes the check)."""
    dim, L, hw, p, B, _, _, _ = SHAPES[name]
    n = (hw[0] // p) * (hw[1] // p)
    G, k3 = 2 * L - 1, 3 * p * p
    meta = (B, n, L, dim)
    shapes = {"state": (B, n, L, dim), "H": (G, B * n, 4 * dim), "C": (B, n, L, dim), "tokens": (B, n, dim),
              "d_levels": (B, n, L, dim), "init_levels": (L, dim), "d_img": (B, 3) + hw, "pos_emb.weight": (n, dim),
              "image_to_tokens.1.bias": (dim,), "image_to_tokens.1.weight": (dim, k3),
              "bottom_up.net.1.weight": (L * 4 * dim, dim, 1), "bottom_up.net.3.weight": (L * dim, 4 * dim, 1),
              "top_down.net.1.bias": ((L - 1) * 4 * dim,), "top_down.net.3.bias": ((L - 1) * dim,)}
    for k, s in shapes.items():
        x = torch.arange(math.prod(s), dtype=torch.float64).reshape(s)
        seen = torch.cat([b.reshape(-1) for b in _blocks(k, x, meta)])
        assert torch.equal(seen.sort().values, x.reshape(-1)), k


# ----------------------------------------------------------------------------- CPU: the bounds catch faults
def _consensus_key_norm_cols(levels, attend_self, mask, cols):
    """_consensus with each key normalised by the norm of its first `cols` columns only."""
    B, n, L, d = levels.shape
    q = levels.permute(0, 2, 1, 3)
    k = (levels / levels[..., :cols].norm(dim=-1, keepdim=True).clamp_min(1e-12)).permute(0, 2, 1, 3)
    sim = (q @ k.transpose(-1, -2)) * d ** -0.5
    if not attend_self:
        sim = sim.masked_fill(torch.eye(n, dtype=torch.bool)[None, None], OT.TOKEN_ATTEND_SELF_VALUE)
    if mask is not None:
        sim = sim.masked_fill(mask[None, None], -torch.finfo(sim.dtype).max)
    return (sim.softmax(-1) @ q).permute(0, 2, 1, 3)


def _patchify_channel_major(img, p):
    """'b c (h p1) (w p2) -> b (h w) (c p1 p2)': the patch vector in the wrong order."""
    B, C, H, W = img.shape
    return img.reshape(B, C, H // p, p, W // p, p).permute(0, 2, 4, 1, 3, 5).reshape(B, (H // p) * (W // p), C * p * p)


def _shape_inputs(name, seed=3):
    """float64 parameters, tokens, positions, state and mask at a GPU-test shape."""
    dim, L, hw, p, B, kw, _, _ = SHAPES[name]
    isz = max(hw)
    P = {k: torch.from_numpy(v).double() for k, v in O.synth_params(dim, L, isz, p, seed=seed).items()}
    n = (hw[0] // p) * (hw[1] // p)
    g = torch.Generator().manual_seed(seed)
    img = torch.randn((B, 3) + hw, generator=g, dtype=torch.float64)
    tok = OT.patchify(img, p) @ P["image_to_tokens.1.weight"].T + P["image_to_tokens.1.bias"]
    S = torch.randn(B, n, L, dim, generator=g, dtype=torch.float64)
    radius = kw.get("local_consensus_radius", 0)
    mask = OT.radius_mask(isz // p, radius) if radius else None
    return P, img, tok, P["pos_emb.weight"][:n].clone(), S, mask, kw.get("consensus_self", False), g


def _fault_forward(name, fault):
    P, _, tok, pos, S, mask, attend_self, _ = _shape_inputs(name)
    B, n, L, d = S.shape
    if fault == "ff1_drops_k_tail":                        # FF1 sums k < 16 floor(d / 16) only
        kt = 16 * (d // 16)
        cut = lambda x: torch.cat([x[..., :kt], torch.zeros_like(x[..., kt:])], -1)   # noqa: E731
        return "H", OT.hidden_activations(P, tok, pos, S), OT.hidden_activations(P, cut(tok), cut(pos), cut(S))
    if fault == "ff1_last_n_tile_zero":                    # H's last partial 64-column tile never written
        good = OT.hidden_activations(P, tok, pos, S)
        bad = good.clone()
        bad[:, :, 64 * (4 * d // 64):] = 0
        return "H", good, bad
    if fault == "attn_drops_last_query_tile":              # no block for the last partial 16-query tile
        good = OT._consensus(S, attend_self, mask)
        bad = good.clone()
        bad[:, 16 * (n // 16):] = 0
        return "C", good, bad
    if fault == "key_norm_first_32_columns":               # the key norm summed over c < 32 only
        return "C", OT._consensus(S, attend_self, mask), _consensus_key_norm_cols(S, attend_self, mask, 32)
    if fault == "top_level_divided_by_4":                  # every level scaled by 1/4 (the top level's 1/3 lost)
        good = OT.column_step(S, tok, pos, P, mask, attend_self)
        bad = good.clone()
        bad[:, :, -1] *= 0.75
        return "state", good, bad
    raise KeyError(fault)


def _fault_backward(name, fault):
    P, img, tok, pos, S, mask, attend_self, g = _shape_inputs(name)
    B, n, L, d = S.shape
    cot = torch.randn(S.shape, generator=g, dtype=torch.float64)
    states = torch.stack([S, S])
    kw = dict(return_all=False, attend_self=attend_self, mask=mask)
    good = OT.grads_at_states(P, tok, pos, states, cot, **kw)
    if fault == "b2_colsum_drops_last_rows":               # the second-layer bias sums skip the last R mod 32 rows
        R = B * n
        contrib = torch.full((L,), 4.0, dtype=torch.float64)
        contrib[-1] = 3.0
        drop = (cot / contrib[:, None]).reshape(R, L, d)[32 * (R // 32):].sum(0)
        bad = dict(good)
        bad["bottom_up.net.3.bias"] = good["bottom_up.net.3.bias"] - drop.reshape(-1)
        bad["top_down.net.3.bias"] = good["top_down.net.3.bias"] - drop[:-1].reshape(-1)
        keys = ("bottom_up.net.3.bias", "top_down.net.3.bias")
    elif fault == "bwd_top_level_divided_by_4":            # scale_by_contrib with 1/4 on the top level too
        cot_bad = cot.clone()
        cot_bad[:, :, -1] *= 0.75
        bad = OT.grads_at_states(P, tok, pos, states, cot_bad, **kw)
        keys = ("d_state0",) + OT.MLP_KEYS
    else:
        raise KeyError(fault)
    rename = {"d_state0": "d_levels"}
    return ({rename.get(k, k): good[k] for k in keys}, {rename.get(k, k): bad[k] for k in keys})


def _fault_tokeniser(name, fault):
    P, img, _, _, S, _, _, g = _shape_inputs(name)
    B, n, _, d = S.shape
    w, b = P["image_to_tokens.1.weight"], P["image_to_tokens.1.bias"]
    p = SHAPES[name][3]
    if fault == "patches_channel_major":                   # MODE_TOK / patchify reading (c, p1, p2)
        return "tokens", OT.patchify(img, p) @ w.T + b, _patchify_channel_major(img, p) @ w.T + b
    cot = torch.randn(B, n, d, generator=g, dtype=torch.float64)
    good = OT.token_grads(img, w, b, p, cot)
    if fault == "unpatchify_p1_p2_swapped":                # the fold writes patch element (p1, p2) to (p2, p1)
        Bi, C, H, W = img.shape
        bad = good["d_img"].reshape(Bi, C, H // p, p, W // p, p).transpose(3, 5).reshape(Bi, C, H, W)
        return "d_img", good["d_img"], bad
    if fault == "token_bias_colsum_drops_last_rows":       # d_bias skips the last R mod 32 rows
        R = B * n
        bad = cot.reshape(R, d)[:32 * (R // 32)].sum(0)
        return "image_to_tokens.1.bias", good["image_to_tokens.1.bias"], bad
    raise KeyError(fault)


# fault -> (kind, GPU-test shape where the faulty part carries weight, the bound of the GPU test that sees it)
FAULTS = {
    "ff1_drops_k_tail": ("forward", "d36_L5_40x40_p5_r2.5_self", "simt_H"),
    "ff1_last_n_tile_zero": ("forward", "d36_L5_40x40_p5_r2.5_self", "simt_H"),
    "attn_drops_last_query_tile": ("forward", "d100_L3_54x54_p2_B1", "simt_C"),
    "key_norm_first_32_columns": ("forward", "d36_L5_40x40_p5_r2.5_self", "simt_C"),
    "top_level_divided_by_4": ("forward", "d4_L2_12x12_p4_B3", "simt"),
    "b2_colsum_drops_last_rows": ("backward", "d132_L2_9x13_p1_B5", "bwd"),
    "bwd_top_level_divided_by_4": ("backward", "d12_L16_16x16_p4_B2", "bwd"),
    "patches_channel_major": ("tokeniser", "d12_L3_15x21_p3_B2", "tok32"),
    "unpatchify_p1_p2_swapped": ("tokeniser", "d12_L3_15x21_p3_B2", "bwd"),
    "token_bias_colsum_drops_last_rows": ("tokeniser", "d132_L2_9x13_p1_B5", "bwd"),
}


@pytest.mark.parametrize("fault", sorted(FAULTS))
def test_bounds_catch_faults(fault):
    """Each faulty reference misses the bound of the GPU test that sees it by >= 3x in both metrics."""
    kind, name, bound = FAULTS[fault]
    dim, L, hw, p, B, _, _, _ = SHAPES[name]
    meta = (B, (hw[0] // p) * (hw[1] // p), L, dim)
    if kind == "backward":
        good, bad = _fault_backward(name, fault)
    else:
        key, g, b = (_fault_forward if kind == "forward" else _fault_tokeniser)(name, fault)
        good, bad = {key: g}, {key: b}
    errs = errors(bad, good, meta)
    rel, ab = max(e[0] for e in errs.values()), max(e[1] for e in errs.values())
    t_rel, t_abs = TOL[bound]
    print(f"[cuda-core-oracle] fault {fault} at {name}: rel {rel:.3e} ({rel / t_rel:.0f}x {bound}) "
          f"abs {ab:.3e} ({ab / t_abs:.0f}x)")
    assert rel >= 3 * t_rel and ab >= 3 * t_abs, (fault, bound, rel, ab)


def test_key_norm_variant_unfaulted_is_the_reference():
    P, _, _, _, S, mask, attend_self, _ = _shape_inputs("d36_L5_40x40_p5_r2.5_self")
    got = _consensus_key_norm_cols(S, attend_self, mask, S.shape[-1])
    want = OT._consensus(S, attend_self, mask)
    assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max())


# ----------------------------------------------------------------------------- CPU: the fp32 consensus limit
def _forward_rc(dim, n, precision):
    """glom_b200_forward with plausible aligned pointers and an empty workspace: an argument error returns
    GLOM_B200_ERR_INVALID before the device query; past the argument checks the call fails on the device query (no GPU)
    or on the workspace size (GPU), before anything is enqueued."""
    from glom_pytorch_b200 import _native
    lib = _native.load()
    cfg = _native.make_cfg(dim, 2, n, False, 0, 0, precision)
    return lib.glom_b200_forward(ctypes.byref(cfg), 1024, 1024, 1024, 1024, None, 2048, 1, 1, 0, 1024, 0, None), \
        lib.glom_b200_last_error().decode()


@pytest.mark.parametrize("dim,n", [(32, 3601), (4, 3629), (36, 3600), (3632, 1)])
def test_fp32_consensus_limit_is_an_argument_error(dim, n):
    rc, msg = _forward_rc(dim, n, "fp32")
    assert rc == TD.INVALID, (rc, msg)
    assert f"dim + n must be <= {ATTN_F32_MAX_DIM_PLUS_N} (got {dim + n})" in msg, msg


@pytest.mark.parametrize("dim,n,precision", [(32, 3600, "fp32"), (4, 3628, "fp32"), (64, 3600, "bf16")])
def test_shapes_within_the_limit_pass_the_argument_checks(dim, n, precision):
    """d + n = 3632 on the fp32 engine, and any d + n on the bf16 engine (its consensus tiles the keys)."""
    rc, msg = _forward_rc(dim, n, precision)
    assert rc != TD.INVALID and "dim + n" not in msg, (rc, msg)


# ----------------------------------------------------------------------------- GPU: fp32 forward
@pytest.mark.gpu
@pytest.mark.parametrize("name", FP32_SHAPES)
def test_fp32_one_step(name):
    """One step from a random carried state: S_1, H and C per fp32 tile against float64 at the engine's tokens and S_0;
    a second identical call is bit-identical; iters = 0 returns S_0 (carried, or init_levels broadcast) bit for bit."""
    m, img, S, n, _ = _model(name)
    out, H, C = _f32_engine(m, img, S, 1)
    out2, H2, C2 = _f32_engine(m, img, S, 1)
    assert torch.equal(out, out2) and torch.equal(H, H2) and torch.equal(C, C2), "two identical calls differ"
    tok, P, pos, mask = FO._ref_inputs(m, img, n)
    errs = errors({"state": out, "H": H, "C": C}, _f32_refs(m, tok, P, pos, mask, S), tuple(S.shape))
    _report(name, "one step", errs)
    check(errs, FWD_TOL, name)
    with torch.no_grad():
        assert torch.equal(m(img.to(DEV), iters=0, levels=S.to(DEV)).cpu(), S)
        z = m(img.to(DEV), iters=0).cpu()
    assert torch.equal(z, m.init_levels.detach().cpu()[None, None].expand_as(S))


@pytest.mark.gpu
@pytest.mark.parametrize("carried", [True, False], ids=["carried", "init_levels"])
@pytest.mark.parametrize("name", FP32_SHAPES)
def test_fp32_chained_steps(name, carried):
    """forward(iters=3, return_all=True): slab t+1 against column_step at the engine's slab t.  forward(iters=3) and
    forward(iters=2) (the ping-pong between state_out and the workspace slab) equal the matching slabs bit for bit, and
    the H and C they leave in the workspace are those of their last step."""
    T = 3
    m, img, S, n, _ = _model(name, seed=1)
    start = S if carried else None
    with torch.no_grad():
        states = m(img.to(DEV), iters=T, levels=None if start is None else start.to(DEV), return_all=True).cpu()
    s0 = S if carried else m.init_levels.detach().cpu()[None, None].expand_as(S)
    assert torch.equal(states[0], s0)
    tok, P, pos, mask = FO._ref_inputs(m, img, n)
    meta = tuple(S.shape)
    worst = {}
    for t in range(T):
        e = errors({"state": states[t + 1]}, {"state": FO._exact(m, tok, P, pos, mask, states[t])}, meta)
        check(e, TOL["simt"], (name, carried, t))
        worst[f"state@{t + 1}"] = e["state"]
    for iters in (T, T - 1):
        last, H, C = _f32_engine(m, img, start, iters)
        assert torch.equal(last, states[iters]), iters
        ref = _f32_refs(m, tok, P, pos, mask, states[iters - 1])
        e = errors({"H": H, "C": C}, {k: ref[k] for k in ("H", "C")}, meta)
        check(e, FWD_TOL, (name, carried, iters))
        worst.update({f"{k}@{iters}": v for k, v in e.items()})
    _report(name, f"T={T} carried={carried}", worst)


@pytest.mark.gpu
def test_fp32_consensus_limit_raises_before_launch():
    """dim + n = 3636 on the fp32 engine: the argument error names the limit, and the module still runs afterwards."""
    import glom_pytorch_b200 as G
    m = G.Glom(dim=36, levels=2, image_size=240, patch_size=4, precision="fp32").to(DEV)
    img = torch.randn(1, 3, 240, 240, device=DEV)
    with torch.no_grad():
        with pytest.raises(RuntimeError, match=r"fp32 consensus keeps 16 \(dim \+ n\) floats per block in shared "
                                               r"memory: dim \+ n must be <= 3632 \(got 3636\)"):
            m(img, iters=1)
        out = m(img[:, :, :120, :120], iters=1)
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()


# ----------------------------------------------------------------------------- GPU: the two bf16 rows' forward
@pytest.mark.gpu
@pytest.mark.parametrize("name", BF16_SHAPES)
def test_bf16_forward(name):
    """One step (S_1, H, C against step_forward_bf16; S_1 against column_step) and three chained steps from init_levels,
    with test_forward_oracle's bounds."""
    m, img, S, n, _ = _model(name)
    out, H, C, _ = FO._engine(m, img, S, 1)
    tok, P, pos, mask = FO._ref_inputs(m, img, n)
    meta = tuple(S.shape)
    emu = FO._emu(m, tok, P, pos, mask, S)
    errs = FO.errors({"state": out, "H": H, "C": C}, {k: emu[k] for k in ("state", "H", "C")}, meta)
    _report(name, "one step vs step_forward_bf16", errs)
    FO.check(errs, TOL["emu"], name)
    errs = FO.errors({"state": out}, {"state": FO._exact(m, tok, P, pos, mask, S)}, meta)
    _report(name, "one step vs column_step", errs)
    FO.check(errs, TOL["tc"], name)
    with torch.no_grad():
        states = m(img.to(DEV), iters=3, return_all=True).cpu()
    for t in range(3):
        errs = FO.errors({"state": states[t + 1]}, {"state": FO._emu(m, tok, P, pos, mask, states[t])["state"]}, meta)
        FO.check(errs, TOL["emu"], (name, t))


# ----------------------------------------------------------------------------- GPU: the backward
def _grads(m, img, start, iters, return_all, cot, det):
    if det:
        return TD._three_runs(m, img, start, iters, return_all, cot)
    with TD.deterministic(False):
        return BO._engine_run(m, img, start, iters, return_all, cot)


@pytest.mark.gpu
@pytest.mark.parametrize("det", [False, True], ids=["default", "deterministic"])
@pytest.mark.parametrize("name", BWD_SHAPES)
def test_backward(name, det):
    """One step from a carried state (d_levels); three steps with return_all (a cotangent on every slab); three steps
    from init_levels with the last slab only (d_init_levels).  Every gradient per kernel block against grads_at_states +
    token_grads at the engine's own states; under the deterministic flag three runs (module, deepcopy, second stream)
    are bit-identical."""
    m, img, S, n, g = _model(name, seed=2)
    tol = TOL["tc_bwd"] if SHAPES[name][6] == "bf16" and SHAPES[name][0] % 256 == 0 else TOL["bwd"]
    T = 3
    meta = tuple(S.shape)
    worst = {}
    for case, (start, iters, return_all) in {"one_step": (S, 1, False), "T3_return_all": (S, T, True),
                                             "T3_last_slab_init": (None, T, False)}.items():
        cot = torch.randn(((iters + 1,) if return_all else ()) + meta, generator=g)
        out, got = _grads(m, img, start, iters, return_all, cot, det)
        if return_all:
            states = out.cpu()
        elif start is not None:
            states = torch.stack([S, out.cpu()])
        else:
            with torch.no_grad():
                states = m(img.to(DEV), iters=iters, return_all=True).cpu()
            assert torch.equal(states[iters], out.cpu())
        ref, _, _ = BO._reference(m, img, states, cot, return_all=return_all, carried=start is not None)
        assert set(got) == set(ref), set(got) ^ set(ref)
        errs = errors(got, ref, meta)
        check(errs, tol, (name, det, case))
        worst[case] = (max(e[0] for e in errs.values()), max(e[1] for e in errs.values()))
    _report(name, f"backward det={det}", worst)


# ----------------------------------------------------------------------------- GPU: the tokeniser
# patch, (H, W), batch: p from 1 to 16, non-square images in both orientations, row counts that are not multiples of 64
TOK_GEOMS = [(1, (9, 13), 5),      # k3 = 3, 585 rows
             (2, (22, 14), 3),     # k3 = 12, 231 rows
             (3, (15, 27), 2),     # k3 = 27, 90 rows
             (5, (40, 25), 3),     # k3 = 75 (one 64-column tile and a partial one of d_weight), 120 rows
             (7, (35, 21), 2),     # k3 = 147, 30 rows
             (16, (32, 48), 3)]    # k3 = 768, 18 rows
TOK_IDS = [f"p{p}_{h}x{w}_B{b}" for p, (h, w), b in TOK_GEOMS]


def _tok_model(dim, p, hw, B, precision, seed=4):
    import glom_pytorch_b200 as G
    isz = max(hw)
    params = O.synth_params(dim, 2, isz, p, seed=seed)
    m = G.Glom(dim=dim, levels=2, image_size=isz, patch_size=p, precision=precision)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=False)
    m = m.to(DEV)
    g = torch.Generator().manual_seed(seed + 1)
    img = torch.randn((B, 3) + hw, generator=g)
    w, b = (torch.from_numpy(params[k]).double() for k in ("image_to_tokens.1.weight", "image_to_tokens.1.bias"))
    return m, img, w, b, g


@pytest.mark.gpu
@pytest.mark.parametrize("geom", TOK_GEOMS, ids=TOK_IDS)
@pytest.mark.parametrize("dim", [4, 36, 100, 128])
def test_fp32_tokeniser(dim, geom):
    """MODE_TOK (K = 3p^2) against float64 patchify(img) W^T + b per 64 x 64 tile."""
    p, hw, B = geom
    m, img, w, b, _ = _tok_model(dim, p, hw, B, "fp32")
    with torch.no_grad():
        tok = m.tokens(img.to(DEV)).cpu()
    ref = OT.patchify(img.double(), p) @ w.T + b
    errs = errors({"tokens": tok}, {"tokens": ref}, (B, tok.shape[1], 1, dim))
    _report(f"d{dim}", f"fp32 tokeniser {TOK_IDS[TOK_GEOMS.index(geom)]}", errs)
    check(errs, TOL["tok32"], (dim, geom))


@pytest.mark.gpu
@pytest.mark.parametrize("geom", TOK_GEOMS, ids=TOK_IDS)
@pytest.mark.parametrize("dim", [64, 192])
def test_tensor_core_tokeniser_patch_sizes(dim, geom):
    """The tensor-core tokeniser (k3 padded to a multiple of 64) against the bf16-operand tokeniser in float64."""
    p, hw, B = geom
    m, img, w, b, _ = _tok_model(dim, p, hw, B, "bf16")
    with torch.no_grad():
        tok = m.tokens(img.to(DEV)).cpu()
    ref = OT.bf16(OT.patchify(img.double(), p)) @ OT.bf16(w).T + b
    errs = errors({"tokens": tok}, {"tokens": ref}, (B, tok.shape[1], 1, dim))
    _report(f"d{dim}", f"tensor-core tokeniser {TOK_IDS[TOK_GEOMS.index(geom)]}", errs)
    check(errs, TOL["tok"], (dim, geom))


NEEDS = {"image": (True, False, False), "weight": (False, True, False), "bias": (False, False, True),
         "all": (True, True, True)}
TOK_BWD_DIMS = [4, 36, 100, 132, 12, 100]          # one per TOK_GEOMS entry


def _tok_backward(m, img, cot, needs):
    lin = m.image_to_tokens[1]
    x = img.to(DEV).requires_grad_(needs[0])
    w = lin.weight.detach().clone().requires_grad_(needs[1])
    b = lin.bias.detach().clone().requires_grad_(needs[2])
    from glom_pytorch_b200.glom import _Tokenize
    tok = _Tokenize.apply(m, x, w, b)
    (tok * cot.to(DEV)).sum().backward()
    torch.cuda.synchronize()
    return {"d_img": x.grad, "image_to_tokens.1.weight": w.grad, "image_to_tokens.1.bias": b.grad}


@pytest.mark.gpu
@pytest.mark.parametrize("det", [False, True], ids=["default", "deterministic"])
@pytest.mark.parametrize("need", list(NEEDS))
@pytest.mark.parametrize("geom", TOK_GEOMS, ids=TOK_IDS)
def test_tokeniser_backward(geom, need, det):
    """_Tokenize.apply with only the image, only the weight, only the bias, or all three requiring grad: the requested
    gradients against token_grads, the others None; under the deterministic flag three runs (two on the current stream,
    one on a second stream) are bit-identical."""
    p, hw, B = geom
    dim = TOK_BWD_DIMS[TOK_GEOMS.index(geom)]
    m, img, w, b, g = _tok_model(dim, p, hw, B, "fp32")
    n = (hw[0] // p) * (hw[1] // p)
    cot = torch.randn(B, n, dim, generator=g)
    needs = NEEDS[need]
    with TD.deterministic(det):
        got = _tok_backward(m, img, cot, needs)
        if det:
            again = _tok_backward(m, img, cot, needs)
            side = torch.cuda.Stream(DEV)
            side.wait_stream(torch.cuda.current_stream(DEV))
            with torch.cuda.stream(side):
                third = _tok_backward(m, img, cot, needs)
            torch.cuda.synchronize()
            for k, v in got.items():
                assert (v is None) == (again[k] is None) == (third[k] is None), k
                if v is not None:
                    assert torch.equal(v, again[k]) and torch.equal(v, third[k]), k
    ref = OT.token_grads(img, w, b, p, cot)
    for k, want in zip(ref, needs):
        assert (got[k] is not None) == want, (k, need)
    ref = {k: v for k, v in ref.items() if got[k] is not None}
    errs = errors(got, ref, (B, n, 2, dim))
    _report(f"d{dim}", f"tokeniser backward {TOK_IDS[TOK_GEOMS.index(geom)]} {need} det={det}", errs)
    check(errs, TOL["bwd"], (geom, need, det))
