"""The forward against float64 references evaluated at the engine's own states (oracle/glom_oracle_torch.py).

`step_forward_bf16` is one K1 -> K3 -> K2 step of the bf16 engine in float64 with bf16 rounding at exactly the points
where the kernels round (shadows, weight packs, H, the consensus probabilities and C, the exact-maximum path's second
rounding, the key passes beyond 576 keys).  Fed the engine's own state S_t, it predicts S_{t+1}, H and C to within the
kernels' fp32 summation order.  `column_step` is the plain float64 step.  Every step is checked from the state the
engine itself produced, so drift over T steps drops out and a chain of T steps is T one-step checks.

Metric (`errors`): every compared tensor is cut into the blocks its kernel tiles -- S_{t+1} per (256-row block of the
B*n rows, level, K2 column tile of 256 / 128 / 64), H per (group, 128-row block, 256-column tile), C per (image, level,
128-query tile), the squared-norm partials per (row, level, part), tokens per (256-row block, column tile) -- and each
block's rel-Frobenius error is taken against max(|ref block|, FLOOR * rms block norm of the tensor).  `rel` is the worst
block over every tensor, `abs` the worst max-abs error over the tensor's max |ref|.

The CPU tests pin the reference (equal to `column_step` to 1e-12 with its roundings switched off, close to the numpy
bf16 emulation with them on), pin the kernel GELU fit, and show that each bound is missed by >= 3x by plausible kernel
faults.  The GPU tests run one step and chains of steps at the shapes where the kernels tile, mask, pass over keys and
switch stabiliser.

Bounds (rel, abs), set at about 3x the worst value observed over all the GPU tests of the path on one H100 80GB HBM3
(700 W power limit); observed maxima in brackets:
  emu   bf16 engine (S_{t+1}, H, C) vs step_forward_bf16 at the engine's S_t
        (1e-3, 1.3e-2)   [rel 3.3e-4 (H, configs[1] dims from init_levels), abs 4.3e-3 (H, d256_n576_r2.5): one bf16
                          ulp of H; S_{t+1} <= 1.3e-4 / 1.9e-3, C <= 2.7e-4 / 4.2e-3]
  tc    bf16 engine S_{t+1} vs column_step at the engine's S_t
        (1.2e-2, 3.2e-2) [rel 3.8e-3, abs 1.06e-2 at cons_d128_n576_exact, whose logits span ~10 log2 units;
                          <= 2.9e-3, 4.8e-3 elsewhere]
  simt  fp32 engine S_{t+1} vs column_step at the engine's S_t
        (8e-7, 1.2e-6)   [rel 2.7e-7, abs 3.9e-7]
  nsq   the squared-norm partials vs float64 sums of squares of the returned state
        (5e-7, 3.5e-7)   [rel 1.7e-7, abs 1.1e-7]
  tok   the tensor-core tokeniser vs the bf16-operand tokeniser
        (1.5e-6, 3e-6)   [rel 5.1e-7, abs 9.7e-7]
The key rows at norms 0 .. 2e-12 ("subeps") and the self-only rows of a radius below 1, with both stabilisers (H100
80GB HBM3, 700 W): emu <= 3.5e-4 / 3.9e-3 (H), tc <= 3.1e-3 / 2.6e-3, simt <= 2.6e-7 / 3.5e-7.
No kernel missed the reference by more than rounding explains.  The faults of test_bounds_catch_faults miss these
bounds by 17x (rel) and 4.8x (abs) at least.
"""
import math

import numpy as np
import pytest
import torch

from oracle import glom_oracle as O
from oracle import glom_oracle_torch as OT

DEV = "cuda:0"
FLOOR = 0.1
TOL = {"emu": (1e-3, 1.3e-2), "tc": (1.2e-2, 3.2e-2), "simt": (8e-7, 1.2e-6), "nsq": (5e-7, 3.5e-7),
       "tok": (1.5e-6, 3e-6)}
NUMPY_EMU_TOL = (2.5e-3, 5e-3)  # step_forward_bf16 vs glom_forward(emulate="bf16") (observed 8.5e-4, 1.6e-3)
GELU_FIT_MAX = 1.9e-6          # ptx.cuh, gelu_fit


# ----------------------------------------------------------------------------- metric
def _blocks(key, x, meta):
    """-> list of blocks of x (float64 CPU) along the structure its kernel tiles; meta = (B, n, L, d)."""
    B, n, L, d = meta
    R = B * n
    bn, _ = OT.forward_tiles(d)
    if key == "state":                                                       # K2 tiles
        x = x.reshape(R, L, d)
        return [x[r:r + 256, l, c:c + bn] for r in range(0, R, 256) for l in range(L) for c in range(0, d, bn)]
    if key == "H":                                                           # K1 tiles
        return [x[g, r:r + 128, c:c + 256] for g in range(x.shape[0]) for r in range(0, R, 128)
                for c in range(0, 4 * d, 256)]
    if key == "C":                                                           # K3 items
        return [x[b, i:i + 128, l] for b in range(B) for l in range(L) for i in range(0, n, 128)]
    if key == "tokens":                                                      # tokeniser tiles
        x = x.reshape(R, d)
        return [x[r:r + 256, c:c + bn] for r in range(0, R, 256) for c in range(0, d, bn)]
    raise KeyError(key)


def errors(got, ref, meta):
    """-> {key: (worst block rel-Frobenius, max-abs / max |ref|)} for the keys of `ref`."""
    out = {}
    for k, r in ref.items():
        g = torch.as_tensor(got[k]).detach().to("cpu", torch.float64)
        r = torch.as_tensor(r).to("cpu", torch.float64)
        assert g.shape == r.shape, (k, tuple(g.shape), tuple(r.shape))
        assert torch.isfinite(g).all(), k
        if k == "nsq":                                                       # one block per (row, level, part)
            rms = float(torch.linalg.norm(r)) / math.sqrt(r.numel())
            rel = float(((g - r).abs() / r.abs().clamp_min(max(FLOOR * rms, 1e-300))).max())
        else:
            gb, rb = _blocks(k, g, meta), _blocks(k, r, meta)
            rms = float(torch.linalg.norm(r)) / math.sqrt(len(rb))
            rel = max(float(torch.linalg.norm(a - b)) / max(float(torch.linalg.norm(b)), FLOOR * rms, 1e-300)
                      for a, b in zip(gb, rb))
        ab = float((g - r).abs().max()) / max(float(r.abs().max()), 1e-300)
        out[k] = (rel, ab)
    return out


def worst(errs):
    return max(e[0] for e in errs.values()), max(e[1] for e in errs.values())


def check(errs, tol, what):
    bad = {k: e for k, e in errs.items() if e[0] > tol[0] or e[1] > tol[1]}
    assert not bad, (what, tol, bad)
    return worst(errs)


def _report(name, what, errs):
    rel, ab = worst(errs)
    print(f"[fwd-oracle] {name} {what}: rel {rel:.3e} abs {ab:.3e} "
          + " ".join(f"{k}=({e[0]:.2e},{e[1]:.2e})" for k, e in errs.items()))


# ----------------------------------------------------------------------------- CPU: the reference itself
def _small(d=32, L=3, isz=16, p=4, B=3, seed=1, rms=1.0):
    P = {k: torch.from_numpy(v).double() for k, v in O.synth_params(d, L, isz, p, seed=seed).items()}
    n = (isz // p) ** 2
    g = torch.Generator().manual_seed(seed)
    tok = torch.randn(B, n, d, generator=g, dtype=torch.float64)
    S = torch.randn(B, n, L, d, generator=g, dtype=torch.float64) * rms
    return P, tok, P["pos_emb.weight"][:n].clone(), S


# (d, L, image_size, patch, B, radius, attend_self): masks with and without self; n = 784 > 576 keys in two passes, the
# radius leaving rows with no unmasked key in the first pass
IDENTITY_CASES = {
    "plain": (32, 3, 16, 4, 3, 0, False),
    "radius_self": (32, 3, 16, 4, 3, 1.5, True),
    "radius": (64, 2, 16, 4, 2, 1.0, False),
    "passes_radius_self": (32, 2, 56, 2, 1, 6.5, True),
    "passes": (32, 2, 56, 2, 1, 0, False),
}


@pytest.mark.parametrize("name", sorted(IDENTITY_CASES))
def test_step_forward_bf16_without_rounding_is_column_step(name, monkeypatch):
    """With bf16 rounding switched off, step_forward_bf16 (bound stabiliser or exact maximum everywhere) is the exact
    step; with it on, it moves the result by about 2^-9 relative."""
    d, L, isz, p, B, radius, attend_self = IDENTITY_CASES[name]
    P, tok, pos, S = _small(d, L, isz, p, B)
    mask = OT.radius_mask(isz // p, radius) if radius else None
    exact = OT.column_step(S, tok, pos, P, mask, attend_self)
    meta = tuple(S.shape)
    _, part_w = OT.forward_tiles(d)
    nsq = exact.reshape(-1, L, d // part_w, part_w).square().sum(-1)
    for bound_max in (OT.ATTN_BOUND_MAX, -math.inf):
        monkeypatch.setattr(OT, "bf16", lambda x: x)
        monkeypatch.setattr(OT, "ATTN_BOUND_MAX", bound_max)
        got = OT.step_forward_bf16(P, tok, pos, S, attend_self=attend_self, mask=mask)
        monkeypatch.undo()
        for k, r in (("state", exact), ("C", OT._consensus(S, attend_self, mask)), ("nsq", nsq)):
            err = float((got[k] - r).abs().max()) / float(r.abs().max())
            assert err <= 1e-12, (name, bound_max, k, err)
    rounded = OT.step_forward_bf16(P, tok, pos, S, attend_self=attend_self, mask=mask)
    rel, _ = worst(errors(rounded, {"state": exact}, meta))
    assert 1e-4 < rel < 5e-2, rel


@pytest.mark.parametrize("name", ["plain", "radius_self", "passes"])
def test_step_forward_bf16_agrees_with_numpy_emulation(name):
    """The numpy oracle's emulate="bf16" rounds the same operands but stabilises the softmax with the row maximum and
    computes in fp32: one step agrees to that difference."""
    d, L, isz, p, B, radius, attend_self = IDENTITY_CASES[name]
    P, tok, pos, S = _small(d, L, isz, p, B)
    mask = OT.radius_mask(isz // p, radius) if radius else None
    got = OT.step_forward_bf16(P, tok, pos, S, attend_self=attend_self, mask=mask)
    params = {k: v.numpy().astype(np.float32) for k, v in P.items()}
    emu = O.glom_forward(params, None, patch_size=p, iters=1, levels=S.numpy().astype(np.float32),
                         tokens=tok.numpy().astype(np.float32), consensus_self=attend_self, local_consensus_radius=radius,
                         image_size=isz, dtype=np.float32, emulate="bf16")
    errs = errors({"state": torch.from_numpy(emu)}, {"state": got["state"]}, tuple(S.shape))
    _report(name, "step_forward_bf16 vs numpy emulate=bf16", errs)
    check(errs, NUMPY_EMU_TOL, name)


def _gelu_fit_f32(x):
    """ptx.cuh gelu_fit evaluated in float32 as written: each fmaf rounded once, ex2.approx as a rounded exp2."""
    f32 = np.float32

    def fmaf(a, b, c):                              # overflow to +-inf far outside [-6, 6], as in float32
        with np.errstate(over="ignore", invalid="ignore"):
            return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(f32)
    x = x.astype(f32)
    u = (x.view(np.uint32) | np.uint32(0x80000000)).view(f32)
    q = fmaf(np.full_like(u, 0.00036467931931838393), u, np.full_like(u, 0.006363349035382271))
    for c in (0.05013200640678406, -0.4617065489292145, 1.150075078010559, -1.0001276731491089):
        q = fmaf(q, u, np.full_like(u, c))
    e = np.exp2(q.astype(np.float64)).astype(f32)
    return fmaf(u, e, np.maximum(x, f32(0)))


def test_gelu_fit_within_documented_bound():
    """K1's GELU (a degree-5 fit of log2 Phi(-|x|) on [0, 6], no clamp) stays within 1.9e-6 of the erf form, including
    far outside the fit interval and at +-0."""
    x = np.concatenate([np.linspace(-12, 12, 2_000_001), [0.0, -0.0, 6.0, -6.0, 30.0, -30.0, 1e4, -1e4, 1e30, -1e30,
                                                         3.4e38, -3.4e38]]).astype(np.float32)
    got = _gelu_fit_f32(x).astype(np.float64)
    xd = x.astype(np.float64)
    want = np.where(np.abs(xd) > 40, np.maximum(xd, 0.0), O._gelu_block(np.clip(xd, -40, 40)))
    err = np.abs(got - want)
    assert np.isfinite(got).all()
    assert err.max() <= GELU_FIT_MAX, (float(err.max()), float(xd[err.argmax()]))
    assert got[np.where(x == 0)].max() == 0.0


# ----------------------------------------------------------------------------- CPU: the bounds catch faults
_ORIG = {k: getattr(OT, k) for k in ("_fwd_k1_operands", "_fwd_key_norm", "_fwd_attn_logits", "_fwd_attn_passes",
                                     "_fwd_k2")}


def _k2_no_h_last_block(S, H, C, w2bu, w2td, b2, contrib):
    R = H.shape[1]
    H = H.clone()
    H[:, 128 * (R // 128):] = 0
    return _ORIG["_fwd_k2"](S, H, C, w2bu, w2td, b2, contrib)


def _k1_last_td_reads_sb(xb, sb, sp):
    ops = _ORIG["_fwd_k1_operands"](xb, sb, sp)
    ops[-2] = sb[:, :, -1]                           # group 2L-3 = top-down L-2 reads S[L-1] without pos
    return ops


def _k3_diag_first_tile_only(q, rs, attend_self, mask):
    x = _ORIG["_fwd_attn_logits"](q, rs, attend_self, mask)
    raw = _ORIG["_fwd_attn_logits"](q, rs, True, mask)
    return torch.where((torch.arange(q.shape[-2]) >= 128)[:, None], raw, x)


def _k2_b2_from_neighbour(S, H, C, w2bu, w2td, b2, contrib):
    bn, _ = OT.forward_tiles(S.shape[-1])
    b2 = b2.clone()
    b2[:, -bn:] = b2[:, -2 * bn:-bn]                 # the last column tile takes the one before
    return _ORIG["_fwd_k2"](S, H, C, w2bu, w2td, b2, contrib)


# fault -> (patched helper, replacement, (d, L, image_size, patch, B, state rms, second-layer bias scale)) of inputs
# where that part carries weight: 300 rows (the last 128-row block holds 44); n = 256 > 128 queries with a peaked
# diagonal; n = 784 (passes 512 + 272); d = 192 (six squared-norm partials, a peaked softmax); d = 192 (three 64-column
# K2 tiles) with second-layer biases of a trained network's size
FAULTS = {
    "k2_no_h_last_partial_block": ("_fwd_k2", _k2_no_h_last_block, (64, 3, 40, 4, 3, 1.0, 1.0)),
    "k1_last_td_without_pos": ("_fwd_k1_operands", _k1_last_td_reads_sb, (64, 3, 40, 4, 3, 1.0, 1.0)),
    "k3_diag_only_in_tile_0": ("_fwd_attn_logits", _k3_diag_first_tile_only, (64, 2, 64, 4, 1, 4.0, 1.0)),
    "k3_drops_last_pass": ("_fwd_attn_passes", lambda n: _ORIG["_fwd_attn_passes"](n)[:-1], (64, 2, 56, 2, 1, 2.0, 1.0)),
    "key_norm_drops_last_part": ("_fwd_key_norm", lambda nsq: nsq[..., :-1].sum(-1).sqrt(), (192, 2, 24, 4, 2, 30.0, 1.0)),
    "k2_b2_of_neighbour_tile": ("_fwd_k2", _k2_b2_from_neighbour, (192, 2, 24, 4, 2, 0.1, 10.0)),
}


def _fault_case(spec):
    d, L, isz, p, B, rms, b2_scale = spec
    P, tok, pos, S = _small(d, L, isz, p, B, seed=3, rms=rms)
    for k in ("bottom_up.net.3.bias", "top_down.net.3.bias"):
        P[k] = P[k] * b2_scale
    return P, tok, pos, S


@pytest.mark.parametrize("fault", sorted(FAULTS))
def test_bounds_catch_faults(fault, monkeypatch):
    """Each faulty reference misses every bound of the GPU tests by >= 3x in both metrics, so a kernel with that fault
    fails them."""
    helper, bad_fn, spec = FAULTS[fault]
    P, tok, pos, S = _fault_case(spec)
    good = OT.step_forward_bf16(P, tok, pos, S)
    monkeypatch.setattr(OT, helper, bad_fn)
    bad = OT.step_forward_bf16(P, tok, pos, S)
    monkeypatch.undo()
    rel, ab = worst(errors(bad, good, tuple(S.shape)))
    print(f"[fwd-oracle] fault {fault}: rel {rel:.3e} abs {ab:.3e}")
    for path, (t_rel, t_abs) in TOL.items():
        assert rel >= 3 * t_rel and ab >= 3 * t_abs, (fault, path, rel, ab)


def test_unfaulted_helpers_are_the_reference(monkeypatch):
    """The fault helpers without a fault reproduce the reference (so the faults, not the helpers, make the difference)."""
    for fault, (helper, _, spec) in FAULTS.items():
        P, tok, pos, S = _fault_case(spec)
        good = OT.step_forward_bf16(P, tok, pos, S)
        monkeypatch.setattr(OT, helper, lambda *a, _f=_ORIG[helper]: _f(*a))
        again = OT.step_forward_bf16(P, tok, pos, S)
        monkeypatch.undo()
        for k in good:
            assert torch.equal(again[k], good[k]), (fault, k)


# ----------------------------------------------------------------------------- GPU
# name: dim, L, image_size, patch, img_hw, B, kwargs, state rms ("edge": see _edge_state)
SHAPES = {
    # 27 rows (one partial block), BN 64, 2 parts, one 16-key block with 7 padding keys
    "d64_n9": (64, 3, 12, 4, None, 3, {}, 1.0),
    # BN 64, 6 parts (general norm path), three K1 N tiles, 108 rows
    "d192_n36": (192, 3, 24, 4, None, 3, {}, 1.0),
    # BN 64, 10 parts, O slices 256 + 64, a ragged 256-key block, 720 rows, radius mask
    "d320_n144_r3": (320, 2, 48, 4, None, 5, dict(local_consensus_radius=3), 1.0),
    # BN 128, the masked logits with attend_self
    "d128_n256_r2_self": (128, 3, 64, 4, None, 2, dict(local_consensus_radius=2, consensus_self=True), 1.0),
    # BN 128, 6 parts, 300 rows
    "d384_n100": (384, 2, 40, 4, None, 3, {}, 1.0),
    # n = 32 of 64 patches: position rows of a non-square image
    "d256_nonsquare": (256, 3, 32, 4, (16, 32), 2, {}, 1.0),
    # five 128-key blocks (the last holds 64), five query tiles
    "d256_n576_r2.5": (256, 2, 96, 4, None, 1, dict(local_consensus_radius=2.5), 1.0),
    # 12 parts, a single top-down group, half-cost top-level tiles
    "d768_L2": (768, 2, 32, 4, None, 3, {}, 1.0),
    # 20 parts (> 16: the general norm path at BN 256), five O slices
    "d1280_n64": (1280, 2, 32, 4, None, 1, {}, 1.0),
    # key passes of 512 + 272, rows with no unmasked key in pass 0
    "d128_n784_r6.5_self": (128, 2, 56, 2, None, 1, dict(local_consensus_radius=6.5, consensus_self=True), 1.0),
    # four key passes, 13 query tiles
    "d64_n1600": (64, 2, 80, 2, None, 1, {}, 1.0),
    # logit bounds at 0.9x and 1.1x of the stabiliser switch in the same warps, a zero level (the 1e-12 eps)
    "d256_bound_edge": (256, 3, 32, 4, None, 2, {}, "edge"),
    "d256_bound_edge_self": (256, 3, 32, 4, None, 2, dict(consensus_self=True), "edge"),
    # key rows at norms on both sides of the 1e-12 eps, facing aligned queries (see _subeps_state)
    "d256_n144_subeps": (256, 3, 48, 4, None, 5, {}, "subeps"),
    "d256_n576_r2.5_self_subeps": (256, 2, 96, 4, None, 1, dict(local_consensus_radius=2.5, consensus_self=True),
                                   "subeps"),
    "d192_n144_r3_self_subeps": (192, 3, 48, 4, None, 2, dict(local_consensus_radius=3, consensus_self=True), "subeps"),
    # a radius below 1: every row's only key is itself (the diagonal's constant logit without attend_self), every other
    # key block and pass of the row is empty; n = 784 in passes of 512 + 272; with both stabilisers at the edge states
    "d256_n256_self_only": (256, 2, 64, 4, None, 2, dict(local_consensus_radius=0.5), 1.0),
    "d256_n784_self_only_self": (256, 2, 56, 2, None, 1, dict(local_consensus_radius=0.5, consensus_self=True), 1.0),
    "d256_n256_self_only_self_edge": (256, 3, 64, 4, None, 2, dict(local_consensus_radius=0.5, consensus_self=True),
                                      "edge"),
    "d256_n784_self_only_edge": (256, 3, 56, 2, None, 2, dict(local_consensus_radius=0.5), "edge"),
    "d192_n144_self_only": (192, 3, 48, 4, None, 2, dict(local_consensus_radius=0.5), 1.0),
    # configs[1] dims
    "config2_dims": (512, 6, 224, 14, None, 2, {}, 1.0),
    # the consensus kernel's own cases: one query tile; a 256-key block of real keys (the unmasked straight-line path);
    # the exact maximum on every warp over five 128-key blocks (P rounded twice); radius mask; attend_self
    "cons_d128_n64": (128, 3, 32, 4, None, 2, {}, 2.0),
    "cons_d512_n256": (512, 2, 64, 4, None, 2, {}, 2.0),
    "cons_d128_n576_exact": (128, 2, 96, 4, None, 1, {}, 80.0),
    "cons_d128_n256_r3": (128, 2, 64, 4, None, 2, dict(local_consensus_radius=3), 2.0),
    "cons_d128_n256_self": (128, 2, 64, 4, None, 2, dict(consensus_self=True), 2.0),
}


def _edge_state(B, n, L, d, g):
    """Unit rows scaled so that the logit bound d^-1/2 log2e |S_i| is 0.9x / 1.1x of ATTN_BOUND_MAX on alternate rows of
    the even 16-row warps and 0.9x on every row of the odd ones; level 2 of image 1 is all zeros."""
    S = torch.randn(B, n, L, d, generator=g)
    S = S / S.norm(dim=-1, keepdim=True)
    edge = OT.ATTN_BOUND_MAX / (d ** -0.5 * OT.LOG2E)
    i = torch.arange(n)
    f = torch.where((i // 16) % 2 == 0, torch.where(i % 2 == 0, 0.9, 1.1), torch.tensor(0.9))
    S = S * (edge * f)[None, :, None, None]
    S[1, :, 2] = 0
    return S


SUBEPS_NORMS = (0.0, 1e-30, 0.3e-12, 0.9e-12, 0.999e-12, 1.001e-12, 2e-12)
SUBEPS_LEVEL = 1


def _subeps_state(B, n, L, d, g, dtype=torch.float32):
    """Rows of rms 1, except level SUBEPS_LEVEL of image 0: there every row is c_i v for one unit vector v, so that its
    queries are aligned with its keys, with |c_i| of rms 1 per element and both signs, and rows 0..6 have the norms
    SUBEPS_NORMS: zero, one whose squares underflow in fp32, and rows just below and above F.normalize's eps 1e-12."""
    S = torch.randn(B, n, L, d, generator=g, dtype=dtype)
    v = torch.randn(d, generator=g, dtype=dtype)
    v = v / v.norm()
    c = (0.5 + torch.rand(n, generator=g, dtype=dtype)) * math.sqrt(d)
    c = torch.where(torch.rand(n, generator=g, dtype=dtype) < 0.5, -c, c)
    c[:len(SUBEPS_NORMS)] = torch.tensor(SUBEPS_NORMS, dtype=dtype)
    S[0, :, SUBEPS_LEVEL] = c[:, None] * v
    return S


def _state(kind, B, n, L, d, g):
    """A random state of rms `kind`, or one of the named kinds "edge" (_edge_state) and "subeps" (_subeps_state)."""
    if kind == "edge":
        return _edge_state(B, n, L, d, g)
    if kind == "subeps":
        return _subeps_state(B, n, L, d, g)
    return torch.randn(B, n, L, d, generator=g) * kind


def _model(name, precision, seed=0, batch=None):
    dim, L, isz, p, hw, B, kw, rms = SHAPES[name]
    B = batch or B
    import glom_pytorch_b200 as G
    params = O.synth_params(dim, L, isz, p, seed=seed)
    m = G.Glom(dim=dim, levels=L, image_size=isz, patch_size=p, precision=precision, **kw)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=False)
    m = m.to(DEV)
    hw = hw or (isz, isz)
    n = (hw[0] // p) * (hw[1] // p)
    g = torch.Generator().manual_seed(seed + 29)
    img = torch.randn((B, 3) + hw, generator=g)
    return m, img, _state(rms, B, n, L, dim, g), n


def _mask(m, n):
    side, d2 = m.attention.mask_params(n)
    if not side:
        return None
    co = torch.stack(torch.meshgrid(torch.arange(side), torch.arange(side), indexing="ij"), -1).reshape(-1, 2)
    return ((co[:, None] - co[None]) ** 2).sum(-1) > d2


def _ref_inputs(m, img, n):
    """The engine's own tokens, the parameters and positions, the mask."""
    with torch.no_grad():
        tok = m.tokens(img.to(DEV)).cpu()
    P = {k: q.detach().cpu() for k, q in m.named_parameters()}
    return tok, P, P["pos_emb.weight"][:n], _mask(m, n)


def _engine(m, img, S, iters):
    """forward(iters) from S (None: init_levels) -> (S_iters, H, C, nsq) with H, C and the squared-norm partials read
    from workspace buffers 0-2: after the call H and C are those of the last step and buffer 2 holds the partials of
    S_iters for even iters (of S_{iters-1} for odd)."""
    from glom_pytorch_b200 import _native
    with torch.no_grad():
        out = m(img.to(DEV), iters=iters, levels=None if S is None else S.to(DEV))
    torch.cuda.synchronize()
    B, n, L, d = out.shape
    cfg = m.engine_cfg(n)
    ws = m._workspace

    def buf(which):
        off, nb = _native.workspace_offset(cfg, B, iters, False, which)
        return ws[off:off + nb]
    R, G, m128 = B * n, 2 * L - 1, (B * n + 127) // 128
    H = buf(0).view(torch.bfloat16).reshape(G, m128, 4 * d // 64, 128, 64).permute(0, 1, 3, 2, 4)
    H = H.reshape(G, m128 * 128, 4 * d)[:, :R].float().cpu()
    C = buf(1).view(torch.bfloat16).reshape(B, n, L, d).float().cpu()
    _, part_w = OT.forward_tiles(d)
    nsq = buf(2).view(torch.float32).reshape(R, L, d // part_w).cpu()
    return out.cpu(), H, C, nsq


def _emu(m, tok, P, pos, mask, S):
    return OT.step_forward_bf16(P, tok, pos, S, attend_self=m.attention.attend_self, mask=mask)


def _exact(m, tok, P, pos, mask, S):
    return OT.column_step(OT._f64(S), OT._f64(tok), OT._f64(pos), {k: OT._f64(P[k]) for k in OT.MLP_KEYS}, mask,
                          m.attention.attend_self)


def _sumsq_parts(S):
    B, n, L, d = S.shape
    _, part_w = OT.forward_tiles(d)
    return S.double().reshape(B * n, L, d // part_w, part_w).square().sum(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SHAPES))
def test_one_step(name):
    """One step from a random carried state: S_1, H and C against step_forward_bf16 and S_1 against column_step; a
    second identical call is bit-identical; after two steps the squared-norm partials against float64 sums of squares
    of the returned S_2."""
    m, img, S, n = _model(name, "bf16")
    out, H, C, _ = _engine(m, img, S, 1)
    out2, _, C2, _ = _engine(m, img, S, 1)
    assert torch.equal(out, out2) and torch.equal(C, C2), "two identical calls differ"
    tok, P, pos, mask = _ref_inputs(m, img, n)
    meta = tuple(S.shape)
    emu = _emu(m, tok, P, pos, mask, S)
    errs = errors({"state": out, "H": H, "C": C}, {k: emu[k] for k in ("state", "H", "C")}, meta)
    _report(name, "one step vs step_forward_bf16", errs)
    check(errs, TOL["emu"], name)
    errs = errors({"state": out}, {"state": _exact(m, tok, P, pos, mask, S)}, meta)
    _report(name, "one step vs column_step", errs)
    check(errs, TOL["tc"], name)
    s2, _, _, nsq = _engine(m, img, S, 2)
    errs = errors({"nsq": nsq}, {"nsq": _sumsq_parts(s2)}, meta)
    _report(name, "nsq of S_2", errs)
    check(errs, TOL["nsq"], name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["d64_n9", "cons_d128_n64", "d256_nonsquare", "config2_dims"])
def test_one_step_from_init_levels(name):
    """One step from init_levels (every row of a level equal; step 0 reads the broadcast init_levels)."""
    m, img, S, n = _model(name, "bf16")
    out, H, C, _ = _engine(m, img, None, 1)
    B, n, L, d = S.shape
    S0 = m.init_levels.detach().cpu()[None, None].expand(B, n, L, d)
    tok, P, pos, mask = _ref_inputs(m, img, n)
    emu = _emu(m, tok, P, pos, mask, S0)
    errs = errors({"state": out, "H": H, "C": C}, {k: emu[k] for k in ("state", "H", "C")}, tuple(S.shape))
    _report(name, "one step from init_levels vs step_forward_bf16", errs)
    check(errs, TOL["emu"], name)


CHAINED = {"d64_n9": 3, "d192_n36": 3, "d320_n144_r3": 3, "d128_n256_r2_self": 3, "d256_nonsquare": 3,
           "d128_n784_r6.5_self": 3, "d256_bound_edge": 3, "config2_dims": 12}


@pytest.mark.gpu
@pytest.mark.parametrize("carried", [True, False], ids=["carried", "init_levels"])
@pytest.mark.parametrize("name", sorted(CHAINED))
def test_chained_steps(name, carried):
    """forward(iters=T, return_all=True): slab t+1 against one reference step at the engine's own slab t (the prep
    kernel's and K2's shadows, group 0's H reused after step 0, the ping-pong buffers); forward(iters=T) and
    forward(iters=T-1) are bit-identical to the matching slabs."""
    T = CHAINED[name]
    m, img, S, n = _model(name, "bf16", seed=1)
    start = S.to(DEV) if carried else None
    with torch.no_grad():
        states = m(img.to(DEV), iters=T, levels=start, return_all=True).cpu()
        for t in (T, T - 1):
            assert torch.equal(m(img.to(DEV), iters=t, levels=start).cpu(), states[t]), t
    tok, P, pos, mask = _ref_inputs(m, img, n)
    worst_errs = {}
    for t in range(T):
        errs = errors({"state": states[t + 1]}, {"state": _emu(m, tok, P, pos, mask, states[t])["state"]},
                      tuple(S.shape))
        check(errs, TOL["emu"], (name, carried, t))
        worst_errs[f"state@{t + 1}"] = errs["state"]
    _report(name, f"T={T} carried={carried} vs step_forward_bf16", worst_errs)


@pytest.mark.gpu
@pytest.mark.parametrize("name,steps", [("d320_n144_r3", [2, 0, 3, 1, 3]), ("d128_n784_r6.5_self", [1, 3])])
def test_per_image_steps(name, steps):
    """forward(iters=<vector>, return_all=True) runs the SETTLE kernel instantiations: a running image's slab t+1 passes
    the one-step check at its slab t, a stopped image's later slabs equal its last one bit for bit."""
    m, img, S, n = _model(name, "bf16", seed=2, batch=len(steps))
    T = max(steps)
    with torch.no_grad():
        states = m(img.to(DEV), iters=torch.tensor(steps), levels=S.to(DEV), return_all=True).cpu()
    tok, P, pos, mask = _ref_inputs(m, img, n)
    _, _, L, d = S.shape
    worst_errs = {}
    for t in range(T):
        ref = _emu(m, tok, P, pos, mask, states[t])["state"]
        for b, k in enumerate(steps):
            if k <= t:
                assert torch.equal(states[t + 1, b], states[t, b]), (b, t)
                continue
            errs = errors({"state": states[t + 1, b:b + 1]}, {"state": ref[b:b + 1]}, (1, n, L, d))
            check(errs, TOL["emu"], (name, b, t))
            worst_errs[f"img{b}@{t + 1}"] = errs["state"]
    _report(name, f"steps={steps} vs step_forward_bf16", worst_errs)


# dim, patch, (H, W), batch: tokeniser tiles of 64 / 128 / 256 columns, 3p^2 = 48 and 588 (not multiples of 64), rows
# that end in a partial 256-row block
TOKENISER = [(64, 4, (12, 12), 3), (128, 14, (70, 98), 9), (192, 14, (42, 56), 5), (256, 4, (40, 40), 3),
             (512, 14, (224, 224), 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("dim,p,hw,B", TOKENISER, ids=[f"d{t[0]}_p{t[1]}_{t[2][0]}x{t[2][1]}_B{t[3]}" for t in TOKENISER])
def test_tensor_core_tokeniser(dim, p, hw, B):
    """m.tokens (bf16 patches and weight, wgmma GEMM) against the bf16-operand tokeniser in float64."""
    import glom_pytorch_b200 as G
    isz = max(hw)
    params = O.synth_params(dim, 2, isz, p, seed=4)
    m = G.Glom(dim=dim, levels=2, image_size=isz, patch_size=p, precision="bf16")
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=False)
    m = m.to(DEV)
    img = torch.randn((B, 3) + hw, generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        tok = m.tokens(img.to(DEV)).cpu()
    w, b = (torch.from_numpy(params[k]).double() for k in ("image_to_tokens.1.weight", "image_to_tokens.1.bias"))
    ref = OT.bf16(OT.patchify(img.double(), p)) @ OT.bf16(w).T + b
    n = tok.shape[1]
    errs = errors({"tokens": tok}, {"tokens": ref}, (B, n, 1, dim))
    _report(f"d{dim}_p{p}", "tokeniser", errs)
    check(errs, TOL["tok"], (dim, p, hw, B))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["d192_n36", "d128_n256_r2_self", "d192_n144_r3_self_subeps", "d192_n144_self_only"])
def test_fp32_engine_steps(name):
    """The fp32 CUDA-core engine: one step from a carried state and a chain of 3 steps from init_levels, each slab
    against column_step at the engine's previous slab."""
    m, img, S, n = _model(name, "fp32")
    tok, P, pos, mask = _ref_inputs(m, img, n)
    with torch.no_grad():
        out = m(img.to(DEV), iters=1, levels=S.to(DEV)).cpu()
        states = m(img.to(DEV), iters=3, return_all=True).cpu()
    errs = {"one step": errors({"state": out}, {"state": _exact(m, tok, P, pos, mask, S)}, tuple(S.shape))["state"]}
    for t in range(3):
        errs[f"state@{t + 1}"] = errors({"state": states[t + 1]}, {"state": _exact(m, tok, P, pos, mask, states[t])},
                                        tuple(S.shape))["state"]
    _report(name, "fp32 engine vs column_step", errs)
    check(errs, TOL["simt"], name)
