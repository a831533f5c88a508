"""The backward against a float64 reference evaluated at the engine's own states (oracle/glom_oracle_torch.py).

`grads_at_states` chains one-step float64 VJPs of `column_step`, each taken at the forward's states S_0..S_T: that is
what the engine's backward computes (its fp32 or tensor-core backward at the states its forward produced), so the
forward's own rounding drops out and the bounds hold at every step count.  `step_backward_bf16` is one reverse step of
the tensor-core backward with the engine's bf16 roundings and nothing else: a tighter check of the same launch.

Metric (`errors`): every gradient is cut into the blocks its kernels tile -- state-like tensors per (image, level),
weight gradients per group and 256 x 256 tile, biases per group, d_pos per 64-row block (rows >= n must be exactly zero),
d_img per image -- and each block's rel-Frobenius error is taken against max(|ref block|, FLOOR * rms block norm of the
tensor).  `rel` is the worst block over every tensor, `abs` the worst max-abs error over the tensor's max |ref|.

The CPU tests pin the reference (identities with full autograd to ~1e-12, the live reference's golden gradients) and
show that each bound catches plausible kernel faults by >= 3x.  The GPU tests run every backward path at the shapes
where its kernels tile, mask and skip.

Bounds (rel, abs), set at about 3x the worst value observed over all the GPU tests of the path on one H100 80GB HBM3
(400 W power limit); observed maxima in brackets:
  tc      bf16 engine with tensor-core MLPs (and tensor-core attention when n % 8 == 0) vs grads_at_states
          (2e-2, 3.5e-2)  [rel 7.0e-3, abs 1.11e-2, both at the rms-20 peaky shape; 3.5e-3 .. 4.3e-3 elsewhere]
  tc_emu  the same one-step gradients vs step_backward_bf16
          (1e-3, 7e-3)    [rel 2.8e-4, abs 2.4e-3 (mixed shape)]
  simt    fp32 CUDA-core backward (fp32 engine, or bf16 engine with dim % 256 != 0) vs grads_at_states
          (3e-6, 6e-6)    [rel 8.5e-7, abs 1.9e-6]
The mixed path (tensor-core MLPs, CUDA-core attention when n % 8 != 0) takes the tc bounds; no path failed.

The edge cases, one H100 80GB HBM3 (700 W power limit), observed (rel, abs) in brackets:
  "subeps" states (key rows at norms 0 .. 2e-12 around F.normalize's eps, facing aligned queries): tc [7.7e-3, 1.3e-2],
  the clamped rows' d_levels row by row <= 1.4e-2; simt [6.4e-7, 1.1e-6], rows <= 1.6e-7.  Before the normalisation
  backward dropped the tangent projection on clamped rows these were tc 0.93 and simt 0.57.  The same states at
  tc_d256_n144_B5 and mixed_d256_n100 measured tc 2.9e-2 and fp32 4.6e-6 on d_levels, over the bounds, and are not in
  SHAPES: the clamped rows' dkhat cancels over the aligned queries and the bounds are not widened for them.
  Saturated GELUs (first-layer biases of -1e6 / +1e6 on whole tiles): tc [4.1e-3, 4.1e-3], tc_emu [1.7e-4, 6.9e-4],
  simt [6.6e-7, 9.7e-7].  With BW_PRE's old GELU tail, -1e6 gave tc rel 9.8e-2 and +1e6 tc_emu rel 8.2e-3.
  Self-only rows (radius 0.5): tc [1.2e-2, 2.1e-2] at the edge states, tc_emu [1.9e-4, 1.1e-3]; simt [6.6e-7, 8.4e-7].
  rms 80 (the forward's exact-maximum scale): tc [1.27e-2, 3.45e-2], at the edge of the abs bound, as bf16 logits of
  magnitude ~80 move A; tc_emu [1.3e-4, 5.1e-4].
The faults of test_bounds_catch_faults miss these bounds by 5.6x (rel) and 4.2x (abs) at least (projection_when_clamped
at tc).  gelu_tail_clamped is shown at biases of -1e8 (20x at tc abs); at -1e6 it misses tc by 5.1x in rel only (abs
7.0e-3), and at +1e6 only tc_emu's rel, by 6x: the saturated GPU cases therefore also run against step_backward_bf16.
"""
import math

import numpy as np
import pytest
import torch

from cases import GRAD_CASES, grad_inputs
from golden_util import GOLDEN_DIR
from oracle import glom_oracle as O
from oracle import glom_oracle_torch as OT

import test_forward_oracle as FO

DEV = "cuda:0"
FLOOR = 0.1
TOL = {"tc": (2e-2, 3.5e-2), "tc_emu": (1e-3, 7e-3), "simt": (3e-6, 6e-6)}
GOLDEN_TOL = (2e-6, 2e-6)      # fp64 reference vs the live reference's fp32 autograd (observed <= 4.1e-7)
BWD_GELU_MAX = (6e-7, 7e-6)    # normal_cdf_pdf over every float32: |gelu|, |gelu'| error (observed 3.8e-7, 4.5e-6)

NAMES = ("bottom_up.net.1.weight", "bottom_up.net.1.bias", "bottom_up.net.3.weight", "bottom_up.net.3.bias",
         "top_down.net.1.weight", "top_down.net.1.bias", "top_down.net.3.weight", "top_down.net.3.bias")


# ----------------------------------------------------------------------------- metric
def _blocks(key, x, L, n):
    """-> list of blocks of x (float64 CPU) along the structure the kernels tile."""
    if key in ("d_levels", "d_state0"):                                      # (B, n, L, d)
        return [x[b, :, l] for b in range(x.shape[0]) for l in range(x.shape[2])]
    if key in ("d_img", "d_tokens", "init_levels"):                          # per image / per level
        return list(x)
    if key == "pos_emb.weight":
        return [x[r:min(r + 64, n)] for r in range(0, n, 64)]
    if key == "image_to_tokens.1.bias":
        return [x]
    if key.endswith("bias"):                                                 # per group
        G = L if key.startswith("bottom_up") else L - 1
        return list(x.reshape(G, -1))
    if key == "image_to_tokens.1.weight":
        G, w = 1, x[None]
    else:
        G = L if key.startswith("bottom_up") else L - 1
        w = x.reshape(G, x.shape[0] // G, x.shape[1])
    return [w[g, i:i + 256, j:j + 256] for g in range(G) for i in range(0, w.shape[1], 256)
            for j in range(0, w.shape[2], 256)]


def errors(got, ref, L, n):
    """-> {key: (worst block rel-Frobenius, max-abs / max |ref|)} for the keys of `ref`."""
    out = {}
    for k, r in ref.items():
        g = torch.as_tensor(got[k]).detach().to("cpu", torch.float64)
        r = torch.as_tensor(r).to("cpu", torch.float64)
        assert g.shape == r.shape, (k, tuple(g.shape), tuple(r.shape))
        assert torch.isfinite(g).all(), k
        if k == "pos_emb.weight":
            assert not g[n:].any(), "d_pos rows >= n must be exactly zero"
        gb, rb = _blocks(k, g, L, n), _blocks(k, r, L, n)
        rms = float(torch.linalg.norm(r)) / math.sqrt(len(rb))
        rel = max(float(torch.linalg.norm(a - b)) / max(float(torch.linalg.norm(b)), FLOOR * rms, 1e-300)
                  for a, b in zip(gb, rb))
        ab = float((g - r).abs().max()) / max(float(r.abs().max()), 1e-300)
        out[k] = (rel, ab)
    return out


def worst(errs):
    return max(e[0] for e in errs.values()), max(e[1] for e in errs.values())


def check(errs, tol, what):
    rel, ab = worst(errs)
    bad = {k: e for k, e in errs.items() if e[0] > tol[0] or e[1] > tol[1]}
    assert not bad, (what, tol, bad)
    return rel, ab


# ----------------------------------------------------------------------------- CPU: the reference itself
def _small(d=32, L=3, isz=16, p=4, B=3, seed=1):
    P = {k: torch.from_numpy(v).double() for k, v in O.synth_params(d, L, isz, p, seed=seed).items()}
    n = (isz // p) ** 2
    g = torch.Generator().manual_seed(seed)
    tok = torch.randn(B, n, d, generator=g, dtype=torch.float64)
    S = torch.randn(B, n, L, d, generator=g, dtype=torch.float64)
    return P, tok, P["pos_emb.weight"][:n].clone(), S, g


def _full_autograd(P, tok, pos, S0, T, cot, return_all, steps, mask, attend_self):
    """loss = sum(out * cot) through T steps of column_step with torch autograd (per-image steps: torch.where)."""
    P = {k: P[k].clone().requires_grad_(True) for k in NAMES}
    tok, pos, S0 = (x.clone().requires_grad_(True) for x in (tok, pos, S0))
    s, hid = S0, [S0]
    for t in range(T):
        nxt = OT.column_step(s, tok, pos, P, mask, attend_self)
        if steps is not None:
            nxt = torch.where((torch.as_tensor(steps) > t)[:, None, None, None], nxt, s)
        s = nxt
        hid.append(s)
    out = torch.stack(hid) if return_all else s
    leaves = [S0, tok, pos] + [P[k] for k in NAMES]
    gr = torch.autograd.grad((out * cot).sum(), leaves, allow_unused=True)
    res = dict(zip(["d_state0", "d_tokens", "d_pos"] + list(NAMES), gr))
    return {k: (torch.zeros_like(leaves[i]) if v is None else v) for i, (k, v) in enumerate(res.items())}, torch.stack(hid)


@pytest.mark.parametrize("return_all,steps,radius,attend_self,init", [
    (True, None, 0, False, False),
    (False, None, 1.5, True, False),
    (False, None, 0, False, True),
    (True, [3, 1, 0], 1.0, False, False),
    (False, [2, 3, 1], 0, True, True),
], ids=["return_all", "last_slab_radius_self", "init_levels", "steps_return_all_radius", "steps_last_slab_init"])
def test_grads_at_states_equals_full_autograd(return_all, steps, radius, attend_self, init):
    """At the reference's own states the chain of one-step VJPs is exactly autograd through T steps."""
    T = 3
    P, tok, pos, S, g = _small()
    B, n, L, d = S.shape
    if init:                                             # carried levels vs the broadcast init_levels
        S = P["init_levels"][None, None].expand(B, n, L, d).clone()
    mask = OT.radius_mask(4, radius) if radius else None
    cot = torch.randn(((T + 1,) if return_all else ()) + (B, n, L, d), generator=g, dtype=torch.float64)
    ref, states = _full_autograd(P, tok, pos, S, T, cot, return_all, steps, mask, attend_self)
    got = OT.grads_at_states(P, tok, pos, states, cot, return_all=return_all, steps=steps, attend_self=attend_self,
                             mask=mask)
    for k, r in ref.items():
        err = float((got[k] - r).abs().max()) / max(float(r.abs().max()), 1e-300)
        assert err <= 1e-12, (k, err)
    if init:
        d_init = got["d_state0"].sum((0, 1))
        assert torch.allclose(d_init, ref["d_state0"].sum((0, 1)), rtol=1e-12, atol=0)


def test_column_step_is_glom_forward():
    """glom_forward runs column_step: float64 chains agree to the last bit."""
    P, tok, pos, S, _ = _small()
    params = {k: v.numpy() for k, v in P.items()}
    img = np.random.default_rng(0).standard_normal((3, 3, 16, 16))
    out = OT.glom_forward(params, img, patch_size=4, iters=2, levels=S, return_all=True, dtype=torch.float64)
    tok = OT.patchify(torch.from_numpy(img), 4) @ P["image_to_tokens.1.weight"].T + P["image_to_tokens.1.bias"]
    s = S
    for t in range(2):
        s = OT.column_step(s, tok, pos, P, None, False)
        assert torch.equal(s, out[t + 1])


def test_step_backward_bf16_without_rounding_is_the_exact_step(monkeypatch):
    """step_backward_bf16 is a hand-written backward: with its roundings switched off it must equal the autograd VJP,
    also on rows whose norm F.normalize clamps at 1e-12 (test_forward_oracle._subeps_state)."""
    for kind in ("random", "subeps"):
        _check_step_backward_bf16(kind, monkeypatch)


def _check_step_backward_bf16(kind, monkeypatch):
    P, tok, pos, S, g = _small(L=3)
    if kind == "subeps":
        S = FO._subeps_state(*S.shape, g, dtype=torch.float64)
    cot = torch.randn(S.shape, generator=g, dtype=torch.float64)
    for attn_tc in (True, False):
        for mask, attend_self in ((None, False), (OT.radius_mask(4, 1.5), True), (OT.radius_mask(4, 1.0), False)):
            exact = OT.grads_at_states(P, tok, pos, torch.stack([S, S]), cot, return_all=False,
                                       attend_self=attend_self, mask=mask)
            monkeypatch.setattr(OT, "bf16", lambda x: x)
            got = OT.step_backward_bf16(P, tok, pos, S, cot, attend_self=attend_self, mask=mask, attn_tc=attn_tc)
            monkeypatch.undo()
            got["d_state0"] = got.pop("d_state")
            for k, r in exact.items():
                err = float((got[k] - r).abs().max()) / float(r.abs().max())
                assert err <= 1e-12, (kind, k, attn_tc, err)
            if kind == "subeps":                      # and row by row on the clamped rows (rows just above the eps
                # lose ~1e-4 of their gradient to float64 cancellation of two 1e12-scale terms in either formula)
                r, a = exact["d_state0"][0, :5, FO.SUBEPS_LEVEL], got["d_state0"][0, :5, FO.SUBEPS_LEVEL]
                err = float(((a - r).norm(dim=-1) / r.norm(dim=-1)).max())
                assert err <= 1e-12, (kind, attn_tc, err)
            # and the roundings are live: bf16 moves every tensor by about 2^-9 relative
            rounded = OT.step_backward_bf16(P, tok, pos, S, cot, attend_self=attend_self, mask=mask, attn_tc=attn_tc)
            rel, _ = worst(errors(rounded, {k: exact[k] for k in NAMES}, 3, 16))
            assert 1e-4 < rel < 5e-2, rel


def _golden_reference(name):
    """grads_at_states at the float64 oracle's own states for a GRAD_CASES fixture, mapped to the reference's names."""
    case = GRAD_CASES[name]
    params = O.synth_params(case["dim"], case["levels"], case["image_size"], case["patch_size"], seed=case["param_seed"])
    img, lv, cot = grad_inputs(case)
    p, L = case["patch_size"], case["levels"]
    radius = case.get("local_consensus_radius", 0)
    states = OT.glom_forward(params, img, patch_size=p, iters=case["iters"], levels=lv, return_all=True,
                             consensus_self=case.get("consensus_self", False), local_consensus_radius=radius,
                             dtype=torch.float64)
    P = {k: torch.from_numpy(v).double() for k, v in params.items()}
    tok = OT.patchify(torch.from_numpy(img).double(), p) @ P["image_to_tokens.1.weight"].T + P["image_to_tokens.1.bias"]
    n = tok.shape[1]
    mask = OT.radius_mask(case["image_size"] // p, radius) if radius else None
    g = OT.grads_at_states(P, tok, P["pos_emb.weight"][:n], states, cot, return_all=case["return_all"],
                           attend_self=case.get("consensus_self", False), mask=mask)
    return case, params, img, n, g


def _map_reference(g, params, img, p, n, carried):
    """grads_at_states output -> the engine's / reference's parameter names (+ d_img, d_levels or d_init_levels)."""
    out = {k: g[k] for k in NAMES}
    tg = OT.token_grads(img, params["image_to_tokens.1.weight"], params["image_to_tokens.1.bias"], p, g["d_tokens"])
    out.update(tg)
    dpos = torch.zeros(params["pos_emb.weight"].shape, dtype=torch.float64)
    dpos[:n] = g["d_pos"]
    out["pos_emb.weight"] = dpos
    if carried:
        out["d_levels"] = g["d_state0"]
    else:
        out["init_levels"] = g["d_state0"].sum((0, 1))
    return out


@pytest.mark.parametrize("name", sorted(GRAD_CASES))
def test_reference_matches_golden_gradients(name):
    """The float64 reference against the live reference's fp32 autograd (tests/golden/make_golden_grads.py)."""
    import os
    case, params, img, n, g = _golden_reference(name)
    with np.load(os.path.join(GOLDEN_DIR, name + ".npz")) as z:
        gold = {k: z[k] for k in z.files}
    carried = bool(case.get("with_levels"))
    got = _map_reference(g, params, img, case["patch_size"], n, carried)
    ref = {k: gold[k] for k in got if k in ("d_img", "d_levels")}
    ref.update({k: gold["d_" + k] for k in got if k not in ("d_img", "d_levels")})
    if carried:
        assert not gold["d_init_levels"].any()
    check(errors(got, ref, case["levels"], n), GOLDEN_TOL, name)


def _normal_cdf_pdf_f32(x, tail_clamped=False):
    """tc_bwd_kernels.cu normal_cdf_pdf in float32 as written (each fmaf rounded once, ex2.approx as a rounded exp2),
    -> (gelu, gelu') = (x cdf, fmaf(x, pdf, cdf)) as BW_PRE forms them.  tail_clamped: the fit evaluated at min(|x|, 6)
    past 6 as well, as it was before the tail was zeroed there."""
    f32 = np.float32

    def fmaf(a, b, c):
        return (a.astype(np.float64) * b.astype(np.float64) + c).astype(f32)
    x = np.asarray(x, f32)
    a = np.abs(x)
    t = np.minimum(a, f32(6))
    q = np.full_like(t, 3.290448512416333e-05)
    for c in (-0.0007621519616805017, 0.008038812316954136, -0.05331535264849663, -0.45887142419815063,
              -1.1511567831039429, -0.9999995827674866):
        q = fmaf(q, t, f32(c))
    tail = np.exp2(q.astype(np.float64)).astype(f32)
    if not tail_clamped:
        tail = np.where(a > 6, f32(0), tail)
    cdf = np.where(x >= 0, f32(1) - tail, tail)
    hz = np.full_like(t, 7.497369551856536e-06)
    for c in (-0.00023059015802573413, 0.003048981074243784, -0.023022783920168877, 0.11135400831699371,
              0.6360868811607361, 0.7979033589363098):
        hz = fmaf(hz, t, f32(c))
    pdf = tail * hz
    return x * cdf, fmaf(x, pdf, cdf)


def test_backward_gelu_fit_within_documented_bound():
    """BW_PRE's GELU and GELU derivative (a fit of Phi(-|x|) and of the hazard on [0, 6], the tail zero past 6) stay
    within BWD_GELU_MAX of the erf form for every float32, finite, including +-0 and +-3.4e38."""
    from scipy.special import ndtr
    x = np.concatenate([np.linspace(-12, 12, 2_000_001), [0.0, -0.0, 6.0, -6.0, 30.0, -30.0, 1e4, -1e4, 1e30, -1e30,
                                                         3.4e38, -3.4e38]]).astype(np.float32)
    h, gp = _normal_cdf_pdf_f32(x)
    xd = x.astype(np.float64)
    with np.errstate(over="ignore"):
        pdf = np.exp(-0.5 * xd * xd) / math.sqrt(2 * math.pi)
    cdf = ndtr(xd)
    assert np.isfinite(h).all() and np.isfinite(gp).all()
    for what, got, want, bound in (("gelu", h, xd * cdf, BWD_GELU_MAX[0]),
                                   ("gelu'", gp, cdf + np.where(pdf > 0, xd * pdf, 0.0), BWD_GELU_MAX[1])):
        err = np.abs(got.astype(np.float64) - want)
        print(f"[bwd-oracle] BW_PRE {what} fit: max error {err.max():.3e} at x = {xd[err.argmax()]:.6g}")
        assert err.max() <= bound, (what, float(err.max()), float(xd[err.argmax()]))
    assert h[x == 0].max() == 0.0
    # before the tail was zeroed past 6 the derivative grew as x phi(6)
    _, old = _normal_cdf_pdf_f32(np.float32([-1e6, 1e6, 3.4e38]), tail_clamped=True)
    assert abs(old[0]) > 6e-3 and old[1] > 1.006 and old[2] > 1e30, old


# ----------------------------------------------------------------------------- CPU: the bounds catch faults
SATURATED = 1e6


def _saturate(params, d, sign, scale=SATURATED, seed=7):
    """First-layer biases of bottom-up group 1 and top-down group 0 (numpy arrays, modified in place): units 0..255, a
    whole 256-unit tile of BW_PRE, at sign * scale, far outside the GELU fit's interval [-6, 6]; the other units of both
    groups at magnitudes 10^1 .. 10^6 of both signs."""
    rng = np.random.default_rng(seed)
    for key, grp in (("bottom_up.net.1.bias", 1), ("top_down.net.1.bias", 0)):
        b = params[key].reshape(-1, 4 * d)
        b[grp] = rng.choice([-1.0, 1.0], 4 * d) * 10.0 ** rng.uniform(1, 6, 4 * d)
        b[grp, :256] = sign * scale


def _fault_inputs(d, L, isz, B, kind):
    """One reverse step at a state of rms `kind` (p = 4: an (isz/4)^2 grid of columns), or at a "subeps" state, or at a
    random state with first-layer biases saturated at a signed scale such as "-1e6" (_saturate)."""
    P, tok, pos, S, g = _small(d=d, L=L, isz=isz, p=4, B=B, seed=3)
    if kind == "subeps":
        S = FO._subeps_state(*S.shape, g, dtype=torch.float64)
    elif isinstance(kind, str) and kind[0] in "+-":
        _saturate({k: P[k].numpy() for k in ("bottom_up.net.1.bias", "top_down.net.1.bias")}, d,
                  math.copysign(1.0, float(kind)), abs(float(kind)))
    else:
        S = S * kind
    return P, tok, pos, torch.stack([S, S]), torch.randn(S.shape, generator=g, dtype=torch.float64)


class _GeluTailClamped(torch.autograd.Function):
    """gelu and its derivative as BW_PRE computed them before the tail was zeroed past |x| = 6."""
    @staticmethod
    def forward(ctx, x):
        h, gp = _normal_cdf_pdf_f32(x.detach().numpy(), tail_clamped=True)
        ctx.save_for_backward(torch.from_numpy(gp.astype(np.float64)))
        return torch.from_numpy(h.astype(np.float64))

    @staticmethod
    def backward(ctx, g):
        return g * ctx.saved_tensors[0]


def _gelu_tail_clamped_ff(x, w1, b1, w2, b2):
    B, n, G, d = x.shape
    a = x.permute(2, 0, 1, 3).reshape(G, B * n, d)
    h = _GeluTailClamped.apply(torch.baddbmm(b1.reshape(G, 1, 4 * d), a, w1.reshape(G, 4 * d, d).transpose(1, 2)))
    y = torch.baddbmm(b2.reshape(G, 1, d), h, w2.reshape(G, d, 4 * d).transpose(1, 2))
    return y.reshape(G, B, n, d).permute(1, 2, 0, 3)


def _faulty_ff(x, w1, b1, w2, b2):
    """Rows of the last partial 128-row block add nothing to the weight gradients (their dx is still right)."""
    B, n, G, d = x.shape
    R = B * n
    keep = torch.zeros(R, dtype=torch.bool)
    keep[:128 * (R // 128)] = True
    keep = keep.reshape(B, n)[..., None, None]
    live = _ORIG_FF(x, w1, b1, w2, b2)
    dead = _ORIG_FF(x, w1.detach(), b1.detach(), w2.detach(), b2.detach())
    return torch.where(keep, live, dead)


_ORIG_FF = OT._grouped_ff
_ORIG_CONS = OT._consensus


def _consensus_variant(fault):
    def cons(levels, attend_self, mask):
        B, n, L, d = levels.shape
        q = levels.permute(0, 2, 1, 3)
        norm = levels.norm(dim=-1, keepdim=True).clamp_min(1e-12)
        if fault == "projection_when_clamped":       # (dk - khat (khat . dk)) / max(|S|, eps) on every row
            s0, r0 = levels.detach(), 1.0 / norm.detach()
            k = levels * (r0 - r0 ** 3 * (s0 * (levels - s0)).sum(-1, keepdim=True))
        else:
            k = levels / (norm.detach() if fault == "no_projection" else norm)
        k = k.permute(0, 2, 1, 3)
        sim = torch.matmul(q, k.transpose(-1, -2)) * (d ** -0.5)
        if not attend_self:
            eye = torch.eye(n, dtype=torch.bool)[None, None]
            if fault == "diag_grad":                     # forward value filled, gradient not zeroed
                sim = torch.where(eye, sim - sim.detach() + OT.TOKEN_ATTEND_SELF_VALUE, sim)
            else:
                sim = sim.masked_fill(eye, OT.TOKEN_ATTEND_SELF_VALUE)
        if mask is not None:
            sim = sim.masked_fill(mask[None, None], -torch.finfo(sim.dtype).max)
        attn = sim.softmax(dim=-1)
        v = q
        if fault == "dv_keys_256":
            v = torch.cat((q[:, :, :256], q[:, :, 256:].detach()), dim=2)
        return torch.matmul(attn, v).permute(0, 2, 1, 3)
    return cons


def _faulty_pos_step(levels, tokens, pos, P, mask, attend_self):
    """The last top-down group gets the positional embedding without its gradient."""
    L = levels.shape[2]
    contrib = torch.full((L,), 4.0, dtype=levels.dtype)
    contrib[-1] = 3.0
    lwi = torch.cat((tokens[:, :, None, :], levels), dim=-2)
    bu = OT._grouped_ff(lwi[..., :-1, :], P["bottom_up.net.1.weight"], P["bottom_up.net.1.bias"],
                        P["bottom_up.net.3.weight"], P["bottom_up.net.3.bias"])
    pe = pos[None, :, None, :].expand(1, pos.shape[0], L - 1, pos.shape[1])
    pe = torch.cat((pe[:, :, :-1], pe[:, :, -1:].detach()), dim=2)
    td = OT._grouped_ff(lwi[..., 2:, :] + pe, P["top_down.net.1.weight"], P["top_down.net.1.bias"],
                        P["top_down.net.3.weight"], P["top_down.net.3.bias"])
    td = torch.nn.functional.pad(td, (0, 0, 0, 1))
    return (levels + bu + td + OT._consensus(levels, attend_self, mask)) / contrib[None, None, :, None]


# fault -> (d, L, image_size, B, rms) of inputs where that part of the backward carries weight: 800 rows (the last
# 128-row block holds 32) and n = 400 > 256 keys; rms 20 makes the softmax peaky so dsim and the normalisation matter;
# the diagonal of a 2 x 2 grid holds a quarter of each softmax row; rows of one level below the eps of F.normalize;
# 512 hidden units per group, half of them saturated
FAULTS = {
    "partial_block_dw": (64, 3, 80, 2, 1.0),
    "dv_keys_256": (64, 3, 80, 2, 20.0),
    "diag_grad": (64, 2, 8, 2, 10.0),
    "no_projection": (64, 3, 80, 2, 20.0),
    "missing_td_pos": (64, 3, 80, 2, 1.0),
    "projection_when_clamped": (64, 3, 80, 2, "subeps"),
    "gelu_tail_clamped": (128, 3, 40, 2, "-1e8"),
}


@pytest.mark.parametrize("fault", sorted(FAULTS))
def test_bounds_catch_faults(fault, monkeypatch):
    """Each faulty reference misses every bound of the GPU tests by >= 3x in both metrics, so a kernel with that fault
    fails them."""
    P, tok, pos, states, cot = _fault_inputs(*FAULTS[fault])
    kw = dict(return_all=False, attend_self=False, mask=None)
    good = OT.grads_at_states(P, tok, pos, states, cot, **kw)
    if fault == "partial_block_dw":
        monkeypatch.setattr(OT, "_grouped_ff", _faulty_ff)
    elif fault == "gelu_tail_clamped":
        monkeypatch.setattr(OT, "_grouped_ff", _gelu_tail_clamped_ff)
    elif fault == "missing_td_pos":
        monkeypatch.setattr(OT, "column_step", _faulty_pos_step)
    else:
        monkeypatch.setattr(OT, "_consensus", _consensus_variant(fault))
    bad = OT.grads_at_states(P, tok, pos, states, cot, **kw)
    monkeypatch.undo()
    rel, ab = worst(errors(bad, good, states.shape[3], states.shape[2]))
    print(f"[bwd-oracle] fault {fault}: rel {rel:.3e} abs {ab:.3e}")
    for path, (t_rel, t_abs) in TOL.items():
        assert rel >= 3 * t_rel and ab >= 3 * t_abs, (fault, path, rel, ab)


def test_unfaulted_variants_are_the_reference(monkeypatch):
    """The fault helpers without a fault reproduce the reference (so the faults, not the helpers, make the difference)."""
    P, tok, pos, states, cot = _fault_inputs(*FAULTS["dv_keys_256"])
    good = OT.grads_at_states(P, tok, pos, states, cot, return_all=False)
    monkeypatch.setattr(OT, "_consensus", _consensus_variant(None))
    again = OT.grads_at_states(P, tok, pos, states, cot, return_all=False)
    assert worst(errors(again, good, 3, states.shape[2]))[0] <= 1e-12


# ----------------------------------------------------------------------------- GPU
# name: dim, L, image_size, patch, img_hw, B, kwargs, path, rms
SHAPES = {
    # rows 720 (ragged 128 / 256 blocks), n % 64 = 16 (partial K blocks in BW_BATCH)
    "tc_d256_n144_B5": (256, 3, 48, 4, None, 5, {}, "tc", 1.0),
    # three M tiles per BW_BATCH problem (the last one 64 rows), 9 K blocks, radius mask + self in a_b / dsim_b
    "tc_d256_n576_mask_self": (256, 2, 96, 4, None, 1, dict(local_consensus_radius=2.5, consensus_self=True), "tc", 1.0),
    # four M tiles, 16 K blocks
    "tc_d256_n1024": (256, 2, 64, 2, None, 1, {}, "tc", 1.0),
    # sparse mask without self, peaky softmax
    "tc_d256_n256_r1_peaky": (256, 4, 64, 4, None, 2, dict(local_consensus_radius=1), "tc", 20.0),
    # d / 256 = 3 (BW_DW / BW_DX tiling), L = 2
    "tc_d768_L2": (768, 2, 32, 4, None, 3, {}, "tc", 1.0),
    # configs[1] dims (G = 11)
    "tc_config2_dims": (512, 6, 224, 14, None, 2, {}, "tc", 1.0),
    # tensor-core MLP + CUDA-core attention (n % 8 = 4), rows 300
    "mixed_d256_n100": (256, 3, 40, 4, None, 3, {}, "mixed", 1.0),
    # ragged gemm_f32 tiles, masked softmax backward
    "simt_d192_n144_mask_self": (192, 3, 48, 4, None, 2, dict(local_consensus_radius=3, consensus_self=True), "simt", 1.0),
    # d slices, long rows
    "simt_d320_n576": (320, 2, 96, 4, None, 1, {}, "simt", 1.0),
    # non-square image: n = 32 of 64 patches, d_pos rows >= n exactly zero
    "simt_d128_nonsquare": (128, 3, 32, 4, (16, 32), 2, {}, "simt", 1.0),
    # key rows at norms 0 .. 2e-12, on both sides of F.normalize's eps, facing aligned queries
    # (test_forward_oracle._subeps_state): their gradients, ~1e8 .. 1e11, are dkhat / eps with no projection
    "tc_d256_n576_mask_self_subeps": (256, 2, 96, 4, None, 1, dict(local_consensus_radius=2.5, consensus_self=True),
                                      "tc", "subeps"),
    "simt_d192_n144_mask_self_subeps": (192, 3, 48, 4, None, 2, dict(local_consensus_radius=3, consensus_self=True),
                                        "simt", "subeps"),
    # a radius below 1: every row's only key is itself, A is one-hot and dsim exactly zero; n = 784 runs the forward in
    # key passes of 512 + 272; "edge" (test_forward_oracle._edge_state) puts both forward stabilisers on such rows
    "tc_d256_n256_self_only": (256, 2, 64, 4, None, 2, dict(local_consensus_radius=0.5), "tc", 1.0),
    "tc_d256_n784_self_only_self": (256, 2, 56, 2, None, 1, dict(local_consensus_radius=0.5, consensus_self=True), "tc",
                                    1.0),
    "tc_d256_n256_self_only_self_edge": (256, 3, 64, 4, None, 2, dict(local_consensus_radius=0.5, consensus_self=True),
                                         "tc", "edge"),
    "tc_d256_n784_self_only_edge": (256, 3, 56, 2, None, 2, dict(local_consensus_radius=0.5), "tc", "edge"),
    "simt_d192_n144_self_only": (192, 3, 48, 4, None, 2, dict(local_consensus_radius=0.5), "simt", 1.0),
    # logits of magnitude ~80, the forward's exact-maximum scale (test_forward_oracle cons_d128_n576_exact)
    "tc_d256_n576_rms80": (256, 2, 96, 4, None, 1, {}, "tc", 80.0),
}
# first-layer biases saturated at a signed scale (_saturate): a table of its own, as a +1e6 bias grows the state by
# ~1e6 per step, so the chained runs of SHAPES do not apply; the signs are separate cases because a 1e6-scale dW tile
# raises the FLOOR * rms under which the other tiles are compared
GELU_SHAPES = {
    "tc_d256_n144_gelu_neg": (256, 3, 48, 4, None, 2, {}, "tc", "-1e6"),
    "tc_d256_n144_gelu_pos": (256, 3, 48, 4, None, 2, {}, "tc", "+1e6"),
    "simt_d192_n144_gelu_neg": (192, 3, 48, 4, None, 2, {}, "simt", "-1e6"),
    "simt_d192_n144_gelu_pos": (192, 3, 48, 4, None, 2, {}, "simt", "+1e6"),
}
TC_SHAPES = [k for k, v in SHAPES.items() if v[7] != "simt"]
SIMT_SHAPES = [k for k, v in SHAPES.items() if v[7] == "simt"]
CHAINED = ["tc_d256_n144_B5", "tc_d256_n576_mask_self", "tc_d768_L2", "mixed_d256_n100", "simt_d192_n144_mask_self",
           "simt_d128_nonsquare"]


def _spec(name):
    return SHAPES[name] if name in SHAPES else GELU_SHAPES[name]


def _model(name, precision, seed=0, batch=None):
    dim, L, isz, p, hw, B, kw, path, kind = _spec(name)
    B = batch or B
    import glom_pytorch_b200 as G
    params = O.synth_params(dim, L, isz, p, seed=seed)
    if name in GELU_SHAPES:
        _saturate(params, dim, math.copysign(1.0, float(kind)), abs(float(kind)))
    m = G.Glom(dim=dim, levels=L, image_size=isz, patch_size=p, precision=precision, **kw)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=False)
    m = m.to(DEV)
    hw = hw or (isz, isz)
    n = (hw[0] // p) * (hw[1] // p)
    g = torch.Generator().manual_seed(seed + 17)
    img = torch.randn((B, 3) + hw, generator=g)
    S = FO._state(1.0 if name in GELU_SHAPES else kind, B, n, L, dim, g)
    return m, img, S, n, g


def _mask(m, n):
    side, d2 = m.attention.mask_params(n)
    if not side:
        return None
    co = torch.stack(torch.meshgrid(torch.arange(side), torch.arange(side), indexing="ij"), -1).reshape(-1, 2)
    return ((co[:, None] - co[None]) ** 2).sum(-1) > d2


def _engine_run(m, img, S, iters, return_all, cot):
    """loss = sum(out * cot) through the engine -> (out, gradients by name)."""
    for q in m.parameters():
        q.grad = None
    x = img.to(DEV).requires_grad_(True)
    lv = None if S is None else S.to(DEV).requires_grad_(True)
    out = m(x, iters=iters, levels=lv, return_all=return_all)
    (out * cot.to(DEV)).sum().backward()
    torch.cuda.synchronize()
    got = {"d_img": x.grad}
    if lv is not None:
        got["d_levels"] = lv.grad
    got.update({k: q.grad for k, q in m.named_parameters() if q.grad is not None})
    return out.detach(), got


def _reference(m, img, states, cot, *, return_all, steps=None, carried=True):
    """grads_at_states fed with the engine's own tokens, positions and states."""
    n = states.shape[2]
    with torch.no_grad():
        tok = m.tokens(img.to(DEV)).cpu()
    P = {k: q.detach().cpu() for k, q in m.named_parameters()}
    g = OT.grads_at_states(P, tok, P["pos_emb.weight"][:n], states.cpu(), cot, return_all=return_all, steps=steps,
                           attend_self=m.attention.attend_self, mask=_mask(m, n))
    params = {k: v.numpy() for k, v in P.items()}
    return _map_reference(g, params, img, m.patch_size, n, carried), P, tok


def _report(name, what, errs):
    rel, ab = worst(errs)
    print(f"[bwd-oracle] {name} {what}: rel {rel:.3e} abs {ab:.3e}")


def _path(name, precision):
    return "simt" if precision == "fp32" or _spec(name)[7] == "simt" else "tc"


def _subeps_rows(got, ref, tol, what):
    """On a "subeps" state the clamped rows' gradients swamp their (image, level) block: the d_levels rows whose norm
    is below 1e-12 each against max(|ref row|, FLOOR * rms of the level's ordinary rows).  The rows just above the eps
    are left to the block metric: their keys are aligned with every query, so the exact tangent part of dkhat is zero and
    fp32 leaves ~1e-7 |dkhat| / |S| of it, far above their own O(1) gradient."""
    g = got["d_levels"][0, :, FO.SUBEPS_LEVEL].detach().to("cpu", torch.float64)
    r = torch.as_tensor(ref["d_levels"])[0, :, FO.SUBEPS_LEVEL].to(torch.float64)
    k = sum(x < 1e-12 for x in FO.SUBEPS_NORMS)
    rms = float(r[len(FO.SUBEPS_NORMS):].norm(dim=-1).square().mean().sqrt())
    err = (g[:k] - r[:k]).norm(dim=-1) / r[:k].norm(dim=-1).clamp_min(FLOOR * rms)
    print(f"[bwd-oracle] {what} d_levels, clamped rows: " + " ".join(f"{float(e):.2e}" for e in err))
    assert float(err.max()) <= tol[0], (what, tol, err.tolist())


def _one_step(name, precision):
    m, img, S, n, g = _model(name, precision)
    cot = torch.randn(S.shape, generator=g)
    out, got = _engine_run(m, img, S, 1, False, cot)
    ref, P, tok = _reference(m, img, torch.stack([S, out.cpu()]), cot, return_all=False)
    errs = errors(got, ref, m.levels, n)
    _report(name, f"one step {precision}", errs)
    check(errs, TOL[_path(name, precision)], (name, precision))
    if _spec(name)[8] == "subeps":
        _subeps_rows(got, ref, TOL[_path(name, precision)], (name, precision))
    return m, img, S, n, cot, got, P, tok


def _vs_step_backward_bf16(name):
    m, img, S, n, cot, got, P, tok = _one_step(name, "bf16")
    emu = OT.step_backward_bf16(P, tok, P["pos_emb.weight"][:n], S, cot, attend_self=m.attention.attend_self,
                                mask=_mask(m, n), attn_tc=_spec(name)[7] == "tc")
    emu["d_state0"] = emu.pop("d_state")
    ref = _map_reference(emu, {k: v.numpy() for k, v in P.items()}, img, m.patch_size, n, True)
    errs = errors(got, ref, m.levels, n)
    _report(name, "one step vs step_backward_bf16", errs)
    check(errs, TOL["tc_emu"], name)
    if _spec(name)[8] == "subeps":
        _subeps_rows(got, ref, TOL["tc_emu"], (name, "step_backward_bf16"))


@pytest.mark.gpu
@pytest.mark.parametrize("name", TC_SHAPES)
def test_tensor_core_backward_one_step(name):
    """One step at a random state: every gradient against grads_at_states, and against step_backward_bf16 (the same
    roundings as the kernels) with a tighter bound."""
    _vs_step_backward_bf16(name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GELU_SHAPES))
def test_backward_one_step_saturated_gelu(name):
    """One step with whole 256-unit tiles of pre at -1e6 or +1e6: BW_PRE's gelu and gelu' (tensor-core path, also
    against step_backward_bf16) or gelu_bwd_kernel (CUDA-core path, both engines) far outside the GELU fit's interval."""
    if GELU_SHAPES[name][7] == "simt":
        for precision in ("bf16", "fp32"):
            _one_step(name, precision)
    else:
        _vs_step_backward_bf16(name)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("name", SIMT_SHAPES)
def test_cuda_core_backward_one_step(name, precision):
    _one_step(name, precision)


def _chained(name, precision, return_all, carried):
    T = 3
    m, img, S, n, g = _model(name, precision, seed=1)
    cot = torch.randn(((T + 1,) if return_all else ()) + tuple(S.shape), generator=g)
    start = S if carried else None
    if return_all:
        out, got = _engine_run(m, img, start, T, True, cot)
        states = out.cpu()
    else:
        with torch.no_grad():
            states = m(img.to(DEV), iters=T, levels=None if start is None else start.to(DEV), return_all=True).cpu()
        out, got = _engine_run(m, img, start, T, False, cot)
        assert torch.equal(out.cpu(), states[T])
    ref, _, _ = _reference(m, img, states, cot, return_all=return_all, carried=carried)
    errs = errors(got, ref, m.levels, n)
    _report(name, f"T={T} return_all={return_all} carried={carried} {precision}", errs)
    check(errs, TOL[_path(name, precision)], (name, precision, return_all, carried))


@pytest.mark.gpu
@pytest.mark.parametrize("name", CHAINED)
def test_backward_chained_return_all(name):
    """forward(iters=3, return_all=True) with a cotangent on every slab, at the returned slabs."""
    _chained(name, "bf16", True, True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tc_d256_n576_mask_self", "mixed_d256_n100", "simt_d128_nonsquare"])
def test_backward_chained_last_slab_from_init_levels(name):
    """Without return_all, starting from init_levels: d_init_levels sums dL/dS_0 over images and columns."""
    _chained(name, "bf16", False, False)


@pytest.mark.gpu
@pytest.mark.parametrize("name", SIMT_SHAPES)
def test_fp32_engine_backward_chained(name):
    _chained(name, "fp32", True, True)
    _chained(name, "fp32", False, False)


@pytest.mark.gpu
@pytest.mark.parametrize("name,steps", [("mixed_d256_n100", [3, 1, 0]), ("tc_d256_n576_mask_self", [1, 3]),
                                        ("tc_d256_n144_B5", [0, 3, 1, 3, 2])])
def test_backward_per_image_steps(name, steps):
    """forward(iters=<vector>, return_all=True): a stopped image is the identity, its cotangents pass through."""
    m, img, S, n, g = _model(name, "bf16", seed=2, batch=len(steps))
    T = max(steps)
    cot = torch.randn((T + 1,) + tuple(S.shape), generator=g)
    out, got = _engine_run(m, img, S, torch.tensor(steps), True, cot)
    ref, _, _ = _reference(m, img, out.cpu(), cot, return_all=True, steps=steps)
    errs = errors(got, ref, m.levels, n)
    _report(name, f"steps={steps}", errs)
    check(errs, TOL["tc"], (name, steps))
