"""settle's implicit backward (glom_b200_backward_implicit) against float64 at the backward oracle's shapes and value
regimes, pass by pass.

The implicit backward is the one caller of backward_run that sets `state_only` (adjoint passes: no BW_DW, no bias sums,
no token / pos scatter), `relin` (passes 2..K and the parameter pass reuse pass 1's pre / h, shadows, khat / rnorm and
softmax probabilities; only gs -> gsb is recast) and `skip_attn` (the parameter pass has no consensus backward).
test_settle_implicit.py checks it at four shapes at ordinary values; this file runs it where the shared kernels were
once wrong (test_backward_oracle.py): keys below F.normalize's eps, self-only softmax rows, rms-80 logits, saturated
GELUs, n up to 1024, d 768 and configs[1] dims.

GPU:
  (1) adjoint_tol = -1, adjoint_iters = K in {0, 1, 3} at every shape of test_backward_oracle's SHAPES and GELU_SHAPES,
      at the state S of that table: every gradient per block against implicit_grads (K + 1 copies of S in float64),
      at the backward oracle's bound of the path.  K = 0 is the parameter pass alone, K = 1 one state-only pass and a
      relinearised parameter pass, K = 3 adds relinearised adjoint passes.  The identity holds at any S.
      At the tensor-core and mixed shapes also against the same passes with the kernels' bf16 roundings (EMU_TOL).
  (2) the same call against the engine's own explicit backward of K + 1 steps at repeated states: the same bits at
      K = 0, EXPLICIT_TOL at K = 1 and 3;
  (3) partial stops inside shared 128 / 256-row blocks (four images per 256-row block; configs[1] dims with a ragged last
      block): K_b and q are settle's rule on the engine's own q table, the gradients match implicit_grads with the
      per-image K_b, a zero cotangent stops its image at pass 1 with q = 0 and contributes exactly zero, and a level
      without cotangent does not stop its image;
  (4) gradients at 2^k cot are 2^k times those at cot bit for bit, K_b and q identical, for k in [-24, 24];
  (5) two runs and SM-count targets 2 and 3 give the default grid's bits at the regime shapes.
CPU: the pass-by-pass float64 reference is implicit_grads, the reference is linear in the cotangent bit for bit, and
each fault of (6) misses the bounds of (1) and (3) by >= 3x in both metrics.

Observed values are beside each bound below and in DESIGN.md, "Implicit gradients through settle".
"""
import contextlib
import math

import numpy as np
import pytest
import torch

from glom_pytorch_b200 import _native
from glom_pytorch_b200.glom import _aligned_bytes
from oracle import glom_oracle_torch as OT

import test_backward_oracle as BO
import test_forward_oracle as FO
import test_settle_implicit as TSI

DEV = "cuda:0"
FIXED_K = (0, 1, 3)
# engine Grads fields -> the reference's names (d_pos under the name whose blocks BO.errors cuts per 64 rows)
GRAD_KEYS = dict(zip(("d_bu_w1", "d_bu_b1", "d_bu_w2", "d_bu_b2", "d_td_w1", "d_td_b1", "d_td_w2", "d_td_b2"),
                     OT.MLP_KEYS))
GRAD_KEYS.update(d_tokens="d_tokens", d_pos="pos_emb.weight")
REGIMES = sorted(BO.SHAPES) + sorted(BO.GELU_SHAPES)
FLT_MAX, FLT_MIN = float(np.finfo(np.float32).max), float(np.finfo(np.float32).tiny)


def _report(what, errs):
    rel, ab = BO.worst(errs)
    wr, wa = max(errs, key=lambda k: errs[k][0]), max(errs, key=lambda k: errs[k][1])
    print(f"[implicit-oracle] {what}: rel {rel:.3e} ({wr}) abs {ab:.3e} ({wa})")


def _named(got):
    return {GRAD_KEYS[k]: v for k, v in got.items()}


# ---------------------------------------------------------------------------------------------- float64, pass by pass
def _vjp_state(P, tok, pos, S, v, attend_self, mask):
    s = S.clone().requires_grad_(True)
    return torch.autograd.grad(OT.column_step(s, tok, pos, P, mask, attend_self), s, v)[0]


def _vjp_params(P, tok, pos, S, v, attend_self, mask):
    Pl = {k: P[k].clone().requires_grad_(True) for k in OT.MLP_KEYS}
    tk, ps = tok.clone().requires_grad_(True), pos.clone().requires_grad_(True)
    out = OT.column_step(S, tk, ps, Pl, mask, attend_self)
    gr = torch.autograd.grad(out, [tk, ps] + [Pl[k] for k in OT.MLP_KEYS], v)
    return dict(zip(["d_tokens", "pos_emb.weight"] + list(OT.MLP_KEYS), gr))


_ORIG_CONS = OT._consensus


def _no_consensus_grad(levels, attend_self, mask):
    return _ORIG_CONS(levels.detach(), attend_self, mask)


@contextlib.contextmanager
def _fault_in(fault, phase, relin):
    """The reference's step as the engine would run it with `fault`, in an adjoint pass or the parameter pass."""
    swap = {}
    if fault == "adjoint_without_consensus" and phase == "adjoint":
        swap["_consensus"] = _no_consensus_grad
    elif fault == "projection_when_clamped" and relin:
        swap["_consensus"] = BO._consensus_variant("projection_when_clamped")
    elif fault == "gelu_tail_clamped" and relin:
        swap["_grouped_ff"] = BO._gelu_tail_clamped_ff
    old = {k: getattr(OT, k) for k in swap}
    for k, v in swap.items():
        setattr(OT, k, v)
    try:
        yield
    finally:
        for k, v in old.items():
            setattr(OT, k, v)


def implicit_by_passes(P, tok, pos, S, cot, K, *, attend_self=False, mask=None, fault=None):
    """The engine's algorithm in float64: u_0 = g; pass k = 1..max K_b computes J^T u_{k-1} at S and sets
    u_k = g + J^T u_{k-1} for the images with K_b >= k; then one parameter VJP at S with cotangent u.
    -> ([u_0, u_1, ...], {d_tokens, pos_emb.weight (n rows), MLP_KEYS}).  `fault` names a fault of (6)."""
    P = {k: OT._f64(P[k]) for k in OT.MLP_KEYS}
    tok, pos, S, cot = (OT._f64(x) for x in (tok, pos, S, cot))
    K = torch.as_tensor(K).to("cpu", torch.int64)
    us = [cot]
    for k in range(1, int(K.max()) + 1):
        with _fault_in(fault, "adjoint", k > 1):
            jtu = _vjp_state(P, tok, pos, S, us[-1], attend_self, mask)
        running = (K >= k)[:, None, None, None]
        stopped = jtu if fault == "stopped_u_overwritten" else us[-1]
        us.append(torch.where(running, cot + jtu, stopped))
    with _fault_in(fault, "param", len(us) > 1):
        grads = _vjp_params(P, tok, pos, S, us[-1], attend_self, mask)
        if fault == "stale_gsb" and len(us) > 1:         # the MLPs see bf16(u_{K-1}), the b2 sums fp32 u_K
            stale = _vjp_params(P, tok, pos, S, us[-2], attend_self, mask)
            grads = {k: (v if k.endswith("net.3.bias") else stale[k]) for k, v in grads.items()}
    return us, grads


def emulated_by_passes(P, tok, pos, S, cot, K, *, attend_self=False, mask=None, attn_tc=True):
    """The same passes with the tensor-core backward's bf16 roundings: pass k is OT.step_backward_bf16 at S with
    cotangent u_{k-1} (the relinearised passes reuse pass 1's shadows, pre / h, khat and probabilities, which are what a
    fresh step at S rounds them to), the parameter pass its MLP gradients with cotangent u_K."""
    K = torch.as_tensor(K).to("cpu", torch.int64)
    cot = OT._f64(cot)
    u = cot
    for k in range(1, int(K.max()) + 1):
        ds = OT.step_backward_bf16(P, tok, pos, S, u, attend_self=attend_self, mask=mask, attn_tc=attn_tc)["d_state"]
        u = torch.where((K >= k)[:, None, None, None], cot + ds, u)
    g = OT.step_backward_bf16(P, tok, pos, S, u, attend_self=attend_self, mask=mask, attn_tc=attn_tc)
    out = {k: g[k] for k in OT.MLP_KEYS}
    out["d_tokens"], out["pos_emb.weight"] = g["d_tokens"], g["d_pos"]
    return out


def _reference(P, tok, pos, S, cot, K, attend_self=False, mask=None):
    g = TSI.implicit_grads(P, tok, pos, S, cot, K, attend_self=attend_self, mask=mask)
    g["pos_emb.weight"] = g.pop("d_pos")
    return g


def _close(got, want, tol, what):
    for k, w in want.items():
        err = float((got[k] - w).abs().max()) / max(float(w.abs().max()), 1e-300)
        assert err <= tol, (what, k, err)


# ---------------------------------------------------------------------------------------------------------- CPU
def _tiny_case(kind, K):
    """A tiny contracting float64 model at its fixed point, or at a "subeps" state, or with first-layer biases
    saturated at a signed scale such as "-1e6" (BO._saturate); a cotangent; the per-image pass counts K."""
    if kind == "subeps":
        P, tok, pos, S, cot = TSI._tiny(seed=3, d=16, side=3, scale=0.6)
        S = FO._subeps_state(*S.shape, torch.Generator().manual_seed(4), dtype=torch.float64)
    elif isinstance(kind, str):
        P, tok, pos, S, cot = TSI._tiny(seed=3, d=64, scale=0.6)
        BO._saturate({k: P[k].numpy() for k in ("bottom_up.net.1.bias", "top_down.net.1.bias")}, 64,
                     math.copysign(1.0, float(kind)), abs(float(kind)))
    else:
        P, tok, pos, S, cot = TSI._tiny(seed=3, scale=0.6)
    return P, tok, pos, S, cot, torch.tensor(K)


def test_passes_are_implicit_grads():
    """The pass-by-pass reference (the engine's order: Neumann sum first, one parameter VJP) is implicit_grads (K + 1
    copies of S, the cotangent chained through them) at ordinary, sub-eps and saturated states."""
    for kind, K in ((1.0, [3, 1]), (1.0, [0, 0]), ("subeps", [3, 2]), ("-1e6", [3, 3]), ("+1e6", [2, 3])):
        P, tok, pos, S, cot, K = _tiny_case(kind, K)
        us, got = implicit_by_passes(P, tok, pos, S, cot, K)
        assert len(us) == int(K.max()) + 1
        _close(got, _reference(P, tok, pos, S, cot, K), 1e-11, (kind, K.tolist()))


def test_emulation_without_rounding_is_the_reference(monkeypatch):
    """emulated_by_passes with bf16 rounding switched off is implicit_grads, on both attention paths."""
    for kind, K in ((1.0, [3, 1]), ("subeps", [2, 3])):
        P, tok, pos, S, cot, K = _tiny_case(kind, K)
        want = _reference(P, tok, pos, S, cot, K)
        monkeypatch.setattr(OT, "bf16", lambda x: x)
        for attn_tc in (True, False):
            _close(emulated_by_passes(P, tok, pos, S, cot, K, attn_tc=attn_tc), want, 1e-11, (kind, attn_tc))
        monkeypatch.undo()


def test_reference_is_linear_in_the_cotangent_bit_for_bit():
    """Every float64 operation on the cotangent commutes with 2^k: the premise of the GPU scaling test."""
    P, tok, pos, S, cot, K = _tiny_case(1.0, [3, 1])
    base = _reference(P, tok, pos, S, cot, K)
    for k in (-24, -7, 5, 24):
        got = _reference(P, tok, pos, S, cot * 2.0 ** k, K)
        for key, v in base.items():
            assert torch.equal(got[key], v * 2.0 ** k), (k, key)


# fault -> (state kind, K): each in the regime it hides in.  adjoint_without_consensus: skip_attn leaking into the
# state-only passes; projection_when_clamped: the tangent projection on clamped rows in passes 2..K; gelu_tail_clamped:
# gelu' held at its value at 6 past |x| = 6 in the relinearised passes; stale_gsb: the parameter pass with u_{K-1}
# (gsb not recast after the last update; the second-layer bias sums read fp32 gs = u_K); stopped_u_overwritten: a
# stopped image's u replaced by J^T u in the passes after it stopped
FAULTS = {
    "adjoint_without_consensus": (1.0, [3, 2]),
    "projection_when_clamped": ("subeps", [3, 3]),
    "gelu_tail_clamped_neg": ("-1e8", [3, 3]),
    "gelu_tail_clamped_pos": ("+1e8", [3, 3]),
    "stale_gsb": (1.0, [3, 3]),
    "stopped_u_overwritten": (1.0, [1, 3]),
}


@pytest.mark.parametrize("fault", sorted(FAULTS))
def test_bounds_catch_faults(fault):
    """Each fault misses the bounds of the GPU comparisons with implicit_grads (BO.TOL tc and simt) by >= 3x in both
    metrics; its unfaulted twin is the reference."""
    P, tok, pos, S, cot, K = _tiny_case(*FAULTS[fault])
    B, n, L, d = S.shape
    good = _reference(P, tok, pos, S, cot, K)
    _close(implicit_by_passes(P, tok, pos, S, cot, K)[1], good, 1e-11, (fault, "twin"))
    _, bad = implicit_by_passes(P, tok, pos, S, cot, K, fault=fault.replace("_neg", "").replace("_pos", ""))
    errs = BO.errors(bad, good, L, n)
    _report(f"fault {fault}", errs)
    rel, ab = BO.worst(errs)
    for path in ("tc", "simt"):
        t_rel, t_abs = BO.TOL[path]
        assert rel >= 3 * t_rel and ab >= 3 * t_abs, (fault, path, rel, ab)


# ---------------------------------------------------------------------------------------------------------- GPU
def _regime_case(name):
    """test_backward_oracle's model and state S of `name`, a random cotangent and the engine's tokens (on the GPU)."""
    m, img, S, n, g = BO._model(name, "bf16")
    cot = torch.randn(S.shape, generator=g)
    with torch.no_grad():
        tokens = m.tokens(img.to(DEV))
    return m, tokens, S.to(DEV).contiguous(), cot.to(DEV), n


def _engine_reference(m, tokens, S, cot, K, emulated=False, attn_tc=True):
    n = S.shape[1]
    P = {k: q.detach().cpu() for k, q in m.named_parameters()}
    args = (P, tokens.cpu(), P["pos_emb.weight"][:n], S.cpu(), cot.cpu(), K)
    kw = dict(attend_self=m.attention.attend_self, mask=BO._mask(m, n))
    return emulated_by_passes(*args, attn_tc=attn_tc, **kw) if emulated else _reference(*args, **kw)


# the engine against emulated_by_passes: each pass adds one step's worth of rounding decisions that fall differently in
# fp32 and float64 (BO.TOL["tc_emu"] bounds one step), so the bound is set at ~3x the worst of K = 3 on one H100 80GB
# HBM3 (rel 1.37e-3 at tc_config2_dims, abs 2.5e-3 at tc_d768_L2; K = 0: 2.8e-4, 1.8e-3; K = 1: 6.0e-4, 2.4e-3)
EMU_TOL = (4e-3, 7.5e-3)
# the engine against its explicit backward on repeated states, ~3x the worst observed (rel 6.0e-3, abs 5.9e-3, both at
# tc_d256_n576_rms80 K = 3; 2.9e-3 .. 4.6e-3 elsewhere)
EXPLICIT_TOL = (2e-2, 2e-2)
# (name, K) whose float64 comparison exceeds the tensor-core bound by the bf16 algorithm's own error: the engine matches
# the bf16 emulation there (EMU_TOL; rel 4.6e-4 and 6.0e-4), and the bound is not widened for them.  Observed (rel, abs) on
# one H100 80GB HBM3:
F64_OVER = {
    # u_1's clamped rows (~1e11) are one reverse step's, whose dkhat cancels over the aligned queries (the block metric's
    # per-row 1.4e-2 of test_backward_oracle); the level-1 second-layer bias sums those rows and cancels again
    ("tc_d256_n576_mask_self_subeps", 1): (2.2e-2, 5.0e-2),
    # bf16 logits of magnitude ~80 move A (one step: at the edge of the abs bound), three passes compound it
    ("tc_d256_n576_rms80", 3): (2.0e-2, 8.6e-2),
}


@pytest.mark.gpu
@pytest.mark.parametrize("K", FIXED_K)
@pytest.mark.parametrize("name", REGIMES)
def test_fixed_passes_match_the_reference(name, K):
    m, tokens, S, cot, n = _regime_case(name)
    got, steps, _ = TSI._engine(m, tokens, S, cot, K, -1.0)
    B = S.shape[0]
    assert steps.tolist() == [K] * B
    Kb = torch.full((B,), K)
    errs = BO.errors(_named(got), _engine_reference(m, tokens, S, cot, Kb), m.levels, n)
    _report(f"{name} K={K}", errs)
    path = BO._path(name, "bf16")
    if (name, K) not in F64_OVER:
        BO.check(errs, BO.TOL[path], (name, K))
    if path == "tc":            # and the bf16 algorithm: what the kernels round, pass by pass
        emu = _engine_reference(m, tokens, S, cot, Kb, emulated=True, attn_tc=BO._spec(name)[7] == "tc")
        errs = BO.errors(_named(got), emu, m.levels, n)
        _report(f"{name} K={K} vs the bf16 emulation", errs)
        BO.check(errs, EMU_TOL, (name, K, "emulated"))


def _explicit(m, tokens, S, cot, K):
    """glom_b200_backward (deterministic) of K + 1 steps at S, K + 2 repeated states, the cotangent on the last."""
    b, n = tokens.shape[:2]
    cfg = m.engine_cfg(n)
    wts = [q.detach().float().contiguous() for q in m._mlp_params()]
    names = ("d_bu_w1", "d_bu_b1", "d_bu_w2", "d_bu_b2", "d_td_w1", "d_td_b1", "d_td_w2", "d_td_b2")
    want = {"d_tokens": torch.zeros_like(tokens), "d_pos": torch.zeros(n, m.dim, device=DEV)}
    want.update({k: torch.zeros_like(w) for k, w in zip(names, wts)})
    want["d_state0"] = torch.zeros_like(S)
    states = S[None].expand((K + 2,) + tuple(S.shape)).contiguous()
    ws = _aligned_bytes(_native.backward_workspace_bytes(cfg, b), torch.device(DEV))
    pos = m.pos_emb.weight[:n].detach().contiguous()
    _native.backward(cfg, [w.data_ptr() for w in wts], tokens.data_ptr(), pos.data_ptr(), states.data_ptr(),
                         cot.data_ptr(), {k: v.data_ptr() for k, v in want.items()}, b, K + 1, False, ws.data_ptr(),
                         ws.numel(), torch.cuda.current_stream().cuda_stream, deterministic=True)
    torch.cuda.synchronize()
    want.pop("d_state0")
    return want


EXPLICIT = BO.TC_SHAPES + sorted(k for k, v in BO.GELU_SHAPES.items() if v[7] != "simt")


@pytest.mark.gpu
@pytest.mark.parametrize("name", EXPLICIT)
def test_fixed_passes_match_the_explicit_backward(name):
    """K = 0: the parameter pass (no consensus backward) is the explicit one-step backward's MLP half, bit for bit.
    K = 1, 3: u_K = sum_k (J^T)^k g rounded to bf16 once, against the unrolled backward rounding each (J^T)^k g."""
    m, tokens, S, cot, n = _regime_case(name)
    for K in FIXED_K:
        got = TSI._engine(m, tokens, S, cot, K, -1.0)[0]
        want = _explicit(m, tokens, S, cot, K)
        if K == 0:
            for k in got:
                assert torch.equal(got[k], want[k]), (name, k)
            continue
        errs = BO.errors(_named(got), _named(want), m.levels, n)
        _report(f"{name} K={K} vs the explicit backward", errs)
        BO.check(errs, EXPLICIT_TOL, (name, K))


# (dim, levels, image_size, patch_size, consensus_self, local_consensus_radius, batch, path): TSI.SHAPES' layout
PARTIAL = {
    # n = 64: four images per 256-row block, two per 128-row block
    "tc_d256_n64_B8": (256, 3, 32, 4, False, 0, 8, "tc"),
    # configs[1] dims at n = 144: 432 rows, images 1 and 2 straddle 256-row blocks, the last block holds 176 rows
    "tc_config2_dims_n144_B3": (512, 6, 168, 14, False, 0, 3, "tc"),
}
PASSES = 6


def _partial_case(name, monkeypatch):
    """TSI._setup's settled state at a PARTIAL shape, and a cotangent with per-image structure: image 0 none at all,
    image 1 none on its top level, the others their levels scaled over one to three decades (up or down)."""
    monkeypatch.setitem(TSI.SHAPES, name, PARTIAL[name])
    m, tokens, S, cot = TSI._settled(name)
    B, L = S.shape[0], S.shape[2]
    cot = cot.clone()
    cot[0] = 0
    cot[1, :, L - 1] = 0
    for b in range(2, B):
        sign = 1 if b % 2 else -1
        cot[b] *= (10.0 ** (sign * (b // 2) * torch.arange(L, device=DEV) / (L - 1)))[None, :, None]
    return m, tokens, S, cot.contiguous()


def _q_table(m, tokens, S, cot):
    """q of passes 1..PASSES with no image stopped: (PASSES, B, L)."""
    table = []
    for k in range(1, PASSES + 1):
        _, K, q = TSI._engine(m, tokens, S, cot, k, -1.0)
        assert K.tolist() == [k] * S.shape[0]
        table.append(q.cpu())
    return torch.stack(table)


def _splitting_tol(table):
    """The q value of the table at which settle's rule gives the most distinct K_b."""
    cands = sorted(set(float(x) for x in table.amax(-1).flatten() if 0 < float(x) < 1))
    return max(cands, key=lambda t: (len(torch.unique(OT.settle_rule(table, t))), -t))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(PARTIAL))
def test_partial_stops_inside_shared_blocks(name, monkeypatch):
    m, tokens, S, cot = _partial_case(name, monkeypatch)
    B, n, L, d = S.shape
    table = _q_table(m, tokens, S, cot)
    assert torch.isfinite(table).all()
    assert not table[:, 0].any()                                      # 0/0 = 0 on every level of image 0
    assert float(table[0, 1, L - 1]) == 1.0                           # u_0 = 0 there: |u_1 - u_0| = |u_1|
    assert (table[:, 1:] > 0).all()
    split = _splitting_tol(table)
    first = table.amax(-1)                                            # (PASSES, B)
    exact = float(first[2, 2])
    alone = float(table[0, 1, :L - 1].max())                          # image 1's other levels meet it at pass 1
    tols = [split, exact, float(np.nextafter(np.float32(exact), np.float32(0))), alone]
    for tol in tols:
        got, K, q = TSI._engine(m, tokens, S, cot, PASSES, tol)
        want = OT.settle_rule(table, tol)
        assert torch.equal(K.cpu(), want), (name, tol, K.tolist(), want.tolist())
        for b, k in enumerate(want.tolist()):
            assert torch.equal(q[b].cpu(), table[k - 1, b]), (name, tol, b)
        assert int(K[0]) == 1 and not q[0].any() and not got["d_tokens"][0].any(), (name, tol)
        print(f"[implicit-oracle] {name} tol {tol:.9g}: K {K.tolist()}")
        if tol == split:
            assert len(torch.unique(K)) >= 3, (name, K.tolist())
            errs = BO.errors(_named(got), _engine_reference(m, tokens, S, cot, K.cpu()), L, n)
            _report(f"{name} K={K.tolist()}", errs)
            BO.check(errs, BO.TOL["tc"], (name, K.tolist()))
    assert int(OT.settle_rule(table, exact)[2]) <= 3
    if alone < 1:
        assert int(OT.settle_rule(table, alone)[1]) >= 2                # the level without cotangent keeps it running


# (source, name, adjoint_iters, adjoint_tol): real settled states (TSI._settled) under settle's rule, and a state of
# test_backward_oracle with three fixed passes
SCALE_CASES = {
    "tc_settled": ("TSI", "tensor_core_bwd_n144", 8, 1e-4),
    "simt_settled": ("TSI", "cuda_core_bwd_n64", 8, 1e-4),
    "tc_relin_K3": ("BO", "tc_d256_n144_B5", 3, -1.0),
}
SCALES = range(-24, 25)
MARGIN = 2.0 ** 8               # between the float64 extremes below and fp32's range, for the engine's own rounding


def _check_scale_range(us, grads, part_w, what):
    """From the float64 reference: at every 2^k of SCALES, every element of u_k and of the gradients, and every squared
    partial of u_k - u_{k-1} and u_k over part_w columns, stays finite in fp32 and (if non-zero) normal."""
    B, n, L, d = us[0].shape
    k_lo, k_hi = min(SCALES), max(SCALES)
    vals, sq = [], []
    for k, u in enumerate(us):
        vals.append(u.flatten())
        if k:
            for x in (u - us[k - 1], u):
                sq.append(x.reshape(B * n, L, d // part_w, part_w).square().sum(-1).flatten())
    vals += [v.flatten() for v in grads.values()]
    for what_, x, p in (("elements", torch.cat(vals).abs(), 1), ("squared partials", torch.cat(sq), 2)):
        nz = x[x > 0]
        hi, lo = float(nz.max()), float(nz.min())
        print(f"[implicit-oracle] {what} {what_}: {lo:.3e} .. {hi:.3e}")
        assert hi * 2.0 ** (p * k_hi) * MARGIN < FLT_MAX, (what, what_, hi)
        assert lo * 2.0 ** (p * k_lo) > FLT_MIN * MARGIN, (what, what_, lo)


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(SCALE_CASES))
def test_power_of_two_scaling_is_exact(case):
    src, name, iters, tol = SCALE_CASES[case]
    if src == "TSI":
        m, tokens, S, cot = TSI._settled(name)
    else:
        m, tokens, S, cot, _ = _regime_case(name)
    torch.use_deterministic_algorithms(True)
    try:
        base, K, q = TSI._engine(m, tokens, S, cot, iters, tol)
        n = S.shape[1]
        P = {k: v.detach().cpu() for k, v in m.named_parameters()}
        us, grads = implicit_by_passes(P, tokens.cpu(), P["pos_emb.weight"][:n], S.cpu(), cot.cpu(), K.cpu(),
                                       attend_self=m.attention.attend_self, mask=BO._mask(m, n))
        _check_scale_range(us, grads, OT.forward_tiles(m.dim)[1], case)
        for k in SCALES:
            got, K2, q2 = TSI._engine(m, tokens, S, (cot * 2.0 ** k).contiguous(), iters, tol)
            assert torch.equal(K2, K) and torch.equal(q2, q), (case, k, K2.tolist(), K.tolist())
            for key, v in base.items():
                assert torch.equal(got[key], v * 2.0 ** k), (case, k, key)
    finally:
        torch.use_deterministic_algorithms(False)
    print(f"[implicit-oracle] {case}: K {K.tolist()}, 2^k cot for k in [{min(SCALES)}, {max(SCALES)}] bit for bit")


GRID_REGIMES = [k for k in REGIMES if k in BO.GELU_SHAPES or BO.SHAPES[k][8] != 1.0 or "self_only" in k]


@pytest.mark.gpu
@pytest.mark.parametrize("name", GRID_REGIMES + sorted(PARTIAL))
def test_bits_across_runs_and_sm_counts(name, monkeypatch):
    """Under the deterministic flag: a second run and SM-count targets 2 and 3 give the default grid's bits (three fixed
    passes at the regime shapes, settle's rule with a splitting tol at the partial-stop shapes)."""
    import test_sm_count as TS
    from test_deterministic_backward import deterministic
    if name in PARTIAL:
        m, tokens, S, cot = _partial_case(name, monkeypatch)
        iters, tol = PASSES, _splitting_tol(_q_table(m, tokens, S, cot))
    else:
        m, tokens, S, cot, _ = _regime_case(name)
        iters, tol = 3, -1.0
    B, n, L, d = S.shape

    def run():
        return TS._cpu(TSI._engine(m, tokens, S, cot, iters, tol))
    with deterministic():
        want = TS._across_targets(run, (2, 3), (d, L, n, B), name)
        TS._same(run(), want, (name, "second run"))
    print(f"[implicit-oracle] {name}: K {want[1].tolist()} at the default grid, targets 2 and 3, and again")
