"""Multi-threaded torch-CPU restatement of the GLOM column update  --  TEST / BASELINE INFRASTRUCTURE, NOT PRODUCT CODE.

Same algorithm and citations as ``oracle/glom_oracle.py`` (the numpy oracle, pinned on the reference's golden
outputs), written with batched torch CPU ops (``torch.bmm`` over the MLP groups, ``F.gelu``, ``torch.softmax``) so
that it uses every host core the way the reference's own torch/oneDNN path does.  ``bench.py`` times it as the CPU
arm (``kind: "port"``) ONLY when the unmodified reference package is not importable on the box
(``$GLOM_REF_PATH`` -> ``baseline/_ref`` -> ``/root/reference``); ``tests/test_oracle_golden.py`` checks it against
the same golden fixtures as the numpy oracle.  ``column_step`` is the loop body as a differentiable float64-capable
function and ``hidden_activations`` its MLPs' hidden layer (``tests/test_cuda_core_oracle.py``);
``grads_at_states`` and ``step_backward_bf16`` are the backward references of ``tests/test_backward_oracle.py``,
``step_forward_bf16`` the one-step forward reference of ``tests/test_forward_oracle.py``, ``settle_change``,
``settle_ratio`` and ``settle_rule`` the settle references of ``tests/test_settle_oracle.py``.
Only ``tests/`` and ``bench.py``'s CPU legs may import this module.

Restates (``glom_pytorch/glom_pytorch.py``): GroupedFeedForward :23-36, ConsensusAttention.forward :56-73
(F.normalize eps 1e-12 :58, d**-0.5 :60, diagonal -5e-4 :11/:62-65 before the radius mask :67-69), image_to_tokens
:94-97, Glom.forward :110-150 (contributions 4..4,3 :128-129, Jacobi loop :131-145, return_all :147-148).
"""
import math

import torch
import torch.nn.functional as F

TOKEN_ATTEND_SELF_VALUE = -5e-4  # glom_pytorch.py:11


def _grouped_ff(x, w1, b1, w2, b2):
    """x (B, n, G, d) -> (B, n, G, d): per-group d -> 4d -> d MLP with exact-erf GELU (:27-33)."""
    B, n, G, d = x.shape
    a = x.permute(2, 0, 1, 3).reshape(G, B * n, d)                       # group-major rows
    h = F.gelu(torch.baddbmm(b1.reshape(G, 1, 4 * d), a, w1.reshape(G, 4 * d, d).transpose(1, 2)))
    y = torch.baddbmm(b2.reshape(G, 1, d), h, w2.reshape(G, d, 4 * d).transpose(1, 2))
    return y.reshape(G, B, n, d).permute(1, 2, 0, 3)


def _consensus(levels, attend_self, mask):
    """ConsensusAttention.forward (:56-73); levels (B, n, L, d)."""
    B, n, L, d = levels.shape
    q = levels.permute(0, 2, 1, 3)                                       # b l i d
    k = F.normalize(levels, dim=-1).permute(0, 2, 1, 3)                  # (:58)
    sim = torch.matmul(q, k.transpose(-1, -2)) * (d ** -0.5)             # (:60)
    if not attend_self:                                                  # (:62-65)
        eye = torch.eye(n, dtype=torch.bool)
        sim = sim.masked_fill(eye[None, None], TOKEN_ATTEND_SELF_VALUE)
    if mask is not None:                                                 # (:67-69)
        sim = sim.masked_fill(mask[None, None], -torch.finfo(sim.dtype).max)
    attn = sim.softmax(dim=-1)                                           # (:71)
    return torch.matmul(attn, q).permute(0, 2, 1, 3)                     # (:72)


def radius_mask(side, radius):
    """non_local_mask (:44-54): 'ij' meshgrid, '(h w) c' coordinates, cdist > radius."""
    ar = torch.arange(side)
    hh, ww = torch.meshgrid(ar, ar, indexing="ij")
    co = torch.stack((hh.reshape(-1), ww.reshape(-1)), -1).float()
    return torch.cdist(co, co) > radius


def column_step(levels, tokens, pos, P, mask, attend_self):
    """One step of the Jacobi loop (:132-144), differentiable.  levels (B, n, L, d), tokens (B, n, d), pos (n, d),
    P: reference state_dict keys -> tensors, mask: (n, n) bool (True = masked) or None."""
    L = levels.shape[2]
    contrib = torch.full((L,), 4.0, dtype=levels.dtype)                                  # (:128)
    contrib[-1] = 3.0                                                                     # (:129)
    lwi = torch.cat((tokens[:, :, None, :], levels), dim=-2)                              # (:132)
    bu = _grouped_ff(lwi[..., :-1, :], P["bottom_up.net.1.weight"], P["bottom_up.net.1.bias"],
                     P["bottom_up.net.3.weight"], P["bottom_up.net.3.bias"])              # (:134)
    td = _grouped_ff(lwi[..., 2:, :] + pos[None, :, None, :], P["top_down.net.1.weight"], P["top_down.net.1.bias"],
                     P["top_down.net.3.weight"], P["top_down.net.3.bias"])                # (:136)
    td = F.pad(td, (0, 0, 0, 1))                                                          # (:137)
    cons = _consensus(levels, attend_self, mask)                                          # (:139)
    return (levels + bu + td + cons) / contrib[None, None, :, None]                       # (:141-142)


MLP_KEYS = ("bottom_up.net.1.weight", "bottom_up.net.1.bias", "bottom_up.net.3.weight", "bottom_up.net.3.bias",
            "top_down.net.1.weight", "top_down.net.1.bias", "top_down.net.3.weight", "top_down.net.3.bias")


def _f64(x):
    return torch.as_tensor(x).detach().to(device="cpu", dtype=torch.float64)


def grads_at_states(P, tokens, pos, states, cot, *, return_all, steps=None, attend_self=False, mask=None):
    """The backward of T column steps as a chain of one-step VJPs in float64, each taken at the GIVEN states.

    states: (>= T+1, B, n, L, d) with S_0..S_T (e.g. the engine's own return_all slabs; S_T is not read); T = the
    number of steps = cot.shape[0] - 1 with `return_all` (cot: one cotangent per slab), else states.shape[0] - 1 (cot:
    the cotangent of S_T).  steps (B,) ints or None: image b is the identity at step t when steps[b] <= t: its cotangent
    passes through, and the step runs on the other images only, so it adds nothing to any other gradient whatever its
    states hold (NaN and inf included).  This is what the engine's backward computes: its fp32
    (or tensor-core) backward evaluated at its forward's states, so the forward's own rounding drops out.
    Returns float64 CPU tensors: d_state0 (dL/dS_0), d_tokens, d_pos (n, d) and one entry per MLP_KEYS name."""
    P = {k: _f64(P[k]).requires_grad_(True) for k in MLP_KEYS}
    tokens = _f64(tokens).requires_grad_(True)
    pos = _f64(pos).requires_grad_(True)
    states = _f64(states)
    cot = _f64(cot)
    T = cot.shape[0] - 1 if return_all else states.shape[0] - 1
    if mask is not None:
        mask = torch.as_tensor(mask, dtype=torch.bool, device="cpu")
    live_all = None if steps is None else torch.as_tensor(steps).to("cpu", torch.int64)
    acc = {k: torch.zeros_like(v) for k, v in P.items()}
    acc["d_tokens"] = torch.zeros_like(tokens)
    acc["d_pos"] = torch.zeros_like(pos)
    g = cot[T] if return_all else cot
    for t in range(T - 1, -1, -1):
        live = slice(None) if live_all is None else (live_all > t).nonzero().flatten()
        if live_all is None or live.numel():
            s = states[t][live].clone().requires_grad_(True)
            out = column_step(s, tokens[live], pos, P, mask, attend_self)
            leaves = [s, tokens, pos] + [P[k] for k in MLP_KEYS]
            gr = torch.autograd.grad(out, leaves, g[live], allow_unused=True)
            for k, v in zip(["d_tokens", "d_pos"] + list(MLP_KEYS), gr[1:]):
                if v is not None:
                    acc[k] += v
            g = g.clone()
            g[live] = gr[0]                                   # frozen images: the identity
        if return_all:
            g = g + cot[t]
    acc["d_state0"] = g
    return acc


def hidden_activations(P, tokens, pos, levels):
    """The MLPs' hidden activations of one step in float64: (2L-1, B*n, 4d), group g = 2l the bottom-up MLP of level l
    (input tokens for l = 0, else levels[:, :, l-1]), g = 2l+1 the top-down MLP of level l (input levels[:, :, l+1] +
    pos), H_g = gelu(A_g W1_g^T + b1_g) with the exact-erf GELU (:27-33, :134-136).  This is the engine's group order."""
    P = {k: _f64(P[k]) for k in MLP_KEYS}
    tokens, pos, levels = _f64(tokens), _f64(pos), _f64(levels)
    B, n, L, d = levels.shape
    w1 = [P["bottom_up.net.1.weight"].reshape(L, 4 * d, d), P["top_down.net.1.weight"].reshape(L - 1, 4 * d, d)]
    b1 = [P["bottom_up.net.1.bias"].reshape(L, 4 * d), P["top_down.net.1.bias"].reshape(L - 1, 4 * d)]
    H = []
    for g in range(2 * L - 1):
        net, l = g & 1, g >> 1
        a = levels[:, :, l + 1] + pos[None] if net else (tokens if l == 0 else levels[:, :, l - 1])
        H.append(F.gelu(a.reshape(B * n, d) @ w1[net][l].T + b1[net][l]))
    return torch.stack(H)


def patchify(img, p):
    """'b c (h p1) (w p2) -> b (h w) (p1 p2 c)' (:95)."""
    B, C, H, W = img.shape
    return img.reshape(B, C, H // p, p, W // p, p).permute(0, 2, 4, 3, 5, 1).reshape(B, (H // p) * (W // p), p * p * C)


def token_grads(img, weight, bias, patch_size, d_tokens):
    """image_to_tokens (:94-97) backward in float64: d_tokens (B, n, d) -> d_img, d_weight, d_bias."""
    img = _f64(img).requires_grad_(True)
    w = _f64(weight).requires_grad_(True)
    b = _f64(bias).requires_grad_(True)
    tok = F.linear(patchify(img, patch_size), w, b)
    gi, gw, gb = torch.autograd.grad(tok, (img, w, b), _f64(d_tokens))
    return {"d_img": gi, "image_to_tokens.1.weight": gw, "image_to_tokens.1.bias": gb}


def bf16(x):
    """Round to the nearest bfloat16 (ties to even), back in the input's dtype."""
    return x.to(torch.float32).to(torch.bfloat16).to(x.dtype)


def _gelu_and_grad(x):
    cdf = 0.5 * (1.0 + torch.erf(x * (0.5 ** 0.5)))
    pdf = torch.exp(-0.5 * x * x) * (2.0 * math.pi) ** -0.5
    return x * cdf, cdf + x * pdf


def step_backward_bf16(P, tokens, pos, s, g, *, attend_self=False, mask=None, attn_tc=True):
    """One reverse step of the bf16 engine's tensor-core backward, float64 except for bf16 rounding at exactly the
    points where the engine rounds.  s = S_t (B, n, L, d), g = dL/dS_{t+1} (plus that slab's own cotangent).
    Returns d_state (dL/dS_t), d_tokens, d_pos and the MLP_KEYS gradients of this step.

    Roundings (bwd_kernels.cu / tc_bwd_kernels.cu):
      bf16 shadows: xb = bf16(tokens), sb = bf16(S_t), sp = bf16(S_t[:, :, 1:] + pos), gsb = bf16(g / c)
      (cast_bf16_rows, bwd_shadows_kernel); weights w1p = w1t = bf16(W1), w2t = bf16(W2); b1 stays fp32.
      BW_PRE: pre = xb W1^T + b1 -> h = bf16(gelu(pre)), gp = bf16(gelu'(pre)).
      BW_DH: dpre = (gsb W2) * gp -> bf16(dpre); the b1 gradient sums the UNROUNDED dpre, the b2 gradient sums g / c.
      BW_DX: dx = bf16(dpre) W1.  BW_DW: dW2 += gsb^T h, dW1 += bf16(dpre)^T xb.
    With attn_tc (n % 8 == 0) the consensus backward runs on tensor cores too:
      khat_b = bf16(khat) (normalize_rows_kernel); logits = sb khat_b^T; a_b = bf16(A) (attn_softmax_kernel);
      dA = gsb sb^T; dsim_b = bf16(scale * dsim) (attn_softmax_bwd_kernel); ds += a_b^T gsb + dsim_b khat_b;
      dkhat = dsim_b^T sb; the normalisation backward is fp32 on khat, rnorm (dkhat * rnorm on rows clamped at 1e-12).
    Without attn_tc (the mixed path) the consensus backward is fp32 on S_t and g / c: exact here."""
    P = {k: _f64(P[k]) for k in MLP_KEYS}
    tokens, pos, s, g = _f64(tokens), _f64(pos), _f64(s), _f64(g)
    B, n, L, d = s.shape
    contrib = torch.full((L,), 4.0, dtype=torch.float64)
    contrib[-1] = 3.0
    gs = g / contrib[None, None, :, None]
    gsb = bf16(gs)
    sb = bf16(s)
    out = {k: torch.zeros_like(v) for k, v in P.items()}
    out["d_tokens"] = torch.zeros_like(tokens)
    out["d_pos"] = torch.zeros_like(pos)
    ds = gs.clone()                                                           # residual term (:141)
    for net, groups in (("bottom_up", L), ("top_down", L - 1)):
        W1 = P[f"{net}.net.1.weight"].reshape(groups, 4 * d, d)
        b1 = P[f"{net}.net.1.bias"].reshape(groups, 4 * d)
        W2 = P[f"{net}.net.3.weight"].reshape(groups, d, 4 * d)
        dW1, dW2 = torch.zeros_like(W1), torch.zeros_like(W2)
        db1, db2 = torch.zeros_like(b1), torch.zeros(groups, d, dtype=torch.float64)
        for l in range(groups):
            if net == "bottom_up":
                x = bf16(tokens if l == 0 else s[:, :, l - 1])
            else:
                x = bf16(s[:, :, l + 1] + pos[None])
            x = x.reshape(B * n, d)
            dy = gsb[:, :, l].reshape(B * n, d)
            w1b, w2b = bf16(W1[l]), bf16(W2[l])
            hv, gp = _gelu_and_grad(x @ w1b.T + b1[l])
            h, gp = bf16(hv), bf16(gp)
            dpre = (dy @ w2b) * gp
            db1[l] = dpre.sum(0)
            db2[l] = gs[:, :, l].reshape(B * n, d).sum(0)
            dpre = bf16(dpre)
            dW2[l] = dy.T @ h
            dW1[l] = dpre.T @ x
            dx = (dpre @ w1b).reshape(B, n, d)
            if net == "bottom_up" and l == 0:
                out["d_tokens"] += dx
            elif net == "bottom_up":
                ds[:, :, l - 1] += dx
            else:
                ds[:, :, l + 1] += dx
                out["d_pos"] += dx.sum(0)
        out[f"{net}.net.1.weight"] = dW1.reshape(groups * 4 * d, d, 1)
        out[f"{net}.net.1.bias"] = db1.reshape(-1)
        out[f"{net}.net.3.weight"] = dW2.reshape(groups * d, 4 * d, 1)
        out[f"{net}.net.3.bias"] = db2.reshape(-1)
    # consensus (:56-73), per (image, level): q = v = S_t, k = normalize(S_t)
    q = s.permute(0, 2, 1, 3)                                                 # b l i d
    dc = gs.permute(0, 2, 1, 3)
    nrm = q.norm(dim=-1, keepdim=True)
    rn = 1.0 / nrm.clamp_min(1e-12)
    khat = q * rn
    scale = d ** -0.5
    fixed = torch.zeros(n, n, dtype=torch.bool)
    if not attend_self:
        fixed |= torch.eye(n, dtype=torch.bool)
    if mask is not None:
        fixed |= torch.as_tensor(mask, dtype=torch.bool)
    if attn_tc:
        qs, kk, dcs = bf16(q), bf16(khat), bf16(dc)
    else:
        qs, kk, dcs = q, khat, dc
    logits = (qs @ kk.transpose(-1, -2)) * scale
    if not attend_self:
        logits = logits.masked_fill(torch.eye(n, dtype=torch.bool)[None, None], TOKEN_ATTEND_SELF_VALUE)
    if mask is not None:
        logits = logits.masked_fill(torch.as_tensor(mask, dtype=torch.bool)[None, None], -math.inf)
    A = logits.softmax(-1)
    dA = dcs @ qs.transpose(-1, -2)
    dsim = (A * (dA - (A * dA).sum(-1, keepdim=True))).masked_fill(fixed[None, None], 0.0)
    if attn_tc:
        ab, dsb = bf16(A), bf16(scale * dsim)
    else:
        ab, dsb = A, scale * dsim
    dq = ab.transpose(-1, -2) @ dcs + dsb @ kk
    dk = dsb.transpose(-1, -2) @ qs
    # a row clamped at eps (|S| < 1e-12) is S / 1e-12, linear in S: its gradient has no tangent projection
    dq = dq + torch.where(nrm < 1e-12, dk, dk - khat * (khat * dk).sum(-1, keepdim=True)) * rn
    ds += dq.permute(0, 2, 1, 3)
    out["d_state"] = ds
    return out


LOG2E = 1.4426950408889634
ATTN_BOUND_MAX = 96.0          # attn_kernel: a 16-row warp with a logit bound beyond this takes the exact running maximum


def forward_tiles(d):
    """(bn, part_w) of the bf16 engine at dim d: K2's N tile and the columns of one squared-norm partial."""
    bn = 256 if d % 256 == 0 else 128 if d % 128 == 0 else 64
    return bn, 64 if bn == 256 else bn // 2


def _fwd_k1_operands(xb, sb, sp):
    """K1's A operand of each MLP group, (B, n, d): group 2l = bottom-up l (tokens, then S[l-1]), 2l+1 = top-down l."""
    L = sb.shape[2]
    ops = []
    for l in range(L):
        ops.append(xb if l == 0 else sb[:, :, l - 1])
        if l < L - 1:
            ops.append(sp[:, :, l])
    return ops


def _fwd_key_norm(nsq):
    """attn_row_norm: |S_j| from its squared-norm partials (..., nparts)."""
    return nsq.sum(-1).sqrt()


def _fwd_attn_logits(q, rs, attend_self, mask):
    """attn_kernel's logits in log2 units, (b, l, i, j): (sb_i . sb_j) rs_j, then the diagonal fill, then the mask."""
    n = q.shape[-2]
    x = (q @ q.transpose(-1, -2)) * rs[..., None, :]
    if not attend_self:
        x = x.masked_fill(torch.eye(n, dtype=torch.bool), TOKEN_ATTEND_SELF_VALUE * LOG2E)
    if mask is not None:
        x = x.masked_fill(mask, -math.inf)
    return x


def _fwd_attn_passes(n):
    """Key ranges (key0, nk) of the launches of attn_kernel: one up to 576 keys, else passes of 512."""
    if n <= 576:
        return [(0, n)]
    return [(k0, min(512, n - k0)) for k0 in range(0, n, 512)]


def _fwd_consensus(sb, nrm, attend_self, mask):
    """attn_kernel (K3) in float64 with its bf16 roundings.  sb (B, n, L, d) bf16 values, nrm (B, n, L) key norms."""
    B, n, L, d = sb.shape
    q = sb.permute(0, 2, 1, 3)                                                # b l i d
    nrm = nrm.permute(0, 2, 1)
    c = d ** -0.5 * LOG2E
    rs, bound = c / nrm.clamp_min(1e-12), c * nrm
    logits = _fwd_attn_logits(q, rs, attend_self, mask)
    n16 = -(-n // 16) * 16
    over = F.pad(~(bound <= ATTN_BOUND_MAX), (0, n16 - n)).reshape(B, L, n16 // 16, 16).any(-1)
    exact = over.repeat_interleave(16, -1)[..., :n, None]                      # per 16-row warp
    bnd = bound[..., None]
    passes = _fwd_attn_passes(n)
    keys = 256 if len(passes) == 1 and 128 < n16 <= 256 else 128
    ninf = torch.tensor(-math.inf, dtype=torch.float64)
    zero = torch.zeros((), dtype=torch.float64)
    m_acc = torch.full_like(bnd, -math.inf)
    l_acc = torch.zeros_like(bnd)
    o_acc = torch.zeros(B, L, n, d, dtype=torch.float64)
    for k0, nk in passes:
        m_run = torch.where(exact, ninf, bnd)
        l_run = torch.zeros_like(bnd)
        blocks = []
        for j0 in range(k0, k0 + nk, keys):
            x = logits[..., j0:min(j0 + keys, k0 + nk)]
            m_new = torch.maximum(m_run, x.amax(-1, keepdim=True))
            m_ex = torch.where(m_new == -math.inf, zero, m_new)
            l_run = torch.where(exact & (m_run > -math.inf), l_run * torch.exp2(m_run - m_ex), torch.where(exact, zero, l_run))
            m_run = torch.where(exact, m_new, m_run)
            m_safe = torch.where(exact, m_ex, bnd)
            e = torch.exp2(x - m_safe)
            l_run = l_run + e.sum(-1, keepdim=True)
            blocks.append((bf16(e), m_safe))
        # exact path: every block's P onto the final maximum, rounded to bf16 a second time
        m_fin = torch.where(m_run == -math.inf, zero, m_run)
        p = torch.cat([torch.where(exact & (mu != m_fin), bf16(pb * torch.exp2(mu - m_fin)), pb) for pb, mu in blocks], -1)
        o = p @ q[..., k0:k0 + nk, :]
        m_pass = torch.where(l_run == 0, ninf, m_run)                        # no unmasked key in this pass
        m_new = torch.maximum(m_acc, m_pass)
        f_old = torch.where(m_acc == -math.inf, zero, torch.exp2(m_acc - m_new))
        f_new = torch.where(m_pass == -math.inf, zero, torch.exp2(m_pass - m_new))
        l_acc = l_acc * f_old + l_run * f_new
        o_acc = o_acc * f_old + o * f_new
        m_acc = m_new
    return bf16(o_acc / l_acc).permute(0, 2, 1, 3)


def _fwd_k2(S, H, C, w2bu, w2td, b2, contrib):
    """K2: S' = ((S + (acc + b2)) + C) / c_l with acc = H_bu,l W2bu_l^T + H_td,l W2td_l^T.  H (G, B*n, 4d)."""
    B, n, L, d = S.shape
    acc = []
    for l in range(L):
        a = H[2 * l] @ w2bu[l].T
        if l < L - 1:
            a = a + H[2 * l + 1] @ w2td[l].T
        acc.append(a.reshape(B, n, d))
    acc = torch.stack(acc, 2)
    return ((S + (acc + b2)) + C) / contrib[None, None, :, None]


def step_forward_bf16(P, tokens, pos, S, *, attend_self=False, mask=None):
    """One step of the bf16 engine (K1 -> K3 -> K2), float64 except for bf16 rounding at exactly the points where the
    kernels round.  S = S_t (B, n, L, d), tokens (B, n, d), pos (n, d), mask (n, n) bool (True = masked) or None.
    Returns {"state": S_{t+1}, "H": (2L-1, B*n, 4d) hidden activations by group (bu_0, td_0, bu_1, ...), "C": (B, n, L, d)
    consensus, "nsq": (B*n, L, nparts) squared-norm partials of S_{t+1}}.

    Roundings (prep_state_kernel, pack_weights_kernel, gemm_kernel, attn_kernel):
      shadows xb = bf16(tokens), sb = bf16(S), sp = bf16(fp32(S[:, :, 1:] + pos)); W1, W2 in bf16; b1, b2 stay fp32
      (b2 = bu_b2 + td_b2, summed in fp32 by the packer: below this reference's resolution, kept in float64 here).
      K1: H_g = bf16(gelu(A_g W1_g^T + b1_g)); the kernel's GELU fit is within 1.9e-6 of the erf form used here.
      K3: key norm |S_j| from the partials of S, logits (sb_i . sb_j) d^-1/2 log2e / max(|S_j|, 1e-12) in log2 units,
          diagonal -5e-4 log2e unless attend_self, masked keys -inf; stabiliser = the Cauchy-Schwarz bound
          d^-1/2 log2e |S_i| unless a row of the 16-row warp has a bound > ATTN_BOUND_MAX, then the exact running maximum
          per key block (256 keys for a single pass of 129..256 padded keys, else 128), each block's P rounded at its own
          maximum and rescaled and rounded again onto the final one; P = bf16(2^(logit - m)), row sum of the unrounded
          values, C = bf16(P sb / l); beyond 576 keys, passes of 512 with (m, l, O) carried between them.
      K2: S_{t+1} = ((S + (acc + b2)) + C) / 3 on the top level, * 0.25 elsewhere; nsq = sum of squares of S_{t+1}
          over each part_w-column part."""
    P = {k: _f64(P[k]) for k in MLP_KEYS}
    tokens, pos, S = _f64(tokens), _f64(pos), _f64(S)
    B, n, L, d = S.shape
    _, part_w = forward_tiles(d)
    if mask is not None:
        mask = torch.as_tensor(mask, dtype=torch.bool, device="cpu")
    xb, sb = bf16(tokens), bf16(S)
    sp = bf16(S[:, :, 1:] + pos[None, :, None, :])
    w1 = [P["bottom_up.net.1.weight"].reshape(L, 4 * d, d), P["top_down.net.1.weight"].reshape(L - 1, 4 * d, d)]
    b1 = [P["bottom_up.net.1.bias"].reshape(L, 4 * d), P["top_down.net.1.bias"].reshape(L - 1, 4 * d)]
    H = []
    for g, a in enumerate(_fwd_k1_operands(xb, sb, sp)):
        net, l = g & 1, g >> 1
        H.append(bf16(F.gelu(a.reshape(B * n, d) @ bf16(w1[net][l]).T + b1[net][l])))
    H = torch.stack(H)
    nsq_in = S.reshape(B, n, L, d // part_w, part_w).square().sum(-1)
    C = _fwd_consensus(sb, _fwd_key_norm(nsq_in), attend_self, mask)
    contrib = torch.full((L,), 4.0, dtype=torch.float64)
    contrib[-1] = 3.0
    b2 = P["bottom_up.net.3.bias"].reshape(L, d).clone()
    b2[:-1] += P["top_down.net.3.bias"].reshape(L - 1, d)
    w2bu = bf16(P["bottom_up.net.3.weight"].reshape(L, d, 4 * d))
    w2td = bf16(P["top_down.net.3.weight"].reshape(L - 1, d, 4 * d))
    state = _fwd_k2(S, H, C, w2bu, w2td, b2, contrib)
    nsq = state.reshape(B * n, L, d // part_w, part_w).square().sum(-1)
    return {"state": state, "H": H, "C": C, "nsq": nsq}


def settle_change(s_prev, s_next, part_w):
    """K2's squared-change partials of a settle step in float64: (B, n, L, d) states S_{k-1}, S_k -> (B*n, L, nparts),
    sum of |S_k - S_{k-1}|^2 over each part_w-column part (part_w as in forward_tiles)."""
    s_prev, s_next = _f64(s_prev), _f64(s_next)
    B, n, L, d = s_next.shape
    return (s_next - s_prev).reshape(B * n, L, d // part_w, part_w).square().sum(-1)


def settle_ratio(dsq, s_next):
    """settle_converge_kernel's ratio in float64: q[b, l] = sqrt(sum_i dsq[b, i, l] / sum_i |S_k[b, i, l]|^2) from the
    change partials (B*n, L, nparts) and S_k (B, n, L, d); 0/0 counts as 0, x/0 (x > 0) as inf."""
    s_next = _f64(s_next)
    B, n, L, d = s_next.shape
    num = _f64(dsq).reshape(B, n, L, -1).sum(dim=(1, 3))
    den = s_next.square().sum(dim=(1, 3))
    return torch.where((num == 0) & (den == 0), torch.zeros_like(num), (num / den).sqrt())


def settle_rule(q_per_step, tol):
    """The stopping rule: q_per_step (K, B, L), the ratios of steps 1..K -> steps (B,) int32, the first k at which every
    level has q <= tol (a NaN never stops an image), K for an image that never stops."""
    hit = (torch.as_tensor(q_per_step) <= tol).all(dim=-1)              # (K, B)
    K = hit.shape[0]
    first = torch.where(hit, torch.arange(1, K + 1)[:, None], torch.full_like(hit, K + 1, dtype=torch.long))
    return first.amin(dim=0).clamp_max(K).to(torch.int32)


@torch.no_grad()
def glom_forward(params, img, *, patch_size, iters=None, levels=None, return_all=False, consensus_self=False,
                 local_consensus_radius=0, dtype=torch.float32):
    """Glom.forward (:110-150).  ``params``: reference state_dict keys -> tensors / arrays; img (B, 3, H, W)."""
    P = {k: torch.as_tensor(v).to(dtype) for k, v in params.items() if k != "attention.non_local_mask"}
    L, d = P["init_levels"].shape
    img = torch.as_tensor(img).to(dtype)
    B, C, H, W = img.shape
    p = patch_size
    x = img.reshape(B, C, H // p, p, W // p, p).permute(0, 2, 4, 3, 5, 1).reshape(B, (H // p) * (W // p), p * p * C)
    tokens = F.linear(x, P["image_to_tokens.1.weight"], P["image_to_tokens.1.bias"])      # (:114)
    n = tokens.shape[1]
    iters = 2 * L if iters is None else iters                                             # (:112)
    if levels is None:
        levels = P["init_levels"][None, None].expand(B, n, L, d)                          # (:123-124)
    else:
        levels = torch.as_tensor(levels).to(dtype)
    mask = None
    if local_consensus_radius > 0:
        mask = radius_mask(int(round(math.sqrt(P["pos_emb.weight"].shape[0]))), local_consensus_radius)
    hiddens = [levels]
    for _ in range(iters):                                                                # (:131)
        levels = column_step(levels, tokens, P["pos_emb.weight"][:n], P, mask, consensus_self)
        hiddens.append(levels)                                                            # (:145)
    if return_all:
        return torch.stack(hiddens)                                                       # (:147-148)
    return levels                                                                         # (:150)
