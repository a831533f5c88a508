"""Implicit gradients through settle: Glom.settle(differentiable="implicit") and glom_b200_backward_implicit.

The settled state S* = f(S*) has the implicit-function-theorem gradient: with J = df/dS at S* and g = dL/dS*, the adjoint
u = sum_k (J^T)^k g (per image, truncated where the adjoint iteration u_k = g + J^T u_{k-1} meets settle's rule), then
the gradients of one step f at S* with cotangent u.  Backpropagating through K + 1 copies of the same step at S* gives
exactly these parameter gradients, so `implicit_grads` below is grads_at_states on repeated states.

CPU: the new symbols, the argument errors of the ABI and of settle (reported before any device query), the workspace
size, the float64 reference against an explicit Neumann sum and against a dense solve of (I - J^T) u = g, and the
faults the GPU bounds must catch.
GPU: the forward is settle's, bit for bit; the gradients match the float64 reference at the engine's own S* and K_b on
the tensor-core, CUDA-core and mixed backward paths; they match the existing backward on repeated states; K_b and q are
settle's rule applied to the engine's own q table; a NaN-filled workspace, a NaN cotangent, determinism, the saved
tensors and batch slicing."""
import copy
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

import glom_pytorch_b200 as G
from glom_pytorch_b200 import _native
from glom_pytorch_b200.glom import _aligned_bytes
from oracle import glom_oracle_torch as OT

import test_backward_oracle as BO

DEV = "cuda:0"
FAKE = 0x100000          # 1024-aligned, never dereferenced: every error below is reported before any device work
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = OT.MLP_KEYS


# ---------------------------------------------------------------------------------------------------- float64 reference
def implicit_grads(P, tokens, pos, state, cot, adjoint_steps, *, attend_self=False, mask=None):
    """The implicit gradients of the settled state `state` (B, n, L, d) given its cotangent `cot`, with image b's adjoint
    truncated after adjoint_steps[b] passes: grads_at_states on T + 1 copies of S*, T = max K_b + 1, the cotangent on
    slab T only and image b live for K_b + 1 steps.  -> d_tokens, d_pos and the MLP_KEYS gradients (float64 CPU)."""
    steps = torch.as_tensor(adjoint_steps).to("cpu", torch.int64) + 1
    T = int(steps.max())
    states = OT._f64(state)[None].expand((T + 1,) + tuple(state.shape))
    g = OT.grads_at_states(P, tokens, pos, states, cot, return_all=False, steps=steps, attend_self=attend_self, mask=mask)
    g.pop("d_state0")
    return g


def _tiny(seed=0, B=2, L=3, d=8, side=2, scale=0.3):
    """A tiny float64 model whose step contracts (second MLP layers scaled), its fixed point and a cotangent."""
    gen = torch.Generator().manual_seed(seed)
    n, G_ = side * side, 2 * L - 1
    P = {}
    for net, groups in (("bottom_up", L), ("top_down", L - 1)):
        P[f"{net}.net.1.weight"] = torch.randn(groups * 4 * d, d, 1, generator=gen, dtype=torch.float64) / math.sqrt(d)
        P[f"{net}.net.1.bias"] = torch.randn(groups * 4 * d, generator=gen, dtype=torch.float64) * 0.1
        P[f"{net}.net.3.weight"] = torch.randn(groups * d, 4 * d, 1, generator=gen, dtype=torch.float64) * scale / math.sqrt(4 * d)
        P[f"{net}.net.3.bias"] = torch.randn(groups * d, generator=gen, dtype=torch.float64) * 0.1
    tokens = torch.randn(B, n, d, generator=gen, dtype=torch.float64)
    pos = torch.randn(n, d, generator=gen, dtype=torch.float64)
    S = torch.randn(B, n, L, d, generator=gen, dtype=torch.float64)
    with torch.no_grad():
        for _ in range(200):
            S = OT.column_step(S, tokens, pos, P, None, False)
    cot = torch.randn(S.shape, generator=gen, dtype=torch.float64)
    return P, tokens, pos, S, cot


def _step_vjp(P, tokens, pos, S, v):
    """-> (J^T v, {d_tokens, d_pos, MLP_KEYS: parameter VJPs of one step at S with cotangent v})."""
    Pl = {k: P[k].clone().requires_grad_(True) for k in NAMES}
    s = S.clone().requires_grad_(True)
    tk, ps = tokens.clone().requires_grad_(True), pos.clone().requires_grad_(True)
    out = OT.column_step(s, tk, ps, Pl, None, False)
    gr = torch.autograd.grad(out, [s, tk, ps] + [Pl[k] for k in NAMES], v)
    return gr[0], dict(zip(["d_tokens", "d_pos"] + list(NAMES), gr[1:]))


def _errors(got, want, L, n):
    return BO.worst(BO.errors({k: got[k] for k in want}, want, L, n))


# ---------------------------------------------------------------------------------------------------------- CPU
def test_new_symbols_are_exported_and_declared():
    with open(os.path.join(ROOT, "include", "glom_b200.h")) as f:
        header = f.read()
    lib = _native.load()
    for name in ("glom_b200_backward_implicit_workspace_bytes", "glom_b200_backward_implicit"):
        assert name in _native.EXPORTS and name in _native.SIGNATURES
        assert re.search(r"GLOM_B200_API int " + name + r"\(", header), name
        assert hasattr(lib, name)
    assert _native.ABI_VERSION == 1 and lib.glom_b200_abi_version() == 1


def _cfg(precision="bf16", dim=128, levels=3, n=64):
    return _native.make_cfg(dim, levels, n, False, 0, 0, precision)


def _implicit_rc(cfg=None, batch=2, adjoint_iters=4, tol=0.1, det=0, steps=FAKE, q=None, d_state0=None, d_init=None):
    lib = _native.load()
    cfg = cfg or _cfg()
    p = ctypes.c_void_p(FAKE)
    w = _native.WeightsRef(ctypes.sizeof(_native.WeightsRef), *([FAKE] * 8))
    names = [k for k, _ in _native.Grads._fields_[1:]]
    vals = {k: FAKE for k in names}
    vals["d_state0"], vals["d_init"] = d_state0, d_init
    g = _native.Grads(ctypes.sizeof(_native.Grads), *[vals[k] for k in names])
    return lib.glom_b200_backward_implicit(ctypes.byref(cfg), ctypes.byref(w), p, p, p, p, ctypes.byref(g), batch,
                                           adjoint_iters, ctypes.c_float(tol), det, steps, q, p, 1 << 30, None)


@pytest.mark.parametrize("what,kw,msg", [
    ("fp32 engine", dict(cfg=_cfg("fp32")), "bf16"),
    ("batch 0", dict(batch=0), "batch"),
    ("negative adjoint_iters", dict(adjoint_iters=-1), "adjoint_iters"),
    ("NaN adjoint_tol", dict(tol=float("nan")), "NaN"),
    ("deterministic 2", dict(det=2), "deterministic"),
    ("NULL adjoint_steps_out", dict(steps=None), "adjoint_steps_out"),
    ("misaligned adjoint_steps_out", dict(steps=FAKE + 2), "aligned"),
    ("misaligned adjoint_q_out", dict(q=FAKE + 2), "aligned"),
    ("d_state0 given", dict(d_state0=FAKE), "d_state0"),
    ("d_init given", dict(d_init=FAKE), "d_init"),
])
def test_backward_implicit_argument_errors(what, kw, msg):
    assert _implicit_rc(**kw) == -1, what
    assert msg in _native.load().glom_b200_last_error().decode(), what


def test_implicit_workspace_holds_the_backward_workspace_and_the_adjoint():
    cfg = _cfg(dim=512, levels=6, n=256)                               # configs[1]
    bwd = _native.backward_workspace_bytes(cfg, 32)
    assert bwd == 2_267_308_032
    rows, L, d, nparts = 32 * 256, 6, 512, 512 // 64
    extra = rows * L * d * 4 + 2 * rows * L * nparts * 4 + (32 + 32 * L + 32) * 4
    assert _native.backward_implicit_workspace_bytes(cfg, 32) >= bwd + extra
    with pytest.raises(_native.GlomB200Error, match="bf16"):
        _native.backward_implicit_workspace_bytes(_cfg("fp32"), 4)


def test_settle_implicit_python_errors():
    m = G.Glom(dim=64, levels=3, image_size=28, patch_size=7)
    img = torch.randn(1, 3, 28, 28)
    for kw, msg in ((dict(differentiable="implicit", return_all=True), "return_all"),
                    (dict(adjoint_tol=1e-3), "implicit"),
                    (dict(differentiable=True, adjoint_iters=3), "implicit"),
                    (dict(differentiable="implicit", adjoint_tol=float("nan")), "NaN"),
                    (dict(differentiable="implicit", adjoint_iters=-1), "adjoint_iters"),
                    (dict(differentiable="unrolled"), "differentiable")):
        with pytest.raises(ValueError, match=msg):
            m.settle(img, 1e-3, **kw)
    m32 = G.Glom(dim=64, levels=3, image_size=28, patch_size=7, precision="fp32")
    with pytest.raises(RuntimeError, match="bf16"):
        m32.settle(img, 1e-3, differentiable="implicit")


def test_reference_is_the_neumann_sum_of_one_step_vjps():
    P, tokens, pos, S, cot = _tiny()
    K = torch.tensor([3, 1])
    got = implicit_grads(P, tokens, pos, S, cot, K)
    want = {k: 0 for k in got}
    for b in range(S.shape[0]):                                        # per image: u = sum_{k <= K_b} (J^T)^k g
        v = torch.zeros_like(cot)
        v[b] = cot[b]
        u = v.clone()
        for _ in range(int(K[b])):
            v = _step_vjp(P, tokens, pos, S, v)[0]
            v[:b], v[b + 1:] = 0, 0
            u = u + v
        _, pv = _step_vjp(P, tokens, pos, S, u)
        for k in want:
            want[k] = want[k] + pv[k]
    for k in got:
        assert float((got[k] - want[k]).abs().max()) <= 1e-12 * max(1.0, float(want[k].abs().max())), k


def test_reference_approaches_the_dense_solve():
    P, tokens, pos, S, cot = _tiny()
    J = torch.autograd.functional.jacobian(lambda s: OT.column_step(s, tokens, pos, P, None, False), S)
    N = S.numel()
    J = J.reshape(N, N)
    assert float(torch.linalg.matrix_norm(J, 2)) < 0.9                 # the model contracts
    u = torch.linalg.solve(torch.eye(N, dtype=torch.float64) - J.T, cot.reshape(N)).reshape(S.shape)
    _, exact = _step_vjp(P, tokens, pos, S, u)
    errs = []
    for K in (0, 2, 5, 10, 30, 90):
        g = implicit_grads(P, tokens, pos, S, cot, torch.full((S.shape[0],), K))
        errs.append(max(float((g[k] - exact[k]).norm() / exact[k].norm()) for k in exact))
    assert all(b < a for a, b in zip(errs, errs[1:])), errs
    assert errs[-1] < 1e-9, errs


def test_bounds_catch_faults():
    """Plausible faults of the implicit backward miss every GPU bound of this file by >= 3x in both metrics."""
    P, tokens, pos, S, cot = _tiny(seed=3, scale=0.6)
    B, n, L, d = S.shape
    K = torch.tensor([1, 2])
    good = implicit_grads(P, tokens, pos, S, cot, K)
    good["init_levels"] = torch.zeros(L, d, dtype=torch.float64)
    S0 = S + 0.3 * torch.randn(S.shape, generator=torch.Generator().manual_seed(9), dtype=torch.float64)
    one_step = implicit_grads(P, tokens, pos, S, cot, 0 * K)           # the g term alone
    faults = {
        "one Neumann term too few": implicit_grads(P, tokens, pos, S, cot, K - 1),
        "g term dropped": {k: v - one_step[k] for k, v in good.items() if k in one_step},
        "parameter pass at S_0": implicit_grads(P, tokens, pos, S0, cot, K),
        "nonzero d_init": dict(good, init_levels=cot.sum((0, 1))),
    }
    for name, bad in faults.items():
        bad = dict(bad)
        bad.setdefault("init_levels", good["init_levels"])
        rel, ab = BO.worst(BO.errors(bad, good, L, n))
        print(f"[implicit] fault {name}: rel {rel:.3e} abs {ab:.3e}")
        for path, (t_rel, t_abs) in TOL.items():
            assert rel >= 3 * t_rel and ab >= 3 * t_abs, (name, path, rel, ab)


# ---------------------------------------------------------------------------------------------------------- GPU
# bounds of the comparison with the float64 reference: those of test_backward_oracle.py, per path
TOL = {"tc": BO.TOL["tc"], "simt": BO.TOL["simt"]}
# (dim, levels, image_size, patch_size, consensus_self, local_consensus_radius, batch, path)
SHAPES = {
    "tensor_core_bwd_n144": (256, 3, 48, 4, False, 0, 5, "tc"),        # rows 720: ragged 128 / 256-row blocks
    "cuda_core_bwd_n64": (128, 3, 32, 4, False, 0, 8, "simt"),
    "mixed_n100": (256, 3, 40, 4, False, 0, 3, "tc"),                  # tensor-core MLPs, CUDA-core attention
    "radius_self_n144": (192, 3, 48, 4, True, 3, 5, "simt"),
}
MAX_ITERS = 12


def _setup(name, w2_scale=0.05):
    """A contracting model (small second MLP layers: every weight gets a gradient), a start near its fixed point with
    noise over six decades (one size per image), and a tol at which the images stop at different steps."""
    dim, L, isz, p, attend_self, radius, B, _ = SHAPES[name]
    torch.manual_seed(0)
    m = G.Glom(dim=dim, levels=L, image_size=isz, patch_size=p, consensus_self=attend_self,
               local_consensus_radius=radius).to(DEV)
    with torch.no_grad():
        m.bottom_up.net[3].weight.mul_(w2_scale)
        m.top_down.net[3].weight.mul_(w2_scale)
    img = torch.randn(B, 3, isz, isz, generator=torch.Generator().manual_seed(1)).to(DEV)
    with torch.no_grad():
        base = m(img, iters=40)
        noise = torch.randn(base.shape, generator=torch.Generator().manual_seed(2)).to(DEV)
        eps = torch.tensor([10.0 ** (1 - 6 * b / max(B - 1, 1)) for b in range(B)], device=DEV).view(B, 1, 1, 1)
        start = (base + eps * noise * base.abs().mean()).contiguous()
    cot = torch.randn(base.shape, generator=torch.Generator().manual_seed(5)).to(DEV)
    return m, img, start, cot


def _grads(m, img, start, cot, **kw):
    """loss = sum(levels * cot) through settle(differentiable="implicit") -> (levels, steps, grads by name)."""
    m.zero_grad(set_to_none=True)
    x = img.clone().requires_grad_(True)
    lv = start.clone().requires_grad_(True)
    levels, steps = m.settle(x, 1e-4, MAX_ITERS, levels=lv, differentiable="implicit", **kw)
    (levels * cot).sum().backward()
    assert lv.grad is None and m.init_levels.grad is None
    g = {k: q.grad.clone() for k, q in m.named_parameters() if q.grad is not None}
    g["d_img"] = x.grad.clone()
    return levels.detach(), steps, g


def _mask(m, n):
    return BO._mask(m, n)


def _reference(m, img, S, cot, K):
    n = S.shape[1]
    with torch.no_grad():
        tok = m.tokens(img).cpu()
    P = {k: q.detach().cpu() for k, q in m.named_parameters()}
    g = implicit_grads(P, tok, P["pos_emb.weight"][:n], S.cpu(), cot.cpu(), K.cpu(),
                       attend_self=m.attention.attend_self, mask=_mask(m, n))
    g["d_state0"] = None
    params = {k: v.numpy() for k, v in P.items()}
    out = BO._map_reference(g, params, img.cpu(), m.patch_size, n, True)
    out.pop("d_levels")
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SHAPES))
def test_forward_is_settle_and_gradients_match_the_reference(name):
    m, img, start, cot = _setup(name)
    with torch.no_grad():
        want, want_steps = m.settle(img, 1e-4, MAX_ITERS, levels=start)
    levels, steps, got = _grads(m, img, start, cot, adjoint_tol=1e-4, adjoint_iters=8)
    assert torch.equal(levels, want) and torch.equal(steps, want_steps)
    K, q = m.last_adjoint
    assert K.dtype == torch.int32 and q.shape == (img.shape[0], m.levels)
    assert int(K.min()) >= 1 and int(K.max()) <= 8
    ref = _reference(m, img, levels, cot, K)
    L, n = m.levels, levels.shape[1]
    rel, ab = _errors(got, ref, L, n)
    print(f"[implicit] {name}: K {K.tolist()} rel {rel:.3e} abs {ab:.3e}")
    BO.check(BO.errors({k: got[k] for k in ref}, ref, L, n), TOL[SHAPES[name][7]], name)


def _engine(m, tokens, S, cot, adjoint_iters, adjoint_tol, deterministic=True, ws=None):
    """glom_b200_backward_implicit on the engine's tokens -> (grads by Grads field, K, q)."""
    b, n = tokens.shape[:2]
    cfg = m.engine_cfg(n)
    wts = [q.detach().float().contiguous() for q in m._mlp_params()]
    names = ("d_bu_w1", "d_bu_b1", "d_bu_w2", "d_bu_b2", "d_td_w1", "d_td_b1", "d_td_w2", "d_td_b2")
    g = {"d_tokens": torch.zeros_like(tokens), "d_pos": torch.zeros(n, m.dim, device=DEV)}
    g.update({k: torch.zeros_like(w) for k, w in zip(names, wts)})
    K = torch.empty(b, dtype=torch.int32, device=DEV)
    q = torch.empty(b, m.levels, device=DEV)
    if ws is None:
        ws = _aligned_bytes(_native.backward_implicit_workspace_bytes(cfg, b), torch.device(DEV))
    pos = m.pos_emb.weight[:n].detach().contiguous()
    _native.backward_implicit(cfg, [w.data_ptr() for w in wts], tokens.data_ptr(), pos.data_ptr(), S.data_ptr(),
                              cot.data_ptr(), {k: v.data_ptr() for k, v in g.items()}, b, adjoint_iters, adjoint_tol,
                              K.data_ptr(), q.data_ptr(), ws.data_ptr(), ws.numel(),
                              torch.cuda.current_stream().cuda_stream, deterministic=deterministic)
    torch.cuda.synchronize()
    return g, K, q


def _settled(name):
    m, img, start, cot = _setup(name)
    with torch.no_grad():
        S, _ = m.settle(img, 1e-4, MAX_ITERS, levels=start)
        tokens = m.tokens(img)
    return m, tokens, S.contiguous(), cot


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tensor_core_bwd_n144", "cuda_core_bwd_n64"])
def test_fixed_passes_match_the_backward_on_repeated_states(name):
    """adjoint_tol = -1, adjoint_iters = K: the backward of K + 1 steps at S*, with the cotangent on the last state."""
    m, tokens, S, cot = _settled(name)
    K = 3
    got, steps, _ = _engine(m, tokens, S, cot, K, -1.0, deterministic=False)
    assert steps.tolist() == [K] * S.shape[0]
    b, n = tokens.shape[:2]
    cfg = m.engine_cfg(n)
    wts = [q.detach().float().contiguous() for q in m._mlp_params()]
    want = {k: torch.zeros_like(v) for k, v in got.items()}
    want["d_state0"] = torch.zeros_like(S)
    states = S[None].expand((K + 2,) + tuple(S.shape)).contiguous()
    ws = _aligned_bytes(_native.backward_workspace_bytes(cfg, b), torch.device(DEV))
    pos = m.pos_emb.weight[:n].detach().contiguous()
    _native.backward(cfg, [w.data_ptr() for w in wts], tokens.data_ptr(), pos.data_ptr(), states.data_ptr(),
                     cot.data_ptr(), {k: v.data_ptr() for k, v in want.items()}, b, K + 1, False, ws.data_ptr(),
                     ws.numel(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    # the tensor-core path rounds u_k (the implicit sum) and (J^T)^k g (the unrolled one) to bf16: its bound
    bound = 1e-5 if SHAPES[name][7] == "simt" else BO.TOL["tc"][0]
    for k, v in got.items():
        r = float((v - want[k]).norm() / want[k].norm().clamp_min(1e-30))
        assert r <= bound, (name, k, r)


@pytest.mark.gpu
def test_stopping_decisions_are_settle_rule_on_the_q_table():
    m, tokens, S, cot = _settled("tensor_core_bwd_n144")
    P = 6
    table = []                                                        # q of pass k, no image stopped: (P, B, L)
    for k in range(1, P + 1):
        _, K, q = _engine(m, tokens, S, cot, k, -1.0)
        assert K.tolist() == [k] * S.shape[0]
        table.append(q.cpu())
    table = torch.stack(table)
    assert torch.isfinite(table).all() and (table > 0).all()
    first = table.amax(-1)                                            # (P, B)
    tols = [float(first[2, 0]), float(np.nextafter(np.float32(first[2, 0]), np.float32(0))),
            float(first[:, 1].median()), float(first.min()) / 2, float(first.max()) * 2]
    for tol in tols:
        _, K, q = _engine(m, tokens, S, cot, P, tol)
        want = OT.settle_rule(table, tol)
        assert torch.equal(K.cpu(), want), (tol, K.tolist(), want.tolist())
        for b, k in enumerate(want.tolist()):
            assert torch.equal(q[b].cpu(), table[k - 1, b]), (tol, b)
    # the exact threshold stops image 0 at pass 3 (or earlier), the next float32 below does not stop it there
    assert int(OT.settle_rule(table, tols[0])[0]) <= 3


def _det_grads(m, img, start, cot, ws_fill=None, stream=None, **kw):
    with torch.cuda.stream(stream or torch.cuda.current_stream()):
        m.zero_grad(set_to_none=True)
        x = img.clone().requires_grad_(True)
        levels, _ = m.settle(x, 1e-4, MAX_ITERS, levels=start, differentiable="implicit", **kw)
        if ws_fill is not None:
            dev = torch.device(DEV)
            n = levels.shape[1]
            ws = m._get_workspace(_native.backward_implicit_workspace_bytes(m.engine_cfg(n), img.shape[0]), dev,
                                  "_implicit_workspace")
            ws.fill_(ws_fill)
        (levels * cot).sum().backward()
        torch.cuda.synchronize()
    g = {k: q.grad.clone() for k, q in m.named_parameters() if q.grad is not None}
    g["d_img"] = x.grad.clone()
    return g, m.last_adjoint[0].clone()


def _same_bits(a, b, what):
    assert set(a) == set(b), what
    for k in a:
        assert torch.equal(a[k], b[k]), (what, k)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tensor_core_bwd_n144", "cuda_core_bwd_n64"])
def test_nan_workspace_nan_cotangent_and_determinism(name):
    m, img, start, cot = _setup(name)
    torch.use_deterministic_algorithms(True)
    try:
        ref, K = _det_grads(m, img, start, cot, adjoint_iters=8)
        nan_ws, K_nan = _det_grads(m, img, start, cot, ws_fill=0xFF, adjoint_iters=8)   # 0xFF..: NaN in fp32 and bf16
        zero_ws, K_zero = _det_grads(m, img, start, cot, ws_fill=0, adjoint_iters=8)
        _same_bits(nan_ws, zero_ws, "NaN workspace")
        _same_bits(ref, zero_ws, "zeroed workspace")
        assert torch.equal(K_nan, K) and torch.equal(K_zero, K)
        twin, K_twin = _det_grads(copy.deepcopy(m), img, start, cot, adjoint_iters=8)
        _same_bits(ref, twin, "deepcopy")
        side, K_side = _det_grads(m, img, start, cot, stream=torch.cuda.Stream(), adjoint_iters=8)
        _same_bits(ref, side, "second stream")
        assert torch.equal(K_twin, K) and torch.equal(K_side, K)
        bad = cot.clone()
        bad[0, 0, 0, 0] = float("nan")
        g_bad, K_bad = _det_grads(m, img, start, bad, adjoint_iters=8)
        assert int(K_bad[0]) == 8
        assert torch.equal(K_bad[1:], K[1:])
        assert torch.equal(g_bad["d_img"][1:], ref["d_img"][1:])
    finally:
        torch.use_deterministic_algorithms(False)


@pytest.mark.gpu
def test_graph_saves_one_state():
    m, img, start, cot = _setup("tensor_core_bwd_n144")
    shape = tuple(start.shape)
    saved = []

    def pack(t):
        saved.append(tuple(t.shape))
        return t

    with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
        levels, _ = m.settle(img.clone().requires_grad_(True), 1e-4, MAX_ITERS, levels=start, differentiable="implicit")
    assert sum(s == shape for s in saved) == 1, saved
    saved.clear()
    with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
        m.settle(img.clone().requires_grad_(True), 1e-4, MAX_ITERS, levels=start, differentiable=True)
    assert (MAX_ITERS + 1,) + shape in saved                          # the unrolled form keeps the trajectory
    (levels * cot).sum().backward()


@pytest.mark.gpu
def test_batch_slicing_at_production_size():
    torch.manual_seed(0)
    m = G.Glom(dim=512, levels=6, image_size=224, patch_size=14).to(DEV)
    with torch.no_grad():
        m.bottom_up.net[3].weight.mul_(0.1)
        m.top_down.net[3].weight.mul_(0.1)
    img = torch.randn(32, 3, 224, 224, generator=torch.Generator().manual_seed(1)).to(DEV)
    cot = torch.randn(32, 256, 6, 512, generator=torch.Generator().manual_seed(5)).to(DEV)
    torch.use_deterministic_algorithms(True)
    try:
        def run(sl):
            x = img[sl].clone().requires_grad_(True)
            levels, _ = m.settle(x, 1e-3, 12, differentiable="implicit")
            (levels * cot[sl]).sum().backward()
            return x.grad.clone(), m.last_adjoint[0].clone()
        d_img, K = run(slice(0, 32))
        for i in range(0, 32, 2):
            d2, K2 = run(slice(i, i + 2))
            assert torch.equal(d2, d_img[i:i + 2]), i
            assert torch.equal(K2, K[i:i + 2]), i
    finally:
        torch.use_deterministic_algorithms(False)
