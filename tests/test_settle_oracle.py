"""Glom.settle against float64 references at the engine's own states (oracle/glom_oracle_torch.py), down to each
threshold decision.

`settle_change` is K2's squared-change partials (B*n, L, nparts) of one step, `settle_ratio` the convergence kernel's
q[b, l] = sqrt(sum dsq / sum |S_k|^2) (0/0 = 0, x/0 = inf), `settle_rule` the first step at which every level has
q <= tol (a NaN never stops an image).  The settle buffers are read through glom_b200_settle_workspace_offset.

(a) settle(tol=-1, max_iters=k) for k = 1..K stops no image: its result is bit-identical to forward(iters=k), and the
    change partials and ratios of step k are compared with the references at the engine's own S_{k-1}, S_k (from
    forward(return_all=True)): dsq per (row, level, part) with the metric of test_forward_oracle.py (|err| over
    max(|ref|, FLOOR * rms)), q per (image, level), relative.  Both settle and settle_all.
(b) The decisions are checked exactly against the rule applied to the engine's own fp32 q tables from (a), at tol values
    that spread the images, at a tol equal to one image's max_l q_k (it must stop at k: the comparison is <=) and at the
    next float32 below (it must not): steps, the final q of every image, frozen and block_frozen.  Where the float64 q
    stays further from tol than the q bound, steps also equal the rule on the float64 q.
(c) The documented special values: an image whose S_1 is exactly 0 has q = 0/0 = 0 (stops at tol = 0, never at -1); an
    image holding a NaN never stops and changes nothing for the other images.

The CPU tests pin the references to test_settle.py's float64 criterion, check the rule on hand-built tables, show that
plausible kernel faults miss the bounds by >= 3x and that plausible rule faults flip decisions that (b) asserts, and
check the settle buffer offsets of the C ABI.

Bounds, set at about 3x the worst value observed over the GPU tests on one H100 80GB HBM3 (400 W power limit);
observed maxima in brackets:
  dsq   change partials vs settle_change at the engine's states    (rel 5e-7, abs 4e-7)  [rel 1.78e-7, abs 1.32e-7, both
                                                                                          at config2_dims]
  q     level_q vs settle_ratio of the engine's states, relative   4.5e-7                [1.46e-7 at n256_whole_blocks]
The kernel faults of test_bounds_catch_kernel_faults miss these bounds by 1.8e4x at least.  No kernel missed its
reference by more than rounding explains.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import glom_pytorch_b200 as G
import test_settle as TS
from glom_pytorch_b200 import _native
from oracle import glom_oracle_torch as OT

DEV = "cuda:0"
FLOOR = 0.1                       # as in test_forward_oracle.py
TOL = {"dsq": (5e-7, 4e-7), "q": 4.5e-7}


# ----------------------------------------------------------------------------- metric
def dsq_errors(got, ref):
    """-> (worst per-(row, level, part) error over max(|ref|, FLOOR * rms), max-abs error over max |ref|)."""
    g, r = torch.as_tensor(got).double(), torch.as_tensor(ref).double()
    assert g.shape == r.shape and torch.isfinite(g).all()
    rms = float(torch.linalg.norm(r)) / math.sqrt(r.numel())
    rel = float(((g - r).abs() / r.abs().clamp_min(max(FLOOR * rms, 1e-300))).max())
    return rel, float((g - r).abs().max()) / max(float(r.abs().max()), 1e-300)


def q_error(got, ref):
    """-> worst relative error per (image, level); both zero counts as exact."""
    g, r = torch.as_tensor(got).double(), torch.as_tensor(ref).double()
    assert g.shape == r.shape and torch.isfinite(g).all() and torch.isfinite(r).all()
    return float(((g - r).abs() / r.abs().clamp_min(1e-300)).max())


def _part_w(d):
    return OT.forward_tiles(d)[1]


def _ratios(states):
    """float64 q of every step from states (K+1, B, n, L, d) -> (K, B, L)."""
    s = states.double()
    return torch.stack([OT.settle_ratio(OT.settle_change(s[k - 1], s[k], _part_w(s.shape[-1])), s[k])
                        for k in range(1, s.shape[0])])


def _tols(Q):
    """Thresholds for (b) from a q table (K, B, L) float32: geometric means between neighbouring max_l q values at least
    1 % apart near the 25 / 50 / 75 % quantiles, then (tol_eq, b, k): tol_eq = max_l q_k[b] as float32 for an image b
    whose ratio at every earlier step is larger (the latest such k < K), and the next float32 below it."""
    r = Q.double().amax(dim=-1)                                             # (K, B)
    vals = np.unique(r[torch.isfinite(r) & (r > 0)].numpy())
    gaps = [(a, b) for a, b in zip(vals[:-1], vals[1:]) if b > a * 1.01]
    spread = []
    for f in (0.25, 0.5, 0.75):
        a, b = gaps[min(int(f * len(gaps)), len(gaps) - 1)]
        spread.append(float(np.float32(math.sqrt(a * b))))
    K, B = r.shape
    best = None
    for b in range(B):
        for k in range(1, K):
            if all(r[j, b] > r[k - 1, b] for j in range(k - 1)) and (best is None or k > best[2]):
                best = (float(Q[k - 1, b].amax()), b, k)
    tol_eq, b, k = best
    below = float(np.nextafter(np.float32(tol_eq), np.float32(-np.inf)))
    return sorted(set(spread)), (tol_eq, below, b, k)


# ----------------------------------------------------------------------------- CPU: the references
def _cpu_chain(B, n, L, d, K=3, seed=0):
    """States (K+1, B, n, L, d) float32 of a settling chain: the change of step k is 2^-k times a size spread over images
    (1e-1 .. 1e-3) and levels (x 3^l)."""
    g = torch.Generator().manual_seed(seed)
    eps = torch.tensor([10.0 ** (-1 - 2 * b / max(B - 1, 1)) for b in range(B)]).view(B, 1, 1, 1)
    eps = eps * (3.0 ** torch.arange(L)).view(1, 1, L, 1)
    s = [torch.randn(B, n, L, d, generator=g)]
    for k in range(1, K + 1):
        s.append(s[-1] + eps * 0.5 ** k * torch.randn(B, n, L, d, generator=g))
    return torch.stack(s).float()


# name: (dim, levels, image_size, patch, consensus_self, radius, batch, K); random weights, random start
SHAPES = {
    "n256_whole_blocks": (256, 3, 64, 4, False, 0, 6, 4),
    "n64_four_images_per_block": (128, 3, 32, 4, False, 0, 8, 4),
    "n625_key_passes": (64, 2, 100, 4, False, 0, 4, 4),
    "n144_radius_self": (192, 3, 48, 4, True, 3, 5, 4),
    "d64_two_parts": (64, 3, 32, 4, False, 0, 3, 3),
    "d320_ten_parts": (320, 2, 24, 4, False, 0, 3, 3),
    "n100_ragged_rows": (128, 3, 40, 4, False, 0, 3, 3),                 # 300 rows: the last 256-row block holds 44
    "config2_dims": (512, 6, 224, 14, False, 0, 2, 12),
}


def _shape_dims(name):
    dim, L, isz, p, _, _, B, K = SHAPES[name]
    return B, (isz // p) ** 2, L, dim, K


def test_reference_is_test_settle_criterion():
    """max_l settle_ratio(settle_change(S_{k-1}, S_k)) is test_settle.py's float64 change criterion, to 1e-12."""
    for name in ("n625_key_passes", "d320_ten_parts", "d64_two_parts"):
        B, n, L, d, K = _shape_dims(name)
        states = _cpu_chain(B, n, L, d, K)
        want = torch.from_numpy(TS._change(states))                          # (B, K)
        got = _ratios(states).amax(dim=-1).T
        assert float(((got - want).abs() / want).max()) <= 1e-12, name


def test_change_partials_follow_k2_parts():
    """settle_change sums each part_w-column part (64 columns at d % 256 == 0, else bn2 / 2) of each (row, level)."""
    for d, part_w in ((64, 32), (128, 64), (192, 32), (320, 32), (384, 64), (512, 64)):
        assert _part_w(d) == part_w, d
        s = _cpu_chain(2, 5, 2, d, 1)
        dsq = OT.settle_change(s[0], s[1], part_w)
        assert dsq.shape == (10, 2, d // part_w)
        diff = (s[1].double() - s[0].double()).reshape(10, 2, d)
        assert torch.allclose(dsq[:, :, -1], diff[:, :, -part_w:].square().sum(-1), rtol=1e-14, atol=0)


def test_rule_semantics_on_hand_built_tables():
    nan, inf = float("nan"), float("inf")
    # (K=3, B=6, L=2): ties stop (<=); a NaN never stops; inf stops only at tol = inf; 0 stops at tol >= 0
    Q = torch.tensor([
        [[0.5, 0.1], [0.2, 0.2], [nan, 0.0], [inf, 0.0], [0.0, 0.0], [0.3, 0.3]],
        [[0.2, 0.1], [0.1, 0.1], [0.0, 0.0], [0.1, 0.1], [0.0, 0.0], [0.3, nan]],
        [[0.1, 0.1], [0.1, 0.1], [0.0, 0.0], [0.1, 0.1], [0.0, 0.0], [nan, nan]],
    ], dtype=torch.float64)
    assert OT.settle_rule(Q, 0.2).tolist() == [2, 1, 2, 2, 1, 3]
    assert OT.settle_rule(Q, 0.1).tolist() == [3, 2, 2, 2, 1, 3]
    assert OT.settle_rule(Q, 0.0).tolist() == [3, 3, 2, 3, 1, 3]
    assert OT.settle_rule(Q, -1.0).tolist() == [3, 3, 3, 3, 3, 3]
    assert OT.settle_rule(Q, inf).tolist() == [1, 1, 2, 1, 1, 1]
    # the ratio: 0/0 = 0, x/0 = inf, both from the partials
    s_prev = torch.zeros(3, 4, 2, 64)
    s_next = torch.zeros(3, 4, 2, 64)
    s_prev[1, :, 0] = 1.0                              # image 1, level 0: S_k = 0 after a change -> x/0 = inf
    s_prev[2] = 1.0
    s_next[2] = 2.0                                    # image 2: |dS| / |S| = 1/2
    q = OT.settle_ratio(OT.settle_change(s_prev, s_next, 32), s_next)
    assert q.tolist() == [[0.0, 0.0], [inf, 0.0], [0.5, 0.5]]


# faults of the kernels: (name, what they change).  Each returns (dsq, q) of step k from the chain s (K+1, B, n, L, d)
def _good(s, k, part_w):
    dsq = OT.settle_change(s[k - 1], s[k], part_w)
    return dsq, OT.settle_ratio(dsq, s[k])


def _k2_drops_last_part(s, k, part_w):
    dsq = OT.settle_change(s[k - 1], s[k], part_w)
    dsq[:, :, -1] = 0
    return dsq, OT.settle_ratio(dsq, s[k])


def _ratio_first_256_rows(s, k, part_w):
    dsq = OT.settle_change(s[k - 1], s[k], part_w)
    B, n = s.shape[1], s.shape[2]
    keep = (torch.arange(n) < 256).double()
    cut = (dsq.reshape(B, n, *dsq.shape[1:]) * keep[None, :, None, None]).reshape(dsq.shape)
    return dsq, OT.settle_ratio(cut, s[k] * keep[None, :, None, None].float())


def _change_against_k_minus_2(s, k, part_w):
    dsq = OT.settle_change(s[k - 2], s[k], part_w)
    return dsq, OT.settle_ratio(dsq, s[k])


def _denominator_of_previous_state(s, k, part_w):
    dsq = OT.settle_change(s[k - 1], s[k], part_w)
    return dsq, OT.settle_ratio(dsq, s[k - 1])


KERNEL_FAULTS = {"k2_drops_last_change_partial": _k2_drops_last_part,
                 "ratio_sums_rows_below_256": _ratio_first_256_rows,
                 "change_against_s_k_minus_2": _change_against_k_minus_2,
                 "denominator_uses_s_k_minus_1": _denominator_of_previous_state}


@pytest.mark.parametrize("fault", sorted(KERNEL_FAULTS))
def test_bounds_catch_kernel_faults(fault):
    """At the GPU test shapes, on CPU states, each faulty reference misses the dsq bound (both metrics) or the q bound by
    >= 3x at some shape."""
    worst = 0.0
    for name in sorted(SHAPES):
        B, n, L, d, _ = _shape_dims(name)
        s = _cpu_chain(B, n, L, d, 2, seed=5)
        good = _good(s, 2, _part_w(d))
        bad = KERNEL_FAULTS[fault](s, 2, _part_w(d))
        rel, ab = dsq_errors(bad[0], good[0])
        miss = max(min(rel / TOL["dsq"][0], ab / TOL["dsq"][1]), q_error(bad[1], good[1]) / TOL["q"])
        print(f"[settle-oracle] fault {fault} at {name}: dsq rel {rel:.2e} abs {ab:.2e}, "
              f"q {q_error(bad[1], good[1]):.2e}")
        worst = max(worst, miss)
    assert worst >= 3, (fault, worst)


def _rule_lt(Q, tol):
    return OT.settle_rule(torch.where(torch.as_tensor(Q) < tol, 0.0, 1.0), 0.5)


def _rule_level0(Q, tol):
    return OT.settle_rule(torch.as_tensor(Q)[..., :1], tol)


def _rule_min(Q, tol):
    return OT.settle_rule(torch.as_tensor(Q).amin(dim=-1, keepdim=True), tol)


RULE_FAULTS = {"lt_not_le": _rule_lt, "level_0_only": _rule_level0, "min_over_levels": _rule_min}


@pytest.mark.parametrize("fault", sorted(RULE_FAULTS))
def test_rule_faults_flip_an_asserted_decision(fault):
    """On a q table of the chain's float32 ratios, each faulty rule gives other steps than settle_rule at one of the tol
    values that (b) picks with _tols."""
    B, n, L, d, _ = _shape_dims("n256_whole_blocks")
    s = _cpu_chain(B, n, L, d, 6, seed=2)
    Q = _ratios(s).float()
    spread, (tol_eq, below, b, k) = _tols(Q)
    assert OT.settle_rule(Q, tol_eq)[b] == k and OT.settle_rule(Q, below)[b] > k
    flips = [t for t in spread + [tol_eq, below] if not torch.equal(RULE_FAULTS[fault](Q, t), OT.settle_rule(Q, t))]
    assert flips, fault


@pytest.mark.parametrize("dim,levels,n,batch,iters", [
    (512, 6, 256, 32, 12), (128, 3, 64, 5, 4), (64, 2, 625, 3, 6), (192, 3, 144, 7, 1), (320, 2, 100, 3, 3)])
@pytest.mark.parametrize("return_all", [False, True])
def test_settle_workspace_offsets(dim, levels, n, batch, iters, return_all):
    cfg = TS._cfg(dim=dim, levels=levels, n=n)
    total = (_native.settle_all_workspace_bytes if return_all else _native.settle_workspace_bytes)(cfg, batch, iters)
    fwd = _native.workspace_bytes(cfg, batch, iters, return_all)
    rows, nparts = batch * n, dim // _part_w(dim)
    want = [rows * levels * nparts * 4, batch * levels * 4, batch * 4, (rows + 255) // 256 * 4]
    spans = []
    for which, nbytes in enumerate(want):
        off, nb = _native.settle_workspace_offset(cfg, batch, iters, return_all, which)
        assert nb == nbytes, which
        assert off % 16 == 0 and off >= fwd and off + nb <= total, (which, off, nb, fwd, total)
        spans.append((off, off + nb))
    spans.sort()
    assert all(a[1] <= b[0] for a, b in zip(spans[:-1], spans[1:])), spans
    for which in (4, -1):
        with pytest.raises(_native.GlomB200Error, match="unknown settle buffer id"):
            _native.settle_workspace_offset(cfg, batch, iters, return_all, which)


def test_settle_workspace_offset_argument_errors():
    lib = _native.load()
    off, nb = ctypes.c_size_t(), ctypes.c_size_t()
    for cfg, batch, iters, msg in ((TS._cfg("fp32"), 2, 4, "bf16"), (TS._cfg(), 0, 4, "batch"),
                                   (TS._cfg(), 2, 0, "max_iters")):
        rc = lib.glom_b200_settle_workspace_offset(ctypes.byref(cfg), batch, iters, 0, 0, ctypes.byref(off),
                                                   ctypes.byref(nb))
        assert rc == -1 and msg in lib.glom_b200_last_error().decode(), msg
    cfg = TS._cfg()
    assert lib.glom_b200_settle_workspace_offset(ctypes.byref(cfg), 2, 4, 0, 0, None, ctypes.byref(nb)) == -1


# ----------------------------------------------------------------------------- GPU
def _model(name, seed=0, contracting=False, zero_second_layer=False):
    dim, L, isz, p, attend_self, radius, B, _ = SHAPES[name]
    torch.manual_seed(seed)
    m = G.Glom(dim=dim, levels=L, image_size=isz, patch_size=p, consensus_self=attend_self,
               local_consensus_radius=radius).to(DEV).eval()
    with torch.no_grad():
        for net in (m.bottom_up.net, m.top_down.net):
            if contracting or zero_second_layer:
                net[3].weight.zero_()
            if zero_second_layer:
                net[3].bias.zero_()
    g = torch.Generator().manual_seed(seed + 1)
    n = (isz // p) ** 2
    img = torch.randn(B, 3, isz, isz, generator=g).to(DEV)
    start = torch.randn(B, n, L, dim, generator=g).to(DEV)
    return m, img, start


def _settle(m, img, tol, max_iters, start, return_all=False):
    """settle -> (out, steps, dsq, level_q, frozen, block_frozen), the buffers read from the workspace after the call."""
    with torch.no_grad():
        out, steps = m.settle(img, tol, max_iters=max_iters, levels=start, return_all=return_all)
    torch.cuda.synchronize()
    B, n = start.shape[0], start.shape[1]
    cfg = m.engine_cfg(n)
    ws = m._workspace

    def buf(which, dtype):
        off, nb = _native.settle_workspace_offset(cfg, B, max_iters, return_all, which)
        return ws[off:off + nb].view(dtype).cpu()
    L, d = start.shape[2], start.shape[3]
    dsq = buf(0, torch.float32).reshape(B * n, L, d // _part_w(d))
    return (out, steps.cpu(), dsq, buf(1, torch.float32).reshape(B, L), buf(2, torch.int32),
            buf(3, torch.int32))


def _q_table(m, img, start, K, return_all=False, check=None):
    """The engine's q of steps 1..K, (K, B, L) float32, from settle(tol=-1, max_iters=k); `check(k, out, dsq, q)` sees
    each call."""
    qs = []
    for k in range(1, K + 1):
        out, steps, dsq, q, frozen, _ = _settle(m, img, -1.0, k, start, return_all)
        assert (steps == k).all() and (frozen == 0).all(), (k, steps, frozen)
        if check:
            check(k, out, dsq, q)
        qs.append(q)
    return torch.stack(qs)


@pytest.mark.gpu
@pytest.mark.parametrize("return_all", [False, True], ids=["settle", "settle_all"])
@pytest.mark.parametrize("name", sorted(SHAPES))
def test_partials_and_ratio_per_step(name, return_all):
    """(a): no image stops at tol = -1; the result is bit-identical to forward, and dsq / q of every step match the
    float64 references at the engine's own S_{k-1}, S_k."""
    m, img, start = _model(name)
    B, n, L, d, K = _shape_dims(name)
    with torch.no_grad():
        states = m(img, iters=K, levels=start, return_all=True).cpu()
    worst = {"dsq_rel": 0.0, "dsq_abs": 0.0, "q": 0.0}

    def check(k, out, dsq, q):
        with torch.no_grad():
            ref_out = m(img, iters=k, levels=start, return_all=return_all)
        assert torch.equal(out, ref_out), (name, k)
        rel, ab = dsq_errors(dsq, OT.settle_change(states[k - 1], states[k], _part_w(d)))
        qe = q_error(q, OT.settle_ratio(dsq.double(), states[k]))
        qe64 = q_error(q, OT.settle_ratio(OT.settle_change(states[k - 1], states[k], _part_w(d)), states[k]))
        worst["dsq_rel"], worst["dsq_abs"] = max(worst["dsq_rel"], rel), max(worst["dsq_abs"], ab)
        worst["q"] = max(worst["q"], qe, qe64)
        assert rel <= TOL["dsq"][0] and ab <= TOL["dsq"][1], (name, k, rel, ab)
        assert qe64 <= TOL["q"] and qe <= TOL["q"], (name, k, qe64, qe)
    _q_table(m, img, start, K, return_all, check)
    print(f"[settle-oracle] {name} return_all={return_all}: " + " ".join(f"{k} {v:.3e}" for k, v in worst.items()))


def _check_decisions(m, img, start, Q, Q64, tol, what):
    """(b) at one tol: steps, final q, frozen, block_frozen against the rule on the engine's own q table Q."""
    K, B, L = Q.shape
    n = start.shape[1]
    _, steps, _, q, frozen, block_frozen = _settle(m, img, tol, K, start)
    want = OT.settle_rule(Q, tol)
    assert torch.equal(steps, want), (what, tol, steps, want)
    last = Q[steps.long() - 1, torch.arange(B)]                              # q of each image's last step
    assert torch.equal(q.view(torch.int32), last.contiguous().view(torch.int32)), (what, tol)
    met = (last <= tol).all(dim=-1).int()
    assert torch.equal(frozen, met), (what, tol, frozen, met)
    rows = B * n
    want_blk = [int(all(met[b] for b in range(m0 * 256 // n, (min(rows, m0 * 256 + 256) - 1) // n + 1)))
                for m0 in range((rows + 255) // 256)]
    assert block_frozen.tolist() == want_blk, (what, tol)
    r64 = Q64.amax(dim=-1)                                                   # (K, B)
    safe = ((r64 / tol - 1).abs() > TOL["q"]).all(dim=0) if tol > 0 else torch.ones(B, dtype=torch.bool)
    assert torch.equal(steps[safe], OT.settle_rule(Q64, tol)[safe]), (what, tol)
    return steps


@pytest.mark.gpu
@pytest.mark.parametrize("start_kind", ["contracting", "random_weights"])
@pytest.mark.parametrize("name", ["n256_whole_blocks", "n64_four_images_per_block", "n625_key_passes"])
def test_decisions_from_the_engines_own_q(name, start_kind):
    """(b): settle's steps, q, frozen and block_frozen are the rule applied to the engine's own fp32 q table exactly,
    including at a tol equal to one image's max_l q_k and at the next float32 below it."""
    if start_kind == "contracting":                                          # test_settle.py's start
        m, img = TS._model(name, contracting=True)
        with torch.no_grad():
            base = m(img, iters=60)
            noise = torch.randn(base.shape, generator=torch.Generator().manual_seed(2)).to(DEV)
            B = img.shape[0]
            eps = torch.tensor([10.0 ** (1 - 6 * b / (B - 1)) for b in range(B)], device=DEV).view(B, 1, 1, 1)
            start = (base + eps * noise * base.abs().mean()).contiguous()
        K = TS.MAX_ITERS
    else:
        m, img, start = _model(name, seed=3)
        K = 8
    Q = _q_table(m, img, start, K)
    with torch.no_grad():
        Q64 = _ratios(m(img, iters=K, levels=start, return_all=True).cpu())
    print(f"[settle-oracle] {name} {start_kind}: q {q_error(Q, Q64):.3e}")
    assert q_error(Q, Q64) <= TOL["q"]
    spread, (tol_eq, below, b, k) = _tols(Q)
    seen = set()
    for tol in spread:
        seen.update(_check_decisions(m, img, start, Q, Q64, tol, (name, start_kind)).tolist())
    assert len(seen) >= 2, (name, start_kind, seen)
    assert _check_decisions(m, img, start, Q, Q64, tol_eq, (name, start_kind, "eq"))[b] == k
    assert _check_decisions(m, img, start, Q, Q64, below, (name, start_kind, "below"))[b] > k


@pytest.mark.gpu
def test_zero_image_counts_as_converged():
    """Second MLP layers zero (weights and biases), image 0 started from zero levels: its S_1 is exactly 0, so q = 0/0
    = 0 at every level: it stops at step 1 with tol = 0 and never with tol = -1."""
    m, img, start = _model("n64_four_images_per_block", zero_second_layer=True)
    start[0] = 0
    K = 4
    out, steps, _, q, frozen, _ = _settle(m, img, 0.0, K, start)
    assert (out[0] == 0).all() and steps[0] == 1 and frozen[0] == 1 and (q[0] == 0).all()
    assert (steps[1:] == K).all() and (frozen[1:] == 0).all() and (q[1:] > 0).all()
    out, steps, _, q, frozen, _ = _settle(m, img, -1.0, K, start)
    assert (steps == K).all() and (frozen == 0).all() and (q[0] == 0).all()


@pytest.mark.gpu
def test_nan_image_never_stops_and_changes_nothing_else():
    """One NaN in image 1's carried levels: image 1 runs max_iters steps and is not frozen; every other image's steps
    and levels are bit-identical to those of the same batch with image 1 finite."""
    m, img = TS._model("n64_four_images_per_block", contracting=True)
    with torch.no_grad():
        base = m(img, iters=60)
        noise = torch.randn(base.shape, generator=torch.Generator().manual_seed(2)).to(DEV)
        B = img.shape[0]
        eps = torch.tensor([10.0 ** (1 - 6 * b / (B - 1)) for b in range(B)], device=DEV).view(B, 1, 1, 1)
        start = (base + eps * noise * base.abs().mean()).contiguous()
        r = TS._change(m(img, iters=TS.MAX_ITERS, levels=start, return_all=True))
    tol = TS._pick_tol(r)
    out, steps, _, _, frozen, _ = _settle(m, img, tol, TS.MAX_ITERS, start)
    bad = start.clone()
    bad[1, 3, 1, 5] = float("nan")
    out_n, steps_n, _, _, frozen_n, _ = _settle(m, img, tol, TS.MAX_ITERS, bad)
    assert steps_n[1] == TS.MAX_ITERS and frozen_n[1] == 0
    others = torch.arange(B) != 1
    assert len(np.unique(steps[others].numpy())) >= 2
    assert torch.equal(steps_n[others], steps[others]) and torch.equal(frozen_n[others], frozen[others])
    assert torch.equal(out_n[others.to(DEV)], out[others.to(DEV)])
