"""The engine on every SM count from one pair to a full H100: no result may depend on the grid.

K1, K2, the tokeniser GEMM and the tensor-core backward GEMMs launch min(tiles, pairs) two-CTA pairs, K3 min(items, SMs)
CTAs, so which tiles a CTA walks, and how many, depends on the SM count of the card.  A tile's or item's arithmetic and
its accumulation order are fixed by the shapes (DESIGN.md, "Deterministic backward"), so the grid may change only when a
value is computed, never what is computed.  glom_b200_set_sm_count_target plans every launch for fewer SMs than the card
has; this file runs the engine at such targets and demands the bits of the default grid:

  (a-c) at the shapes of test_forward_oracle / test_backward_oracle / test_settle_implicit, where the default run is
        checked against float64, targets 2 (one pair, two K3 CTAs) and 3 (one pair, three K3 CTAs): one pair then walks
        every tile, so bit-identity carries those suites' per-tile bounds over to the multi-tile machinery (ring phases
        carried over, the wait on the previous tile's bulk store, K2's half-cost dealing, K3's scale hand-off, SETTLE and
        block_fresh skips in the middle of a tile list);
  production  configs[1] at batch 32 at the SM counts of other parts: 16, 32, 60, 64, 114 (H100 PCIe) and 14 (seven
        pairs, which divide no tile count evenly);
  (d)   the target bites: the grids of every tensor-core launch, read from a torch.profiler trace, are those `grids`
        predicts, and a process whose first call ran at a target launches the full grid once the target is cleared.

Every mbarrier wait traps after about 4e9 cycles (GLOM_WAIT_TIMEOUT_CYCLES, about 2 s).  `launch_ms_estimate` scales
DESIGN.md's measured configs[1] kernel times to a shape and a grid; each case asserts it stays far below that.

Observed on one H100 80GB HBM3 (132 SMs, 700 W power limit): see DESIGN.md, "How grid sizes are tested".
"""
import contextlib
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import glom_pytorch_b200 as G
from glom_pytorch_b200 import _native
import test_backward_oracle as BO
import test_cuda_core_oracle as CCO
import test_forward_oracle as FO
import test_production_batch as PB
import test_settle as ST
import test_settle_implicit as TSI
import test_settle_oracle as TSO
from oracle import glom_oracle_torch as OT

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@contextlib.contextmanager
def sm_target(sms):
    """Every launch inside the block planned for at most `sms` SMs; the device's own count (0) restored afterwards."""
    _native.set_sm_count_target(sms)
    try:
        yield
    finally:
        _native.set_sm_count_target(0)


# ----------------------------------------------------------------------------- the grid model
def grids(d, L, n, B, sms, occ_pairs):
    """{launch kind: (work, CTAs)} of every persistent launch at these shapes when `sms` SMs are planned for and at most
    `occ_pairs` two-CTA clusters of a GEMM are co-resident (tc_kernels.cu launch_gemm_impl / launch_attention /
    tokenize_tc, tc_bwd_kernels.cu launch, which has no cluster and so no occupancy bound).  Work is tiles (GEMMs) or
    items per key pass (K3), counted as test_production_batch.regime counts them."""
    pairs, rows, G_ = min(sms // 2, occ_pairs), B * n, 2 * L - 1
    num_m = (rows + 255) // 256
    bn2, _ = OT.forward_tiles(d)

    def gemm(tiles, p=pairs):
        return tiles, 2 * min(tiles, p)
    out = {"k1_g0": gemm(G_ * num_m * (4 * d // 256)),              # step 0 (and the settle queue): group 0 included
           "k1": gemm((G_ - 1) * num_m * (4 * d // 256)),
           "k2": gemm(L * num_m * (d // bn2)),
           "tok": gemm(num_m * (d // bn2))}
    items = ((n + 127) // 128) * L * B
    out["k3"] = (items, min(items, sms))
    if d % 256 == 0:
        bp = sms // 2
        out.update({"bw_pre": gemm(G_ * num_m * (4 * d // 256), bp), "bw_dh": gemm(G_ * num_m * (4 * d // 256), bp),
                    "bw_dx": gemm(G_ * num_m * (d // 256), bp), "bw_dw": gemm(G_ * 2 * (d // 256) * (4 * d // 256), bp),
                    "bw_batch_n": gemm(B * L * ((n + 255) // 256) * ((n + 255) // 256), bp),
                    "bw_batch_d": gemm(B * L * ((n + 255) // 256) * ((d + 255) // 256), bp)})
    return out


def bites(d, L, n, B, sms):
    """The launch kinds whose work exceeds what `sms` SMs give them (pairs or CTAs): their grid is smaller than on a
    full H100 (66 pairs, 132 SMs) wherever the full part's grid exceeds the target's."""
    return sorted(k for k, (work, ctas) in grids(d, L, n, B, sms, sms).items() if work > ctas // (1 if k == "k3" else 2))


# DESIGN.md's measured configs[1] (batch 32) times on one H100 80GB HBM3 at 66 pairs / 132 SMs: K1 5.82, K2 6.29 and
# attention 1.22 ms per 12-step forward; the deterministic backward 65.66 ms per 12 reverse steps (all its launches)
C1_MS = {"k1": 5.82 / 12, "k2": 6.29 / 12, "k3": 1.22 / 12, "bwd_step": 65.66 / 12}
WAIT_TIMEOUT_MS = 2000.0


def launch_ms_estimate(d, L, n, B, sms, backward=True):
    """Estimated longest launch (ms) at `sms` SMs: the configs[1] time scaled by the work (MLP: rows * G * d^2;
    attention: B * L * n^2 * d) and by the grid (66 pairs / the target's, 132 CTAs / the target's).  With `backward`,
    a whole reverse step counts as one launch.  An estimate, not a measurement."""
    mlp = (B * n * (2 * L - 1) * d * d) / (32 * 256 * 11 * 512 * 512)
    att = (B * L * n * n * d) / (32 * 6 * 256 * 256 * 512)
    pairs, ctas = max(1, sms // 2), sms
    est = max(C1_MS["k1"] * mlp * 66 / pairs, C1_MS["k2"] * mlp * 66 / pairs, C1_MS["k3"] * att * 132 / ctas)
    return max(est, C1_MS["bwd_step"] * max(mlp, att) * 66 / pairs) if backward else est


def check_case(d, L, n, B, sms, backward=True):
    """The target changes the grid at these shapes, and the estimated longest launch stays below a tenth of the wait
    timeout."""
    est = launch_ms_estimate(d, L, n, B, sms, backward)
    assert est < WAIT_TIMEOUT_MS / 10, ("a launch could approach the mbarrier wait timeout", d, L, n, B, sms, est)
    b = bites(d, L, n, B, sms)
    assert b, ("the target changes no grid here", d, L, n, B, sms)
    return b


# ----------------------------------------------------------------------------- CPU
def test_symbol_is_exported_and_declared():
    hdr = open(os.path.join(ROOT, "include", "glom_b200.h")).read()
    assert re.search(r"GLOM_B200_API\s+int\s+glom_b200_set_sm_count_target\s*\(\s*int\s+sms\s*\)", hdr)
    assert "glom_b200_set_sm_count_target" in _native.EXPORTS


def test_target_round_trip_and_argument_errors():
    """-1 and 1 are rejected (the target is left as it was); a valid value returns the previous one.  No device is
    touched (this runs without one)."""
    lib = _native.load()
    assert lib.glom_b200_set_sm_count_target(0) == 0
    try:
        for bad in (-1, 1, -132):
            assert lib.glom_b200_set_sm_count_target(bad) == -1, bad
            assert "SM-count target" in lib.glom_b200_last_error().decode()
        assert lib.glom_b200_set_sm_count_target(14) == 0
        assert lib.glom_b200_set_sm_count_target(1) == -1
        assert lib.glom_b200_set_sm_count_target(1000) == 14          # larger than any part: clamped at launch
        assert _native.set_sm_count_target(2) == 1000
        with pytest.raises(_native.GlomB200Error, match="SM-count target"):
            _native.set_sm_count_target(1)
        with sm_target(3):
            assert lib.glom_b200_set_sm_count_target(3) == 3
    finally:
        lib.glom_b200_set_sm_count_target(0)
    assert lib.glom_b200_set_sm_count_target(0) == 0


def test_grid_model_arithmetic():
    """grids() at configs[1], batch 32 on a full H100 (132 SMs, 66 co-resident pairs), at one pair and at seven; its
    work over pairs / SMs is test_production_batch.regime."""
    g = grids(512, 6, 256, 32, 132, 66)
    assert g["k1_g0"] == (2816, 132) and g["k1"] == (2560, 132) and g["k2"] == (384, 132) and g["k3"] == (384, 132)
    assert g["tok"] == (64, 128) and g["bw_batch_n"] == (192, 132) and g["bw_batch_d"] == (384, 132)
    assert g["bw_pre"] == (2816, 132) and g["bw_dx"] == (704, 132) and g["bw_dw"] == (352, 132)
    r = PB.regime(512, 6, 256, 32, 132)
    assert (g["k1"][0] / 66, g["k2"][0] / 66, g["k3"][0] / 132, g["tok"][0] / 66) == (r["k1"], r["k2"], r["k3"], r["tok"])
    assert min(v[0] for k, v in g.items() if k.startswith("bw_")) / 66 == r["bwd"]
    for sms, ctas, k3 in ((2, 2, 2), (3, 2, 3), (14, 14, 14)):
        g = grids(512, 6, 256, 32, sms, 66)
        assert all(v[1] == (k3 if k == "k3" else ctas) for k, v in g.items()), (sms, g)
    # the occupancy bound lowers the forward GEMMs only
    g = grids(512, 6, 256, 32, 132, 60)
    assert g["k1"][1] == 120 and g["k3"][1] == 132 and g["bw_dw"][1] == 132
    # a small shape: d64_n9 (27 rows, one row block) still has more K1 tiles and K3 items than one pair / two CTAs
    assert grids(64, 3, 9, 3, 2, 66)["k1"] == (4, 2) and grids(64, 3, 9, 3, 3, 66)["k3"] == (9, 3)
    assert bites(64, 3, 9, 3, 2) == ["k1", "k1_g0", "k2", "k3"]
    assert "tok" not in bites(512, 6, 256, 32, 132) and "tok" in bites(512, 6, 256, 32, 114)


def test_launch_estimates_stay_below_the_timeout():
    """configs[1] at batch 32: K2 at one pair is the longest forward launch (~35 ms); a whole reverse step at seven
    pairs ~52 ms.  Every oracle shape this file runs at target 2 stays below a tenth of the 2 s wait timeout."""
    assert launch_ms_estimate(512, 6, 256, 32, 2, backward=False) == pytest.approx(C1_MS["k2"] * 66, rel=1e-12)
    assert launch_ms_estimate(512, 6, 256, 32, 14) == pytest.approx(C1_MS["bwd_step"] * 66 / 7, rel=1e-12)
    for name, (dim, L, isz, p, hw, B, _, _) in FO.SHAPES.items():
        hw = hw or (isz, isz)
        assert launch_ms_estimate(dim, L, (hw[0] // p) * (hw[1] // p), B, 2) < WAIT_TIMEOUT_MS / 10, name
    for name, (dim, L, isz, p, hw, B, _, _, _) in BO.SHAPES.items():
        hw = hw or (isz, isz)
        assert launch_ms_estimate(dim, L, (hw[0] // p) * (hw[1] // p), B, 2) < WAIT_TIMEOUT_MS / 10, name


# ----------------------------------------------------------------------------- helpers
def _same(a, b, what):
    """Bit for bit, tensors or dicts / tuples of tensors."""
    if isinstance(a, dict):
        assert set(a) == set(b), (what, set(a) ^ set(b))
        for k in a:
            _same(a[k], b[k], (what, k))
        return
    if isinstance(a, (tuple, list)):
        assert len(a) == len(b), what
        for i, (x, y) in enumerate(zip(a, b)):
            _same(x, y, (what, i))
        return
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape, a.dtype, b.dtype)
    if not torch.equal(a, b):
        diff = a != b
        if a.is_floating_point():
            diff = diff & ~(torch.isnan(a) & torch.isnan(b))
            if not diff.any():
                return
        idx = diff.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(diff.sum())} of {a.numel()} elements differ, first at {idx}: "
                             f"{a[tuple(idx)].item()!r} vs {b[tuple(idx)].item()!r}")


def _across_targets(run, targets, dims, what):
    """run() at the default grid, then at every target: each must give the default's bits."""
    want = run()
    for t in targets:
        check_case(*dims, t)
        with sm_target(t):
            _same(run(), want, (what, t))
    return want


def _cpu(x):
    if isinstance(x, dict):
        return {k: _cpu(v) for k, v in x.items()}
    if isinstance(x, (tuple, list)):
        return type(x)(_cpu(v) for v in x)
    return x.detach().cpu().clone()


def _split_tol(r):
    """A tol between the images' smallest changes (r: (B, T) from test_settle._change), so some stop early and the rest
    run on; one image: between its smallest and largest change."""
    lo = np.sort(r.min(axis=1))
    vals = np.unique(lo[lo > 0]) if len(lo) > 1 else np.unique(r[r > 0])
    if len(vals) < 2:
        return float(vals[0]) if len(vals) else 1e-3
    mid = len(vals) // 2
    return float(np.sqrt(vals[mid - 1] * vals[mid]))


def _spread(m, img, max_iters):
    """test_production_batch._spread's start (noise over six decades across the images) and a tol that splits them."""
    N = img.shape[0]
    with torch.no_grad():
        base = m(img, iters=60)
        noise = torch.randn(base.shape, generator=torch.Generator().manual_seed(2)).to(DEV)
        eps = torch.tensor([10.0 ** (1 - 6 * b / (N - 1)) for b in range(N)], device=DEV).view(N, 1, 1, 1)
        start = (base + eps * noise * base.abs().mean()).contiguous()
        r = ST._change(m(img, iters=max_iters, levels=start, return_all=True))
    return start, _split_tol(r)


# ----------------------------------------------------------------------------- GPU (a): forward at the oracle shapes
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(FO.SHAPES))
def test_forward_bits_at_one_pair(name):
    """forward(iters=3, return_all=True) from a carried state and from init_levels; S_1 with the workspace H, C and
    squared-norm partials (test_forward_oracle._engine, after one and two steps); a per-image step vector with
    return_all; settle at a tol that splits the images, with its change partials, ratios and flags."""
    m, img, S, n = FO._model(name, "bf16")
    img, S = img.to(DEV), S.to(DEV)
    B, L, d = img.shape[0], m.levels, m.dim
    steps = torch.tensor([3] + [(3 * b + 1) % 4 for b in range(1, B)])      # T = 3, images at 0 .. 3
    with torch.no_grad():
        r = ST._change(m(img, iters=3, levels=S, return_all=True))
    # between the two smallest first-step changes: one image stops after step 1, the rest later (one image: between its
    # first two changes, so it stops before step 3)
    first = np.unique(r[:, 0]) if B > 1 else np.sort(r[0, :2])
    tol = float(np.sqrt(first[0] * first[1]))

    def run():
        out = {}
        with torch.no_grad():
            out["carried"] = m(img, iters=3, levels=S, return_all=True)
            out["init"] = m(img, iters=3, return_all=True)
            out["steps"] = m(img, iters=steps, levels=S, return_all=True)
        out["one_step"] = FO._engine(m, img, S, 1)
        out["two_steps_nsq"] = FO._engine(m, img, S, 2)[3]
        out["settle"] = TSO._settle(m, img, tol, 3, S)
        return _cpu(out)
    want = _across_targets(run, (2, 3), (d, L, n, B), name)
    settled = want["settle"][1].numpy()
    assert settled.min() < 3 and (B == 1 or len(np.unique(settled)) >= 2), settled
    print(f"[sm-count] {name}: bit-identical at targets 2, 3; settle steps {want['settle'][1].tolist()}")


@pytest.mark.gpu
@pytest.mark.parametrize("dim,p,hw,B", FO.TOKENISER, ids=[f"d{t[0]}_p{t[1]}_{t[2][0]}x{t[2][1]}_B{t[3]}" for t in FO.TOKENISER])
def test_tokeniser_bits_at_one_pair(dim, p, hw, B):
    from oracle import glom_oracle as O
    isz = max(hw)
    params = O.synth_params(dim, 2, isz, p, seed=4)
    m = G.Glom(dim=dim, levels=2, image_size=isz, patch_size=p, precision="bf16")
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=False)
    m = m.to(DEV)
    img = torch.randn((B, 3) + hw, generator=torch.Generator().manual_seed(5)).to(DEV)

    def run():
        with torch.no_grad():
            return m.tokens(img).cpu()
    want = run()
    for t in (2, 3):
        with sm_target(t):
            _same(run(), want, ("tokens", dim, p, hw, B, t))


# ----------------------------------------------------------------------------- GPU (b): backward at the oracle shapes
def _bwd_runs(m, img, S, g, B):
    T = 3
    cot1 = torch.randn(S.shape, generator=g)
    cotT = torch.randn((T + 1,) + tuple(S.shape), generator=g)
    steps = torch.tensor([3] + [(3 * b + 1) % 4 for b in range(1, B)])      # T = 3, images at 0 .. 3

    def run():
        out = {}
        for key, it, ra, cot in (("one_step", 1, False, cot1), ("chain", T, True, cotT), ("steps", steps, True, cotT)):
            o, got = BO._engine_run(m, img, S, it, ra, cot)
            out[key] = (o, got)
        return _cpu(out)
    return run


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(BO.SHAPES))
def test_deterministic_backward_bits_at_one_pair(name):
    """Under torch.use_deterministic_algorithms: one step, a T = 3 chain with return_all and a per-image step vector,
    every gradient bit for bit at targets 2 and 3 (tensor-core, mixed and CUDA-core paths).  The default (atomic)
    backward at target 2 is within test_production_batch.DEFAULT_TOL of the deterministic default grid."""
    from test_deterministic_backward import deterministic
    m, img, S, n, g = BO._model(name, "bf16")
    B = img.shape[0]
    run = _bwd_runs(m, img, S, g, B)
    with deterministic():
        want = _across_targets(run, (2, 3), (m.dim, m.levels, n, B), name)
    with deterministic(False), sm_target(2):
        plain = run()
    for key in want:
        errs = BO.errors(plain[key][1], want[key][1], m.levels, n)
        BO._report(name, f"{key}: atomic at target 2 vs deterministic default", errs)
        BO.check(errs, PB.DEFAULT_TOL, (name, key, "atomic"))


# ----------------------------------------------------------------------------- GPU (c): implicit, queue, video
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(TSI.SHAPES))
def test_implicit_backward_bits_at_one_pair(name):
    """settle(differentiable="implicit") under the deterministic flag: levels, steps, every gradient, K_b and q."""
    from test_deterministic_backward import deterministic
    m, img, start, cot = TSI._setup(name)
    dim, L, isz, p, _, _, B, _ = TSI.SHAPES[name]

    def run():
        with torch.no_grad():
            levels, steps = m.settle(img, 1e-4, TSI.MAX_ITERS, levels=start)
        grads, K = TSI._det_grads(m, img, start, cot, adjoint_iters=8)
        return _cpu((levels, steps, grads, K, m.last_adjoint[1]))
    with deterministic():
        want = _across_targets(run, (2, 3), (dim, L, (isz // p) ** 2, B), name)
    print(f"[sm-count] implicit {name}: steps {want[1].tolist()} K {want[3].tolist()}")


QUEUE_DIMS = (256, 3, 48, 4)          # n = 144: 2 x 144 = 288 rows, so a slot's rows straddle 256-row blocks


@pytest.mark.gpu
@pytest.mark.parametrize("N", [5, 9])
def test_settle_queue_bits(N):
    """settle_queue(N images, 3 slots): the images enter at different steps, so K1's block_fresh group-0 tiles sit in
    the middle of its tile list."""
    m = PB._contracting(*QUEUE_DIMS)
    img = torch.randn(N, 3, 48, 48, generator=torch.Generator().manual_seed(N)).to(DEV)
    start, tol = _spread(m, img, 12)

    def run():
        with torch.no_grad():
            return _cpu(m.settle_queue(img, tol, max_iters=12, levels=start, slots=3))
    want = _across_targets(run, (2, 3, 7), (256, 3, 144, 3), ("queue", N))
    assert len(np.unique(want[1].numpy())) >= 2, want[1]
    print(f"[sm-count] settle_queue N={N}: steps {want[1].tolist()}")


@pytest.mark.gpu
def test_settle_video_bits():
    """settle_video(3 streams x 4 frames, 2 slots)."""
    m = PB._contracting(*QUEUE_DIMS)
    frames = torch.randn(3, 4, 3, 48, 48, generator=torch.Generator().manual_seed(7)).to(DEV)
    with torch.no_grad():
        base = m(frames[:, 0], iters=60)
    noise = torch.randn(base.shape, generator=torch.Generator().manual_seed(2)).to(DEV)
    start = (base + noise * base.abs().mean() * torch.tensor([1.0, 1e-2, 1e-4], device=DEV).view(3, 1, 1, 1))

    def run():
        with torch.no_grad():
            return _cpu(m.settle_video(frames, 1e-3, max_iters=12, levels=start, slots=2))
    want = _across_targets(run, (2, 3, 7), (256, 3, 144, 2), "video")
    print(f"[sm-count] settle_video: steps {want[1].tolist()}")


# ----------------------------------------------------------------------------- GPU: the fp32 engine at one pair
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["d132_L2_9x13_p1_B5", "d36_L5_40x40_p5_r2.5_self"])
def test_fp32_engine_bits_at_one_pair(name):
    """The fp32 engine's grid-stride loops wrap many times at two SMs: a 3-step chain from a carried state and its
    deterministic backward with a cotangent on every slab."""
    from test_deterministic_backward import deterministic
    m, img, S, n, g = CCO._model(name)
    cot = torch.randn((4,) + tuple(S.shape), generator=g)

    def run():
        with torch.no_grad():
            chain = m(img.to(DEV), iters=3, levels=S.to(DEV), return_all=True)
        return _cpu((chain, BO._engine_run(m, img, S, 3, True, cot)))
    with deterministic():
        want = run()
        with sm_target(2):
            _same(run(), want, (name, 2))


# ----------------------------------------------------------------------------- GPU: production shapes, other parts
PROD_TARGETS = [16, 32, 60, 64, 114, 14]


@pytest.fixture(scope="module")
def prod():
    """configs[1] at batch 32: every production check and its result at the default grid."""
    from test_deterministic_backward import deterministic
    B, T = 32, 12
    m, img, S, n, _ = PB._bwd_model(B)
    img, S = img.to(DEV), S.to(DEV)
    steps = torch.tensor([12 if b % 2 == 0 else (b // 2) % 12 for b in range(B)])
    cot = torch.randn((T + 1,) + tuple(S.shape), generator=torch.Generator(device=DEV).manual_seed(3), device=DEV)
    c = PB._contracting(512, 6, 224, 14)
    imgs = torch.randn(64, 3, 224, 224, generator=torch.Generator().manual_seed(1)).to(DEV)
    q_start, q_tol = _spread(c, imgs, 12)
    s_img, s_start, s_tol = imgs[::2].contiguous(), q_start[::2].contiguous(), q_tol     # every decade of noise
    imp = G.Glom(dim=512, levels=6, image_size=224, patch_size=14).to(DEV)
    with torch.no_grad():
        imp.bottom_up.net[3].weight.mul_(0.05)
        imp.top_down.net[3].weight.mul_(0.05)
        imp_start = imp(imgs[:B], iters=40)
        imp_start = imp_start + torch.randn(imp_start.shape, generator=torch.Generator().manual_seed(2)).to(DEV) * 1e-3
    imp_cot = torch.randn(imp_start.shape, generator=torch.Generator().manual_seed(5)).to(DEV)

    def forward():
        with torch.no_grad():
            return m(img, iters=T, return_all=True)

    def settle():
        with torch.no_grad():
            return c.settle(s_img, s_tol, max_iters=12, levels=s_start)

    def queue():
        with torch.no_grad():
            return c.settle_queue(imgs, q_tol, max_iters=12, levels=q_start, slots=32)

    def train():
        with deterministic():
            return PB._grads(m, img.clone(), S.clone(), steps, lambda out: (out * cot).sum())

    def implicit():
        with deterministic():
            g, K = TSI._det_grads(imp, imgs[:B], imp_start, imp_cot, adjoint_iters=8)
        return g, K, imp.last_adjoint[1].clone()
    runs = {"forward": forward, "settle": settle, "settle_queue": queue, "train": train, "implicit": implicit}
    case = {"runs": runs, "want": {k: f() for k, f in runs.items()}, "n": n}
    print(f"[sm-count] configs[1] B=32: settle steps {case['want']['settle'][1].tolist()}, queue steps "
          f"{case['want']['settle_queue'][1].tolist()}")
    assert len(np.unique(case["want"]["settle"][1].cpu().numpy())) >= 3
    yield case
    case.clear()


@pytest.mark.gpu
@pytest.mark.parametrize("target", PROD_TARGETS)
def test_configs1_bits_at_other_sm_counts(target, prod):
    """forward(iters=12, return_all=True), settle, settle_queue(N=64, slots=32), bench.py's deterministic training step
    with a per-image step vector and a cotangent on every slab (every gradient), and the deterministic implicit backward:
    the default grid's bits at the SM counts of other parts."""
    case = prod
    b = check_case(512, 6, case["n"], 32, target)
    with sm_target(target):
        for k, f in case["runs"].items():
            _same(f(), case["want"][k], (k, target))
    print(f"[sm-count] configs[1] B=32 at {target} SMs: bit-identical ({', '.join(b)} re-dealt)")


@pytest.mark.gpu
def test_configs1_forward_bits_at_one_pair(prod):
    case = prod
    check_case(512, 6, case["n"], 32, 2, backward=False)
    with sm_target(2):
        _same(case["runs"]["forward"](), case["want"]["forward"], ("forward", 2))


# ----------------------------------------------------------------------------- GPU (d): the target bites
def _launches(fn, path):
    """[(kind, grid x)] of the tensor-core launches fn() makes, from a torch.profiler trace written to `path`."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    prof.export_chrome_trace(str(path))
    return _parse_trace(path)


BWD_MODES = {0: "bw_pre", 1: "bw_dh", 2: "bw_dx", 3: "bw_dw", 4: "bw_batch"}
FWD_MODES = {0: "k1", 1: "k2", 2: "tok"}


def _parse_trace(path):
    with open(path) as f:
        events = json.load(f)["traceEvents"]
    kernels = [e for e in events if e.get("cat") == "kernel"]
    assert kernels, "the profiler trace holds no kernel events"
    out = []
    for e in kernels:
        name, grid = e["name"], e["args"]["grid"][0]
        mb, mf = re.search(r"bwd_gemm_kernel<(\d+)", name), re.search(r"\bgemm_kernel<(\d+)", name)
        if mb:
            out.append((BWD_MODES[int(mb.group(1))], grid))
        elif mf:
            out.append((FWD_MODES[int(mf.group(1))], grid))
        elif re.search(r"\battn_kernel<", name):
            out.append(("k3", grid))
    return out


BITE_SHAPE = (512, 6, 224, 14, 8)     # configs[1] at batch 8: dim, levels, image_size, patch_size, batch


def _bite_model():
    from oracle import glom_oracle as O
    dim, L, isz, p, B = BITE_SHAPE
    params = O.synth_params(dim, L, isz, p, seed=0)
    m = G.Glom(dim=dim, levels=L, image_size=isz, patch_size=p, precision="bf16")
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=False)
    m = m.to(DEV)
    img = torch.randn(B, 3, isz, isz, generator=torch.Generator().manual_seed(3)).to(DEV)
    return m, img, (isz // p) ** 2


def _expected(kind, g):
    """The grid(s) a launch of `kind` may have under the model g = grids(...)."""
    if kind == "k1":
        return {g["k1"][1], g["k1_g0"][1]}
    if kind == "bw_batch":
        return {g["bw_batch_n"][1], g["bw_batch_d"][1]}
    return {g[kind][1]}


@pytest.mark.gpu
@pytest.mark.parametrize("target", [2, 3, 14, 0])
def test_target_sets_every_grid(target, tmp_path):
    """One forward (iters=2 from init_levels, return_all, the tokeniser included) and its backward under the profiler:
    every gemm_kernel, attn_kernel and bwd_gemm_kernel launch has the grid grids() predicts, which is at most the
    target's bound and reaches it where the work exceeds it.  At 0 the forward GEMMs' pair count is the device's
    co-resident cluster count, at most SMs / 2."""
    dim, L, isz, p, B = BITE_SHAPE
    m, img, n = _bite_model()
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    if target:
        check_case(dim, L, n, B, target)

    def step():
        x = img.clone().requires_grad_(True)
        m(x, iters=2, return_all=True).square().mean().backward()
    step()                                                     # warm-up: packed weights, workspaces
    with sm_target(target):
        got = _launches(step, tmp_path / "trace.json")
    kinds = {k for k, _ in got}
    assert kinds == {"k1", "k2", "k3", "tok", "bw_pre", "bw_dh", "bw_dx", "bw_dw", "bw_batch"}, kinds
    planned = target or sms
    occ = planned // 2
    if target == 0:
        occ = max(gr for k, gr in got if k == "k1") // 2
        assert 1 <= occ <= sms // 2, (occ, sms)
    g = grids(dim, L, n, B, planned, occ)
    for kind, grid in got:
        assert grid in _expected(kind, g), (target, kind, grid, _expected(kind, g))
        bound = planned if kind == "k3" else 2 * ((occ if kind in FWD_MODES.values() else planned // 2))
        assert grid <= bound, (target, kind, grid, bound)
    for kind, (work, ctas) in g.items():
        bound = planned if kind == "k3" else 2 * ((occ if not kind.startswith("bw_") else planned // 2))
        if work * (1 if kind == "k3" else 2) > bound:
            assert ctas == bound
    seen = {}
    for kind, grid in got:
        seen.setdefault(kind, set()).add(grid)
    print(f"[sm-count] target {target} ({planned} SMs, {occ} pairs): "
          + " ".join(f"{k}={sorted(v)}" for k, v in sorted(seen.items())))


FRESH_PROCESS = r"""
import os
import sys
import torch
for sub in ("", "tests", "tests/golden"):
    sys.path.insert(0, os.path.join(sys.argv[2], sub))
import test_sm_count as T
from glom_pytorch_b200 import _native
m, img, n = T._bite_model()
_native.set_sm_count_target(4)                       # the process's first engine call runs at four SMs
with torch.no_grad():
    m(img, iters=2)
torch.cuda.synchronize()
_native.set_sm_count_target(0)
def fwd():
    with torch.no_grad():
        m(img, iters=2)
T._launches(fwd, sys.argv[1])
"""


@pytest.mark.gpu
def test_first_call_at_a_target_does_not_pin_the_pair_count(tmp_path):
    """A fresh process whose first call runs at target 4, then at 0: K1 and K2 launch the default grid, which is the
    co-resident pair count and not the two pairs of the first call (the occupancy query is cached per device and the
    SM count bounds it on every call)."""
    dim, L, isz, p, B = BITE_SHAPE
    m, img, n = _bite_model()

    def fwd():
        with torch.no_grad():
            m(img, iters=2)
    here = _launches(fwd, tmp_path / "here.json")
    trace = tmp_path / "fresh.json"
    script = tmp_path / "fresh.py"
    script.write_text(FRESH_PROCESS)
    r = subprocess.run([sys.executable, str(script), str(trace), ROOT], capture_output=True, text=True, timeout=600,
                       cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    fresh = _parse_trace(trace)
    by_kind = lambda ls, k: sorted({gr for kk, gr in ls if kk == k})
    g = grids(dim, L, n, B, 4, 66)
    for kind in ("k1", "k2"):
        assert by_kind(fresh, kind) == by_kind(here, kind), (kind, by_kind(fresh, kind), by_kind(here, kind))
        assert max(by_kind(fresh, kind)) > max(_expected(kind, g)), (kind, by_kind(fresh, kind))
    print(f"[sm-count] fresh process after target 4: k1 {by_kind(fresh, 'k1')} k2 {by_kind(fresh, 'k2')}")
