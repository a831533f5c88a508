"""The engine at production batch sizes, where every persistent kernel walks several tiles or items per CTA.

K1, K2, the tokeniser GEMM and the tensor-core backward GEMMs launch min(tiles, pairs) two-CTA clusters and K3
min(items, SMs) CTAs, so at the batches of the oracle suites (1 to 5 images) each CTA gets one tile and the per-CTA
machinery never runs: ring phases carried from tile to tile, the wait on the previous tile's bulk store, K2's half-cost
top-level dealing, the attention kernel's double-buffered scale hand-off, SETTLE skips in the middle of a tile list.
Every GPU case here first asserts, from the shapes and the SM count, that it is in that regime (`regime`).

Two kinds of check:
  per tile   one step (forward) or one reverse step (backward) at the production batch against the float64 references
             of test_forward_oracle / test_backward_oracle, per block of the kernels' tiling, at their bounds;
  slicing    rows, consensus items and tiles are independent across images (DESIGN.md), so a call at batch B must
             equal, bit for bit, the same call made on slices of the batch sizes the oracle suites pin: two images at
             configs[1] (as config2_dims / tc_config2_dims at B = 2), one or a few images elsewhere.  Those slices
             still deal a few K1 tiles per pair (2.4 at configs[1]), and the backward's BW_DW deals the same tiles
             at any batch, but every such launch is checked against float64 there.  This holds for the forward,
             settle, settle_queue, the tokeniser and, under torch.use_deterministic_algorithms, for the per-image
             gradients (d_img, d_levels).
The batch-summed gradients (weights, biases, pos_emb, init_levels, tokeniser) sum rows of every image in fp32, so they
are compared with the float64 sum of the slices' gradients at batch_sum_tol (3.0e-4 at configs[1]); the CPU tests show
that plausible faults of the multi-tile schedule miss that bound by >= 3x (18x at least).

Observed on one H100 80GB HBM3 (400 W power limit, 132 SMs, 66 pairs): every slicing check bit-identical; per tile at
most rel 3.3e-4 / abs 6.1e-3 (emu), 1.2e-3 / 1.2e-3 (tc, forward), 4.3e-3 / 5.4e-3 (tc, backward), 1.5e-4 / 6.9e-4
(tc_emu), tokeniser 5.1e-7 / 8.6e-7; deterministic batch sums within 2.9e-5 of the slices; the default mode's batch
sums within 1.4e-3 and its d_img / d_levels within 7.0e-4; about 90 s for the file.
"""
import math
import os
import subprocess

import numpy as np
import pytest
import torch

import glom_pytorch_b200 as G
import test_backward_oracle as BO
import test_forward_oracle as FO
from oracle import glom_oracle as O
from oracle import glom_oracle_torch as OT

DEV = "cuda:0"
U32 = 2.0 ** -24          # fp32 unit roundoff


# ----------------------------------------------------------------------------- the regime guard
def regime(d, L, n, B, num_sms):
    """Work items over grid size of each persistent launch at these shapes (tc_kernels.cu step_bf16 /
    launch_attention / tokenize_tc, tc_bwd_kernels.cu).  Pairs are bounded by num_sms / 2: the occupancy query the
    GEMM launch also applies can only lower that, which only raises the ratios."""
    pairs, rows, G_ = num_sms // 2, B * n, 2 * L - 1
    num_m = (rows + 255) // 256
    bn2, _ = OT.forward_tiles(d)
    k1 = (G_ - 1) * num_m * (4 * d // 256)                      # steps after the first skip group 0
    k2 = L * num_m * (d // bn2)
    k3 = ((n + 127) // 128) * L * B                              # per key pass
    tok = num_m * (d // bn2)                                     # the tokeniser's N tile is K2's
    out = {"k1": k1 / pairs, "k2": k2 / pairs, "k3": k3 / num_sms, "tok": tok / pairs}
    if d % 256 == 0:                                             # tensor-core backward
        nm = (rows + 255) // 256
        bw = {"pre": G_ * nm * (4 * d // 256), "dx": G_ * nm * (d // 256), "dw": G_ * 2 * (d // 256) * (4 * d // 256),
              "batch": B * L * ((n + 255) // 256) * ((min(n, d) + 255) // 256)}
        out["bwd"] = min(bw.values()) / pairs
    return out


def guard(d, L, n, B, kernels=("k1", "k2", "k3")):
    """Assert that every kernel of `kernels` runs several tiles / items per CTA: K1 and K2 >= 3 tiles per pair; K3 and
    the backward GEMMs (BW_BATCH: 192 problems at configs[1], B = 32) >= 2; the tokeniser more tiles than pairs."""
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    r = regime(d, L, n, B, sms)
    need = {"k1": 3, "k2": 3, "bwd": 2, "k3": 2, "tok": 1 + 1e-9}
    low = {k: r[k] for k in kernels if r[k] < need[k]}
    print(f"[production] d{d} L{L} n{n} B{B} on {sms} SMs ({sms // 2} pairs): "
          + " ".join(f"{k}={r[k]:.2f}" for k in kernels))
    assert not low, ("back in the one-tile regime", sms, low)
    return r


def test_regime_arithmetic():
    """The guard's counts at configs[1], B = 32 on 132 SMs: 38.8 K1 tiles per pair, 5.8 K2 tiles, 2.9 K3 items per
    CTA; the tokeniser needs B >= 34 to give the 66 pairs more than one tile."""
    r = regime(512, 6, 256, 32, 132)
    assert (round(r["k1"], 1), round(r["k2"], 1), round(r["k3"], 1)) == (38.8, 5.8, 2.9)
    assert r["tok"] < 1 and regime(512, 6, 256, 34, 132)["tok"] > 1
    assert regime(1024, 8, 576, 8, 132)["k2"] == pytest.approx(576 / 66)


# ----------------------------------------------------------------------------- CPU: K1 / K2 schedule, every pair count
def _nvcc():
    import shutil
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    return None


def test_gemm_schedule_for_every_pair_count(tmp_path):
    """tests/native/sched_tile_harness.cu, compiled from gemm_sched.cuh (the kernels' own decode_tile / sched_tile):
    for C = 1..66 pairs (H100 PCIe, SXM, NVL and MIG slices have different SM counts; a GPU run covers one) and the
    tile counts of L = 2..8, num_n in {1..5, 8, 16}, num_m = 1..40, every K1 and K2 tile is dealt exactly once, K2's
    half-cost tiles are the top level's, and K2's per-pair cost (full 2, half 1) differs by at most 2."""
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    here = os.path.dirname(os.path.abspath(__file__))
    csrc = os.path.join(os.path.dirname(here), "glom_pytorch_b200", "csrc")
    exe = str(tmp_path / "sched_tile_harness")
    subprocess.run([nvcc, "-std=c++17", "-O2", "-gencode", "arch=compute_90a,code=sm_90a", "-I", csrc,
                    os.path.join(here, "native", "sched_tile_harness.cu"), "-o", exe], check=True, capture_output=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(r.stdout)
    assert r.returncode == 0, r.stdout
    last = r.stdout.strip().splitlines()[-1].split()
    assert last[:4] == ["configs", "129360", "failures", "0"], r.stdout
    assert int(last[5]) <= 2 and int(last[7]) <= 1, r.stdout


# ----------------------------------------------------------------------------- helpers
def _glom(dim, L, isz, p, *, seed=0, **kw):
    """A bf16 model with synth_params weights (eval mode: the resume path of carried states is live)."""
    params = O.synth_params(dim, L, isz, p, seed=seed)
    m = G.Glom(dim=dim, levels=L, image_size=isz, patch_size=p, precision="bf16", **kw)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=False)
    m.image_side = isz
    return m.to(DEV).eval()


def _inputs(m, B, seed):
    """(B, 3, isz, isz) images and a random carried state on the GPU, and n."""
    g = torch.Generator().manual_seed(seed)
    isz = m.image_side
    img = torch.randn(B, 3, isz, isz, generator=g)
    n = (isz // m.patch_size) ** 2
    S = torch.randn(B, n, m.levels, m.dim, generator=g)
    return img.to(DEV), S.to(DEV), n


def _sliced(fn, B, k, dim=0):
    """fn(lo, hi) over slices of k images, concatenated along `dim`."""
    return torch.cat([fn(lo, min(lo + k, B)) for lo in range(0, B, k)], dim=dim)


def _equal(a, b, what):
    assert a.shape == b.shape, (what, a.shape, b.shape)
    if not torch.equal(a, b):
        diff = (a != b)
        idx = diff.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(diff.sum())} elements differ, first at {idx}")


def _per_tile_step(m, img, S, n, name):
    """test_one_step at this batch: S_1, H, C vs step_forward_bf16 (emu), S_1 vs column_step (tc), the squared-norm
    partials of S_2 vs float64 sums of squares (nsq).  S = None: from init_levels (then emu only)."""
    out, H, C, _ = FO._engine(m, img, S, 1)
    B = img.shape[0]
    S0 = m.init_levels.detach().cpu()[None, None].expand(B, n, m.levels, m.dim) if S is None else S.cpu()
    tok, P, pos, mask = FO._ref_inputs(m, img, n)
    meta = tuple(S0.shape)
    emu = FO._emu(m, tok, P, pos, mask, S0)
    errs = FO.errors({"state": out, "H": H, "C": C}, {k: emu[k] for k in ("state", "H", "C")}, meta)
    FO._report(name, f"B={B} one step vs step_forward_bf16", errs)
    FO.check(errs, FO.TOL["emu"], name)
    if S is None:
        return
    errs = FO.errors({"state": out}, {"state": FO._exact(m, tok, P, pos, mask, S0)}, meta)
    FO._report(name, f"B={B} one step vs column_step", errs)
    FO.check(errs, FO.TOL["tc"], name)
    s2, _, _, nsq = FO._engine(m, img, S, 2)
    errs = FO.errors({"nsq": nsq}, {"nsq": FO._sumsq_parts(s2)}, meta)
    FO._report(name, f"B={B} nsq of S_2", errs)
    FO.check(errs, FO.TOL["nsq"], name)


CFG1 = (512, 6, 224, 14)          # configs[1]: dim, levels, image_size, patch_size
CFG3 = (1024, 8, 384, 16)         # configs[3]


# ----------------------------------------------------------------------------- GPU: forward, configs[1] B = 32
@pytest.mark.gpu
@pytest.mark.parametrize("carried", [True, False], ids=["carried", "init_levels"])
def test_configs1_one_step_per_tile(carried):
    m = _glom(*CFG1)
    img, S, n = _inputs(m, 32, seed=11)
    guard(512, 6, n, 32)
    _per_tile_step(m, img, S.cpu() if carried else None, n, "configs[1]")


@pytest.mark.gpu
@pytest.mark.parametrize("carried", [True, False], ids=["carried", "init_levels"])
def test_configs1_equals_two_image_slices(carried):
    """forward(iters=12, return_all=True) and forward(iters=12) at B = 32 against 16 two-image calls, slab for slab."""
    m = _glom(*CFG1)
    img, S, n = _inputs(m, 32, seed=12)
    guard(512, 6, n, 32)
    start = S if carried else None

    def call(lo, hi, return_all):
        return m(img[lo:hi], iters=12, levels=None if start is None else start[lo:hi], return_all=return_all)
    with torch.no_grad():
        full = m(img, iters=12, levels=start, return_all=True)
        _equal(full, _sliced(lambda a, b: call(a, b, True), 32, 2, dim=1), "return_all")
        del full
        full = m(img, iters=12, levels=start)
        _equal(full, _sliced(lambda a, b: call(a, b, False), 32, 2), "last slab")


@pytest.mark.gpu
def test_configs4_chain_equals_slices():
    """configs[4]: 12 -> 10 -> 6 with the state carried (the resume path) at B = 32 equals the chain run per slice."""
    m = _glom(*CFG1)
    imgs = [_inputs(m, 32, seed=20 + f)[0] for f in range(3)]
    guard(512, 6, 256, 32)

    def chain(lo, hi):
        lv = m(imgs[0][lo:hi], iters=12)
        lv = m(imgs[1][lo:hi], iters=10, levels=lv)
        return m(imgs[2][lo:hi], iters=6, levels=lv)
    with torch.no_grad():
        full = chain(0, 32)
        _equal(full, _sliced(chain, 32, 2), "configs[4] chain")


# ----------------------------------------------------------------------------- GPU: forward, configs[3] B = 8
@pytest.mark.gpu
def test_configs3_equals_one_image_slices():
    """configs[3] (d 1024, L 8, n 576) at B = 8 for 16 steps equals eight one-image calls; one step of a one-image slice
    passes the per-tile check."""
    m = _glom(*CFG3)
    img, S, n = _inputs(m, 8, seed=13)
    guard(1024, 8, n, 8)
    with torch.no_grad():
        full = m(img, iters=16)
        _equal(full, _sliced(lambda a, b: m(img[a:b], iters=16), 8, 1), "configs[3] iters=16")
        full = m(img, iters=16, levels=S, return_all=True)
        _equal(full, _sliced(lambda a, b: m(img[a:b], iters=16, levels=S[a:b], return_all=True), 8, 1, dim=1),
               "configs[3] return_all carried")
    del full
    _per_tile_step(m, img[:1], S[:1].cpu(), n, "configs[3] slice")


# ----------------------------------------------------------------------------- GPU: the other K2 widths and K3 paths
# name in test_forward_oracle.SHAPES -> batch that passes the guard (K2 tiles per pair, K3 items per CTA on 132 SMs)
OTHER = {
    "d320_n144_r3": 72,           # K2 BN 64 (6.2), radius mask (2.2)
    "d384_n100": 136,             # K2 BN 128, 256-row blocks straddling images of 100 rows (4.9, 2.1)
    "d64_n1600": 16,              # four key passes (3.0, 3.2 per pass)
    "d128_n256_r2_self": 72,      # masked logits with attend_self (3.3, 3.3)
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(OTHER))
def test_other_paths_per_tile_and_slices(name):
    B = OTHER[name]
    m, img, S, n = FO._model(name, "bf16", batch=B)
    guard(m.dim, m.levels, n, B)
    img, S = img.to(DEV), S.to(DEV)
    with torch.no_grad():
        for start in (S, None):
            full = m(img, iters=4, levels=start, return_all=True)
            k = max(1, 256 // n)                   # slices of at most 256 rows, as the oracle's batches
            ref = _sliced(lambda a, b: m(img[a:b], iters=4, levels=None if start is None else start[a:b],
                                         return_all=True), B, k, dim=1)
            _equal(full, ref, (name, start is None))
    del full, ref
    _per_tile_step(m, img, S.cpu(), n, name)


# ----------------------------------------------------------------------------- GPU: per-image steps
PER_IMAGE = {
    # whole 256-row blocks frozen early
    "configs[1]": (CFG1, 32, lambda B: [(3 * b) % 13 for b in range(B)]),
    # n = 64: four images per 256-row block, blocks partly frozen
    "configs[1]_n64": ((512, 6, 112, 14), 72, lambda B: [0, 2] * 4 + [(5 * b + 1) % 12 + 1 for b in range(B - 8)]),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(PER_IMAGE))
def test_per_image_steps_equal_scalar_slices(name):
    """forward(iters=<vector>, return_all=True): every image equals its slice's scalar-iters call, slab for slab (slab t
    of image b = S_min(t, steps[b]))."""
    (dim, L, isz, p), B, steps_fn = PER_IMAGE[name]
    steps = steps_fn(B)
    m = _glom(dim, L, isz, p)
    img, S, n = _inputs(m, B, seed=14)
    guard(dim, L, n, B)
    T = max(steps)
    with torch.no_grad():
        full = m(img, iters=torch.tensor(steps), levels=S, return_all=True)
        for b, k in enumerate(steps):
            one = m(img[b:b + 1], iters=k, levels=S[b:b + 1], return_all=True)
            _equal(full[:k + 1, b:b + 1], one, (name, b, k))
            for t in range(k + 1, T + 1):
                _equal(full[t, b], one[k, 0], (name, b, k, t))


# ----------------------------------------------------------------------------- GPU: settle and the queue
def _contracting(dim, L, isz, p, seed=0):
    """test_settle's contracting model: both second MLP layers zeroed."""
    torch.manual_seed(seed)
    m = G.Glom(dim=dim, levels=L, image_size=isz, patch_size=p).to(DEV).eval()
    with torch.no_grad():
        m.bottom_up.net[3].weight.zero_()
        m.top_down.net[3].weight.zero_()
    return m


def _spread(m, img, max_iters):
    """A start near the fixed point with noise spread over six decades across the images, and test_settle's tol."""
    import test_settle as ST
    N = img.shape[0]
    base = m(img, iters=60)
    noise = torch.randn(base.shape, generator=torch.Generator().manual_seed(2)).to(DEV)
    eps = torch.tensor([10.0 ** (1 - 6 * b / (N - 1)) for b in range(N)], device=DEV).view(N, 1, 1, 1)
    start = (base + eps * noise * base.abs().mean()).contiguous()
    del base, noise
    r = ST._change(m(img, iters=max_iters, levels=start, return_all=True))
    return start, ST._pick_tol(r)


@pytest.mark.gpu
def test_configs1_settle_and_queue():
    """settle at B = 32 gives per image the bits and steps of forward(iters=steps[b]) on its slice; settle_queue(N = 96,
    slots = 32) equals settle on all 96 images."""
    m = _contracting(*CFG1)
    imgs = torch.randn(96, 3, 224, 224, generator=torch.Generator().manual_seed(1)).to(DEV)
    guard(512, 6, 256, 32)
    with torch.no_grad():
        img = imgs[:32]
        start, tol = _spread(m, img, 12)
        levels, steps = m.settle(img, tol, max_iters=12, levels=start)
        sh = steps.cpu().numpy()
        assert len(np.unique(sh)) >= 3, sh
        for b, k in enumerate(sh):
            _equal(levels[b:b + 1], m(img[b:b + 1], iters=int(k), levels=start[b:b + 1]), ("settle", b, int(k)))
        del levels, start
        start, tol = _spread(m, imgs, 12)
        want, want_steps = m.settle(imgs, tol, max_iters=12, levels=start)
        got, got_steps = m.settle_queue(imgs, tol, max_iters=12, levels=start, slots=32)
        assert len(np.unique(want_steps.cpu().numpy())) >= 3
        _equal(got_steps, want_steps, "queue steps")
        _equal(got, want, "queue levels")


@pytest.mark.gpu
def test_settle_and_queue_beyond_256_images():
    """The settle / queue kernels loop over images and slots in strides of 256 threads: settle at B = 300 equals its
    100-image slices, settle_queue(N = 700, slots = 300) equals settle on all 700 (d 64, L 2, n 16)."""
    m = _contracting(64, 2, 16, 4)
    imgs = torch.randn(700, 3, 16, 16, generator=torch.Generator().manual_seed(1)).to(DEV)
    with torch.no_grad():
        img = imgs[:300]
        start, tol = _spread(m, img, 12)
        levels, steps = m.settle(img, tol, max_iters=12, levels=start)
        assert len(np.unique(steps.cpu().numpy())) >= 3
        parts = [m.settle(img[a:a + 100], tol, max_iters=12, levels=start[a:a + 100]) for a in range(0, 300, 100)]
        _equal(steps, torch.cat([p[1] for p in parts]), "settle steps")
        _equal(levels, torch.cat([p[0] for p in parts]), "settle levels")
        start, tol = _spread(m, imgs, 12)
        want, want_steps = m.settle(imgs, tol, max_iters=12, levels=start)
        got, got_steps = m.settle_queue(imgs, tol, max_iters=12, levels=start, slots=300)
        assert len(np.unique(want_steps.cpu().numpy())) >= 3
        _equal(got_steps, want_steps, "queue steps")
        _equal(got, want, "queue levels")


# ----------------------------------------------------------------------------- GPU: the tokeniser at B = 128
@pytest.mark.gpu
def test_tokeniser_configs1_dims_batch128():
    """256 tiles of 256 rows x 256 columns: per tile against bf16(patchify(img)) @ bf16(W)^T + b in float64, and equal
    to its 16-image slices bit for bit."""
    m = _glom(*CFG1)
    B = 128
    img = torch.randn(B, 3, 224, 224, generator=torch.Generator().manual_seed(5)).to(DEV)
    guard(512, 6, 256, B, kernels=("tok",))
    with torch.no_grad():
        tok = m.tokens(img)
        _equal(tok, _sliced(lambda a, b: m.tokens(img[a:b]), B, 16), "tokens")
    w = m.image_to_tokens[1].weight.detach().cpu().double()
    bias = m.image_to_tokens[1].bias.detach().cpu().double()
    ref = OT.bf16(OT.patchify(img.cpu().double(), 14)) @ OT.bf16(w).T + bias
    errs = FO.errors({"tokens": tok.cpu()}, {"tokens": ref}, (B, 256, 1, 512))
    FO._report("configs[1] B=128", "tokeniser", errs)
    FO.check(errs, FO.TOL["tok"], "tokeniser B=128")


# ----------------------------------------------------------------------------- backward: the batch-summed bound
BATCH_SUMMED = ("pos_emb.weight", "image_to_tokens.1.weight", "image_to_tokens.1.bias", "init_levels") + BO.NAMES


# the default (atomic) backward against the deterministic slices: 2^-8, one bf16 rounding (relative) of every element.
# Only a small fraction of its bf16 cotangent shadows round the other way, so it stays well inside
DEFAULT_TOL = (2.0 ** -8, 2.0 ** -8)


def batch_sum_tol(T, R):
    """(rel, abs) bound on a batch-summed gradient of T reverse steps over R rows against the float64 sum of its
    slices' gradients.  Both sides multiply the same bf16 operands (the per-row cotangents are bit-identical), so they
    differ only in the fp32 summation over the T * R row-steps.  A sum of N fp32 terms of random sign is off by about
    u sqrt(N) of its size; 16x that covers the tensor cores' truncating accumulation and the partial sums' order."""
    b = 16 * U32 * math.sqrt(T * R)
    return b, b


# ----------------------------------------------------------------------------- CPU: the bound catches faults
# d 32, L 2, n 16, B 512, T 12: the rows (8192) and steps of bench.py's training step at configs[1], so each fault
# removes the same fraction of the row-steps as it would there
FAULT_SHAPE = dict(d=32, L=2, isz=16, p=4, B=512, T=12)


def _fault_case():
    f = FAULT_SHAPE
    P = {k: torch.from_numpy(v).double() for k, v in O.synth_params(f["d"], f["L"], f["isz"], f["p"], seed=7).items()}
    n = (f["isz"] // f["p"]) ** 2
    g = torch.Generator().manual_seed(7)
    tok = torch.randn(f["B"], n, f["d"], generator=g, dtype=torch.float64)
    pos = P["pos_emb.weight"][:n].clone()
    s = torch.randn(f["B"], n, f["L"], f["d"], generator=g, dtype=torch.float64)
    states = [s]
    for _ in range(f["T"]):
        states.append(OT.column_step(states[-1], tok, pos, P, None, False))
    states = torch.stack(states)
    cot = torch.randn(states.shape, generator=g, dtype=torch.float64)
    return P, tok, pos, states, cot


def _step_grads(P, tok, pos, states, cot, t0, imgs=slice(None)):
    """Step t0's own contribution to the batch-summed gradients, from images `imgs` only."""
    G_next = OT.grads_at_states(P, tok[imgs], pos, states[t0 + 1:, imgs], cot[t0 + 1:, imgs], return_all=True)
    return OT.grads_at_states(P, tok[imgs], pos, states[t0:t0 + 2, imgs], G_next["d_state0"], return_all=False)


def _summed(g):
    """grads_at_states output -> the batch-summed keys the GPU test compares (tokens stand in for the tokeniser)."""
    out = {k: g[k] for k in BO.NAMES}
    out["pos_emb.weight"] = g["d_pos"]
    out["init_levels"] = g["d_state0"].sum((0, 1))
    return out


@pytest.mark.parametrize("fault", ["dw_tile_dropped", "dw_kblock_skipped", "batch_problem_dropped"])
def test_batch_sum_bound_catches_faults(fault):
    """Each fault of the multi-tile schedule misses batch_sum_tol at configs[1]'s T and rows by >= 3x in both metrics:
    a BW_DW tile (one group's weight tile at one step) dropped; one 64-row k-block of BW_DW skipped at one step; one
    BW_BATCH problem (image 22 = z >= 132 at L 6, one level) left out at one step."""
    f = FAULT_SHAPE
    P, tok, pos, states, cot = _fault_case()
    n, L, t0 = tok.shape[1], f["L"], f["T"] // 2
    good = OT.grads_at_states(P, tok, pos, states, cot, return_all=True)
    bad = {k: v.clone() for k, v in good.items()}
    if fault == "dw_tile_dropped":
        step = _step_grads(P, tok, pos, states, cot, t0)
        w = bad["bottom_up.net.3.weight"].view(L, f["d"], 4 * f["d"])
        w[1] -= step["bottom_up.net.3.weight"].view(L, f["d"], 4 * f["d"])[1]
    elif fault == "dw_kblock_skipped":
        step = _step_grads(P, tok, pos, states, cot, t0, slice(100, 104))          # 64 rows
        for k in BO.NAMES:
            if k.endswith("weight"):
                bad[k] -= step[k]
    else:
        b0, l0 = 22, 1
        G_next = OT.grads_at_states(P, tok[b0:b0 + 1], pos, states[t0 + 1:, b0:b0 + 1], cot[t0 + 1:, b0:b0 + 1],
                                    return_all=True)["d_state0"]
        s = states[t0, b0:b0 + 1].clone().requires_grad_(True)
        cons = OT._consensus(s, False, None)[:, :, l0] / (3.0 if l0 == L - 1 else 4.0)
        (dcons,) = torch.autograd.grad(cons, s, G_next[:, :, l0])
        # the missing dL/dS_t0 of that image propagates through steps t0-1 .. 0
        lost = OT.grads_at_states(P, tok[b0:b0 + 1], pos, states[:t0 + 1, b0:b0 + 1], dcons, return_all=False)
        for k in BO.NAMES:
            bad[k] -= lost[k]
        bad["d_pos"] -= lost["d_pos"]
        bad["d_state0"][b0:b0 + 1] -= lost["d_state0"]
    tol = batch_sum_tol(12, 32 * 256)
    rel, ab = BO.worst(BO.errors(_summed(bad), _summed(good), L, n))
    print(f"[production] fault {fault}: rel {rel:.3e} abs {ab:.3e} vs bound {tol[0]:.2e}")
    assert rel >= 3 * tol[0] and ab >= 3 * tol[1], (fault, rel, ab, tol)


def test_fault_step_decomposition_is_exact():
    """The fault helpers' per-step contributions add up to the T-step gradients (so the faults remove what they say)."""
    f = FAULT_SHAPE
    P, tok, pos, states, cot = _fault_case()
    sl = slice(0, 8)
    states, cot, tok = states[:4, sl], cot[:4, sl], tok[sl]
    good = OT.grads_at_states(P, tok, pos, states, cot, return_all=True)
    total = {k: sum(_step_grads(P, tok, pos, states, cot, t)[k] for t in range(3)) for k in BO.NAMES}
    for k in BO.NAMES:
        assert torch.allclose(total[k], good[k], rtol=1e-10, atol=1e-12 * float(good[k].abs().max())), k


# ----------------------------------------------------------------------------- GPU: backward, bench.py's training step
def _bwd_model(B):
    m, img, S, n, g = BO._model("tc_config2_dims", "bf16", batch=B)
    return m, img, S, n, g


@pytest.mark.gpu
def test_configs1_backward_one_step_per_tile():
    """One reverse step at B = 32 (BW_BATCH: 192 problems): every gradient per block against grads_at_states (tc) and
    step_backward_bf16 (tc_emu)."""
    m, img, S, n, g = _bwd_model(32)
    guard(512, 6, n, 32, kernels=("bwd",))
    cot = torch.randn(S.shape, generator=g)
    out, got = BO._engine_run(m, img, S, 1, False, cot)
    ref, P, tok = BO._reference(m, img, torch.stack([S, out.cpu()]), cot, return_all=False)
    errs = BO.errors(got, ref, m.levels, n)
    BO._report("configs[1] B=32", "one step vs grads_at_states", errs)
    BO.check(errs, BO.TOL["tc"], "B=32 tc")
    emu = OT.step_backward_bf16(P, tok, P["pos_emb.weight"][:n], S, cot, attend_self=m.attention.attend_self,
                                mask=None, attn_tc=True)
    emu["d_state0"] = emu.pop("d_state")
    ref = BO._map_reference(emu, {k: v.numpy() for k, v in P.items()}, img, m.patch_size, n, True)
    errs = BO.errors(got, ref, m.levels, n)
    BO._report("configs[1] B=32", "one step vs step_backward_bf16", errs)
    BO.check(errs, BO.TOL["tc_emu"], "B=32 tc_emu")


def _grads(m, img, S, iters, loss_fn):
    """loss_fn(out) through the engine -> gradients by name (d_img, d_levels when S is given, parameters)."""
    for q in m.parameters():
        q.grad = None
    x = img.to(DEV).requires_grad_(True)
    lv = None if S is None else S.to(DEV).requires_grad_(True)
    loss_fn(m(x, iters=iters, levels=lv, return_all=True)).backward()
    torch.cuda.synchronize()
    got = {"d_img": x.grad}
    if lv is not None:
        got["d_levels"] = lv.grad
    got.update({k: q.grad.clone() for k, q in m.named_parameters() if q.grad is not None})
    return got


CASES_T12 = {
    # bench.py's training step: iters=12, return_all, loss mean(levels[7, :, :, -1] ** 2) at B = 32, from init_levels
    "bench_loss": (None, False),
    # a random cotangent on every slab, from a carried state
    "random_cot": (None, True),
    # the same with a per-image step vector: odd images stop after 0 .. 11 steps (whole 256-row blocks frozen), even
    # images run all 12, so every two-image slice returns the same 13 slabs as the full batch
    "random_cot_steps": ([12 if b % 2 == 0 else (b // 2) % 12 for b in range(32)], True),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES_T12))
def test_configs1_backward_T12_slices(case):
    """T = 12 at B = 32 under torch.use_deterministic_algorithms: d_img and d_levels equal 16 two-image runs bit for
    bit, and the batch-summed gradients are within batch_sum_tol of the float64 sum of the slices' gradients.

    The default (atomic) mode reduces the top-down groups' dx into dL/dS in no fixed order, so its per-row cotangents
    differ from the slices' in the last fp32 bits; where such a value sits near a bf16 rounding boundary its bf16
    shadow (gsb) moves by a whole bf16 ulp, and over 12 reverse steps the batch sums move by ~1e-3 (1.4e-3 observed
    with a random cotangent).  That mode is held to DEFAULT_TOL, the relative size of one bf16 rounding, for the batch
    sums and for d_img / d_levels against the deterministic slices."""
    from test_deterministic_backward import deterministic
    steps, carried = CASES_T12[case]
    B, T = 32, 12
    m, img, S, n, g = _bwd_model(B)
    guard(512, 6, n, B, kernels=("k1", "k2", "k3", "bwd"))
    iters = T if steps is None else torch.tensor(steps)
    start = S if carried else None
    scale = 1.0 / (B * n * m.dim)                  # bench's mean at B = 32; the same constant in every slice
    if case == "bench_loss":
        cot = None
    else:
        cot = torch.randn((T + 1,) + tuple(S.shape), generator=torch.Generator(device=DEV).manual_seed(3), device=DEV)

    def loss(lo, hi):
        if cot is None:
            return lambda out: out[7, :, :, -1].square().sum() * scale
        return lambda out: (out * cot[:, lo:hi]).sum()

    def run(lo, hi):
        it = iters if steps is None else iters[lo:hi]
        return _grads(m, img[lo:hi], None if start is None else start[lo:hi], it, loss(lo, hi))
    with deterministic():
        full = run(0, B)
        parts = [run(lo, lo + 2) for lo in range(0, B, 2)]
    per_image = [k for k in ("d_img", "d_levels") if k in full]
    for k in per_image:
        _equal(full[k], torch.cat([p[k] for p in parts]), (case, k))
    summed = {k: sum(p[k].double().cpu() for p in parts) for k in full if k not in per_image}
    assert set(summed) == set(BATCH_SUMMED) - ({"init_levels"} if carried else set()), set(summed)
    tol = batch_sum_tol(T, B * n)
    errs = BO.errors(full, summed, m.levels, n)
    BO._report(f"configs[1] B=32 T=12 {case}", f"deterministic batch sums vs slices (bound {tol[0]:.2e})", errs)
    BO.check(errs, tol, (case, "deterministic"))
    with deterministic(False):
        plain = run(0, B)
    errs = BO.errors(plain, summed, m.levels, n)
    BO._report(f"configs[1] B=32 T=12 {case}", f"default batch sums vs slices (bound {DEFAULT_TOL[0]:.2e})", errs)
    BO.check(errs, DEFAULT_TOL, (case, "default"))
    errs = BO.errors(plain, {k: full[k] for k in per_image}, m.levels, n)
    BO._report(f"configs[1] B=32 T=12 {case}", f"default per-image gradients vs slices (bound {DEFAULT_TOL[0]:.2e})",
               errs)
    BO.check(errs, DEFAULT_TOL, (case, "default per image"))
