"""Images are independent: NaN, inf and overflowing values in one image never reach another image's results.

Every batching feature leans on this (DESIGN.md, "Where S_k stays"): settle_queue / settle_video refill a slot's rows
with the next image, settle skips frozen 256-row blocks, the image-independent path copies image 0's rows out, and the
production-batch tests require batch = slices bit for bit.  With finite data a kernel that reads another image's value
and multiplies it by zero (a padded row of a shared 128 / 256-row tile, a masked key, a stale row of a refilled slot, a
frozen row of a partially frozen block) still gives the same bits, so the suites above cannot see it.  Here one image
gets a poison, an ordinary float input the public API accepts:

* values: NaN, +inf, -inf, 3e38 (finite; its squares and its first-layer products overflow) and 1e20 (only the fp32
  squared norms overflow);
* places: one element of the carried levels at level 0, at the top level and at a middle level, the image's first and
  last patch (the rows next to the neighbouring image inside a shared tile), one pixel of its first and of its last
  patch, and in backward tests the cotangent;
* images: image 0 (the representative image of the image-independent path), an image in the middle of a shared
  256-row block, the last image (ragged tail).

The clean and the poisoned input run with everything else equal, and every output of every other image must have the
same bits (compared through integer views, since NaN != NaN): levels, return_all slabs, steps, settle's q and frozen
flags, last_adjoint, per-image gradients, island fields.  For a NaN poison the poisoned image itself is checked step by
step against ``column_step`` in float64 at the engine's own states: the set of (patch, level) with a non-finite element
must match.  With a radius mask, ``column_step`` (the reference's masked_fill + P V) still spreads a masked key's NaN to
every query through 0 x NaN, so there the engine's set must contain the mask-exact set (patches with an unmasked
non-finite key or a non-finite input of their own) and lie inside column_step's.

A stopped image (per-image step count 0) must add nothing to the shared gradients whatever its levels hold
(``test_stopped_image_adds_nothing``).  The CPU self-tests run the same harness over small fake kernels with the faults
it exists to catch, and show that a finite perturbation misses each of them.
"""
import itertools
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import test_backward_oracle as BO
import test_deterministic_backward as DB
import test_forward_oracle as FO
import test_image_independent_levels as II
import test_settle as TS
import test_settle_oracle as TSO
from oracle import glom_oracle as O
from oracle import glom_oracle_torch as OT
from oracle import islands_oracle as IO

DEV = "cuda:0"
VALUES = {"nan": float("nan"), "+inf": float("inf"), "-inf": float("-inf"), "3e38": 3.0e38, "1e20": 1e20}
LEVEL_PLACES = ("level0", "top_level", "mid_level", "first_patch", "last_patch")
PIXEL_PLACES = ("first_pixel", "last_pixel")
PLACES = LEVEL_PLACES + PIXEL_PLACES
STATE_DIMS = ("image", "row", "level", "col")
SLAB_DIMS = ("slab",) + STATE_DIMS
FINITE = 0.25             # the finite perturbation of the self-tests: a well-scaled value that changes nothing else


# ----------------------------------------------------------------------------- the comparator
def bits(t):
    """t as integers of its width, so that NaN payloads compare like any other bits and +0 != -0."""
    t = t.detach().contiguous()
    if t.dtype == torch.float32:
        return t.view(torch.int32)
    if t.dtype == torch.float64:
        return t.view(torch.int64)
    return t


def differing(a, b, mode="bits"):
    """Element mask where a and b differ: by bits, or by value ("value": NaN equals NaN, +0 equals -0)."""
    assert a.shape == b.shape, (tuple(a.shape), tuple(b.shape))
    if mode == "bits":
        return bits(a) != bits(b)
    return ~((a == b) | (torch.isnan(a) & torch.isnan(b)))


def first_difference(a, b, what, *, skip=(), image_dim=0, dims=None, mode="bits"):
    """None if a and b agree outside images `skip` (indices along `image_dim`), else a message naming the first
    differing element by its dimension names, e.g. (image 2, row 17, level 1, col 5)."""
    diff = differing(a, b, mode)
    if skip:
        diff.index_fill_(image_dim, torch.tensor(sorted(skip), device=diff.device), False)
    if not diff.any():
        return None
    idx = diff.nonzero()[0].tolist()
    names = dims or tuple(f"dim{i}" for i in range(a.dim()))
    where = ", ".join(f"{k} {i}" for k, i in zip(names, idx))
    return (f"{what}: {int(diff.sum())} of {diff.numel()} elements differ, first at ({where}): "
            f"{a[tuple(idx)].item()!r} vs {b[tuple(idx)].item()!r}")


def assert_same(a, b, what, **kw):
    msg = first_difference(a, b, what, **kw)
    assert msg is None, msg


def nonfinite(x):
    """(..., d) -> (...) bool: the row holds a non-finite element."""
    return ~torch.isfinite(x).all(-1)


# ----------------------------------------------------------------------------- poisons
def poison(img, S, b, place, value):
    """Copies of img (B, 3, H, W) and S (B, n, L, d) or None with `value` at `place` of image b."""
    img = img.clone()
    S = None if S is None else S.clone()
    if place == "first_pixel":
        img[b, 1, 0, 0] = value
    elif place == "last_pixel":
        img[b, 2, -1, -1] = value
    else:
        _, n, L, d = S.shape
        row, level = {"level0": (n // 2, 0), "top_level": (n // 3, L - 1), "mid_level": ((2 * n) // 3, L // 2),
                      "first_patch": (0, L // 2), "last_patch": (n - 1, 0)}[place]
        S[b, row, level, d // 3] = value
    return img, S


def pick_images(n, B):
    """Image 0, an image in the middle of a shared 256-row block (not the first or the last if one exists), the last."""
    mid = B // 2
    for r in range(128, n * B, 256):
        if 0 < r // n < B - 1:
            mid = r // n
            break
    return sorted({0, mid, B - 1})


def cases(images, values=VALUES, places=PLACES):
    """Every (value, place), each at one of `images` in turn: each image meets every value and most places."""
    return [(v, p, images[i % len(images)]) for i, (v, p) in enumerate(itertools.product(values, places))]


# ----------------------------------------------------------------------------- the poisoned image itself
def mask_exact(S, tok, mask):
    """(B, n, L) bool: rows of the next step that take a non-finite value from their own inputs (the row, its
    bottom-up input S[l-1] or the token, its top-down input S[l+1]) or from an unmasked non-finite key of their level."""
    nf = nonfinite(S)                                                     # (B, n, L)
    own = nf.clone()
    own[:, :, 0] |= nonfinite(tok)
    own[:, :, 1:] |= nf[:, :, :-1]
    own[:, :, :-1] |= nf[:, :, 1:]
    seen = torch.ones(S.shape[1], S.shape[1], dtype=torch.float64) if mask is None else (~mask).double()
    keys = torch.einsum("ij,bjl->bil", seen, nf.double()) > 0
    return own | keys


def check_nan_steps(states, tok, params, pos, mask, attend_self, what):
    """One image's slabs (T+1, 1, n, L, d): at each step the engine's non-finite (patch, level) set against
    column_step's in float64 at the engine's own state: equal without a mask, between the mask-exact set and
    column_step's with one.  -> the number of extra patches (engine beyond mask-exact) per step."""
    extras = []
    P = {k: OT._f64(params[k]) for k in OT.MLP_KEYS}
    for t in range(states.shape[0] - 1):
        S = states[t].cpu()
        ref = nonfinite(OT.column_step(OT._f64(S), OT._f64(tok), OT._f64(pos), P, mask, attend_self))
        got = nonfinite(states[t + 1].cpu())
        exact = mask_exact(S, tok.cpu(), mask)
        missing = exact & ~got
        assert not missing.any(), f"{what} step {t + 1}: engine finite at (patch, level) {missing[0].nonzero()[:4].tolist()}"
        beyond = got & ~ref
        assert not beyond.any(), f"{what} step {t + 1}: non-finite beyond float64 at {beyond[0].nonzero()[:4].tolist()}"
        if mask is None:
            assert torch.equal(ref, exact), what
        extras.append(int((got & ~exact).sum()))
    if any(extras):
        print(f"[isolation] {what}: patches non-finite beyond the mask-exact set per step {extras}")
    return extras


def _params(m):
    return {k: q.detach().cpu() for k, q in m.named_parameters()}


# ----------------------------------------------------------------------------- CPU: the harness catches each fault
def _x(B=4, n=6, d=5, seed=0):
    return torch.randn(B, n, d, generator=torch.Generator().manual_seed(seed))


def _others_fail(kernel, x, b, value):
    """The isolation check over a fake kernel: its outputs with x[b] poisoned at one element, against clean."""
    bad = x.clone()
    bad[b, 1, 2] = value
    return first_difference(kernel(x), kernel(bad), "fake", skip=(b,), dims=("image", "row", "col"))


def _neighbour_read(x):
    return torch.tanh(x) + 0 * x.roll(-1, 0)


def _fmax_swallow(x):
    return torch.fmax(x, torch.zeros_like(x)).cumsum(1)


def _fmax_exact(x):
    return torch.maximum(x, torch.zeros_like(x)).cumsum(1)


def _settle_steps(x, batch_wide, tol=1e-3, iters=30):
    """Per-image contraction x_k = x_{k-1} / 2 stopped when max |x_k - x_{k-1}| <= tol; `batch_wide`: one decision for
    every image, from the maximum change over images."""
    B = x.shape[0]
    steps = torch.full((B,), iters)
    done = torch.zeros(B, dtype=torch.bool)
    cur = x.double()
    for k in range(1, iters + 1):
        nxt = cur / 2
        ch = (nxt - cur).abs().amax((1, 2))
        stop = (ch <= tol).expand(B) if not batch_wide else (ch.max() <= tol).expand(B)
        stop = stop & ~done
        steps[stop] = k
        done |= stop
        cur = nxt
    return steps


def _shared_grad(x, live, masked):
    """A shared weight gradient over images: frozen images (live = 0) scaled by zero, or dropped (`masked`)."""
    per = x * torch.linspace(0.5, 1.5, x.shape[-1])
    if masked:
        return torch.where(live[:, None, None], per, torch.zeros_like(per)).sum(0)
    return (live[:, None, None].double() * per).sum(0)


def _stopped_fail(x, b, value, masked):
    """The stopped-image check: image b frozen, its values poisoned; the shared sum must be finite and equal (as
    values) to the same call with x[b] = 0."""
    live = torch.ones(x.shape[0], dtype=torch.bool)
    live[b] = False
    bad, zero = x.clone(), x.clone()
    bad[b, 1, 2] = value
    zero[b] = 0
    got = _shared_grad(bad, live, masked)
    if not torch.isfinite(got).all():
        return "shared gradient not finite"
    return first_difference(got, _shared_grad(zero, live, masked), "shared", mode="value")


@pytest.mark.parametrize("value", ["nan", "+inf", "-inf"])
def test_harness_catches_a_masked_read_of_the_neighbour(value):
    x = _x()
    assert _others_fail(_neighbour_read, x, 2, VALUES[value]) is not None
    assert _others_fail(_neighbour_read, x, 2, FINITE) is None
    assert _others_fail(torch.tanh, x, 2, VALUES[value]) is None


def test_harness_catches_a_nan_swallowing_fmax():
    x = _x()
    x[1, 1, 2] = float("nan")
    got, ref = nonfinite(_fmax_swallow(x)), nonfinite(_fmax_exact(x.double()))
    assert not torch.equal(got, ref)
    x[1, 1, 2] = FINITE
    assert torch.equal(nonfinite(_fmax_swallow(x)), nonfinite(_fmax_exact(x.double())))


def test_harness_catches_a_batch_wide_stopping_decision():
    x = _x() * torch.tensor([1.0, 10.0, 100.0, 1000.0])[:, None, None]
    clean = _settle_steps(x, batch_wide=False)
    assert len(set(clean.tolist())) == 4

    def run(batch_wide, value):
        bad = x.clone()
        bad[0, 1, 2] = value
        return first_difference(_settle_steps(x, batch_wide), _settle_steps(bad, batch_wide), "steps", skip=(0,))
    assert run(True, float("nan")) is not None
    assert run(True, FINITE) is None
    assert run(False, float("nan")) is None


@pytest.mark.parametrize("value", ["nan", "+inf", "3e38"])
def test_harness_catches_a_frozen_row_multiplied_by_zero(value):
    x = _x()
    v = VALUES[value] if value != "3e38" else float("inf")      # the overflow of a 3e38 product, in float64 here
    assert _stopped_fail(x, 1, v, masked=False) is not None
    assert _stopped_fail(x, 1, FINITE, masked=False) is None
    assert _stopped_fail(x, 1, v, masked=True) is None


def test_comparator_bits_and_values():
    a = torch.tensor([float("nan"), 0.0, 1.0])
    assert not torch.equal(a, a.clone())                                    # why bit views are needed
    assert first_difference(a, a.clone(), "nan payload") is None
    other = a.clone()
    other.view(torch.int32)[0] = 0x7fc00001                                  # a NaN with another payload
    assert first_difference(a, other, "payload") is not None
    assert first_difference(a, other, "payload", mode="value") is None
    neg = a.clone()
    neg[1] = -0.0
    assert "(dim0 1)" in first_difference(a, neg, "signed zero")
    assert first_difference(a, neg, "signed zero", mode="value") is None
    assert first_difference(a, neg, "skipped", skip=(1,)) is None


def test_pick_images_finds_a_block_middle_and_the_tail():
    assert pick_images(64, 8) == [0, 2, 7]            # rows 128..191: images 0-3 share the first 256-row block
    assert pick_images(144, 5) == [0, 2, 4]           # row 384: images 1-3 share rows 256..511
    assert pick_images(256, 3) == [0, 1, 2]
    assert pick_images(784, 2) == [0, 1]


def test_mask_exact_set():
    S = torch.zeros(1, 4, 3, 2)
    tok = torch.zeros(1, 4, 2)
    S[0, 1, 1, 0] = float("nan")
    mask = torch.ones(4, 4, dtype=torch.bool)
    mask[torch.arange(4), torch.arange(4)] = False
    mask[0, 1] = False                                                     # patch 0 sees patch 1's key
    got = mask_exact(S, tok, mask)[0]
    want = torch.zeros(4, 3, dtype=torch.bool)
    want[1, :] = True                                                      # its own row and both neighbour levels
    want[0, 1] = True                                                      # patch 0 through the unmasked key
    assert torch.equal(got, want)
    assert mask_exact(S, tok, None)[0][:, 1].all()


def test_grads_at_states_drops_a_stopped_image():
    """A frozen image with NaN and inf in its states adds nothing: every gradient equals the same call without the
    image, and its d_state0 is its cotangent."""
    P, tok, pos, S, g = BO._small(B=3)
    T = 2
    states = torch.stack([S, S + 0.1, S + 0.2])
    states[:, 1, 2, 1, 3] = float("nan")
    states[:, 1, 0, 0, 0] = float("inf")
    cot = torch.randn(S.shape, generator=g, dtype=torch.float64)
    got = OT.grads_at_states(P, tok, pos, states, cot, return_all=False, steps=[T, 0, T])
    keep = [0, 2]
    ref = OT.grads_at_states(P, tok[keep], pos, states[:, keep], cot[keep], return_all=False)
    for k, v in ref.items():
        assert torch.isfinite(got[k]).all(), k
        w = got[k][keep] if k in ("d_tokens", "d_state0") else got[k]
        assert torch.equal(w, v), k
    assert torch.equal(got["d_state0"][1], cot[1]) and not got["d_tokens"][1].any()


# ----------------------------------------------------------------------------- GPU: forward
FORWARD = {      # name: (test_forward_oracle.SHAPES entry, precision, batch)
    "n64": ("cons_d128_n64", "bf16", 8),
    "n144_B5_r3": ("d320_n144_r3", "bf16", 5),
    "n100": ("d384_n100", "bf16", 3),
    "n784_r6.5_self": ("d128_n784_r6.5_self", "bf16", 2),
    "self_only": ("d192_n144_self_only", "bf16", 3),
    "nonsquare": ("d256_nonsquare", "bf16", 3),
    "config2_dims": ("config2_dims", "bf16", 3),
    "fp32_n36": ("d192_n36", "fp32", 3),
    "fp32_n256_r2_self": ("d128_n256_r2_self", "fp32", 3),
}


def _forward_outputs(m, img, S):
    return {"T3_all": m(img, iters=3, levels=S, return_all=True), "T1": m(img, iters=1, levels=S)}


def _check_forward_outputs(clean, got, b, what):
    for k in clean:
        assert_same(clean[k], got[k], f"{what} {k}", skip=(b,), image_dim=1 if k.endswith("all") else 0,
                    dims=SLAB_DIMS if k.endswith("all") else STATE_DIMS)


def _nan_parity(m, img, states, b, n, what):
    with torch.no_grad():
        tok = m.tokens(img)[b:b + 1].cpu()
    P = _params(m)
    return check_nan_steps(states[:, b:b + 1], tok, P, P["pos_emb.weight"][:n], FO._mask(m, n),
                           m.attention.attend_self, what)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(FORWARD))
def test_forward(name):
    """forward T = 1 and T = 3 (return_all) from carried levels: every poison at every place, the other images' bits
    unchanged; the NaN image against column_step at a level and at a pixel."""
    shape, precision, B = FORWARD[name]
    m, img, S, n = FO._model(shape, precision, batch=B)
    img, S = img.to(DEV), S.to(DEV)
    images = pick_images(n, B)
    with torch.no_grad():
        clean = _forward_outputs(m, img, S)
        for value, place, b in cases(images):
            pi, pS = poison(img, S, b, place, VALUES[value])
            got = _forward_outputs(m, pi, pS)
            _check_forward_outputs(clean, got, b, f"{name} {value} at {place} of image {b}")
            if value == "nan" and place in ("mid_level", "first_pixel", "last_patch"):
                _nan_parity(m, pi, got["T3_all"], b, n, f"{name} NaN at {place} of image {b}")


@pytest.mark.gpu
def test_resume_chain():
    """The second call of a resume chain (eval, levels = the tensor the first call returned) poisoned through its pixels:
    the other images' bits equal those of the same call without resume, and of the clean resumed call."""
    m, img, S, n = FO._model("cons_d128_n64", "bf16", batch=8)
    m.eval()
    img = img.to(DEV)
    img2 = img.flip(0).contiguous()
    with torch.no_grad():
        clean = m(img2, iters=2, levels=m(img, iters=2))
        for value, place, b in cases(pick_images(n, 8), places=PIXEL_PLACES):
            p2, _ = poison(img2, None, b, place, VALUES[value])
            first = m(img, iters=2)
            resumed = m(p2, iters=2, levels=first)
            plain = m(p2, iters=2, levels=first.clone())
            what = f"resume {value} at {place} of image {b}"
            assert_same(plain, resumed, what, skip=(b,), dims=STATE_DIMS)
            assert_same(clean, resumed, what, skip=(b,), dims=STATE_DIMS)


def _check_init_path(m, img, images, iters, values, parity):
    with torch.no_grad():
        clean = m(img, iters=iters, return_all=True)
        for value, place, b in cases(images, values, PIXEL_PLACES):
            pi, _ = poison(img, None, b, place, VALUES[value])
            got = m(pi, iters=iters, return_all=True)
            what = f"init_levels {value} at {place} of image {b}"
            assert_same(clean, got, what, skip=(b,), image_dim=1, dims=SLAB_DIMS)
            if parity and value == "nan":
                _nan_parity(m, pi, got, b, got.shape[2], what)
            del got


@pytest.mark.gpu
@pytest.mark.parametrize("name,images", [("L2_n64", [0]), ("n576", [0, 1]), ("n784", [0, 7])])
def test_image_independent_path(name, images):
    """forward from init_levels, where image 0's rows (at n = 576 images 0-1, at n = 784 images 0-7) stand in for every
    image's image-independent levels: pixel poison in those representative images."""
    dim, L, isz, p, B = II.SHAPES[name]
    m = II._glom(dim, L, isz, p)
    _check_init_path(m, II._images(m, B, 3), images, 2 * L, VALUES, parity=name == "L2_n64")


@pytest.mark.gpu
def test_image_independent_level_fill_configs1_batch32():
    """configs[1] at batch 32 with return_all: level_fill_kernel copies the representative image's levels out."""
    m = II._glom(512, 6, 224, 14)
    _check_init_path(m, II._images(m, 32, 1), [0], 7, {k: VALUES[k] for k in ("nan", "+inf", "3e38")}, parity=False)


@pytest.mark.gpu
@pytest.mark.parametrize("name,B", [("d320_n144_r3", 5), ("cons_d128_n64", 8)])
def test_per_image_iters(name, B):
    """forward(iters=<vector>, return_all=True) with the poisoned image at 0 steps (its slabs are its poisoned start) and
    at the maximum."""
    m, img, S, n = FO._model(name, "bf16", batch=B)
    img, S = img.to(DEV), S.to(DEV)
    base = torch.tensor([1 + (b % 3) for b in range(B)])
    for value, place, b in cases(pick_images(n, B)):
        for k in (0, 4):
            vec = base.clone()
            vec[b] = k
            pi, pS = poison(img, S, b, place, VALUES[value])
            with torch.no_grad():
                clean = m(img, iters=vec, levels=S, return_all=True)
                got = m(pi, iters=vec, levels=pS, return_all=True)
            what = f"iters {vec.tolist()} {value} at {place} of image {b}"
            assert_same(clean, got, what, skip=(b,), image_dim=1, dims=SLAB_DIMS)
            if k == 0:
                assert_same(got[:, b], pS[b].expand_as(got[:, b]), what + ": a stopped image is its start")


# ----------------------------------------------------------------------------- GPU: settle, queue, video
def _settle_start(shape):
    m, img = TS._model(shape, contracting=True)
    B = img.shape[0]
    with torch.no_grad():
        base = m(img, iters=60)
        noise = torch.randn(base.shape, generator=torch.Generator().manual_seed(2)).to(DEV)
        eps = torch.tensor([10.0 ** (1 - 6 * b / max(B - 1, 1)) for b in range(B)], device=DEV).view(B, 1, 1, 1)
        start = (base + eps * noise * base.abs().mean()).contiguous()
        r = TS._change(m(img, iters=TS.MAX_ITERS, levels=start, return_all=True))
    tol = float(np.quantile(r[np.isfinite(r) & (r > 0)], 0.5))
    return m, img, start, tol


@pytest.mark.gpu
@pytest.mark.parametrize("shape", sorted(TS.SHAPES))
def test_settle(shape):
    """settle: the poisoned image never stops (NaN), the others' levels, steps, per-level q and frozen flags keep their
    bits."""
    m, img, start, tol = _settle_start(shape)
    B, n = img.shape[0], start.shape[1]
    out, steps, _, q, frozen, _ = TSO._settle(m, img, tol, TS.MAX_ITERS, start)
    for value, place, b in cases(pick_images(n, B)):
        pi, pS = poison(img, start, b, place, VALUES[value])
        out_p, steps_p, _, q_p, frozen_p, _ = TSO._settle(m, pi, tol, TS.MAX_ITERS, pS)
        what = f"settle {shape} {value} at {place} of image {b}"
        assert_same(out, out_p, what, skip=(b,), dims=STATE_DIMS)
        assert_same(steps, steps_p, what + " steps", skip=(b,))
        assert_same(q, q_p, what + " q", skip=(b,))
        assert_same(frozen, frozen_p, what + " frozen", skip=(b,))
        if value == "nan":
            assert steps_p[b] == TS.MAX_ITERS and frozen_p[b] == 0, what


@pytest.mark.gpu
@pytest.mark.parametrize("slots", [1, 3, 8])
def test_settle_queue(slots):
    """settle_queue with the poisoned image first in the queue: with one slot every later image runs in the rows the
    poisoned one used."""
    m, img, start, tol = _settle_start("n64_four_images_per_block")
    with torch.no_grad():
        out, steps = m.settle_queue(img, tol, TS.MAX_ITERS, levels=start, slots=slots)
        for value, place in itertools.product(VALUES, ("mid_level", "last_patch", "first_pixel")):
            pi, pS = poison(img, start, 0, place, VALUES[value])
            out_p, steps_p = m.settle_queue(pi, tol, TS.MAX_ITERS, levels=pS, slots=slots)
            what = f"queue slots={slots} {value} at {place}"
            assert_same(out, out_p, what, skip=(0,), dims=STATE_DIMS)
            assert_same(steps, steps_p, what + " steps", skip=(0,))
            if value == "nan":
                assert int(steps_p[0]) == TS.MAX_ITERS, what


@pytest.mark.gpu
@pytest.mark.parametrize("slots", [1, 2])
def test_settle_video(slots):
    """settle_video over 3 streams of 4 frames: a poisoned stream (its start levels or its first frame), and one
    poisoned frame in the middle of a stream; the other streams keep their levels and steps."""
    m, img, start, tol = _settle_start("n64_four_images_per_block")
    S, Fr = 3, 4
    g = torch.Generator().manual_seed(5)
    frames = (img[:S, None] + 0.05 * torch.randn(S, Fr, *img.shape[1:], generator=g).to(DEV)).contiguous()
    lv = start[:S].contiguous()
    with torch.no_grad():
        out, steps = m.settle_video(frames, tol, TS.MAX_ITERS, levels=lv, slots=slots)
        for value, (s, how) in itertools.product(("nan", "+inf", "3e38"),
                                                 [(0, "levels"), (2, "frame0"), (1, "frame2")]):
            pf, pl = frames.clone(), lv.clone()
            if how == "levels":
                pl[s, 5, 1, 7] = VALUES[value]
            else:
                pf[s, int(how[-1]), 0, 3, 3] = VALUES[value]
            out_p, steps_p = m.settle_video(pf, tol, TS.MAX_ITERS, levels=pl, slots=slots)
            what = f"video slots={slots} {value} in stream {s} {how}"
            assert_same(out, out_p, what, skip=(s,), dims=("stream", "frame") + STATE_DIMS[1:])
            assert_same(steps, steps_p, what + " steps", skip=(s,))
            if how == "frame2":
                assert_same(out[s, :2], out_p[s, :2], what + ": frames before the poisoned one")


# ----------------------------------------------------------------------------- GPU: tokeniser
@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("dim,p,hw,B", [(64, 4, (12, 12), 3), (128, 14, (70, 98), 9), (512, 14, (224, 224), 2)])
def test_tokeniser(dim, p, hw, B, precision):
    """The other images and the other patches of the poisoned image keep their bits; a NaN patch row is non-finite
    exactly where float64 Linear's is."""
    import glom_pytorch_b200 as G
    isz = max(hw)
    params = O.synth_params(dim, 2, isz, p, seed=4)
    m = G.Glom(dim=dim, levels=2, image_size=isz, patch_size=p, precision=precision)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=False)
    m = m.to(DEV)
    img = torch.randn((B, 3) + hw, generator=torch.Generator().manual_seed(5)).to(DEV)
    n = (hw[0] // p) * (hw[1] // p)
    w, bias = (torch.from_numpy(params[k]).double() for k in ("image_to_tokens.1.weight", "image_to_tokens.1.bias"))
    with torch.no_grad():
        clean = m.tokens(img)
        for value, place, b in cases(pick_images(n, B), places=PIXEL_PLACES):
            pi, _ = poison(img, None, b, place, VALUES[value])
            got = m.tokens(pi)
            patch = 0 if place == "first_pixel" else n - 1
            what = f"tokens {precision} {value} at {place} of image {b}"
            assert_same(clean, got, what, skip=(b,), dims=("image", "patch", "col"))
            rest = torch.arange(n, device=DEV) != patch
            assert_same(clean[b, rest], got[b, rest], what + ": other patches")
            if value == "nan":
                ref = F.linear(OT.patchify(pi[b:b + 1].double().cpu(), p), w, bias)[0, patch]
                assert torch.equal(~torch.isfinite(ref), ~torch.isfinite(got[b, patch].cpu())), what


# ----------------------------------------------------------------------------- GPU: backward
BACKWARD = {"tc_d256_n144_B5": 5, "mixed_d256_n100": 3, "simt_d192_n144_mask_self": 3}


def _grads(m, img, S, iters, return_all, cot, det=True):
    with DB.deterministic(det):
        _, got = BO._engine_run(m, img, S, iters, return_all, cot)
    return got


def _check_image_grads(clean, got, b, what):
    assert_same(clean["d_img"], got["d_img"], what + " d_img", skip=(b,), dims=("image", "chan", "y", "x"))
    assert_same(clean["d_levels"], got["d_levels"], what + " d_levels", skip=(b,), dims=STATE_DIMS)


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 3])
@pytest.mark.parametrize("name", sorted(BACKWARD))
def test_backward(name, T):
    """return_all backward under the deterministic flag: a poisoned forward input with a finite cotangent, and a poisoned
    cotangent with a finite input; the other images' d_img and d_levels keep their bits.  In atomic mode they stay
    finite and within 2^-8 of the deterministic result."""
    m, img, S, n, g = BO._model(name, "bf16", batch=BACKWARD[name])
    B = S.shape[0]
    cot = torch.randn((T + 1,) + tuple(S.shape), generator=g)
    clean = _grads(m, img, S, T, True, cot)
    images = pick_images(n, B)
    runs = [(v, p, b, "input") for v, p, b in cases(images, ("nan", "+inf", "3e38"), ("mid_level", "last_patch", "first_pixel"))]
    runs += [(v, "cot", images[i % len(images)], "cot") for i, v in enumerate(("nan", "+inf", "-inf"))]
    for value, place, b, kind in runs:
        what = f"{name} T={T} {value} at {place} of image {b}"
        if kind == "input":
            pi, pS = poison(img, S, b, place, VALUES[value])
            pc = cot
        else:
            pi, pS, pc = img, S, cot.clone()
            pc[T, b, n - 1, 0, 3] = VALUES[value]
        got = _grads(m, pi, pS, T, True, pc)
        _check_image_grads(clean, got, b, what)
        if value == "nan" and kind == "input":
            atomic = _grads(m, pi, pS, T, True, pc, det=False)
            keep = [i for i in range(B) if i != b]
            for k in ("d_img", "d_levels"):
                a, d = atomic[k][keep], got[k][keep]
                assert torch.isfinite(a).all(), (what, k)
                err = float((a - d).abs().max() / d.abs().max())
                assert err <= 2.0 ** -8, (what, k, err)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [True, "implicit"])
def test_settle_differentiable(mode):
    """settle(differentiable=True / "implicit") under the deterministic flag: the other images' d_img, steps and, for
    the implicit backward, K_b and q of last_adjoint keep their bits."""
    m, img, start, tol = _settle_start("n64_four_images_per_block")
    B = img.shape[0]
    cot = torch.randn(start.shape, generator=torch.Generator().manual_seed(3)).to(DEV)

    def run(x, lv):
        x = x.clone().requires_grad_(True)
        with DB.deterministic():
            out, steps = m.settle(x, tol, TS.MAX_ITERS, levels=lv, differentiable=mode)
            (out * cot).sum().backward()
        torch.cuda.synchronize()
        adj = m.last_adjoint if mode == "implicit" else None
        return x.grad, steps, adj
    d_img, steps, adj = run(img, start)
    for value, place, b in cases(pick_images(start.shape[1], B), ("nan", "+inf", "3e38"), ("mid_level", "first_pixel")):
        pi, pS = poison(img, start, b, place, VALUES[value])
        g_p, steps_p, adj_p = run(pi, pS)
        what = f"settle {mode} {value} at {place} of image {b}"
        assert_same(d_img, g_p, what + " d_img", skip=(b,), dims=("image", "chan", "y", "x"))
        assert_same(steps, steps_p, what + " steps", skip=(b,))
        if adj is not None:
            assert_same(adj[0], adj_p[0], what + " K_b", skip=(b,))
            assert_same(adj[1], adj_p[1], what + " q", skip=(b,), dims=("image", "level"))


# ----------------------------------------------------------------------------- GPU: islands, parse tree, tracks
def _island_states(T=3, B=3, side=8, L=3, d=64):
    g = torch.Generator().manual_seed(9)
    S = torch.randn(T, B, side * side, L, d, generator=g)
    S[..., :d // 2] += 3.0                                                # neighbours mostly agree: real islands
    return S.to(DEV)


def _fields(t):
    return {k: v for k, v in t._asdict().items() if v is not None}


@pytest.mark.gpu
@pytest.mark.parametrize("value", list(VALUES))
def test_islands_parse_tree_tracks(value):
    """A poisoned slab (t = 1, b = 1): islands leave the other slabs, and the poisoned slab's other levels, unchanged in
    every field; parse_tree(embeddings=True) the other slabs; track_islands the other sequences.  NaN cosine maps are
    non-finite where float64 edges are."""
    import glom_pytorch_b200 as G
    S = _island_states()
    T, B, n, L, d = S.shape
    bad = S.clone()
    bad[1, 1, 27, 1, 5] = VALUES[value]
    flat, flat_bad = S.view(T * B, n, L, d), bad.view(T * B, n, L, d)
    slab = 1 * B + 1
    isl, isl_p = _fields(G.islands(flat)), _fields(G.islands(flat_bad))
    for k in isl:
        assert_same(isl[k], isl_p[k], f"islands {value} {k}", skip=(slab,))
        if isl[k].dim() == 3:                                               # (slabs, L, n): the other levels
            keep = [l for l in range(L) if l != 1]
            assert_same(isl[k][slab, keep], isl_p[k][slab, keep], f"islands {value} {k} other levels")
    if value == "nan":
        cr, cd = IO.edges(flat_bad[slab].cpu().numpy(), 8, 8)
        assert np.array_equal(~np.isfinite(cr), ~torch.isfinite(isl_p["cos_right"][slab]).cpu().numpy())
        assert np.array_equal(~np.isfinite(cd), ~torch.isfinite(isl_p["cos_down"][slab]).cpu().numpy())
    tree, tree_p = _fields(G.parse_tree(flat, embeddings=True)), _fields(G.parse_tree(flat_bad, embeddings=True))
    for k in tree:
        assert_same(tree[k], tree_p[k], f"parse_tree {value} {k}", skip=(slab,))
    tr, tr_p = _fields(G.track_islands(S)), _fields(G.track_islands(bad))
    for k in tr:
        assert_same(tr[k], tr_p[k], f"track_islands {value} {k}", skip=(1,), image_dim=1)


# ----------------------------------------------------------------------------- GPU: SM-count targets
@pytest.mark.gpu
@pytest.mark.parametrize("sms", [2, 3])
def test_sm_count_targets(sms):
    """One pair of CTAs walks tiles across every image boundary: forward, settle and the deterministic backward."""
    m, img, S, n = FO._model("cons_d128_n64", "bf16", batch=8)
    img, S = img.to(DEV), S.to(DEV)
    bm, bimg, bS, bn, g = BO._model("tc_d256_n144_B5", "bf16")
    cot = torch.randn((2,) + tuple(bS.shape), generator=g)
    sm, simg, sstart, tol = _settle_start("n64_four_images_per_block")
    with II._sm_target(sms):
        with torch.no_grad():
            clean = _forward_outputs(m, img, S)
            s_clean = TSO._settle(sm, simg, tol, TS.MAX_ITERS, sstart)
        b_clean = _grads(bm, bimg, bS, 1, True, cot)
        for value, b in itertools.product(("nan", "+inf", "3e38"), (2, 3)):
            with torch.no_grad():
                pi, pS = poison(img, S, b, "first_patch", VALUES[value])
                _check_forward_outputs(clean, _forward_outputs(m, pi, pS), b, f"target {sms} {value} image {b}")
                pi, pS = poison(simg, sstart, b, "last_patch", VALUES[value])
                s_got = TSO._settle(sm, pi, tol, TS.MAX_ITERS, pS)
                for k, (x, y) in enumerate(zip(s_clean, s_got)):
                    if k in (0, 1, 3, 4):                                   # levels, steps, q, frozen
                        assert_same(x, y, f"target {sms} settle {value} image {b} output {k}", skip=(b,))
            pi, pS = poison(bimg, bS, b, "last_patch", VALUES[value])
            _check_image_grads(b_clean, _grads(bm, pi, pS, 1, True, cot), b, f"target {sms} backward {value} image {b}")


# ----------------------------------------------------------------------------- GPU: a stopped image adds nothing
STOPPED = {      # name: (test_backward_oracle.SHAPES entry or a spec of its own, batch, the images tried)
    "n100_mixed": ("mixed_d256_n100", 3, (1, 2)),
    "n144_B5": ("tc_d256_n144_B5", 5, (0, 4)),
    "n256_aligned": ((256, 3, 64, 4, None, 3, {}, "tc", 1.0), 3, (0, 1)),
    "simt_n144": ("simt_d192_n144_mask_self", 3, (0, 1)),
}
SHARED = BO.NAMES + ("pos_emb.weight", "image_to_tokens.1.weight", "image_to_tokens.1.bias")


def _stopped_model(name):
    spec, B, _ = STOPPED[name]
    if isinstance(spec, str):
        return BO._model(spec, "bf16", batch=B)
    key = f"_isolation_{name}"
    BO.SHAPES.setdefault(key, spec)
    try:
        return BO._model(key, "bf16", batch=B)
    finally:
        BO.SHAPES.pop(key, None)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(STOPPED))
def test_stopped_image_adds_nothing(name):
    """forward(iters=vec, levels=...) with image b at 0 steps and NaN, +inf or 3e38 in its levels: its d_levels is its
    cotangent, its d_img zero, every shared gradient finite, equal (as values, deterministic flag) to the same call with
    its levels zeroed, and within the backward oracle's bounds of grads_at_states without it."""
    m, img, S, n, g = _stopped_model(name)
    B = S.shape[0]
    cot = torch.randn(S.shape, generator=g)
    path = BO.TOL["simt" if STOPPED[name][0] == "simt_d192_n144_mask_self" else "tc"]
    for b, value in itertools.product(STOPPED[name][2], ("nan", "+inf", "3e38")):
        vec = torch.full((B,), 2)
        vec[b] = 0
        bad, zero = S.clone(), S.clone()
        bad[b, n // 2, 0, 3] = VALUES[value]
        bad[b, n - 1, m.levels - 1, 7] = VALUES[value]
        zero[b] = 0
        what = f"{name} image {b} stopped with {value}"
        got = _grads(m, img, bad, vec, False, cot)
        bad_keys = [k for k in SHARED if not torch.isfinite(got[k]).all()]
        print(f"[isolation] {what}: non-finite shared gradients {bad_keys}, "
              f"d_levels[b] == cot[b]: {torch.equal(got['d_levels'][b].cpu(), cot[b])}, "
              f"max |d_img[b]| {float(got['d_img'][b].abs().max())}")
        assert torch.equal(got["d_levels"][b].cpu(), cot[b]), what + ": d_levels is not the cotangent"
        assert not got["d_img"][b].any(), what + ": d_img is not zero"
        assert not bad_keys, (what, bad_keys)
        ref_zero = _grads(m, img, zero, vec, False, cot)
        for k in SHARED:
            assert_same(ref_zero[k], got[k], f"{what} {k} vs levels zeroed", mode="value")
        with torch.no_grad():
            states = m(img.to(DEV), iters=vec, levels=bad.to(DEV), return_all=True).cpu()
        ref, _, _ = BO._reference(m, img, states, cot, return_all=False, steps=vec.tolist())
        errs = BO.errors({k: got[k] for k in SHARED}, {k: ref[k] for k in SHARED}, m.levels, n)
        BO._report(name, what + " shared vs grads_at_states", errs)
        BO.check(errs, path, what)


@pytest.mark.gpu
def test_fp32_engine_has_no_stopped_images():
    """The fp32 engine rejects per-image step counts, so no image of it is ever frozen in a backward."""
    m, img, S, n = FO._model("d192_n36", "fp32")
    with pytest.raises(RuntimeError, match="per-image iters need precision='bf16'"):
        m(img.to(DEV), iters=[0, 1, 2], levels=S.to(DEV))
