"""Training through Glom.settle: settle(return_all=True) and settle(differentiable=True).

CPU: argument errors of glom_b200_settle_all (reported before any device query), its workspace size, and the Python errors
of the differentiable path.
GPU: on the contracting model and start of test_settle.py at its four shapes, settle(return_all=True) gives the states of
forward(iters=k, return_all=True) for each image's k, with the slabs after k equal to slab k, and the differentiable call
gives the same values and steps.  Gradients of the one-pass settle match the two-pass recipe (settle under no_grad, then
forward(iters=steps)) on the tensor-core backward (dim 256, with the attention-backward skip) and the CUDA-core one
(dim 128), with every image stopped at least 3 steps before max_iters, so that the last reverse steps have every image
frozen; from a carried start the images stop at >= 3 distinct steps.  A backward workspace filled with NaN bytes gives the same gradients as a zeroed one, so no skipped store is
read.  An in-place edit of the returned steps does not change the gradients."""
import ctypes

import numpy as np
import pytest
import torch

import glom_pytorch_b200 as G
from glom_pytorch_b200 import _native

DEV = "cuda:0"
FAKE = 0x100000          # 1024-aligned, never dereferenced: every error below is reported before any device work


# ---------------------------------------------------------------------------------------------------------- CPU
def _cfg(precision="bf16", dim=128, levels=3, n=64):
    return _native.make_cfg(dim, levels, n, False, 0, 0, precision)


def _settle_all_rc(cfg, max_iters=4, tol=0.1, steps=FAKE):
    lib = _native.load()
    p = ctypes.c_void_p(FAKE)
    return lib.glom_b200_settle_all(ctypes.byref(cfg), p, p, p, None, p, p, 2, max_iters, ctypes.c_float(tol), steps, p,
                                    1 << 30, None)


@pytest.mark.parametrize("what,kw,msg", [
    ("fp32 engine", dict(cfg=_cfg("fp32")), "bf16"),
    ("max_iters = 0", dict(max_iters=0), "max_iters"),
    ("NaN tol", dict(tol=float("nan")), "NaN"),
    ("NULL steps_out", dict(steps=None), "steps_out"),
    ("misaligned steps_out", dict(steps=FAKE + 2), "aligned"),
])
def test_settle_all_argument_errors(what, kw, msg):
    cfg = kw.pop("cfg", _cfg())
    assert _settle_all_rc(cfg, **kw) == -1, what
    assert msg in _native.load().glom_b200_last_error().decode(), what


@pytest.mark.parametrize("dim,levels,n,batch,iters", [(512, 6, 256, 32, 12), (128, 3, 64, 8, 6), (64, 2, 625, 3, 6)])
def test_settle_all_workspace_is_the_return_all_forward_steps_workspace(dim, levels, n, batch, iters):
    cfg = _cfg(dim=dim, levels=levels, n=n)
    assert _native.settle_all_workspace_bytes(cfg, batch, iters) == \
        _native.forward_steps_workspace_bytes(cfg, batch, iters, True)
    with pytest.raises(_native.GlomB200Error, match="max_iters"):
        _native.settle_all_workspace_bytes(cfg, batch, 0)


def test_differentiable_settle_rejects_fp32_model_and_cpu_input():
    m = G.Glom(dim=64, levels=3, image_size=28, patch_size=7, precision="fp32")
    with pytest.raises(RuntimeError, match="bf16"):
        m.settle(torch.randn(1, 3, 28, 28), 1e-3, differentiable=True)
    m = G.Glom(dim=64, levels=3, image_size=28, patch_size=7)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m.settle(torch.randn(1, 3, 28, 28), 1e-3, differentiable=True)


# ---------------------------------------------------------------------------------------------------------- GPU
# (dim, levels, image_size, patch_size, consensus_self, local_consensus_radius, batch), as in test_settle.py
SHAPES = {
    "n256_whole_blocks": (256, 3, 64, 4, False, 0, 6),
    "n64_four_images_per_block": (128, 3, 32, 4, False, 0, 8),
    "n625_key_passes": (64, 2, 100, 4, False, 0, 4),
    "n144_radius_self": (192, 3, 48, 4, True, 3, 5),
}
# the two backward paths of test_per_image_iters.py
GRAD_SHAPES = {
    "tensor_core_bwd_n144": (256, 3, 48, 4, False, 0, 5),        # rows = 720: not a multiple of 128 / 256
    "cuda_core_bwd_n64": (128, 3, 32, 4, False, 0, 8),
}
MAX_ITERS = 12


def _change(states):
    """r[b, k - 1] = max_l sqrt(sum_i |S_k - S_{k-1}|^2 / sum_i |S_k|^2) in float64, states (T+1, B, n, L, d)."""
    s = states.double()
    num = ((s[1:] - s[:-1]) ** 2).sum(dim=(2, 4))
    den = (s[1:] ** 2).sum(dim=(2, 4))
    q = torch.where((num == 0) & (den == 0), torch.zeros_like(num), (num / den).sqrt())
    return q.amax(dim=2).T.cpu().numpy()                              # (B, T)


def _first_stop(r, tol):
    hit = r <= tol
    return np.where(hit.any(axis=1), hit.argmax(axis=1) + 1, r.shape[1]).astype(np.int32)


def _setup(spec, w2_scale):
    """Model whose second MLP layers are scaled by w2_scale (0: the contracting model of test_settle.py), and a start
    near its fixed point with noise over six decades, one size per image."""
    dim, L, isz, p, attend_self, radius, B = spec
    torch.manual_seed(0)
    m = G.Glom(dim=dim, levels=L, image_size=isz, patch_size=p, consensus_self=attend_self,
               local_consensus_radius=radius).to(DEV).eval()
    with torch.no_grad():
        m.bottom_up.net[3].weight.mul_(w2_scale)
        m.top_down.net[3].weight.mul_(w2_scale)
    img = torch.randn(B, 3, isz, isz, generator=torch.Generator().manual_seed(1)).to(DEV)
    with torch.no_grad():
        base = m(img, iters=60)
        noise = torch.randn(base.shape, generator=torch.Generator().manual_seed(2)).to(DEV)
        eps = torch.tensor([10.0 ** (1 - 6 * b / (B - 1)) for b in range(B)], device=DEV).view(B, 1, 1, 1)
        start = (base + eps * noise * base.abs().mean()).contiguous()
        r = _change(m(img, iters=MAX_ITERS, levels=start, return_all=True))
    return m, img, start, r


def _tol_spread(r):
    """A tol (1e-3 relative away from every r) at which the images stop at >= 3 distinct steps, one never stops."""
    vals = np.unique(r[np.isfinite(r) & (r > 0)])
    best = None
    for a, b in zip(vals[:-1], vals[1:]):
        if b <= a * 1.01:
            continue
        tol = float(np.sqrt(a * b))
        score = len(np.unique(_first_stop(r, tol)))
        if (r > tol).all(axis=1).any() and (best is None or score > best[0]):
            best = (score, tol)
    assert best is not None and best[0] >= 3, f"the contracting model does not spread the images: {r}"
    return best[1]


def _tol_all_stop_early(r, min_distinct):
    """Among the tols between two well separated r values at which every image stops by step MAX_ITERS - 3 (so that the
    backward ends with >= 3 reverse steps in which every image is frozen), the one with the most distinct steps."""
    vals = np.unique(r[np.isfinite(r) & (r > 0)])
    best = None
    for a, b in zip(vals[:-1], vals[1:]):
        if b <= a * 1.01:
            continue
        tol = float(np.sqrt(a * b))
        if (r[:, :MAX_ITERS - 3] <= tol).any(axis=1).all():
            score = len(np.unique(_first_stop(r, tol)))
            if best is None or score > best[0]:
                best = (score, tol)
    assert best is not None and best[0] >= min_distinct, (best, r)
    return best[1]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_settle_return_all_values(shape):
    m, img, start, r = _setup(SHAPES[shape], 0.0)
    tol = _tol_spread(r)
    with torch.no_grad():
        levels, steps = m.settle(img, tol, max_iters=MAX_ITERS, levels=start)
        states, steps_all = m.settle(img, tol, max_iters=MAX_ITERS, levels=start, return_all=True)
    assert states.shape == (MAX_ITERS + 1,) + tuple(start.shape)
    assert torch.equal(steps_all, steps)
    assert torch.equal(states[MAX_ITERS], levels)
    steps_h = steps.cpu().numpy()
    assert len(np.unique(steps_h)) >= 3
    with torch.no_grad():
        for k in np.unique(steps_h):
            k = int(k)
            ref = m(img, iters=k, levels=start, return_all=True)
            for b in np.nonzero(steps_h == k)[0]:
                for t in range(MAX_ITERS + 1):
                    assert torch.equal(states[t, b], ref[min(t, k), b]), (shape, int(b), k, t)
    # with parameters that require grad, the differentiable call computes the same values and steps
    for return_all, want in ((False, levels), (True, states)):
        got, got_steps = m.settle(img, tol, max_iters=MAX_ITERS, levels=start, return_all=return_all, differentiable=True)
        assert got.requires_grad and not got_steps.requires_grad
        assert torch.equal(got.detach(), want) and torch.equal(got_steps, steps), return_all


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _grads(m, img, lv, loss_fn):
    m.zero_grad(set_to_none=True)
    img = img.clone().requires_grad_(True)
    lv = None if lv is None else lv.clone().requires_grad_(True)
    loss_fn(img, lv).backward()
    g = {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}
    g["img"] = img.grad.clone()
    if lv is not None:
        g["levels"] = lv.grad.clone()
    return g


def _assert_close(got, want, what):
    assert set(got) == set(want), what
    for k in want:
        assert torch.isfinite(got[k]).all(), (what, k)
        assert _rel(got[k], want[k]) <= 1e-5, (what, k, _rel(got[k], want[k]))


def _grad_setup(shape, carried=True):
    """The model with small second MLP layers (every weight gets a gradient), the start (None: init_levels), a tol at
    which every image stops by step MAX_ITERS - 3, and the steps settle picks.  From a carried start the images stop at
    >= 3 distinct steps.  From init_levels every image starts at the same state and may stop at the same step: that case
    checks the all-frozen tail against the scalar two-pass path."""
    m, img, start, r = _setup(GRAD_SHAPES[shape], 0.05)
    lv = start if carried else None
    if not carried:
        with torch.no_grad():
            r = _change(m(img, iters=MAX_ITERS, return_all=True))
    tol = _tol_all_stop_early(r, 3 if carried else 1)
    with torch.no_grad():
        _, steps = m.settle(img, tol, max_iters=MAX_ITERS, levels=lv)
    assert int(steps.max()) <= MAX_ITERS - 3, (steps, tol)
    m.train()
    return m, img, lv, tol, steps


def _one_pass_loss(m, tol, lv_cot, return_all):
    def loss(x, s):
        out, _ = m.settle(x, tol, max_iters=MAX_ITERS, levels=s, return_all=return_all, differentiable=True)
        return (out * lv_cot).sum()
    return loss


@pytest.mark.gpu
@pytest.mark.parametrize("return_all", [False, True])
@pytest.mark.parametrize("carried", [False, True])
@pytest.mark.parametrize("shape", sorted(GRAD_SHAPES))
def test_settle_gradients_match_the_two_pass_recipe(shape, carried, return_all):
    m, img, lv, tol, steps = _grad_setup(shape, carried)
    T = int(steps.max())
    shape_s = (img.shape[0], (img.shape[2] // m.patch_size) ** 2, m.levels, m.dim)
    cot = torch.randn(((MAX_ITERS + 1,) if return_all else ()) + shape_s,
                      generator=torch.Generator().manual_seed(5)).to(DEV)

    got = _grads(m, img, lv, _one_pass_loss(m, tol, cot, return_all))

    def two_pass(x, s):
        out = m(x, iters=steps, levels=s, return_all=return_all)
        if not return_all:
            return (out * cot).sum()
        # slabs T.. of the one-pass states all equal slab T: fold their cotangents into slab T, in the order of the
        # backward's pass-through steps (from the last slab down), so that both backwards see the same fp32 cotangent
        fold = cot[MAX_ITERS]
        for t in range(MAX_ITERS - 1, T - 1, -1):
            fold = fold + cot[t]
        return (out * torch.cat([cot[:T], fold[None]])).sum()

    want = _grads(m, img, lv, two_pass)
    _assert_close(got, want, (shape, carried, return_all))


@pytest.mark.gpu
@pytest.mark.parametrize("shape", sorted(GRAD_SHAPES))
def test_skipped_backward_stores_are_never_read(shape):
    m, img, start, tol, _ = _grad_setup(shape)
    cot = torch.randn((MAX_ITERS + 1,) + tuple(start.shape), generator=torch.Generator().manual_seed(5)).to(DEV)
    loss = _one_pass_loss(m, tol, cot, True)
    _grads(m, img, start, loss)                              # creates the cached backward workspace
    dev = torch.device(DEV)
    key = ("_bwd_workspace", dev.index, torch.cuda.current_stream(dev).cuda_stream)

    def filled(byte):
        def run(x, s):
            out = loss(x, s)
            m._scratch[key].fill_(byte)                      # between the forward and the backward
            return out
        return run

    nan_ws = _grads(m, img, start, filled(0xFF))             # 0xFFFF... is a NaN in fp32 and bf16
    zero_ws = _grads(m, img, start, filled(0))
    _assert_close(nan_ws, zero_ws, shape)


@pytest.mark.gpu
def test_backward_keeps_its_own_steps():
    m, img, start, tol, _ = _grad_setup("tensor_core_bwd_n144")
    cot = torch.randn(tuple(start.shape), generator=torch.Generator().manual_seed(5)).to(DEV)

    def edited(x, s):
        out, steps = m.settle(x, tol, max_iters=MAX_ITERS, levels=s, differentiable=True)
        steps.zero_()
        return (out * cot).sum()

    _assert_close(_grads(m, img, start, edited), _grads(m, img, start, _one_pass_loss(m, tol, cot, False)), "steps.zero_()")
