"""Glom.settle: per-image early stopping on the GPU.

CPU: argument errors of the C ABI (reached before any device query) and the workspace sizes.
GPU: on a contracting model (both second MLP layers zeroed, so the bottom-up / top-down outputs are constants) started
from a fixed point plus noise of sizes spread over decades, each image stops at its own step; every settled image is
bit-identical to forward(iters=steps[b]) on the same batch, and `steps` is the first k whose change criterion, recomputed
in float64 from forward(return_all=True), is <= tol.  Covered: n = 256 (whole 256-row blocks skipped), n = 64 (four images
per block: row masking inside running tiles), n = 625 (consensus key passes; blocks and bands straddle images) and
n = 144 with a radius mask and consensus_self.  Also the tol = -1 / tol = inf limits with random weights, determinism,
the following forward's ordinary prologue, and the errors."""
import ctypes

import numpy as np
import pytest
import torch

import glom_pytorch_b200 as G
from glom_pytorch_b200 import _native

DEV = "cuda:0"


# ---------------------------------------------------------------------------------------------------------- CPU
def _cfg(precision="bf16", dim=128, levels=3, n=64):
    return _native.make_cfg(dim, levels, n, False, 0, 0, precision)


def _settle_rc(cfg, max_iters=4, tol=0.1, steps=0x1000):
    lib = _native.load()
    ws = ctypes.c_void_p(0x100000)
    return lib.glom_b200_settle(ctypes.byref(cfg), ws, ws, ws, None, ws, ws, 2, max_iters, ctypes.c_float(tol),
                                steps, ws, 1 << 30, None)


@pytest.mark.parametrize("what,kw,msg", [
    ("fp32 engine", dict(cfg=_cfg("fp32")), "bf16"),
    ("max_iters = 0", dict(max_iters=0), "max_iters"),
    ("NaN tol", dict(tol=float("nan")), "NaN"),
    ("NULL steps_out", dict(steps=None), "steps_out"),
])
def test_settle_argument_errors(what, kw, msg):
    cfg = kw.pop("cfg", _cfg())
    rc = _settle_rc(cfg, **kw)
    assert rc == -1, what
    assert msg in _native.load().glom_b200_last_error().decode(), what


def test_settle_workspace_bytes_errors():
    with pytest.raises(_native.GlomB200Error, match="bf16"):
        _native.settle_workspace_bytes(_cfg("fp32"), 2, 4)
    with pytest.raises(_native.GlomB200Error, match="max_iters"):
        _native.settle_workspace_bytes(_cfg(), 2, 0)


@pytest.mark.parametrize("dim,levels,n,batch,iters,fwd_bytes", [
    (512, 6, 256, 32, 12, 716177408),       # configs[1]
    (128, 3, 64, 8, 6, 5267456),
    (64, 2, 625, 3, 6, 7123968),
])
def test_settle_workspace_extends_the_forward_workspace(dim, levels, n, batch, iters, fwd_bytes):
    cfg = _cfg(dim=dim, levels=levels, n=n)
    fwd = _native.workspace_bytes(cfg, batch, iters, False)
    assert fwd == fwd_bytes                  # the forward layout is unchanged by settle
    st = _native.settle_workspace_bytes(cfg, batch, iters)
    nparts = dim // (64 if dim % 128 == 0 else 32)
    # + squared-change partials (rows, L, nparts) + per-image / per-block flags
    assert st >= fwd + batch * n * levels * nparts * 4 + batch * 4
    assert st % 1024 == 0


def test_settle_rejects_fp32_model_and_cpu_input():
    m = G.Glom(dim=64, levels=3, image_size=28, patch_size=7, precision="fp32")
    with torch.no_grad(), pytest.raises(RuntimeError, match="bf16"):
        m.settle(torch.randn(1, 3, 28, 28), 1e-3)
    m = G.Glom(dim=64, levels=3, image_size=28, patch_size=7)
    with torch.no_grad(), pytest.raises(RuntimeError, match="no CPU fallback"):
        m.settle(torch.randn(1, 3, 28, 28), 1e-3)


# ---------------------------------------------------------------------------------------------------------- GPU
# (dim, levels, image_size, patch_size, consensus_self, local_consensus_radius, batch)
SHAPES = {
    "n256_whole_blocks": (256, 3, 64, 4, False, 0, 6),
    "n64_four_images_per_block": (128, 3, 32, 4, False, 0, 8),
    "n625_key_passes": (64, 2, 100, 4, False, 0, 4),
    "n144_radius_self": (192, 3, 48, 4, True, 3, 5),
}
MAX_ITERS = 12


def _model(shape, contracting):
    dim, L, isz, p, attend_self, radius, B = SHAPES[shape]
    torch.manual_seed(0)
    m = G.Glom(dim=dim, levels=L, image_size=isz, patch_size=p, consensus_self=attend_self,
               local_consensus_radius=radius).to(DEV).eval()
    if contracting:
        with torch.no_grad():
            m.bottom_up.net[3].weight.zero_()
            m.top_down.net[3].weight.zero_()
    g = torch.Generator().manual_seed(1)
    img = torch.randn(B, 3, isz, isz, generator=g).to(DEV)
    return m, img


def _change(states):
    """r[b, k - 1] = max_l sqrt(sum_i |S_k - S_{k-1}|^2 / sum_i |S_k|^2) in float64, states (T+1, B, n, L, d)."""
    s = states.double()
    num = ((s[1:] - s[:-1]) ** 2).sum(dim=(2, 4))                     # (T, B, L)
    den = (s[1:] ** 2).sum(dim=(2, 4))
    q = torch.where((num == 0) & (den == 0), torch.zeros_like(num), (num / den).sqrt())
    return q.amax(dim=2).T.cpu().numpy()                              # (B, T)


def _first_stop(r, tol):
    hit = r <= tol
    return np.where(hit.any(axis=1), hit.argmax(axis=1) + 1, r.shape[1]).astype(np.int32)


def _pick_tol(r):
    """The tol that spreads the images over the most distinct stopping steps while one image never stops, at least
    1e-3 (relative) away from every r."""
    vals = np.unique(r[np.isfinite(r) & (r > 0)])
    best = None
    for a, b in zip(vals[:-1], vals[1:]):
        if b <= a * 1.01:
            continue
        tol = float(np.sqrt(a * b))
        steps = _first_stop(r, tol)
        never = (r > tol).all(axis=1)
        score = len(np.unique(steps))
        if never.any() and (best is None or score > best[0]):
            best = (score, tol)
    assert best is not None and best[0] >= 3, f"the contracting model does not spread the images: {r}"
    return best[1]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_settle_contracting_model(shape):
    m, img = _model(shape, contracting=True)
    B = img.shape[0]
    with torch.no_grad():
        base = m(img, iters=60)                                       # (close to) the fixed point
        noise = torch.randn(base.shape, generator=torch.Generator().manual_seed(2)).to(DEV)
        eps = torch.tensor([10.0 ** (1 - 6 * b / (B - 1)) for b in range(B)], device=DEV).view(B, 1, 1, 1)
        start = (base + eps * noise * base.abs().mean()).contiguous()
        states = m(img, iters=MAX_ITERS, levels=start, return_all=True)
        r = _change(states)
        tol = _pick_tol(r)
        assert np.abs(r / tol - 1).min() > 1e-3
        levels, steps = m.settle(img, tol, max_iters=MAX_ITERS, levels=start)
        steps_h = steps.cpu().numpy()
        assert steps.dtype == torch.int32 and steps.is_cuda
        assert np.array_equal(steps_h, _first_stop(r, tol)), (steps_h, r, tol)
        assert (steps_h == MAX_ITERS).any() and len(np.unique(steps_h)) >= 3
        for k in np.unique(steps_h):
            ref = m(img, iters=int(k), levels=start)
            for b in np.nonzero(steps_h == k)[0]:
                assert torch.equal(levels[b], ref[b]), (shape, int(b), int(k))
        # determinism: a second call gives the same bits
        levels2, steps2 = m.settle(img, tol, max_iters=MAX_ITERS, levels=start)
        assert torch.equal(levels, levels2) and torch.equal(steps, steps2)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["n256_whole_blocks", "n64_four_images_per_block", "n625_key_passes"])
def test_settle_limits_with_random_weights(shape):
    m, img = _model(shape, contracting=False)
    B = img.shape[0]
    with torch.no_grad():
        levels, steps = m.settle(img, -1.0, max_iters=5)
        assert torch.equal(steps.cpu(), torch.full((B,), 5, dtype=torch.int32))
        assert torch.equal(levels, m(img, iters=5))
        levels, steps = m.settle(img, float("inf"), max_iters=5)
        assert torch.equal(steps.cpu(), torch.ones(B, dtype=torch.int32))
        assert torch.equal(levels, m(img, iters=1))
        levels, steps = m.settle(img, float("inf"))                  # max_iters = None -> 2L, stops after one step
        assert torch.equal(steps.cpu(), torch.ones(B, dtype=torch.int32))


@pytest.mark.gpu
def test_forward_after_settle_takes_the_ordinary_prologue():
    m, img = _model("n64_four_images_per_block", contracting=False)
    with torch.no_grad():
        out1 = m(img, iters=3)                       # the workspace now holds out1's shadows
        settled, _ = m.settle(img, 1e-2, max_iters=4, levels=out1)
        a = m(img, iters=2, levels=out1)
        b = m(img, iters=2, levels=out1.clone())
        assert torch.equal(a, b)
        c = m(img, iters=2, levels=settled)
        d = m(img, iters=2, levels=settled.clone())
        assert torch.equal(c, d)


@pytest.mark.gpu
def test_settle_errors_on_gpu():
    m, img = _model("n64_four_images_per_block", contracting=False)
    with pytest.raises(RuntimeError, match="inference only"):
        m.settle(img, 1e-3)                          # parameters require grad, grad mode on
    with torch.no_grad(), pytest.raises(ValueError, match="max_iters"):
        m.settle(img, 1e-3, max_iters=0)
    f = G.Glom(dim=64, levels=3, image_size=28, patch_size=7, precision="fp32").to(DEV).eval()
    with torch.no_grad(), pytest.raises(RuntimeError, match="bf16"):
        f.settle(torch.randn(1, 3, 28, 28, device=DEV), 1e-3)
