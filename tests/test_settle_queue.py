"""Glom.settle_queue: N images settled through fixed batch slots, each slot refilled on the GPU as its image stops.

CPU: argument errors of the C ABI (reached before any device query) and the workspace sizes.
GPU: on the contracting model of test_settle (second MLP layers zeroed, start = fixed point + noise spread over decades)
with N = 3 * slots + 1 images, every image's levels and step count are bit-identical to settle on the whole N-image batch,
with and without a start state, at slots = 1, at a slot count that does not divide N and at slots >= N, for each
test_settle shape.  Also the tol = -1 / tol = inf limits, determinism, a workspace pre-filled with NaN bytes (no stale
shadow, token, group-0 or flag read in a refilled slot) and the errors."""
import ctypes

import numpy as np
import pytest
import torch

import glom_pytorch_b200 as G
from glom_pytorch_b200 import _native
from test_settle import SHAPES, _change, _pick_tol

DEV = "cuda:0"
MAX_ITERS = 12


# ---------------------------------------------------------------------------------------------------------- CPU
def _cfg(precision="bf16", dim=128, levels=3, n=64):
    return _native.make_cfg(dim, levels, n, False, 0, 0, precision)


def _queue_rc(fn, cfg, images=5, slots=2, max_iters=4, tol=0.1, steps=0x1000):
    lib = _native.load()
    p = ctypes.c_void_p(0x100000)
    if fn == "begin":
        return lib.glom_b200_settle_queue_begin(ctypes.byref(cfg), p, p, None, p, p, steps, images, slots, max_iters,
                                                ctypes.c_float(tol), p, 1 << 30, None)
    return lib.glom_b200_settle_queue_run(ctypes.byref(cfg), p, p, p, None, p, p, steps, images, slots, max_iters,
                                          ctypes.c_float(tol), p, 1 << 30, None, 0, max_iters, None)


@pytest.mark.parametrize("fn", ["begin", "run"])
@pytest.mark.parametrize("what,kw,msg", [
    ("fp32 engine", dict(cfg=_cfg("fp32")), "bf16"),
    ("images = 0", dict(images=0), "images"),
    ("slots = 0", dict(slots=0), "slots"),
    ("max_iters = 0", dict(max_iters=0), "max_iters"),
    ("NaN tol", dict(tol=float("nan")), "NaN"),
    ("NULL steps_out", dict(steps=None), "steps_out"),
    ("misaligned steps_out", dict(steps=0x1002), "steps_out"),
])
def test_settle_queue_argument_errors(fn, what, kw, msg):
    kw = dict(kw)
    cfg = kw.pop("cfg", _cfg())
    rc = _queue_rc(fn, cfg, **kw)
    assert rc == -1, what
    assert msg in _native.load().glom_b200_last_error().decode(), what


def test_settle_queue_workspace_bytes_errors():
    with pytest.raises(_native.GlomB200Error, match="bf16"):
        _native.settle_queue_workspace_bytes(_cfg("fp32"), 2, 4)
    with pytest.raises(_native.GlomB200Error, match="slots"):
        _native.settle_queue_workspace_bytes(_cfg(), 0, 4)
    with pytest.raises(_native.GlomB200Error, match="max_iters"):
        _native.settle_queue_workspace_bytes(_cfg(), 2, 0)


@pytest.mark.parametrize("dim,levels,n,slots,iters", [
    (512, 6, 256, 32, 12),        # configs[1]
    (128, 3, 64, 8, 6),
    (64, 2, 625, 3, 6),
    (192, 3, 144, 1, 12),
])
def test_settle_queue_workspace_extends_the_settle_workspace(dim, levels, n, slots, iters):
    cfg = _cfg(dim=dim, levels=levels, n=n)
    q = _native.settle_queue_workspace_bytes(cfg, slots, iters)
    st = _native.settle_workspace_bytes(cfg, slots, iters)
    # + a second fp32 state slab of the slots + five per-slot ints, the per-block fresh flags and two counters
    assert q >= st + slots * n * levels * dim * 4 + 5 * slots * 4 + 8
    assert q % 1024 == 0
    assert _native.settle_queue_workspace_bytes(cfg, slots + 1, iters) > q


# ---------------------------------------------------------------------------------------------------------- GPU
def _model(shape, contracting, images):
    dim, L, isz, p, attend_self, radius, _ = SHAPES[shape]
    torch.manual_seed(0)
    m = G.Glom(dim=dim, levels=L, image_size=isz, patch_size=p, consensus_self=attend_self,
               local_consensus_radius=radius).to(DEV).eval()
    if contracting:
        with torch.no_grad():
            m.bottom_up.net[3].weight.zero_()
            m.top_down.net[3].weight.zero_()
    img = torch.randn(images, 3, isz, isz, generator=torch.Generator().manual_seed(1)).to(DEV)
    return m, img


def _spread_start(m, img):
    """A start near the fixed point with noise of sizes spread over six decades, and a tol that spreads the stops."""
    N = img.shape[0]
    base = m(img, iters=60)
    noise = torch.randn(base.shape, generator=torch.Generator().manual_seed(2)).to(DEV)
    eps = torch.tensor([10.0 ** (1 - 6 * b / (N - 1)) for b in range(N)], device=DEV).view(N, 1, 1, 1)
    start = (base + eps * noise * base.abs().mean()).contiguous()
    r = _change(m(img, iters=MAX_ITERS, levels=start, return_all=True))
    return start, _pick_tol(r)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_settle_queue_equals_settle_on_the_whole_batch(shape):
    slots = 4
    N = 3 * slots + 1
    m, img = _model(shape, contracting=True, images=N)
    with torch.no_grad():
        start, tol = _spread_start(m, img)
        for levels in (start, None):
            want, want_steps = m.settle(img, tol, max_iters=MAX_ITERS, levels=levels)
            if levels is not None:
                assert len(np.unique(want_steps.cpu().numpy())) >= 3
            for s in (slots, 1, 5, N, N + 3):              # 5 does not divide 13; N + 3 is clipped to N
                got, steps = m.settle_queue(img, tol, max_iters=MAX_ITERS, levels=levels, slots=s)
                assert steps.dtype == torch.int32 and steps.is_cuda and got.shape == want.shape
                assert torch.equal(steps, want_steps), (shape, s, levels is None, steps, want_steps)
                assert torch.equal(got, want), (shape, s, levels is None)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["n256_whole_blocks", "n64_four_images_per_block", "n625_key_passes"])
def test_settle_queue_limits_with_random_weights(shape):
    N = 7
    m, img = _model(shape, contracting=False, images=N)
    with torch.no_grad():
        levels, steps = m.settle_queue(img, -1.0, max_iters=5, slots=3)
        assert torch.equal(steps.cpu(), torch.full((N,), 5, dtype=torch.int32))
        assert torch.equal(levels, m(img, iters=5))
        levels, steps = m.settle_queue(img, float("inf"), max_iters=5, slots=3)
        assert torch.equal(steps.cpu(), torch.ones(N, dtype=torch.int32))
        assert torch.equal(levels, m(img, iters=1))
        _, steps = m.settle_queue(img, float("inf"), slots=2)           # max_iters = None -> 2L
        assert torch.equal(steps.cpu(), torch.ones(N, dtype=torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["n64_four_images_per_block", "n144_radius_self"])
def test_settle_queue_is_deterministic_and_reads_no_stale_workspace(shape):
    slots = 3
    m, img = _model(shape, contracting=True, images=3 * slots + 1)
    with torch.no_grad():
        start, tol = _spread_start(m, img)
        a, sa = m.settle_queue(img, tol, max_iters=MAX_ITERS, levels=start, slots=slots)
        b, sb = m.settle_queue(img, tol, max_iters=MAX_ITERS, levels=start, slots=slots)
        assert torch.equal(a, b) and torch.equal(sa, sb)
        ws = m._workspace
        for fill in (0xFF, 0x00):                   # 0xFF bytes: NaN floats and bf16, -1 ints
            ws.fill_(fill)
            c, sc = m.settle_queue(img, tol, max_iters=MAX_ITERS, levels=start, slots=slots)
            assert m._workspace.data_ptr() == ws.data_ptr()
            assert torch.equal(a, c) and torch.equal(sa, sc), fill


@pytest.mark.gpu
def test_settle_queue_errors_on_gpu():
    m, img = _model("n64_four_images_per_block", contracting=False, images=3)
    with pytest.raises(RuntimeError, match="inference only"):
        m.settle_queue(img, 1e-3)                    # parameters require grad, grad mode on
    with torch.no_grad():
        with pytest.raises(ValueError, match="max_iters"):
            m.settle_queue(img, 1e-3, max_iters=0)
        with pytest.raises(ValueError, match="NaN"):
            m.settle_queue(img, float("nan"))
        with pytest.raises(ValueError, match="slots"):
            m.settle_queue(img, 1e-3, slots=0)
        with pytest.raises(RuntimeError, match="levels must have shape"):
            m.settle_queue(img, 1e-3, levels=torch.zeros(2, 64, 3, 128, device=DEV))
    f = G.Glom(dim=64, levels=3, image_size=28, patch_size=7, precision="fp32").to(DEV).eval()
    with torch.no_grad(), pytest.raises(RuntimeError, match="bf16"):
        f.settle_queue(torch.randn(1, 3, 28, 28, device=DEV), 1e-3)


def test_settle_queue_rejects_fp32_model_and_cpu_input():
    m = G.Glom(dim=64, levels=3, image_size=28, patch_size=7, precision="fp32")
    with torch.no_grad(), pytest.raises(RuntimeError, match="bf16"):
        m.settle_queue(torch.randn(1, 3, 28, 28), 1e-3)
    m = G.Glom(dim=64, levels=3, image_size=28, patch_size=7)
    with torch.no_grad(), pytest.raises(RuntimeError, match="no CPU fallback"):
        m.settle_queue(torch.randn(1, 3, 28, 28), 1e-3)
