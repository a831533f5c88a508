"""Glom.settle_video: S video streams settled frame by frame through fixed batch slots, each frame starting from the
levels its stream's previous frame settled at.

CPU: argument errors of the C ABI (reached before any device query), the workspace sizes and the Python-side errors that
need no device.
GPU: on a token-sensitive contracting model (both second MLP layers scaled down, so that the columns settle and the
tokens still move the fixed point) with frames base_s + drift_s * f * noise_s, drift sizes spread over decades across
streams, every frame's levels and step count are bit-identical to the host loop of settle over the frames, with and
without a start state, at slots = S, 1, a count that does not divide S and > S, for each test_settle shape.  Also F = 1
against settle_queue, chunked calls, the tol = -1 / tol = inf limits, a NaN stream, determinism and stale workspace
reads, the following forward, a production batch at configs[1] and the errors."""
import copy
import ctypes

import pytest
import torch

import glom_pytorch_b200 as G
from glom_pytorch_b200 import _native
from test_settle import SHAPES

DEV = "cuda:0"
MAX_ITERS = 12
FRAMES = 4
SECOND_LAYER_SCALE = 0.1     # contracting, but the tokens still move the fixed point


# ---------------------------------------------------------------------------------------------------------- CPU
def _cfg(precision="bf16", dim=128, levels=3, n=64):
    return _native.make_cfg(dim, levels, n, False, 0, 0, precision)


P = 0x100000                 # a 1024-byte aligned stand-in pointer; never dereferenced (errors come first)


def _video_rc(fn, cfg, streams=3, frames=4, slots=2, max_iters=4, tol=0.1, steps=0x1000, tokens=P, state_in=None,
              init=P, state_out=P + 0x400000, ws=P, ws_bytes=1 << 30, pos=P):
    lib = _native.load()
    if fn == "begin":
        return lib.glom_b200_settle_video_begin(ctypes.byref(cfg), tokens, pos, state_in, init, state_out, steps, streams,
                                                frames, slots, max_iters, ctypes.c_float(tol), ws, ws_bytes, None)
    return lib.glom_b200_settle_video_run(ctypes.byref(cfg), P, tokens, pos, state_in, init, state_out, steps, streams,
                                          frames, slots, max_iters, ctypes.c_float(tol), ws, ws_bytes, None, 0, max_iters,
                                          None)


@pytest.mark.parametrize("fn", ["begin", "run"])
@pytest.mark.parametrize("what,kw,rc,msg", [
    ("fp32 engine", dict(cfg=_cfg("fp32")), -1, "bf16"),
    ("streams = 0", dict(streams=0), -1, "streams must be >= 1"),
    ("frames = 0", dict(frames=0), -1, "frames must be >= 1"),
    ("streams x frames overflows", dict(streams=1 << 16, frames=1 << 15), -1, "2^31"),
    ("slots = 0", dict(slots=0), -1, "slots"),
    ("max_iters = 0", dict(max_iters=0), -1, "max_iters"),
    ("NaN tol", dict(tol=float("nan")), -1, "NaN"),
    ("NULL steps_out", dict(steps=None), -1, "steps_out"),
    ("misaligned steps_out", dict(steps=0x1002), -1, "steps_out"),
    ("NULL tokens", dict(tokens=None), -1, "required pointer"),
    ("NULL pos", dict(pos=None), -1, "required pointer"),
    ("NULL state_out", dict(state_out=None), -1, "required pointer"),
    ("no start", dict(init=None), -1, "state_in or init_levels"),
    ("state_out aliases state_in", dict(state_in=P + 0x400000), -1, "alias"),
    ("misaligned workspace", dict(ws=P + 16), -1, "1024-byte"),
    ("misaligned tensor", dict(tokens=P + 4), -1, "16-byte"),
    ("small workspace", dict(ws_bytes=1024), -2, "workspace"),
])
def test_settle_video_argument_errors(fn, what, kw, rc, msg):
    kw = dict(kw)
    cfg = kw.pop("cfg", _cfg())
    assert _video_rc(fn, cfg, **kw) == rc, what
    err = _native.load().glom_b200_last_error().decode()
    assert err.startswith("settle_video") and msg in err, (what, err)


def test_settle_video_run_argument_errors():
    lib = _native.load()
    cfg = _cfg()

    def run(packed=P, first=0, num=4, remaining=None):
        return lib.glom_b200_settle_video_run(ctypes.byref(cfg), packed, P, P, None, P, P + 0x400000, 0x1000, 3, 4, 2, 4,
                                              ctypes.c_float(0.1), P, 1 << 30, None, first, num, remaining)
    for what, kw, msg in [("NULL packed weights", dict(packed=None), "packed"),
                          ("misaligned packed weights", dict(packed=P + 64), "packed"),
                          ("negative first_step", dict(first=-1), "first_step"),
                          ("negative num_steps", dict(num=-1), "num_steps"),
                          ("misaligned remaining_out", dict(remaining=0x1002), "remaining_out")]:
        assert run(**kw) == -1, what
        err = lib.glom_b200_last_error().decode()
        assert err.startswith("settle_video") and msg in err, (what, err)


def test_settle_video_workspace_bytes_errors():
    with pytest.raises(_native.GlomB200Error, match="settle_video: bf16"):
        _native.settle_video_workspace_bytes(_cfg("fp32"), 2, 4)
    with pytest.raises(_native.GlomB200Error, match="settle_video: slots"):
        _native.settle_video_workspace_bytes(_cfg(), 0, 4)
    with pytest.raises(_native.GlomB200Error, match="settle_video: max_iters"):
        _native.settle_video_workspace_bytes(_cfg(), 2, 0)


@pytest.mark.parametrize("dim,levels,n,slots,iters", [
    (512, 6, 256, 32, 12),        # configs[1]
    (128, 3, 64, 8, 6),
    (64, 2, 625, 3, 6),
    (192, 3, 144, 1, 12),
])
def test_settle_video_workspace_bytes(dim, levels, n, slots, iters):
    cfg = _cfg(dim=dim, levels=levels, n=n)
    v = _native.settle_video_workspace_bytes(cfg, slots, iters)
    assert v >= _native.settle_queue_workspace_bytes(cfg, slots, iters)
    assert v % 1024 == 0
    assert _native.settle_video_workspace_bytes(cfg, slots + 1, iters) > v


def test_settle_video_rejects_fp32_model_and_cpu_input():
    m = G.Glom(dim=64, levels=3, image_size=28, patch_size=7, precision="fp32")
    with torch.no_grad(), pytest.raises(RuntimeError, match="bf16"):
        m.settle_video(torch.randn(1, 2, 3, 28, 28), 1e-3)
    m = G.Glom(dim=64, levels=3, image_size=28, patch_size=7)
    with torch.no_grad(), pytest.raises(RuntimeError, match="no CPU fallback"):
        m.settle_video(torch.randn(1, 2, 3, 28, 28), 1e-3)


# ---------------------------------------------------------------------------------------------------------- GPU
def _model(dim, L, isz, p, attend_self=False, radius=0, contracting=True):
    torch.manual_seed(0)
    m = G.Glom(dim=dim, levels=L, image_size=isz, patch_size=p, consensus_self=attend_self,
               local_consensus_radius=radius).to(DEV).eval()
    if contracting:
        with torch.no_grad():
            m.bottom_up.net[3].weight.mul_(SECOND_LAYER_SCALE)
            m.top_down.net[3].weight.mul_(SECOND_LAYER_SCALE)
    return m


def _shape_model(shape, contracting=True):
    dim, L, isz, p, attend_self, radius, S = SHAPES[shape]
    return _model(dim, L, isz, p, attend_self, radius, contracting), S, isz


def _frames(S, F, isz, seed=1):
    """(S, F, 3, isz, isz): frame f of stream s is base_s + drift_s * f * noise_s, drift_s spread over six decades (in
    shuffled stream order)."""
    g = torch.Generator().manual_seed(seed)
    base = torch.randn(S, 1, 3, isz, isz, generator=g)
    noise = torch.randn(S, 1, 3, isz, isz, generator=g)
    order = torch.randperm(S, generator=g).double()
    drift = (10.0 ** (-6 * order / max(S - 1, 1))).float().view(S, 1, 1, 1, 1)
    f = torch.arange(F, dtype=torch.float32).view(1, F, 1, 1, 1)
    return (base + drift * f * noise).to(DEV)


def _start(m, frames):
    """A start for frame 0 near its fixed point, with noise of sizes spread over decades across the streams."""
    S = frames.shape[0]
    base = m(frames[:, 0], iters=40)
    noise = torch.randn(base.shape, generator=torch.Generator().manual_seed(2)).to(DEV)
    eps = torch.tensor([10.0 ** (-1 - 4 * s / max(S - 1, 1)) for s in range(S)], device=DEV).view(S, 1, 1, 1)
    return (base + eps * noise * base.abs().mean()).contiguous()


def _host_loop(m, frames, tol, levels=None, max_iters=MAX_ITERS):
    """The per-frame settle loop settle_video must equal -> (levels (S, F, n, L, d), steps (S, F))."""
    outs, steps, lv = [], [], levels
    for f in range(frames.shape[1]):
        lv, st = m.settle(frames[:, f], tol, max_iters=max_iters, levels=lv)
        outs.append(lv)
        steps.append(st)
    return torch.stack(outs, 1), torch.stack(steps, 1)


def _pick_tol(m, frames, levels):
    """The tol (on a half-decade grid) whose host loop spreads the steps of frames >= 1 over the most distinct values."""
    best = None
    for k in range(4, 17):
        tol = 10.0 ** (-k / 2)
        _, st = _host_loop(m, frames, tol, levels)
        score = len(torch.unique(st[:, 1:]))
        if best is None or score > best[0]:
            best = (score, tol)
    return best[1]


def _mixed(steps):
    return len(torch.unique(steps[:, 1:])) >= 3


def _not_dividing(S):
    return next(k for k in range(2, S + 1) if S % k) if S > 2 else 2


@pytest.mark.gpu
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_settle_video_equals_the_host_loop(shape):
    m, S, isz = _shape_model(shape)
    frames = _frames(S, FRAMES, isz)
    with torch.no_grad():
        for levels in (_start(m, frames), None):
            tol = _pick_tol(m, frames, levels)
            want, want_steps = _host_loop(m, frames, tol, levels)
            assert _mixed(want_steps), (shape, levels is None, want_steps)
            for slots in (S, 1, _not_dividing(S), S + 3):              # S + 3: clipped to S
                got, steps = m.settle_video(frames, tol, max_iters=MAX_ITERS, levels=levels, slots=slots)
                assert steps.dtype == torch.int32 and steps.is_cuda and steps.shape == (S, FRAMES)
                assert got.dtype == torch.float32 and got.shape == want.shape
                assert torch.equal(steps, want_steps), (shape, slots, levels is None, steps, want_steps)
                assert torch.equal(got, want), (shape, slots, levels is None)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_settle_video_of_one_frame_is_settle_queue(shape):
    m, S, isz = _shape_model(shape)
    frames = _frames(S, 1, isz)
    with torch.no_grad():
        start = _start(m, frames)
        for levels in (start, None):
            for slots in (S, 2):
                got, steps = m.settle_video(frames, 1e-4, max_iters=MAX_ITERS, levels=levels, slots=slots)
                want, want_steps = m.settle_queue(frames[:, 0], 1e-4, max_iters=MAX_ITERS, levels=levels, slots=slots)
                assert torch.equal(steps[:, 0], want_steps) and torch.equal(got[:, 0], want), (shape, slots)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["n64_four_images_per_block", "n625_key_passes"])
def test_settle_video_in_chunks_equals_one_call(shape):
    m, S, isz = _shape_model(shape)
    F = 6
    frames = _frames(S, F, isz, seed=3)
    with torch.no_grad():
        tol = _pick_tol(m, frames[:, :3], None)
        whole, whole_steps = m.settle_video(frames, tol, max_iters=MAX_ITERS, slots=3)
        assert _mixed(whole_steps)
        for k in (1, 4):
            a, sa = m.settle_video(frames[:, :k], tol, max_iters=MAX_ITERS, slots=3)
            b, sb = m.settle_video(frames[:, k:], tol, max_iters=MAX_ITERS, levels=a[:, -1], slots=2)
            assert torch.equal(torch.cat([sa, sb], 1), whole_steps), k
            assert torch.equal(torch.cat([a, b], 1), whole), k


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["n256_whole_blocks", "n64_four_images_per_block", "n625_key_passes"])
def test_settle_video_limits_with_random_weights(shape):
    m, S, isz = _shape_model(shape, contracting=False)
    F = 3
    frames = _frames(S, F, isz)
    with torch.no_grad():
        levels, steps = m.settle_video(frames, -1.0, max_iters=5, slots=3)
        assert torch.equal(steps.cpu(), torch.full((S, F), 5, dtype=torch.int32))
        prev = None
        for f in range(F):
            prev = m(frames[:, f], iters=5, levels=None if prev is None else prev.clone())
            assert torch.equal(levels[:, f], prev), f
        levels, steps = m.settle_video(frames, float("inf"), max_iters=5, slots=3)
        assert torch.equal(steps.cpu(), torch.ones((S, F), dtype=torch.int32))
        prev = None
        for f in range(F):
            prev = m(frames[:, f], iters=1, levels=None if prev is None else prev.clone())
            assert torch.equal(levels[:, f], prev), f
        _, steps = m.settle_video(frames, float("inf"), slots=2)          # max_iters = None -> 2L
        assert torch.equal(steps.cpu(), torch.ones((S, F), dtype=torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["n64_four_images_per_block", "n144_radius_self"])
def test_settle_video_nan_stream_leaves_the_others_alone(shape):
    m, S, isz = _shape_model(shape)
    frames = _frames(S, FRAMES, isz)
    with torch.no_grad():
        tol = _pick_tol(m, frames, None)
        want, want_steps = m.settle_video(frames, tol, max_iters=MAX_ITERS, slots=3)
        nan = torch.full_like(frames[:1], float("nan"))
        with_nan = torch.cat([frames[:1], nan, frames[1:]]).contiguous()
        got, steps = m.settle_video(with_nan, tol, max_iters=MAX_ITERS, slots=3)
        assert torch.equal(steps[1].cpu(), torch.full((FRAMES,), MAX_ITERS, dtype=torch.int32))
        keep = [0] + list(range(2, S + 1))
        assert torch.equal(steps[keep], want_steps) and torch.equal(got[keep], want)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["n64_four_images_per_block", "n144_radius_self"])
def test_settle_video_is_deterministic_and_reads_no_stale_workspace(shape):
    m, S, isz = _shape_model(shape)
    frames = _frames(S, FRAMES, isz)
    with torch.no_grad():
        start = _start(m, frames)
        tol = _pick_tol(m, frames, start)
        a, sa = m.settle_video(frames, tol, max_iters=MAX_ITERS, levels=start, slots=3)
        assert _mixed(sa)
        b, sb = m.settle_video(frames, tol, max_iters=MAX_ITERS, levels=start, slots=3)
        assert torch.equal(a, b) and torch.equal(sa, sb)
        ws = m._workspace
        for fill in (0xFF, 0x00):                   # 0xFF bytes: NaN floats and bf16, -1 ints
            ws.fill_(fill)
            c, sc = m.settle_video(frames, tol, max_iters=MAX_ITERS, levels=start, slots=3)
            assert m._workspace.data_ptr() == ws.data_ptr()
            assert torch.equal(a, c) and torch.equal(sa, sc), fill


@pytest.mark.gpu
def test_forward_after_settle_video_takes_the_ordinary_prologue():
    m, S, isz = _shape_model("n64_four_images_per_block", contracting=False)
    frames = _frames(S, 3, isz)
    with torch.no_grad():
        m(frames[:, 0], iters=3)                     # the workspace now holds that state's shadows
        out, _ = m.settle_video(frames, 1e-2, max_iters=4, slots=3)
        a = m(frames[:, -1], levels=out[:, -1], iters=2)
        fresh = copy.deepcopy(m)
        b = fresh(frames[:, -1], levels=out[:, -1], iters=2)
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_settle_video_production_batch():
    """configs[1] dims, 40 streams x 3 frames through 32 slots: K1, K2 and K3 deal several tiles per CTA."""
    m = _model(512, 6, 224, 14)
    S, F = 40, 3
    rows = 32 * 256
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert (rows // 256) * (4 * 512 // 256) * 11 > sms            # K1: more tiles than CTAs
    frames = _frames(S, F, 224)
    with torch.no_grad():
        start = _start(m, frames)
        for tol, levels in ((1e-4, start), (1e-3, None)):
            want, want_steps = _host_loop(m, frames, tol, levels)
            got, steps = m.settle_video(frames, tol, max_iters=MAX_ITERS, levels=levels, slots=32)
            assert torch.equal(steps, want_steps), (tol, steps, want_steps)
            assert torch.equal(got, want), tol


@pytest.mark.gpu
def test_settle_video_errors_on_gpu():
    m, S, isz = _shape_model("n64_four_images_per_block", contracting=False)
    frames = _frames(2, 2, isz)
    with pytest.raises(RuntimeError, match="inference only"):
        m.settle_video(frames, 1e-3)                 # parameters require grad, grad mode on
    with torch.no_grad():
        with pytest.raises(ValueError, match="max_iters"):
            m.settle_video(frames, 1e-3, max_iters=0)
        with pytest.raises(ValueError, match="NaN"):
            m.settle_video(frames, float("nan"))
        with pytest.raises(ValueError, match="slots"):
            m.settle_video(frames, 1e-3, slots=0)
        with pytest.raises(RuntimeError, match="not \\(S, F, 3, H, W\\)"):
            m.settle_video(frames[:, 0], 1e-3)       # 4-D
        with pytest.raises(RuntimeError, match="not \\(S, F, 3, H, W\\)"):
            m.settle_video(frames[:, :, :2], 1e-3)   # 2 channels
        with pytest.raises(RuntimeError, match="not \\(S, F, 3, H, W\\)"):
            m.settle_video(frames[..., :-1], 1e-3)   # W not a multiple of the patch size
        with pytest.raises(RuntimeError, match="at least one"):
            m.settle_video(frames[:, :0], 1e-3)
        with pytest.raises(RuntimeError, match="levels must have shape"):
            m.settle_video(frames, 1e-3, levels=torch.zeros(2, 2, 64, 3, 128, device=DEV))   # per-frame levels
        with pytest.raises(RuntimeError, match="levels must have shape"):
            m.settle_video(frames, 1e-3, levels=torch.zeros(3, 64, 3, 128, device=DEV))
    f = G.Glom(dim=64, levels=3, image_size=28, patch_size=7, precision="fp32").to(DEV).eval()
    with torch.no_grad(), pytest.raises(RuntimeError, match="bf16"):
        f.settle_video(torch.randn(1, 2, 3, 28, 28, device=DEV), 1e-3)
