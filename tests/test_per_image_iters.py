"""Glom.forward with a per-image step count: iters = a (B,) vector, each image runs its own number of steps.

CPU: argument errors of glom_b200_forward_steps / glom_b200_backward_steps (reported before any device query), the
workspace size, and the Python argument errors that need no device.
GPU: random weights, a step vector holding 0, the maximum and values in between, with and without a carried-in state, at
n = 256 (whole 256-row blocks frozen), n = 64 (four images per block: masked rows inside running tiles), n = 625
(consensus key passes) and n = 144 with a radius mask and consensus_self.  Every image is bit-identical to
forward(iters=steps[b]) with and without return_all; the settled levels of Glom.settle are reproduced; a uniform vector
is the scalar call; out-of-range entries are clamped on the device.  Gradients of sum(out * cot) match the sum over the
distinct step counts k of the same loss on forward(iters=k) with the cotangent restricted to the images that run k
steps, on the tensor-core backward (dim 256) and the CUDA-core backward (dim 128)."""
import ctypes

import numpy as np
import pytest
import torch

import glom_pytorch_b200 as G
from glom_pytorch_b200 import _native
from glom_pytorch_b200.glom import _aligned_bytes

DEV = "cuda:0"


# ---------------------------------------------------------------------------------------------------------- CPU
def _cfg(precision="bf16", dim=128, levels=3, n=64):
    return _native.make_cfg(dim, levels, n, False, 0, 0, precision)


FAKE = 0x100000          # 1024-aligned, never dereferenced: every error below is reported before any device work


def _forward_steps_rc(cfg, steps=FAKE, max_steps=4):
    lib = _native.load()
    p = ctypes.c_void_p(FAKE)
    return lib.glom_b200_forward_steps(ctypes.byref(cfg), p, p, p, None, p, p, 2, steps, max_steps, 0, p, 1 << 30, None)


def _backward_steps_rc(cfg, steps=FAKE, max_steps=4, grads=True):
    lib = _native.load()
    p = ctypes.c_void_p(FAKE)
    w = _native.WeightsRef(ctypes.sizeof(_native.WeightsRef), *([FAKE] * 8))
    names = [k for k, _ in _native.Grads._fields_[1:]]
    g = _native.Grads(ctypes.sizeof(_native.Grads), *[(FAKE if grads and k != "d_state0" else None) for k in names])
    return lib.glom_b200_backward_steps(ctypes.byref(cfg), ctypes.byref(w), p, p, p, p, ctypes.byref(g), 2, steps,
                                        max_steps, 0, p, 1 << 30, None)


@pytest.mark.parametrize("what,call,msg", [
    ("forward: NULL steps", lambda: _forward_steps_rc(_cfg(), steps=None), "steps is NULL"),
    ("forward: max_steps < 0", lambda: _forward_steps_rc(_cfg(), max_steps=-1), "max_steps"),
    ("forward: fp32 engine", lambda: _forward_steps_rc(_cfg("fp32")), "bf16"),
    ("backward: NULL steps", lambda: _backward_steps_rc(_cfg(), steps=None), "steps is NULL"),
    ("backward: max_steps < 0", lambda: _backward_steps_rc(_cfg(), max_steps=-1), "max_steps"),
    ("backward: NULL gradients", lambda: _backward_steps_rc(_cfg(), grads=False), "gradient pointers"),
])
def test_steps_abi_argument_errors(what, call, msg):
    assert call() == -1, what
    assert msg in _native.load().glom_b200_last_error().decode(), what


@pytest.mark.parametrize("dim,levels,n,batch,max_steps", [(512, 6, 256, 32, 12), (128, 3, 64, 8, 6), (64, 2, 625, 3, 0)])
@pytest.mark.parametrize("return_all", [False, True])
def test_forward_steps_workspace_bytes(dim, levels, n, batch, max_steps, return_all):
    cfg = _cfg(dim=dim, levels=levels, n=n)
    fwd = _native.workspace_bytes(cfg, batch, max_steps, return_all)
    ws = _native.forward_steps_workspace_bytes(cfg, batch, max_steps, return_all)
    assert ws >= fwd + batch * 4 + (batch * n + 255) // 256 * 4        # + per-image and per-256-row-block flags
    assert ws % 1024 == 0
    with pytest.raises(_native.GlomB200Error, match="bf16"):
        _native.forward_steps_workspace_bytes(_cfg("fp32"), batch, max_steps, return_all)
    with pytest.raises(_native.GlomB200Error, match="max_steps"):
        _native.forward_steps_workspace_bytes(cfg, batch, -1, return_all)


@pytest.mark.parametrize("iters,err", [
    ([1, 2], ValueError),                                  # wrong length
    (torch.tensor([1.0, 2.0, 3.0]), ValueError),           # not an integer dtype
    (torch.tensor([[1, 2, 3]]), ValueError),               # more than one dimension
    (torch.tensor([1, -1, 3]), ValueError),                # a negative entry
    ([1, 2.5, 3], ValueError),                             # a list entry that is not an integer
])
def test_per_image_iters_python_errors_without_a_device(iters, err):
    m = G.Glom(dim=64, levels=3, image_size=28, patch_size=7)
    with torch.no_grad(), pytest.raises(err):
        m(torch.randn(3, 3, 28, 28), iters=iters)


def test_per_image_iters_need_the_bf16_engine():
    m = G.Glom(dim=64, levels=3, image_size=28, patch_size=7, precision="fp32")
    with torch.no_grad(), pytest.raises(RuntimeError, match="bf16"):
        m(torch.randn(2, 3, 28, 28), iters=[1, 2])


# ---------------------------------------------------------------------------------------------------------- GPU
# (dim, levels, image_size, patch_size, consensus_self, local_consensus_radius, step vector)
SHAPES = {
    "n256_whole_blocks": (256, 3, 64, 4, False, 0, [0, 4, 1, 3, 4, 2]),
    "n64_four_images_per_block": (128, 3, 32, 4, False, 0, [0, 4, 1, 3, 2, 4, 0, 1]),
    "n625_key_passes": (64, 2, 100, 4, False, 0, [2, 0, 4, 1]),
    "n144_radius_self": (192, 3, 48, 4, True, 3, [3, 4, 0, 1, 4]),
}
GRAD_SHAPES = {
    "tensor_core_bwd_n144": (256, 3, 48, 4, False, 0, [0, 4, 1, 3, 2]),        # rows = 720: not a multiple of 128 / 256
    "cuda_core_bwd_n64": (128, 3, 32, 4, False, 0, [0, 4, 1, 3, 2, 4, 0, 1]),
}


def _model(spec, seed=0):
    dim, L, isz, p, attend_self, radius, steps = spec
    torch.manual_seed(seed)
    m = G.Glom(dim=dim, levels=L, image_size=isz, patch_size=p, consensus_self=attend_self,
               local_consensus_radius=radius).to(DEV).eval()
    g = torch.Generator().manual_seed(seed + 1)
    img = torch.randn(len(steps), 3, isz, isz, generator=g).to(DEV)
    n = (isz // p) ** 2
    start = torch.randn(len(steps), n, L, dim, generator=g).to(DEV)
    return m, img, start, steps


@pytest.mark.gpu
@pytest.mark.parametrize("carried", [False, True])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_per_image_iters_bit_identical(shape, carried):
    m, img, start, steps = _model(SHAPES[shape])
    lv = start if carried else None
    T = max(steps)
    st = np.array(steps)
    with torch.no_grad():
        out = m(img, iters=torch.tensor(steps, device=DEV), levels=lv)
        out_all = m(img, iters=steps, levels=lv, return_all=True)
        assert out.shape == (len(steps),) + tuple(start.shape[1:])
        assert out_all.shape == (T + 1, len(steps)) + tuple(start.shape[1:])
        for k in np.unique(st):
            ref = m(img, iters=int(k), levels=lv)
            ref_all = m(img, iters=int(k), levels=lv, return_all=True)
            for b in np.nonzero(st == k)[0]:
                assert torch.equal(out[b], ref[b]), (shape, int(b), int(k))
                for t in range(T + 1):
                    assert torch.equal(out_all[t, b], ref_all[min(t, int(k)), b]), (shape, int(b), int(k), t)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["n256_whole_blocks", "n64_four_images_per_block"])
def test_uniform_vector_is_the_scalar_call(shape):
    m, img, start, steps = _model(SHAPES[shape])
    B = len(steps)
    with torch.no_grad():
        for lv in (None, start):
            ref = m(img, iters=3, levels=lv)
            assert torch.equal(m(img, iters=torch.full((B,), 3, device=DEV), levels=lv), ref)
            assert torch.equal(m(img, iters=[3] * B, levels=lv), ref)
            assert torch.equal(m(img, iters=torch.zeros(B, dtype=torch.int32), levels=lv), m(img, iters=0, levels=lv))


@pytest.mark.gpu
def test_steps_are_clamped_on_the_device():
    m, img, start, _ = _model(SHAPES["n64_four_images_per_block"])
    raw = torch.tensor([-3, 9, 1, 4, -1, 2, 100, 3], dtype=torch.int32, device=DEV)
    max_steps = 4
    with torch.no_grad():
        want = m(img, iters=raw.clamp(0, max_steps), levels=start)
        want_all = m(img, iters=raw.clamp(0, max_steps), levels=start, return_all=True)
        n = (img.shape[2] // m.patch_size) ** 2
        tokens = m.tokens(img)
        with torch.cuda.device(img.device):
            stream = torch.cuda.current_stream().cuda_stream
            cfg = m.engine_cfg(n)
            packed = m._packed_weights(cfg, img.device, stream)
            pos = m.pos_emb.weight[:n].detach().contiguous()
            init = m.init_levels.detach().contiguous()
            for return_all, ref in ((False, want), (True, want_all)):
                out = torch.empty_like(ref)
                nb = _native.forward_steps_workspace_bytes(cfg, img.shape[0], max_steps, return_all)
                ws = _aligned_bytes(nb, img.device)
                _native.forward_steps(cfg, packed.data_ptr(), tokens.data_ptr(), pos.data_ptr(), start.data_ptr(),
                                      init.data_ptr(), out.data_ptr(), img.shape[0], raw.data_ptr(), max_steps, return_all,
                                      ws.data_ptr(), nb, stream)
                assert torch.equal(out, ref), return_all


def _change(states):
    """r[b, k - 1] = max_l sqrt(sum_i |S_k - S_{k-1}|^2 / sum_i |S_k|^2) in float64, states (T+1, B, n, L, d)."""
    s = states.double()
    num = ((s[1:] - s[:-1]) ** 2).sum(dim=(2, 4))
    den = (s[1:] ** 2).sum(dim=(2, 4))
    q = torch.where((num == 0) & (den == 0), torch.zeros_like(num), (num / den).sqrt())
    return q.amax(dim=2).T.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_forward_at_the_settled_depth_reproduces_settle(shape):
    m, img, _, steps = _model(SHAPES[shape])
    B = len(steps)
    with torch.no_grad():
        m.bottom_up.net[3].weight.zero_()                   # contracting: the MLP outputs are constants
        m.top_down.net[3].weight.zero_()
        base = m(img, iters=60)
        noise = torch.randn(base.shape, generator=torch.Generator().manual_seed(2)).to(DEV)
        eps = torch.tensor([10.0 ** (1 - 6 * b / (B - 1)) for b in range(B)], device=DEV).view(B, 1, 1, 1)
        start = (base + eps * noise * base.abs().mean()).contiguous()
        r = _change(m(img, iters=12, levels=start, return_all=True))
        # a tol between two well separated change values near the middle: the images stop at different steps
        vals = np.sort(r[np.isfinite(r) & (r > 0)].ravel())
        gaps = [(i, vals[i + 1] / vals[i]) for i in range(len(vals) - 1) if vals[i + 1] > vals[i] * 1.01]
        i = min(gaps, key=lambda g: abs(g[0] - len(vals) // 2))[0]
        tol = float(np.sqrt(vals[i] * vals[i + 1]))
        levels, settled_steps = m.settle(img, tol, max_iters=12, levels=start)
        assert len(torch.unique(settled_steps)) >= 2, (settled_steps, tol)
        again = m(img, iters=settled_steps, levels=start)
        assert torch.equal(again, levels)


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


@pytest.mark.gpu
@pytest.mark.parametrize("return_all", [False, True])
@pytest.mark.parametrize("carried", [False, True])
@pytest.mark.parametrize("shape", sorted(GRAD_SHAPES))
def test_per_image_iters_gradients(shape, carried, return_all):
    m, img, start, steps = _model(GRAD_SHAPES[shape])
    m.train()
    lv = start if carried else None
    st = torch.tensor(steps, device=DEV)
    T, B = max(steps), len(steps)
    cot = torch.randn(((T + 1,) if return_all else ()) + tuple(start.shape), generator=torch.Generator().manual_seed(5))
    cot = cot.to(DEV)

    got = _grads(m, img, lv, lambda x, s: (m(x, iters=st, levels=s, return_all=return_all) * cot).sum())

    def reference(x, s):
        loss = 0.0
        for k in sorted(set(steps)):
            sel = (st == k).view(-1, 1, 1, 1).float()
            if return_all:
                c = torch.cat([cot[:k], cot[k:].sum(0, keepdim=True)]) * sel            # slabs k..T all equal S_k
            else:
                c = cot * sel
            loss = loss + (m(x, iters=k, levels=s, return_all=return_all) * c).sum()
        return loss

    want = _grads(m, img, lv, reference)
    assert set(got) == set(want)
    for k in want:
        assert torch.isfinite(got[k]).all(), k
        assert _rel(got[k], want[k]) <= 1e-4, (shape, k, _rel(got[k], want[k]))
    if carried and not return_all:
        for b in range(B):
            if steps[b] == 0:
                assert torch.equal(got["levels"][b], cot[b])      # a 0-step image passes its cotangent straight through


@pytest.mark.gpu
def test_per_image_iters_errors_on_gpu():
    m, img, _, steps = _model(SHAPES["n64_four_images_per_block"])
    with torch.no_grad():
        with pytest.raises(ValueError):
            m(img, iters=torch.tensor([1, -1] * 4, device=DEV))
        with pytest.raises(ValueError):
            m(img, iters=torch.tensor(steps[:-1], device=DEV))
    f = G.Glom(dim=64, levels=3, image_size=28, patch_size=7, precision="fp32").to(DEV).eval()
    with torch.no_grad(), pytest.raises(RuntimeError, match="bf16"):
        f(torch.randn(2, 3, 28, 28, device=DEV), iters=[1, 2])
