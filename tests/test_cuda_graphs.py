"""Every engine call under CUDA graph capture and on concurrent streams.

A captured graph freezes the pointers and the kernel list its capture saw, so whatever one call leaves behind for the
next (the packed weights, the per-stream workspaces, the resume record, staged tokens, the radius-mask key) must never
leak into a capture.  A call under capture packs the weights inside its graph into a buffer of its own, takes its
workspaces from buffers no other call touches, neither resumes nor leaves a resume record, and reads nothing on the
host (DESIGN.md, "CUDA graphs and streams").

Every check is bit for bit against an eager call on ``copy.deepcopy`` of the module taken before any capture: the copy
starts with empty caches, so it takes the ordinary path that the oracle suites pin against float64.  Graphs are
replayed after new inputs are copied into their static tensors, in orders that differ from the capture order.

Cases that are expected to break a capture (host reads inside a capture, the first engine call of a process inside a
capture) run in a subprocess.  Stale buffers stay allocated: eager buffers are poisoned with 0xFF and kept referenced.

Observed on one H100 80GB HBM3 (700 W power limit): every case bit-identical to eager (the default-mode training
captures within DEFAULT_TOL); about 70 s for the file, 9.5 GiB peak allocated (the configs[1] B = 32 capture matrix).
"""
import contextlib
import copy
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

import glom_pytorch_b200 as G
from glom_pytorch_b200 import _native
from glom_pytorch_b200 import glom as glom_mod

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG1 = (512, 6, 224, 14)


# ----------------------------------------------------------------------------- helpers
def _equal(a, b, what):
    assert a.shape == b.shape, (what, tuple(a.shape), tuple(b.shape))
    if not torch.equal(a, b):
        diff = a != b
        raise AssertionError(f"{what}: {int(diff.sum())} of {a.numel()} elements differ, first at "
                             f"{diff.nonzero()[0].tolist()}")


@contextlib.contextmanager
def _deterministic(on=True):
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def _capture(fn, **kw):
    """-> (graph, fn's outputs captured into it)."""
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, **kw):
        out = fn()
    return g, out


def _glom(dim, L, isz, p, seed=0, **kw):
    import test_production_batch as PB
    return PB._glom(dim, L, isz, p, seed=seed, **kw)


def _images(m, B, seed):
    g = torch.Generator().manual_seed(seed)
    isz = m.image_side
    n = (isz // m.patch_size) ** 2
    return torch.randn(B, 3, isz, isz, generator=g).to(DEV), torch.randn(B, n, m.levels, m.dim, generator=g).to(DEV)


def _spread_tol(r):
    """The tol between two observed changes that gives the images the most distinct stopping steps."""
    import test_settle as ST
    vals = np.unique(r[np.isfinite(r) & (r > 0)])
    best = (0, float(vals[len(vals) // 2]) if len(vals) else 1e-3)
    for a, b in zip(vals[:-1], vals[1:]):
        if b > a * 1.01:
            tol = float(np.sqrt(a * b))
            best = max(best, (len(np.unique(ST._first_stop(r, tol))), tol))
    return best[1]


def _fresh(m):
    """(m, its deepcopy) with empty caches: the deepcopy is the eager reference."""
    assert m._packed is None and not m._scratch and m._resume is None
    return m, copy.deepcopy(m)


# ----------------------------------------------------------------------------- CPU
def _no_host_reads(monkeypatch):
    def refuse(*_a, **_k):
        raise AssertionError("host read")
    monkeypatch.setattr(torch.Tensor, "item", refuse)
    monkeypatch.setattr(torch.Tensor, "tolist", refuse)
    monkeypatch.setattr(torch, "equal", refuse)


@pytest.mark.parametrize("how", ["constructed", "to", "double", "load_state_dict", "deepcopy", "pickle"])
def test_mask_params_need_no_host_read(how, monkeypatch):
    """The radius mask is checked on the host when the buffer is created, moved, loaded or copied, so mask_params (which
    every engine call makes, also under capture) reads nothing; an in-place edit is re-checked on the next call."""
    m = G.Glom(dim=64, levels=2, image_size=32, patch_size=4, local_consensus_radius=2)
    want = m.attention.mask_params(64)
    other = G.Glom(dim=64, levels=2, image_size=32, patch_size=4, local_consensus_radius=2)
    m = {"constructed": lambda: m, "to": lambda: m.to("cpu"), "double": lambda: m.double(),
         "load_state_dict": lambda: (m.load_state_dict(other.state_dict()), m)[1],
         "deepcopy": lambda: copy.deepcopy(m), "pickle": lambda: pickle.loads(pickle.dumps(m))}[how]()
    with monkeypatch.context() as mp:
        _no_host_reads(mp)
        assert m.attention.mask_params(64) == want
    with torch.no_grad():
        m.attention.non_local_mask[0, 0, 1] = ~m.attention.non_local_mask[0, 0, 1]
    with pytest.raises(RuntimeError, match="not a radius mask"):
        m.attention.mask_params(64)
    with torch.no_grad():
        m.attention.non_local_mask[0, 0, 1] = ~m.attention.non_local_mask[0, 0, 1]
    assert m.attention.mask_params(64) == want
    sd = m.state_dict()
    bad = torch.zeros_like(sd["attention.non_local_mask"])
    bad[0, 0, 1] = True
    sd["attention.non_local_mask"] = bad                                  # loads, then raises on use
    m.load_state_dict(sd)
    with pytest.raises(RuntimeError, match="not a radius mask"):
        m.attention.mask_params(64)


def test_host_reads_are_refused_under_capture(monkeypatch):
    """With the current stream capturing, the calls that read the device on the host raise an error that names graph
    capture before they enqueue anything, and the stale-mask check refuses to read the buffer."""
    m = G.Glom(dim=64, levels=2, image_size=32, patch_size=4, local_consensus_radius=2)
    img = torch.randn(2, 3, 32, 32)
    calls = []
    monkeypatch.setattr(glom_mod, "_capturing", lambda: True)
    monkeypatch.setattr(G.Glom, "tokens", lambda *a, **k: calls.append("tokens"))
    for iters in ([1, 2], (3, 1), torch.tensor([1, 2]), torch.tensor([2, 2])):
        with torch.no_grad(), pytest.raises(ValueError, match="graph capture") as e:
            m(img, iters=iters)
        assert "settle(" in str(e.value)
    with torch.no_grad():
        for fn in (lambda: m.settle_queue(img, 1e-3), lambda: m.settle_video(img[None], 1e-3),
                   lambda: m.stage_tokens(img)):
            with pytest.raises(RuntimeError, match="CUDA graph"):
                fn()
    assert not calls
    with torch.no_grad():
        m.attention.non_local_mask[0, 0, 1] = True
    with pytest.raises(RuntimeError, match="CUDA graph"):
        m.attention.mask_params(64)


# ----------------------------------------------------------------------------- GPU: the capture matrix (eval)
MATRIX = {
    "d256_L3_n64": lambda: (_glom(256, 3, 32, 4), 2),
    "configs1_B2": lambda: (_glom(*CFG1), 2),
    "configs1_B32": lambda: (_glom(*CFG1), 32),
    "d128_n256_r2_self": lambda: (_glom(128, 3, 64, 4, local_consensus_radius=2, consensus_self=True), 2),
    "d320_n144_r3": lambda: (_glom(320, 2, 48, 4, local_consensus_radius=3), 3),
    "d384_n100": lambda: (_glom(384, 2, 40, 4), 3),
    "d64_n1600": lambda: (_glom(64, 2, 80, 2), 1),
}


def _matrix_calls(m, x, S, tol, ra_iters):
    """The eval calls of the matrix, each returning tensors; `m` is the captured module or its eager reference."""
    from glom_pytorch_b200.islands import islands
    o1 = m(x, iters=1, levels=S)
    out = {"iters0": m(x, iters=0), "iters0_all": m(x, iters=0, return_all=True),
           "iters1_levels": o1, "iters12": m(x, iters=12),
           "iters12_carried": m(x, iters=12, levels=o1),
           f"iters{ra_iters}_all_levels": m(x, iters=ra_iters, levels=S, return_all=True),
           "tokens": m.tokens(x)}
    out["settle"], out["settle_steps"] = m.settle(x, tol, max_iters=12, levels=S)
    out["settle_all"], out["settle_all_steps"] = m.settle(x, tol, max_iters=ra_iters, levels=S, return_all=True)
    isl = islands(out[f"iters{ra_iters}_all_levels"])
    out.update({f"islands_{k}": v for k, v in isl._asdict().items()})
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(MATRIX))
def test_capture_matrix_eval(name):
    """A fresh module captured with no earlier eager call: forward at iters 0, 1 and 12 with and without return_all, from
    init_levels and from carried levels, settle with and without return_all, tokens and islands of a captured slab; two
    replays with new inputs equal eager calls on the deepcopy."""
    m, B = MATRIX[name]()
    m, ref = _fresh(m)
    x, S = _images(m, B, 1)
    ra_iters = 12 if B * S[0].numel() * 4 * 13 <= (256 << 20) else 1
    with torch.no_grad():
        sample = ref(x[:4], iters=12, levels=S[:4], return_all=True)
        import test_settle as ST
        tol = _spread_tol(ST._change(sample))
        del sample
        g, static = _capture(lambda: _matrix_calls(m, x, S, tol, ra_iters))
        for seed in (2, 3):
            xn, Sn = _images(m, B, seed)
            x.copy_(xn)
            S.copy_(Sn)
            g.replay()
            want = _matrix_calls(ref, xn, Sn.clone(), tol, ra_iters)
            for k in want:
                _equal(static[k], want[k], (name, seed, k))
        print(f"[graphs] {name} B={B}: settle steps {sorted(set(want['settle_steps'].tolist()))}")


@pytest.mark.gpu
def test_capture_fp32_engine_forward():
    import test_forward_oracle as FO
    m, img, S, n = FO._model("d128_n256_r2_self", "fp32")
    m, ref = _fresh(m.eval())
    x, S = img.to(DEV), S.to(DEV)
    with torch.no_grad():
        g, static = _capture(lambda: (m(x, iters=3), m(x, iters=2, levels=S, return_all=True)))
        for seed in (5, 6):
            gen = torch.Generator().manual_seed(seed)
            x.copy_(torch.randn(x.shape, generator=gen))
            S.copy_(torch.randn(S.shape, generator=gen))
            g.replay()
            _equal(static[0], ref(x, iters=3), ("fp32", seed, "iters3"))
            _equal(static[1], ref(x, iters=2, levels=S.clone(), return_all=True), ("fp32", seed, "return_all"))


# ----------------------------------------------------------------------------- GPU: several graphs on one module
@pytest.mark.gpu
@pytest.mark.parametrize("shared_pool", [False, True], ids=["private_pools", "shared_pool"])
def test_several_graphs_replay_in_any_order(shared_pool):
    """Graphs at B = 1, 8, 32 and a second B = 8 graph with other iters, all on the default capture stream: each packs
    the weights itself, so any replay order is right, and after load_state_dict every graph reads the new weights."""
    m, ref = _fresh(_glom(*CFG1))
    specs = {"g1": (1, 12), "g8": (8, 12), "g32": (32, 12), "g8b": (8, 3)}
    static, graphs, pool = {}, {}, None
    with torch.no_grad():
        for k, (B, T) in specs.items():
            static[k] = _images(m, B, 10 + B)[0]
            graphs[k], static[k + "_out"] = _capture(lambda: m(static[k], iters=T), pool=pool)
            if shared_pool and pool is None:
                pool = graphs[k].pool()

        def replay(order, seed):
            for k in order:
                B, T = specs[k]
                static[k].copy_(_images(m, B, seed + B)[0])
                graphs[k].replay()
                _equal(static[k + "_out"], ref(static[k], iters=T), (order, k))
        replay(["g8b"], 20)
        replay(["g8", "g1"], 30)
        replay(["g1", "g32", "g8", "g32"], 40)
        other = _glom(*CFG1, seed=1).state_dict()
        m.load_state_dict(other)
        ref.load_state_dict(other)
        replay(["g32", "g8b", "g1", "g8"], 50)


# ----------------------------------------------------------------------------- GPU: capture-owned buffers
_RANGED = {"pack_weights": (None, 2, 3), "forward": (1, 10, 11), "forward_resume": (1, 9, 10), "settle": (1, 12, 13),
           "forward_steps": (1, 11, 12), "tokenize": (None, 10, 11), "backward": (None, 10, 11),
           "backward_implicit": (None, 12, 13), "tokenize_backward": (None, 11, 12)}


def _record_ranges(monkeypatch):
    """Wrap the _native entry points: -> list of (capturing, lo, hi) of every workspace and packed-weight range."""
    seen = []
    for name, (packed_at, ptr_at, size_at) in _RANGED.items():
        orig = getattr(_native, name)

        def wrap(*a, _orig=orig, _p=packed_at, _w=ptr_at, _s=size_at, _name=name, **k):
            cap = torch.cuda.is_current_stream_capturing()
            if a[_w] is not None:
                seen.append((cap, a[_w], a[_w] + a[_s], _name))
            if _p is not None:
                seen.append((cap, a[_p], a[_p] + _native.packed_weight_bytes(a[0]), _name + ".packed"))
            return _orig(*a, **k)
        monkeypatch.setattr(_native, name, wrap)
    return seen


def _poison_eager(m, sizes, stream):
    """Fill the eager buffers the module holds with 0xFF, and poison the blocks its eager calls freed by allocating and
    filling blocks of their sizes on `stream`; everything stays referenced."""
    keep = [t for t in m._scratch.values() if isinstance(t, torch.Tensor)]
    if m._packed is not None:
        keep.append(m._packed[1])
    with torch.cuda.stream(stream):
        keep += [torch.empty(nb + 1024, dtype=torch.uint8, device=DEV) for nb in sizes]
    for t in keep:
        t.fill_(0xFF)
    return keep


@pytest.mark.gpu
@pytest.mark.parametrize("train", [False, True], ids=["eval", "train"])
def test_capture_after_eager_warmup_owns_its_buffers(train, monkeypatch):
    """Eager calls on stream s, then a capture on s; after it, eager calls on s at the same and a larger batch and on the
    default stream, with every eager buffer poisoned: the replay still equals eager, and no workspace or packed-weight
    range passed inside the capture meets one passed by an eager call."""
    import test_backward_oracle as BO
    m, img, S, n, g = BO._model("tc_config2_dims", "bf16", batch=4)
    m, ref = _fresh(m.train(train))
    seen = _record_ranges(monkeypatch)
    x = img.to(DEV)
    big = torch.randn((8,) + tuple(img.shape[1:]), generator=g).to(DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())

    def step(xx, model):
        if not train:
            return (model(xx, iters=4),)
        out = model(xx, iters=4, return_all=True)
        out[2, :, :, -1].square().mean().backward()
        return (out,) + tuple(p.grad for p in model.parameters())

    with torch.set_grad_enabled(train), _deterministic(True):
        with torch.cuda.stream(s):
            for _ in range(2):
                m.zero_grad(set_to_none=True)
                step(x, m)
        torch.cuda.current_stream().wait_stream(s)
        m.zero_grad(set_to_none=True)
        graph, static = _capture(lambda: step(x, m), stream=s)
        sizes = [nb for cap, lo, hi, _ in seen if not cap for nb in [hi - lo]]
        with torch.cuda.stream(s):
            for xx in (x, big):
                m.zero_grad(set_to_none=True)               # the graph's static gradients stay its own
                step(xx, m)
        torch.cuda.current_stream().wait_stream(s)
        m.zero_grad(set_to_none=True)
        step(x, m)
        torch.cuda.synchronize()
        keep = _poison_eager(m, sorted(set(sizes)), s)
        for seed in (1, 2):
            x.copy_(torch.randn(x.shape, generator=torch.Generator().manual_seed(seed)))
            with torch.cuda.stream(s):
                graph.replay()
            torch.cuda.current_stream().wait_stream(s)
            ref.zero_grad(set_to_none=True)
            for i, (a, b) in enumerate(zip(static, step(x, ref))):
                _equal(a, b, ("replay", train, seed, i))
    del keep
    cap = [(lo, hi, w) for c, lo, hi, w in seen if c]
    eager = [(lo, hi, w) for c, lo, hi, w in seen if not c]
    assert cap and eager
    hits = [(a, b) for a in cap for b in eager if a[0] < b[1] and b[0] < a[1]]
    assert not hits, hits[:4]


# ----------------------------------------------------------------------------- GPU: cross-call state
@pytest.mark.gpu
def test_captured_carried_state_does_not_resume():
    """g2 = m(x2, levels=<g1's output>) is captured without the resume path, so replaying g3 between g1 and g2 changes
    nothing; eager resumed chains after the replays still equal plain calls; a staged frame does not leak into a
    capture."""
    m, ref = _fresh(_glom(256, 3, 32, 4))
    B = 3
    xs = [_images(m, B, s)[0] for s in (1, 2, 3)]
    with torch.no_grad():
        g1, out1 = _capture(lambda: m(xs[0], iters=4))
        g2, out2 = _capture(lambda: m(xs[1], iters=3, levels=out1))
        g3, out3 = _capture(lambda: m(xs[2], iters=4))
        for seed in (4, 5):
            for i, x in enumerate(xs):
                x.copy_(_images(m, B, 10 * seed + i)[0])
            g1.replay()
            g3.replay()
            g2.replay()
            _equal(out1, ref(xs[0], iters=4), "g1")
            _equal(out3, ref(xs[2], iters=4), "g3")
            _equal(out2, ref(xs[1], iters=3, levels=out1.clone()), "g2 after g3")
        a = m(xs[0], iters=4)
        b = m(xs[1], iters=3, levels=a)                   # resumed eagerly
        _equal(b, ref(xs[1], iters=3, levels=a.clone()), "eager resume after replays")
        g3.replay()
        c = m(xs[1], iters=2, levels=b)                   # resumes from b; the replay touched no eager buffer
        _equal(c, ref(xs[1], iters=2, levels=b.clone()), "eager resume across a replay")

        static_x = xs[0].clone()
        m.stage_tokens(static_x)
        g4, out4 = _capture(lambda: m(static_x, iters=2))
        static_x.copy_(xs[2])
        g4.replay()
        _equal(out4, ref(xs[2], iters=2), "capture after stage_tokens")


# ----------------------------------------------------------------------------- GPU: training capture
LOSSES = {
    "bench": lambda m, x: m(x, iters=12, return_all=True)[7, :, :, -1].square().mean(),
    "settle_unrolled": lambda m, x: m.settle(x, 0.05, max_iters=6, differentiable=True, return_all=True)[0][
        :, :, :, -1].square().mean(),
    "settle_implicit": lambda m, x: m.settle(x, 0.05, max_iters=6, differentiable="implicit")[0][:, :, -1].square().mean(),
}


def _train_case(name, loss_fn, graph_deterministic, k=2):
    """Warm-up, capture of loss.backward(); opt.step() with SGD + momentum, k replays; the deepcopy of (model, optimiser)
    taken after the warm-up runs k eager steps under torch.use_deterministic_algorithms.  -> pairs to compare."""
    import test_backward_oracle as BO
    m, img, S, n, g = BO._model(name, "bf16", batch=8 if name == "tc_config2_dims" else None)
    m.train()
    x = img.to(DEV)
    imgs = [torch.randn(x.shape, generator=g).to(DEV) for _ in range(k)]
    opt = torch.optim.SGD(m.parameters(), lr=0.05, momentum=0.9)
    with _deterministic(graph_deterministic):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                opt.zero_grad(set_to_none=True)
                loss_fn(m, x).backward()
                opt.step()
        torch.cuda.current_stream().wait_stream(s)
        ref, ref_opt = copy.deepcopy((m, opt))
        opt.zero_grad(set_to_none=True)

        def step():
            loss = loss_fn(m, x)
            loss.backward()
            opt.step()
            return loss
        graph, loss = _capture(step)
    pairs = []
    for i in range(k):
        x.copy_(imgs[i])
        graph.replay()
        with _deterministic(True):
            ref_opt.zero_grad(set_to_none=True)
            rl = loss_fn(ref, imgs[i])
            rl.backward()
            ref_opt.step()
        pairs.append((f"loss{i}", loss.clone(), rl))
    for (pn, p), q in zip(m.named_parameters(), ref.parameters()):
        pairs += [(pn, p, q)]
        if q.grad is None:                      # settle(differentiable="implicit"): no gradient for init_levels
            assert p.grad is None and "momentum_buffer" not in opt.state[p], pn
            continue
        pairs += [(pn + ".grad", p.grad, q.grad),
                  (pn + ".momentum", opt.state[p]["momentum_buffer"], ref_opt.state[q]["momentum_buffer"])]
    if m.last_adjoint is not None:
        pairs += [("adjoint_steps", m.last_adjoint[0], ref.last_adjoint[0]), ("adjoint_q", m.last_adjoint[1],
                                                                               ref.last_adjoint[1])]
    return pairs


@pytest.mark.gpu
@pytest.mark.parametrize("loss", sorted(LOSSES))
@pytest.mark.parametrize("name", ["tc_config2_dims", "mixed_d256_n100", "simt_d192_n144_mask_self"])
def test_training_step_capture_deterministic(name, loss):
    """Under torch.use_deterministic_algorithms, k replays of a captured training step leave the parameters, gradients,
    momentum buffers (and the implicit adjoint's steps and ratios) bit-identical to k eager steps."""
    for what, a, b in _train_case(name, LOSSES[loss], True):
        _equal(a.detach(), b.detach(), (name, loss, what))


@pytest.mark.gpu
@pytest.mark.parametrize("loss", sorted(LOSSES))
def test_training_step_capture_default_mode(loss):
    """The default (atomic) backward captured: within test_production_batch.DEFAULT_TOL of the deterministic eager run."""
    from test_production_batch import DEFAULT_TOL
    _, ab = DEFAULT_TOL
    for what, a, b in _train_case("mixed_d256_n100", LOSSES[loss], False):
        if what.startswith("adjoint"):          # the adjoint's stopping decisions may move with the atomics' bits
            continue
        a, b = a.detach().double(), b.detach().double()
        err = (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)
        assert err <= ab, (loss, what, err)


@pytest.mark.gpu
def test_make_graphed_callables_training():
    """torch.cuda.make_graphed_callables(model, (img,)) in train mode, deterministic: one memory pool for the forward
    and backward graphs; outputs and gradients of 3 calls equal eager."""
    import test_backward_oracle as BO
    m, img, S, n, g = BO._model("mixed_d256_n100", "bf16")
    m, ref = _fresh(m.train())
    x = img.to(DEV)
    with _deterministic(True):
        gm = torch.cuda.make_graphed_callables(m, (x,))
        for i in range(3):
            xi = torch.randn(x.shape, generator=g).to(DEV)
            m.zero_grad(set_to_none=True)           # the graphed backward returns its static gradient buffers
            ref.zero_grad(set_to_none=True)
            out = gm(xi)
            want = ref(xi)
            _equal(out.detach(), want.detach(), ("output", i))
            out[:, :, -1].square().mean().backward()
            want[:, :, -1].square().mean().backward()
            for (pn, p), q in zip(m.named_parameters(), ref.parameters()):
                _equal(p.grad, q.grad, ("grad", i, pn))


# ----------------------------------------------------------------------------- GPU: concurrent streams
@pytest.mark.gpu
def test_concurrent_streams_eager_and_graphs():
    """One module issues forwards and settles at different batches on two streams with no synchronisation until a final
    join: equal to the sequential results.  Two graphs captured on two streams and replayed concurrently equal eager."""
    m, ref = _fresh(_glom(256, 3, 32, 4))
    (xa, Sa), (xb, Sb) = _images(m, 5, 1), _images(m, 2, 2)
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.no_grad():
        want = [ref(xa, iters=6), ref.settle(xb, 1e-2, max_iters=6, levels=Sb), ref(xb, iters=3, levels=Sb),
                ref.settle(xa, 1e-2, max_iters=8, levels=Sa)]
        for st in (sa, sb):
            st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(sa):
            r0 = m(xa, iters=6)
        with torch.cuda.stream(sb):
            r2 = m(xb, iters=3, levels=Sb)
        with torch.cuda.stream(sa):
            r1 = m.settle(xb, 1e-2, max_iters=6, levels=Sb)
        with torch.cuda.stream(sb):
            r3 = m.settle(xa, 1e-2, max_iters=8, levels=Sa)
        got = [r0, r1, r2, r3]
        for st in (sa, sb):
            torch.cuda.current_stream().wait_stream(st)
        for i, (a, b) in enumerate(zip(got, want)):
            for u, v in zip(a if isinstance(a, tuple) else (a,), b if isinstance(b, tuple) else (b,)):
                _equal(u, v, ("streams", i))

        m2, ref2 = _fresh(_glom(256, 3, 32, 4, seed=3))
        ga, oa = _capture(lambda: m2(xa, iters=5), stream=sa)
        gb, ob = _capture(lambda: m2.settle(xb, 1e-2, max_iters=7, levels=Sb), stream=sb)
        xa.copy_(_images(m, 5, 7)[0])
        xb.copy_(_images(m, 2, 8)[0])
        for st in (sa, sb):
            st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(sa):
            ga.replay()
        with torch.cuda.stream(sb):
            gb.replay()
        for st in (sa, sb):
            torch.cuda.current_stream().wait_stream(st)
        _equal(oa, ref2(xa, iters=5), "concurrent graph a")
        wl, ws = ref2.settle(xb, 1e-2, max_iters=7, levels=Sb)
        _equal(ob[0], wl, "concurrent graph b levels")
        _equal(ob[1], ws, "concurrent graph b steps")


# ----------------------------------------------------------------------------- GPU: in a process of their own
def _run_in_subprocess(fn_name, tmp_path):
    script = tmp_path / "case.py"
    script.write_text(
        "import json, os, sys\n"
        "for sub in ('', 'tests', 'tests/golden'):\n"
        "    sys.path.insert(0, os.path.join(sys.argv[2], sub))\n"
        "import test_cuda_graphs as T\n"
        "print('RESULT ' + json.dumps(getattr(T, sys.argv[1])()))\n")
    r = subprocess.run([sys.executable, str(script), fn_name, ROOT], capture_output=True, text=True, timeout=600,
                       cwd=ROOT)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")]
    assert r.returncode == 0 and lines, r.stdout[-4000:] + r.stderr[-4000:]
    return json.loads(lines[-1][len("RESULT "):])


def _first_call(kind):
    """The process's first engine call is made inside a capture; the replay must equal an eager run made afterwards."""
    if kind == "mask":
        m = _glom(128, 3, 64, 4, local_consensus_radius=2, consensus_self=True)
    else:
        m = _glom(*CFG1)
    ref = copy.deepcopy(m)
    x = _images(m, 2, 1)[0]
    if kind == "train":
        m.train()
        ref.train()

        def step(model, xx):
            model(xx, iters=3, return_all=True)[2, :, :, -1].square().mean().backward()
            return [p.grad for p in model.parameters()]
        with _deterministic(True):
            g, static = _capture(lambda: step(m, x))
            x.copy_(_images(m, 2, 2)[0])
            g.replay()
            want = step(ref, x)
    else:
        with torch.no_grad():
            g, static = _capture(lambda: [m(x, iters=4)])
            x.copy_(_images(m, 2, 2)[0])
            g.replay()
            want = [ref(x, iters=4)]
    return [bool(torch.equal(a, b)) for a, b in zip(static, want)]


def first_call_forward():
    return _first_call("forward")


def first_call_mask():
    return _first_call("mask")


def first_call_train():
    return _first_call("train")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["forward", "mask", "train"])
def test_first_engine_call_of_a_process_inside_a_capture(kind, tmp_path):
    """The lazy one-time work (device queries, the tensor-map encoder, occupancy and shared-memory opt-in, module
    loading) and a fresh radius-mask model's mask check all work when the first call is captured."""
    eq = _run_in_subprocess(f"first_call_{kind}", tmp_path)
    assert eq and all(eq), eq


def host_read_guards():
    """Inside a live capture each host-reading call raises an error naming graph capture; the capture then continues
    with a valid call, and its replay equals eager."""
    m = _glom(128, 3, 32, 4)
    ref = copy.deepcopy(m)
    x = _images(m, 2, 1)[0]
    frames = x[None]
    cpu_vec, cuda_vec, cuda_scalar = torch.tensor([1, 2]), torch.tensor([1, 2], device=DEV), torch.tensor(2, device=DEV)
    cases = {"iters_list": lambda: m(x, iters=[1, 2]), "iters_cpu_vector": lambda: m(x, iters=cpu_vec),
             "iters_cuda_vector": lambda: m(x, iters=cuda_vec), "iters_cuda_scalar": lambda: m(x, iters=cuda_scalar),
             "settle_queue": lambda: m.settle_queue(x, 1e-3), "settle_video": lambda: m.settle_video(frames, 1e-3),
             "stage_tokens": lambda: m.stage_tokens(x)}
    out = {}
    for name, fn in cases.items():
        res = {"error": None, "equal": False}
        try:
            with torch.no_grad():
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    try:
                        fn()
                    except (ValueError, RuntimeError) as e:
                        res["error"] = f"{type(e).__name__}: {e}"
                    y = m(x, iters=2)
                x.copy_(_images(m, 2, 3)[0])
                g.replay()
                res["equal"] = bool(torch.equal(y, ref(x, iters=2)))
        except Exception as e:                                  # a capture the call invalidated
            res["capture"] = f"{type(e).__name__}: {e}"[:300]
        out[name] = res
    return out


@pytest.mark.gpu
def test_host_reads_under_capture_raise_and_leave_the_capture_intact(tmp_path):
    res = _run_in_subprocess("host_read_guards", tmp_path)
    for name, r in res.items():
        assert r["error"] and "graph" in r["error"] and "capture" in r["error"], (name, r)
        assert "capture" not in r and r["equal"], (name, r)
    assert "settle(" in res["iters_cuda_vector"]["error"]
