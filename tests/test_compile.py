"""Glom under torch.compile and torch.export: the engine as glom_b200 custom ops (glom_pytorch_b200/ops.py).

CPU: the ops and their schemas, the fake implementations' shapes on fake CUDA tensors, and exported graphs of forward,
settle(differentiable=True) and a loss-plus-backward step that call glom_b200 ops and aten view ops only.

GPU: everything compiled or exported is bit for bit equal to eager calls on ``copy.deepcopy`` of the module (training
under the default atomic reductions: within the backward oracle's tolerance), with no graph break where the op path
promises none; the host loops run eagerly behind a graph break; an in-place edit of the radius mask after compiling
raises; eager calls never reach a glom_b200 op.
"""
import copy
import io

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode
from torch.utils._python_dispatch import TorchDispatchMode

import glom_pytorch_b200 as G

DEV = "cuda:0"
CFG1 = (512, 6, 224, 14)

SCHEMAS = {
    "tokenize": "glom_b200::tokenize(Tensor img, Tensor weight, Tensor bias, SymInt patch, str precision) -> Tensor",
    "tokenize_backward": "glom_b200::tokenize_backward(Tensor img, Tensor weight, Tensor d_tokens, SymInt patch, "
                         "bool need_img, bool need_weight, bool need_bias, bool deterministic) -> (Tensor, Tensor, "
                         "Tensor)",
    "column_update": "glom_b200::column_update(Tensor tokens, Tensor pos, Tensor? state0, Tensor init_levels, "
                     "Tensor bu_w1, Tensor bu_b1, Tensor bu_w2, Tensor bu_b2, Tensor td_w1, Tensor td_b1, "
                     "Tensor td_w2, Tensor td_b2, Tensor? steps, bool attend_self, SymInt mask_side, "
                     "SymInt mask_d2_max, Tensor? mask_checked, str precision, SymInt iters, bool return_all, "
                     "bool keep_states) -> Tensor",
    "settle": "glom_b200::settle(Tensor tokens, Tensor pos, Tensor? state0, Tensor init_levels, Tensor bu_w1, "
              "Tensor bu_b1, Tensor bu_w2, Tensor bu_b2, Tensor td_w1, Tensor td_b1, Tensor td_w2, Tensor td_b2, "
              "bool attend_self, SymInt mask_side, SymInt mask_d2_max, Tensor? mask_checked, float tol, "
              "SymInt max_iters, bool return_all, bool keep_states) -> (Tensor, Tensor)",
    "check_radius_mask": "glom_b200::check_radius_mask(Tensor mask, SymInt mask_side, SymInt mask_d2_max) -> Tensor",
    "column_update_backward": "glom_b200::column_update_backward(Tensor tokens, Tensor pos, Tensor states, "
                              "Tensor grad_out, Tensor bu_w1, Tensor bu_b1, Tensor bu_w2, Tensor bu_b2, Tensor td_w1, "
                              "Tensor td_b1, Tensor td_w2, Tensor td_b2, Tensor? steps, bool attend_self, "
                              "SymInt mask_side, SymInt mask_d2_max, str precision, SymInt iters, bool grad_all, "
                              "bool has_state0, bool deterministic) -> Tensor[]",
    "islands": "glom_b200::islands(Tensor states, SymInt side_h, SymInt side_w, float threshold) -> (Tensor, Tensor, "
               "Tensor, Tensor, Tensor)",
}

# (dim, levels, image (h, w), patch, Glom kwargs): configs[0], configs[1], a radius mask with self, a non-square image,
# the fp32 engine
FAKE_SHAPES = {
    "configs0": (64, 3, (28, 28), 7, {}),
    "configs1": (512, 6, (224, 224), 14, {}),
    "radius_self": (128, 3, (64, 64), 4, dict(local_consensus_radius=2, consensus_self=True)),
    "nonsquare": (256, 3, (16, 32), 4, dict(image_size=32)),
    "fp32": (128, 3, (64, 64), 4, dict(precision="fp32")),
}
VIEW_OPS = {"aten.slice.Tensor", "aten.select.int", "aten.view.default", "aten.alias.default", "aten.detach.default",
            "<built-in function getitem>"}


def test_ops_are_registered_with_their_schemas():
    for name, schema in SCHEMAS.items():
        assert str(getattr(torch.ops.glom_b200, name).default._schema) == schema, name
    # the mask check stays out of CUDA graphs recorded by mode="reduce-overhead", so it runs on every call
    assert torch.Tag.cudagraph_unsafe in torch.ops.glom_b200.check_radius_mask.default.tags


def test_ops_refuse_tensors_off_cuda():
    """The ops check their arguments on the host before any pointer reaches the library."""
    m = G.Glom(dim=64, levels=3, image_size=28, patch_size=7)
    img = torch.randn(2, 3, 28, 28)
    lin = m.image_to_tokens[1]
    with pytest.raises(ValueError, match="CUDA device"):
        torch.ops.glom_b200.tokenize(img, lin.weight, lin.bias, 7, "bf16")
    tokens = torch.randn(2, 16, 64)
    with pytest.raises(ValueError, match="CUDA device"):
        torch.ops.glom_b200.column_update(tokens, m.pos_emb.weight[:16], None, m.init_levels, *m._mlp_params(), None,
                                          False, 0, 0, None, "bf16", 2, False, False)


def _fake_model(name, mode):
    dim, L, (h, w), p, kw = FAKE_SHAPES[name]
    kw = dict(kw)
    isz = kw.pop("image_size", h)
    m = G.Glom(dim=dim, levels=L, image_size=isz, patch_size=p, **kw)
    with mode:
        m = m.to(DEV)
        img = torch.randn(2, 3, h, w, device=DEV)
    return m, img, (h // p) * (w // p)


@pytest.mark.parametrize("name", sorted(FAKE_SHAPES))
def test_fake_shapes_match_the_eager_api(name, monkeypatch):
    """Under FakeTensorMode with fake CUDA tensors, the op path (what torch.compile / torch.export trace) gives the
    shapes, dtypes and device the eager API returns, and gradients shaped like their parameters."""
    mode = FakeTensorMode(allow_non_fake_inputs=True)
    m, img, n = _fake_model(name, mode)
    B, L, d = img.shape[0], m.levels, m.dim
    monkeypatch.setattr(torch.compiler, "is_compiling", lambda: True)

    def check(t, shape, dtype=torch.float32):
        assert tuple(t.shape) == shape and t.dtype == dtype and t.device == torch.device(DEV), (t.shape, t.dtype)
    with mode:
        with torch.no_grad():
            for iters in (0, 1, 12):
                check(m(img, iters=iters), (B, n, L, d))
                check(m(img, iters=iters, return_all=True), (iters + 1, B, n, L, d))
            check(m.tokens(img), (B, n, d))
            states = m(img, iters=2, return_all=True)
            isl = G.islands(states, grid=(img.shape[2] // m.patch_size, img.shape[3] // m.patch_size))
            for k in ("cos_right", "cos_down", "agreement"):
                check(getattr(isl, k), (3, B, L, n))
            check(isl.labels, (3, B, L, n), torch.int32)
            check(isl.num_islands, (3, B, L), torch.int32)
            if m.precision == "bf16":
                lv, steps = m.settle(img, 1e-3, max_iters=5)
                check(lv, (B, n, L, d))
                check(steps, (B,), torch.int32)
                lv, steps = m.settle(img, 1e-3, max_iters=5, return_all=True)
                check(lv, (6, B, n, L, d))
                check(steps, (B,), torch.int32)
        # the backward ops (the autograd engine itself needs a device, so they are called as the formulas call them)
        lin = m.image_to_tokens[1]
        d_i, d_w, d_b = torch.ops.glom_b200.tokenize_backward(img, lin.weight, m.tokens(img), m.patch_size, True, True,
                                                              True, False)
        check(d_i, tuple(img.shape))
        check(d_w, tuple(lin.weight.shape))
        check(d_b, tuple(lin.bias.shape))
        side, d2, mask = m.attention._op_mask_args(n)
        checked = None if mask is None else torch.ops.glom_b200.check_radius_mask(mask, side, d2)
        if mask is not None:
            check(checked, (0,), torch.bool)
        args = (m.tokens(img), m.pos_emb.weight[:n])
        weights = m._mlp_params()
        for state0, steps in ((None, None), (torch.randn(B, n, L, d, device=DEV), None),
                              (None, torch.ones(B, dtype=torch.int32, device=DEV))):
            if steps is not None and m.precision != "bf16":
                continue
            states = torch.ops.glom_b200.column_update(*args, state0, m.init_levels, *weights, steps,
                                                      m.attention.attend_self, side, d2, checked, m.precision, 4,
                                                      False,
                                                      True)
            check(states, (5, B, n, L, d))
            for grad_all in (False, True):
                g = torch.ops.glom_b200.column_update_backward(
                    *args, states, states if grad_all else states[4], *weights, steps, m.attention.attend_self, side,
                    d2, m.precision, 4, grad_all, state0 is not None, True)
                want = [args[0].shape, args[1].shape, (B, n, L, d) if state0 is not None else (0,),
                        (0,) if state0 is not None else (L, d)] + [w.shape for w in weights]
                assert len(g) == 12
                for t, shape in zip(g, want):
                    check(t, tuple(shape))


def _targets(gm):
    return {str(nd.target) for nd in gm.graph.nodes if nd.op == "call_function"}


def _export(m, fn, img):
    class Call(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.m = m

        def forward(self, x):
            return fn(self.m, x)
    return torch.export.export(Call(), (img,))


@pytest.mark.parametrize("name", ["configs1", "radius_self"])
def test_exported_graphs_call_engine_ops_and_views_only(name):
    """torch.export of forward (with and without autograd), settle(differentiable=True) and islands on fake CUDA inputs:
    one graph (export has no graph breaks) of glom_b200 ops and aten view / slice ops only.  (The loss-plus-backward
    trace needs the autograd engine, which needs a device: test_loss_and_backward_trace_reaches_the_backward_ops.)"""
    mode = FakeTensorMode(allow_non_fake_inputs=True)
    m, img, n = _fake_model(name, mode)
    calls = {
        "forward": lambda mm, x: mm(x, iters=12, return_all=True),
        "forward_last": lambda mm, x: mm(x, iters=12),
        "settle_differentiable": lambda mm, x: mm.settle(x, 1e-3, max_iters=6, differentiable=True),
        "islands": lambda mm, x: tuple(G.islands(mm(x, iters=2, return_all=True))),
    }
    with mode:
        for what, fn in calls.items():
            for grad in (False, True):
                with torch.set_grad_enabled(grad):
                    ep = _export(m, fn, img)
                ts = _targets(ep.graph_module)
                engine = {t for t in ts if t.startswith("glom_b200.")}
                assert engine and ts - engine <= VIEW_OPS, (what, grad, ts)


# ----------------------------------------------------------------------------- GPU helpers
def _equal(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape, a.dtype, b.dtype)
    if not torch.equal(a, b):
        diff = a != b
        raise AssertionError(f"{what}: {int(diff.sum())} of {a.numel()} elements differ, first at "
                             f"{diff.nonzero()[0].tolist()}")


def _flat(x):
    if isinstance(x, torch.Tensor):
        return [x]
    return [t for v in x for t in _flat(v)]


def _equal_all(a, b, what):
    a, b = _flat(a), _flat(b)
    assert len(a) == len(b), what
    for i, (u, v) in enumerate(zip(a, b)):
        _equal(u.detach(), v.detach(), (what, i))


class _EngineOpCounter(TorchDispatchMode):
    """Counts the glom_b200 ops dispatched while it is active."""

    def __init__(self):
        super().__init__()
        self.calls = []

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        if func.namespace == "glom_b200":
            self.calls.append(func.name())
        return func(*args, **(kwargs or {}))


def _glom(dim, L, isz, p, seed=0, **kw):
    import test_production_batch as PB
    return PB._glom(dim, L, isz, p, seed=seed, **kw)


def _images(m, B, seed):
    import test_cuda_graphs as CG
    return CG._images(m, B, seed)


def _compile(m, **kw):
    torch._dynamo.reset()
    return torch.compile(m, fullgraph=True, **kw)


def _breaks(fn, *args, **kw):
    return torch._dynamo.explain(fn)(*args, **kw).graph_break_count


def _eval_calls(m, x, S, tol):
    from glom_pytorch_b200.islands import islands
    o1 = m(x, iters=1, levels=S)
    out = {"iters_none": m(x), "iters0": m(x, iters=0), "iters0_all": m(x, iters=0, return_all=True), "iters1": o1,
           "iters12": m(x, iters=12), "iters12_carried": m(x, iters=12, levels=o1),
           "iters3_all": m(x, iters=3, levels=S, return_all=True), "tokens": m.tokens(x),
           "settle": m.settle(x, tol, max_iters=12, levels=S),
           "settle_all": m.settle(x, tol, max_iters=3, levels=S, return_all=True)}
    out["islands"] = tuple(islands(out["iters3_all"]))
    return out


MATRIX = {
    "configs1_B32": lambda: (_glom(*CFG1), 32),
    "d320_n144_r3": lambda: (_glom(320, 2, 48, 4, local_consensus_radius=3), 5),
    "d128_n256_r2_self": lambda: (_glom(128, 3, 64, 4, local_consensus_radius=2, consensus_self=True), 2),
    "d384_n100_ragged": lambda: (_glom(384, 2, 40, 4), 3),
    "d256_n576_key_blocks": lambda: (_glom(256, 2, 96, 4, local_consensus_radius=2.5), 1),
}


# ----------------------------------------------------------------------------- GPU: opcheck
@pytest.mark.gpu
def test_opcheck_every_op():
    """torch.library.opcheck at small oracle shapes: schema, fake implementation, autograd registration, AOT dispatch."""
    m = _glom(64, 3, 28, 7, local_consensus_radius=1, consensus_self=True).train()
    x, S = _images(m, 2, 1)
    lin = m.image_to_tokens[1]
    w = [p.detach().clone().requires_grad_(True) for p in m._mlp_params()]
    side, d2, mask = m.attention._op_mask_args(16)
    tok = torch.ops.glom_b200.tokenize(x, lin.weight.detach(), lin.bias.detach(), 7, "bf16")
    tok = tok.detach().requires_grad_(True)
    pos = m.pos_emb.weight.detach()[:16].clone().requires_grad_(True)
    init = m.init_levels.detach().clone().requires_grad_(True)
    cfg = (True, side, d2, torch.ops.glom_b200.check_radius_mask(mask, side, d2))
    states = torch.ops.glom_b200.column_update(tok, pos, None, init, *w, None, *cfg, "bf16", 3, False, True).detach()
    steps = torch.tensor([1, 3], dtype=torch.int32, device=DEV)
    cases = [
        (torch.ops.glom_b200.tokenize, (x.clone().requires_grad_(True), lin.weight.detach().clone().requires_grad_(True),
                                        lin.bias.detach().clone().requires_grad_(True), 7, "bf16")),
        (torch.ops.glom_b200.tokenize_backward, (x, lin.weight.detach(), torch.randn_like(tok), 7, True, True, True,
                                                 True)),
        (torch.ops.glom_b200.column_update, (tok, pos, None, init, *w, None, *cfg, "bf16", 3, True, True)),
        (torch.ops.glom_b200.column_update, (tok, pos, S.clone().requires_grad_(True), init, *w, steps, *cfg, "bf16",
                                             3, False, True)),
        (torch.ops.glom_b200.column_update, (tok.detach(), pos.detach(), None, init.detach(), *[t.detach() for t in w],
                                             None, *cfg, "bf16", 2, False, False)),
        (torch.ops.glom_b200.settle, (tok, pos, S, init, *w, *cfg, 1e-2, 4, False, True)),
        (torch.ops.glom_b200.column_update_backward, (tok.detach(), pos.detach(), states, torch.randn_like(states),
                                                      *[t.detach() for t in w], None, True, side, d2, "bf16", 3, True,
                                                      False, True)),
        (torch.ops.glom_b200.islands, (states, 4, 4, 0.9)),
        (torch.ops.glom_b200.check_radius_mask, (mask, side, d2)),
    ]
    for op, args in cases:
        torch.library.opcheck(op, args, test_utils=("test_schema", "test_faketensor", "test_autograd_registration",
                                                    "test_aot_dispatch_dynamic"))


@pytest.mark.gpu
def test_loss_and_backward_trace_reaches_the_backward_ops():
    """make_fx(tracing_mode="fake") of a loss-plus-backward step through the exported forward: one graph whose engine
    work is the four glom_b200 ops, forward and backward."""
    from torch.fx.experimental.proxy_tensor import make_fx
    m = _glom(*CFG1).train()
    x = _images(m, 2, 1)[0]
    ep = _export(m, lambda mm, xx: mm(xx, iters=12, return_all=True), x)
    params = list(m.parameters())

    def step(xx):
        loss = ep.module()(xx)[7, :, :, -1].square().mean()
        return torch.autograd.grad(loss, params + [xx])
    ts = _targets(make_fx(step, tracing_mode="fake", _allow_non_fake_inputs=True)(x.clone().requires_grad_(True)))
    engine = {t for t in ts if t.startswith("glom_b200.")}
    assert engine == {f"glom_b200.{op}.default" for op in ("tokenize", "column_update", "column_update_backward",
                                                           "tokenize_backward")}, ts


# ----------------------------------------------------------------------------- GPU: eval calls compiled
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(MATRIX))
def test_compiled_eval_calls_are_eager_bits(name):
    """forward (iters None / 0 / 1 / 12, return_all, carried levels), tokens, settle with and without return_all and
    islands, each compiled with fullgraph=True and free of graph breaks: bit-identical to eager on a deepcopy."""
    import test_cuda_graphs as CG
    m, B = MATRIX[name]()
    ref = copy.deepcopy(m)
    x, S = _images(m, B, 1)
    with torch.no_grad():
        import test_settle as ST
        tol = CG._spread_tol(ST._change(ref(x[:4], iters=12, levels=S[:4], return_all=True)))
        want = _eval_calls(ref, x, S, tol)
        torch._dynamo.reset()
        fn = torch.compile(lambda xx, SS: _eval_calls(m, xx, SS, tol), fullgraph=True)
        for seed in (1, 2):
            if seed == 2:
                x, S = _images(m, B, seed)
                want = _eval_calls(ref, x, S, tol)
            got = fn(x, S)
            for k in want:
                _equal_all(got[k], want[k], (name, seed, k))
        torch._dynamo.reset()
        assert _breaks(lambda xx, SS: _eval_calls(m, xx, SS, tol), x, S) == 0


@pytest.mark.gpu
def test_compiled_fp32_engine_is_eager_bits():
    import test_forward_oracle as FO
    m, img, S, n = FO._model("d128_n256_r2_self", "fp32")
    m = m.eval()
    ref = copy.deepcopy(m)
    x, S = img.to(DEV), S.to(DEV)
    cm = _compile(m)
    with torch.no_grad():
        for kw in (dict(iters=3), dict(iters=2, levels=S, return_all=True), dict(iters=0)):
            _equal(cm(x, **kw), ref(x, **kw), ("fp32", kw))
        _equal(torch.compile(m.tokens, fullgraph=True)(x), ref.tokens(x), "fp32 tokens")
        assert _breaks(m, x, iters=3) == 0


# ----------------------------------------------------------------------------- GPU: training
LOSSES = {
    # exact cotangents (a fixed weight c on one slab or on the result): the backward ops see eager's bits
    "forward_all": lambda m, x, c, S: (m(x, iters=12, return_all=True)[7, :, :, -1] * c).sum(),
    "forward_carried": lambda m, x, c, S: (m(x, iters=3, levels=S)[:, :, -1] * c).sum(),
    "settle_differentiable": lambda m, x, c, S: (m.settle(x, 0.05, max_iters=6, differentiable=True)[0][:, :, -1]
                                                 * c).sum(),
    "settle_differentiable_all": lambda m, x, c, S: (m.settle(x, 0.05, max_iters=6, differentiable=True,
                                                              return_all=True)[0][4, :, :, -1] * c).sum(),
}


def _train_model(name="mixed_d256_n100"):
    """-> (model in train mode, image, cotangent weight c, carried state S that requires grad, generator)."""
    import test_backward_oracle as BO
    m, img, S, n, g = BO._model(name, "bf16")
    c = torch.randn(img.shape[0], n, m.dim, generator=g).to(DEV)
    return m.train(), img.to(DEV), c, S.to(DEV).requires_grad_(True), g


def _train_steps(m, step_fn, xs, c, S, deterministic, k=2):
    """k steps of step_fn's loss, backward and SGD with momentum -> [(name, tensor)] to compare."""
    import test_cuda_graphs as CG
    opt = torch.optim.SGD(m.parameters(), lr=0.05, momentum=0.9)
    out = []
    with CG._deterministic(deterministic):
        for i in range(k):
            opt.zero_grad(set_to_none=True)
            S.grad = None
            loss = step_fn(m, xs[i], c, S)
            loss.backward()
            out.append((f"loss{i}", loss.detach().clone()))
            out += [(pn + f".grad{i}", p.grad.clone()) for pn, p in m.named_parameters() if p.grad is not None]
            if S.grad is not None:
                out.append((f"levels.grad{i}", S.grad.clone()))
            opt.step()
    return out + [(pn, p.detach().clone()) for pn, p in m.named_parameters()]


@pytest.mark.gpu
@pytest.mark.parametrize("loss", sorted(LOSSES))
@pytest.mark.parametrize("deterministic", [True, False], ids=["deterministic", "default"])
def test_compiled_training_step(loss, deterministic):
    """A compiled forward + loss, loss.backward() and an SGD step, twice: bit-identical to eager under
    torch.use_deterministic_algorithms, within the backward oracle's tolerance under the default atomic reductions."""
    import test_backward_oracle as BO
    m, x, c, S, g = _train_model()
    ref = copy.deepcopy(m)
    xs = [x, torch.randn(x.shape, generator=g).to(DEV)]
    torch._dynamo.reset()
    compiled = torch.compile(LOSSES[loss], fullgraph=True)
    got = _train_steps(m, compiled, xs, c, S, deterministic)
    want = _train_steps(ref, LOSSES[loss], xs, c, S, True)
    assert [k for k, _ in got] == [k for k, _ in want]
    _, rel = BO.TOL["tc"]
    for (k, a), (_, b) in zip(got, want):
        if deterministic and k.startswith("loss"):   # the loss's own sum is inductor's reduction, not the engine's
            assert torch.allclose(a, b, rtol=1e-5, atol=0), (loss, k, a, b)
        elif deterministic:
            _equal(a, b, (loss, k))
        else:
            err = (a.double() - b.double()).abs().max().item() / max(b.abs().max().item(), 1e-30)
            assert err <= rel, (loss, k, err)
    torch._dynamo.reset()
    assert _breaks(LOSSES[loss], m, x, c, S) == 0


@pytest.mark.gpu
def test_deterministic_flag_toggled_between_calls_of_one_compiled_step(monkeypatch):
    """One compiled step called with the flag off, on, off, on: every call's backwards are launched in that call's mode
    (the flag is part of dynamo's global-state guard, so a toggle recompiles rather than replaying the other mode), and
    each deterministic call's gradients are the eager deterministic bits."""
    import test_cuda_graphs as CG
    from glom_pytorch_b200 import _native
    seen = []
    for name in ("backward", "tokenize_backward"):
        orig = getattr(_native, name)

        def wrap(*a, _orig=orig, _name=name, **k):
            seen.append((_name, bool(k.get("deterministic", False))))
            return _orig(*a, **k)
        monkeypatch.setattr(_native, name, wrap)
    m, x, c, S, g = _train_model()
    ref = copy.deepcopy(m)
    torch._dynamo.reset()
    compiled = torch.compile(LOSSES["forward_all"], fullgraph=True)
    for mode in (False, True, False, True):
        with CG._deterministic(mode):
            m.zero_grad(set_to_none=True)
            seen.clear()
            compiled(m, x, c, S).backward()
            assert sorted(seen) == [("backward", mode), ("tokenize_backward", mode)], (mode, seen)
            if mode:
                ref.zero_grad(set_to_none=True)
                LOSSES["forward_all"](ref, x, c, S).backward()
                for (pn, p), q in zip(m.named_parameters(), ref.parameters()):
                    _equal(p.grad, q.grad, ("deterministic", pn))


# ----------------------------------------------------------------------------- GPU: cudagraph trees, dynamic, export
@pytest.mark.gpu
def test_reduce_overhead_reads_new_weights():
    """mode="reduce-overhead": repeated calls equal eager; after an optimiser step and after load_state_dict the next
    call reads the new weights."""
    m = _glom(256, 3, 32, 4)
    ref = copy.deepcopy(m)
    cm = _compile(m, mode="reduce-overhead")
    with torch.no_grad():
        for seed in range(4):
            x = _images(m, 4, seed)[0]
            _equal(cm(x, iters=6).clone(), ref(x, iters=6), ("replay", seed))
        opt, ref_opt = (torch.optim.SGD(mm.parameters(), lr=0.1) for mm in (m, ref))
        for mm, o in ((m, opt), (ref, ref_opt)):
            for p in mm.parameters():
                p.grad = torch.full_like(p, 0.01)
            o.step()
        x = _images(m, 4, 9)[0]
        _equal(cm(x, iters=6).clone(), ref(x, iters=6), "after optimiser step")
        other = _glom(256, 3, 32, 4, seed=3).state_dict()
        m.load_state_dict(other)
        ref.load_state_dict(other)
        _equal(cm(x, iters=6).clone(), ref(x, iters=6), "after load_state_dict")


@pytest.mark.gpu
def test_dynamic_batch_does_not_recompile():
    m = _glom(256, 3, 32, 4)
    ref = copy.deepcopy(m)
    counts = torch._dynamo.utils.counters
    cm = _compile(m, dynamic=True)
    with torch.no_grad():
        frames = []
        for B in (2, 3, 5):
            x = _images(m, B, B)[0]
            _equal(cm(x, iters=5, return_all=True), ref(x, iters=5, return_all=True), ("dynamic", B))
            frames.append(counts["stats"]["unique_graphs"])
    assert frames[0] == frames[1] == frames[2], frames


@pytest.mark.gpu
def test_export_and_save_load_round_trip():
    m = _glom(*CFG1)
    ref = copy.deepcopy(m)
    x = _images(m, 4, 1)[0]
    with torch.no_grad():
        ep = torch.export.export(m, (x,), {"iters": 12})
        want = ref(x, iters=12)
        _equal(ep.module()(x, iters=12), want, "export")
        buf = io.BytesIO()
        torch.export.save(ep, buf)
        buf.seek(0)
        loaded = torch.export.load(buf)
        _equal(loaded.module()(x, iters=12), want, "export save / load")


# ----------------------------------------------------------------------------- GPU: eager behind a graph break
@pytest.mark.gpu
def test_host_loops_and_implicit_settle_run_eagerly_under_compile():
    """settle_queue, settle_video, stage_tokens and settle(differentiable="implicit") run eagerly behind a graph break:
    eager bits, and the implicit backward still sets last_adjoint."""
    m = _glom(256, 3, 32, 4)
    ref = copy.deepcopy(m)
    x = _images(m, 5, 1)[0]
    with torch.no_grad():
        torch._dynamo.reset()
        got = torch.compile(lambda xx: (m.settle_queue(xx, 1e-2, max_iters=6, slots=2),
                                        m.settle_video(xx.view(1, 5, *xx.shape[1:]), 1e-2, max_iters=6)))(x)
        want = (ref.settle_queue(x, 1e-2, max_iters=6, slots=2),
                ref.settle_video(x.view(1, 5, *x.shape[1:]), 1e-2, max_iters=6))
        _equal_all(got, want, "settle_queue / settle_video")
        torch._dynamo.reset()
        torch.compile(m.stage_tokens)(x)
        _equal(m(x, iters=3), ref(x, iters=3), "after a compiled stage_tokens")

    mt, xt, c, _, _ = _train_model()
    rt = copy.deepcopy(mt)

    def implicit(mm, xx):
        return (mm.settle(xx, 0.05, max_iters=6, differentiable="implicit")[0][:, :, -1] * c).sum()
    import test_cuda_graphs as CG
    with CG._deterministic(True):
        torch._dynamo.reset()
        torch.compile(implicit)(mt, xt).backward()
        implicit(rt, xt).backward()
    for (pn, p), q in zip(mt.named_parameters(), rt.parameters()):
        if q.grad is None:
            assert p.grad is None, pn
            continue
        _equal(p.grad, q.grad, ("implicit", pn))
    _equal_all(mt.last_adjoint, rt.last_adjoint, "last_adjoint")


@pytest.mark.gpu
def test_per_image_iters_break_once_then_run_the_steps_op():
    m = _glom(256, 3, 32, 4)
    ref = copy.deepcopy(m)
    x = _images(m, 3, 1)[0]
    iters = torch.tensor([1, 4, 2], device=DEV)
    from glom_pytorch_b200 import ops
    calls = []
    orig = ops._engine_call

    def counting(*a):
        calls.append(a[5] is not None)                  # the steps argument
        return orig(*a)
    with torch.no_grad():
        torch._dynamo.reset()
        ops._engine_call = counting
        try:
            got = torch.compile(m)(x, iters=iters)
        finally:
            ops._engine_call = orig
        _equal(got, ref(x, iters=iters), "per-image iters")
        assert calls == [True], calls
        torch._dynamo.reset()
        assert _breaks(m, x, iters=iters) == 1


@pytest.mark.gpu
def test_compiled_islands_of_states_that_require_grad():
    """islands of a training forward's states inside a compiled step: no gradient flows through the analytics (as
    eagerly), the step compiles without a break, and its analytics and gradients are the eager bits."""
    import test_cuda_graphs as CG
    from glom_pytorch_b200.islands import islands
    m, x, c, S, g = _train_model()
    ref = copy.deepcopy(m)

    def step(mm, xx):
        states = mm(xx, iters=3, return_all=True)
        isl = islands(states)
        return (states[2, :, :, -1] * c).sum(), isl.agreement, isl.cos_right, isl.labels, isl.agreement.mean()
    with CG._deterministic(True):
        torch._dynamo.reset()
        got = torch.compile(step, fullgraph=True)(m, x)
        want = step(ref, x)
        assert not any(t.requires_grad for t in got[1:]), [t.requires_grad for t in got[1:]]
        got[0].backward()
        want[0].backward()
    for i, (a, b) in enumerate(zip(got[1:4], want[1:4])):
        _equal(a, b, ("islands", i))
    assert torch.allclose(got[4], want[4], rtol=1e-5, atol=0)      # the mean is inductor's reduction, not the engine's
    for (pn, p), q in zip(m.named_parameters(), ref.parameters()):
        _equal(p.grad, q.grad, ("grad", pn))
    torch._dynamo.reset()
    assert _breaks(step, m, x) == 0


@pytest.mark.gpu
def test_ops_check_their_arguments():
    """Direct calls with wrong shapes or mixed devices raise before the library is called."""
    m = _glom(64, 3, 28, 7, local_consensus_radius=1)
    x, S = _images(m, 2, 1)
    lin = m.image_to_tokens[1]
    w = list(m._mlp_params())
    tok = torch.ops.glom_b200.tokenize(x, lin.weight, lin.bias, 7, "bf16")
    pos, init = m.pos_emb.weight[:16], m.init_levels
    side, d2, mask = m.attention._op_mask_args(16)

    def update(*args, steps=None, state0=None, iters=2):
        return torch.ops.glom_b200.column_update(*args[:2], state0, args[2], *args[3:], steps, False, side, d2, None,
                                                 "bf16", iters, False, False)
    with torch.no_grad():
        for what, call in {
            "bu_w1 has shape": lambda: update(tok, pos, init, w[0][:-1], *w[1:]),
            "td_b2 has shape": lambda: update(tok, pos, init, *w[:7], w[7][:-1]),
            "pos has shape": lambda: update(tok, pos[:-1], init, *w),
            "init_levels must be": lambda: update(tok, pos, init[:, :-1], *w),
            "state0 has shape": lambda: update(tok, pos, init, *w, state0=S[:1]),
            "steps has shape": lambda: update(tok, pos, init, *w, steps=torch.ones(3, dtype=torch.int32, device=DEV)),
            "pos is on cpu": lambda: update(tok, pos.cpu(), init, *w),
            "iters must be": lambda: update(tok, pos, init, *w, iters=-1),
            "weight must be": lambda: torch.ops.glom_b200.tokenize(x, lin.weight[:, :-1], lin.bias, 7, "bf16"),
            "not \\(B, 3, H, W\\)": lambda: torch.ops.glom_b200.tokenize(x[:, :, :-1], lin.weight, lin.bias, 7,
                                                                         "bf16"),
            "mask must be": lambda: torch.ops.glom_b200.check_radius_mask(mask[:, :-1], side, d2),
            "states must be": lambda: torch.ops.glom_b200.column_update_backward(
                tok, pos, S[None].expand(2, -1, -1, -1, -1), S, *w, None, False, side, d2, "bf16", 3, False, False,
                True),
        }.items():
            with pytest.raises(ValueError, match=what):
                call()


# ----------------------------------------------------------------------------- GPU: radius mask, eager untouched
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["default", "reduce-overhead"])
def test_in_place_mask_edit_after_compiling_never_uses_the_stale_radius(mode):
    """An in-place edit of the radius mask after compiling raises on the next call, also once mode="reduce-overhead" has
    recorded its CUDA graph (the mask check is left out of the graph); after the host check the call retraces."""
    m = _glom(128, 3, 64, 4, local_consensus_radius=2, consensus_self=True)
    x = _images(m, 2, 1)[0]
    cm = _compile(m, **({} if mode == "default" else {"mode": mode}))
    with torch.no_grad():
        want = copy.deepcopy(m)(x, iters=2)
        for _ in range(3):                                                 # warm-up, record, replay
            _equal(cm(x, iters=2).clone(), want, (mode, "before the edit"))
        wider = G.Glom(dim=128, levels=3, image_size=64, patch_size=4, local_consensus_radius=3).attention
        m.attention.non_local_mask.copy_(wider.non_local_mask)            # in place: a radius-3 mask
        with pytest.raises(RuntimeError, match="edited in place after tracing"):
            cm(x, iters=2)
        m.attention.mask_params(256)                                       # the host check the error asks for
        ref = copy.deepcopy(m)
        _equal(cm(x, iters=2).clone(), ref(x, iters=2), (mode, "retraced with the edited mask"))
        assert m.attention._mask_key[1] == 9


@pytest.mark.gpu
def test_eager_calls_never_reach_the_ops():
    """Eager forward, settle, training and resume: no glom_b200 op, the same last_launches as a deepcopy, and a carried
    state still takes forward_resume."""
    from glom_pytorch_b200 import _native
    m = _glom(256, 3, 32, 4)
    ref = copy.deepcopy(m)
    x, S = _images(m, 3, 1)
    resumed = []
    orig = _native.forward_resume

    def counting(*a, **k):
        resumed.append(1)
        return orig(*a, **k)
    with _EngineOpCounter() as seen:
        with torch.no_grad():
            a = m(x, iters=4)
            _native.forward_resume = counting
            try:
                b = m(x, iters=3, levels=a)
            finally:
                _native.forward_resume = orig
            launches = m.last_launches
            m.settle(x, 1e-2, max_iters=6, levels=S)
            m.tokens(x)
        m.train()
        m(x, iters=3, return_all=True).sum().backward()
    assert not seen.calls, seen.calls
    assert resumed == [1]
    with torch.no_grad():
        ra = ref(x, iters=4)
        rb = ref(x, iters=3, levels=ra)
    assert ref.last_launches == launches
    _equal(b, rb, "resumed")
