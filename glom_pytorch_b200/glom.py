"""Drop-in `Glom` for lucidrains/glom-pytorch whose column-update loop runs on the H100 (sm_90a) engine.

Mirrors the reference's public surface (glom_pytorch/glom_pytorch.py):
  * ``Glom.__init__(*, dim, levels, image_size, patch_size, consensus_self,
    local_consensus_radius)``  (:78-87), attribute ``self.levels`` (:92);
  * ``state_dict()`` keys/shapes: ``init_levels``, ``image_to_tokens.1.{weight,bias}``,
    ``pos_emb.weight``, ``bottom_up.net.{1,3}.{weight,bias}``, ``top_down.net.{1,3}.{weight,bias}``,
    ``attention.non_local_mask`` (radius > 0 only)  -- so ``load_state_dict(ref.state_dict())`` works;
  * ``forward(img, iters=None, levels=None, return_all=False)`` (:110): ``iters=None -> 2L`` (:112),
    ``iters=0`` returns S_0, output ``(B, n, L, d)`` or ``(T+1, B, n, L, d)`` fp32.

What differs: the loop body (:131-145) plus GroupedFeedForward.forward / ConsensusAttention.forward is
one call into ``libglom_b200.so`` (C ABI in include/glom_b200.h).  CUDA sm_90a (H100) only; there is no CPU / eager
fallback -- inputs on other devices raise.  Under autograd the loop is a ``torch.autograd.Function`` whose backward
is ``glom_b200_backward`` (bf16 engine: the MLP and consensus GEMMs of the reverse pass on wgmma tensor cores, the
softmax / normalisation / bias reductions in fp32 on CUDA cores; fp32 engine: everything fp32 on CUDA cores): the
forward keeps S_0..S_T and the reverse pass recomputes each step's intermediates (README.md:58-90 training use).
The backward is once-differentiable.  By default it accumulates some sums with ``red.add`` atomics, so gradients are
reproducible only up to fp32 summation order; under ``torch.use_deterministic_algorithms(True)`` (read when the
backward runs, ``warn_only`` included) it reduces in an order fixed by the shapes instead, and the gradients are
bit-identical from run to run on the same GPU model and build (DESIGN.md, "Deterministic backward").
``settle(differentiable="implicit")`` is trained by the implicit gradient of the settled state instead
(``_SettleImplicit``, ``glom_b200_backward_implicit``; DESIGN.md, "Implicit gradients through settle").

Packed weights: the MLP weights are repacked (one small kernel) on EVERY call while ``self.training``; in eval mode
the packed copy is cached and keyed on each parameter's ``(data_ptr, _version)`` and dropped by ``load_state_dict``,
``.to()`` / ``.cuda()`` / ``.half()``-style ``_apply`` calls and ``invalidate_packed()``.  In-place edits through
``param.data`` do not bump ``_version``: call ``invalidate_packed()`` after them in eval mode.  A call made under CUDA
graph capture packs inside its graph into a buffer of its own and uses workspaces no other call touches, so its graph
reads the parameters at replay and depends on no other call (DESIGN.md, "CUDA graphs and streams").  While
torch.compile / torch.export trace, forward, settle, tokens and islands call the ``glom_b200`` custom ops of ops.py,
which run the same host bodies as eager calls (``_engine_forward`` and its siblings below) in buffers of their own, with
the semantics of a captured call; ``last_launches`` is then not updated, and a compiled step's backward runs in the
deterministic mode in effect at its forward call (DESIGN.md, "torch.compile and torch.export").

Engine-only knob (keyword-only, additive): ``precision`` = ``"bf16"`` (default; wgmma tensor cores,
bf16 operands, fp32 accumulate and fp32 state -- the arithmetic of the reference under
``torch.autocast(dtype=torch.bfloat16)``) or ``"fp32"`` (CUDA-core path: each step within 8e-7 relative, per
kernel tile, of the same step in float64 from the same state; tests/test_cuda_core_oracle.py).  The fp32 engine needs
dim + n <= 3632 (its consensus keeps a block's 16 query rows and logits in shared memory).
"""
from math import prod, sqrt

import operator
import weakref

import torch
from torch import nn

from . import _native


def _aligned_bytes(nbytes, device, align=1024):
    """uint8 device buffer whose data_ptr is `align`-byte aligned (TMA / swizzle-128B bases)."""
    raw = torch.empty(nbytes + align, dtype=torch.uint8, device=device)
    off = (-raw.data_ptr()) % align
    return raw[off:off + nbytes]


def _contiguous16(t):
    """t contiguous with a 16-byte aligned data_ptr, as the engine's fp32 tensor arguments must be: a contiguous view
    that starts mid-row of a larger buffer (e.g. ``big.view(-1)[1:1 + k].view(shape)``) is copied."""
    t = t.contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()


def _f32(t, device=None):
    """t detached, as fp32 (on `device` if given), contiguous and 16-byte aligned: an fp32 tensor argument of the engine."""
    return _contiguous16(t.detach().to(device=device, dtype=torch.float32))


def _ptr(t):
    return None if t is None else t.data_ptr()


def _stream(device):
    return torch.cuda.current_stream(device).cuda_stream


_GRADS = tuple(k for k, _ in _native.Grads._fields_[1:])     # d_tokens, d_pos, d_state0, d_init, then the 8 MLP weights'


# ---------------------------------------------------------------------- the host side of each engine call
# One body per C operation, shared by eager Glom and the glom_b200 custom ops (ops.py).  They differ only in where the
# buffers come from: `workspace` is a callable nbytes -> uint8 device tensor (eager: the module's cached workspace of a
# slot, or a buffer of the capture's own; ops: a fresh _aligned_bytes), and eager passes its cached packed weights.
def _pack_weights(cfg, params, packed):
    """glom_b200_pack_weights: the 8 MLP parameters in the reference layout, packed for cfg into `packed` -> packed."""
    srcs = [_f32(p) for p in params]
    with torch.cuda.device(packed.device):
        _native.pack_weights(cfg, [t.data_ptr() for t in srcs], packed.data_ptr(), packed.numel(),
                             _stream(packed.device))
    return packed


def _engine_inputs(tokens, pos, state0, init_levels):
    """The fp32 tensor arguments of a forward, settle or queue call -> (tokens, pos, state0 or None, init_levels)."""
    return (_f32(tokens), _f32(pos), None if state0 is None else _f32(state0, tokens.device), _f32(init_levels))


def _engine_forward(cfg, packed, tokens, pos, state0, init_levels, iters, keep_all, workspace, steps=None, tol=None):
    """One forward engine call from state0 (None: init_levels) with the packed weights of cfg:
    * glom_b200_forward: `iters` steps;
    * `steps`, a (B,) integer tensor with maximum `iters` (glom_b200_forward_steps): steps[b] steps for image b;
    * `tol` (glom_b200_settle / _settle_all): up to `iters` steps, each image stopped on the GPU.
    -> (iters+1, B, n, L, d) fp32 if keep_all, else (B, n, L, d); with `tol` (states, steps (B,) int32)."""
    device = tokens.device
    b, n = tokens.shape[0], tokens.shape[1]
    with torch.cuda.device(device):
        stream = _stream(device)
        tokens, pos, state0, init = _engine_inputs(tokens, pos, state0, init_levels)
        shape = (b, n) + tuple(init.shape)
        out = torch.empty(((iters + 1,) + shape) if keep_all else shape, dtype=torch.float32, device=device)
        args = (cfg, packed.data_ptr(), tokens.data_ptr(), pos.data_ptr(), _ptr(state0), init.data_ptr(), out.data_ptr(), b)
        if tol is not None:
            steps = torch.empty(b, dtype=torch.int32, device=device)
            ws = workspace((_native.settle_all_workspace_bytes if keep_all else _native.settle_workspace_bytes)(cfg, b, iters))
            _native.settle(*args, iters, keep_all, tol, steps.data_ptr(), ws.data_ptr(), ws.numel(), stream)
            return out, steps
        if steps is None:
            ws = workspace(_native.workspace_bytes(cfg, b, iters, keep_all))
            _native.forward(*args, iters, keep_all, ws.data_ptr(), ws.numel(), stream)
        else:
            steps = steps.to(device=device, dtype=torch.int32).contiguous()
            ws = workspace(_native.forward_steps_workspace_bytes(cfg, b, iters, keep_all))
            _native.forward_steps(*args, steps.data_ptr(), iters, keep_all, ws.data_ptr(), ws.numel(), stream)
    return out


def _zero_grads(tokens, pos, weights, d_state0=None, d_init=None):
    """The gradient buffers of a backward, by _native.Grads field name: zeroed fp32 tensors shaped like tokens, pos and
    the weights, and d_state0 / d_init of the shapes given (None: absent)."""
    shapes = (tokens.shape, pos.shape, d_state0, d_init, *(w.shape for w in weights))
    return {k: None if s is None else torch.zeros(s, dtype=torch.float32, device=tokens.device)
            for k, s in zip(_GRADS, shapes)}


def _engine_backward(cfg, tokens, pos, states, grad_out, weights, iters, grad_all, steps, has_state0, deterministic,
                     workspace):
    """glom_b200_backward from the kept states (iters+1, B, n, L, d) and the cotangent of every slab (grad_all) or of
    slab `iters`; with `steps` (the forward's per-image step counts) glom_b200_backward_steps, with `deterministic` the
    fixed-order reductions of glom_b200_backward_ex.  -> the 12 gradients by Grads field name: d_state0 is None
    without a start state, d_init with one."""
    device = states.device
    b = states.shape[1]
    with torch.cuda.device(device):
        grad_out = _f32(grad_out)
        wts = [_f32(w) for w in weights]
        tokens, pos = _f32(tokens), _f32(pos)
        g = _zero_grads(tokens, pos, wts, states.shape[1:] if has_state0 else None,
                        None if has_state0 else states.shape[-2:])
        ws = workspace(_native.backward_workspace_bytes(cfg, b))
        if steps is not None:
            steps = steps.to(device=device, dtype=torch.int32).contiguous()
        _native.backward(cfg, [w.data_ptr() for w in wts], tokens.data_ptr(), pos.data_ptr(), states.data_ptr(),
                         grad_out.data_ptr(), {k: _ptr(v) for k, v in g.items()}, b, iters, grad_all, ws.data_ptr(),
                         ws.numel(), _stream(device), _ptr(steps), deterministic=deterministic)
    return g


def _engine_tokenize(img, weight, bias, patch, precision, workspace):
    """glom_b200_tokenize: image_to_tokens of a (B, 3, H, W) image -> (B, n, dim) fp32."""
    img = img.detach().float().contiguous()
    b, _, h, w = img.shape
    dim = weight.shape[0]
    device = img.device
    with torch.cuda.device(device):
        out = torch.empty(b, (h // patch) * (w // patch), dim, dtype=torch.float32, device=device)
        wt, bs = _f32(weight), _f32(bias)
        nbytes = _native.tokenize_workspace_bytes(b, h, w, patch, dim, precision)
        ws = workspace(nbytes) if nbytes else None
        _native.tokenize(img.data_ptr(), wt.data_ptr(), bs.data_ptr(), out.data_ptr(), b, h, w, patch, dim, precision,
                         _ptr(ws), nbytes, _stream(device))
    return out


def _engine_tokenize_backward(img, weight, d_tokens, patch, need_img, need_weight, need_bias, deterministic, workspace):
    """glom_b200_tokenize_backward (deterministic: _ex, d_bias by a fixed-order column sum) -> (d_img, d_weight,
    d_bias), each None when not needed."""
    img = img.detach().float().contiguous()
    b, _, h, w = img.shape
    dim = weight.shape[0]
    device = img.device
    d_tokens = d_tokens.to(torch.float32).contiguous()
    wt = _f32(weight)

    def zeros(shape, need):
        return torch.zeros(shape, dtype=torch.float32, device=device) if need else None
    d_w, d_b, d_i = zeros(wt.shape, need_weight), zeros(dim, need_bias), zeros(img.shape, need_img)
    with torch.cuda.device(device):
        ws = workspace(_native.tokenize_backward_workspace_bytes(b, h, w, patch, need_img))
        _native.tokenize_backward(img.data_ptr(), wt.data_ptr(), d_tokens.data_ptr(), _ptr(d_w), _ptr(d_b), _ptr(d_i),
                                  b, h, w, patch, dim, ws.data_ptr(), ws.numel(), _stream(device),
                                  deterministic=deterministic)
    return d_i, d_w, d_b


def _capturing():
    """True inside a CUDA graph capture on the current stream.  Such a call may only enqueue: it reads nothing on the
    host, and it uses buffers of its own that no other call touches (Glom._capture_owned).  Never true while
    torch.compile / torch.export trace: that path calls the custom ops (ops.py), which always work in buffers of their
    own."""
    return (not torch.compiler.is_compiling() and torch.cuda.is_available()
            and torch.cuda.is_current_stream_capturing())


def _no_capture(what, why):
    if _capturing():
        raise RuntimeError(f"{what} cannot be captured in a CUDA graph: {why}")


def _require_cuda(img):
    if not img.is_cuda:
        raise RuntimeError("glom_pytorch_b200.Glom runs on CUDA sm_90a (H100) only (no CPU fallback); "
                           "move the module and inputs to an H100")


def radius_mask_d2(mask, side):
    """d2_max of a (1, n, n) radius mask on a side x side patch grid (True = masked: squared distance > d2_max), or None
    if the mask is no such mask.  Reads the mask on the host."""
    mask = mask[0].cpu()
    ar = torch.arange(side)
    hh, ww = torch.meshgrid(ar, ar, indexing="ij")
    co = torch.stack((hh.reshape(-1), ww.reshape(-1)), -1)
    d2 = ((co[:, None, :] - co[None, :, :]) ** 2).sum(-1)
    kept = d2[~mask]
    d2_max = int(kept.max().item()) if kept.numel() else -1
    return d2_max if torch.equal(d2 > d2_max, mask) else None


class _Patchify(nn.Module):
    """Parameter-free placeholder at index 0 so the Linear keeps the key ``image_to_tokens.1.*``
    (the reference has an einops Rearrange there, glom_pytorch.py:95)."""

    def __init__(self, patch_size):
        super().__init__()
        self.patch_size = patch_size

    def forward(self, img):
        b, c, h, w = img.shape
        p = self.patch_size
        x = img.reshape(b, c, h // p, p, w // p, p).permute(0, 2, 4, 3, 5, 1)   # b h w p1 p2 c
        return x.reshape(b, (h // p) * (w // p), p * p * c)


class GroupedFeedForward(nn.Module):
    """Parameter container with the reference's layout (glom_pytorch.py:23-36): two grouped 1x1
    Conv1d at ``net.1`` and ``net.3``.  The engine consumes the weights repacked; this module has
    no forward of its own."""

    def __init__(self, *, dim, groups, mult=4):
        super().__init__()
        total = dim * groups
        self.net = nn.Sequential(
            nn.Identity(),
            nn.Conv1d(total, total * mult, 1, groups=groups),
            nn.GELU(),
            nn.Conv1d(total * mult, total, 1, groups=groups),
            nn.Identity(),
        )

    def forward(self, *_):
        raise RuntimeError("GroupedFeedForward runs inside the fused column update engine; call Glom.forward")


class ConsensusAttention(nn.Module):
    """Holds attend_self / radius and the ``non_local_mask`` buffer (glom_pytorch.py:39-54)."""

    def __init__(self, num_patches_side, attend_self=True, local_consensus_radius=0):
        super().__init__()
        self.attend_self = attend_self
        self.local_consensus_radius = local_consensus_radius
        self.num_patches_side = num_patches_side
        if local_consensus_radius > 0:
            ar = torch.arange(num_patches_side)
            hh, ww = torch.meshgrid(ar, ar, indexing="ij")
            co = torch.stack((hh.reshape(-1), ww.reshape(-1)), -1).float()     # (h w) c
            dist = torch.cdist(co, co)
            self.register_buffer("non_local_mask", (dist > local_consensus_radius)[None])
        self._mask_key = None
        self._derive_mask()

    def forward(self, *_):
        raise RuntimeError("ConsensusAttention runs inside the fused column update engine; call Glom.forward")

    def mask_params(self, n):
        """(mask_side, mask_d2_max) for the engine's analytic mask, derived from the buffer so a
        loaded state_dict is honoured; raises if the buffer is not a radial mask on the grid.  The buffer is checked on
        the host when it is created, moved, loaded or copied, so this call reads nothing from the device (and may run
        inside a CUDA graph capture) unless the buffer was edited in place since."""
        return self._mask_args(n, recheck=True)[:2]

    def _mask_args(self, n, recheck):
        """-> (mask_side, mask_d2_max, mask buffer or None), checked; `recheck`: re-derive d2_max from the buffer first
        if it was edited in place since its last host check."""
        if self.local_consensus_radius <= 0:
            return 0, 0, None
        side = self.num_patches_side
        if n != side * side:
            raise RuntimeError(f"local_consensus_radius needs n == num_patches ({side * side}), got {n} "
                               "(the reference's masked_fill_ fails the same way)")
        if recheck and not self._mask_fresh():
            _no_capture("a call after an in-place edit of attention.non_local_mask",
                        "checking the edited mask reads it on the host; make one call outside the capture first")
            self._derive_mask()
        if self._mask_key[1] is None:
            raise RuntimeError("attention.non_local_mask is not a radius mask on the patch grid")
        return side, self._mask_key[1], self.non_local_mask

    def _mask_fresh(self):
        key = getattr(self, "_mask_key", None)
        return key is not None and key[0] is self.non_local_mask and key[2] == self.non_local_mask._version

    def _derive_mask(self):
        """Key the buffer with its d2_max (None if it is not a radius mask on the grid), read from a host copy."""
        if self.local_consensus_radius <= 0:
            return
        self._mask_key = (self.non_local_mask, radius_mask_d2(self.non_local_mask, self.num_patches_side),
                          self.non_local_mask._version)

    def _op_mask_args(self, n):
        """mask_params for the custom-op path (glom_pytorch_b200.ops), which torch.compile / torch.export trace:
        -> (mask_side, mask_d2_max, mask buffer or None).  The radius is the one of the last host check, a constant of
        the trace (dynamo guards on ``_mask_key``); the op check_radius_mask re-checks the buffer when it runs, so an
        in-place edit made after tracing raises instead of running with the old radius."""
        return self._mask_args(n, recheck=False)

    def _apply(self, fn, *args, **kwargs):                 # .to() / .cuda() replace the buffer: its d2_max carries over
        if self.local_consensus_radius > 0 and not self._mask_fresh():
            self._derive_mask()
        out = super()._apply(fn, *args, **kwargs)
        if self.local_consensus_radius > 0:
            self._mask_key = (self.non_local_mask, self._mask_key[1], self.non_local_mask._version)
        return out

    def _load_from_state_dict(self, *args, **kwargs):     # a loaded mask (copied in place) is re-derived
        out = super()._load_from_state_dict(*args, **kwargs)
        self._derive_mask()
        return out

    def __getstate__(self):                               # pickle / deepcopy: the key travels as d2_max alone
        st = super().__getstate__() if hasattr(super(), "__getstate__") else self.__dict__.copy()
        st = dict(st)
        st.pop("_mask_key", None)
        if self.local_consensus_radius > 0:
            if not self._mask_fresh():
                self._derive_mask()
            st["_mask_d2"] = self._mask_key[1]
        return st

    def __setstate__(self, st):
        st = dict(st)
        carried = "_mask_d2" in st
        d2 = st.pop("_mask_d2", None)
        super().__setstate__(st)
        self._mask_key = None
        if carried:
            self._mask_key = (self.non_local_mask, d2, self.non_local_mask._version)
        else:
            self._derive_mask()


class _ColumnUpdate(torch.autograd.Function):
    """The loop glom_pytorch.py:131-145 as one differentiable op: forward = the engine call with all states kept,
    backward = glom_b200_backward (recompute per step; tensor-core GEMMs for the bf16 engine).  With `steps` (the
    engine's (B,) int32 copy of a per-image step vector, iters = its maximum): forward_steps / backward_steps.  With
    `tol` (Glom.settle(differentiable=True), iters = max_iters): settle_all / backward_steps with the settle's own step
    counts, which are constants of the backward exactly as in forward(iters=steps); the outputs are then
    (levels, steps), and steps is not differentiable."""

    @staticmethod
    def forward(ctx, module, iters, steps, tol, return_all, tokens, pos, state0, init_levels, *weights):
        tokens, pos = _contiguous16(tokens), _contiguous16(pos)
        states = module._run(tokens, pos, state0, init_levels, iters, True, steps=steps, tol=tol)   # (T+1, B, n, L, d)
        if tol is not None:
            states, steps = states
            ctx.mark_non_differentiable(steps)
        ctx.module, ctx.iters, ctx.return_all = module, iters, return_all
        # settle: the backward reads its own copy, so an in-place edit of the returned steps changes no gradient
        ctx.steps = steps if tol is None else steps.clone()
        ctx.had_state0 = state0 is not None
        ctx.want_state0 = state0 is not None and state0.requires_grad
        ctx.save_for_backward(tokens, pos, states, *weights)
        out = states if return_all else states[iters]
        return out if tol is None else (out, steps)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out, *_grad_steps):
        module = ctx.module
        tokens, pos, states, *weights = ctx.saved_tensors
        device = states.device
        with torch.cuda.device(device):
            cfg = module.engine_cfg(tokens.shape[1])           # bf16 engine: MLP GEMMs of the backward on tensor cores
            g = _engine_backward(cfg, tokens, pos, states, grad_out, weights, ctx.iters, ctx.return_all, ctx.steps,
                                 ctx.had_state0, torch.are_deterministic_algorithms_enabled(),
                                 lambda nb: module._get_workspace(nb, device, "_bwd_workspace"))   # cached across steps
        return (None, None, None, None, None, g["d_tokens"], g["d_pos"], g["d_state0"] if ctx.want_state0 else None,
                g["d_init"], *[g[k] for k in _GRADS[4:]])


class _SettleImplicit(torch.autograd.Function):
    """Glom.settle(differentiable="implicit"): forward = glom_b200_settle (the same call as under no_grad), backward =
    glom_b200_backward_implicit, the implicit-function-theorem gradient of the settled state S* = f(S*).  The graph
    keeps S*, the tokens, pos and the weights, no trajectory.  The start state and init_levels get no gradient: the
    fixed point does not depend on where the iteration started.  Outputs (levels, steps); steps is not differentiable."""

    @staticmethod
    def forward(ctx, module, max_iters, tol, adjoint_tol, adjoint_iters, tokens, pos, state0, init_levels, *weights):
        tokens, pos = _contiguous16(tokens), _contiguous16(pos)
        levels, steps = module._run(tokens, pos, state0, init_levels, max_iters, False, tol=tol)
        ctx.mark_non_differentiable(steps)
        ctx.module, ctx.adjoint_tol, ctx.adjoint_iters = module, adjoint_tol, adjoint_iters
        ctx.save_for_backward(tokens, pos, levels, *weights)
        return levels, steps

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out, *_grad_steps):
        module = ctx.module
        tokens, pos, state, *weights = ctx.saved_tensors
        device = state.device
        b, n = tokens.shape[0], tokens.shape[1]
        grad_out = _f32(grad_out)
        wts = [_f32(w) for w in weights]
        g = _zero_grads(tokens, pos, wts)
        adj_steps = torch.empty(b, dtype=torch.int32, device=device)
        adj_q = torch.empty(b, module.levels, dtype=torch.float32, device=device)
        with torch.cuda.device(device):
            cfg = module.engine_cfg(n)
            ws_bytes = _native.backward_implicit_workspace_bytes(cfg, b)
            ws = module._get_workspace(ws_bytes, device, "_implicit_workspace")      # cached across steps
            _native.backward_implicit(cfg, [w.data_ptr() for w in wts], tokens.data_ptr(), pos.data_ptr(),
                                      state.data_ptr(), grad_out.data_ptr(), {k: _ptr(v) for k, v in g.items()}, b,
                                      ctx.adjoint_iters, ctx.adjoint_tol, adj_steps.data_ptr(), adj_q.data_ptr(),
                                      ws.data_ptr(), ws.numel(), _stream(device),
                                      deterministic=torch.are_deterministic_algorithms_enabled())
        module.last_adjoint = (adj_steps, adj_q)
        return (None, None, None, None, None, g["d_tokens"], g["d_pos"], None, None, *[g[k] for k in _GRADS[4:]])


class _Tokenize(torch.autograd.Function):
    """image_to_tokens (glom_pytorch.py:94-97, :114) as a differentiable op on the engine's own kernels: forward =
    glom_b200_tokenize (the same arithmetic with and without autograd), backward = glom_b200_tokenize_backward (fp32
    CUDA-core GEMMs for d_weight / d_img, a column sum for d_bias).  No torch / cuBLAS kernel runs in the training step."""

    @staticmethod
    def forward(ctx, module, img, weight, bias):
        img = img.float().contiguous()
        ctx.module = module
        ctx.save_for_backward(img, weight)
        ctx.need = (img.requires_grad, weight.requires_grad, bias.requires_grad)
        return module.tokens(img)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, d_tokens):
        module = ctx.module
        img, weight = ctx.saved_tensors
        device = img.device
        with torch.cuda.device(device):
            d_i, d_w, d_b = _engine_tokenize_backward(img, weight, d_tokens, module.patch_size, *ctx.needs_input_grad[1:4],
                                                      torch.are_deterministic_algorithms_enabled(),
                                                      lambda nb: module._get_workspace(nb, device, "_tok_bwd_ws"))
        return None, d_i, d_w, d_b


class Glom(nn.Module):
    def __init__(self, *, dim=512, levels=6, image_size=224, patch_size=14, consensus_self=False,
                 local_consensus_radius=0, precision="bf16"):
        super().__init__()
        if precision not in _native.PRECISION:
            raise ValueError(f"precision must be one of {sorted(_native.PRECISION)}")
        num_patches_side = image_size // patch_size
        num_patches = num_patches_side ** 2
        self.levels = levels
        self.dim = dim
        self.patch_size = patch_size
        self.precision = precision

        # creation order matches the reference (:94-108) so seeded default init is identical
        self.image_to_tokens = nn.Sequential(_Patchify(patch_size), nn.Linear(patch_size ** 2 * 3, dim))
        self.pos_emb = nn.Embedding(num_patches, dim)
        self.init_levels = nn.Parameter(torch.randn(levels, dim))
        self.bottom_up = GroupedFeedForward(dim=dim, groups=levels)
        self.top_down = GroupedFeedForward(dim=dim, groups=levels - 1)
        self.attention = ConsensusAttention(num_patches_side, attend_self=consensus_self,
                                            local_consensus_radius=local_consensus_radius)
        self.__dict__.update(self._empty_scratch())
        self.use_native_tokenizer = True
        self.last_launches = 0
        self.last_adjoint = None      # settle(differentiable="implicit"): (steps (B,) int32, q (B, L) f32) of the last backward

    # ------------------------------------------------------------------ cache hygiene
    @staticmethod
    def _empty_scratch():
        """The device-side caches, empty.  .to() / .cuda() / .float() (parameters are replaced), pickling and deepcopy
        reset them to this (.to() keeps the buffers of captured calls: graphs may still use them)."""
        return {"_packed": None,    # (key, tensor)
                "_scratch": {},     # (slot, device index, stream) -> buffer, grown on demand, reused across calls
                "_resume": None,    # cross-call persistence: what the workspace still holds about the last returned state
                "_staged": None,    # tokens of the next frame computed ahead on a side stream (stage_tokens)
                "_captured": []}    # the packed weights and workspaces of calls made under CUDA graph capture

    def invalidate_packed(self):
        """Drop the cached packed copy of the MLP weights (needed after in-place ``param.data`` edits in eval mode)."""
        self._packed = None

    def _apply(self, fn, *args, **kwargs):
        captured = self._captured
        self.__dict__.update(self._empty_scratch())
        self._captured = captured
        return super()._apply(fn, *args, **kwargs)

    def _capture_owned(self, nbytes, device):
        """A buffer for one call under CUDA graph capture.  Its graph's replays are its only users: the module keeps it
        for its lifetime, so it is never freed or handed to another call or capture, and graphs captured on one module
        share nothing (any replay order, or replays on concurrent streams, are safe)."""
        buf = _aligned_bytes(nbytes, device)
        self._captured.append(buf)
        return buf

    def _load_from_state_dict(self, *args, **kwargs):      # load_state_dict copies in place: versions bump, but be explicit
        self._packed = None
        return super()._load_from_state_dict(*args, **kwargs)

    def __getstate__(self):                                # torch.save(model) / pickle: no scratch buffers
        st = dict(super().__getstate__() if hasattr(super(), "__getstate__") else self.__dict__)
        st.update(self._empty_scratch())
        return st

    def __deepcopy__(self, memo):
        import copy
        cls = self.__class__
        new = cls.__new__(cls)
        memo[id(self)] = new
        empty = self._empty_scratch()
        for k, v in self.__dict__.items():
            new.__dict__[k] = empty[k] if k in empty else copy.deepcopy(v, memo)
        return new

    @property
    def _workspace(self):
        """The forward workspace of the current device / stream (diagnostics and tests)."""
        dev = torch.cuda.current_device()
        return self._scratch.get(("_workspace", dev, torch.cuda.current_stream(dev).cuda_stream))

    # ------------------------------------------------------------------ engine plumbing
    def _mlp_params(self):
        return (self.bottom_up.net[1].weight, self.bottom_up.net[1].bias,
                self.bottom_up.net[3].weight, self.bottom_up.net[3].bias,
                self.top_down.net[1].weight, self.top_down.net[1].bias,
                self.top_down.net[3].weight, self.top_down.net[3].bias)

    def _packed_weights(self, cfg, device, stream):
        params = self._mlp_params()
        key = (self.precision, (device, stream), tuple((p.data_ptr(), p._version) for p in params))
        capturing = _capturing()
        # training: parameters change between calls in ways the key cannot always see (optimisers that write through
        # .data, EMA updates): repack every call (one ~30 us kernel).  eval: cached on (data_ptr, _version).  Under
        # graph capture the pack is part of the graph, into a buffer of its own: a replay reads the parameters as they
        # are then, and depends on no other call or graph.
        if not self.training and not capturing and self._packed is not None and self._packed[0] == key:
            return self._packed[1]
        nbytes = _native.packed_weight_bytes(cfg)
        if capturing:
            packed = self._capture_owned(nbytes, device)
        elif self._packed is not None and self._packed[1].device == device and self._packed[1].numel() == nbytes \
                and self._packed[0][:2] == key[:2]:
            packed = self._packed[1]            # same stream order as the kernels that read it: safe to overwrite
        else:
            packed = _aligned_bytes(nbytes, device)
        _pack_weights(cfg, params, packed)
        if not capturing:
            self._packed = (key, packed)
        return packed

    def _get_workspace(self, nbytes, device, slot="_workspace"):
        """Scratch buffer per (purpose, device, stream): two forwards of one module on different streams never share
        H / C / shadow buffers, and a buffer is only ever reused by work enqueued on the stream that last used it.
        Under graph capture: a fresh buffer that only the graph uses (_capture_owned)."""
        if _capturing():
            return self._capture_owned(nbytes, device)
        key = (slot, device.index if device.index is not None else torch.cuda.current_device(),
               torch.cuda.current_stream(device).cuda_stream)
        ws = self._scratch.get(key)
        if ws is None or ws.numel() < nbytes:
            ws = _aligned_bytes(nbytes, device)
            self._scratch[key] = ws
        return ws

    def engine_cfg(self, n, precision=None):
        side, d2 = self.attention.mask_params(n)
        return _native.make_cfg(self.dim, self.levels, n, self.attention.attend_self, side, d2,
                                precision or self.precision)

    def tokens(self, img):
        """image_to_tokens (:114): fp32 CUDA-core kernel (precision fp32) or bf16 gather + wgmma GEMM (bf16)."""
        lin = self.image_to_tokens[1]
        self._check_input(img, loop=False)
        if not self.use_native_tokenizer:
            return lin(self.image_to_tokens[0](img.float())).contiguous()
        if torch.compiler.is_compiling():        # torch.compile / torch.export: the custom op (ops.py)
            return torch.ops.glom_b200.tokenize(img, lin.weight, lin.bias, self.patch_size, self.precision)
        device = img.device
        with torch.cuda.device(device):          # the library launches on the CURRENT device
            out = _engine_tokenize(img, lin.weight, lin.bias, self.patch_size, self.precision,
                                   lambda nb: self._get_workspace(nb, device, "_tok_ws"))
        self._tok_launches = _native.last_launch_count()
        return out

    # ------------------------------------------------------------------ cross-call persistence
    @torch.compiler.disable
    def stage_tokens(self, img):
        """Video / multi-frame use (README.md:94-112): compute image_to_tokens of the NEXT frame now, on a side stream, so
        that it overlaps the tail of the forward call already enqueued for the current frame.  The following
        ``forward(img, ...)`` with this very tensor (unmodified) picks the tokens up instead of tokenising again.
        No-grad inference only; returns nothing.  Not capturable: it forks to a stream of its own, and a captured forward
        tokenises inside its graph anyway."""
        _no_capture("stage_tokens", "it tokenises on a side stream for the next eager forward; a captured forward "
                                    "tokenises inside its graph")
        if not img.is_cuda:
            raise RuntimeError("stage_tokens needs a CUDA tensor")
        device = img.device
        with torch.cuda.device(device):
            side = self._scratch.get(("_side_stream", device.index))
            if side is None:
                side = torch.cuda.Stream(device)
                self._scratch[("_side_stream", device.index)] = side
            cur = torch.cuda.current_stream(device)
            side.wait_stream(cur)                       # the frame may still be on its way (H2D copy on the caller's stream)
            with torch.cuda.stream(side), torch.no_grad():
                tokens = self.tokens(img)
                img.record_stream(side)
            ev = torch.cuda.Event()
            ev.record(side)
        self._staged = {"ref": weakref.ref(img), "version": img._version, "tokens": tokens, "event": ev,
                        "weights": tuple((p.data_ptr(), p._version) for p in self.image_to_tokens[1].parameters())}

    def _take_staged(self, img):
        st, self._staged = self._staged, None
        if st is None or st["ref"]() is not img or img._version != st["version"]:
            return None
        if st["weights"] != tuple((p.data_ptr(), p._version) for p in self.image_to_tokens[1].parameters()):
            return None
        cur = torch.cuda.current_stream(img.device)
        cur.wait_event(st["event"])
        st["tokens"].record_stream(cur)
        return st["tokens"]

    # ------------------------------------------------------------------ engine call
    def _run(self, tokens, pos, state_in, init, iters, return_all, *, steps=None, tol=None, allow_resume=False):
        """One engine call (_engine_forward) with the module's packed weights and workspace.  tokens (B,n,d), pos (n,d),
        state_in (B,n,L,d) or None, init (L,d): CUDA tensors.
        * Plain (glom_b200_forward): `iters` steps.  allow_resume (eval, no autograd): when `state_in` IS the tensor the
          previous call returned, unmodified, and the workspace is the same, the engine still holds that state's bf16
          shadows / norm partials: the state prologue is skipped (glom_b200_forward_resume).
        * `steps` (glom_b200_forward_steps): image b runs steps[b] steps (steps: the engine's (B,) int32 CUDA tensor,
          iters its maximum).
        * `tol` (glom_b200_settle / _settle_all): up to `iters` steps, each image stopped on the GPU -> (out, steps).
        After a per-image run the shadows of stopped images are stale: the next forward takes the ordinary prologue.
        Under graph capture the call neither resumes nor leaves a resume record (its workspace is its graph's own), and
        the record of the last eager call stays valid."""
        device = tokens.device
        b, n = tokens.shape[0], tokens.shape[1]
        capturing = _capturing()
        resume = None
        if capturing:
            allow_resume = False
        else:
            resume, self._resume = self._resume, None
        allow_resume = allow_resume and steps is None and tol is None and iters >= 1 and self.precision == "bf16"
        ws = None

        def workspace(nbytes):
            nonlocal ws
            ws = self._get_workspace(nbytes, device)
            return ws
        with torch.cuda.device(device):
            stream = _stream(device)
            pos_key = (self.pos_emb.weight.data_ptr(), self.pos_emb.weight._version)
            call_key = (device.index, stream, b, n, self.precision, pos_key)
            use_resume = (allow_resume and resume is not None and state_in is not None and resume["ref"]() is state_in
                          and state_in._version == resume["version"] and resume["key"] == call_key)
            cfg = self.engine_cfg(n)
            packed = self._packed_weights(cfg, device, stream)
            if use_resume and workspace(_native.workspace_bytes(cfg, b, iters, return_all)).data_ptr() == resume["ws"]:
                tokens, pos, state_in, _ = _engine_inputs(tokens, pos, state_in, init)
                shape = (b, n, self.levels, self.dim)
                out = torch.empty(((iters + 1,) + shape) if return_all else shape, dtype=torch.float32, device=device)
                parity = _native.forward_resume(cfg, packed.data_ptr(), tokens.data_ptr(), pos.data_ptr(),
                                                state_in.data_ptr(), out.data_ptr(), b, iters, return_all, ws.data_ptr(),
                                                ws.numel(), stream, resume["parity"])
            else:
                parity = iters & 1
                out = _engine_forward(cfg, packed, tokens, pos, state_in, init, iters, return_all, workspace, steps=steps,
                                      tol=tol)
            self.last_launches = _native.last_launch_count() + getattr(self, "_tok_launches", 0)
            if allow_resume and not return_all:
                self._resume = {"ref": weakref.ref(out), "version": out._version, "key": call_key, "ws": ws.data_ptr(),
                                "parity": parity}
        return out

    def _parse_iters(self, iters, b):
        """-> (iters, steps): a scalar step count and None, or, for a per-image vector whose entries differ, its maximum
        and the vector itself (the caller's tensor, or an int64 CPU tensor made from a list).  Reads min / max of a
        vector once on the host, so under graph capture only an int or a CPU scalar tensor is accepted."""
        if iters is None:
            return self.levels * 2, None                                     # (:112)
        if _capturing() and (isinstance(iters, (list, tuple))
                             or isinstance(iters, torch.Tensor) and (iters.dim() > 0 or iters.is_cuda)):
            raise ValueError("forward(iters=...) with a per-image list or tensor, or a CUDA scalar, reads the step counts "
                             "on the host, which CUDA graph capture cannot do: capture with an int iters, or let the GPU "
                             "pick each image's steps with settle(img, tol, levels=..., differentiable=True), which is "
                             "capturable")
        if isinstance(iters, (list, tuple)):
            try:
                iters = torch.tensor([operator.index(v) for v in iters], dtype=torch.int64)
            except TypeError:
                raise ValueError("a per-image iters list must hold integers") from None
        if not isinstance(iters, torch.Tensor) or iters.dim() == 0:
            return int(iters), None
        if iters.dim() != 1:
            raise ValueError(f"per-image iters must be a 1-D tensor, got {iters.dim()} dimensions")
        if iters.dtype.is_floating_point or iters.dtype.is_complex or iters.dtype == torch.bool:
            raise ValueError(f"per-image iters must have an integer dtype, got {iters.dtype}")
        if iters.shape[0] != b:
            raise ValueError(f"per-image iters must have one entry per image ({b}), got {iters.shape[0]}")
        lo, hi = torch.stack(torch.aminmax(iters)).tolist()                 # one device-to-host read for a CUDA tensor
        if lo < 0:
            raise ValueError(f"per-image iters must be >= 0, got {lo}")
        if lo == hi:
            return int(hi), None
        return int(hi), iters

    # ------------------------------------------------------------------ the reference's forward (:110)
    def forward(self, img, iters=None, levels=None, return_all=False):
        """The reference's forward.  ``iters`` is an int (None = 2L), or a per-image step count: a 1-D integer tensor
        (CPU or CUDA) or a list of length B with entries >= 0.  With T = max(iters), image b then gets S_{iters[b]}
        (``return_all``: (T+1, B, n, L, d), slab t of image b = S_{min(t, iters[b])}), bit-identical to
        ``forward(img, iters=iters[b], levels=same)[b]``; under autograd a stopped image is the identity at the later
        steps.  min / max of the vector are read once on the host (one device-to-host read for a CUDA tensor); a
        vector whose entries are all equal takes the scalar path.  Per-image counts need precision='bf16' and clear
        the resume state."""
        iters, steps = self._parse_iters(iters, img.shape[0])
        if steps is not None and self.precision != "bf16":
            raise RuntimeError("per-image iters need precision='bf16' (the fp32 engine has no per-image freezing)")
        _require_cuda(img)
        if steps is not None:    # the engine's own int32 copy: later in-place edits of the caller's tensor change nothing
            steps = steps.to(device=img.device, dtype=torch.int32, copy=True)
        return self._column_update(img, levels, self._needs_grad(img, levels), iters, return_all, steps=steps)

    def _needs_grad(self, img, levels):
        return torch.is_grad_enabled() and (img.requires_grad or (levels is not None and levels.requires_grad)
                                            or any(p.requires_grad for p in self.parameters()))

    def _check_input(self, img, levels=None, loop=True):
        """-> (b, n) of a (B, 3, H, W) image with H, W multiples of the patch size.  For the column update (`loop`) the
        n patches must fit pos_emb, and `levels`, if given, must have shape (b, n, L, d)."""
        p = self.patch_size
        if img.dim() != 4 or img.shape[1] != 3 or img.shape[2] % p or img.shape[3] % p:
            raise RuntimeError(f"image {tuple(img.shape)} is not (B, 3, H, W) with H, W multiples of {p}")
        b, n = img.shape[0], (img.shape[2] // p) * (img.shape[3] // p)
        if loop and n > self.pos_emb.num_embeddings:
            raise IndexError(f"{n} patches exceed pos_emb size {self.pos_emb.num_embeddings}")   # (:117)
        if levels is not None and tuple(levels.shape) != (b, n, self.levels, self.dim):          # (:123)
            raise RuntimeError(f"levels must have shape {(b, n, self.levels, self.dim)}, got {tuple(levels.shape)}")
        return b, n

    def _column_update(self, img, levels, needs_grad, iters, return_all, *, steps=None, tol=None, adjoint=None):
        """forward and settle after their own argument checks: check the image and `levels`, take the tokens, and run the
        engine (`_run`'s arguments), through the autograd Function _ColumnUpdate when gradients are needed, or
        _SettleImplicit with `adjoint` = (adjoint_tol, adjoint_iters) (settle(differentiable="implicit"))."""
        if torch.compiler.is_compiling():
            if adjoint is not None:
                return self._settle_implicit_eager(img, levels, needs_grad, iters, return_all, tol=tol, adjoint=adjoint)
            return self._column_update_ops(img, levels, needs_grad, iters, return_all, steps, tol)
        _, n = self._check_input(img, levels)
        if not needs_grad:
            tokens = None if _capturing() else self._take_staged(img)      # a graph tokenises for itself
            if tokens is None:
                tokens = self.tokens(img)                                    # (:114) engine tokeniser
            return self._run(tokens, self.pos_emb.weight[:n], levels, self.init_levels, iters, return_all, steps=steps,
                             tol=tol, allow_resume=not self.training)
        # training: the tokeniser and the loop are the engine's differentiable ops (the same kernels as without autograd);
        # only the parameter views (pos_emb slice) are plain torch ops
        lin = self.image_to_tokens[1]
        if self.use_native_tokenizer:
            tokens = _Tokenize.apply(self, img, lin.weight, lin.bias)                           # (:114)
        else:
            self._tok_launches = 0
            tokens = lin(self.image_to_tokens[0](img.float()))
        pos = self.pos_emb.weight[:n]                                                            # (:117)
        state0 = None if levels is None else levels.to(device=img.device, dtype=torch.float32)
        if adjoint is not None:
            return _SettleImplicit.apply(self, iters, tol, *adjoint, tokens, pos, state0, self.init_levels,
                                         *self._mlp_params())
        return _ColumnUpdate.apply(self, iters, steps, tol, return_all, tokens, pos, state0, self.init_levels,
                                   *self._mlp_params())

    @torch.compiler.disable
    def _settle_implicit_eager(self, *args, **kwargs):
        """settle(differentiable="implicit") under torch.compile: the eager autograd Function behind a graph break (its
        backward sets ``last_adjoint``)."""
        return self._column_update(*args, **kwargs)

    def _column_update_ops(self, img, levels, needs_grad, iters, return_all, steps, tol):
        """_column_update while torch.compile / torch.export trace: the same engine calls as custom ops (ops.py), with
        the semantics of a call under CUDA graph capture (no resume, no staged tokens, no packed-weight cache, the
        parameters read when the op runs; ``last_launches`` is not updated).  With gradients the op keeps every state
        for its backward and the last one is sliced here, as _ColumnUpdate does."""
        _, n = self._check_input(img, levels)
        mask_side, mask_d2_max, mask = self.attention._op_mask_args(n)
        checked = None if mask is None else torch.ops.glom_b200.check_radius_mask(mask, mask_side, mask_d2_max)
        tokens = self.tokens(img)                                            # (:114)
        pos = self.pos_emb.weight[:n]                                        # (:117)
        state0 = None if levels is None else levels.to(device=img.device, dtype=torch.float32)
        args = (tokens, pos, state0, self.init_levels, *self._mlp_params())
        cfg = (self.attention.attend_self, mask_side, mask_d2_max, checked)
        if tol is None:
            out = torch.ops.glom_b200.column_update(*args, steps, *cfg, self.precision, iters, return_all, needs_grad)
        else:
            out, steps = torch.ops.glom_b200.settle(*args, *cfg, tol, iters, return_all, needs_grad)
        if needs_grad and not return_all:
            out = out[iters]
        return out if tol is None else (out, steps)

    # ------------------------------------------------------------------ inference until the columns settle
    def settle(self, img, tol, max_iters=None, levels=None, *, return_all=False, differentiable=False, adjoint_tol=None,
               adjoint_iters=None):
        """Run each image's column update until its levels stop changing -> ``(levels, steps)``.

        After step k the change of image b is ``max_l sqrt(sum_i |S_k[b,i,l] - S_{k-1}[b,i,l]|^2 / sum_i |S_k[b,i,l]|^2)``
        (sums over the image's columns, fp32); the first k where it is ``<= tol`` stops the image.  ``levels[b]`` is then
        S_k, bit-identical to ``forward(img, iters=k, levels=same_start)[b]`` on the same batch, and ``steps[b] = k``.
        Images that never meet the rule run ``max_iters`` steps (``None`` = 2L as in ``forward``).  The stopping decisions
        are taken on the GPU inside the call: ``steps`` is a (B,) int32 CUDA tensor the host never reads, so the call does
        not synchronise.  bf16 engine only.

        ``return_all=True`` returns every state, ``(max_iters+1, B, n, L, d)``: slab t of image b is S_min(t, steps[b]),
        as in ``forward(iters=steps, return_all=True)``, with the same ``steps``.

        By default settle is inference only and raises if autograd would be needed.  With ``differentiable=True`` it
        settles and trains in one forward: under autograd the result is differentiable exactly like
        ``forward(img, iters=steps, levels=levels, return_all=return_all)`` with the steps as constants, but without
        running the steps a second time and without a host read of ``steps``.  The returned ``steps`` is not
        differentiable; the backward keeps its own copy.  That path holds all max_iters+1 states in fp32 until the
        backward, with or without ``return_all``: about 1.3 GB at dim 512, 6 levels, 256 patches, batch 32 and
        max_iters 12.  Without autograd ``differentiable`` changes nothing.

        ``differentiable="implicit"`` trains the settled state itself instead of the path that reached it: the forward is
        the plain settle call (``levels`` and ``steps`` bit-identical to it under no_grad) and the graph keeps only S*,
        the tokens, pos and the weights.  The backward is the implicit-function-theorem gradient of S* = f(S*): with
        J = df/dS at each image's S* and g = dL/dS*, it iterates ``u_0 = g, u_k = g + J^T u_{k-1}`` per image, stops an
        image by settle's rule applied to u (``adjoint_tol``, default ``tol``) or after ``adjoint_iters`` passes (default
        ``max_iters``; 0 gives the one-step "Jacobian-free" gradient), and returns the gradients of one step at S* with
        cotangent u_K (the MLP weights, pos, the tokens and through them the image and the tokeniser).  ``levels`` and
        ``init_levels`` get no gradient: the fixed point does not depend on the start.  An image whose adjoint does not
        converge gets the truncated Neumann sum.  ``self.last_adjoint`` then holds ``(steps, q)`` of that backward:
        each image's K_b ((B,) int32) and its last pass's per-level ratios ((B, L) float32), on the GPU.  No
        ``return_all``."""
        if self.precision != "bf16":
            raise RuntimeError("Glom.settle needs precision='bf16' (the fp32 engine has no early stopping)")
        implicit = isinstance(differentiable, str)
        if implicit and differentiable != "implicit":
            raise ValueError(f"differentiable must be False, True or 'implicit', got {differentiable!r}")
        if not implicit and (adjoint_tol is not None or adjoint_iters is not None):
            raise ValueError("adjoint_tol / adjoint_iters need differentiable='implicit'")
        if implicit:
            if return_all:
                raise ValueError("differentiable='implicit' has no trajectory to return: return_all must be False")
            if adjoint_tol is not None:
                adjoint_tol = float(adjoint_tol)
                if adjoint_tol != adjoint_tol:
                    raise ValueError("adjoint_tol is NaN")
            if adjoint_iters is not None:
                adjoint_iters = operator.index(adjoint_iters)
                if adjoint_iters < 0:
                    raise ValueError(f"adjoint_iters must be >= 0, got {adjoint_iters}")
        _require_cuda(img)
        needs_grad = self._needs_grad(img, levels)
        if needs_grad and not differentiable:
            raise RuntimeError("Glom.settle is inference only: call it under torch.no_grad() / torch.inference_mode() "
                               "or with parameters and inputs that do not require grad, or pass differentiable=True")
        tol, max_iters = self._settle_limits(tol, max_iters)
        adjoint = None
        if implicit and needs_grad:
            adjoint = (tol if adjoint_tol is None else adjoint_tol, max_iters if adjoint_iters is None else adjoint_iters)
        return self._column_update(img, levels, needs_grad, max_iters, return_all, tol=tol, adjoint=adjoint)

    # ------------------------------------------------------------------ settling a stream of images
    @torch.compiler.disable
    def settle_queue(self, img, tol, max_iters=None, levels=None, *, slots=32):
        """Settle N images through ``slots`` batch slots -> ``(levels, steps)``, as ``settle`` returns them for the whole
        batch.

        Contract: ``levels[i]`` and ``steps[i]`` are bit-identical to ``settle(img, tol, max_iters, levels)`` on the whole
        N-image batch, and so to ``forward(img, iters=steps[i], levels=same_start)[i]``.  Rows, consensus items and tiles
        are independent across images, so which slot holds an image, and when, changes no bit.

        The engine keeps ``slots`` images in flight (the batch of each step, clipped to N).  When an image stops, its
        slot takes the next queued image on the next step, on the GPU, so the throughput follows the mean step count of
        the images rather than each batch's slowest image.  Arguments, errors and the stopping rule are those of
        ``settle``: bf16 engine only, inference only, ``max_iters >= 1`` (None = 2L), NaN ``tol`` rejected; no
        ``return_all`` or ``differentiable``.  ``levels`` (N, n, L, d) or None, result (N, n, L, d) fp32 and ``steps``
        (N,) int32 on the GPU.

        The tokens of all N images are computed up front by one tokeniser call: N * n * d * 4 bytes (512 MB for 1024
        images at dim 512 and 256 patches).  The call synchronises once per ``max_iters`` steps to read the number of
        unfinished images (4 bytes), so it cannot be captured in a CUDA graph."""
        tol, max_iters, slots = self._slot_args("settle_queue", img, levels, tol, max_iters, slots)
        num, n = self._check_input(img, levels)
        self._resume = None
        tokens = self.tokens(img)                                           # (:114) all N images, one engine call
        return self._settle_slots("settle_queue", tokens, levels, (num,), n, tol, max_iters, min(slots, num))

    @torch.compiler.disable
    def settle_video(self, frames, tol, max_iters=None, levels=None, *, slots=32):
        """Settle S video streams frame by frame -> ``(levels, steps)``, each frame starting from the levels its stream's
        previous frame settled at.  ``frames`` is (S, F, 3, H, W); ``levels`` (S, n, L, d) or None (``init_levels``) is
        the start of each stream's frame 0.  Result: ``levels`` (S, F, n, L, d) fp32 and ``steps`` (S, F) int32 on the GPU.

        Contract: ``(levels[s, f], steps[s, f])`` are bit-identical to the host loop
        ``lv = levels; for f in range(F): lv, st = settle(frames[:, f], tol, max_iters, levels=lv)`` at index s, and so
        to ``forward(frames[:, f], iters=steps[:, f], levels=<frame f-1's levels>)[s]``.  So F = 1 is ``settle_queue`` on
        ``frames[:, 0]``, and a long clip can be settled in chunks: ``settle_video(frames[:, k:], levels=out[:, k-1])``
        continues ``out = settle_video(frames[:, :k])`` with the same bits as one call over all F frames.

        The engine keeps ``slots`` streams in flight (clipped to S).  When a frame stops, its slot takes the stream's
        next frame on the next step, on the GPU, starting from the state the slot already holds; after the last frame it
        takes the next queued stream.  A static stream thus runs ahead of one with a cut instead of waiting for it at
        every frame.  Arguments, errors and the stopping rule are those of ``settle_queue``: bf16 engine only, inference
        only, ``max_iters >= 1`` (None = 2L), NaN ``tol`` rejected, ``slots >= 1``; no ``return_all`` or
        ``differentiable``.  The tokens of all S * F frames are computed up front by one tokeniser call, and the call
        reads the number of unfinished frames once per ``max_iters`` steps (4 bytes)."""
        tol, max_iters, slots = self._slot_args("settle_video", frames, levels, tol, max_iters, slots)
        p = self.patch_size
        if frames.dim() != 5 or frames.shape[2] != 3 or frames.shape[3] % p or frames.shape[4] % p:
            raise RuntimeError(f"frames {tuple(frames.shape)} is not (S, F, 3, H, W) with H, W multiples of {p}")
        num, num_frames = frames.shape[0], frames.shape[1]
        if num < 1 or num_frames < 1:
            raise RuntimeError(f"frames {tuple(frames.shape)} needs at least one stream and one frame")
        flat = frames.reshape((num * num_frames,) + tuple(frames.shape[2:]))
        _, n = self._check_input(flat)
        if levels is not None and tuple(levels.shape) != (num, n, self.levels, self.dim):
            raise RuntimeError(f"levels must have shape {(num, n, self.levels, self.dim)}, got {tuple(levels.shape)}")
        self._resume = None
        tokens = self.tokens(flat)                                          # (:114) all S * F frames, one engine call
        out, steps = self._settle_slots("settle_video", tokens, levels, (num, num_frames), n, tol, max_iters,
                                        min(slots, num))
        return out.view(num, num_frames, n, self.levels, self.dim), steps.view(num, num_frames)

    def _settle_limits(self, tol, max_iters):
        """settle's tol (not NaN) and max_iters (None = 2L, >= 1) -> (tol, max_iters)."""
        max_iters = self.levels * 2 if max_iters is None else int(max_iters)
        if max_iters < 1:
            raise ValueError(f"max_iters must be >= 1, got {max_iters}")
        tol = float(tol)
        if tol != tol:
            raise ValueError("tol is NaN")
        return tol, max_iters

    def _slot_args(self, name, img, levels, tol, max_iters, slots):
        """The argument checks of settle_queue / settle_video -> (tol, max_iters, slots)."""
        _no_capture(f"Glom.{name}", "its host loop reads the number of unfinished images between engine calls; capture "
                                    "settle(img, tol, ...) on fixed batches instead (differentiable=True for training)")
        if self.precision != "bf16":
            raise RuntimeError(f"Glom.{name} needs precision='bf16' (the fp32 engine has no early stopping)")
        _require_cuda(img)
        if self._needs_grad(img, levels):
            raise RuntimeError(f"Glom.{name} is inference only: call it under torch.no_grad() / torch.inference_mode() "
                               "or with parameters and inputs that do not require grad")
        tol, max_iters = self._settle_limits(tol, max_iters)
        slots = int(slots)
        if slots < 1:
            raise ValueError(f"slots must be >= 1, got {slots}")
        return tol, max_iters, slots

    def _settle_slots(self, name, tokens, levels, counts, n, tol, max_iters, slots):
        """The host loop of glom_b200_<name>_begin / _run: settle_queue with counts = (N,), settle_video with counts =
        (S, F) and tokens stream-major.  -> (out (prod(counts), n, L, d), steps (prod(counts),))."""
        device = tokens.device
        images = prod(counts)
        begin, run = getattr(_native, name + "_begin"), getattr(_native, name + "_run")
        with torch.cuda.device(device):
            stream = _stream(device)
            tokens, pos, state_in, init = _engine_inputs(tokens, self.pos_emb.weight[:n], levels, self.init_levels)
            cfg = self.engine_cfg(n)
            packed = self._packed_weights(cfg, device, stream)
            out = torch.empty(images, n, self.levels, self.dim, dtype=torch.float32, device=device)
            steps = torch.empty(images, dtype=torch.int32, device=device)
            remaining = torch.empty(1, dtype=torch.int32, device=device)
            ws = self._get_workspace(getattr(_native, name + "_workspace_bytes")(cfg, slots, max_iters), device)
            args = (tokens.data_ptr(), pos.data_ptr(), _ptr(state_in), init.data_ptr(), out.data_ptr(), steps.data_ptr(),
                    *counts, slots, max_iters, tol, ws.data_ptr(), ws.numel(), stream)
            begin(cfg, *args)
            launches, first = _native.last_launch_count(), 0
            while True:
                run(cfg, packed.data_ptr(), *args, first, max_iters, remaining.data_ptr())
                launches += _native.last_launch_count()
                first += max_iters
                if int(remaining.item()) == 0:                              # the only host read
                    break
            run(cfg, packed.data_ptr(), *args, first, 0, None)              # the last stopped images' states
            self.last_launches = launches + _native.last_launch_count() + getattr(self, "_tok_launches", 0)
        return out, steps
