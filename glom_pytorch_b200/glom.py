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

Packed weights: the MLP weights are repacked (one small kernel) on EVERY call while ``self.training``; in eval mode
the packed copy is cached and keyed on each parameter's ``(data_ptr, _version)`` and dropped by ``load_state_dict``,
``.to()`` / ``.cuda()`` / ``.half()``-style ``_apply`` calls and ``invalidate_packed()``.  In-place edits through
``param.data`` do not bump ``_version``: call ``invalidate_packed()`` after them in eval mode.

Engine-only knob (keyword-only, additive): ``precision`` = ``"bf16"`` (default; wgmma tensor cores,
bf16 operands, fp32 accumulate and fp32 state -- the arithmetic of the reference under
``torch.autocast(dtype=torch.bfloat16)``) or ``"fp32"`` (CUDA-core path matching the reference's fp32
forward to ~1e-5).
"""
from math import sqrt

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


def _require_cuda(img):
    if not img.is_cuda:
        raise RuntimeError("glom_pytorch_b200.Glom runs on CUDA sm_90a (H100) only (no CPU fallback); "
                           "move the module and inputs to an H100")


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

    def forward(self, *_):
        raise RuntimeError("ConsensusAttention runs inside the fused column update engine; call Glom.forward")

    def mask_params(self, n):
        """(mask_side, mask_d2_max) for the engine's analytic mask, derived from the buffer so a
        loaded state_dict is honoured; raises if the buffer is not a radial mask on the grid."""
        if self.local_consensus_radius <= 0:
            return 0, 0
        side = self.num_patches_side
        mask = self.non_local_mask[0]
        if n != side * side:
            raise RuntimeError(f"local_consensus_radius needs n == num_patches ({side * side}), got {n} "
                               "(the reference's masked_fill_ fails the same way)")
        key = getattr(self, "_mask_key", None)
        if key is None or key[0] is not self.non_local_mask or key[2] != self.non_local_mask._version:
            ar = torch.arange(side, device=mask.device)
            hh, ww = torch.meshgrid(ar, ar, indexing="ij")
            co = torch.stack((hh.reshape(-1), ww.reshape(-1)), -1)
            d2 = ((co[:, None, :] - co[None, :, :]) ** 2).sum(-1)
            kept = d2[~mask]
            d2_max = int(kept.max().item()) if kept.numel() else -1
            if not torch.equal(d2 > d2_max, mask):
                raise RuntimeError("attention.non_local_mask is not a radius mask on the patch grid")
            self._mask_key = (self.non_local_mask, d2_max, self.non_local_mask._version)
        return side, self._mask_key[1]

    def _load_from_state_dict(self, *args, **kwargs):     # a loaded mask (copied in place) is re-derived
        self._mask_key = None
        return super()._load_from_state_dict(*args, **kwargs)

    def __getstate__(self):
        st = super().__getstate__() if hasattr(super(), "__getstate__") else self.__dict__.copy()
        st = dict(st)
        st.pop("_mask_key", None)
        return st


class _ColumnUpdate(torch.autograd.Function):
    """The loop glom_pytorch.py:131-145 as one differentiable op: forward = the engine call with all states kept,
    backward = glom_b200_backward (recompute per step; tensor-core GEMMs for the bf16 engine).  With `steps` (the
    engine's (B,) int32 copy of a per-image step vector, iters = its maximum): forward_steps / backward_steps.  With
    `tol` (Glom.settle(differentiable=True), iters = max_iters): settle_all / backward_steps with the settle's own step
    counts, which are constants of the backward exactly as in forward(iters=steps); the outputs are then
    (levels, steps), and steps is not differentiable."""

    @staticmethod
    def forward(ctx, module, iters, steps, tol, return_all, tokens, pos, state0, init_levels, *weights):
        tokens, pos = tokens.contiguous(), pos.contiguous()
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
        module, iters = ctx.module, ctx.iters
        tokens, pos, states, *weights = ctx.saved_tensors
        device = states.device
        b, n = tokens.shape[0], tokens.shape[1]
        grad_out = grad_out.to(torch.float32).contiguous()
        wts = [w.detach().to(torch.float32).contiguous() for w in weights]
        zeros = torch.zeros
        g = {"d_tokens": zeros_like32(tokens), "d_pos": zeros_like32(pos),
             "d_state0": zeros(states.shape[1:], dtype=torch.float32, device=device) if ctx.had_state0 else None,
             "d_init": None if ctx.had_state0 else zeros(module.levels, module.dim, dtype=torch.float32, device=device)}
        names = ("d_bu_w1", "d_bu_b1", "d_bu_w2", "d_bu_b2", "d_td_w1", "d_td_b1", "d_td_w2", "d_td_b2")
        for k, w in zip(names, wts):
            g[k] = zeros_like32(w)
        with torch.cuda.device(device):
            cfg = module.engine_cfg(n)           # bf16 engine: MLP GEMMs of the backward on tensor cores
            ws_bytes = _native.backward_workspace_bytes(cfg, b)
            ws = module._get_workspace(ws_bytes, device, "_bwd_workspace")      # cached across steps
            ptrs = {k: (None if v is None else v.data_ptr()) for k, v in g.items()}
            _native.backward(cfg, [w.data_ptr() for w in wts], tokens.data_ptr(), pos.data_ptr(), states.data_ptr(),
                             grad_out.data_ptr(), ptrs, b, iters, ctx.return_all, ws.data_ptr(), ws.numel(),
                             torch.cuda.current_stream(device).cuda_stream,
                             None if ctx.steps is None else ctx.steps.data_ptr(),
                             deterministic=torch.are_deterministic_algorithms_enabled())
        return (None, None, None, None, None, g["d_tokens"], g["d_pos"], g["d_state0"] if ctx.want_state0 else None,
                g["d_init"], *[g[k] for k in names])


def zeros_like32(t):
    return torch.zeros(t.shape, dtype=torch.float32, device=t.device)


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
        need_img, need_w, need_b = ctx.needs_input_grad[1], ctx.needs_input_grad[2], ctx.needs_input_grad[3]
        device = img.device
        b, _, h, w = img.shape
        p = module.patch_size
        d_tokens = d_tokens.to(torch.float32).contiguous()
        wt = weight.detach().to(torch.float32).contiguous()
        d_w = zeros_like32(wt) if need_w else None
        d_b = torch.zeros(module.dim, dtype=torch.float32, device=device) if need_b else None
        d_i = zeros_like32(img) if need_img else None
        with torch.cuda.device(device):
            ws_bytes = _native.tokenize_backward_workspace_bytes(b, h, w, p, need_img)
            ws = module._get_workspace(ws_bytes, device, "_tok_bwd_ws")
            _native.tokenize_backward(img.data_ptr(), wt.data_ptr(), d_tokens.data_ptr(),
                                      None if d_w is None else d_w.data_ptr(), None if d_b is None else d_b.data_ptr(),
                                      None if d_i is None else d_i.data_ptr(), b, h, w, p, module.dim,
                                      ws.data_ptr(), ws.numel(), torch.cuda.current_stream(device).cuda_stream,
                                      deterministic=torch.are_deterministic_algorithms_enabled())
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

    # ------------------------------------------------------------------ cache hygiene
    @staticmethod
    def _empty_scratch():
        """The device-side caches, empty.  .to() / .cuda() / .float() (parameters are replaced), pickling and deepcopy
        reset them to this."""
        return {"_packed": None,    # (key, tensor)
                "_scratch": {},     # (slot, device index, stream) -> buffer, grown on demand, reused across calls
                "_resume": None,    # cross-call persistence: what the workspace still holds about the last returned state
                "_staged": None}    # tokens of the next frame computed ahead on a side stream (stage_tokens)

    def invalidate_packed(self):
        """Drop the cached packed copy of the MLP weights (needed after in-place ``param.data`` edits in eval mode)."""
        self._packed = None

    def _apply(self, fn, *args, **kwargs):
        self.__dict__.update(self._empty_scratch())
        return super()._apply(fn, *args, **kwargs)

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
        # training: parameters change between calls in ways the key cannot always see (optimisers that write through
        # .data, EMA updates): repack every call (one ~30 us kernel).  eval: cached on (data_ptr, _version).
        if not self.training and self._packed is not None and self._packed[0] == key:
            return self._packed[1]
        srcs = []
        for p in params:
            t = p.detach()
            if t.dtype != torch.float32 or not t.is_contiguous():
                t = t.float().contiguous()
            srcs.append(t)
        nbytes = _native.packed_weight_bytes(cfg)
        if self._packed is not None and self._packed[1].device == device and self._packed[1].numel() == nbytes \
                and self._packed[0][:2] == key[:2]:
            packed = self._packed[1]            # same stream order as the kernels that read it: safe to overwrite
        else:
            packed = _aligned_bytes(nbytes, device)
        _native.pack_weights(cfg, [t.data_ptr() for t in srcs], packed.data_ptr(), nbytes, stream)
        self._packed = (key, packed)
        return packed

    def _get_workspace(self, nbytes, device, slot="_workspace"):
        """Scratch buffer per (purpose, device, stream): two forwards of one module on different streams never share
        H / C / shadow buffers, and a buffer is only ever reused by work enqueued on the stream that last used it."""
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
        _, _, h, w = img.shape
        b, n = self._check_input(img, loop=False)
        p = self.patch_size
        if not self.use_native_tokenizer:
            return lin(self.image_to_tokens[0](img.float())).contiguous()
        img = img.float().contiguous()
        with torch.cuda.device(img.device):      # the library launches on the CURRENT device
            out = torch.empty(b, n, self.dim, dtype=torch.float32, device=img.device)
            wt, bs = lin.weight.detach().float().contiguous(), lin.bias.detach().float().contiguous()
            tws_bytes = _native.tokenize_workspace_bytes(b, h, w, p, self.dim, self.precision)
            tws = self._get_workspace(tws_bytes, img.device, "_tok_ws") if tws_bytes else None
            _native.tokenize(img.data_ptr(), wt.data_ptr(), bs.data_ptr(), out.data_ptr(), b, h, w, p, self.dim,
                             self.precision, tws.data_ptr() if tws_bytes else None, tws_bytes,
                             torch.cuda.current_stream(img.device).cuda_stream)
        self._tok_launches = _native.last_launch_count()
        return out

    # ------------------------------------------------------------------ cross-call persistence
    def stage_tokens(self, img):
        """Video / multi-frame use (README.md:94-112): compute image_to_tokens of the NEXT frame now, on a side stream, so
        that it overlaps the tail of the forward call already enqueued for the current frame.  The following
        ``forward(img, ...)`` with this very tensor (unmodified) picks the tokens up instead of tokenising again.
        No-grad inference only; returns nothing."""
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
        """One engine call.  tokens (B,n,d), pos (n,d), state_in (B,n,L,d) or None, init (L,d): CUDA tensors.
        * Plain (glom_b200_forward): `iters` steps.  allow_resume (eval, no autograd): when `state_in` IS the tensor the
          previous call returned, unmodified, and the workspace is the same, the engine still holds that state's bf16
          shadows / norm partials: the state prologue is skipped (glom_b200_forward_resume).
        * `steps` (glom_b200_forward_steps): image b runs steps[b] steps (steps: the engine's (B,) int32 CUDA tensor,
          iters its maximum).
        * `tol` (glom_b200_settle / _settle_all): up to `iters` steps, each image stopped on the GPU -> (out, steps).
        After a per-image run the shadows of stopped images are stale: the next forward takes the ordinary prologue."""
        device = tokens.device
        b, n = tokens.shape[0], tokens.shape[1]
        resume, self._resume = self._resume, None
        plain = steps is None and tol is None
        with torch.cuda.device(device):
            stream = torch.cuda.current_stream(device).cuda_stream
            pos_key = (self.pos_emb.weight.data_ptr(), self.pos_emb.weight._version)
            call_key = (device.index, stream, b, n, self.precision, pos_key)
            use_resume = (plain and allow_resume and resume is not None and state_in is not None and iters >= 1
                          and self.precision == "bf16" and resume["ref"]() is state_in
                          and state_in._version == resume["version"] and resume["key"] == call_key)
            tokens = tokens.detach().to(torch.float32).contiguous()
            pos = pos.detach().to(torch.float32).contiguous()
            init = init.detach().to(torch.float32).contiguous()
            if state_in is not None:
                state_in = state_in.detach().to(device=device, dtype=torch.float32).contiguous()
            state_ptr = None if state_in is None else state_in.data_ptr()
            cfg = self.engine_cfg(n)
            packed = self._packed_weights(cfg, device, stream)
            shape = (b, n, self.levels, self.dim)
            out = torch.empty(((iters + 1,) + shape) if return_all else shape, dtype=torch.float32, device=device)
            if tol is not None:
                steps = torch.empty(b, dtype=torch.int32, device=device)
            if plain:
                ws_bytes = _native.workspace_bytes(cfg, b, iters, return_all)
            elif tol is None:
                ws_bytes = _native.forward_steps_workspace_bytes(cfg, b, iters, return_all)
            else:
                ws_bytes = (_native.settle_all_workspace_bytes if return_all else _native.settle_workspace_bytes)(cfg, b, iters)
            ws = self._get_workspace(ws_bytes, device)
            if tol is not None:
                _native.settle(cfg, packed.data_ptr(), tokens.data_ptr(), pos.data_ptr(), state_ptr, init.data_ptr(),
                               out.data_ptr(), b, iters, return_all, tol, steps.data_ptr(), ws.data_ptr(), ws.numel(), stream)
            elif steps is not None:
                _native.forward_steps(cfg, packed.data_ptr(), tokens.data_ptr(), pos.data_ptr(), state_ptr, init.data_ptr(),
                                      out.data_ptr(), b, steps.data_ptr(), iters, return_all, ws.data_ptr(), ws.numel(),
                                      stream)
            elif use_resume and ws.data_ptr() == resume["ws"]:
                parity = _native.forward_resume(cfg, packed.data_ptr(), tokens.data_ptr(), pos.data_ptr(), state_ptr,
                                                out.data_ptr(), b, iters, return_all, ws.data_ptr(), ws.numel(), stream,
                                                resume["parity"])
            else:
                parity = iters & 1
                _native.forward(cfg, packed.data_ptr(), tokens.data_ptr(), pos.data_ptr(), state_ptr, init.data_ptr(),
                                out.data_ptr(), b, iters, return_all, ws.data_ptr(), ws.numel(), stream)
            self.last_launches = _native.last_launch_count() + getattr(self, "_tok_launches", 0)
            if plain and allow_resume and not return_all and iters >= 1 and self.precision == "bf16":
                self._resume = {"ref": weakref.ref(out), "version": out._version, "key": call_key, "ws": ws.data_ptr(),
                                "parity": parity}
        return out if tol is None else (out, steps)

    def _parse_iters(self, iters, b):
        """-> (iters, steps): a scalar step count and None, or, for a per-image vector whose entries differ, its maximum
        and the vector itself (the caller's tensor, or an int64 CPU tensor made from a list).  Reads min / max of a
        vector once on the host."""
        if iters is None:
            return self.levels * 2, None                                     # (:112)
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

    def _column_update(self, img, levels, needs_grad, iters, return_all, *, steps=None, tol=None):
        """forward and settle after their own argument checks: check the image and `levels`, take the tokens, and run the
        engine (`_run`'s arguments), through the autograd Function _ColumnUpdate when gradients are needed."""
        _, n = self._check_input(img, levels)
        if not needs_grad:
            tokens = self._take_staged(img)
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
        return _ColumnUpdate.apply(self, iters, steps, tol, return_all, tokens, pos, state0, self.init_levels,
                                   *self._mlp_params())

    # ------------------------------------------------------------------ inference until the columns settle
    def settle(self, img, tol, max_iters=None, levels=None, *, return_all=False, differentiable=False):
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
        max_iters 12.  Without autograd ``differentiable`` changes nothing."""
        if self.precision != "bf16":
            raise RuntimeError("Glom.settle needs precision='bf16' (the fp32 engine has no early stopping)")
        _require_cuda(img)
        needs_grad = self._needs_grad(img, levels)
        if needs_grad and not differentiable:
            raise RuntimeError("Glom.settle is inference only: call it under torch.no_grad() / torch.inference_mode() "
                               "or with parameters and inputs that do not require grad, or pass differentiable=True")
        max_iters = self.levels * 2 if max_iters is None else int(max_iters)
        if max_iters < 1:
            raise ValueError(f"max_iters must be >= 1, got {max_iters}")
        tol = float(tol)
        if tol != tol:
            raise ValueError("tol is NaN")
        return self._column_update(img, levels, needs_grad, max_iters, return_all, tol=tol)

    # ------------------------------------------------------------------ settling a stream of images
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
        if self.precision != "bf16":
            raise RuntimeError("Glom.settle_queue needs precision='bf16' (the fp32 engine has no early stopping)")
        _require_cuda(img)
        if self._needs_grad(img, levels):
            raise RuntimeError("Glom.settle_queue is inference only: call it under torch.no_grad() / torch.inference_mode() "
                               "or with parameters and inputs that do not require grad")
        max_iters = self.levels * 2 if max_iters is None else int(max_iters)
        if max_iters < 1:
            raise ValueError(f"max_iters must be >= 1, got {max_iters}")
        tol = float(tol)
        if tol != tol:
            raise ValueError("tol is NaN")
        slots = int(slots)
        if slots < 1:
            raise ValueError(f"slots must be >= 1, got {slots}")
        num, n = self._check_input(img, levels)
        self._resume = None
        slots = min(slots, num)
        tokens = self.tokens(img)                                           # (:114) all N images, one engine call
        device = tokens.device
        with torch.cuda.device(device):
            stream = torch.cuda.current_stream(device).cuda_stream
            pos = self.pos_emb.weight[:n].detach().to(torch.float32).contiguous()
            init = self.init_levels.detach().to(torch.float32).contiguous()
            state_in = None if levels is None else levels.detach().to(device=device, dtype=torch.float32).contiguous()
            state_ptr = None if state_in is None else state_in.data_ptr()
            cfg = self.engine_cfg(n)
            packed = self._packed_weights(cfg, device, stream)
            out = torch.empty(num, n, self.levels, self.dim, dtype=torch.float32, device=device)
            steps = torch.empty(num, dtype=torch.int32, device=device)
            remaining = torch.empty(1, dtype=torch.int32, device=device)
            ws = self._get_workspace(_native.settle_queue_workspace_bytes(cfg, slots, max_iters), device)
            args = (tokens.data_ptr(), pos.data_ptr(), state_ptr, init.data_ptr(), out.data_ptr(), steps.data_ptr(), num,
                    slots, max_iters, tol, ws.data_ptr(), ws.numel(), stream)
            _native.settle_queue_begin(cfg, *args)
            launches, first = _native.last_launch_count(), 0
            while True:
                _native.settle_queue_run(cfg, packed.data_ptr(), *args, first, max_iters, remaining.data_ptr())
                launches += _native.last_launch_count()
                first += max_iters
                if int(remaining.item()) == 0:                              # the only host read
                    break
            _native.settle_queue_run(cfg, packed.data_ptr(), *args, first, 0, None)   # the last stopped images' states
            self.last_launches = launches + _native.last_launch_count() + getattr(self, "_tok_launches", 0)
        return out, steps
