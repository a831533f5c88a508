"""The engine as ``torch.library`` custom ops in the namespace ``glom_b200``, so that ``torch.compile`` (also with
``fullgraph=True``) and ``torch.export`` trace ``Glom`` instead of stopping at its ctypes calls.

Each op runs the same host body as the eager path (glom.py's ``_engine_*`` functions and ``_pack_weights``, one per C
entry point of include/glom_b200.h) and is functional: its outputs, packed weights and workspace come from the torch
allocator when it runs, and it mutates no input.  Fake implementations give the output shapes from the (possibly
symbolic) input shapes, and the differentiable ops carry their autograd formulas, whose backwards are ops of their own.
``Glom`` routes ``forward``, ``settle``, ``tokens``, ``islands`` and ``parse_tree`` through these ops while
``torch.compiler.is_compiling()`` (DESIGN.md, "torch.compile and torch.export"); eager calls never reach them.

  tokenize(img, weight, bias, patch, precision) -> tokens                      glom_b200_tokenize
  tokenize_backward(img, weight, d_tokens, patch, need_img, need_weight, need_bias, deterministic)
      -> (d_img, d_weight, d_bias)                                              glom_b200_tokenize_backward[_ex]
  check_radius_mask(mask, mask_side, mask_d2_max) -> zero-size token          (host check, no device work)
  column_update(tokens, pos, state0?, init_levels, 8 MLP weights, steps?, attend_self, mask_side, mask_d2_max,
      mask_checked?, precision, iters, return_all, keep_states) -> states       pack_weights + glom_b200_forward
                                                                                (steps: glom_b200_forward_steps)
  settle(tokens, pos, state0?, init_levels, 8 MLP weights, attend_self, mask_side, mask_d2_max, mask_checked?, tol,
      max_iters, return_all, keep_states) -> (states, steps)                    pack_weights + glom_b200_settle[_all]
  column_update_backward(tokens, pos, states, grad_out, 8 MLP weights, steps?, attend_self, mask_side, mask_d2_max,
      precision, iters, grad_all, has_state0, deterministic) -> 12 gradients    glom_b200_backward[_steps|_ex]
  islands(states, side_h, side_w, threshold) -> 5 tensors                       glom_b200_islands
  parse_tree(states, side_h, side_w, threshold, embeddings) -> 9 tensors        glom_b200_islands +
                                                                                glom_b200_island_tree

``column_update`` / ``settle`` return every state, (T+1, B, n, L, d), when ``return_all`` or ``keep_states``, else the
last one.  ``keep_states`` is what the autograd formula needs: the backward recomputes each step from the states, so a
differentiable call keeps them and the caller takes slab T itself; ``return_all`` then says whether the loss may read
every slab (``grad_all``) or only slab T.  Gradients an op does not compute come back as zero-size tensors.

The engine computes the radius mask from ``mask_side`` / ``mask_d2_max``, constants of the trace taken from the mask
buffer's last host check.  ``check_radius_mask`` checks the buffer itself when it runs (on the host, once per buffer
and again after each in-place edit, as ``ConsensusAttention.mask_params`` does) and raises if it no longer is that mask.
Its zero-size result is the ``mask_checked`` argument of ``column_update`` / ``settle``, so the check runs before them
and is never dropped as dead code.  It is tagged ``cudagraph_unsafe``: under ``mode="reduce-overhead"`` inductor leaves
it out of the recorded CUDA graphs, so it runs on every call there too.

The ops check their arguments' shapes, dtypes and devices on the host before any pointer reaches the library.
"""
import weakref

import torch
from torch import Tensor

from . import _native
from .glom import (_aligned_bytes, _engine_backward, _engine_forward, _engine_tokenize, _engine_tokenize_backward,
                   _pack_weights, radius_mask_d2)


_checked_masks = {}      # id(mask) -> (weakref to mask, its _version, its d2_max or None)


def _check_mask(mask, side, d2_max):
    _require(mask.dim() == 3 and tuple(mask.shape) == (1, side * side, side * side) and mask.dtype == torch.bool,
             f"mask must be a (1, {side * side}, {side * side}) bool tensor, got {tuple(mask.shape)} {mask.dtype}")
    key = id(mask)
    hit = _checked_masks.get(key)
    if hit is None or hit[0]() is not mask or hit[1] != mask._version:
        hit = (weakref.ref(mask, lambda _, k=key: _checked_masks.pop(k, None)), mask._version,
               radius_mask_d2(mask, side))
        _checked_masks[key] = hit
    if hit[2] != d2_max:
        raise RuntimeError(f"attention.non_local_mask is no longer the radius mask (d2_max {d2_max}) this graph was "
                           "traced with: it was edited in place after tracing.  Make one eager call (or call "
                           "model.attention.mask_params(n)) so the edit is checked; the next compiled call then "
                           "retraces with the new mask")


def _require(ok, what):
    if not ok:
        raise ValueError(f"glom_b200 op: {what}")


def _check_floats(device, **tensors):
    """Every tensor given is a floating-point tensor on `device` (a CUDA device)."""
    _require(device.type == "cuda", f"tensors must be on a CUDA device, got {device}")
    for name, t in tensors.items():
        if t is not None:
            _require(t.device == device, f"{name} is on {t.device}, expected {device}")
            _require(t.dtype.is_floating_point, f"{name} must be floating point, got {t.dtype}")


def _check_shape(name, t, shape):
    _require(tuple(t.shape) == tuple(shape), f"{name} has shape {tuple(t.shape)}, expected {tuple(shape)}")


def _check_weights(weights, levels, dim):
    """The 8 MLP tensors in the layout of GroupedFeedForward's two grouped Conv1d (bottom-up: L groups, top-down:
    L-1)."""
    names = ("bu_w1", "bu_b1", "bu_w2", "bu_b2", "td_w1", "td_b1", "td_w2", "td_b2")
    for i, groups in ((0, levels), (4, levels - 1)):
        shapes = ((groups * 4 * dim, dim, 1), (groups * 4 * dim,), (groups * dim, 4 * dim, 1), (groups * dim,))
        for j, shape in enumerate(shapes):
            _check_shape(names[i + j], weights[i + j], shape)


def _check_column_args(tokens, pos, state0, init_levels, weights, steps, iters):
    """The arguments of column_update / settle / column_update_backward that the C library takes as raw pointers."""
    _require(tokens.dim() == 3, f"tokens must be (B, n, d), got {tuple(tokens.shape)}")
    b, n, dim = tokens.shape
    _require(init_levels.dim() == 2 and init_levels.shape[1] == dim,
             f"init_levels must be (L, {dim}), got {tuple(init_levels.shape)}")
    levels = init_levels.shape[0]
    _check_floats(tokens.device, tokens=tokens, pos=pos, state0=state0, init_levels=init_levels,
                  **{f"weight {i}": w for i, w in enumerate(weights)})
    _check_shape("pos", pos, (n, dim))
    if state0 is not None:
        _check_shape("state0", state0, (b, n, levels, dim))
    _check_weights(weights, levels, dim)
    _require(iters >= 0, f"iters must be >= 0, got {iters}")
    if steps is not None:
        _require(steps.device == tokens.device and not steps.dtype.is_floating_point and steps.dtype != torch.bool,
                 f"steps must be an integer tensor on {tokens.device}, got {steps.dtype} on {steps.device}")
        _check_shape("steps", steps, (b,))


def _check_image_args(img, weight, patch):
    _require(img.dim() == 4 and img.shape[1] == 3 and patch > 0 and img.shape[2] % patch == 0
             and img.shape[3] % patch == 0, f"img {tuple(img.shape)} is not (B, 3, H, W) with H, W multiples of {patch}")
    _require(weight.dim() == 2 and weight.shape[1] == patch * patch * 3,
             f"weight must be (dim, {patch * patch * 3}), got {tuple(weight.shape)}")


def _fresh(device):
    """The workspace provider of an op: a buffer of its own from the torch allocator."""
    return lambda nbytes: _aligned_bytes(nbytes, device)


def _or_empty(t, device):
    """A gradient the engine did not compute (None) as the zero-size tensor of the op's schema."""
    return torch.zeros(0, dtype=torch.float32, device=device) if t is None else t


def _state_shape(tokens, init_levels):
    return (tokens.shape[0], tokens.shape[1], init_levels.shape[0], tokens.shape[2])


def _engine_call(tokens, pos, state0, init_levels, weights, steps, attend_self, mask_side, mask_d2_max, precision,
                 iters, engine_all, tol):
    """The body of column_update and settle: one engine call in buffers of its own -> states (, steps)."""
    _check_column_args(tokens, pos, state0, init_levels, weights, steps, iters)
    device = tokens.device
    cfg = _native.make_cfg(tokens.shape[2], init_levels.shape[0], tokens.shape[1], attend_self, mask_side, mask_d2_max,
                           precision)
    packed = _pack_weights(cfg, weights, _aligned_bytes(_native.packed_weight_bytes(cfg), device))
    return _engine_forward(cfg, packed, tokens, pos, state0, init_levels, iters, engine_all, _fresh(device), steps=steps,
                           tol=tol)


# ----------------------------------------------------------------------------- radius mask
@torch.library.custom_op("glom_b200::check_radius_mask", mutates_args=(), tags=(torch.Tag.cudagraph_unsafe,))
def check_radius_mask(mask: Tensor, mask_side: int, mask_d2_max: int) -> Tensor:
    """Raise unless `mask` is still the radius mask with this d2_max -> a zero-size bool tensor on its device."""
    _check_mask(mask, mask_side, mask_d2_max)
    return torch.empty(0, dtype=torch.bool, device=mask.device)


@check_radius_mask.register_fake
def _(mask, mask_side, mask_d2_max):
    return mask.new_empty((0,), dtype=torch.bool)


# ----------------------------------------------------------------------------- tokeniser
@torch.library.custom_op("glom_b200::tokenize", mutates_args=())
def tokenize(img: Tensor, weight: Tensor, bias: Tensor, patch: int, precision: str) -> Tensor:
    """image_to_tokens: (B, 3, H, W) -> (B, n, dim) fp32, as Glom.tokens."""
    _check_image_args(img, weight, patch)
    _check_floats(img.device, img=img, weight=weight, bias=bias)
    _check_shape("bias", bias, weight.shape[:1])
    return _engine_tokenize(img, weight, bias, patch, precision, _fresh(img.device))


@tokenize.register_fake
def _(img, weight, bias, patch, precision):
    b, _, h, w = img.shape
    return img.new_empty((b, (h // patch) * (w // patch), weight.shape[0]), dtype=torch.float32)


@torch.library.custom_op("glom_b200::tokenize_backward", mutates_args=())
def tokenize_backward(img: Tensor, weight: Tensor, d_tokens: Tensor, patch: int, need_img: bool, need_weight: bool,
                      need_bias: bool, deterministic: bool) -> tuple[Tensor, Tensor, Tensor]:
    """-> (d_img, d_weight, d_bias), each zero-size when not needed."""
    _check_image_args(img, weight, patch)
    _check_floats(img.device, img=img, weight=weight, d_tokens=d_tokens)
    _check_shape("d_tokens", d_tokens, (img.shape[0], (img.shape[2] // patch) * (img.shape[3] // patch),
                                        weight.shape[0]))
    grads = _engine_tokenize_backward(img, weight, d_tokens, patch, need_img, need_weight, need_bias, deterministic,
                                      _fresh(img.device))
    return tuple(_or_empty(g, img.device) for g in grads)


@tokenize_backward.register_fake
def _(img, weight, d_tokens, patch, need_img, need_weight, need_bias, deterministic):
    def grad(t, need):
        return t.new_empty(t.shape if need else (0,), dtype=torch.float32)
    return grad(img, need_img), grad(weight, need_weight), grad(weight.new_empty(weight.shape[0]), need_bias)


def _tokenize_setup(ctx, inputs, output):
    img, weight, _, patch, _ = inputs
    ctx.save_for_backward(img, weight)
    ctx.patch = patch


def _tokenize_grad(ctx, d_tokens):
    img, weight = ctx.saved_tensors
    need = ctx.needs_input_grad[:3]
    d_i, d_w, d_b = tokenize_backward(img, weight, d_tokens, ctx.patch, *need,
                                      torch.are_deterministic_algorithms_enabled())
    return (d_i if need[0] else None, d_w if need[1] else None, d_b if need[2] else None, None, None)


tokenize.register_autograd(_tokenize_grad, setup_context=_tokenize_setup)


# ----------------------------------------------------------------------------- column update and settle
@torch.library.custom_op("glom_b200::column_update", mutates_args=())
def column_update(tokens: Tensor, pos: Tensor, state0: Tensor | None, init_levels: Tensor, bu_w1: Tensor,
                  bu_b1: Tensor, bu_w2: Tensor, bu_b2: Tensor, td_w1: Tensor, td_b1: Tensor, td_w2: Tensor,
                  td_b2: Tensor, steps: Tensor | None, attend_self: bool, mask_side: int, mask_d2_max: int,
                  mask_checked: Tensor | None, precision: str, iters: int, return_all: bool,
                  keep_states: bool) -> Tensor:
    """`iters` steps from state0 (None: init_levels), or with `steps` ((B,) int32, iters = its maximum) steps[b] for
    image b.  -> (iters+1, B, n, L, d) if return_all or keep_states, else (B, n, L, d).  `mask_checked`: the result of
    check_radius_mask when the model has a radius mask, else None (only its place in the graph matters)."""
    weights = (bu_w1, bu_b1, bu_w2, bu_b2, td_w1, td_b1, td_w2, td_b2)
    return _engine_call(tokens, pos, state0, init_levels, weights, steps, attend_self, mask_side, mask_d2_max,
                        precision, iters, return_all or keep_states, None)


@column_update.register_fake
def _(tokens, pos, state0, init_levels, bu_w1, bu_b1, bu_w2, bu_b2, td_w1, td_b1, td_w2, td_b2, steps, attend_self,
      mask_side, mask_d2_max, mask_checked, precision, iters, return_all, keep_states):
    shape = _state_shape(tokens, init_levels)
    return tokens.new_empty(((iters + 1,) + shape) if return_all or keep_states else shape, dtype=torch.float32)


@torch.library.custom_op("glom_b200::settle", mutates_args=())
def settle(tokens: Tensor, pos: Tensor, state0: Tensor | None, init_levels: Tensor, bu_w1: Tensor, bu_b1: Tensor,
           bu_w2: Tensor, bu_b2: Tensor, td_w1: Tensor, td_b1: Tensor, td_w2: Tensor, td_b2: Tensor, attend_self: bool,
           mask_side: int, mask_d2_max: int, mask_checked: Tensor | None, tol: float, max_iters: int,
           return_all: bool, keep_states: bool) -> tuple[Tensor, Tensor]:
    """Glom.settle's engine call (bf16 engine) -> (states, steps (B,) int32); states as column_update's with
    iters = max_iters, slab t of image b = S_min(t, steps[b])."""
    weights = (bu_w1, bu_b1, bu_w2, bu_b2, td_w1, td_b1, td_w2, td_b2)
    _require(max_iters >= 1, f"max_iters must be >= 1, got {max_iters}")
    return _engine_call(tokens, pos, state0, init_levels, weights, None, attend_self, mask_side, mask_d2_max, "bf16",
                        max_iters, return_all or keep_states, tol)


@settle.register_fake
def _(tokens, pos, state0, init_levels, bu_w1, bu_b1, bu_w2, bu_b2, td_w1, td_b1, td_w2, td_b2, attend_self, mask_side,
      mask_d2_max, mask_checked, tol, max_iters, return_all, keep_states):
    shape = _state_shape(tokens, init_levels)
    out = tokens.new_empty(((max_iters + 1,) + shape) if return_all or keep_states else shape, dtype=torch.float32)
    return out, tokens.new_empty((tokens.shape[0],), dtype=torch.int32)


@torch.library.custom_op("glom_b200::column_update_backward", mutates_args=())
def column_update_backward(tokens: Tensor, pos: Tensor, states: Tensor, grad_out: Tensor, bu_w1: Tensor, bu_b1: Tensor,
                           bu_w2: Tensor, bu_b2: Tensor, td_w1: Tensor, td_b1: Tensor, td_w2: Tensor, td_b2: Tensor,
                           steps: Tensor | None, attend_self: bool, mask_side: int, mask_d2_max: int, precision: str,
                           iters: int, grad_all: bool, has_state0: bool, deterministic: bool) -> list[Tensor]:
    """The backward of column_update / settle from its kept states (iters+1, B, n, L, d) and the cotangent of every
    slab (grad_all) or of slab `iters` -> [d_tokens, d_pos, d_state0, d_init, the 8 MLP weight gradients]; d_state0 is
    zero-size without a start state, d_init with one."""
    weights = (bu_w1, bu_b1, bu_w2, bu_b2, td_w1, td_b1, td_w2, td_b2)
    _require(states.dim() == 5 and states.shape[0] == iters + 1,
             f"states must be (iters+1, B, n, L, d) = ({iters + 1}, ...), got {tuple(states.shape)}")
    _check_column_args(tokens, pos, None, states[0, 0, 0], weights, steps, iters)     # S_0's (L, d) row: init's shape
    _check_floats(tokens.device, states=states, grad_out=grad_out)
    _check_shape("tokens", tokens, (states.shape[1], states.shape[2], states.shape[4]))
    _check_shape("grad_out", grad_out, states.shape if grad_all else states.shape[1:])
    _, n, levels, dim = states.shape[1:]
    cfg = _native.make_cfg(dim, levels, n, attend_self, mask_side, mask_d2_max, precision)
    g = _engine_backward(cfg, tokens, pos, states, grad_out, weights, iters, grad_all, steps, has_state0, deterministic,
                         _fresh(states.device))
    return [_or_empty(t, states.device) for t in g.values()]


@column_update_backward.register_fake
def _(tokens, pos, states, grad_out, bu_w1, bu_b1, bu_w2, bu_b2, td_w1, td_b1, td_w2, td_b2, steps, attend_self,
      mask_side, mask_d2_max, precision, iters, grad_all, has_state0, deterministic):
    def like(t, shape=None):
        return t.new_empty(t.shape if shape is None else shape, dtype=torch.float32)
    levels, dim = states.shape[-2], states.shape[-1]
    return [like(tokens), like(pos), like(states, states.shape[1:] if has_state0 else (0,)),
            like(states, (0,) if has_state0 else (levels, dim))] + [like(w) for w in (bu_w1, bu_b1, bu_w2, bu_b2, td_w1,
                                                                                    td_b1, td_w2, td_b2)]


def _backward_from_states(ctx, grad_states):
    """The autograd formula shared by column_update and settle: the engine backward over the kept states."""
    tokens, pos, states, *weights, steps = ctx.saved_tensors
    if not ctx.kept:
        raise RuntimeError("glom_b200 ops keep the states for their backward only with keep_states=True or "
                           "return_all=True")
    grad = grad_states if ctx.return_all else grad_states[ctx.iters]
    g = column_update_backward(tokens, pos, states, grad, *weights, steps, *ctx.cfg, ctx.iters, ctx.return_all,
                               ctx.has_state0, torch.are_deterministic_algorithms_enabled())
    need = ctx.needs_input_grad
    return (g[0] if need[0] else None, g[1] if need[1] else None,
            g[2] if ctx.has_state0 and need[2] else None, None if ctx.has_state0 or not need[3] else g[3],
            *[gw if nd else None for gw, nd in zip(g[4:], need[4:12])])


def _column_update_setup(ctx, inputs, output):
    tokens, pos, state0, _, *rest = inputs
    weights, steps = rest[:8], rest[8]
    attend_self, mask_side, mask_d2_max, _, precision, iters, return_all, keep_states = rest[9:]
    ctx.save_for_backward(tokens, pos, output, *weights, steps)
    ctx.cfg = (attend_self, mask_side, mask_d2_max, precision)
    ctx.iters, ctx.return_all, ctx.kept, ctx.has_state0 = iters, return_all, return_all or keep_states, state0 is not None


def _column_update_grad(ctx, grad_states):
    return _backward_from_states(ctx, grad_states) + (None,) * 9


column_update.register_autograd(_column_update_grad, setup_context=_column_update_setup)


def _settle_setup(ctx, inputs, output):
    tokens, pos, state0, _, *rest = inputs
    weights = rest[:8]
    attend_self, mask_side, mask_d2_max, _, _, max_iters, return_all, keep_states = rest[8:]
    states, steps = output
    ctx.mark_non_differentiable(steps)
    # the backward reads its own copy, so an in-place edit of the returned steps changes no gradient (as _ColumnUpdate)
    ctx.save_for_backward(tokens, pos, states, *weights, steps.clone())
    ctx.cfg = (attend_self, mask_side, mask_d2_max, "bf16")
    ctx.iters, ctx.return_all, ctx.kept, ctx.has_state0 = max_iters, return_all, return_all or keep_states, \
        state0 is not None


def _settle_grad(ctx, grad_states, _grad_steps):
    return _backward_from_states(ctx, grad_states) + (None,) * 8


settle.register_autograd(_settle_grad, setup_context=_settle_setup)


# ----------------------------------------------------------------------------- island analytics
@torch.library.custom_op("glom_b200::islands", mutates_args=())
def islands(states: Tensor, side_h: int, side_w: int, threshold: float) -> tuple[Tensor, Tensor, Tensor, Tensor,
                                                                                  Tensor]:
    """glom_pytorch_b200.islands on (..., n, L, d) states -> (cos_right, cos_down, agreement, labels, num_islands)."""
    from .islands import islands as eager_islands
    return tuple(eager_islands(states, grid=(side_h, side_w), threshold=threshold))


@islands.register_fake
def _(states, side_h, side_w, threshold):
    *lead, n, levels, _ = states.shape
    shape = (*lead, levels, n)
    return (states.new_empty(shape, dtype=torch.float32), states.new_empty(shape, dtype=torch.float32),
            states.new_empty(shape, dtype=torch.float32), states.new_empty(shape, dtype=torch.int32),
            states.new_empty((*lead, levels), dtype=torch.int32))


@torch.library.custom_op("glom_b200::parse_tree", mutates_args=())
def parse_tree(states: Tensor, side_h: int, side_w: int, threshold: float, embeddings: bool) -> tuple[
        Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor]:
    """glom_pytorch_b200.parse_tree on (..., n, L, d) states -> the 9 ParseTree fields; without embeddings the last three
    are zero-size."""
    from .islands import parse_tree as eager_parse_tree
    out = eager_parse_tree(states, grid=(side_h, side_w), threshold=threshold, embeddings=embeddings)
    return tuple(states.new_empty(0, dtype=torch.float32) if t is None else t for t in out)


@parse_tree.register_fake
def _(states, side_h, side_w, threshold, embeddings):
    *lead, n, levels, dim = states.shape
    shape = (*lead, levels, n)

    def opt(shp):
        return states.new_empty(shp if embeddings else (0,), dtype=torch.float32)
    return (states.new_empty(shape, dtype=torch.int32), states.new_empty((*lead, levels), dtype=torch.int32),
            states.new_empty(shape, dtype=torch.int32), states.new_empty(shape, dtype=torch.int32),
            states.new_empty(shape, dtype=torch.float32), states.new_empty((*lead, levels - 1), dtype=torch.float32),
            opt((*lead, levels, n, dim)), opt(shape), opt(shape))
