"""CPU-side tests: the C-ABI library loads and exports every symbol the header declares, host
logic (layout sizes, argument errors), drop-in surface, and the batch-sharding logic under gloo."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import glom_pytorch_b200 as G
from glom_pytorch_b200 import _native
from glom_pytorch_b200.sharding import shard_range

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "glom_b200.h")).read()
    declared = set(re.findall(r"GLOM_B200_API\s+[\w\s\*]+?\b(glom_b200_\w+)\s*\(", hdr))
    assert declared == set(_native.EXPORTS), declared ^ set(_native.EXPORTS)
    lib = ctypes.CDLL(G.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.glom_b200_abi_version() == 1


def test_layout_sizes_without_gpu():
    cfg = _native.make_cfg(512, 6, 256, False, 0, 0, "bf16")
    pw = _native.packed_weight_bytes(cfg)
    G_, d, L = 11, 512, 6
    assert pw >= (G_ * 4 * d * d + L * d * 8 * d) * 2 + (G_ * 4 * d + L * d) * 4
    ws = _native.workspace_bytes(cfg, 32, 12, False)
    rows = 32 * 256
    assert ws >= rows * G_ * 4 * d * 2 + rows * L * d * 4
    ws_all = _native.workspace_bytes(cfg, 32, 12, True)
    assert ws - ws_all >= rows * L * d * 4 - 4096      # return_all needs no private fp32 slab
    off, nb = _native.workspace_offset(cfg, 32, 12, False, 0)
    assert nb == rows * G_ * 4 * d * 2 and off % 1024 == 0


@pytest.mark.parametrize("kw,msg", [
    (dict(dim=512, levels=1), "levels"),
    (dict(dim=70, levels=3), "dim"),
    (dict(dim=96, levels=3, precision="bf16"), "64"),
])
def test_bad_config_is_an_error_not_a_fallback(kw, msg):
    cfg = _native.make_cfg(kw.get("dim"), kw.get("levels"), 16, False, 0, 0, kw.get("precision", "fp32"))
    with pytest.raises(_native.GlomB200Error, match=msg):
        _native.packed_weight_bytes(cfg)


# ---- argument errors of every launching entry point: exact text and code, and which error wins --------------------------
# The argument checks run before the device is queried, so they are exercised here with made-up device addresses that
# are never dereferenced.  Each case overrides one or more arguments of a valid call.
def _p(i, off=0):
    return 0x100000 + 0x1000 * i + off


_NAN = float("nan")
_W_KEYS = [k for k, _ in _native.WeightsRef._fields_[1:]]
_G_KEYS = [k for k, _ in _native.Grads._fields_[1:]]
_TENSORS = dict(tokens=_p(2), pos=_p(3), state_in=None, init=_p(4), out=_p(5))
_WS = dict(ws=_p(6), ws_bytes=1 << 40, stream=None)
_BWD = dict(cfg={}, w={}, tokens=_p(2), pos=_p(3), states=_p(4), grad_out=_p(5), gr=dict(d_init=None), batch=2)
_QUEUE = dict(cfg={}, **_TENSORS, steps_out=_p(7), items=5, slots=2, max_iters=3, tol=0.1, **_WS)
_VIDEO = dict(cfg={}, **_TENSORS, steps_out=_p(7), items=5, frames=2, slots=2, max_iters=3, tol=0.1, **_WS)
_RUN = dict(first_step=0, num_steps=2, remaining_out=None)
_IMG = dict(batch=2, height=28, width=28, patch=7, dim=64)
_TOKB = dict(img=_p(1), weight=_p(2), d_tokens=_p(3), d_weight=_p(4), d_bias=_p(5), d_img=None, **_IMG)


def _after(d, key, **new):
    """`d` with the entries of `new` inserted after `key` (argument order is dict order)."""
    out = {}
    for k, v in d.items():
        out[k] = v
        if k == key:
            out.update(new)
    return out


_CALLS = {      # symbol -> its arguments, in order, of a call that passes every check
    "pack_weights": dict(cfg={}, w={}, packed=_p(1), packed_bytes=1 << 40, stream=None),
    "forward": dict(cfg={}, packed=_p(1), **_TENSORS, batch=2, iters=3, return_all=0, **_WS),
    "forward_resume": dict(cfg={}, packed=_p(1), tokens=_p(2), pos=_p(3), state_in=_p(4), out=_p(5), batch=2, iters=3,
                           return_all=0, **_WS, shadow_parity=0, out_parity=None),
    "forward_steps": dict(cfg={}, packed=_p(1), **_TENSORS, batch=2, steps=_p(7), max_steps=3, return_all=0, **_WS),
    "settle": dict(cfg={}, packed=_p(1), **_TENSORS, batch=2, max_iters=3, tol=0.1, steps_out=_p(7), **_WS),
    "settle_queue_begin": _QUEUE,
    "settle_queue_run": {**_after(_QUEUE, "cfg", packed=_p(1)), **_RUN},
    "settle_video_begin": _VIDEO,
    "settle_video_run": {**_after(_VIDEO, "cfg", packed=_p(1)), **_RUN},
    "tokenize": dict(img=_p(1), weight=_p(2), bias=_p(3), tokens=_p(4), **_IMG, precision=1, **_WS),
    "tokenize_backward": dict(**_TOKB, **_WS),
    "tokenize_backward_ex": dict(**_TOKB, deterministic=1, **_WS),
    "backward": dict(**_BWD, iters=3, grad_all=0, **_WS),
    "backward_steps": dict(**_BWD, steps=_p(7), max_steps=3, grad_all=0, **_WS),
    "backward_ex": dict(**_BWD, steps=_p(7), max_steps=3, grad_all=0, deterministic=1, **_WS),
    "backward_implicit": dict(**{**_BWD, "gr": dict(d_state0=None, d_init=None)}, adjoint_iters=4, adjoint_tol=0.1,
                              deterministic=1, adjoint_steps_out=_p(7), adjoint_q_out=None, **_WS),
    "islands": dict(states=_p(1), slabs=2, side_h=4, side_w=4, levels=3, dim=64, threshold=0.5, cos_right=_p(2),
                    cos_down=_p(3), agreement=_p(4), labels=_p(5), num_islands=_p(6), stream=None),
}
_CALLS["settle_all"] = _CALLS["settle"]

_INVALID, _WORKSPACE = -1, -2
_FP32 = dict(precision="fp32")
_NO_GRAD = "gradient pointers: all MLP/token/pos outputs and exactly one of d_state0 / d_init"
_STRUCTS = "weights / grads struct missing or wrong size"


def _forward_family(sym, pre=""):
    """The checks forward, forward_steps, settle and settle_all share once their own have passed."""
    return [
        (sym, dict(tokens=None), _INVALID, pre + "a required pointer is NULL"),
        (sym, dict(out=None), _INVALID, pre + "a required pointer is NULL"),
        (sym, dict(init=None), _INVALID, pre + "need state_in or init_levels"),
        (sym, dict(state_in=_p(5)), _INVALID, pre + "state_out must not alias state_in"),
        (sym, dict(pos=_p(3, 8)), _INVALID, pre + "tensor pointers must be 16-byte aligned"),
        (sym, dict(init=_p(4, 4)), _INVALID, pre + "tensor pointers must be 16-byte aligned"),
        (sym, dict(tokens=None, state_in=_p(5)), _INVALID, pre + "a required pointer is NULL"),
        (sym, dict(state_in=_p(5), ws=_p(6, 512)), _INVALID, pre + "state_out must not alias state_in"),
    ]


def _queue_family(begin, run, name, items):
    pre = name + ": "
    small = name + " workspace: need {need} bytes, got 1024"
    cases = []
    for sym in (begin, run):
        cases += _forward_family(sym, pre) + [
            (sym, dict(cfg=None), _INVALID, "cfg is NULL"),
            (sym, dict(cfg=_FP32), _INVALID, pre + "bf16 engine only (precision fp32 given)"),
            (sym, dict(items=0), _INVALID, pre + items + " must be >= 1 (got 0)"),
            (sym, dict(slots=0), _INVALID, pre + "slots must be >= 1 (got 0)"),
            (sym, dict(max_iters=0), _INVALID, pre + "max_iters must be >= 1 (got 0)"),
            (sym, dict(tol=_NAN), _INVALID, pre + "tol is NaN"),
            (sym, dict(steps_out=None), _INVALID, pre + "steps_out is NULL"),
            (sym, dict(steps_out=_p(7, 2)), _INVALID, pre + "steps_out must be 4-byte aligned"),
            (sym, dict(ws=_p(6, 512)), _INVALID, pre + "workspace must be 1024-byte aligned"),
            (sym, dict(ws_bytes=1024), _WORKSPACE, small),
            (sym, dict(ws=None), _WORKSPACE, name + " workspace: need {need} bytes, got " + str(1 << 40)),
            (sym, dict(tol=_NAN, slots=0), _INVALID, pre + "slots must be >= 1 (got 0)"),
            (sym, dict(tol=_NAN, steps_out=None), _INVALID, pre + "tol is NaN"),
            (sym, dict(pos=_p(3, 8), ws_bytes=1024), _INVALID, pre + "tensor pointers must be 16-byte aligned"),
        ]
    cases += [
        (run, dict(packed=None), _INVALID, pre + "packed weights NULL or not 1024-byte aligned"),
        (run, dict(packed=_p(1, 16)), _INVALID, pre + "packed weights NULL or not 1024-byte aligned"),
        (run, dict(first_step=-1), _INVALID, pre + "first_step and num_steps must be >= 0 (got -1, 2)"),
        (run, dict(remaining_out=_p(8, 2)), _INVALID, pre + "remaining_out must be 4-byte aligned"),
        (run, dict(packed=None, tol=_NAN), _INVALID, pre + "packed weights NULL or not 1024-byte aligned"),
        (run, dict(num_steps=-1, tokens=None), _INVALID, pre + "first_step and num_steps must be >= 0 (got 0, -1)"),
        (run, dict(slots=0, packed=None), _INVALID, pre + "slots must be >= 1 (got 0)"),
    ]
    return cases


def _backward_family(sym):
    """The checks backward, backward_steps and backward_ex share once their own have passed."""
    return [
        (sym, dict(cfg=None), _INVALID, "cfg is NULL"),
        (sym, dict(batch=0), _INVALID, "batch must be >= 1 and iters >= 0"),
        (sym, dict(w=None), _INVALID, _STRUCTS),
        (sym, dict(gr=dict(struct_size=8)), _INVALID, _STRUCTS),
        (sym, dict(states=None), _INVALID, "a required pointer is NULL"),
        (sym, dict(w=dict(td_w2=None)), _INVALID, "a weight pointer is NULL"),
        (sym, dict(gr=dict(d_pos=None)), _INVALID, _NO_GRAD),
        (sym, dict(gr=dict(d_init=_p(30))), _INVALID, _NO_GRAD),           # d_state0 and d_init
        (sym, dict(gr=dict(d_state0=None)), _INVALID, _NO_GRAD),           # neither
        (sym, dict(w=dict(struct_size=8), tokens=None), _INVALID, _STRUCTS),
        (sym, dict(grad_out=None, w=dict(bu_w1=None)), _INVALID, "a required pointer is NULL"),
        (sym, dict(w=dict(bu_b1=None), gr=dict(d_td_b2=None)), _INVALID, "a weight pointer is NULL"),
    ]


_ERROR_CASES = [
    ("pack_weights", dict(cfg=None), _INVALID, "cfg is NULL"),
    ("pack_weights", dict(cfg=dict(struct_size=4)), _INVALID, "cfg.struct_size 4 != 32 (ABI mismatch)"),
    ("pack_weights", dict(w=None), _INVALID, "weights struct missing or wrong size"),
    ("pack_weights", dict(w=dict(struct_size=8)), _INVALID, "weights struct missing or wrong size"),
    ("pack_weights", dict(w=dict(bu_b2=None)), _INVALID, "a weight pointer is NULL"),
    ("pack_weights", dict(packed_bytes=512), _WORKSPACE, "packed buffer: need {need} bytes, got 512"),
    ("pack_weights", dict(packed=_p(1, 256)), _INVALID, "packed buffer must be 1024-byte aligned"),
    ("pack_weights", dict(w=dict(bu_b2=None), packed=None), _INVALID, "a weight pointer is NULL"),
    ("pack_weights", dict(packed=_p(1, 256), packed_bytes=512), _WORKSPACE, "packed buffer: need {need} bytes, got 512"),

    *_forward_family("forward"),
    ("forward", dict(cfg=None), _INVALID, "cfg is NULL"),
    ("forward", dict(cfg=dict(levels=1)), _INVALID, "levels must be >= 2 (got 1)"),
    ("forward", dict(batch=0), _INVALID, "batch must be >= 1 and iters >= 0"),
    ("forward", dict(iters=-1), _INVALID, "batch must be >= 1 and iters >= 0"),
    ("forward", dict(cfg=dict(dim=3600, n=64, precision="fp32")), _INVALID,
     "fp32 consensus keeps 16 (dim + n) floats per block in shared memory: dim + n must be <= 3632 (got 3664)"),
    ("forward", dict(packed=_p(1, 16)), _INVALID, "packed weights and workspace must be 1024-byte aligned"),
    ("forward", dict(ws=_p(6, 512)), _INVALID, "packed weights and workspace must be 1024-byte aligned"),
    ("forward", dict(packed=None), _INVALID, "a required pointer is NULL"),
    ("forward", dict(batch=0, tokens=None), _INVALID, "batch must be >= 1 and iters >= 0"),
    ("forward", dict(packed=_p(1, 16), tokens=_p(2, 4)), _INVALID, "packed weights and workspace must be 1024-byte aligned"),

    *_forward_family("forward_resume")[:2],
    ("forward_resume", dict(cfg=None), _INVALID, "forward_resume: bf16 engine only"),
    ("forward_resume", dict(cfg=_FP32), _INVALID, "forward_resume: bf16 engine only"),
    ("forward_resume", dict(state_in=None), _INVALID,
     "forward_resume: need state_in, shadow_parity in {0, 1} and iters >= 1"),
    ("forward_resume", dict(shadow_parity=2), _INVALID,
     "forward_resume: need state_in, shadow_parity in {0, 1} and iters >= 1"),
    ("forward_resume", dict(iters=0), _INVALID, "forward_resume: need state_in, shadow_parity in {0, 1} and iters >= 1"),
    ("forward_resume", dict(state_in=_p(5)), _INVALID, "state_out must not alias state_in"),
    ("forward_resume", dict(cfg=_FP32, shadow_parity=2), _INVALID, "forward_resume: bf16 engine only"),
    ("forward_resume", dict(shadow_parity=2, batch=0), _INVALID,
     "forward_resume: need state_in, shadow_parity in {0, 1} and iters >= 1"),
    ("forward_resume", dict(batch=0, tokens=None), _INVALID, "batch must be >= 1 and iters >= 0"),

    *_forward_family("forward_steps"),
    ("forward_steps", dict(cfg=_FP32), _INVALID, "forward_steps: bf16 engine only (precision fp32 given)"),
    ("forward_steps", dict(batch=0), _INVALID, "forward_steps: batch must be >= 1 (got 0)"),
    ("forward_steps", dict(max_steps=-1), _INVALID, "forward_steps: max_steps must be >= 0 (got -1)"),
    ("forward_steps", dict(steps=None), _INVALID, "forward_steps: steps is NULL"),
    ("forward_steps", dict(steps=_p(7, 2)), _INVALID, "forward_steps: steps must be 4-byte aligned"),
    ("forward_steps", dict(steps=None, tokens=None), _INVALID, "forward_steps: steps is NULL"),
    ("forward_steps", dict(max_steps=-1, steps=None), _INVALID, "forward_steps: max_steps must be >= 0 (got -1)"),

    *[c for sym in ("settle", "settle_all") for c in _forward_family(sym) + [
        (sym, dict(cfg=None), _INVALID, "cfg is NULL"),
        (sym, dict(cfg=_FP32), _INVALID, "settle: bf16 engine only (precision fp32 given)"),
        (sym, dict(batch=0), _INVALID, "settle: batch must be >= 1 (got 0)"),
        (sym, dict(max_iters=0), _INVALID, "settle: max_iters must be >= 1 (got 0)"),
        (sym, dict(tol=_NAN), _INVALID, "settle: tol is NaN"),
        (sym, dict(steps_out=None), _INVALID, "settle: steps_out is NULL"),
        (sym, dict(steps_out=_p(7, 1)), _INVALID, "settle: steps_out must be 4-byte aligned"),
        (sym, dict(tol=_NAN, max_iters=0), _INVALID, "settle: max_iters must be >= 1 (got 0)"),
        (sym, dict(tol=_NAN, steps_out=None), _INVALID, "settle: tol is NaN"),
        (sym, dict(steps_out=None, tokens=None), _INVALID, "settle: steps_out is NULL"),
        (sym, dict(packed=_p(1, 16), out=None), _INVALID, "a required pointer is NULL"),
    ]],

    *_queue_family("settle_queue_begin", "settle_queue_run", "settle_queue", "images"),
    *_queue_family("settle_video_begin", "settle_video_run", "settle_video", "streams"),
    ("settle_video_begin", dict(frames=0), _INVALID, "settle_video: frames must be >= 1 (got 0)"),
    ("settle_video_run", dict(items=1 << 20, frames=1 << 20), _INVALID,
     "settle_video: streams x frames must be < 2^31 (got 1048576 x 1048576)"),
    ("settle_video_run", dict(frames=0, slots=0), _INVALID, "settle_video: frames must be >= 1 (got 0)"),

    ("tokenize", dict(bias=None), _INVALID, "a required pointer is NULL"),
    ("tokenize", dict(patch=5), _INVALID, "image 28x28 is not a positive multiple of patch 5"),
    ("tokenize", dict(patch=0), _INVALID, "image 28x28 is not a positive multiple of patch 0"),
    ("tokenize", dict(width=35, height=3), _INVALID, "image 3x35 is not a positive multiple of patch 7"),
    ("tokenize", dict(batch=0), _INVALID, "image 28x28 is not a positive multiple of patch 7"),
    ("tokenize", dict(dim=0), _INVALID, "image 28x28 is not a positive multiple of patch 7"),
    ("tokenize", dict(precision=7), _INVALID, "unknown precision 7"),
    ("tokenize", dict(img=None, patch=5), _INVALID, "a required pointer is NULL"),
    ("tokenize", dict(width=30, precision=7), _INVALID, "image 28x30 is not a positive multiple of patch 7"),

    *[c for sym in ("tokenize_backward", "tokenize_backward_ex") for c in [
        (sym, dict(d_tokens=None), _INVALID, "a required pointer is NULL"),
        (sym, dict(height=30), _INVALID, "image 30x28 is not a positive multiple of patch 7"),
        (sym, dict(patch=-1), _INVALID, "image 28x28 is not a positive multiple of patch -1"),
        (sym, dict(dim=0), _INVALID, "image 28x28 is not a positive multiple of patch 7"),
        (sym, dict(weight=None, batch=0), _INVALID, "a required pointer is NULL"),
        (sym, dict(img=None, d_tokens=None, width=1), _INVALID, "a required pointer is NULL"),
    ]],
    ("tokenize_backward_ex", dict(deterministic=2), _INVALID, "tokenize_backward_ex: deterministic must be 0 or 1 (got 2)"),
    ("tokenize_backward_ex", dict(deterministic=-1, img=None), _INVALID,
     "tokenize_backward_ex: deterministic must be 0 or 1 (got -1)"),

    *_backward_family("backward"),
    ("backward", dict(iters=-1), _INVALID, "batch must be >= 1 and iters >= 0"),
    *_backward_family("backward_steps"),
    ("backward_steps", dict(steps=None), _INVALID, "backward_steps: steps is NULL"),
    ("backward_steps", dict(steps=_p(7, 2)), _INVALID, "backward_steps: steps must be 4-byte aligned"),
    ("backward_steps", dict(max_steps=-1), _INVALID, "backward_steps: max_steps must be >= 0 (got -1)"),
    ("backward_steps", dict(steps=None, max_steps=-1), _INVALID, "backward_steps: steps is NULL"),
    ("backward_steps", dict(max_steps=-1, cfg=None), _INVALID, "backward_steps: max_steps must be >= 0 (got -1)"),
    *_backward_family("backward_ex"),
    ("backward_ex", dict(deterministic=2), _INVALID, "backward_ex: deterministic must be 0 or 1 (got 2)"),
    ("backward_ex", dict(steps=_p(7, 2)), _INVALID, "backward_ex: steps must be 4-byte aligned"),
    ("backward_ex", dict(max_steps=-1), _INVALID, "backward_ex: max_steps must be >= 0 (got -1)"),
    ("backward_ex", dict(steps=None, max_steps=-1), _INVALID, "batch must be >= 1 and iters >= 0"),
    ("backward_ex", dict(deterministic=2, steps=_p(7, 2)), _INVALID, "backward_ex: deterministic must be 0 or 1 (got 2)"),
    ("backward_ex", dict(steps=_p(7, 2), max_steps=-1), _INVALID, "backward_ex: steps must be 4-byte aligned"),

    *[("backward_implicit", o, rc, m) for o, rc, m in [
        (dict(cfg=None), _INVALID, "cfg is NULL"),
        (dict(cfg=_FP32), _INVALID, "backward_implicit: bf16 engine only (precision fp32 given)"),
        (dict(batch=0), _INVALID, "backward_implicit: batch must be >= 1 (got 0)"),
        (dict(adjoint_iters=-1), _INVALID, "backward_implicit: adjoint_iters must be >= 0 (got -1)"),
        (dict(adjoint_tol=_NAN), _INVALID, "backward_implicit: adjoint_tol is NaN"),
        (dict(deterministic=2), _INVALID, "backward_implicit: deterministic must be 0 or 1 (got 2)"),
        (dict(adjoint_steps_out=None), _INVALID, "backward_implicit: adjoint_steps_out is NULL"),
        (dict(adjoint_steps_out=_p(7, 2)), _INVALID, "backward_implicit: adjoint_steps_out must be 4-byte aligned"),
        (dict(adjoint_q_out=_p(8, 2)), _INVALID, "backward_implicit: adjoint_q_out must be 4-byte aligned"),
        (dict(gr=None), _INVALID, _STRUCTS),
        (dict(w=dict(struct_size=8)), _INVALID, _STRUCTS),
        (dict(pos=None), _INVALID, "a required pointer is NULL"),
        (dict(w=dict(bu_w2=None)), _INVALID, "a weight pointer is NULL"),
        (dict(gr=dict(d_bu_b2=None)), _INVALID, "gradient pointers: all MLP/token/pos outputs are needed"),
        (dict(gr=dict(d_state0=_p(29))), _INVALID,
         "backward_implicit: d_state0 and d_init must be NULL (the fixed point does not depend on the start state)"),
        (dict(gr=dict(d_init=_p(30))), _INVALID,
         "backward_implicit: d_state0 and d_init must be NULL (the fixed point does not depend on the start state)"),
        (dict(adjoint_tol=_NAN, deterministic=2), _INVALID, "backward_implicit: adjoint_tol is NaN"),
        (dict(adjoint_q_out=_p(8, 2), w=None), _INVALID, "backward_implicit: adjoint_q_out must be 4-byte aligned"),
        (dict(gr=dict(d_state0=_p(29), d_tokens=None)), _INVALID, "gradient pointers: all MLP/token/pos outputs are needed"),
        (dict(gr=dict(d_state0=_p(29)), w=dict(td_b1=None)), _INVALID, "a weight pointer is NULL"),
      ]],

    ("islands", dict(labels=None), _INVALID, "a required pointer is NULL"),
    ("islands", dict(slabs=0), _INVALID,
     "islands: need 1 <= slabs, levels <= 65535, side_h * side_w <= 8192, dim % 4 == 0"),
    ("islands", dict(side_h=128, side_w=128), _INVALID,
     "islands: need 1 <= slabs, levels <= 65535, side_h * side_w <= 8192, dim % 4 == 0"),
    ("islands", dict(dim=6), _INVALID, "islands: need 1 <= slabs, levels <= 65535, side_h * side_w <= 8192, dim % 4 == 0"),
    ("islands", dict(states=_p(1, 8)), _INVALID, "states must be 16-byte aligned"),
    ("islands", dict(states=None, levels=0), _INVALID, "a required pointer is NULL"),
    ("islands", dict(levels=0, states=_p(1, 8)), _INVALID,
     "islands: need 1 <= slabs, levels <= 65535, side_h * side_w <= 8192, dim % 4 == 0"),
]


def _struct(cls, keys, first, over):
    if over is None:
        return None
    s = cls(ctypes.sizeof(cls), *[_p(first + i) for i in range(len(keys))])
    for k, v in over.items():
        setattr(s, k, v)
    return s


def _cfg_struct(over):
    if over is None:
        return None
    kw = {**dict(dim=64, levels=3, n=16, precision="bf16"), **over}
    cfg = _native.make_cfg(kw["dim"], kw["levels"], kw["n"], False, 0, 0, kw["precision"])
    cfg.struct_size = kw.get("struct_size", cfg.struct_size)
    return cfg


def _needed_bytes(sym, args, cfg):
    if sym == "pack_weights":
        return _native.packed_weight_bytes(cfg)
    name = "glom_b200_settle_queue_workspace_bytes" if "queue" in sym else "glom_b200_settle_video_workspace_bytes"
    return _native._bytes(name, ctypes.byref(cfg), args["slots"], args["max_iters"])


@pytest.mark.parametrize("sym,over,code,text", _ERROR_CASES,
                         ids=[f"{c[0]}-{i}" for i, c in enumerate(_ERROR_CASES)])
def test_argument_errors_have_exact_text_code_and_order(sym, over, code, text):
    lib = _native.load()
    args = dict(_CALLS[sym])
    for k, v in over.items():        # a dict overrides fields of the struct argument
        args[k] = {**args[k], **v} if isinstance(v, dict) else v
    # the structs must outlive the call
    held = dict(cfg=_cfg_struct(args.get("cfg")), w=_struct(_native.WeightsRef, _W_KEYS, 10, args.get("w")),
                gr=_struct(_native.Grads, _G_KEYS, 20, args.get("gr")))
    call = [(ctypes.byref(held[k]) if held[k] is not None else None) if k in held else v for k, v in args.items()]
    rc = getattr(lib, "glom_b200_" + sym)(*call)
    want = text.replace("{need}", str(_needed_bytes(sym, args, held["cfg"]))) if "{need}" in text else text
    assert (rc, lib.glom_b200_last_error().decode()) == (code, want)


@pytest.mark.parametrize("over", [dict(batch=0), dict(patch=0), dict(dim=0), dict(height=6), dict(width=30), dict(out=False)])
def test_tokeniser_workspace_sizes_reject_bad_geometry(over):
    lib = _native.load()
    a = {**_IMG, "out": True, **over}
    out = ctypes.c_size_t()
    ref = ctypes.byref(out) if a["out"] else None
    assert lib.glom_b200_tokenize_workspace_bytes(a["batch"], a["height"], a["width"], a["patch"], a["dim"], 1, ref) == -1
    assert lib.glom_b200_last_error().decode() == "bad tokeniser geometry"
    if "dim" not in over:       # the backward's scratch does not depend on dim
        assert lib.glom_b200_tokenize_backward_workspace_bytes(a["batch"], a["height"], a["width"], a["patch"], 1, ref) == -1
        assert lib.glom_b200_last_error().decode() == "tokeniser backward: bad arguments"


def test_forward_on_cpu_tensor_raises():
    m = G.Glom(dim=64, levels=3, image_size=28, patch_size=7)
    with torch.no_grad(), pytest.raises(RuntimeError, match="no CPU fallback"):
        m(torch.randn(1, 3, 28, 28))


def test_state_dict_surface_matches_reference_layout():
    m = G.Glom(dim=64, levels=3, image_size=28, patch_size=7, local_consensus_radius=1.5)
    sd = m.state_dict()
    want = {
        "init_levels": (3, 64), "image_to_tokens.1.weight": (64, 147), "image_to_tokens.1.bias": (64,),
        "pos_emb.weight": (16, 64), "bottom_up.net.1.weight": (768, 64, 1), "bottom_up.net.1.bias": (768,),
        "bottom_up.net.3.weight": (192, 256, 1), "bottom_up.net.3.bias": (192,),
        "top_down.net.1.weight": (512, 64, 1), "top_down.net.1.bias": (512,),
        "top_down.net.3.weight": (128, 256, 1), "top_down.net.3.bias": (128,),
        "attention.non_local_mask": (1, 16, 16),
    }
    assert {k: tuple(v.shape) for k, v in sd.items()} == want
    assert m.levels == 3


@pytest.mark.parametrize("how", ["deepcopy", "pickle", "float"])
def test_copies_and_conversions_drop_the_device_caches(how):
    """deepcopy, a pickle round trip and .float() reset the packed weights, the scratch buffers, the resume state and the
    staged tokens; the parameters and the other attributes survive."""
    import copy
    import pickle
    torch.manual_seed(0)
    m = G.Glom(dim=64, levels=3, image_size=28, patch_size=7)
    want = {k: v.clone() for k, v in m.state_dict().items()}
    m._packed = (("key",), torch.zeros(4))
    m._scratch = {("_workspace", 0, 0): torch.zeros(8)}
    m._resume = {"parity": 1}
    m._staged = {"version": 0}
    m._tok_launches = 2
    new = {"deepcopy": lambda: copy.deepcopy(m), "pickle": lambda: pickle.loads(pickle.dumps(m)), "float": m.float}[how]()
    assert new._packed is None and new._scratch == {} and new._resume is None and new._staged is None
    assert new._tok_launches == 2
    got = new.state_dict()
    assert got.keys() == want.keys() and all(torch.equal(got[k], want[k]) for k in want)
    if how != "float":
        assert m._packed is not None and m._scratch and m._resume and m._staged     # the original keeps its caches


def test_radius_mask_params_follow_the_buffer():
    from oracle.glom_oracle import radius_mask
    for side, r in [(4, 1.5), (4, 1), (8, 2), (8, 2.9), (6, 10)]:
        m = G.Glom(dim=64, levels=2, image_size=side * 4, patch_size=4, local_consensus_radius=r)
        assert np.array_equal(m.attention.non_local_mask[0].numpy(), radius_mask(side, r))
        s, d2 = m.attention.mask_params(side * side)
        hh, ww = np.meshgrid(np.arange(side), np.arange(side), indexing="ij")
        co = np.stack([hh.ravel(), ww.ravel()], -1)
        dd = ((co[:, None] - co[None]) ** 2).sum(-1)
        assert s == side and np.array_equal(dd > d2, radius_mask(side, r))


def test_shard_range_covers_batch():
    for batch in (1, 7, 32, 256):
        for world in (1, 2, 3, 8):
            spans = [shard_range(batch, r, world) for r in range(world)]
            assert spans[0][0] == 0 and spans[-1][1] == batch
            assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))


def _gloo_worker(rank, world, port, q):
    import torch.distributed as dist
    from golden_util import inputs, load
    from oracle import glom_oracle as O
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    case, params, outs = load("mid_consensus_self")
    img, _ = inputs(case)
    s, e = shard_range(img.shape[0], rank, world)
    mine = O.glom_forward(params, img[s:e], patch_size=case["patch_size"], iters=case["iters"],
                          consensus_self=True, dtype=np.float32)
    t = torch.from_numpy(np.ascontiguousarray(mine))
    gathered = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(gathered, t)                      # off the timed path; only to check the partition
    elapsed = torch.tensor([1.0 + rank])
    dist.all_reduce(elapsed, op=dist.ReduceOp.MAX)    # bench.py's max-over-ranks timing reduction
    if rank == 0:
        full = torch.cat(gathered).numpy()
        q.put((float(np.abs(full - outs["out0"]).max()), float(elapsed.item())))
    dist.barrier()
    dist.destroy_process_group()


def test_batch_sharding_two_ranks_gloo():
    """world_size 2 on gloo: each rank updates its own images with no data-path collective; the
    concatenation equals the unsharded reference output (golden)."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 2000
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    err, tmax = q.get(timeout=120)
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    assert err <= 1e-4 and tmax == 2.0


def _dp_worker(rank, world, port, q):
    import torch.distributed as dist
    from glom_pytorch_b200.dp import allreduce_gradients, broadcast_parameters
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.manual_seed(100 + rank)                       # deliberately different init per rank
    m = G.Glom(dim=64, levels=3, image_size=28, patch_size=7)
    broadcast_parameters(m, src=0)
    ref = [p.detach().clone() for p in m.parameters()]
    gens = torch.Generator().manual_seed(7)
    for i, p in enumerate(m.parameters()):              # rank r holds gradient (r + 1) * base_i; init_levels has none on rank 1
        base = torch.randn(p.shape, generator=gens)
        p.grad = None if (rank == 1 and i == 0) else (rank + 1) * base
    calls = allreduce_gradients(m, bucket_bytes=64 << 10)
    gens = torch.Generator().manual_seed(7)
    err = 0.0
    for i, p in enumerate(m.parameters()):
        base = torch.randn(p.shape, generator=gens)
        want = base * (1.0 / 2.0 if i == 0 else 1.5)    # mean of (1, 2) * base; param 0: (1, 0) * base
        err = max(err, float((p.grad - want).abs().max()))
    same = all(torch.equal(a, b) for a, b in zip(ref, [p.detach() for p in m.parameters()]))
    t = torch.tensor([float(ref[3].sum())])
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    t2 = torch.tensor([float(ref[3].sum())])
    dist.all_reduce(t2, op=dist.ReduceOp.MIN)
    if rank == 0:
        q.put((err, calls, same, float(t.item() - t2.item())))
    dist.barrier()
    dist.destroy_process_group()


def test_data_parallel_gradient_allreduce_two_ranks_gloo():
    """the only collective of the path -- bucketed gradient averaging over the ranks (NCCL on the
    box, gloo here), incl. a parameter that has no gradient on one rank, and the setup-time parameter broadcast."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + os.getpid() % 2000
    procs = [ctx.Process(target=_dp_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    err, calls, same, spread = q.get(timeout=180)
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    assert err <= 1e-6 and calls >= 2 and same and spread == 0.0
