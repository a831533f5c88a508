"""Memory bounds of every engine entry point: each call reads only its inputs and writes only its outputs.

The oracle suites check the values inside each output.  This file checks the bytes around them.  Every pointer argument
of a C-ABI call gets its own `Fence`: one uint8 buffer laid out as [front guard | payload | back guard].  Each guard is
at least 1 MiB and at least one 256-row tile of that tensor (256 x its row bytes).  The payload sits at the alignment
the ABI demands (1024 for packed weights and workspaces, 16 for fp32 tensors, 4 for int32 vectors) and ends flush
against the back guard.  A workspace payload is exactly the `*_workspace_bytes` value, and that value is what the call
gets as its size.  `pos` is its own slot of exactly n rows, not a view into the whole embedding table.

`fenced_run` fills every buffer with one byte pattern, copies the inputs in, calls through `_native` with raw pointers,
synchronises, and then checks:
  - every guard byte still holds the pattern (a stray store), and every input payload still holds its input;
  - for each pattern in turn: 0x00; 0xFF (NaN in fp32 and bf16, -1 in int32: poisons a read that is masked by a
    multiply with zero); 0x7F (3.39e38 in fp32 and bf16, about 2.1e9 in int32: dominates fmaxf and running maxima,
    which swallow NaN, and breaks int comparisons);
  - the outputs of the three patterns are bit-identical.  A read past an input or an output element left unwritten
    (outputs written in full keep the pattern in their payload) makes them differ;
  - the outputs are bit-identical to the same operation through the public API (Glom.forward, settle, settle_queue,
    settle_video, tokens, islands, the autograd Functions under torch.use_deterministic_algorithms).  The atomic paths
    (the default backward, the default tokeniser d_bias) are instead held to test_backward_oracle.TOL of the
    deterministic run.
Gradients are ACCUMULATED into (include/glom_b200.h).  Their payloads get zeros for the comparisons above, and a second
run pre-fills them with a random R of the gradient's size, one to two times its RMS, with a random sign.  That run must
give |got - (R + g)| <= ACC_C u (|R| + |g|) elementwise, u = 2^-24, g the zero-prefilled result.  An entry point that
overwrites instead of adding misses that bound by about |R| / (ACC_C u |R|) = 2^24 / ACC_C, 1.1e6 (the CPU
self-test shows it).

What this cannot see: a stray access farther than a guard's width from its tensor, and a read whose value never reaches
an output.

CPU: the coverage table against _native.SIGNATURES, and fake torch "kernels" on CPU fences: every fault the harness is
for is flagged, and its in-bounds twin passes.

Observed on one H100 80GB HBM3 (132 SMs): every guard intact and every output bit-identical across the patterns and
to the public API; accumulate contract at most 4.98 u (|R| + |g|) (the fixed-order backward at T = 3), against the
bound of 15; the multi-tile case at B = 17 (K1 20.6, K2 3.1 tiles per pair); about 45 s for the GPU part of the file,
peak allocation 5.35 GiB (the multi-tile case).
"""
import contextlib
import ctypes
import math

import numpy as np
import pytest
import torch

import glom_pytorch_b200 as G
from glom_pytorch_b200 import _native
from glom_pytorch_b200.glom import _ColumnUpdate, _SettleImplicit, _Tokenize
from oracle import glom_oracle as O

import test_backward_oracle as BO
import test_cuda_core_oracle as CC
import test_forward_oracle as FO
import test_production_batch as PB
import test_settle as ST
import test_settle_implicit as SI
import test_settle_video as SV
from test_deterministic_backward import deterministic

DEV = "cuda:0"
PATTERNS = (0x00, 0xFF, 0x7F)
MIN_GUARD = 1 << 20
U32 = 2.0 ** -24
ACC_C = 15.0                  # accumulate contract: |got - (R + g)| <= ACC_C u (|R| + |g|); 4.98 observed
GRAD_FIELDS = tuple(k for k, _ in _native.Grads._fields_[1:])
WEIGHT_FIELDS = tuple(k for k, _ in _native.WeightsRef._fields_[1:])
# ABI gradient names -> the names test_backward_oracle.errors blocks by
BO_NAME = {"d_tokens": "d_tokens", "d_pos": "pos_emb.weight", "d_state0": "d_state0", "d_init": "init_levels",
           **{g: n for g, n in zip(GRAD_FIELDS[4:], BO.NAMES)}}
TOK_BO = {"d_img": "d_img", "d_weight": "image_to_tokens.1.weight", "d_bias": "image_to_tokens.1.bias"}


# ====================================================================================================== the harness
class Fence:
    """One ABI argument in its own uint8 buffer [front guard | payload | back guard].

    kind: "in" (copied in, must be left unchanged), "out" (written in full: its payload keeps the fill pattern, so an
    element left unwritten shows), "acc" (accumulated into: zeros or a given prefill in the payload), "ws" (scratch).
    row_dims: trailing dimensions that make one row (2 for a (.., L, d) state), for the 256-row guard.  shift: bytes
    added to the aligned payload offset (a deliberately misaligned input)."""

    def __init__(self, name, shape, dtype=torch.float32, kind="in", *, align=None, row_dims=1, nbytes=None, shift=0,
                 device=DEV):
        self.name, self.shape, self.dtype, self.kind = name, tuple(shape), dtype, kind
        esize = torch.empty((), dtype=dtype).element_size()
        self.nbytes = nbytes if nbytes is not None else math.prod(self.shape) * esize
        if align is None:
            align = 1024 if dtype == torch.uint8 else 16 if dtype == torch.float32 else esize
        row = math.prod(self.shape[-row_dims:]) * esize if self.shape and dtype != torch.uint8 else 0
        self.guard = max(MIN_GUARD, 256 * row)
        self.raw = torch.empty(2 * self.guard + align + shift + self.nbytes, dtype=torch.uint8, device=device)
        base = self.raw.data_ptr()
        self.off = self.guard + (-(base + self.guard)) % align + shift
        self.payload = self.raw[self.off:self.off + self.nbytes]

    @property
    def ptr(self):
        return self.raw.data_ptr() + self.off

    @property
    def tensor(self):
        return self.payload.view(self.dtype).view(self.shape) if self.dtype != torch.uint8 else self.payload

    def violations(self, pattern):
        """-> text for every guard byte that no longer holds `pattern` (empty list: intact)."""
        out = []
        for side, region, origin in (("front", self.raw[:self.off], self.off), ("back", self.raw[self.off + self.nbytes:], 0)):
            bad = (region != pattern).nonzero().flatten()
            if bad.numel():
                first, last = int(bad[0]) - origin, int(bad[-1]) - origin
                vals = " ".join(f"{v:02x}" for v in region[bad[:16]].tolist())
                where = "the payload start" if side == "front" else "the payload end"
                out.append(f"{self.name}: {bad.numel()} {side}-guard bytes changed at offsets {first} .. {last} "
                           f"relative to {where} (pattern 0x{pattern:02X}; first bytes written: {vals})")
        return out


def _sync(fences):
    if any(f.raw.is_cuda for f in fences.values()):
        torch.cuda.synchronize()


def same_bits(a, b, what):
    a, b = a.contiguous(), b.contiguous()
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape, a.dtype, b.dtype)
    if not torch.equal(a.view(torch.uint8), b.view(torch.uint8)):
        diff = (a.view(torch.uint8) != b.view(torch.uint8)).view(a.shape + (a.element_size(),)).any(-1)
        idx = diff.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(diff.sum())} elements differ, first at {idx}: "
                             f"{a[tuple(idx)].item()} vs {b[tuple(idx)].item()}")


def fenced_run(fences, inputs, call, *, patterns=PATTERNS, prefill=None, exact=True):
    """For each pattern: fill every fence, copy `inputs` (name -> tensor) in, pre-fill the "acc" payloads (`prefill`:
    name -> tensor, default zeros), call(fences), synchronise, and assert that every guard byte still holds the pattern
    and every input is unchanged.  exact: the outputs of all patterns are bit-identical.  -> one {name: output copy}
    per pattern (outputs: the "out" and "acc" fences)."""
    prefill = prefill or {}
    results = []
    for pat in patterns:
        for f in fences.values():
            f.raw.fill_(pat)
        for name, f in fences.items():
            if f.kind == "acc":
                f.tensor.copy_(prefill[name] if name in prefill else torch.zeros(f.shape, dtype=f.dtype))
        for name, v in inputs.items():
            fences[name].tensor.copy_(v)
        call(fences)
        _sync(fences)
        bad = [v for f in fences.values() for v in f.violations(pat)]
        assert not bad, "\n".join(bad)
        for name, v in inputs.items():
            t = fences[name].tensor
            same_bits(t, v.to(t.device, t.dtype).reshape(t.shape), f"input {name} changed (pattern 0x{pat:02X})")
        results.append({k: f.tensor.clone() for k, f in fences.items() if f.kind in ("out", "acc")})
    if exact:
        for pat, r in zip(patterns[1:], results[1:]):
            for k in r:
                same_bits(r[k], results[0][k], f"output {k}: pattern 0x{pat:02X} vs 0x{patterns[0]:02X}")
    return results


def accumulate_ratio(got, R, g):
    """max over elements of |got - (R + g)| / (u (|R| + |g|)), in float64."""
    got, R, g = (t.detach().to("cpu", torch.float64) for t in (got, R, g))
    den = U32 * (R.abs() + g.abs())
    err = (got - (R + g)).abs()
    assert not (err[den == 0] > 0).any()
    return float((err / den.clamp_min(1e-300)).max()) if err.numel() else 0.0


def random_prefill(g, seed):
    """R: one to two times the RMS of g per element, random sign (never near zero, so an overwrite always shows)."""
    gen = torch.Generator().manual_seed(seed)
    rms = max(float(g.double().square().mean().sqrt()), 1e-3) if g.numel() else 1.0
    mag = 1.0 + torch.rand(g.shape, generator=gen, dtype=torch.float64)
    sign = torch.where(torch.rand(g.shape, generator=gen) < 0.5, -1.0, 1.0).double()
    return (rms * mag * sign).float().to(g.device)


OBSERVED = {}                  # accumulate ratios by case (printed; the docstring records the worst)


def check_accumulate(got, R, g, what):
    worst = max(accumulate_ratio(got[k], R[k], g[k]) for k in R)
    OBSERVED[what] = worst
    print(f"[guard] accumulate {what}: {worst:.3g} u (|R| + |g|) (bound {ACC_C:g})")
    assert worst <= ACC_C, (what, worst)


def accumulate_twice(fences, inputs, call, acc_names, what, *, exact=True, seed=0):
    """fenced_run with zero-prefilled gradients, then with R -> (the zero-prefilled outputs of each pattern, the
    R-prefilled outputs minus R of each pattern).  The bound on R + g holds elementwise for the fixed-order paths
    (exact), checked here; the atomic paths sum in another order in each run, so there the caller compares got - R with
    the deterministic result."""
    zero = fenced_run(fences, inputs, call, exact=exact)
    R = {k: random_prefill(zero[0][k], seed + i) for i, k in enumerate(acc_names)}
    withR = fenced_run(fences, inputs, call, prefill=R, exact=exact)
    if exact:
        check_accumulate(withR[0], R, zero[0], what)
    return zero, [{k: r[k] - R[k] if k in R else r[k] for k in r} for r in withR]


def check_gradients(zero, withR, ref, exact, tol, what, bo_name, L, n):
    """Fixed-order paths: every pattern's zero-prefilled gradients are the public ones bit for bit (the R runs met the
    accumulate bound).  Atomic paths: every run, zero-prefilled and R-prefilled minus R, within `tol` of them
    (test_backward_oracle.errors, blocked by the names `bo_name` maps to)."""
    if exact:
        for k in ref:
            same_bits(zero[0][k], ref[k], (what, k))
        return
    for res in zero + withR:
        BO.check(BO.errors({bo_name[k]: res[k] for k in ref}, {bo_name[k]: v for k, v in ref.items()}, L, n), tol, what)


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ====================================================================================================== coverage
# every C-ABI symbol that touches device memory -> the GPU test of this file that runs it fenced
COVERAGE = {
    "glom_b200_pack_weights": "test_forward_fenced",
    "glom_b200_forward": "test_forward_fenced",
    "glom_b200_forward_resume": "test_forward_fenced",
    "glom_b200_forward_steps": "test_steps_and_settle_fenced",
    "glom_b200_settle": "test_steps_and_settle_fenced",
    "glom_b200_settle_all": "test_steps_and_settle_fenced",
    "glom_b200_settle_queue_begin": "test_settle_queue_fenced",
    "glom_b200_settle_queue_run": "test_settle_queue_fenced",
    "glom_b200_settle_video_begin": "test_settle_video_fenced",
    "glom_b200_settle_video_run": "test_settle_video_fenced",
    "glom_b200_tokenize": "test_tokenize_fenced",
    "glom_b200_tokenize_backward": "test_tokenize_fenced",
    "glom_b200_tokenize_backward_ex": "test_tokenize_fenced",
    "glom_b200_backward": "test_backward_fenced",
    "glom_b200_backward_steps": "test_backward_fenced",
    "glom_b200_backward_ex": "test_backward_fenced",
    "glom_b200_backward_implicit": "test_backward_implicit_fenced",
    "glom_b200_islands": "test_islands_fenced",
    "glom_b200_clock_probe": "test_clock_probe_fenced",
}
# host-only queries and measurement aids: no device pointer, or host arrays only
NOT_DEVICE = {"glom_b200_last_error", "glom_b200_last_launch_count", "glom_b200_profile_begin", "glom_b200_profile_end",
              "glom_b200_kernel_clocks", "glom_b200_abi_version"}


def _takes_device_pointer(argtypes):
    return any(a in (ctypes.c_void_p, ctypes.POINTER(_native.WeightsRef), ctypes.POINTER(_native.Grads)) for a in argtypes)


def test_every_device_entry_point_has_a_fenced_case():
    """A symbol of _native.SIGNATURES that takes a device pointer (not a *_bytes / *_offset query or a measurement
    aid) must be run fenced by a GPU test of this file."""
    missing = []
    for name, (_, argtypes) in _native.SIGNATURES.items():
        if name in NOT_DEVICE or name.endswith("_bytes") or name.endswith("_offset"):
            continue
        if _takes_device_pointer(argtypes) and name not in COVERAGE:
            missing.append(name)
    assert not missing, f"entry points without a fenced GPU case: {missing}"
    for name, test in COVERAGE.items():
        assert name in _native.SIGNATURES, name
        fn = globals().get(test)
        assert fn is not None and any(m.name == "gpu" for m in getattr(fn, "pytestmark", [])), (name, test)


# ====================================================================================================== CPU self-tests
def _cpu_fences(**spec):
    return {k: Fence(k, *v[:2], kind=v[2], device="cpu", **(v[3] if len(v) > 3 else {})) for k, v in spec.items()}


def _flags(fences, inputs, call, **kw):
    """-> the AssertionError text fenced_run raises, or None."""
    try:
        fenced_run(fences, inputs, call, **kw)
    except AssertionError as e:
        return str(e)
    return None


X = torch.randn(8, 4, generator=torch.Generator().manual_seed(0))


def _store_past_end(f, twin):
    o = f["out"]
    n = o.nbytes // 4 + (0 if twin else 1)
    o.raw[o.off:o.off + 4 * n].view(torch.float32).copy_(torch.cat([f["x"].tensor.flatten(), torch.ones(1)])[:n])


def _store_before_start(f, twin):
    o = f["out"]
    lo = o.off - (0 if twin else 4)
    o.raw[lo:lo + o.nbytes].view(torch.float32).copy_(f["x"].tensor.flatten())
    if not twin:
        o.tensor.view(-1)[-1] = f["x"].tensor.view(-1)[-1]


def _ws_byte_past(f, twin):
    w = f["ws"]
    w.raw[w.off + w.nbytes - (1 if twin else 0)] = 7
    f["out"].tensor.copy_(f["x"].tensor)


def _unwritten(f, twin):
    f["out"].tensor.view(-1)[:None if twin else -1].copy_(f["x"].tensor.view(-1)[:None if twin else -1])


def _max_past_end(f, twin):
    """out[c] = max over rows of x[:, c], reading one row too many; fmax swallows NaN like fmaxf."""
    x = f["x"]
    rows = x.shape[0] + (0 if twin else 1)
    v = x.raw[x.off:x.off + 4 * rows * x.shape[1]].view(torch.float32).view(rows, x.shape[1])
    out = v[0].clone()
    for r in range(1, rows):
        out = torch.fmax(out, v[r])
    f["out"].tensor.copy_(out)


def _masked_past_end(f, twin):
    """out[c] = sum over rows of x[:, c] * mask[r], reading one row too many with mask 0 for it."""
    x = f["x"]
    rows = x.shape[0] + (0 if twin else 1)
    v = x.raw[x.off:x.off + 4 * rows * x.shape[1]].view(torch.float32).view(rows, x.shape[1])
    mask = torch.ones(rows)
    mask[x.shape[0]:] = 0
    f["out"].tensor.copy_((v * mask[:, None]).sum(0))


def _steps_predicate(f, twin):
    """A warp-collective 'is any image of the block frozen at step t' over lanes 0 .. B, one lane too many."""
    s, t = f["steps"], 2
    lanes = s.shape[0] + (0 if twin else 1)
    v = s.raw[s.off:s.off + 4 * lanes].view(torch.int32)
    frozen = bool((v <= t).any())
    f["out"].tensor.copy_(f["x"].tensor + (0.0 if frozen else 1.0))


@pytest.mark.parametrize("fault", ["store_past_end", "store_before_start", "ws_byte_past_end", "unwritten_element",
                                   "max_read_past_end", "masked_read_past_end", "steps_read_past_end"])
def test_harness_flags_fault_and_passes_twin(fault):
    spec = dict(x=((8, 4), torch.float32, "in"), out=((8, 4), torch.float32, "out"),
                ws=((), torch.uint8, "ws", dict(nbytes=3000)))
    inputs = {"x": X}
    fn = {"store_past_end": _store_past_end, "store_before_start": _store_before_start, "ws_byte_past_end": _ws_byte_past,
          "unwritten_element": _unwritten, "max_read_past_end": _max_past_end,
          "masked_read_past_end": _masked_past_end, "steps_read_past_end": _steps_predicate}[fault]
    if fault in ("max_read_past_end", "masked_read_past_end"):
        spec["out"] = ((4,), torch.float32, "out")
    if fault == "max_read_past_end":
        inputs = {"x": X.abs() + 1.0}              # positive: a zero row changes no maximum either
    if fault == "steps_read_past_end":
        spec["steps"] = ((5,), torch.int32, "in")
        inputs["steps"] = torch.tensor([3, 4, 5, 6, 7], dtype=torch.int32)   # every image live at t = 2
    assert _flags(_cpu_fences(**spec), inputs, lambda f: fn(f, True)) is None
    msg = _flags(_cpu_fences(**spec), inputs, lambda f: fn(f, False))
    assert msg is not None, fault
    print(f"[guard] {fault}: {msg.splitlines()[0]}")
    if fault == "max_read_past_end":               # only 0x7F moves a maximum of positive values past a NaN-swallowing fmax
        assert _flags(_cpu_fences(**spec), inputs, lambda f: fn(f, False), patterns=(0x00, 0xFF)) is None
        assert _flags(_cpu_fences(**spec), inputs, lambda f: fn(f, False), patterns=(0x00, 0x7F)) is not None
    if fault == "masked_read_past_end":            # only 0xFF survives a multiply with zero
        assert _flags(_cpu_fences(**spec), inputs, lambda f: fn(f, False), patterns=(0x00, 0x7F)) is None
        assert _flags(_cpu_fences(**spec), inputs, lambda f: fn(f, False), patterns=(0x00, 0xFF)) is not None
    if fault in ("store_past_end", "store_before_start", "ws_byte_past_end"):
        assert "guard bytes changed" in msg


def test_harness_flags_overwritten_accumulator():
    """d += g passes the accumulate bound; d = g misses it by about 2^24 / ACC_C."""
    g = torch.randn(64, generator=torch.Generator().manual_seed(3))

    def run(overwrite):
        f = _cpu_fences(x=((64,), torch.float32, "in"), d=((64,), torch.float32, "acc"))

        def call(f):
            if overwrite:
                f["d"].tensor.copy_(f["x"].tensor)
            else:
                f["d"].tensor.add_(f["x"].tensor)
        return accumulate_twice(f, {"x": g}, call, ["d"], f"cpu overwrite={overwrite}")
    run(False)
    with pytest.raises(AssertionError):
        run(True)
    assert OBSERVED["cpu overwrite=True"] > 1e5 and OBSERVED["cpu overwrite=False"] <= 1.0


def test_harness_layout():
    """Payload at its alignment, flush against the back guard, guards of at least 1 MiB and one 256-row tile."""
    f = Fence("s", (3, 9, 6, 512), kind="out", row_dims=2, device="cpu")
    assert f.ptr % 16 == 0 and f.guard == 256 * 6 * 512 * 4 and f.off >= f.guard
    assert f.raw.numel() - (f.off + f.nbytes) >= f.guard
    w = Fence("ws", (), torch.uint8, "ws", nbytes=5000, device="cpu")
    assert w.ptr % 1024 == 0 and w.guard == MIN_GUARD and w.payload.numel() == 5000
    m = Fence("lv", (2, 3), shift=4, device="cpu")
    assert m.ptr % 16 == 4


# ====================================================================================================== GPU helpers
def _weights32(m):
    return [q.detach().float().contiguous() for q in m._mlp_params()]


def _packed_sections(d, L, precision):
    """(offset, bytes) of W1, W2, b1, b2 in the packed buffer (glom_api.cu packed_layout); the gaps are padding."""
    es, Gs, out, off = (2 if precision == "bf16" else 4), 2 * L - 1, [], 0
    for nb in (Gs * 4 * d * d * es, L * d * 8 * d * es, Gs * 4 * d * 4, L * d * 4):
        out.append((off, nb))
        off = -(-(off + nb) // 1024) * 1024
    return out, off


def _pack_fenced(m, n, precision):
    """glom_b200_pack_weights fenced -> the packed bytes (sections bit-identical across patterns)."""
    cfg = m.engine_cfg(n, precision)
    nbytes = _native.packed_weight_bytes(cfg)
    sections, total = _packed_sections(m.dim, m.levels, precision)
    assert total == nbytes
    wts = _weights32(m)
    f = {k: Fence(k, w.shape, row_dims=w.dim() - 1 or 1) for k, w in zip(WEIGHT_FIELDS, wts)}
    f["packed"] = Fence("packed", (), torch.uint8, "out", nbytes=nbytes)
    res = fenced_run(f, dict(zip(WEIGHT_FIELDS, wts)),
                     lambda f: _native.pack_weights(cfg, [f[k].ptr for k in WEIGHT_FIELDS], f["packed"].ptr, nbytes,
                                                    _stream()), exact=False)
    for r in res[1:]:
        for off, nb in sections:
            same_bits(r["packed"][off:off + nb], res[0]["packed"][off:off + nb], f"packed section at {off}")
    if precision == m.precision:
        public = m._packed_weights(cfg, torch.device(DEV), _stream())
        for off, nb in sections:
            same_bits(res[0]["packed"][off:off + nb], public[off:off + nb], f"packed vs Glom._packed_weights at {off}")
    return res[0]["packed"]


def _state_fence(name, shape, kind):
    return Fence(name, shape, kind=kind, row_dims=2)


def _engine_inputs(m, img, n):
    with torch.no_grad():
        tokens = m.tokens(img)
    return tokens, m.pos_emb.weight[:n].detach().float().clone(), m.init_levels.detach().float().clone()


# ---------------------------------------------------------------------------------------------- forward shapes
NEW_SHAPES = {
    # (dim, L, image_size, patch, (H, W), B, precision): the smallest legal n, never run by the oracle suites
    "d64_n1": (64, 2, 4, 4, (4, 4), 3, "bf16"),
    "d64_n2": (64, 2, 8, 4, (4, 8), 3, "bf16"),
    # fp32 engine: n = 15 of 25 pos rows, d / 4 = 9
    "fp32_d36_n15": (36, 3, 15, 3, (9, 15), 2, "fp32"),
}
FWD_SHAPES = ["d64_n9", "d192_n36", "d320_n144_r3", "d384_n100", "d256_nonsquare", "d768_L2", "d128_n784_r6.5_self",
              "d64_n1600", "d64_n1", "d64_n2", "fp32_d36_n15", "fp32_d100_L3_54x54_p2_B1"]


def _fwd_model(name, batch=None):
    """-> (model in eval mode, img, S, n) on the GPU."""
    if name in NEW_SHAPES:
        dim, L, isz, p, hw, B, precision = NEW_SHAPES[name]
        B = batch or B
        params = O.synth_params(dim, L, isz, p, seed=0)
        m = G.Glom(dim=dim, levels=L, image_size=isz, patch_size=p, precision=precision)
        m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=False)
        g = torch.Generator().manual_seed(31)
        n = (hw[0] // p) * (hw[1] // p)
        img, S = torch.randn((B, 3) + hw, generator=g), torch.randn(B, n, L, dim, generator=g)
    elif name.startswith("fp32_"):
        m, img, S, n, _ = CC._model(name[len("fp32_"):])
    else:
        m, img, S, n = FO._model(name, "bf16", batch=batch)
    return m.to(DEV).eval(), img.to(DEV), S.to(DEV), n


def _forward_fences(m, B, n, T, return_all, ws_bytes, packed_bytes, outs=("out",)):
    L, d = m.levels, m.dim
    shape = ((T + 1, B, n, L, d) if return_all else (B, n, L, d))
    f = {"packed": Fence("packed", (), torch.uint8, "in", nbytes=packed_bytes),
         "tokens": Fence("tokens", (B, n, d)), "pos": Fence("pos", (n, d)),
         "state_in": _state_fence("state_in", (B, n, L, d), "in"), "init": Fence("init", (L, d)),
         "ws": Fence("ws", (), torch.uint8, "ws", nbytes=ws_bytes)}
    for o in outs:
        f[o] = _state_fence(o, shape, "out")
    return f


@pytest.mark.gpu
@pytest.mark.parametrize("name", FWD_SHAPES)
def test_forward_fenced(name):
    """pack_weights (both precisions), forward at iters 0 / 1 / 3, return_all 0 / 1, state_in NULL / set, then (bf16)
    forward_resume twice on the same fenced workspace (parity 1, then 0) with the previous output as state_in."""
    m, img, S, n = _fwd_model(name)
    B, L, d = img.shape[0], m.levels, m.dim
    packed = {p: _pack_fenced(m, n, p) for p in ("bf16", "fp32") if p == "fp32" or d % 64 == 0}[m.precision]
    tokens, pos, init = _engine_inputs(m, img, n)
    cfg = m.engine_cfg(n)
    for T in (0, 1, 3):
        for return_all in (0, 1):
            for start in (None, S):
                ws_bytes = _native.workspace_bytes(cfg, B, T, return_all)
                f = _forward_fences(m, B, n, T, return_all, ws_bytes, packed.numel())
                inputs = {"packed": packed, "tokens": tokens, "pos": pos, "init": init}
                if start is not None:
                    inputs["state_in"] = start

                def call(f):
                    _native.forward(cfg, f["packed"].ptr, f["tokens"].ptr, f["pos"].ptr,
                                    None if start is None else f["state_in"].ptr, f["init"].ptr, f["out"].ptr, B, T,
                                    return_all, f["ws"].ptr, ws_bytes, _stream())
                got = fenced_run(f, inputs, call)[0]["out"]
                with torch.no_grad():
                    want = m(img, iters=T, levels=start, return_all=bool(return_all))
                same_bits(got, want, (name, T, return_all, start is None))
    if m.precision != "bf16":
        return
    ws_bytes = _native.workspace_bytes(cfg, B, 3, 0)
    assert ws_bytes == _native.workspace_bytes(cfg, B, 1, 0) == _native.workspace_bytes(cfg, B, 2, 0)
    for start in (None, S):
        f = _forward_fences(m, B, n, 0, 0, ws_bytes, packed.numel(), outs=("out1", "out2", "out3"))
        inputs = {"packed": packed, "tokens": tokens, "pos": pos, "init": init}
        if start is not None:
            inputs["state_in"] = start
        parities = []

        def call(f):
            _native.forward(cfg, f["packed"].ptr, f["tokens"].ptr, f["pos"].ptr, None if start is None else f["state_in"].ptr,
                            f["init"].ptr, f["out1"].ptr, B, 3, 0, f["ws"].ptr, ws_bytes, _stream())
            p = _native.forward_resume(cfg, f["packed"].ptr, f["tokens"].ptr, f["pos"].ptr, f["out1"].ptr, f["out2"].ptr,
                                       B, 1, 0, f["ws"].ptr, ws_bytes, _stream(), 1)
            q = _native.forward_resume(cfg, f["packed"].ptr, f["tokens"].ptr, f["pos"].ptr, f["out2"].ptr, f["out3"].ptr,
                                       B, 2, 0, f["ws"].ptr, ws_bytes, _stream(), p)
            parities.append((p, q))
        got = fenced_run(f, inputs, call)[0]
        assert len(set(parities)) == 1, parities
        with torch.no_grad():
            w1 = m(img, iters=3, levels=start)
            w2 = m(img, iters=1, levels=w1)                   # eval mode: the public resume path
            w3 = m(img, iters=2, levels=w2)
        for k, w in (("out1", w1), ("out2", w2), ("out3", w3)):
            same_bits(got[k], w, (name, "resume", k, start is None))


# ---------------------------------------------------------------------------------------------- per-image steps, settle
def _contracting_start(m, img, T):
    """Second MLP layers scaled by 0.1, a start near the fixed point with noise over six decades across the images, and
    a tol between the images' smallest changes: the image with the largest one never stops, the one with the smallest
    stops."""
    with torch.no_grad():
        m.bottom_up.net[3].weight.mul_(0.1)
        m.top_down.net[3].weight.mul_(0.1)
        m.invalidate_packed()
        B = img.shape[0]
        base = m(img, iters=30)
        noise = torch.randn(base.shape, generator=torch.Generator().manual_seed(2)).to(DEV)
        eps = torch.tensor([10.0 ** (-6 * b / max(B - 1, 1)) for b in range(B)], device=DEV).view(B, 1, 1, 1)
        start = (base + eps * noise * base.abs().mean()).contiguous()
        r = ST._change(m(img, iters=T, levels=start, return_all=True))
    vals = np.unique(r[np.isfinite(r) & (r > 0)])
    best = None
    for a, b in zip(vals[:-1], vals[1:]):
        if b > a * 1.02:
            tol = float(np.sqrt(a * b))
            score = len(np.unique(ST._first_stop(r, tol)))
            if best is None or score > best[0]:
                best = (score, tol)
    assert best is not None and best[0] >= 2, r
    return start, best[1]


STEP_SHAPES = {"d64_n9": 3, "d320_n144_r3": 5, "d128_n784_r6.5_self": 3}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(STEP_SHAPES))
def test_steps_and_settle_fenced(name):
    """forward_steps (return_all 0 / 1, steps including 0 and T), settle and settle_all, from state_in and from
    init_levels, with a tol that stops some images and not others."""
    T = 6
    m, img, _, n = _fwd_model(name, batch=STEP_SHAPES[name])
    B, L, d = img.shape[0], m.levels, m.dim
    start, tol = _contracting_start(m, img, T)
    packed = _pack_fenced(m, n, "bf16")
    tokens, pos, init = _engine_inputs(m, img, n)
    cfg = m.engine_cfg(n)
    steps = torch.tensor(([0, T, 2, 5, 1] * B)[:B], dtype=torch.int32)
    for lv in (start, None):
        base = {"packed": packed, "tokens": tokens, "pos": pos, "init": init}
        if lv is not None:
            base["state_in"] = lv
        for return_all in (0, 1):
            ws_bytes = _native.forward_steps_workspace_bytes(cfg, B, T, return_all)
            f = _forward_fences(m, B, n, T, return_all, ws_bytes, packed.numel())
            f["steps"] = Fence("steps", (B,), torch.int32)

            def call(f):
                _native.forward_steps(cfg, f["packed"].ptr, f["tokens"].ptr, f["pos"].ptr,
                                      None if lv is None else f["state_in"].ptr, f["init"].ptr, f["out"].ptr, B,
                                      f["steps"].ptr, T, return_all, f["ws"].ptr, ws_bytes, _stream())
            got = fenced_run(f, dict(base, steps=steps), call)[0]["out"]
            with torch.no_grad():
                want = m(img, iters=steps.tolist(), levels=lv, return_all=bool(return_all))
            same_bits(got, want, (name, "forward_steps", return_all, lv is None))
        for return_all in (0, 1):
            fn = _native.settle_all_workspace_bytes if return_all else _native.settle_workspace_bytes
            ws_bytes = fn(cfg, B, T)
            f = _forward_fences(m, B, n, T, return_all, ws_bytes, packed.numel())
            f["steps_out"] = Fence("steps_out", (B,), torch.int32, "out")

            def call(f):
                _native.settle(cfg, f["packed"].ptr, f["tokens"].ptr, f["pos"].ptr, None if lv is None else f["state_in"].ptr,
                               f["init"].ptr, f["out"].ptr, B, T, return_all, tol, f["steps_out"].ptr, f["ws"].ptr,
                               ws_bytes, _stream())
            got = fenced_run(f, base, call)[0]
            with torch.no_grad():
                want, want_steps = m.settle(img, tol, max_iters=T, levels=lv, return_all=bool(return_all))
            same_bits(got["steps_out"], want_steps, (name, "settle steps", return_all, lv is None))
            same_bits(got["out"], want, (name, "settle", return_all, lv is None))
            if lv is not None:
                assert len(torch.unique(want_steps)) >= 2, want_steps


# ---------------------------------------------------------------------------------------------- queue and video
def _slot_loop(begin, run, f, cfg, packed_ptr, args_of):
    """The host loop of _settle_slots on fenced pointers."""
    begin(cfg, *args_of(f))
    first, rounds = 0, 0
    while True:
        run(cfg, packed_ptr(f), *args_of(f), first, args_of.max_iters, f["remaining"].ptr)
        first += args_of.max_iters
        torch.cuda.synchronize()
        rounds += 1
        if int(f["remaining"].tensor[0]) == 0:
            break
        assert rounds < 64
    run(cfg, packed_ptr(f), *args_of(f), first, 0, None)


QUEUE_CASES = [("d64_n9", 7, 3), ("d64_n9", 5, 5), ("d320_n144_r3", 7, 3), ("d320_n144_r3", 5, 5)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,N,slots", QUEUE_CASES, ids=[f"{a}_N{b}_slots{c}" for a, b, c in QUEUE_CASES])
def test_settle_queue_fenced(name, N, slots):
    T = 6
    m, img, _, n = _fwd_model(name, batch=N)
    L, d = m.levels, m.dim
    start, tol = _contracting_start(m, img, T)
    packed = _pack_fenced(m, n, "bf16")
    tokens, pos, init = _engine_inputs(m, img, n)
    cfg = m.engine_cfg(n)
    ws_bytes = _native.settle_queue_workspace_bytes(cfg, slots, T)
    for lv in (start, None):
        f = {"packed": Fence("packed", (), torch.uint8, "in", nbytes=packed.numel()),
             "tokens": Fence("tokens", (N, n, d)), "pos": Fence("pos", (n, d)),
             "state_in": _state_fence("state_in", (N, n, L, d), "in"), "init": Fence("init", (L, d)),
             "out": _state_fence("out", (N, n, L, d), "out"), "steps": Fence("steps", (N,), torch.int32, "out"),
             "remaining": Fence("remaining", (1,), torch.int32, "out"),
             "ws": Fence("ws", (), torch.uint8, "ws", nbytes=ws_bytes)}
        inputs = {"packed": packed, "tokens": tokens, "pos": pos, "init": init}
        if lv is not None:
            inputs["state_in"] = lv

        def args(f):
            return (f["tokens"].ptr, f["pos"].ptr, None if lv is None else f["state_in"].ptr, f["init"].ptr, f["out"].ptr,
                    f["steps"].ptr, N, slots, T, tol, f["ws"].ptr, ws_bytes, _stream())
        args.max_iters = T
        got = fenced_run(f, inputs, lambda f: _slot_loop(_native.settle_queue_begin, _native.settle_queue_run, f, cfg,
                                                         lambda f: f["packed"].ptr, args))[0]
        with torch.no_grad():
            want, want_steps = m.settle_queue(img, tol, max_iters=T, levels=lv, slots=slots)
        same_bits(got["steps"], want_steps, (name, N, slots, "steps", lv is None))
        same_bits(got["out"], want, (name, N, slots, "levels", lv is None))


@pytest.mark.gpu
def test_settle_video_fenced():
    """S = 5 streams x F = 3 frames through 2 slots, with and without state_in."""
    m, _, isz = SV._shape_model("n64_four_images_per_block")
    S, F, slots, T = 5, 3, 2, SV.MAX_ITERS
    frames = SV._frames(S, F, isz)
    L, d = m.levels, m.dim
    with torch.no_grad():
        tokens = m.tokens(frames.reshape((S * F,) + tuple(frames.shape[2:])))
        start = SV._start(m, frames)
    n = tokens.shape[1]
    packed = _pack_fenced(m, n, "bf16")
    pos, init = m.pos_emb.weight[:n].detach().clone(), m.init_levels.detach().clone()
    cfg = m.engine_cfg(n)
    ws_bytes = _native.settle_video_workspace_bytes(cfg, slots, T)
    for lv in (start, None):
        with torch.no_grad():
            tol = SV._pick_tol(m, frames, lv)
        f = {"packed": Fence("packed", (), torch.uint8, "in", nbytes=packed.numel()),
             "tokens": Fence("tokens", (S * F, n, d)), "pos": Fence("pos", (n, d)),
             "state_in": _state_fence("state_in", (S, n, L, d), "in"), "init": Fence("init", (L, d)),
             "out": _state_fence("out", (S * F, n, L, d), "out"), "steps": Fence("steps", (S * F,), torch.int32, "out"),
             "remaining": Fence("remaining", (1,), torch.int32, "out"),
             "ws": Fence("ws", (), torch.uint8, "ws", nbytes=ws_bytes)}
        inputs = {"packed": packed, "tokens": tokens, "pos": pos, "init": init}
        if lv is not None:
            inputs["state_in"] = lv

        def args(f):
            return (f["tokens"].ptr, f["pos"].ptr, None if lv is None else f["state_in"].ptr, f["init"].ptr, f["out"].ptr,
                    f["steps"].ptr, S, F, slots, T, tol, f["ws"].ptr, ws_bytes, _stream())
        args.max_iters = T
        got = fenced_run(f, inputs, lambda f: _slot_loop(_native.settle_video_begin, _native.settle_video_run, f, cfg,
                                                         lambda f: f["packed"].ptr, args))[0]
        with torch.no_grad():
            want, want_steps = m.settle_video(frames, tol, max_iters=T, levels=lv, slots=slots)
        same_bits(got["steps"], want_steps.reshape(-1), ("video steps", lv is None))
        same_bits(got["out"], want.reshape(got["out"].shape), ("video levels", lv is None))


# ---------------------------------------------------------------------------------------------- tokeniser
# (patch, (H, W), B, dim): p = 1, 3, 14, 16; non-square in both orientations
TOK_CASES = [(1, (9, 13), 2, 64), (3, (15, 9), 2, 64), (14, (28, 42), 2, 128), (16, (48, 32), 3, 64), (3, (9, 15), 2, 36)]
SUBSETS = [(i, w, b) for i in (0, 1) for w in (0, 1) for b in (0, 1) if i or w or b]


@pytest.mark.gpu
@pytest.mark.parametrize("p,hw,B,dim", TOK_CASES, ids=[f"p{c[0]}_{c[1][0]}x{c[1][1]}_d{c[3]}" for c in TOK_CASES])
def test_tokenize_fenced(p, hw, B, dim):
    """tokenize (bf16 where dim % 64 == 0, fp32) and tokenize_backward / _ex (deterministic 0 / 1) with each non-empty
    subset of (d_img, d_weight, d_bias), against _Tokenize under the deterministic flag."""
    H, W = hw
    n = (H // p) * (W // p)
    gen = torch.Generator().manual_seed(9)
    img = torch.randn(B, 3, H, W, generator=gen).to(DEV)
    cot = torch.randn(B, n, dim, generator=gen).to(DEV)
    for precision in (("bf16", "fp32") if dim % 64 == 0 else ("fp32",)):
        torch.manual_seed(0)
        m = G.Glom(dim=dim, levels=2, image_size=max(H, W), patch_size=p, precision=precision).to(DEV)
        lin = m.image_to_tokens[1]
        wt, bs = lin.weight.detach().clone(), lin.bias.detach().clone()
        ws_bytes = _native.tokenize_workspace_bytes(B, H, W, p, dim, precision)
        f = {"img": Fence("img", (B, 3, H, W)), "weight": Fence("weight", wt.shape), "bias": Fence("bias", bs.shape),
             "tokens": Fence("tokens", (B, n, dim), kind="out"), "ws": Fence("ws", (), torch.uint8, "ws", nbytes=ws_bytes)}
        got = fenced_run(f, {"img": img, "weight": wt, "bias": bs},
                         lambda f: _native.tokenize(f["img"].ptr, f["weight"].ptr, f["bias"].ptr, f["tokens"].ptr, B, H, W,
                                                    p, dim, precision, f["ws"].ptr, ws_bytes, _stream()))[0]
        with torch.no_grad():
            same_bits(got["tokens"], m.tokens(img), (precision, "tokens"))
    # the backward is fp32 whatever the precision: the public reference under the deterministic flag
    with deterministic():
        x, w_, b_ = img.clone().requires_grad_(True), wt.clone().requires_grad_(True), bs.clone().requires_grad_(True)
        _Tokenize.apply(m, x, w_, b_).backward(cot)
    ref = {"d_img": x.grad, "d_weight": w_.grad, "d_bias": b_.grad}
    for need in SUBSETS:
        names = [k for k, on in zip(("d_img", "d_weight", "d_bias"), need) if on]
        ws_bytes = _native.tokenize_backward_workspace_bytes(B, H, W, p, need[0])
        for det in (0, 1):
            f = {"img": Fence("img", (B, 3, H, W)), "weight": Fence("weight", wt.shape),
                 "d_tokens": Fence("d_tokens", (B, n, dim)), "ws": Fence("ws", (), torch.uint8, "ws", nbytes=ws_bytes)}
            for k in names:
                f[k] = Fence(k, ref[k].shape, kind="acc")

            def call(f):
                ptrs = [f[k].ptr if k in f else None for k in ("d_weight", "d_bias", "d_img")]
                lib = _native.load()
                if det or need == (1, 1, 1):
                    rc = lib.glom_b200_tokenize_backward_ex(f["img"].ptr, f["weight"].ptr, f["d_tokens"].ptr, *ptrs, B, H, W,
                                                            p, dim, det, f["ws"].ptr, ws_bytes, _stream())
                else:
                    rc = lib.glom_b200_tokenize_backward(f["img"].ptr, f["weight"].ptr, f["d_tokens"].ptr, *ptrs, B, H, W,
                                                         p, dim, f["ws"].ptr, ws_bytes, _stream())
                _native.check(rc)
            inputs = {"img": img, "weight": wt, "d_tokens": cot}
            exact = bool(det) or "d_bias" not in names           # d_weight and d_img never use atomics
            what = f"tokenize_backward p{p} {hw} need={need} det={det}"
            zero, withR = accumulate_twice(f, inputs, call, names, what, exact=exact)
            check_gradients(zero, withR, {k: ref[k] for k in names}, exact, BO.TOL["simt"], what, TOK_BO, 2, n)
            if not exact:                                          # the atomic d_bias aside, every run is the public bits
                for res in zero:
                    for k in names:
                        if k != "d_bias":
                            same_bits(res[k], ref[k], (what, k))


# ---------------------------------------------------------------------------------------------- backward
BWD_SHAPES = ["tc_d256_n144_B5", "tc_d256_n576_mask_self", "mixed_d256_n100", "simt_d192_n144_mask_self",
              "simt_d128_nonsquare", "cc_d256_L12_32x32_p4_bf16"]
# (entry point, deterministic, T, grad_all, start, per-image steps)
BWD_CASES = [("backward", 0, 1, 0, "state0", False), ("backward_ex", 1, 1, 0, "state0", False),
             ("backward_ex", 1, 3, 1, "init", False), ("backward_ex", 1, 3, 0, "state0", False),
             ("backward", 0, 3, 1, "init", False), ("backward_ex", 0, 3, 0, "init", False),
             ("backward_steps", 0, 3, 1, "state0", True), ("backward_ex", 1, 3, 0, "init", True)]


def _bwd_model(name):
    if name.startswith("cc_"):
        m, img, S, n, g = CC._model(name[3:])
        path = "tc"
    else:
        m, img, S, n, g = BO._model(name, "bf16")
        path = BO._path(name, "bf16")
    return m, img.to(DEV), S.to(DEV), n, g, path


def _public_column_grads(m, tokens, pos, S, T, steps, grad_all, cot):
    """_ColumnUpdate (the autograd Function of Glom.forward) under the deterministic flag -> gradients by Grads field."""
    m.zero_grad(set_to_none=True)
    with deterministic():
        tok, ps = tokens.clone().requires_grad_(True), pos.clone().requires_grad_(True)
        s0 = None if S is None else S.clone().requires_grad_(True)
        out = _ColumnUpdate.apply(m, T, steps, None, bool(grad_all), tok, ps, s0, m.init_levels, *m._mlp_params())
        out.backward(cot)
    g = {"d_tokens": tok.grad, "d_pos": ps.grad}
    if S is None:
        g["d_init"] = m.init_levels.grad
    else:
        g["d_state0"] = s0.grad
    g.update({k: q.grad.reshape(q.shape) for k, q in zip(GRAD_FIELDS[4:], m._mlp_params())})
    return g


@pytest.mark.gpu
@pytest.mark.parametrize("name", BWD_SHAPES)
def test_backward_fenced(name):
    """backward, backward_steps and backward_ex (deterministic 0 / 1): one step, and T = 3 with grad_all 0 / 1, from a
    carried state (d_state0) and from init_levels (d_init), with gradients zero-prefilled and R-prefilled."""
    m, img, S, n, gen, path = _bwd_model(name)
    B, L, d = img.shape[0], m.levels, m.dim
    tokens, pos, _ = _engine_inputs(m, img, n)
    wts = _weights32(m)
    cfg = m.engine_cfg(n)
    ws_bytes = _native.backward_workspace_bytes(cfg, B)
    lib = _native.load()
    for entry, det, T, grad_all, start, per_image in BWD_CASES:
        steps = torch.tensor([(T - b) % (T + 1) for b in range(B)], dtype=torch.int32, device=DEV) if per_image else None
        S0 = S if start == "state0" else None
        with torch.no_grad():
            states = m._run(tokens, pos, S0, m.init_levels, T, True, steps=steps)
        cot = torch.randn(((T + 1,) if grad_all else ()) + (B, n, L, d), generator=gen).to(DEV)
        ref = _public_column_grads(m, tokens, pos, S0, T, steps, grad_all, cot)
        f = {"tokens": Fence("tokens", (B, n, d)), "pos": Fence("pos", (n, d)),
             "states": _state_fence("states", (T + 1, B, n, L, d), "in"),
             "grad_out": _state_fence("grad_out", cot.shape, "in"), "ws": Fence("ws", (), torch.uint8, "ws", nbytes=ws_bytes)}
        f.update({k: Fence(k, w.shape) for k, w in zip(WEIGHT_FIELDS, wts)})
        if steps is not None:
            f["steps"] = Fence("steps", (B,), torch.int32)
        for k, v in ref.items():
            f[k] = _state_fence(k, v.shape, "acc") if k == "d_state0" else Fence(k, v.shape, kind="acc")
        inputs = {"tokens": tokens, "pos": pos, "states": states, "grad_out": cot, **dict(zip(WEIGHT_FIELDS, wts))}
        if steps is not None:
            inputs["steps"] = steps

        def call(f):
            w = _native.WeightsRef(ctypes.sizeof(_native.WeightsRef), *[f[k].ptr for k in WEIGHT_FIELDS])
            g = _native.Grads(ctypes.sizeof(_native.Grads), *[f[k].ptr if k in f else None for k in GRAD_FIELDS])
            a = (ctypes.byref(cfg), ctypes.byref(w), f["tokens"].ptr, f["pos"].ptr, f["states"].ptr, f["grad_out"].ptr,
                 ctypes.byref(g), B)
            sp = f["steps"].ptr if "steps" in f else None
            if entry == "backward":
                rc = lib.glom_b200_backward(*a, T, grad_all, f["ws"].ptr, ws_bytes, _stream())
            elif entry == "backward_steps":
                rc = lib.glom_b200_backward_steps(*a, sp, T, grad_all, f["ws"].ptr, ws_bytes, _stream())
            else:
                rc = lib.glom_b200_backward_ex(*a, sp, T, grad_all, det, f["ws"].ptr, ws_bytes, _stream())
            _native.check(rc)
        what = f"{name} {entry} det={det} T={T} grad_all={grad_all} {start} steps={per_image}"
        zero, withR = accumulate_twice(f, inputs, call, list(ref), what, exact=bool(det))
        check_gradients(zero, withR, ref, bool(det), BO.TOL[path], what, BO_NAME, L, n)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SI.SHAPES))
def test_backward_implicit_fenced(name):
    """backward_implicit: deterministic 0 / 1, adjoint_iters 0 and 4, adjoint_q NULL and set, against _SettleImplicit."""
    m, img, start, cot = SI._setup(name)
    B, L, d = img.shape[0], m.levels, m.dim
    with torch.no_grad():
        Sstar, _ = m.settle(img, 1e-4, SI.MAX_ITERS, levels=start)
        tokens = m.tokens(img)
    n = tokens.shape[1]
    pos = m.pos_emb.weight[:n].detach().clone()
    wts = _weights32(m)
    cfg = m.engine_cfg(n)
    ws_bytes = _native.backward_implicit_workspace_bytes(cfg, B)
    path = SI.SHAPES[name][7]
    for det, iters, with_q in ((1, 4, True), (1, 0, False), (0, 4, False), (0, 0, True)):
        m.zero_grad(set_to_none=True)
        with deterministic():
            tok, ps = tokens.clone().requires_grad_(True), pos.clone().requires_grad_(True)
            lv, _ = _SettleImplicit.apply(m, SI.MAX_ITERS, 1e-4, 1e-4, iters, tok, ps, start, m.init_levels, *m._mlp_params())
            (lv * cot).sum().backward()
        same_bits(lv.detach(), Sstar, (name, "implicit forward"))
        ref = {"d_tokens": tok.grad, "d_pos": ps.grad}
        ref.update({k: q.grad.reshape(q.shape) for k, q in zip(GRAD_FIELDS[4:], m._mlp_params())})
        K_ref, q_ref = (t.clone() for t in m.last_adjoint)
        f = {"tokens": Fence("tokens", (B, n, d)), "pos": Fence("pos", (n, d)), "state": _state_fence("state", Sstar.shape, "in"),
             "grad_out": _state_fence("grad_out", cot.shape, "in"), "ws": Fence("ws", (), torch.uint8, "ws", nbytes=ws_bytes),
             "K": Fence("K", (B,), torch.int32, "out")}
        if with_q:
            f["q"] = Fence("q", (B, L), kind="out")
        f.update({k: Fence(k, w.shape) for k, w in zip(WEIGHT_FIELDS, wts)})
        for k, v in ref.items():
            f[k] = Fence(k, v.shape, kind="acc")
        inputs = {"tokens": tokens, "pos": pos, "state": Sstar, "grad_out": cot, **dict(zip(WEIGHT_FIELDS, wts))}

        def call(f):
            _native.backward_implicit(cfg, [f[k].ptr for k in WEIGHT_FIELDS], f["tokens"].ptr, f["pos"].ptr, f["state"].ptr,
                                      f["grad_out"].ptr, {k: f[k].ptr for k in ref}, B, iters, 1e-4, f["K"].ptr,
                                      f["q"].ptr if with_q else None, f["ws"].ptr, ws_bytes, _stream(), deterministic=bool(det))
        what = f"{name} implicit det={det} adjoint_iters={iters} q={with_q}"
        # K and q come from the fixed-order adjoint passes whatever `deterministic` says: exact across patterns
        zero, withR = accumulate_twice(f, inputs, call, list(ref), what, exact=bool(det))
        for res in zero + withR:
            same_bits(res["K"], K_ref, (what, "K"))
            if with_q:
                same_bits(res["q"], q_ref, (what, "q"))
        check_gradients(zero, withR, ref, bool(det), SI.TOL[path], what, BO_NAME, L, n)


# ---------------------------------------------------------------------------------------------- islands, clock probe
ISLAND_GRIDS = [(1, 37), (37, 1), (16, 16), (64, 128)]


@pytest.mark.gpu
@pytest.mark.parametrize("grid", ISLAND_GRIDS, ids=[f"{a}x{b}" for a, b in ISLAND_GRIDS])
def test_islands_fenced(grid):
    """d = 36 (d / 4 odd), L = 2, 3 slabs; neighbouring vectors correlated so that islands form and break."""
    sh, sw = grid
    n, L, d, slabs = sh * sw, 2, 36, 3
    gen = torch.Generator().manual_seed(4)
    base = torch.randn(slabs, 1, L, d, generator=gen)
    states = (base + 0.35 * torch.randn(slabs, n, L, d, generator=gen)).to(DEV)
    f = {"states": _state_fence("states", states.shape, "in")}
    for k in ("cos_right", "cos_down", "agreement"):
        f[k] = Fence(k, (slabs, L, n), kind="out")
    f["labels"] = Fence("labels", (slabs, L, n), torch.int32, "out")
    f["num"] = Fence("num", (slabs, L), torch.int32, "out")
    got = fenced_run(f, {"states": states},
                     lambda f: _native.islands(f["states"].ptr, slabs, sh, sw, L, d, 0.9, f["cos_right"].ptr,
                                               f["cos_down"].ptr, f["agreement"].ptr, f["labels"].ptr, f["num"].ptr,
                                               _stream()))[0]
    want = G.islands(states, grid=grid, threshold=0.9)
    for k, w in zip(("cos_right", "cos_down", "agreement", "labels", "num"), want):
        same_bits(got[k], w, (grid, k))
    assert int(want.num_islands.min()) >= 1


@pytest.mark.gpu
def test_clock_probe_fenced():
    """The probe's two words, {cycles, ns}: written (neither keeps the fill), nothing around them."""
    f = {"out": Fence("out", (2,), torch.int64, "out", align=16)}
    res = fenced_run(f, {}, lambda f: _native.clock_probe(f["out"].ptr, 50, _stream()), exact=False)
    for pat, r in zip(PATTERNS, res):
        cycles, ns = (int(v) for v in r["out"].tolist())
        fill = int.from_bytes(bytes([pat]) * 8, "little", signed=True)
        assert cycles != fill and ns != fill and ns >= 50_000 and 0.3 < cycles / ns < 3.0, (pat, cycles, ns)


# ---------------------------------------------------------------------------------------------- multi-tile regime
@pytest.mark.gpu
def test_configs1_multi_tile_fenced():
    """configs[1] dims at the smallest batch where K1 and K2 deal at least 3 tiles per pair: forward, settle and one
    reverse step (deterministic), fenced, against the public API."""
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    B = next(b for b in range(1, 256) if min(PB.regime(512, 6, 256, b, sms)[k] for k in ("k1", "k2")) >= 3)
    PB.guard(512, 6, 256, B, kernels=("k1", "k2"))
    m = PB._glom(*PB.CFG1)
    img, S, n = PB._inputs(m, B, seed=21)
    L, d = m.levels, m.dim
    packed = _pack_fenced(m, n, "bf16")
    tokens, pos, init = _engine_inputs(m, img, n)
    cfg = m.engine_cfg(n)
    base = {"packed": packed, "tokens": tokens, "pos": pos, "init": init, "state_in": S}
    ws_bytes = _native.workspace_bytes(cfg, B, 1, 0)
    f = _forward_fences(m, B, n, 1, 0, ws_bytes, packed.numel())
    got = fenced_run(f, base, lambda f: _native.forward(cfg, f["packed"].ptr, f["tokens"].ptr, f["pos"].ptr, f["state_in"].ptr,
                                                        f["init"].ptr, f["out"].ptr, B, 1, 0, f["ws"].ptr, ws_bytes,
                                                        _stream()))[0]["out"]
    with torch.no_grad():
        S1 = m(img, iters=1, levels=S)
    same_bits(got, S1, "configs[1] forward")
    ws_bytes = _native.settle_workspace_bytes(cfg, B, 3)
    f = _forward_fences(m, B, n, 3, 0, ws_bytes, packed.numel())
    f["steps_out"] = Fence("steps_out", (B,), torch.int32, "out")
    got = fenced_run(f, base, lambda f: _native.settle(cfg, f["packed"].ptr, f["tokens"].ptr, f["pos"].ptr, f["state_in"].ptr,
                                                       f["init"].ptr, f["out"].ptr, B, 3, 0, 0.05, f["steps_out"].ptr,
                                                       f["ws"].ptr, ws_bytes, _stream()))[0]
    with torch.no_grad():
        want, want_steps = m.settle(img, 0.05, max_iters=3, levels=S)
    same_bits(got["steps_out"], want_steps, "configs[1] settle steps")
    same_bits(got["out"], want, "configs[1] settle")
    states = torch.stack([S, S1])
    cot = torch.randn(S.shape, generator=torch.Generator().manual_seed(6)).to(DEV)
    ref = _public_column_grads(m, tokens, pos, S, 1, None, 0, cot)
    wts = _weights32(m)
    ws_bytes = _native.backward_workspace_bytes(cfg, B)
    f = {"tokens": Fence("tokens", (B, n, d)), "pos": Fence("pos", (n, d)), "states": _state_fence("states", states.shape, "in"),
         "grad_out": _state_fence("grad_out", cot.shape, "in"), "ws": Fence("ws", (), torch.uint8, "ws", nbytes=ws_bytes)}
    f.update({k: Fence(k, w.shape) for k, w in zip(WEIGHT_FIELDS, wts)})
    for k, v in ref.items():
        f[k] = _state_fence(k, v.shape, "acc") if k == "d_state0" else Fence(k, v.shape, kind="acc")

    def call(f):
        _native.backward(cfg, [f[k].ptr for k in WEIGHT_FIELDS], f["tokens"].ptr, f["pos"].ptr, f["states"].ptr,
                         f["grad_out"].ptr, {k: f[k].ptr for k in ref}, B, 1, 0, f["ws"].ptr, ws_bytes, _stream(),
                         deterministic=True)
    what = f"configs[1] B={B} backward"
    zero, withR = accumulate_twice(f, {"tokens": tokens, "pos": pos, "states": states, "grad_out": cot,
                                       **dict(zip(WEIGHT_FIELDS, wts))}, call, list(ref), what)
    check_gradients(zero, withR, ref, True, None, what, BO_NAME, L, n)


# ---------------------------------------------------------------------------------------------- misaligned public inputs
def _misaligned(t):
    """A contiguous copy of t whose data_ptr is 4 bytes past a 16-byte boundary, inside a fence of pattern 0xFF."""
    f = Fence("misaligned", t.shape, shift=4, row_dims=max(t.dim() - 2, 1))
    f.raw.fill_(0xFF)
    f.tensor.copy_(t)
    assert f.tensor.data_ptr() % 16 == 4 and f.tensor.is_contiguous()
    return f


@pytest.mark.gpu
def test_misaligned_contiguous_inputs_through_the_public_api():
    """levels, states and img at a 4-byte offset: the public API gives the bits of the aligned call and leaves the
    bytes around them alone."""
    m, img, S, n = _fwd_model("d64_n9", batch=5)
    start, tol = _contracting_start(m, img, 4)
    fl, fi = _misaligned(start), _misaligned(img)
    with torch.no_grad():
        same_bits(m(fi.tensor, iters=3, levels=fl.tensor), m(img, iters=3, levels=start), "forward")
        a, sa = m.settle(fi.tensor, tol, max_iters=4, levels=fl.tensor)
        b, sb = m.settle(img, tol, max_iters=4, levels=start)
        same_bits(a, b, "settle")
        same_bits(sa, sb, "settle steps")
        a, sa = m.settle_queue(fi.tensor, tol, max_iters=4, levels=fl.tensor, slots=2)
        same_bits(a, b, "settle_queue")
        same_bits(sa, sb, "settle_queue steps")
        fv = _misaligned(img[None].transpose(0, 1).contiguous())
        a, _ = m.settle_video(fv.tensor, tol, max_iters=4, levels=fl.tensor, slots=2)
        same_bits(a[:, 0], b, "settle_video")
        states = m(img, iters=2, return_all=True)
        fs = _misaligned(states)
        for x, y in zip(G.islands(fs.tensor, grid=(3, 3)), G.islands(states, grid=(3, 3))):
            same_bits(x, y, "islands")
    with deterministic():
        grads = []
        for x, lv in ((fi.tensor, fl.tensor), (img, start)):
            m.zero_grad(set_to_none=True)
            x = x.detach().requires_grad_(True) if x is img else x.requires_grad_(True)
            lv = lv.detach().clone().requires_grad_(True) if lv is start else lv.requires_grad_(True)
            m(x, iters=2, levels=lv).square().sum().backward()
            grads.append({"img": x.grad.clone(), "levels": lv.grad.clone(),
                          **{k: q.grad.clone() for k, q in m.named_parameters() if q.grad is not None}})
            if x is not img:
                x.requires_grad_(False)
                lv.requires_grad_(False)
        for k in grads[1]:
            same_bits(grads[0][k], grads[1][k], ("autograd", k))
    for f in (fl, fi, fv, fs):
        bad = f.violations(0xFF)
        assert not bad, bad


@pytest.fixture(autouse=True)
def _peak_memory(request):
    if "gpu" in request.keywords and torch.cuda.is_available():
        torch.cuda.reset_peak_memory_stats()
    yield
    if "gpu" in request.keywords and torch.cuda.is_available():
        print(f"[guard] {request.node.name}: peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
