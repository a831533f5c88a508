"""Island tracks through time (glom_pytorch_b200.track_islands, glom_b200_island_track in include/glom_b200_track.h).

CPU: the numpy oracle (`track_oracle.track`) on hand-built label sequences (a drifting band, a split, a merge, ties in
`prev` and `next`, T = 1, garbage labels); the new header against `_native.TRACK_SIGNATURES`; a fenced GPU case in this
file for each device entry point of that table; the argument errors' exact text and codes (they precede any device
query); the op's fake shapes for time_dim 0, 1 and a middle dimension.

GPU:
  - exact: `labels` / `num_islands` are `islands()`'s bits; `prev`, `overlap`, `next` and `track` equal the oracle run on
    the kernel's own labels.  States are built from designed label sequences (a vector per island plus small noise, so
    `islands` recovers the design at 0.9) whose blocks drift, split and merge over time, in three layouts, and from real
    states: the configs[1] `return_all` slabs, a `settle_video` output, and `settle(return_all=True)` on the contracting
    model, where the slabs after an image's stop are copies and so every island continues its own track;
  - layout: time_dim = k gives the bits of the same states moved to time_dim = 0;
  - bits: two runs, SM-count targets 2, 3 and the full device, a CUDA graph replay, torch.compile(fullgraph=True),
    opcheck and a misaligned state view all give the same bits;
  - guard bands: glom_b200_island_track fenced with the 0x00 / 0xFF / 0x7F fills on real and garbage labels.
"""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import glom_pytorch_b200 as G
from glom_pytorch_b200 import _native
from track_oracle import track

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = G.IslandTracks._fields
TRACK_FIELDS = ("prev", "overlap", "next", "track")


# ====================================================================================================== CPU: oracle
def _seq(*steps):
    """Label maps of one sequence, one level: steps[t] (n,) -> (T, 1, n)."""
    return np.array(steps, dtype=np.int64)[:, None, :]


def test_oracle_drifting_band_keeps_one_track():
    """1 x 10: a band of 3 patches moving one patch per step between two background islands keeps track 0."""
    n, T = 10, 6
    steps = []
    for t in range(T):
        lab = np.arange(n)
        lab[:t] = 0
        lab[t:t + 3] = t
        lab[t + 3:] = t + 3
        steps.append(lab)
    r = track(_seq(*steps))
    for t in range(T):
        assert (r["track"][t, 0, t:t + 3] == 0).all(), t
    assert [int(r["prev"][t, 0, t]) for t in range(1, T)] == list(range(T - 1))
    assert [int(r["overlap"][t, 0, t]) for t in range(1, T)] == [2] * (T - 1)
    assert [int(r["next"][t, 0, t]) for t in range(T - 1)] == list(range(1, T))


def test_oracle_split_gives_the_larger_part_the_track():
    """1 x 8: island [0..5] splits into [0..3] (4 patches) and [4, 5] (2): the larger part keeps track 0, the smaller
    starts t n + j = 8 + 4; [6, 7] continues its own track."""
    r = track(_seq([0, 0, 0, 0, 0, 0, 6, 6], [0, 0, 0, 0, 4, 4, 6, 6]))
    assert r["track"][1, 0].tolist() == [0, 0, 0, 0, 12, 12, 6, 6]
    assert r["prev"][1, 0, [0, 4, 6]].tolist() == [0, 0, 6] and r["overlap"][1, 0, [0, 4, 6]].tolist() == [4, 2, 2]
    assert r["next"][0, 0, [0, 6]].tolist() == [0, 6]
    assert (r["next"][1] == -1).all() and (r["prev"][0] == -1).all() and (r["overlap"][0] == 0).all()


def test_oracle_merge_continues_the_larger_overlap():
    """1 x 8: [0..4] and [5..7] merge: the merged island carries track 0 on (overlap 5 > 3) and track 5 ends."""
    r = track(_seq([0, 0, 0, 0, 0, 5, 5, 5], [0] * 8))
    assert r["track"][1, 0].tolist() == [0] * 8
    assert r["prev"][1, 0, 0] == 0 and r["overlap"][1, 0, 0] == 5
    assert r["next"][0, 0, [0, 5]].tolist() == [0, 0]
    assert 5 not in r["track"][1]
    # the larger overlap wins whichever label is smaller
    r = track(_seq([0, 0, 0, 3, 3, 3, 3, 3], [0] * 8))
    assert r["prev"][1, 0, 0] == 3 and r["overlap"][1, 0, 0] == 5 and r["track"][1, 0].tolist() == [3] * 8


def test_oracle_ties_go_to_the_smaller_label():
    """1 x 8: [0..3], [4..7] -> [0, 1], [2..5], [6, 7].  Island 2 overlaps 0 and 4 twice each: prev 0.  Island 0 at t = 0
    overlaps 0 and 2 twice each: next 0, so island 0 continues track 0 and island 2 starts 8 + 2.  Island 4 at t = 0
    overlaps 2 and 6 twice each: next 2, so island 6 (prev 4) starts 8 + 6 and track 4 ends."""
    r = track(_seq([0, 0, 0, 0, 4, 4, 4, 4], [0, 0, 2, 2, 2, 2, 6, 6]))
    assert r["prev"][1, 0, [0, 2, 6]].tolist() == [0, 0, 4] and r["overlap"][1, 0, [0, 2, 6]].tolist() == [2, 2, 2]
    assert r["next"][0, 0, [0, 4]].tolist() == [0, 2]
    assert r["track"][1, 0].tolist() == [0, 0, 10, 10, 10, 10, 14, 14]


def test_oracle_single_step_is_the_labels():
    lab = np.array([[[0, 0, 2, 2, 2, 5], [0, 1, 1, 1, 4, 4]]])            # (T = 1, L = 2, n = 6)
    for lead in ((1,), (1, 3), (2, 1)):
        labels = np.broadcast_to(lab.reshape((1,) * (len(lead) - 1) + lab.shape), lead + lab.shape[1:])
        td = lead.index(1)
        r = track(labels, time_dim=td)
        assert np.array_equal(r["track"], labels) and (r["prev"] == -1).all() and (r["next"] == -1).all()
        assert (r["overlap"] == 0).all() and r["track"].dtype == np.int32


def test_oracle_skips_garbage_labels():
    """Patch i is a member of j = lab[i] only when 0 <= j <= i and lab[j] == j: non-members get track -1 and count in
    no overlap."""
    bad = [0, 0, -1, 2 ** 31 - 1, 5, 4, 1, 0]                          # members: 0, 0, -, -, -, -, -, 0
    r = track(_seq(bad, [0, 0, 0, 0, 0, 0, 0, 0], bad))
    assert r["track"][0, 0].tolist() == [0, 0, -1, -1, -1, -1, -1, 0]
    assert r["overlap"][1, 0, 0] == 3 and r["prev"][1, 0, 0] == 0
    assert r["track"][1, 0].tolist() == [0] * 8
    assert r["track"][2, 0].tolist() == [0, 0, -1, -1, -1, -1, -1, 0] and r["overlap"][2, 0, 0] == 3


# ====================================================================================================== CPU: ABI
def test_track_header_declares_exactly_the_track_table():
    hdr = open(os.path.join(ROOT, "include", "glom_b200_track.h")).read()
    declared = set(re.findall(r"GLOM_B200_API\s+[\w\s\*]+?\b(glom_b200_\w+)\s*\(", hdr))
    assert declared == set(_native.TRACK_EXPORTS), declared ^ set(_native.TRACK_EXPORTS)
    assert not declared & set(_native.EXPORTS) and not declared & set(_native.TREE_EXPORTS)
    lib = ctypes.CDLL(G.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), name


# every device entry point of _native.TRACK_SIGNATURES -> the GPU test of this file that runs it fenced
COVERAGE = {"glom_b200_island_track": "test_island_track_fenced"}


def test_every_track_entry_point_has_a_fenced_case():
    for name, (_, argtypes) in _native.TRACK_SIGNATURES.items():
        if ctypes.c_void_p in argtypes:
            assert name in COVERAGE, name
    for name, test in COVERAGE.items():
        assert name in _native.TRACK_SIGNATURES, name
        fn = globals().get(test)
        assert fn is not None and any(m.name == "gpu" for m in getattr(fn, "pytestmark", [])), (name, test)


def _p(i, off=0):
    return 0x100000 + 0x1000 * i + off


_TRACK_CALL = dict(labels=_p(1), outer=2, times=13, inner=3, n=256, levels=6, prev=_p(2), overlap=_p(3), next=_p(4),
                   track=_p(5), stream=None)
_NULL = "island_track: a required pointer is NULL"
_SHAPE = "island_track: need 1 <= outer * times * inner <= 65535, 1 <= n <= 8192, 1 <= levels <= 65535"
_A4 = "island_track: labels and outputs must be 4-byte aligned"
TRACK_ERRORS = [
    (dict(labels=None), _NULL), (dict(prev=None), _NULL), (dict(overlap=None), _NULL), (dict(next=None), _NULL),
    (dict(track=None), _NULL), (dict(track=None, n=0), _NULL), (dict(labels=None, prev=_p(2, 1)), _NULL),
    (dict(outer=0), _SHAPE), (dict(times=0), _SHAPE), (dict(inner=0), _SHAPE), (dict(outer=-1, times=-1), _SHAPE),
    (dict(outer=1, times=65536, inner=1), _SHAPE),
    (dict(outer=256, times=256, inner=1), _SHAPE), (dict(outer=65536, times=65536, inner=65536), _SHAPE),
    (dict(outer=2 ** 31 - 1, times=2 ** 31 - 1, inner=2 ** 31 - 1), _SHAPE),
    (dict(n=0), _SHAPE), (dict(n=8193), _SHAPE), (dict(levels=0), _SHAPE), (dict(levels=65536), _SHAPE),
    (dict(n=0, labels=_p(1, 2)), _SHAPE),
    (dict(labels=_p(1, 2)), _A4), (dict(prev=_p(2, 1)), _A4), (dict(overlap=_p(3, 2)), _A4), (dict(next=_p(4, 3)), _A4),
    (dict(track=_p(5, 2)), _A4), (dict(outer=1, times=65535, inner=1, n=8192, levels=65535, labels=_p(1, 2)), _A4),
    (dict(outer=5, times=13107, inner=1, n=1, levels=1, track=_p(5, 2)), _A4),
]


@pytest.mark.parametrize("over,text", TRACK_ERRORS, ids=[",".join(f"{k}={v}" for k, v in o.items()) for o, _ in TRACK_ERRORS])
def test_island_track_argument_errors(over, text):
    """Every error is reported before any device query (the pointers are never dereferenced).  Sizes at the limits
    pass the size check and stop at the alignment check."""
    lib = _native.load()
    args = {**_TRACK_CALL, **over}
    rc = lib.glom_b200_island_track(*args.values())
    assert (rc, lib.glom_b200_last_error().decode()) == (-1, text)


def test_track_islands_op_fake_shapes(monkeypatch):
    """The op path (what torch.compile traces) on fake CUDA tensors: the shapes and dtypes of the eager API for time
    along dimension 0, 1 and a middle dimension with sequences on both sides, and the time_dim errors."""
    from torch._subclasses.fake_tensor import FakeTensorMode
    monkeypatch.setattr(torch.compiler, "is_compiling", lambda: True)
    with FakeTensorMode(allow_non_fake_inputs=True):
        for lead, tds in (((13, 4), (0, 1, -5, -4)), ((3, 5, 2), (0, 1, 2, -4)), ((7,), (0, -4))):
            states = torch.empty(*lead, 12, 4, 8, device=DEV)
            for td in tds:
                t = G.track_islands(states, time_dim=td, grid=(3, 4))
                assert isinstance(t, G.IslandTracks)
                for k in FIELDS:
                    v = getattr(t, k)
                    want = (*lead, 4) if k == "num_islands" else (*lead, 4, 12)
                    assert (tuple(v.shape), v.dtype, v.device) == (want, torch.int32, torch.device(DEV)), (lead, td, k)
            for td in (len(lead), len(lead) + 2, -4 - len(lead)):
                with pytest.raises(RuntimeError, match="time_dim"):
                    G.track_islands(states, time_dim=td, grid=(3, 4))
        with pytest.raises(RuntimeError, match="leading"):
            G.track_islands(torch.empty(12, 4, 8, device=DEV), grid=(3, 4))


# ====================================================================================================== GPU helpers
def _design_seq(sh, sw, L, d, T, rng, phase=0):
    """States (T, n, L, d) of one sequence whose level-l islands at step t are blocks of side 2^(l+1) or 2^(l+2)
    (clipped to the grid; the side doubles or halves every 3 steps, so blocks merge by fours and split again), shifted
    by a drift of (t (l % 2 + 1), t) patches, so blocks also move, appear and leave.  A block holds a Gaussian vector of
    its own (independent across blocks, so neighbouring blocks' cosines stay far below 0.9) plus 0.02 Gaussian noise
    per patch.  -> (states, the designed labels (T, L, n))."""
    n = sh * sw
    h, w = np.divmod(np.arange(n), sw)
    x = np.empty((T, n, L, d), np.float32)
    labels = np.empty((T, L, n), np.int32)
    for t in range(T):
        for l in range(L):
            s = 2 ** min(l + 1 + ((t // 3 + l + phase) % 2), 20)
            bh, bw = (h + t * (l % 2 + 1)) // s, (w + t + phase) // s
            _, first, inv = np.unique(bh * (1 << 20) + bw, return_index=True, return_inverse=True)
            labels[t, l] = first[inv]
            x[t, :, l] = rng.standard_normal((first.size, d))[inv] + 0.02 * rng.standard_normal((n, d))
    return x, labels


LAYOUTS = {"T,B": (0, lambda seqs: np.stack(seqs, 1)), "S,F": (1, lambda seqs: np.stack(seqs, 0)),
           "2,T,3": (1, lambda seqs: np.stack(seqs, 1).reshape((seqs[0].shape[0], 2, 3) + seqs[0].shape[1:]).swapaxes(0, 1))}
NSEQ = {"T,B": 2, "S,F": 2, "2,T,3": 6}


def _designed(sh, sw, L, d, T, layout, seed):
    """-> (states tensor in the layout, time_dim, designed labels (..., L, n) in the same layout)."""
    rng = np.random.default_rng(seed)
    xs, labs = zip(*[_design_seq(sh, sw, L, d, T, rng, phase=q) for q in range(NSEQ[layout])])
    td, stack = LAYOUTS[layout]
    return torch.from_numpy(np.ascontiguousarray(stack(xs))).to(DEV), td, np.ascontiguousarray(stack(labs))


def _np(t):
    return t.detach().cpu().numpy()


def _same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape)
    assert torch.equal(a, b), (what, int((a != b).sum()))


def _same_tracks(a, b, what):
    for k in FIELDS:
        _same(getattr(a, k), getattr(b, k), (what, k))


def check_tracks(t, labels, time_dim, what=""):
    """prev / overlap / next / track against the oracle on `labels` bit for bit."""
    want = track(_np(labels), time_dim)
    for k in TRACK_FIELDS:
        got = _np(getattr(t, k))
        assert got.dtype == want[k].dtype and np.array_equal(got, want[k]), (what, k, int((got != want[k]).sum()))
    return want


def _check_public(states, time_dim, grid=None, what="", threshold=0.9):
    t = G.track_islands(states, time_dim=time_dim, grid=grid, threshold=threshold)
    isl = G.islands(states, grid=grid, threshold=threshold)
    _same(t.labels, isl.labels, (what, "labels"))
    _same(t.num_islands, isl.num_islands, (what, "num_islands"))
    check_tracks(t, t.labels, time_dim, what)
    return t


def _events(t, time_dim):
    """(continued, born after step 0) island counts over every sequence and level, from the kernel's track."""
    tr = np.moveaxis(_np(t.track), time_dim, 0)
    lab = np.moveaxis(_np(t.labels), time_dim, 0)
    n = lab.shape[-1]
    roots = lab == np.arange(n)
    ids = np.where(roots, tr, -1)[1:]
    step = np.arange(1, lab.shape[0]).reshape((-1,) + (1,) * (lab.ndim - 1))
    return int(((ids >= 0) & (ids < step * n)).sum()), int((ids >= step * n).sum())


# ====================================================================================================== GPU: exact
# (side_h, side_w, L, d, T, layout): n = 1; one row; one column; non-square with L = 8; n = 8192; T = 1; T = 13 in
# every layout
SHAPES = [(1, 1, 2, 32, 3, "T,B"), (1, 37, 3, 32, 13, "S,F"), (37, 1, 3, 32, 2, "2,T,3"), (6, 10, 8, 32, 13, "T,B"),
          (64, 128, 2, 32, 2, "S,F"), (16, 16, 2, 64, 1, "T,B"), (16, 16, 4, 32, 13, "2,T,3"), (8, 8, 3, 32, 13, "T,B"),
          (12, 12, 3, 32, 13, "S,F")]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES, ids=[f"{a}x{b}_L{c}_d{d}_T{e}_{f}" for a, b, c, d, e, f in SHAPES])
def test_designed_tracks(shape):
    sh, sw, L, d, T, layout = shape
    states, td, design = _designed(sh, sw, L, d, T, layout, seed=sh * 1000 + sw + L + T)
    t = _check_public(states, td, grid=(sh, sw), what=str(shape))
    assert np.array_equal(_np(t.labels), design), "islands did not recover the designed label sequences"
    cont, born = _events(t, td)
    print(f"[track_islands] {shape}: {cont} islands continue a track, {born} start one after step 0")
    if T >= 13 and min(sh, sw) >= 6:
        assert cont > 0 and born > 0
    if T == 1:
        _same(t.track, t.labels, "T = 1: track is the labels")


CFG1 = (512, 6, 224, 14)


@pytest.mark.gpu
def test_configs1_return_all_slabs():
    """configs[1] (dim 512, 6 levels, 224 / 14, 12 iterations, batch 32): the 13 x 32 return_all slabs."""
    import test_production_batch as PB
    m = PB._glom(*CFG1)
    img = torch.randn(32, 3, 224, 224, generator=torch.Generator().manual_seed(3)).to(DEV)
    with torch.no_grad():
        states = m(img, iters=12, return_all=True)
    t = _check_public(states, 0, what="configs[1]")
    cont, born = _events(t, 0)
    print(f"[track_islands] configs[1]: islands per (slab, level) median {float(np.median(_np(t.num_islands)))}; "
          f"{cont} continue a track, {born} start one after step 0")


@pytest.mark.gpu
def test_settle_video_output():
    """A small settle_video output (S, F, n, L, d), time_dim = 1: 3 streams of 6 frames, each frame its stream's image
    shifted by one more pixel."""
    torch.manual_seed(0)
    m = G.Glom(dim=64, levels=3, image_size=56, patch_size=7).to(DEV).eval()
    base = torch.randn(3, 3, 56, 56, generator=torch.Generator().manual_seed(4))
    frames = torch.stack([torch.roll(base, f, dims=3) for f in range(6)], 1).to(DEV)
    with torch.no_grad():
        out, _ = m.settle_video(frames, 1e-3, max_iters=6)
    for thr in (0.9, 0.5):
        t = _check_public(out, 1, what=f"settle_video {thr}", threshold=thr)
        cont, born = _events(t, 1)
        print(f"[track_islands] settle_video threshold {thr}: islands per (slab, level) median "
              f"{float(np.median(_np(t.num_islands)))}; {cont} continue a track, {born} start one")


@pytest.mark.gpu
def test_settle_return_all_stopped_images_continue_every_track():
    """settle(return_all=True) on the contracting model of test_settle_train.py: the slabs of image b after steps[b]
    are copies of slab steps[b], so there every root j continues its own track, with prev == j, next == j and
    overlap == its size."""
    import test_settle_train as STR
    m, img, start, r = STR._setup(STR.SHAPES["n64_four_images_per_block"], 0.0)
    tol = STR._tol_spread(r)
    with torch.no_grad():
        states, steps = m.settle(img, tol, max_iters=STR.MAX_ITERS, levels=start, return_all=True)
    t = _check_public(states, 0, what="settle return_all")
    lab, prev, ov, nxt, tr = (_np(getattr(t, k)) for k in ("labels", "prev", "overlap", "next", "track"))
    n = lab.shape[-1]
    checked = 0
    for b, k in enumerate(_np(steps).tolist()):
        for s in range(k + 1, STR.MAX_ITERS + 1):
            assert np.array_equal(lab[s, b], lab[s - 1, b]), (b, s)
            for l in range(lab.shape[2]):
                roots = np.flatnonzero(lab[s, b, l] == np.arange(n))
                size = np.bincount(lab[s, b, l], minlength=n)[roots]
                assert (prev[s, b, l, roots] == roots).all() and (nxt[s - 1, b, l, roots] == roots).all(), (b, s, l)
                assert (ov[s, b, l, roots] == size).all(), (b, s, l)
                checked += roots.size
            assert np.array_equal(tr[s, b], tr[s - 1, b]), (b, s)
    assert checked > 0, _np(steps)


@pytest.mark.gpu
def test_time_dim_is_a_layout_choice():
    """track_islands(states, time_dim=k) is track_islands(states.movedim(k, 0), time_dim=0) moved back."""
    states, _, _ = _designed(8, 8, 3, 32, 5, "2,T,3", seed=7)
    for k in (1, -4, 2, 0):
        got = G.track_islands(states, time_dim=k)
        kk = k % 6
        ref = G.track_islands(states.movedim(kk, 0).contiguous(), time_dim=0)
        for f in FIELDS:
            _same(getattr(got, f), getattr(ref, f).movedim(0, kk), (k, f))
        check_tracks(got, got.labels, kk, f"time_dim {k}")


# ====================================================================================================== GPU: bits
def _bits_case():
    states, _, _ = _designed(16, 16, 4, 64, 13, "T,B", seed=11)
    noisy = states + 0.4 * torch.randn(states.shape, generator=torch.Generator().manual_seed(12)).to(DEV)   # ragged
    return torch.cat([states, noisy], 1).contiguous()


@pytest.mark.gpu
def test_runs_and_sm_count_targets_are_bit_identical():
    states = _bits_case()
    ref = G.track_islands(states)
    check_tracks(ref, ref.labels, 0, "bits case")
    _same_tracks(G.track_islands(states), ref, "second run")
    for sms in (2, 3, 0):
        _native.set_sm_count_target(sms)
        try:
            got = G.track_islands(states)
        finally:
            _native.set_sm_count_target(0)
        _same_tracks(got, ref, f"sm target {sms}")
    big, td, _ = _designed(64, 128, 2, 32, 2, "S,F", seed=5)
    ref = G.track_islands(big, time_dim=td, grid=(64, 128))
    _native.set_sm_count_target(2)
    try:
        _same_tracks(G.track_islands(big, time_dim=td, grid=(64, 128)), ref, "n = 8192, sm target 2")
    finally:
        _native.set_sm_count_target(0)


@pytest.mark.gpu
def test_cuda_graph_replay_is_eager_bits():
    states = _bits_case()
    other = torch.flip(states, dims=(1,)).contiguous()
    static = states.clone()
    G.track_islands(static)                                           # warm up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = G.track_islands(static)
    for src in (other, states):
        static.copy_(src)
        g.replay()
        torch.cuda.synchronize()
        _same_tracks(out, G.track_islands(src), "graph")


@pytest.mark.gpu
def test_compiled_track_islands_is_eager_bits_without_graph_breaks():
    states = _bits_case()
    for td in (0, 1):
        torch._dynamo.reset()

        def fn(s):
            return G.track_islands(s * 1.0, time_dim=td)
        got = torch.compile(fn, fullgraph=True)(states)
        _same_tracks(got, G.track_islands(states, time_dim=td), ("compile", td))
        torch._dynamo.reset()
        assert torch._dynamo.explain(fn)(states).graph_break_count == 0


@pytest.mark.gpu
def test_track_islands_opcheck():
    states = _bits_case()[:, :3]
    for td in (0, 1):
        torch.library.opcheck(torch.ops.glom_b200.track_islands, (states.contiguous(), 16, 16, 0.9, td),
                              test_utils=("test_schema", "test_faketensor", "test_autograd_registration"))


@pytest.mark.gpu
def test_misaligned_state_view_gives_the_aligned_bits():
    from test_guard_bands import _misaligned
    states = _bits_case()
    f = _misaligned(states)
    _same_tracks(G.track_islands(f.tensor), G.track_islands(states), "misaligned")
    assert not f.violations(0xFF)


# ====================================================================================================== GPU: guard bands
FENCE_GRIDS = [(1, 37), (16, 16), (64, 128)]


@pytest.mark.gpu
@pytest.mark.parametrize("grid", FENCE_GRIDS, ids=[f"{a}x{b}" for a, b in FENCE_GRIDS])
def test_island_track_fenced(grid):
    """glom_b200_island_track on the labels of islands() and on garbage labels, (outer, times, inner) = (2, T, 3),
    fenced with the three fills: guards and inputs intact, outputs bit-identical across fills, equal to track_islands
    (real labels) or to the oracle (garbage labels)."""
    from test_guard_bands import Fence, fenced_run, same_bits
    from test_parse_tree import _garbage
    sh, sw = grid
    n, L = sh * sw, 3
    T = 4 if n > 1000 else 6
    states, td, _ = _designed(sh, sw, L, 32, T, "2,T,3", seed=sw)
    states = states + 0.3 * torch.randn(states.shape, generator=torch.Generator().manual_seed(sh)).to(DEV)
    public = G.track_islands(states, time_dim=td, grid=grid)
    shape = (2, T, 3, L, n)
    for name, labels in (("real", public.labels), ("garbage", _garbage(public.labels, sh * sw))):
        f = {"labels": Fence("labels", shape, torch.int32)}
        for k in TRACK_FIELDS:
            f[k] = Fence(k, shape, torch.int32, "out")

        def call(f):
            _native.island_track(f["labels"].ptr, 2, T, 3, n, L, f["prev"].ptr, f["overlap"].ptr, f["next"].ptr,
                                 f["track"].ptr, torch.cuda.current_stream().cuda_stream)
        got = fenced_run(f, {"labels": labels}, call)[0]
        if name == "real":
            for k in TRACK_FIELDS:
                same_bits(got[k], getattr(public, k), (grid, name, k))
        else:
            check_tracks(G.IslandTracks(labels, None, *(got[k] for k in TRACK_FIELDS)), labels, td, f"{grid} garbage")
