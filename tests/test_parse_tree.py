"""Part-whole parse trees (glom_pytorch_b200.parse_tree, glom_b200_island_tree in include/glom_b200_tree.h).

CPU: the numpy oracle (`tree_oracle.tree`) on hand-built label sets; the new header against
`_native.TREE_SIGNATURES`; a fenced GPU case in this file for each device entry point of that table; the argument
errors' exact text and codes (they precede any device query); the op's fake shapes.

GPU:
  - exact: `labels` / `num_islands` are `islands()`'s bits; `size`, `parent`, `containment` and `nested` equal the
    oracle run on the kernel's own labels bit for bit.  States are built from designed label sets (a vector per island
    plus small noise, so `islands` recovers the design at 0.9) and from configs[1] `return_all` slabs;
  - tolerance: `embedding` within the fixed-order fp32 summation bound (size + 1) u mean|x| of the float64 means, and
    bit-identical to a sequential fp32 sum in patch order; `member_cos` and `coherence` within 1e-5 of float64;
  - bits: two runs, SM-count targets 2, 3 and the full device, a CUDA graph replay, torch.compile(fullgraph=True) and a
    misaligned state view all give the same bits;
  - guard bands: glom_b200_island_tree fenced with the 0x00 / 0xFF / 0x7F fills on real and garbage labels.
"""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import glom_pytorch_b200 as G
from glom_pytorch_b200 import _native
from tree_oracle import members, tree

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U32 = 2.0 ** -24
COS_TOL = 1e-5
INT_FIELDS = ("size", "parent", "containment", "nested")
EMB_FIELDS = ("embedding", "member_cos", "coherence")


# ====================================================================================================== CPU: oracle
def _tree1(*levels):
    return tree(np.array(levels, dtype=np.int32))


def test_oracle_quadrants_inside_halves():
    """4 x 4 grid: level 0 quadrants, level 1 left / right halves, level 2 one island."""
    q = np.array([[0, 0, 2, 2], [0, 0, 2, 2], [8, 8, 10, 10], [8, 8, 10, 10]]).ravel()
    half = np.tile([0, 0, 2, 2], 4)
    r = _tree1(q, half, np.zeros(16))
    roots = [0, 2, 8, 10]
    assert r["size"][0, roots].tolist() == [4] * 4 and r["size"][0].sum() == 16
    assert r["parent"][0, roots].tolist() == [0, 2, 0, 2]
    assert r["containment"][0, roots].tolist() == [1.0] * 4
    assert r["size"][1, [0, 2]].tolist() == [8, 8] and r["parent"][1, [0, 2]].tolist() == [0, 0]
    assert r["nested"].tolist() == [1.0, 1.0]
    nonroot = np.setdiff1d(np.arange(16), roots)
    assert (r["parent"][0, nonroot] == -1).all() and (r["containment"][0, nonroot] == 0).all()
    assert (r["size"][0, nonroot] == 0).all()


def test_oracle_straddling_island_ties_to_the_smaller_label():
    """1 x 8: level 0 island {2..5} straddles the level-1 halves {0..3}, {4..7} two and two: containment 0.5, parent
    0 (the smaller label); the other islands are contained."""
    r = _tree1([0, 0, 2, 2, 2, 2, 6, 6], [0, 0, 0, 0, 4, 4, 4, 4])
    assert r["size"][0, [0, 2, 6]].tolist() == [2, 4, 2]
    assert r["parent"][0, [0, 2, 6]].tolist() == [0, 0, 4]
    assert r["containment"][0, 2] == np.float32(0.5) and r["containment"][0, [0, 6]].tolist() == [1.0, 1.0]
    assert r["nested"][0] == np.float32(4 / 8)
    # a majority beats the smaller label
    r = _tree1([0, 0, 0, 0, 0, 5, 5, 5], [0, 0, 2, 2, 2, 2, 2, 2])
    assert r["parent"][0, 0] == 2 and r["containment"][0, 0] == np.float32(3 / 5)


def test_oracle_one_island_and_checkerboard():
    r = _tree1(np.zeros(9), np.zeros(9))
    assert r["size"][:, 0].tolist() == [9, 9] and r["parent"][:, 0].tolist() == [0, -1]
    assert r["nested"].tolist() == [1.0]
    n = 12
    r = _tree1(np.arange(n), np.zeros(n))                       # n islands of size 1, each inside the one above
    assert (r["size"][0] == 1).all() and (r["parent"][0] == 0).all() and (r["containment"][0] == 1).all()
    assert r["nested"].tolist() == [1.0]


def test_oracle_top_level_has_no_parent():
    r = _tree1([0, 0, 2, 2], [0, 1, 2, 3], [0, 0, 0, 0])
    assert (r["parent"][-1] == -1).all() and (r["containment"][-1] == 0).all()
    assert r["size"][-1, 0] == 4 and r["nested"].shape == (2,)
    assert r["parent"][1].tolist() == [0, 0, 0, 0] and r["nested"][0] == np.float32(0.0)   # halves split below


def test_oracle_skips_garbage_labels():
    """A patch is a member of j = lab[i] only when 0 <= j <= i and lab[j] == j."""
    lab = np.array([0, 0, -1, 2 ** 31 - 1, 5, 4, 1, 0], dtype=np.int64)
    assert members(lab).tolist() == [0, 0, -1, -1, -1, -1, -1, 0]
    r = tree(np.array([lab, np.zeros(8)], dtype=np.int32), np.ones((8, 2, 4), np.float32))
    assert r["size"][0].tolist() == [3, 0, 0, 0, 0, 0, 0, 0] and r["nested"][0] == np.float32(3 / 8)
    assert (r["member_cos"][0, [0, 1, 7]] == 1).all() and (r["member_cos"][0, 2:7] == 0).all()
    assert r["coherence"][0, 0] == 1 and (r["embedding"][0, 0] == 1).all() and (r["embedding"][0, 1:] == 0).all()


# ====================================================================================================== CPU: ABI
def test_tree_header_declares_exactly_the_tree_table():
    hdr = open(os.path.join(ROOT, "include", "glom_b200_tree.h")).read()
    declared = set(re.findall(r"GLOM_B200_API\s+[\w\s\*]+?\b(glom_b200_\w+)\s*\(", hdr))
    assert declared == set(_native.TREE_EXPORTS), declared ^ set(_native.TREE_EXPORTS)
    assert not declared & set(_native.EXPORTS)
    lib = ctypes.CDLL(G.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), name


# every device entry point of _native.TREE_SIGNATURES -> the GPU test of this file that runs it fenced
COVERAGE = {"glom_b200_island_tree": "test_island_tree_fenced"}


def test_every_tree_entry_point_has_a_fenced_case():
    for name, (_, argtypes) in _native.TREE_SIGNATURES.items():
        if ctypes.c_void_p in argtypes:
            assert name in COVERAGE, name
    for name, test in COVERAGE.items():
        assert name in _native.TREE_SIGNATURES, name
        fn = globals().get(test)
        assert fn is not None and any(m.name == "gpu" for m in getattr(fn, "pytestmark", [])), (name, test)


def _p(i, off=0):
    return 0x100000 + 0x1000 * i + off


_TREE_CALL = dict(labels=_p(1), states=_p(2), slabs=2, n=16, levels=3, dim=64, size=_p(3), parent=_p(4),
                  containment=_p(5), nested=_p(6), embedding=_p(7), member_cos=_p(8), coherence=_p(9), stream=None)
_NULL = "island_tree: a required pointer is NULL"
_ALL = "island_tree: states, embedding, member_cos and coherence are all NULL or all set"
_SHAPE = "island_tree: need 1 <= slabs, levels <= 65535, 1 <= n <= 8192, dim % 4 == 0"
_A16 = "island_tree: states and embedding must be 16-byte aligned"
_A4 = "island_tree: labels and outputs must be 4-byte aligned"
TREE_ERRORS = [
    (dict(labels=None), _NULL), (dict(size=None), _NULL), (dict(parent=None), _NULL), (dict(containment=None), _NULL),
    (dict(nested=None), _NULL), (dict(nested=None, levels=0), _NULL), (dict(labels=None, slabs=0), _NULL),
    (dict(embedding=None), _ALL), (dict(states=None), _ALL), (dict(states=None, embedding=None, member_cos=None), _ALL),
    (dict(coherence=None, slabs=0), _ALL),
    (dict(slabs=0), _SHAPE), (dict(slabs=65536), _SHAPE), (dict(n=0), _SHAPE), (dict(n=8193), _SHAPE),
    (dict(levels=0), _SHAPE), (dict(levels=65536), _SHAPE), (dict(dim=0), _SHAPE), (dict(dim=6), _SHAPE),
    (dict(dim=6, states=_p(2, 8)), _SHAPE),
    (dict(states=_p(2, 8)), _A16), (dict(embedding=_p(7, 4)), _A16), (dict(states=_p(2, 4), labels=_p(1, 2)), _A16),
    (dict(labels=_p(1, 2)), _A4), (dict(nested=_p(6, 1)), _A4), (dict(coherence=_p(9, 2)), _A4),
    (dict(size=_p(3, 2), states=None, embedding=None, member_cos=None, coherence=None), _A4),
]


@pytest.mark.parametrize("over,text", TREE_ERRORS, ids=[",".join(f"{k}={v}" for k, v in o.items()) for o, _ in TREE_ERRORS])
def test_island_tree_argument_errors(over, text):
    lib = _native.load()
    args = {**_TREE_CALL, **over}
    rc = lib.glom_b200_island_tree(*args.values())
    assert (rc, lib.glom_b200_last_error().decode()) == (-1, text)


def test_parse_tree_op_fake_shapes(monkeypatch):
    """The op path (what torch.compile traces) on fake CUDA tensors: the shapes and dtypes of the eager API."""
    from torch._subclasses.fake_tensor import FakeTensorMode
    monkeypatch.setattr(torch.compiler, "is_compiling", lambda: True)
    with FakeTensorMode(allow_non_fake_inputs=True):
        states = torch.empty(3, 2, 12, 4, 8, device=DEV)
        for emb in (False, True):
            t = G.parse_tree(states, grid=(3, 4), embeddings=emb)
            want = dict(labels=((3, 2, 4, 12), torch.int32), num_islands=((3, 2, 4), torch.int32),
                        size=((3, 2, 4, 12), torch.int32), parent=((3, 2, 4, 12), torch.int32),
                        containment=((3, 2, 4, 12), torch.float32), nested=((3, 2, 3), torch.float32))
            if emb:
                want.update(embedding=((3, 2, 4, 12, 8), torch.float32), member_cos=((3, 2, 4, 12), torch.float32),
                            coherence=((3, 2, 4, 12), torch.float32))
            for k in ParseTreeFields:
                v = getattr(t, k)
                if k not in want:
                    assert v is None, k
                    continue
                assert (tuple(v.shape), v.dtype, v.device) == (*want[k], torch.device(DEV)), k


ParseTreeFields = G.ParseTree._fields


# ====================================================================================================== GPU helpers
def _design(sh, sw, L, d, shifted, rng):
    """States (n, L, d) whose level-l islands are the blocks of side 2^l (clipped to the grid), shifted by l % 2 rows
    and columns when `shifted` (so islands straddle the level above).  A block holds 3 e_c + 0.3 g (c one of 4 axes,
    coloured so that neighbouring blocks differ; g Gaussian per block) plus 0.02 Gaussian noise per patch.  -> (states,
    the designed labels (L, n))."""
    n = sh * sw
    h, w = np.divmod(np.arange(n), sw)
    x = np.empty((n, L, d), np.float32)
    labels = np.empty((L, n), np.int32)
    for l in range(L):
        s = 2 ** min(l, 20)
        o = l % 2 if shifted else 0
        bh, bw = (h + o) // s, (w + o) // s
        block = bh * (sw + 2) + bw
        _, first, inv = np.unique(block, return_index=True, return_inverse=True)
        labels[l] = first[inv]
        axis = ((bh % 2) * 2 + (bw % 2)) * (d // 4)
        base = 0.3 * rng.standard_normal((first.size, d))
        base[np.arange(first.size), axis[first]] += 3.0
        x[:, l] = base[inv] + 0.02 * rng.standard_normal((n, d))
    return x, labels


def _designed_slabs(sh, sw, L, d, slabs, shifted, seed):
    rng = np.random.default_rng(seed)
    xs, labs = zip(*[_design(sh, sw, L, d, shifted, rng) for _ in range(slabs)])
    return np.stack(xs), np.stack(labs)


def _np(t):
    return t.detach().cpu().numpy()


def _seq_mean32(x, lab):
    """The kernel's embedding in numpy fp32: members summed one at a time in increasing patch order, then one fp32
    division by the size.  x (n, d) fp32, lab (n,)."""
    m = members(lab)
    n = x.shape[0]
    acc = np.zeros_like(x)
    for i in range(n):
        if m[i] >= 0:
            acc[m[i]] += x[i]
    size = np.bincount(m[m >= 0], minlength=n).astype(np.float32)
    out = np.zeros_like(x)
    roots = size > 0
    out[roots] = acc[roots] / size[roots][:, None]
    return out


def check_tree(t, labels, states=None, slab_subset=None, what=""):
    """size / parent / containment / nested against the oracle on `labels` bit for bit; with states, the embedding
    outputs of the slabs in slab_subset (default all) against float64 and the sequential fp32 sum."""
    lab = _np(labels)
    L, n = lab.shape[-2:]
    want = tree(lab)
    for k in INT_FIELDS:
        got = _np(getattr(t, k))
        assert got.dtype == want[k].dtype and np.array_equal(got, want[k]), (what, k)
    if states is None:
        return {}
    d = states.shape[-1]
    lab2 = lab.reshape(-1, L, n)
    sel = list(range(lab2.shape[0]) if slab_subset is None else slab_subset)
    xs = _np(states.reshape(-1, n, L, d)[sel])                           # only the slabs checked leave the device
    emb, mcos, coh = (_np(getattr(t, k).reshape((-1, L, n) + ((d,) if k == "embedding" else ()))[sel])
                      for k in EMB_FIELDS)
    worst = {"emb": 0.0, "cos": 0.0, "coh": 0.0}
    for q, s in enumerate(sel):
        r = tree(lab2[s], xs[q])
        for l in range(L):
            m = members(lab2[s, l])
            x = xs[q, :, l, :]
            size = r["size"][l].astype(np.float64)
            ok = m >= 0
            mean_abs = np.zeros_like(r["embedding"][l])
            np.add.at(mean_abs, m[ok], np.abs(x[ok].astype(np.float64)))
            roots = size > 0
            mean_abs[roots] /= size[roots][:, None]
            bound = (size[:, None] + 1) * U32 * mean_abs
            err = np.abs(emb[q, l] - r["embedding"][l])
            assert (err <= bound).all(), (what, s, l, float((err - bound).max()))
            worst["emb"] = max(worst["emb"], float((err / np.maximum(bound, 1e-300)).max()))
            assert np.array_equal(emb[q, l], _seq_mean32(x, lab2[s, l])), (what, s, l, "fp32 sequential sum")
        e_cos = np.abs(mcos[q] - r["member_cos"]).max()
        e_coh = np.abs(coh[q] - r["coherence"]).max()
        worst["cos"], worst["coh"] = max(worst["cos"], float(e_cos)), max(worst["coh"], float(e_coh))
        assert e_cos <= COS_TOL and e_coh <= COS_TOL, (what, s, e_cos, e_coh)
    print(f"[parse_tree] {what}: embedding err / bound {worst['emb']:.3g}, member_cos {worst['cos']:.2e}, "
          f"coherence {worst['coh']:.2e}")
    return worst


def _same(a, b, what):
    if a is None or b is None:
        assert a is None and b is None, what
        return
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape)
    assert torch.equal(a.view(torch.uint8) if a.dtype == torch.float32 else a,
                       b.view(torch.uint8) if b.dtype == torch.float32 else b), what


def _same_tree(a, b, what):
    for k in ParseTreeFields:
        _same(getattr(a, k), getattr(b, k), (what, k))


# ====================================================================================================== GPU: exact and tolerance
# (side_h, side_w, L, d, slabs, shifted): n = 1; one row; one column; non-square with L = 8; n = 8192 (the API bound);
# d / 4 = 1, 5, 9, 16, 129; 3000 slabs
SHAPES = [(1, 1, 2, 4, 3, False), (1, 37, 3, 20, 2, True), (37, 1, 3, 36, 2, False), (6, 10, 8, 64, 2, True),
          (64, 128, 2, 12, 1, True), (64, 128, 3, 4, 1, False), (16, 16, 2, 516, 2, True), (8, 8, 4, 4, 4, True),
          (4, 4, 2, 16, 3000, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES, ids=[f"{a}x{b}_L{c}_d{d}_s{e}{'_shift' if f else ''}" for a, b, c, d, e, f in SHAPES])
def test_designed_islands(shape):
    sh, sw, L, d, slabs, shifted = shape
    x, design = _designed_slabs(sh, sw, L, d, slabs, shifted, seed=sh * 1000 + sw + L)
    states = torch.from_numpy(x).to(DEV)
    t = G.parse_tree(states, grid=(sh, sw), threshold=0.9, embeddings=True)
    isl = G.islands(states, grid=(sh, sw), threshold=0.9)
    _same(t.labels, isl.labels, "labels")
    _same(t.num_islands, isl.num_islands, "num_islands")
    assert np.array_equal(_np(t.labels), design), "islands did not recover the designed label sets"
    subset = None if slabs <= 8 else [0, 1, slabs // 2, slabs - 1]
    check_tree(t, t.labels, states, subset, what=str(shape))
    if shifted and min(sh, sw) > 2 and L > 2:
        assert (_np(t.nested) < 1).any()                           # some island straddles its parents
    t2 = G.parse_tree(states, grid=(sh, sw), threshold=0.9)
    for k in ParseTreeFields[:6]:
        _same(getattr(t2, k), getattr(t, k), ("embeddings=False", k))
    assert t2.embedding is None and t2.member_cos is None and t2.coherence is None


CFG1 = (512, 6, 224, 14)


@pytest.mark.gpu
def test_configs1_return_all_slabs():
    """configs[1] (dim 512, 6 levels, 224 / 14, 12 iterations, batch 32): the 13 x 32 return_all slabs.  Exact fields
    on every slab; the embedding outputs on slabs of the first, a middle and the last iteration."""
    import test_production_batch as PB
    m = PB._glom(*CFG1)
    img = torch.randn(32, 3, 224, 224, generator=torch.Generator().manual_seed(3)).to(DEV)
    with torch.no_grad():
        states = m(img, iters=12, return_all=True)
    t = G.parse_tree(states, embeddings=True)
    isl = G.islands(states)
    _same(t.labels, isl.labels, "labels")
    _same(t.num_islands, isl.num_islands, "num_islands")
    counts = _np(t.num_islands)
    print(f"[parse_tree] configs[1]: islands per (slab, level) min {counts.min()} median {np.median(counts)} "
          f"max {counts.max()}; nested mean {float(t.nested.mean()):.3f}")
    check_tree(t, t.labels, states, slab_subset=[0, 5, 6 * 32 + 17, 12 * 32 + 31], what="configs[1]")


# ====================================================================================================== GPU: bits
def _bits_case():
    x, _ = _designed_slabs(16, 16, 4, 64, 6, True, seed=11)
    noisy = x + 0.4 * np.random.default_rng(12).standard_normal(x.shape).astype(np.float32)   # ragged islands
    return torch.from_numpy(np.concatenate([x, noisy])).to(DEV)


@pytest.mark.gpu
def test_runs_and_sm_count_targets_are_bit_identical():
    states = _bits_case()
    ref = G.parse_tree(states, embeddings=True)
    _same_tree(G.parse_tree(states, embeddings=True), ref, "second run")
    for sms in (2, 3, 0):
        _native.set_sm_count_target(sms)
        try:
            got = G.parse_tree(states, embeddings=True)
        finally:
            _native.set_sm_count_target(0)
        _same_tree(got, ref, f"sm target {sms}")
    big = torch.from_numpy(_designed_slabs(64, 128, 2, 8, 1, True, seed=5)[0]).to(DEV)
    ref = G.parse_tree(big, grid=(64, 128), embeddings=True)
    _native.set_sm_count_target(2)
    try:
        _same_tree(G.parse_tree(big, grid=(64, 128), embeddings=True), ref, "n = 8192, sm target 2")
    finally:
        _native.set_sm_count_target(0)


@pytest.mark.gpu
def test_cuda_graph_replay_is_eager_bits():
    states = _bits_case()
    other = torch.flip(states, dims=(0,)).contiguous()
    static = states.clone()
    for emb in (True, False):
        G.parse_tree(static, embeddings=emb)                      # warm up outside the capture
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = G.parse_tree(static, embeddings=emb)
        for src in (other, states):
            static.copy_(src)
            g.replay()
            torch.cuda.synchronize()
            _same_tree(out, G.parse_tree(src, embeddings=emb), ("graph", emb))


@pytest.mark.gpu
def test_compiled_parse_tree_is_eager_bits_without_graph_breaks():
    states = _bits_case()
    for emb in (True, False):
        torch._dynamo.reset()

        def fn(s):
            return G.parse_tree(s * 1.0, embeddings=emb)
        got = torch.compile(fn, fullgraph=True)(states)
        _same_tree(got, G.parse_tree(states, embeddings=emb), ("compile", emb))
        torch._dynamo.reset()
        assert torch._dynamo.explain(fn)(states).graph_break_count == 0


@pytest.mark.gpu
def test_parse_tree_opcheck():
    states = _bits_case()[:3]
    for emb in (True, False):
        torch.library.opcheck(torch.ops.glom_b200.parse_tree, (states, 16, 16, 0.9, emb),
                              test_utils=("test_schema", "test_faketensor", "test_autograd_registration"))


@pytest.mark.gpu
def test_misaligned_state_view_gives_the_aligned_bits():
    from test_guard_bands import _misaligned
    states = _bits_case()
    f = _misaligned(states)
    _same_tree(G.parse_tree(f.tensor, embeddings=True), G.parse_tree(states, embeddings=True), "misaligned")
    assert not f.violations(0xFF)


# ====================================================================================================== GPU: guard bands
FENCE_GRIDS = [(1, 37), (16, 16), (64, 128)]


def _garbage(labels, seed):
    """Real labels with a fifth of the entries of each (slab, level) replaced, in turn, by -1, 2^31 - 1, n, a later
    patch (j > i) and an earlier non-root (when there is one)."""
    flat = labels.cpu().reshape(-1, labels.shape[-1]).numpy().copy()
    n = flat.shape[1]
    rng = np.random.default_rng(seed)
    for r in range(flat.shape[0]):
        nonroot = np.flatnonzero(flat[r] != np.arange(n))
        for q, i in enumerate(rng.permutation(n)[:max(1, n // 5)]):
            early = nonroot[nonroot < i]
            flat[r, i] = (-1, 2 ** 31 - 1, n, i + 1, early[0] if early.size else -1)[q % 5]
    return torch.from_numpy(flat).reshape(labels.shape).to(labels.device)


@pytest.mark.gpu
@pytest.mark.parametrize("grid", FENCE_GRIDS, ids=[f"{a}x{b}" for a, b in FENCE_GRIDS])
def test_island_tree_fenced(grid):
    """glom_b200_island_tree with and without states, on the labels of islands() and on garbage labels, fenced with the
    three fills: guards and inputs intact, outputs bit-identical across fills, equal to parse_tree (real labels) or to
    the oracle (garbage labels)."""
    from test_guard_bands import Fence, fenced_run, same_bits
    sh, sw = grid
    n, L, d, slabs = sh * sw, 3, 36, 2
    x, _ = _designed_slabs(sh, sw, L, d, slabs, True, seed=sw)
    x = x + 0.3 * np.random.default_rng(sh).standard_normal(x.shape).astype(np.float32)
    states = torch.from_numpy(x).to(DEV)
    public = G.parse_tree(states, grid=grid, embeddings=True)
    real = public.labels
    shape = (slabs, L, n)
    for name, labels in (("real", real), ("garbage", _garbage(real, sh * sw))):
        for with_states in (True, False):
            f = {"labels": Fence("labels", shape, torch.int32), "size": Fence("size", shape, torch.int32, "out"),
                 "parent": Fence("parent", shape, torch.int32, "out"), "containment": Fence("containment", shape, kind="out"),
                 "nested": Fence("nested", (slabs, L - 1), kind="out")}
            inputs = {"labels": labels}
            if with_states:
                f["states"] = Fence("states", states.shape, row_dims=2)
                f["embedding"] = Fence("embedding", (slabs, L, n, d), kind="out", row_dims=2)
                f["member_cos"] = Fence("member_cos", shape, kind="out")
                f["coherence"] = Fence("coherence", shape, kind="out")
                inputs["states"] = states

            def call(f):
                p = {k: (f[k].ptr if k in f else None) for k in ("states", "embedding", "member_cos", "coherence")}
                _native.island_tree(f["labels"].ptr, p["states"], slabs, n, L, d, f["size"].ptr, f["parent"].ptr,
                                    f["containment"].ptr, f["nested"].ptr, p["embedding"], p["member_cos"],
                                    p["coherence"], torch.cuda.current_stream().cuda_stream)
            got = fenced_run(f, inputs, call)[0]
            if name == "real":
                for k in got:
                    same_bits(got[k], getattr(public, k), (grid, name, with_states, k))
            else:
                t = G.ParseTree(labels, None, *(got.get(k) for k in ParseTreeFields[2:]))
                check_tree(t, labels, states if with_states else None, what=f"{grid} garbage")
