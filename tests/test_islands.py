"""Island analytics: the numpy oracle on constructed cases (CPU), and the CUDA kernels
(glom_b200_islands through the C ABI) against the oracle (GPU).

The labels are checked bit for bit against `components` run on the kernel's own fp32 cosines, so thresholds may sit on
the data (one equals a kernel cosine: that edge is kept, the comparison is >=).  The cosine maps are compared with the
float64 `edges` per (slab, level), max-abs, within COS_BOUND, set at about 3x the worst error observed on one H100 80GB
HBM3 (400 W power limit) [observed: 1.72e-7 at 64 x 128, d = 12].  Adversarial components at the API bound n = 8192: a serpentine path whose
minimum label must travel the whole path, a checkerboard (n islands), a constant grid (one island)."""
from collections import deque

import numpy as np
import pytest
import torch

from oracle.islands_oracle import components, edges
from oracle.islands_oracle import islands as islands_oracle

COS_BOUND = 5e-7


def _planted(side_h, side_w, L, d, seed=0, noise=0.02):
    """States with planted islands: level l splits the grid into vertical bands of width 2**l (clipped); patches of a
    band share one random direction plus small noise.  Returns (states (n, L, d), expected band id per level)."""
    rng = np.random.default_rng(seed)
    n = side_h * side_w
    x = np.empty((n, L, d), dtype=np.float32)
    bands = np.empty((L, n), dtype=np.int64)
    for l in range(L):
        width = min(side_w, 2 ** l)
        nb = -(-side_w // width)
        dirs = rng.standard_normal((nb, d)).astype(np.float32) * 3.0
        for i in range(n):
            b = (i % side_w) // width
            bands[l, i] = b
            x[i, l] = dirs[b] + noise * rng.standard_normal(d).astype(np.float32)
    return x, bands


def test_oracle_finds_planted_bands():
    x, bands = _planted(6, 8, 4, 64)
    r = islands_oracle(x, 6, 8, threshold=0.9)
    for l in range(4):
        assert r["num_islands"][l] == len(set(bands[l]))
        # same band <=> same label
        lab = r["labels"][l]
        for i in range(48):
            for j in range(48):
                assert (lab[i] == lab[j]) == (bands[l, i] == bands[l, j])
        assert r["labels"][l].min() == 0
    assert r["agreement"].shape == (4, 48) and r["agreement"][3].min() > 0.9       # one band: everybody agrees
    assert np.all(r["cos_right"][:, 7::8] == 0) and np.all(r["cos_down"][:, -8:] == 0)


def test_oracle_single_patch_and_threshold_extremes():
    x = np.random.default_rng(1).standard_normal((1, 2, 8)).astype(np.float32)
    r = islands_oracle(x, 1, 1, 0.5)
    assert r["num_islands"].tolist() == [1, 1] and r["agreement"].tolist() == [[1.0], [1.0]]
    y = np.random.default_rng(2).standard_normal((12, 1, 16)).astype(np.float32)
    assert islands_oracle(y, 3, 4, -2.0)["num_islands"][0] == 1        # every edge kept
    assert islands_oracle(y, 3, 4, 2.0)["num_islands"][0] == 12        # no edge kept


def _direct(x, side_h, side_w, threshold):
    """The definition in include/glom_b200.h, one patch at a time: cosines with np.dot, components by breadth-first
    search from each patch in index order (so each component's id is its smallest patch index)."""
    n, L, _ = x.shape
    x = x.astype(np.float64)
    cr, cd, agr = np.zeros((L, n)), np.zeros((L, n)), np.zeros((L, n))
    labels, counts = np.full((L, n), -1, dtype=np.int32), np.zeros(L, dtype=np.int32)

    def cos(a, b):
        return float(np.dot(a, b) / max(np.linalg.norm(a) * np.linalg.norm(b), 1e-12))
    for l in range(L):
        nbrs = [[] for _ in range(n)]
        for i in range(n):
            h, w = divmod(i, side_w)
            if w + 1 < side_w:
                cr[l, i] = cos(x[i, l], x[i + 1, l])
                nbrs[i].append((i + 1, cr[l, i]))
                nbrs[i + 1].append((i, cr[l, i]))
            if h + 1 < side_h:
                cd[l, i] = cos(x[i, l], x[i + side_w, l])
                nbrs[i].append((i + side_w, cd[l, i]))
                nbrs[i + side_w].append((i, cd[l, i]))
        for i in range(n):
            agr[l, i] = np.mean([c for _, c in nbrs[i]]) if nbrs[i] else 1.0
            if labels[l, i] >= 0:
                continue
            counts[l] += 1
            labels[l, i] = i
            todo = deque([i])
            while todo:
                j = todo.popleft()
                for k, c in nbrs[j]:
                    if c >= threshold and labels[l, k] < 0:
                        labels[l, k] = i
                        todo.append(k)
    return dict(cos_right=cr, cos_down=cd, agreement=agr, labels=labels, num_islands=counts)


@pytest.mark.parametrize("grid", [(6, 8), (1, 9), (9, 1), (5, 7)])
def test_split_oracle_is_the_definition(grid):
    """islands() = edges() + components() + the agreement map equals the patch-by-patch definition, on planted and
    random states, at thresholds on both sides of the data."""
    sh, sw = grid
    x, _ = _planted(sh, sw, 3, 16, seed=3, noise=0.3)
    y = np.random.default_rng(4).standard_normal((sh * sw, 2, 8)).astype(np.float32)
    for states, thr in ((x, 0.9), (x, 0.99), (y, 0.0), (y, 0.3), (y, -2.0)):
        got, want = islands_oracle(states, sh, sw, thr), _direct(states, sh, sw, thr)
        for k in ("cos_right", "cos_down", "agreement"):
            assert np.allclose(got[k], want[k], rtol=0, atol=1e-12), k
        assert np.array_equal(got["labels"], want["labels"]) and np.array_equal(got["num_islands"], want["num_islands"])
        cr, cd = edges(states, sh, sw)
        assert np.array_equal(cr, got["cos_right"]) and np.array_equal(cd, got["cos_down"])


# (T1, B, side_h, side_w, L, d): planted bands; grids of one row / one column / 5 x 13; d = 4, 20, 132, 516 (d / 4 = 1,
# 5, 33, 129 float4 per lane loop); 3000 slabs; n = 8192 (the API bound) and n = 8190
@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(2, 3, 6, 8, 4, 64), (1, 1, 16, 16, 6, 512), (1, 2, 1, 5, 2, 12), (1, 1, 24, 24, 2, 128),
                                   (1, 2, 1, 37, 3, 64), (1, 2, 37, 1, 3, 64), (2, 1, 5, 13, 4, 32),
                                   (1, 2, 6, 8, 3, 4), (1, 2, 6, 8, 2, 20), (1, 1, 6, 8, 2, 132), (1, 1, 4, 4, 2, 516),
                                   (1000, 3, 2, 3, 2, 16), (1, 1, 64, 128, 2, 16), (1, 1, 90, 91, 1, 12)])
def test_gpu_islands_match_oracle(shape):
    import glom_pytorch_b200 as G
    T1, B, sh, sw, L, d = shape
    rng = np.random.default_rng(7)
    xs = np.stack([np.stack([_planted(sh, sw, L, d, seed=int(rng.integers(1 << 30)), noise=0.05 * (t + 1))[0]
                             for _ in range(B)]) for t in range(T1)])               # (T1, B, n, L, d)
    thr = 0.8
    want = islands_oracle(xs, sh, sw, thr)
    got = G.islands(torch.from_numpy(xs).cuda(), grid=(sh, sw), threshold=thr)
    torch.cuda.synchronize()
    for k in ("cos_right", "cos_down", "agreement"):
        assert np.abs(getattr(got, k).cpu().numpy() - want[k]).max() <= 2e-5, k
    safe = (np.abs(want["cos_right"] - thr) > 1e-4).all() and (np.abs(want["cos_down"] - thr) > 1e-4).all()
    assert safe                                                       # planted data keeps clear of the threshold
    assert np.array_equal(got.labels.cpu().numpy(), want["labels"])
    assert np.array_equal(got.num_islands.cpu().numpy(), want["num_islands"])


@pytest.mark.gpu
def test_gpu_islands_on_a_forward_slab():
    """End to end on real states: Glom.forward(return_all=True) -> islands; early iterations of a random-init model have
    no planted structure, so only the oracle comparison of the similarity maps is asserted."""
    import glom_pytorch_b200 as G
    torch.manual_seed(0)
    m = G.Glom(dim=128, levels=4, image_size=32, patch_size=4).cuda().eval()
    with torch.no_grad():
        allv = m(torch.randn(2, 3, 32, 32, device="cuda"), iters=4, return_all=True)
    r = G.islands(allv, threshold=0.5)
    want = islands_oracle(allv.cpu().numpy(), 8, 8, 0.5)
    assert r.labels.shape == (5, 2, 4, 64) and r.num_islands.shape == (5, 2, 4)
    assert np.abs(r.agreement.cpu().numpy() - want["agreement"]).max() <= 2e-5
    # slab 0 is the broadcast init_levels: every patch identical -> one island per level
    assert (r.num_islands[0] == 1).all() and (r.agreement[0] > 0.999).all()


@pytest.mark.gpu
@pytest.mark.parametrize("grid,L,d,slabs", [((16, 16), 3, 16, 4), ((5, 13), 2, 4, 3), ((1, 37), 2, 20, 2),
                                            ((64, 128), 1, 12, 1)])
def test_gpu_labels_from_the_kernels_own_cosines(grid, L, d, slabs):
    """Random (unplanted) states: the cosine maps against the float64 edges() per (slab, level), also for the states
    scaled by 1e-3 and 300; labels and num_islands bit for bit equal to components() on the kernel's own fp32 maps, at
    thresholds at quantiles of the kernel's cosines and at one kernel cosine exactly (that edge is kept)."""
    import glom_pytorch_b200 as G
    sh, sw = grid
    x = np.random.default_rng(11).standard_normal((slabs, sh * sw, L, d)).astype(np.float32)
    want_r, want_d = edges(x, sh, sw)
    worst = 0.0
    for scale in (1.0, 1e-3, 300.0):
        got = G.islands(torch.from_numpy(x * np.float32(scale)).cuda(), grid=grid, threshold=0.5)
        for k, want in (("cos_right", want_r), ("cos_down", want_d)):
            err = np.abs(getattr(got, k).cpu().numpy() - want).reshape(slabs * L, -1).max(axis=1)   # per (slab, level)
            worst = max(worst, float(err.max()))
    print(f"[islands] {grid} L={L} d={d}: cos max-abs {worst:.3e}")
    assert worst <= COS_BOUND, worst
    xd = torch.from_numpy(x).cuda()
    got = G.islands(xd, grid=grid, threshold=0.5)
    cr = got.cos_right.cpu().numpy().reshape(slabs * L, sh, sw)
    cd = got.cos_down.cpu().numpy().reshape(slabs * L, sh, sw)
    inner = np.concatenate([cr[:, :, :-1].ravel(), cd[:, :-1, :].ravel()])
    thresholds = [float(np.quantile(inner, q)) for q in (0.05, 0.3, 0.6, 0.9)]
    if sw > 1:                                               # an interior right edge of the last (slab, level)
        hit = (sh // 2, sw // 2 - 1)
        thresholds.append(float(cr[-1][hit]))
    for thr in thresholds:
        thr = float(np.float32(thr))                         # the kernel compares in fp32
        got = G.islands(xd, grid=grid, threshold=thr)
        lab, num = got.labels.cpu().numpy(), got.num_islands.cpu().numpy()
        want_lab, want_num = components(got.cos_right.cpu().numpy(), got.cos_down.cpu().numpy(), sh, sw, np.float32(thr))
        assert np.array_equal(lab, want_lab) and np.array_equal(num, want_num), thr
    if sw > 1:
        i = hit[0] * sw + hit[1]
        assert lab.reshape(slabs * L, -1)[-1, i] == lab.reshape(slabs * L, -1)[-1, i + 1]    # cos == threshold: kept


def _serpentine(sh, sw, d):
    """Cell k of the boustrophedon path over the grid holds e_(k mod d) + e_((k+1) mod d), d > 2 * side_w: path
    neighbours have cosine 0.5, every other pair of grid neighbours 0 -> one island, a path of n cells."""
    assert d > 2 * sw
    x = np.zeros((sh * sw, 1, d), dtype=np.float32)
    for k in range(sh * sw):
        h, w = divmod(k, sw)
        i = h * sw + (w if h % 2 == 0 else sw - 1 - w)
        x[i, 0, k % d] += 1.0
        x[i, 0, (k + 1) % d] += 1.0
    return x


def _checkerboard(sh, sw, d):
    x = np.zeros((sh * sw, 1, d), dtype=np.float32)
    hw = np.add.outer(np.arange(sh), np.arange(sw)).ravel() % 2
    x[np.arange(sh * sw), 0, hw] = 1.0
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("grid,d", [((64, 128), 260), ((5, 7), 16), ((90, 91), 184)])
def test_gpu_adversarial_components(grid, d):
    """A serpentine path covering the grid (one island whose minimum label walks the whole path), a checkerboard of two
    orthogonal vectors (n islands) and a constant grid (one island), at the API bound n = 8192, at n = 8190 and on a
    small grid."""
    import glom_pytorch_b200 as G
    sh, sw = grid
    n = sh * sw
    rng = np.random.default_rng(5)
    cases = {"serpentine": (_serpentine(sh, sw, d), 1),
             "checkerboard": (_checkerboard(sh, sw, d), n),
             "constant": (np.broadcast_to(rng.standard_normal(d).astype(np.float32), (n, 1, d)).copy(), 1)}
    for name, (x, count) in cases.items():
        got = G.islands(torch.from_numpy(x).cuda(), grid=grid, threshold=0.25)
        want = islands_oracle(x, sh, sw, 0.25)
        assert want["num_islands"][0] == count, name
        assert np.abs(got.cos_right.cpu().numpy() - want["cos_right"]).max() <= COS_BOUND, name
        assert np.abs(got.cos_down.cpu().numpy() - want["cos_down"]).max() <= COS_BOUND, name
        assert np.array_equal(got.labels.cpu().numpy(), want["labels"]), name
        assert got.num_islands.cpu().numpy().tolist() == [count], name
