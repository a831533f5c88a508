"""Island analytics: the numpy oracle on constructed cases (CPU), and the CUDA kernels
(glom_b200_islands through the C ABI) against the oracle (GPU)."""
import numpy as np
import pytest
import torch

from oracle.islands_oracle import islands as islands_oracle


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


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(2, 3, 6, 8, 4, 64), (1, 1, 16, 16, 6, 512), (1, 2, 1, 5, 2, 12), (1, 1, 24, 24, 2, 128)])
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
