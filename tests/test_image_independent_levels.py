"""A forward from init_levels runs the work whose inputs are the same in every image once, for the representative rows.

Every image starts from init_levels, so S_t[l] differs between images only for l <= t - 1.  At the steps t < L the
engine runs the K1 groups, K3 levels and K2 levels whose inputs do not yet differ for the first lcm(n, 128) rows only,
and K2 reads those inputs back from row r mod n (DESIGN.md, "Image-independent levels").  No bit may change:

* a carried state takes the full path, so ``forward(img)`` must equal ``forward(img, levels=init_levels broadcast)``;
* at batch 1 nothing is reduced, so ``forward(img)`` must equal the per-image calls concatenated.

The CPU test enumerates the reduced K1 / K2 / K3 schedules (tests/native/ii_sched_harness.cu) for every pair count.
"""
import contextlib
import os
import subprocess

import pytest
import torch

from glom_pytorch_b200 import _native

DEV = "cuda:0"
HERE = os.path.dirname(os.path.abspath(__file__))


# ----------------------------------------------------------------------------- CPU: the schedules
def test_reduced_schedules_for_every_pair_count(tmp_path):
    """Every required K1 / K2 tile and K3 item is dealt exactly once and nothing else, for pair counts 1..66, L = 2..8 and
    n from 1 to 784 (ragged, non-multiple-of-128 and key-pass shapes); at configs[1] over 12 steps the executed counts
    are 22,296 of 30,976 K1 tiles, 6,898 of 8,448 K2 cost units and 3,306 of 4,608 K3 items."""
    import test_production_batch as PB
    nvcc = PB._nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    csrc = os.path.join(os.path.dirname(HERE), "glom_pytorch_b200", "csrc")
    exe = str(tmp_path / "ii_sched_harness")
    subprocess.run([nvcc, "-std=c++17", "-O2", "-gencode", "arch=compute_90a,code=sm_90a", "-I", csrc,
                    os.path.join(HERE, "native", "ii_sched_harness.cu"), "-o", exe], check=True, capture_output=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(r.stdout)
    assert r.returncode == 0, r.stdout
    lines = r.stdout.strip().splitlines()
    head = lines[-2].split()
    assert head[0] == "configs" and int(head[1]) > 10000 and head[2:] == ["failures", "0"], r.stdout
    assert lines[-1].split() == ["c1", "k1_tiles", "22296", "30976", "k2_cost", "6898", "8448", "k3_items", "3306",
                                 "4608"], r.stdout


# ----------------------------------------------------------------------------- GPU
def _glom(dim, L, isz, p, **kw):
    import test_production_batch as PB
    return PB._glom(dim, L, isz, p, **kw)


def _images(m, B, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, 3, m.image_side, m.image_side, generator=g).to(DEV)


def _equal(a, b, what):
    assert a.shape == b.shape, (what, tuple(a.shape), tuple(b.shape))
    if not torch.equal(a, b):
        diff = a != b
        raise AssertionError(f"{what}: {int(diff.sum())} of {a.numel()} elements differ, first at "
                             f"{diff.nonzero()[0].tolist()}")


def _carried(m, img):
    n = (m.image_side // m.patch_size) ** 2
    return m.init_levels.detach().float().expand(img.shape[0], n, m.levels, m.dim).clone()


def _check(m, img, iters, return_all, slices=True):
    with torch.no_grad():
        out = m(img, iters=iters, return_all=return_all)
        ref = m(img, iters=iters, levels=_carried(m, img), return_all=return_all)
        torch.cuda.synchronize()
        _equal(out, ref, f"init_levels vs carried init_levels, iters={iters} return_all={return_all}")
        if slices:
            per = torch.cat([m(img[b:b + 1], iters=iters, return_all=return_all) for b in range(img.shape[0])],
                            dim=1 if return_all else 0)
            _equal(out, per, f"batch vs per-image calls, iters={iters} return_all={return_all}")
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("iters", [7, 8, 12])
@pytest.mark.parametrize("return_all", [False, True])
def test_configs1_batch32(iters, return_all):
    """configs[1] at B = 32: the reduced steps are 0..5; iters = 7 is the smallest eligible count."""
    m = _glom(512, 6, 224, 14)
    _check(m, _images(m, 32, 1), iters, return_all, slices=(iters == 12))


# (dim, L, image side, patch, batch): L = 2, 3, 8; n = 36, 144, 576 and 784 (lcm(n, 128) spans several images, ragged
# 256-row blocks, key passes beyond 576 columns)
SHAPES = {
    "L2_n64": (128, 2, 32, 4, 6),
    "L3_n144": (256, 3, 48, 4, 12),
    "L8_n64": (128, 8, 32, 4, 5),
    "n36": (128, 4, 24, 4, 40),
    "n576": (256, 3, 96, 4, 4),
    "n784": (128, 3, 112, 4, 10),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SHAPES))
@pytest.mark.parametrize("return_all", [False, True])
def test_shapes(name, return_all):
    dim, L, isz, p, B = SHAPES[name]
    m = _glom(dim, L, isz, p)
    _check(m, _images(m, B, 2), L + 2, return_all)


@pytest.mark.gpu
@pytest.mark.parametrize("attend_self", [False, True])
def test_radius_mask(attend_self):
    m = _glom(256, 4, 48, 4, local_consensus_radius=2, consensus_self=attend_self)
    _check(m, _images(m, 12, 3), 6, True)


@contextlib.contextmanager
def _sm_target(sms):
    _native.set_sm_count_target(sms)
    try:
        yield
    finally:
        _native.set_sm_count_target(0)


@pytest.mark.gpu
@pytest.mark.parametrize("sms", [2, 3])
def test_sm_count_targets(sms):
    """One pair (two K3 CTAs) and an odd K3 CTA count walk the reduced lists: the default grid's bits."""
    m = _glom(256, 3, 48, 4)
    img = _images(m, 12, 4)
    with torch.no_grad():
        full = m(img, iters=5, return_all=True)
    with _sm_target(sms):
        out = _check(m, img, 5, True, slices=False)
    _equal(out, full, f"target {sms} vs default grid")


@pytest.mark.gpu
def test_graph_capture():
    """A captured forward from init_levels replays the eager bits (the reduction is decided on the host)."""
    import copy
    m = _glom(256, 3, 48, 4)
    ref = copy.deepcopy(m)
    img = _images(m, 12, 5)
    static = img.clone()
    with torch.no_grad():
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = m(static, iters=5, return_all=True)
        img2 = _images(m, 12, 6)
        static.copy_(img2)
        g.replay()
        torch.cuda.synchronize()
        _equal(out, _check(ref, img2, 5, True, slices=False), "graph replay vs eager")
