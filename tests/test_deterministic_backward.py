"""The deterministic backward: under torch.use_deterministic_algorithms(True) the gradients of Glom are bit-identical
from run to run (glom_b200_backward_ex / glom_b200_tokenize_backward_ex with deterministic = 1, DESIGN.md
"Deterministic backward").

CPU: the new entry points are exported and check their arguments before any device query; the workspace is the
default one; the only functions of libglom_b200.so with floating-point RED / ATOM instructions are the four default
kernels that the deterministic path replaces.
GPU: at every shape of test_backward_oracle, on both engines, one step and three chained steps: three runs (the module,
a deepcopy with fresh NaN-filled workspaces, a second CUDA stream) give the same bits, within the oracle's bounds of
grads_at_states and of the default (atomic) gradients.  Per-image steps do not read stale workspace, settle's one-pass
gradients equal the two-pass recipe bit for bit, and the flag changes no forward output.
"""
import contextlib
import copy
import ctypes
import os
import re
import shutil
import subprocess

import pytest
import torch

import glom_pytorch_b200 as G
from glom_pytorch_b200 import _native

import test_backward_oracle as BO

DEV = "cuda:0"
INVALID = -1


@contextlib.contextmanager
def deterministic(on=True):
    """torch.use_deterministic_algorithms(on) inside the block, the caller's setting restored afterwards."""
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


# ----------------------------------------------------------------------------------------------------------------- CPU
def test_new_symbols_are_exported():
    lib = ctypes.CDLL(G.LIB_PATH)
    for name in ("glom_b200_backward_ex", "glom_b200_tokenize_backward_ex"):
        assert name in _native.EXPORTS and hasattr(lib, name), name


def _backward_ex_rc(deterministic, tokens=16, steps=None, max_steps=1, grads=True):
    lib = _native.load()
    cfg = _native.make_cfg(256, 3, 16, False, 0, 0, "bf16")
    w = _native.WeightsRef(ctypes.sizeof(_native.WeightsRef), *([1024] * 8))
    g = _native.Grads(ctypes.sizeof(_native.Grads), *([1024, 1024, 1024, None] + [1024] * 8 if grads else [None] * 12))
    return lib.glom_b200_backward_ex(ctypes.byref(cfg), ctypes.byref(w), tokens, 1024, 1024, 1024, ctypes.byref(g), 2,
                                     steps, max_steps, 0, deterministic, 1024, 1 << 30, None)


@pytest.mark.parametrize("kw,msg", [
    (dict(deterministic=2), "deterministic must be 0 or 1"),
    (dict(deterministic=-1), "deterministic must be 0 or 1"),
    (dict(deterministic=1, tokens=None), "NULL"),
    (dict(deterministic=1, grads=False), "gradient pointers"),
    (dict(deterministic=1, steps=1026), "aligned"),
    (dict(deterministic=0, steps=1024, max_steps=-1), "max_steps"),
])
def test_backward_ex_argument_errors_before_device_query(kw, msg):
    """Without a GPU a device query fails with GLOM_B200_ERR_CUDA: INVALID means the check came first."""
    assert _backward_ex_rc(**kw) == INVALID
    assert msg in _native.load().glom_b200_last_error().decode()


@pytest.mark.parametrize("det,img,msg", [(2, 1024, "deterministic must be 0 or 1"), (1, None, "NULL")])
def test_tokenize_backward_ex_argument_errors_before_device_query(det, img, msg):
    lib = _native.load()
    rc = lib.glom_b200_tokenize_backward_ex(img, 1024, 1024, 1024, 1024, None, 2, 32, 32, 4, 64, det, 1024, 1 << 20, None)
    assert rc == INVALID
    assert msg in lib.glom_b200_last_error().decode()


def test_workspace_at_configs1_is_the_default_one():
    """configs[1] (dim 512, 6 levels, 256 patches) at batch 32: the deterministic path's buffers live in workspace
    regions that are dead when it runs, so its size query is the default one, unchanged."""
    cfg = _native.make_cfg(512, 6, 256, False, 0, 0, "bf16")
    assert _native.backward_workspace_bytes(cfg, 32) == 2_267_308_032


def _cuobjdump():
    for c in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if c and os.path.exists(c):
            return c
    return None


def test_sass_float_atomics_only_in_the_default_kernels():
    """The functions with a floating-point RED / ATOM are exactly the four default kernels the deterministic path
    replaces; no deterministic instantiation or reducer is among them."""
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not found")
    sass = subprocess.run([tool, "-sass", G.LIB_PATH], check=True, capture_output=True, text=True).stdout
    found, fn = set(), None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
        elif fn and re.search(r"\b(RED|ATOM)[A-Z]*\.[A-Za-z0-9_.]*\bF(16|32|64)(x\d)?\b", line):
            found.add(fn)
    want = {"bwd_gemm_kernelILi1ELb0E": "BW_DH", "bwd_gemm_kernelILi2ELb0E": "BW_DX", "colsum_acc_kernel": "colsum_acc",
            "init_grad_kernel": "init_grad"}
    matched = {k: [f for f in found if k in f] for k in want}
    assert all(len(v) == 1 for v in matched.values()), matched
    assert len(found) == len(want), sorted(found)


# ----------------------------------------------------------------------------------------------------------------- GPU
def _three_runs(m, img, S, iters, return_all, cot):
    """The gradients under the flag: the module, a deepcopy (fresh workspaces, NaN-filled by torch), a second stream."""
    with deterministic():
        out, g1 = BO._engine_run(m, img, S, iters, return_all, cot)
        _, g2 = BO._engine_run(copy.deepcopy(m), img, S, iters, return_all, cot)
        side = torch.cuda.Stream(DEV)
        side.wait_stream(torch.cuda.current_stream(DEV))
        with torch.cuda.stream(side):
            _, g3 = BO._engine_run(m, img, S, iters, return_all, cot)
    assert set(g1) == set(g2) == set(g3)
    for k in g1:
        assert torch.equal(g1[k], g2[k]), ("deepcopy", k)
        assert torch.equal(g1[k], g3[k]), ("second stream", k)
    return out, g1


@pytest.mark.gpu
@pytest.mark.parametrize("chained", [False, True], ids=["one_step", "chained_T3"])
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("name", list(BO.SHAPES))
def test_gradients_bit_identical(name, precision, chained):
    """One step from a carried state (d_levels), or three steps from init_levels with return_all (d_init_levels)."""
    m, img, S, n, g = BO._model(name, precision, seed=1 if chained else 0)
    T = 3 if chained else 1
    cot = torch.randn(((T + 1,) if chained else ()) + tuple(S.shape), generator=g)
    start = None if chained else S
    with deterministic(False):
        _, plain = BO._engine_run(m, img, start, T, chained, cot)
    out, got = _three_runs(m, img, start, T, chained, cot)
    want = {"d_img", "pos_emb.weight", "image_to_tokens.1.weight", "image_to_tokens.1.bias", *BO.NAMES,
            "init_levels" if chained else "d_levels"}
    assert set(got) == want, set(got) ^ want
    states = out.cpu() if chained else torch.stack([S, out.cpu()])
    ref, _, _ = BO._reference(m, img, states, cot, return_all=chained, carried=not chained)
    tol = BO.TOL[BO._path(name, precision)]
    errs = BO.errors(got, ref, m.levels, n)
    BO._report(name, f"deterministic {precision} T={T}", errs)
    BO.check(errs, tol, (name, precision, T, "vs grads_at_states"))
    BO.check(BO.errors(got, {k: plain[k] for k in ref}, m.levels, n), tol, (name, precision, T, "vs default"))


@pytest.mark.gpu
@pytest.mark.parametrize("name,steps", [("mixed_d256_n100", [3, 1, 0]), ("tc_d256_n576_mask_self", [1, 3]),
                                        ("tc_d256_n144_B5", [0, 3, 1, 3, 2])])
def test_per_image_steps_read_no_stale_workspace(name, steps):
    """forward(iters=<vector>, return_all=True): the backward workspace filled with 0xFF bytes (NaN in fp32 and bf16)
    or zeros before the backward gives the same finite gradients."""
    m, img, S, n, g = BO._model(name, "bf16", seed=2, batch=len(steps))
    T = max(steps)
    cot = torch.randn((T + 1,) + tuple(S.shape), generator=g)
    dev = torch.device(DEV)
    nbytes = _native.backward_workspace_bytes(m.engine_cfg(n), len(steps))
    runs = []
    with deterministic():
        for byte in (0xFF, 0):
            m._get_workspace(nbytes, dev, "_bwd_workspace").fill_(byte)
            runs.append(BO._engine_run(m, img, S, torch.tensor(steps), True, cot)[1])
    for k in runs[0]:
        assert torch.isfinite(runs[0][k]).all(), k
        assert torch.equal(runs[0][k], runs[1][k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("carried", [False, True])
@pytest.mark.parametrize("shape", ["tensor_core_bwd_n144", "cuda_core_bwd_n64"])
def test_settle_gradients_equal_the_two_pass_recipe(shape, carried):
    """settle(differentiable=True, return_all=True) against forward(iters=steps, return_all=True) with the cotangents of
    the frozen tail folded in the backward's order (test_settle_train.py): bit-identical under the flag."""
    import test_settle_train as ST
    m, img, lv, tol, steps = ST._grad_setup(shape, carried)
    T = int(steps.max())
    shape_s = (img.shape[0], (img.shape[2] // m.patch_size) ** 2, m.levels, m.dim)
    cot = torch.randn((ST.MAX_ITERS + 1,) + shape_s, generator=torch.Generator().manual_seed(5)).to(DEV)

    def two_pass(x, s):
        out = m(x, iters=steps, levels=s, return_all=True)
        fold = cot[ST.MAX_ITERS]
        for t in range(ST.MAX_ITERS - 1, T - 1, -1):
            fold = fold + cot[t]
        return (out * torch.cat([cot[:T], fold[None]])).sum()

    with deterministic():
        got = ST._grads(m, img, lv, ST._one_pass_loss(m, tol, cot, True))
        want = ST._grads(m, img, lv, two_pass)
    assert set(got) == set(want)
    for k in want:
        assert torch.isfinite(got[k]).all(), k
        assert torch.equal(got[k], want[k]), (shape, carried, k, ST._rel(got[k], want[k]))


@pytest.mark.gpu
def test_configs1_batch8_bit_identical():
    """configs[1] dims at batch 8 (d_pos sums 8 images x 5 top-down groups per element and step): two flag-on runs give
    the same bits.  The number of elements two default runs disagree on is printed for information only."""
    m, img, S, n, g = BO._model("tc_config2_dims", "bf16", batch=8)
    T = 2
    cot = torch.randn((T + 1,) + tuple(S.shape), generator=g)
    with deterministic(False):
        a = BO._engine_run(m, img, S, T, True, cot)[1]
        b = BO._engine_run(m, img, S, T, True, cot)[1]
    diff = {k: int((a[k] != b[k]).sum()) for k in a}
    print(f"[deterministic] configs[1] dims, batch 8, default backward: elements differing between two runs {diff}")
    with deterministic():
        a = BO._engine_run(m, img, S, T, True, cot)[1]
        b = BO._engine_run(m, img, S, T, True, cot)[1]
    for k in a:
        assert torch.equal(a[k], b[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_forward_outputs_unchanged_by_the_flag(precision):
    """forward, settle and settle_queue under the flag (outputs and fresh workspaces NaN-filled by torch) give the same
    bits as without it."""
    torch.manual_seed(0)
    m = G.Glom(dim=256, levels=3, image_size=48, patch_size=4, precision=precision).to(DEV).eval()
    img = torch.randn(5, 3, 48, 48, generator=torch.Generator().manual_seed(1)).to(DEV)

    def outputs(mod):
        with torch.no_grad():
            res = {"forward": mod(img, iters=3), "return_all": mod(img, iters=3, return_all=True)}
            if precision == "bf16":
                res["settle"], res["settle_steps"] = mod.settle(img, 1e-2, max_iters=6)
                res["queue"], res["queue_steps"] = mod.settle_queue(img, 1e-2, max_iters=6, slots=2)
        torch.cuda.synchronize()
        return res

    off = outputs(m)
    with deterministic():
        on = outputs(copy.deepcopy(m))
    for k in off:
        assert torch.equal(off[k], on[k]), k
