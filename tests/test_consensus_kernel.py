"""Consensus attention kernel (K3) on its own: after one bf16 step from a random state, the consensus C left in the
workspace matches the oracle's bf16 emulation, for the 128-key and 256-key S blocks, the radius mask and attend-self,
and a second identical step reproduces C bit for bit (the producer / consumer hand-offs of the kernel are race-free)."""
import numpy as np
import pytest
import torch

import glom_pytorch_b200 as G
from glom_pytorch_b200 import _native
from oracle import glom_oracle as O

DEV = "cuda:0"

# (dim, levels, image_size, patch_size, consensus_self, local_consensus_radius, batch)
CASES = {
    "n64_one_tile": (128, 3, 32, 4, False, 0, 2),
    "n256_256key_block": (512, 2, 64, 4, False, 0, 2),
    "n576_128key_blocks": (128, 2, 96, 4, False, 0, 1),
    "n256_radius_mask": (128, 2, 64, 4, False, 3, 2),
    "n256_attend_self": (128, 2, 64, 4, True, 0, 2),
}


def _consensus_from_workspace(m, img, state):
    with torch.no_grad():
        m(img, iters=1, levels=state)
    torch.cuda.synchronize()
    B, n, L, d = state.shape
    off, nb = _native.workspace_offset(m.engine_cfg(n), B, 1, False, 1)
    return m._workspace[off:off + nb].view(torch.bfloat16).float().reshape(B, n, L, d).cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_consensus_matches_oracle_and_is_deterministic(name):
    dim, L, isz, p, attend_self, radius, B = CASES[name]
    torch.manual_seed(0)
    m = G.Glom(dim=dim, levels=L, image_size=isz, patch_size=p, consensus_self=attend_self,
               local_consensus_radius=radius, precision="bf16").to(DEV).eval()
    n = (isz // p) ** 2
    rng = np.random.default_rng(1)
    img = torch.from_numpy(rng.standard_normal((B, 3, isz, isz)).astype(np.float32)).to(DEV)
    # a random state (scaled so that the attention is selective) instead of init_levels, whose rows are all equal
    S = (2.0 * rng.standard_normal((B, n, L, dim))).astype(np.float32)
    state = torch.from_numpy(S).to(DEV)

    C = _consensus_from_workspace(m, img, state)
    mask = O.radius_mask(isz // p, radius) if radius > 0 else None
    want = O.consensus(S, attend_self, mask, emulate="bf16")
    err = np.abs(C - want).max()
    assert np.isfinite(C).all()
    assert err <= 2e-2 * max(1.0, np.abs(want).max()), (name, err)
    # C is not trivially the state: the test would not notice a kernel that skipped the softmax otherwise
    assert np.abs(C - O.bf16_round(S)).max() > 10 * max(err, 1e-3)

    C2 = _consensus_from_workspace(m, img, state)
    assert np.array_equal(C, C2), name
