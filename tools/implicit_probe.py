"""Training through settle, unrolled against implicit: settle(differentiable=True) vs settle(differentiable="implicit").

configs[1] (dim 512, 6 levels, 224/14 = 256 patches), batch 32, a contracting model (second MLP layers x 0.1), settle
with tol 1e-3 and max_iters 12 from init_levels, loss = mean(levels[:, :, -1] ** 2).  Rounds alternate the two modes;
each round times --reps training steps with CUDA events (forward and backward separately) and records
torch.cuda.max_memory_allocated of the step.  Also reports the forward steps and the adjoint passes K_b, and the time of
one adjoint pass (implicit backward with 5 passes minus 1 pass, adjoint_tol = -1, over 4) against one reverse step of
the existing backward (glom_b200_backward on 6 minus 2 copies of S*, over 4).  The card's name and power limit are read
in the same run.  Prints one JSON line (and writes it to --out).

    python tools/implicit_probe.py [--rounds 6] [--reps 5] [--out /tmp/implicit_probe.json]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import glom_pytorch_b200 as G  # noqa: E402
from glom_pytorch_b200 import _native  # noqa: E402
from glom_pytorch_b200.glom import _aligned_bytes  # noqa: E402
from tools.deterministic_probe import card  # noqa: E402

DEV = "cuda:0"
TOL, MAX_ITERS = 1e-3, 12


def step(model, img, mode, ev):
    model.zero_grad(set_to_none=True)
    torch.cuda.reset_peak_memory_stats()
    ev[0].record()
    levels, steps = model.settle(img, TOL, MAX_ITERS, differentiable=mode)
    loss = levels[:, :, -1].square().mean()
    ev[1].record()
    loss.backward()
    ev[2].record()
    return steps


def timed(fn, reps=5):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for _ in range(reps):
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return statistics.median(out)


def pass_costs(model, img):
    """-> (ms of one adjoint pass, ms of one reverse step of glom_b200_backward), both at S*."""
    with torch.no_grad():
        tokens = model.tokens(img)
        S, _ = model.settle(img, TOL, MAX_ITERS)
    b, n = tokens.shape[:2]
    cfg = model.engine_cfg(n)
    wts = [q.detach().float().contiguous() for q in model._mlp_params()]
    pos = model.pos_emb.weight[:n].detach().contiguous()
    cot = torch.randn_like(S)
    names = ("d_bu_w1", "d_bu_b1", "d_bu_w2", "d_bu_b2", "d_td_w1", "d_td_b1", "d_td_w2", "d_td_b2")
    g = {"d_tokens": torch.zeros_like(tokens), "d_pos": torch.zeros_like(pos)}
    g.update({k: torch.zeros_like(w) for k, w in zip(names, wts)})
    ptrs = {k: v.data_ptr() for k, v in g.items()}
    stream = torch.cuda.current_stream().cuda_stream
    K = torch.empty(b, dtype=torch.int32, device=DEV)
    ws = _aligned_bytes(_native.backward_implicit_workspace_bytes(cfg, b), torch.device(DEV))

    def implicit(passes):
        _native.backward_implicit(cfg, [w.data_ptr() for w in wts], tokens.data_ptr(), pos.data_ptr(), S.data_ptr(),
                                  cot.data_ptr(), ptrs, b, passes, -1.0, K.data_ptr(), None, ws.data_ptr(), ws.numel(),
                                  stream)
    one, five = timed(lambda: implicit(1)), timed(lambda: implicit(5))
    del ws
    states = S[None].expand((7,) + tuple(S.shape)).contiguous()
    d_state0 = torch.zeros_like(S)
    bws = _aligned_bytes(_native.backward_workspace_bytes(cfg, b), torch.device(DEV))

    def unrolled(steps):
        _native.backward(cfg, [w.data_ptr() for w in wts], tokens.data_ptr(), pos.data_ptr(), states.data_ptr(),
                         cot.data_ptr(), dict(ptrs, d_state0=d_state0.data_ptr()), b, steps, False, bws.data_ptr(),
                         bws.numel(), stream)
    two, six = timed(lambda: unrolled(2)), timed(lambda: unrolled(6))
    return (five - one) / 4, (six - two) / 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.manual_seed(0)
    model = G.Glom(dim=512, levels=6, image_size=224, patch_size=14).to(DEV).train()
    with torch.no_grad():
        model.bottom_up.net[3].weight.mul_(0.1)
        model.top_down.net[3].weight.mul_(0.1)
    img = torch.randn(32, 3, 224, 224, generator=torch.Generator().manual_seed(1)).to(DEV)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    modes = (True, "implicit")
    res = {m: {"forward_ms": [], "backward_ms": [], "max_memory_gb": []} for m in modes}
    steps = {}
    for mode in modes:                                              # warm-up: workspaces, packing, first launches
        for _ in range(2):
            steps[mode] = step(model, img, mode, ev)
    torch.cuda.synchronize()
    for r in range(args.rounds):
        for mode in (modes if r % 2 == 0 else modes[::-1]):
            for _ in range(args.reps):
                step(model, img, mode, ev)
                torch.cuda.synchronize()
                res[mode]["forward_ms"].append(ev[0].elapsed_time(ev[1]))
                res[mode]["backward_ms"].append(ev[1].elapsed_time(ev[2]))
                res[mode]["max_memory_gb"].append(torch.cuda.max_memory_allocated() / 1e9)
    adjoint_steps = model.last_adjoint[0].tolist()
    adjoint_ms, reverse_ms = pass_costs(model, img)
    out = {"card": card(), "config": "configs[1] dim=512 L=6 224/14 batch=32, second MLP layers x0.1, settle tol 1e-3 "
                                     "max_iters 12, loss mean(levels[:, :, -1]^2)",
           "rounds": args.rounds, "reps": args.reps, "forward_steps": steps["implicit"].tolist(),
           "adjoint_steps": adjoint_steps}
    for mode, tag in ((True, "unrolled"), ("implicit", "implicit")):
        out[tag] = {k: round(statistics.median(v), 3) for k, v in res[mode].items()}
    out["adjoint_pass_ms"] = round(adjoint_ms, 3)
    out["reverse_step_ms"] = round(reverse_ms, 3)
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
