"""Training through Glom.settle at configs[1] shapes (dim=512 L=6 224/14, batch 32, max_iters 12, bf16).

A training step is: settle, then the loss on slab 7's top level of the return_all states (as in bench.py's train step),
then its backward.  It is done two ways:
  one-pass  states, _ = settle(img, tol, return_all=True, differentiable=True)
  two-pass  _, steps = settle(img, tol) under no_grad, then forward(img, iters=steps, return_all=True)
            (slab min(7, max(steps)), the same values: slabs past an image's step count repeat its last state).
On the contracting model of tools/settle_probe.py (b) (both second MLP layers zeroed, start = fixed point + noise):
  (a) even images stop by step 3, odd ones never;
  (b) every image stops by step 3: the one-pass backward then runs 12 - max(steps) reverse steps in which every image is
      frozen; their cost per step is (one-pass backward - two-pass backward) / (12 - max(steps)).
On the randomly initialised bench model:
  (c) the backward of forward(iters=<half at 3, half at 12>) and of forward(iters=12), as in tools/iters_probe.py (c).

Forward and backward milliseconds are reported separately: medians of interleaved rounds of CUDA-event-timed steps.  The
card's name and power limit are read in the same run.  Prints one JSON line (and writes it to --out).

    python tools/settle_train_probe.py [--rounds 5] [--reps 5] [--out /tmp/settle_train_probe.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import glom_pytorch_b200 as G  # noqa: E402

MAX_ITERS = 12
B = 32


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, limit = (q.stdout.strip().split(", ") + ["?", "?"])[:2] if q.returncode == 0 else (torch.cuda.get_device_name(0), "?")
    return {"name": name, "power_limit": limit}


def summary(v):
    return {"median_ms": round(statistics.median(v), 4), "min_ms": round(min(v), 4), "max_ms": round(max(v), 4)}


def step_times(model, loss_fn, reps):
    """(forward ms, backward ms) of a training step, averaged over `reps` steps timed with CUDA events."""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    f = b = 0.0
    for _ in range(reps):
        model.zero_grad(set_to_none=True)
        ev[0].record()
        loss = loss_fn()
        ev[1].record()
        loss.backward()
        ev[2].record()
        torch.cuda.synchronize()
        f += ev[0].elapsed_time(ev[1])
        b += ev[1].elapsed_time(ev[2])
    return f / reps, b / reps


def compare(model, fns, rounds, reps):
    for fn in fns.values():                          # warm-up of every shape
        step_times(model, fn, 2)
    runs = {k: ([], []) for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            f, b = step_times(model, fn, reps)
            runs[k][0].append(f)
            runs[k][1].append(b)
    return {k: {"forward": summary(f), "backward": summary(b), "step_median_ms": round(statistics.median(
        [x + y for x, y in zip(f, b)]), 4)} for k, (f, b) in runs.items()}


def change(states):
    """r[b, k - 1] = max_l sqrt(sum_i |S_k - S_{k-1}|^2 / sum_i |S_k|^2), float64, from (T+1, B, n, L, d) states."""
    out = []
    for k in range(1, states.shape[0]):
        s1, s0 = states[k].double(), states[k - 1].double()
        num, den = ((s1 - s0) ** 2).sum(dim=(1, 3)), (s1 ** 2).sum(dim=(1, 3))
        out.append((num / den).sqrt().amax(dim=1))
    return torch.stack(out, 1).cpu()


def settle_case(m, img, base, noise, eps, rounds, reps):
    start = (base + eps.view(B, 1, 1, 1) * noise * base.abs().mean()).contiguous()
    with torch.no_grad():
        r = change(m(img, iters=MAX_ITERS, levels=start, return_all=True))
        near = eps <= 1e-3
        tol = float(r[near.cpu(), 2].max()) * 1.001            # the near images stop by step 3
        _, steps = m.settle(img, tol, max_iters=MAX_ITERS, levels=start)
    hist = {int(k): int(c) for k, c in zip(*torch.unique(steps, return_counts=True))}

    def one_pass():
        states, _ = m.settle(img, tol, max_iters=MAX_ITERS, levels=start, return_all=True, differentiable=True)
        return states[7, :, :, -1].square().mean()

    def two_pass():
        with torch.no_grad():
            _, st = m.settle(img, tol, max_iters=MAX_ITERS, levels=start)
        states = m(img, iters=st, levels=start, return_all=True)
        return states[min(7, states.shape[0] - 1), :, :, -1].square().mean()

    with torch.no_grad():
        assert torch.equal(one_pass(), two_pass())          # the same loss, bit for bit
    res = {"tol": tol, "steps": hist, "timing": compare(m, {"one_pass": one_pass, "two_pass": two_pass}, rounds, reps)}
    return res, int(steps.max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("settle_train_probe needs a CUDA device (an H100)")
    dev = torch.device("cuda:0")
    res = {"card": card(), "config": "dim=512 L=6 224/14 batch=32 max_iters=12 bf16",
           "rounds": args.rounds, "reps": args.reps}

    # (c) the random-init bench model: per-image backward against uniform 12 steps
    torch.manual_seed(0)
    m = G.Glom(dim=512, levels=6, image_size=224, patch_size=14).to(dev).train()
    img = torch.randn(B, 3, 224, 224, generator=torch.Generator().manual_seed(1)).to(dev)
    half = torch.tensor([3 if b % 2 == 0 else MAX_ITERS for b in range(B)], dtype=torch.int32, device=dev)
    res["c_backward"] = compare(m, {
        "uniform_12": lambda: m(img, iters=MAX_ITERS, return_all=True)[7, :, :, -1].square().mean(),
        "per_image_half_3_half_12": lambda: m(img, iters=half, return_all=True)[7, :, :, -1].square().mean(),
    }, args.rounds, args.reps)

    # (a), (b): the contracting model
    with torch.no_grad():
        for net in (m.bottom_up, m.top_down):
            net.net[3].weight.zero_()
        base = m(img, iters=60)
        noise = torch.randn(base.shape, generator=torch.Generator().manual_seed(2)).to(dev)
    half_near = torch.tensor([1e-4 if b % 2 == 0 else 3.0 for b in range(B)], device=dev)
    res["a_half_stop_by_3"], _ = settle_case(m, img, base, noise, half_near, args.rounds, args.reps)
    res["b_all_stop_by_3"], t_max = settle_case(m, img, base, noise, torch.full((B,), 1e-4, device=dev), args.rounds,
                                                args.reps)
    tb = res["b_all_stop_by_3"]["timing"]
    res["b_all_stop_by_3"]["frozen_reverse_steps"] = MAX_ITERS - t_max
    res["b_all_stop_by_3"]["ms_per_frozen_reverse_step"] = round(
        (tb["one_pass"]["backward"]["median_ms"] - tb["two_pass"]["backward"]["median_ms"]) / (MAX_ITERS - t_max), 4)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
