"""Glom.settle at configs[1] shapes (dim=512 L=6 224/14, batch 32, max_iters 12), against forward(iters=12).

  (a) settle(tol=-1): nothing stops, so the difference to the forward is the cost of the stopping rule and the flags;
  (b) a contracting model (both second MLP layers zeroed) started from its fixed point plus noise, with half of the
      images (= half of the 256-row blocks, n = 256) small enough to stop after about 3 steps and the other half never:
      time and the `steps` histogram;
  (c) the `steps` histogram of the randomly initialised bench model at a few tols (for information).

Times are medians of interleaved rounds of CUDA-event-timed calls.  Prints one JSON line (and writes it to --out).

    python tools/settle_probe.py [--rounds 5] [--reps 10] [--out /tmp/settle_probe.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import glom_pytorch_b200 as G  # noqa: E402
from glom_pytorch_b200 import _native  # noqa: E402

MAX_ITERS = 12


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, limit = (q.stdout.strip().split(", ") + ["?", "?"])[:2] if q.returncode == 0 else (torch.cuda.get_device_name(0), "?")
    return {"name": name, "power_limit": limit}


def timed(fn, reps):
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def compare(fns, rounds, reps):
    """{name: median ms} of `rounds` interleaved rounds of `reps` calls each."""
    ms = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            ms[k].append(timed(fn, reps))
    return {k: {"median_ms": round(statistics.median(v), 4), "min_ms": round(min(v), 4), "max_ms": round(max(v), 4)}
            for k, v in ms.items()}


def kernel_ms(fn, reps=5):
    """Per-kernel-kind milliseconds per call (CUDA events around each launch, glom_b200_profile_begin / _end); the
    stopping rule's own launches are not bracketed."""
    fn()
    torch.cuda.synchronize()
    _native.profile_begin()
    for _ in range(reps):
        fn()
    prof = _native.profile_end()
    return {k: round(ms / reps, 4) for k, (ms, n) in prof.items() if n}


def histogram(steps):
    v, c = np.unique(steps.cpu().numpy(), return_counts=True)
    return {int(a): int(b) for a, b in zip(v, c)}


def change(states):
    """r[b, k - 1] = max_l sqrt(sum_i |S_k - S_{k-1}|^2 / sum_i |S_k|^2), float64, from (T+1, B, n, L, d) states."""
    out = []
    for k in range(1, states.shape[0]):
        s1, s0 = states[k].double(), states[k - 1].double()
        num, den = ((s1 - s0) ** 2).sum(dim=(1, 3)), (s1 ** 2).sum(dim=(1, 3))
        out.append((num / den).sqrt().amax(dim=1))
    return torch.stack(out, 1).cpu().numpy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("settle_probe needs a CUDA device (an H100)")
    dev = torch.device("cuda:0")
    res = {"card": card(), "config": "dim=512 L=6 224/14 batch=32 max_iters=12 bf16"}

    torch.manual_seed(0)
    m = G.Glom(dim=512, levels=6, image_size=224, patch_size=14).to(dev).eval()
    img = torch.randn(32, 3, 224, 224, generator=torch.Generator().manual_seed(1)).to(dev)
    with torch.no_grad():
        # (a) nothing stops
        lv, st = m.settle(img, -1.0, max_iters=MAX_ITERS)
        assert torch.equal(lv, m(img, iters=MAX_ITERS)) and bool((st == MAX_ITERS).all())
        res["a_no_stop"] = compare({"forward_iters12": lambda: m(img, iters=MAX_ITERS),
                                    "settle_tol_-1": lambda: m.settle(img, -1.0, max_iters=MAX_ITERS)},
                                   args.rounds, args.reps)
        res["a_kernel_ms"] = {"forward_iters12": kernel_ms(lambda: m(img, iters=MAX_ITERS)),
                              "settle_tol_-1": kernel_ms(lambda: m.settle(img, -1.0, max_iters=MAX_ITERS))}

        # (c) the random-init bench model
        res["c_random_init_steps"] = {str(tol): histogram(m.settle(img, tol, max_iters=MAX_ITERS)[1])
                                      for tol in (1e-1, 3e-2, 1e-2, 3e-3, 1e-3)}
        r = change(m(img, iters=MAX_ITERS, return_all=True))
        res["c_random_init_change_median_by_step"] = [float(f"{x:.4g}") for x in np.median(r, axis=0)]

        # (b) contracting model: even images start 1e-4 away from the fixed point, odd ones far away
        for net in (m.bottom_up, m.top_down):
            net.net[3].weight.zero_()
        base = m(img, iters=60)
        noise = torch.randn(base.shape, generator=torch.Generator().manual_seed(2)).to(dev)
        eps = torch.tensor([1e-4 if b % 2 == 0 else 3.0 for b in range(32)], device=dev).view(32, 1, 1, 1)
        start = (base + eps * noise * base.abs().mean()).contiguous()
        del base, noise
        r = change(m(img, iters=MAX_ITERS, levels=start, return_all=True))
        tol = float(r[0::2, 2].max()) * 1.001          # the near images stop by step 3
        lv, st = m.settle(img, tol, max_iters=MAX_ITERS, levels=start)
        res["b_contracting"] = {
            "tol": tol, "steps": histogram(st),
            "far_images_min_change": float(r[1::2].min()),
            "timing": compare({"forward_iters12": lambda: m(img, iters=MAX_ITERS, levels=start),
                               "settle": lambda: m.settle(img, tol, max_iters=MAX_ITERS, levels=start)},
                              args.rounds, args.reps),
        }
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
