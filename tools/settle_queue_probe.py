"""Glom.settle_queue against batch-by-batch settle and forward at configs[1] shapes (dim=512 L=6 224/14, max_iters 12).

A contracting model (both second MLP layers zeroed) started from its fixed point plus noise whose size is spread over
six decades across 1024 images (in shuffled order), so that the images stop after anywhere from 1 to 12 steps.  Arms, in
interleaved rounds, each timed with a host clock around work that ends in a device synchronise (tokeniser included):
  (A) settle over consecutive 32-image batches;
  (B) settle_queue(slots=32) over all 1024 images;
  (C) forward(iters=12) over consecutive 32-image batches.
Reports the median images/s of each arm, the `steps` histogram, the card's name and power limit, and whether (B) equals
(A) bit for bit.  Prints one JSON line (and writes it to --out).

    python tools/settle_queue_probe.py [--images 1024] [--rounds 3] [--out /tmp/settle_queue_probe.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import glom_pytorch_b200 as G  # noqa: E402

MAX_ITERS = 12
BATCH = 32


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, limit = (q.stdout.strip().split(", ") + ["?", "?"])[:2] if q.returncode == 0 else (torch.cuda.get_device_name(0), "?")
    return {"name": name, "power_limit": limit}


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


def batched(fn, img, start):
    """fn over consecutive BATCH-image slices; results concatenated (tuples element-wise)."""
    parts = [fn(img[i:i + BATCH], start[i:i + BATCH]) for i in range(0, img.shape[0], BATCH)]
    if isinstance(parts[0], tuple):
        return tuple(torch.cat(p) for p in zip(*parts))
    return torch.cat(parts)


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("settle_queue_probe needs a CUDA device (an H100)")
    dev = torch.device("cuda:0")
    N = args.images
    res = {"card": card(), "config": f"dim=512 L=6 224/14 images={N} batch/slots={BATCH} max_iters={MAX_ITERS} bf16, "
                                     "contracting model"}

    torch.manual_seed(0)
    m = G.Glom(dim=512, levels=6, image_size=224, patch_size=14).to(dev).eval()
    img = torch.randn(N, 3, 224, 224, generator=torch.Generator().manual_seed(1)).to(dev)
    with torch.no_grad():
        for net in (m.bottom_up, m.top_down):
            net.net[3].weight.zero_()
        base = batched(lambda x, _: m(x, iters=60), img, img)
        noise = torch.randn(base.shape, generator=torch.Generator().manual_seed(2)).to(dev)
        order = torch.randperm(N, generator=torch.Generator().manual_seed(3))
        eps = (10.0 ** (1 - 6 * order.double() / (N - 1))).float().to(dev).view(N, 1, 1, 1)
        start = (base + eps * noise * base.abs().mean()).contiguous()
        del base, noise
        # tol: about half of a sample of images has stopped by step 6
        r = change(m(img[:BATCH], iters=MAX_ITERS, levels=start[:BATCH], return_all=True))
        tol = float(np.median(r[:, 5]))
        res["tol"] = tol

        arms = {
            "A_settle_batches": lambda: batched(lambda x, s: m.settle(x, tol, max_iters=MAX_ITERS, levels=s), img, start),
            "B_settle_queue": lambda: m.settle_queue(img, tol, max_iters=MAX_ITERS, levels=start, slots=BATCH),
            "C_forward_batches": lambda: batched(lambda x, s: m(x, iters=MAX_ITERS, levels=s), img, start),
        }
        outs = {k: fn() for k, fn in arms.items()}                  # warm-up, and the results compared below
        (la, sa), (lb, sb) = outs["A_settle_batches"], outs["B_settle_queue"]
        res["B_equals_A_bitwise"] = bool(torch.equal(la, lb) and torch.equal(sa, sb))
        res["steps"] = histogram(sa)
        res["mean_steps"] = float(sa.double().mean())
        del outs, la, lb
        secs = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, fn in arms.items():
                t, out = wall(fn)
                del out
                secs[k].append(t)
        res["images_per_s"] = {k: {"median": round(N / statistics.median(v), 1), "min": round(N / max(v), 1),
                                   "max": round(N / min(v), 1)} for k, v in secs.items()}
        res["B_over_A"] = round(statistics.median(secs["A_settle_batches"]) / statistics.median(secs["B_settle_queue"]), 3)
        res["B_over_C"] = round(statistics.median(secs["C_forward_batches"]) / statistics.median(secs["B_settle_queue"]), 3)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
