"""Times glom_pytorch_b200.track_islands next to islands() alone, on two inputs of the configs[1] model (dim 512,
6 levels, 224 / 14 -> n 256):
  return_all    forward(iters=12, return_all=True) at batch 32: 13 x 32 slabs of (256, 6, 512) fp32, 1.31 GB, time_dim 0
  settle_video  settle_video of 32 streams x 16 frames (each frame its stream's image shifted by one more pixel,
                tol 1e-3, max_iters 12): 32 x 16 slabs, 1.61 GB, time_dim 1
Device events around `--calls` back-to-back calls, medians over `--rounds`; the two calls are interleaved round by
round.  Writes nothing; the card's name and power limit are printed with the numbers.

Algorithmic bytes (what the call must move at least, each byte once):
  islands  states read (S n L d 4) + cos_right / cos_down / agreement / labels written (16 S L n) + num_islands
  tracks   + labels read (4 S L n) + prev / overlap / next / track written (16 S L n)
The tracking kernels touch int32 per (patch, level), 1/d of the state bytes.

    python tools/track_islands_probe.py [--rounds 5] [--calls 10]
"""
import argparse
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import glom_pytorch_b200 as G  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def timed(fn, calls):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(calls):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / calls


def run(name, states, time_dim, args):
    lead = states.shape[:-3]
    n, L, d = states.shape[-3:]
    S = int(np.prod(lead))
    isl_bytes = S * n * L * d * 4 + 16 * S * L * n + 4 * S * L
    trk_bytes = isl_bytes + 20 * S * L * n
    cases = {"islands": (lambda: G.islands(states), isl_bytes),
             "track_islands": (lambda: G.track_islands(states, time_dim=time_dim), trk_bytes)}
    for fn, _ in cases.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    samples = {k: [] for k in cases}
    for _ in range(args.rounds):
        for k, (fn, _) in cases.items():
            samples[k].append(timed(fn, args.calls))
    t = G.track_islands(states, time_dim=time_dim)
    tr = torch.movedim(t.track, time_dim, 0)
    lab = torch.movedim(t.labels, time_dim, 0)
    roots = lab == torch.arange(n, device=lab.device)
    step = torch.arange(lab.shape[0], device=lab.device).view((-1,) + (1,) * (lab.dim() - 1))
    cont = int((roots & (tr < step * n))[1:].sum())
    born = int((roots & (tr >= step * n))[1:].sum())
    print(f"{name}: states {tuple(states.shape)} fp32, time_dim {time_dim}; islands per (slab, level) median "
          f"{float(t.num_islands.float().median()):.0f}; after the first step {cont} islands continue a track and "
          f"{born} start one")
    for k, (_, nbytes) in cases.items():
        ms = statistics.median(samples[k])
        gbs = nbytes / (ms * 1e-3) / 1e9
        print(f"  {k:14s} median {ms:8.3f} ms/call (min {min(samples[k]):.3f}, max {max(samples[k]):.3f}); "
              f"{nbytes / 1e9:.3f} GB algorithmic -> {gbs:7.1f} GB/s, {gbs * 1e9 / HBM_BYTES_PER_S:.1%} of 3.35 TB/s")
    extra = statistics.median(samples["track_islands"]) - statistics.median(samples["islands"])
    print(f"  tracking kernels ~{extra:.3f} ms ({extra / statistics.median(samples['islands']):.1%} of islands) "
          f"(difference of medians)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=10)
    args = ap.parse_args()
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip()
    except OSError:
        smi = "nvidia-smi unavailable"
    print(f"device: {torch.cuda.get_device_name()} ({smi}), torch {torch.__version__}")
    torch.manual_seed(0)
    m = G.Glom(dim=512, levels=6, image_size=224, patch_size=14).cuda().eval()
    with torch.no_grad():
        states = m(torch.randn(32, 3, 224, 224, device="cuda"), iters=12, return_all=True)
    run("return_all", states, 0, args)
    del states
    base = torch.randn(32, 3, 224, 224, device="cuda")
    frames = torch.stack([torch.roll(base, f, dims=3) for f in range(16)], 1)
    with torch.no_grad():
        video, _ = m.settle_video(frames, 1e-3, max_iters=12)
    del frames
    run("settle_video", video, 1, args)


if __name__ == "__main__":
    main()
