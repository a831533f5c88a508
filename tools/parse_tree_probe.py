"""Times glom_pytorch_b200.parse_tree on the configs[1] return_all slabs (dim 512, 6 levels, 224 / 14 -> n 256,
12 iterations, batch 32: 13 x 32 slabs of (256, 6, 512) fp32, 1.31 GB), with and without embeddings, next to islands()
alone.  Device events around `--calls` back-to-back calls, medians over `--rounds`; the three calls are interleaved
round by round.  Writes nothing; the card's name and power limit are printed with the numbers.

Algorithmic bytes (what the call must move at least, each byte once):
  islands     states read (S n L d 4) + cos_right / cos_down / agreement / labels written (16 S L n) + num_islands
  tree        + labels read (4 S L n) + size / parent / containment written (12 S L n) + nested
  embeddings  + states read once more for the sums (S n L d 4) + embedding written (S L n d 4) + member_cos /
              coherence written (8 S L n)
GB/s is those bytes over the median time; the share of peak is against the H100 SXM's 3.35 TB/s HBM3.

    python tools/parse_tree_probe.py [--rounds 5] [--calls 10]
"""
import argparse
import os
import statistics
import subprocess
import sys

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
    T1, B, n, L, d = states.shape
    S = T1 * B
    isl_bytes = S * n * L * d * 4 + 16 * S * L * n + 4 * S * L
    tree_bytes = isl_bytes + 16 * S * L * n + 4 * S * (L - 1)
    emb_bytes = tree_bytes + 2 * S * n * L * d * 4 + 8 * S * L * n
    cases = {"islands": (lambda: G.islands(states), isl_bytes),
             "parse_tree": (lambda: G.parse_tree(states), tree_bytes),
             "parse_tree embeddings": (lambda: G.parse_tree(states, embeddings=True), emb_bytes)}
    for fn, _ in cases.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    samples = {k: [] for k in cases}
    for _ in range(args.rounds):
        for k, (fn, _) in cases.items():
            samples[k].append(timed(fn, args.calls))
    t = G.parse_tree(states)
    print(f"states {tuple(states.shape)} fp32; islands per (slab, level): median "
          f"{float(t.num_islands.float().median()):.0f}, max {int(t.num_islands.max())}; nested mean "
          f"{float(t.nested.mean()):.3f}")
    for k, (_, nbytes) in cases.items():
        ms = statistics.median(samples[k])
        gbs = nbytes / (ms * 1e-3) / 1e9
        print(f"{k:22s} median {ms:8.3f} ms/call (min {min(samples[k]):.3f}, max {max(samples[k]):.3f}); "
              f"{nbytes / 1e9:.3f} GB algorithmic -> {gbs:7.1f} GB/s, {gbs * 1e9 / HBM_BYTES_PER_S:.1%} of 3.35 TB/s")
    tree_ms = statistics.median(samples["parse_tree"]) - statistics.median(samples["islands"])
    emb_ms = statistics.median(samples["parse_tree embeddings"]) - statistics.median(samples["parse_tree"])
    print(f"tree kernel ~{tree_ms:.3f} ms, embedding kernel ~{emb_ms:.3f} ms "
          f"({(emb_bytes - tree_bytes) / (emb_ms * 1e-3) / 1e9:.1f} GB/s on its own bytes) (differences of medians)")


if __name__ == "__main__":
    main()
