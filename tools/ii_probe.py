"""Time a forward from init_levels against the same forward from a carried state, and count the FLOPs each executes.

    python tools/ii_probe.py [--batch 32] [--iters 12] [--rounds 5] [--calls 10]

configs[1] shapes (dim 512, L 6, 224/14), bf16.  Arm "init" is ``forward(img, iters)``: its steps t < L run the work
whose inputs are the same in every image for the representative rows only (DESIGN.md, "Image-independent levels").
Arm "carried" is ``forward(img, iters, levels=<init_levels broadcast>)``: the same start and the same bits, but a carried
state always takes the full path, so it is the control.  Medians of interleaved rounds, CUDA events.  The executed
FLOPs are counted from the schedules (K1 / K2 tiles, K3 items) as the engine deals them; ``bench.py``'s roofline counts
the algorithmic FLOPs of the full path.
"""
import argparse
import math
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def executed_flops(d, L, n, B, iters, reduced):
    """(K1, K3, K2) FLOPs of one call, from the tile / item counts of step_bf16's launches."""
    rows, G = B * n, 2 * L - 1
    num_m = (rows + 255) // 256
    nrep = (n // math.gcd(n, 128) * 128 + 255) // 256
    bn2 = 256 if d % 256 == 0 else 128 if d % 128 == 0 else 64
    ntiles = (n + 127) // 128
    keys = (n + 15) // 16 * 16
    k1 = k2 = k3 = 0
    for t in range(iters):
        red = reduced and t < L
        for z in range(0 if t == 0 else 1, G):
            full = not red or (z <= 2 * t - 3 if z % 2 else z <= 2 * t)
            k1 += (num_m if full else nrep) * (4 * d // 256) * 2 * 256 * 256 * d
        for l in range(L):
            full = not red or l <= t
            kdim = 4 * d if l == L - 1 else 8 * d
            k2 += (num_m if full else nrep) * (d // bn2) * 2 * 256 * bn2 * kdim
            items = B * ntiles if (not red or l <= t - 1) else ntiles
            k3 += items * 2 * 2 * 128 * keys * d          # S = Q K^T and O = P V
    return k1, k3, k2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=12)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=10)
    args = ap.parse_args()
    import torch
    import glom_pytorch_b200 as G

    d, L, isz, p = 512, 6, 224, 14
    n = (isz // p) ** 2
    B, T = args.batch, args.iters
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip()
    except OSError:
        smi = "nvidia-smi unavailable"
    print(f"device: {torch.cuda.get_device_name(0)} ({smi})")
    torch.manual_seed(0)
    m = G.Glom(dim=d, levels=L, image_size=isz, patch_size=p, precision="bf16").cuda().eval()
    img = torch.randn(B, 3, isz, isz, device="cuda")
    carried = m.init_levels.detach().float().expand(B, n, L, d).clone()

    def init():
        return m(img, iters=T)

    def carry():
        return m(img, iters=T, levels=carried)

    with torch.no_grad():
        a, b = init(), carry()
        torch.cuda.synchronize()
        print(f"bit-identical: {torch.equal(a, b)}")
        times = {"init": [], "carried": []}
        for _ in range(args.rounds):
            for name, fn in (("init", init), ("carried", carry)):
                for _ in range(2):
                    fn()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.calls):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1) / args.calls)
    for name, reduced in (("init", True), ("carried", False)):
        eligible = reduced and T >= L + 1 and (n // math.gcd(n, 128) * 128 + 255) // 256 < (B * n + 255) // 256
        k1, k3, k2 = executed_flops(d, L, n, B, T, eligible)
        ts = times[name]
        print(f"{name:8s} median {statistics.median(ts):.3f} ms (min {min(ts):.3f}, max {max(ts):.3f})  "
              f"executed GFLOP per call: K1 {k1 / 1e9:.1f}  K3 {k3 / 1e9:.1f}  K2 {k2 / 1e9:.1f}  "
              f"total {(k1 + k2 + k3) / 1e9:.1f}  -> {(k1 + k2 + k3) / (statistics.median(ts) * 1e-3) / 1e12:.0f} TFLOP/s")


if __name__ == "__main__":
    main()
