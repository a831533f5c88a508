"""Per-image step counts (Glom.forward with iters = a (B,) vector) at configs[1] shapes (dim=512 L=6 224/14, batch 32, bf16).

  (a) no-grad forward with every image at 12 steps but one at 11, against forward(iters=12): the cost of the per-image
      path itself (the schedule launches, the SETTLE builds of the step kernels, the final gather);
  (b) no-grad forward with half of the images at 3 steps and half at 12, against forward(iters=12);
  (c) a training step (return_all, loss on slab 7's top level as in bench.py's train step) with the step vector of (b),
      against uniform 12 steps; forward and backward milliseconds separately.

Times are medians of interleaved rounds of CUDA-event-timed calls.  The card's name and power limit are read in the same
run.  Prints one JSON line (and writes it to --out).

    python tools/iters_probe.py [--rounds 5] [--reps 5] [--out /tmp/iters_probe.json]
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

T = 12


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


def summary(v):
    return {"median_ms": round(statistics.median(v), 4), "min_ms": round(min(v), 4), "max_ms": round(max(v), 4)}


def compare(fns, rounds, reps):
    """{name: median ms} of `rounds` interleaved rounds of `reps` calls each."""
    ms = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            ms[k].append(timed(fn, reps))
    return {k: summary(v) for k, v in ms.items()}


def train_times(model, img, iters, reps):
    """(forward ms, backward ms) per training step, averaged over `reps` steps timed with CUDA events."""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    f = b = 0.0
    for _ in range(reps):
        model.zero_grad(set_to_none=True)
        ev[0].record()
        loss = model(img, iters=iters, return_all=True)[7, :, :, -1].square().mean()
        ev[1].record()
        loss.backward()
        ev[2].record()
        torch.cuda.synchronize()
        f += ev[0].elapsed_time(ev[1])
        b += ev[1].elapsed_time(ev[2])
    return f / reps, b / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("iters_probe needs a CUDA device (an H100)")
    dev = torch.device("cuda:0")
    res = {"card": card(), "config": "dim=512 L=6 224/14 batch=32 bf16"}

    torch.manual_seed(0)
    m = G.Glom(dim=512, levels=6, image_size=224, patch_size=14).to(dev).eval()
    img = torch.randn(32, 3, 224, 224, generator=torch.Generator().manual_seed(1)).to(dev)
    one_short = torch.full((32,), T, dtype=torch.int32, device=dev)
    one_short[5] = T - 1
    half = torch.tensor([3 if b % 2 == 0 else T for b in range(32)], dtype=torch.int32, device=dev)
    with torch.no_grad():
        ref = m(img, iters=T)
        out = m(img, iters=one_short)
        assert torch.equal(out[one_short == T], ref[one_short == T])
        res["a_one_image_short"] = compare({"forward_iters12": lambda: m(img, iters=T),
                                            "per_image_12_but_one_11": lambda: m(img, iters=one_short)},
                                           args.rounds, args.reps)
        res["b_half_at_3"] = compare({"forward_iters12": lambda: m(img, iters=T),
                                      "per_image_half_3_half_12": lambda: m(img, iters=half)},
                                     args.rounds, args.reps)
        del ref, out

    m.train()
    train_times(m, img, T, 2)                       # warm-up of both shapes
    train_times(m, img, half, 2)
    runs = {"uniform_12": ([], []), "per_image_half_3_half_12": ([], [])}
    for _ in range(args.rounds):
        for name, iters in (("uniform_12", T), ("per_image_half_3_half_12", half)):
            f, b = train_times(m, img, iters, args.reps)
            runs[name][0].append(f)
            runs[name][1].append(b)
    res["c_train_step"] = {k: {"forward": summary(f), "backward": summary(b)} for k, (f, b) in runs.items()}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
