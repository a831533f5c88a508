"""Cost and effect of the deterministic backward (torch.use_deterministic_algorithms), on bench.py's training step.

configs[1] (dim 512, 6 levels, 224/14 = 256 patches), batch 32, forward(iters=12, return_all=True), loss =
mean(all_levels[7, :, :, -1] ** 2), as in bench.py.  Rounds alternate flag off / flag on; each round times --reps
training steps with CUDA events (forward and backward separately).  Reports the median forward and backward ms of
each mode, the elements that differ per gradient between two flag-off steps on the same input, and whether two flag-on
steps gave the same bits.  The card's name and power limit are read in the same run.  Prints one JSON line (and writes it
to --out).

    python tools/deterministic_probe.py [--rounds 6] [--reps 5] [--out /tmp/deterministic_probe.json]
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

DEV = "cuda:0"


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, limit = (q.stdout.strip().split(", ") + ["?", "?"])[:2] if q.returncode == 0 else (torch.cuda.get_device_name(0), "?")
    return {"name": name, "power_limit": limit}


def step(model, img, ev):
    model.zero_grad(set_to_none=True)
    ev[0].record()
    loss = model(img, iters=12, return_all=True)[7, :, :, -1].square().mean()
    ev[1].record()
    loss.backward()
    ev[2].record()


def grads(model):
    return {k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.manual_seed(0)
    model = G.Glom(dim=512, levels=6, image_size=224, patch_size=14).to(DEV).train()
    img = torch.randn(32, 3, 224, 224, generator=torch.Generator().manual_seed(1)).to(DEV).requires_grad_(True)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    times = {False: {"forward_ms": [], "backward_ms": []}, True: {"forward_ms": [], "backward_ms": []}}
    runs = {False: [], True: []}
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        for mode in (False, True):                                  # warm-up: workspaces, packing, first launches
            torch.use_deterministic_algorithms(mode)
            for _ in range(2):
                step(model, img, ev)
        torch.cuda.synchronize()
        for r in range(args.rounds):
            for mode in ((False, True) if r % 2 == 0 else (True, False)):
                torch.use_deterministic_algorithms(mode)
                for i in range(args.reps):
                    img.grad = None
                    step(model, img, ev)
                    torch.cuda.synchronize()
                    times[mode]["forward_ms"].append(ev[0].elapsed_time(ev[1]))
                    times[mode]["backward_ms"].append(ev[1].elapsed_time(ev[2]))
                    if len(runs[mode]) < 2:
                        g = grads(model)
                        g["d_img"] = img.grad.detach().clone()
                        runs[mode].append(g)
    finally:
        torch.use_deterministic_algorithms(prev)
    a, b = runs[False]
    differ = {k: int((a[k] != b[k]).sum()) for k in a}
    same_on = all(torch.equal(runs[True][0][k], runs[True][1][k]) for k in runs[True][0])
    res = {"card": card(), "config": "configs[1] dim=512 L=6 224/14 batch=32 iters=12 return_all, loss slab 7 top level",
           "rounds": args.rounds, "reps": args.reps}
    for mode, tag in ((False, "default"), (True, "deterministic")):
        res[tag] = {k: round(statistics.median(v), 3) for k, v in times[mode].items()}
    res["backward_cost_pct"] = round(100 * (res["deterministic"]["backward_ms"] / res["default"]["backward_ms"] - 1), 2)
    res["default_elements_differing_between_two_runs"] = differ
    res["deterministic_runs_bit_identical"] = same_on
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
