"""Glom.settle_video against the per-frame settle loop and the per-frame forward continuation at configs[1] shapes
(dim=512 L=6 224/14, max_iters 12), 32 streams x 16 frames.

A token-sensitive contracting model: both second MLP layers scaled by 0.1 (zeroed, the tokens would have no effect and
every continuing frame would stop after one step).  Every stream starts from init_levels.  Two clips:
  drift:       frame f of stream s is base_s + drift_s * f * noise_s, with drift sizes spread over six decades across
               the streams (in shuffled order), so the same streams are slow at every frame;
  scene_cuts:  drift sizes from 1e-2 down over four decades, and stream s cuts to a new scene at frame 1 + s % 15, so
               the slow frames are the cuts, in a different stream at each frame.
For each clip, tol is the half-decade value whose per-frame settle loop over the first four frames gives frames 1..3 a
mean step count closest to 6.  Arms, in interleaved rounds, each timed with a host clock around work that ends in a
device synchronise (tokeniser included):
  (A) the per-frame loop  lv, st = settle(frames[:, f], tol, 12, levels=lv);
  (B) settle_video(frames, tol, 12, slots=32);
  (C) the per-frame continuation  lv = forward(frames[:, f], iters=12, levels=lv).
Reports frames/s (median, min, max) of each arm, the steps histogram per frame index, sum_f max_s steps (what (A)'s time
follows) and max_s sum_f steps (what (B)'s follows), whether (B) equals (A) bit for bit, and the card's name and power
limit.  Prints one JSON line (and writes it to --out).

    python tools/settle_video_probe.py [--streams 32] [--frames 16] [--rounds 5] [--out /tmp/settle_video_probe.json]
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
SLOTS = 32
SECOND_LAYER_SCALE = 0.1


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, limit = (q.stdout.strip().split(", ") + ["?", "?"])[:2] if q.returncode == 0 else (torch.cuda.get_device_name(0), "?")
    return {"name": name, "power_limit": limit}


def settle_loop(m, frames, tol, levels=None):
    outs, steps, lv = [], [], levels
    for f in range(frames.shape[1]):
        lv, st = m.settle(frames[:, f], tol, max_iters=MAX_ITERS, levels=lv)
        outs.append(lv)
        steps.append(st)
    return torch.stack(outs, 1), torch.stack(steps, 1)


def forward_loop(m, frames):
    outs, lv = [], None
    for f in range(frames.shape[1]):
        lv = m(frames[:, f], iters=MAX_ITERS, levels=lv)
        outs.append(lv)
    return outs


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def make_frames(S, F, cuts):
    """(S, F, 3, 224, 224) on the CPU: base_s + drift_s * f * noise_s, drift_s spread over six decades from 1 (shuffled).
    With `cuts`, the drifts are spread over four decades from 1e-2 instead, and stream s cuts to a new scene (a second
    base) at frame 1 + s % (F - 1)."""
    g = torch.Generator().manual_seed(1)
    base = torch.randn(S, 1, 3, 224, 224, generator=g)
    noise = torch.randn(S, 1, 3, 224, 224, generator=g)
    order = torch.randperm(S, generator=g).double()
    top, decades = (-2, 4) if cuts else (0, 6)
    drift = (10.0 ** (top - decades * order / max(S - 1, 1))).float().view(S, 1, 1, 1, 1)
    frames = base + drift * torch.arange(F, dtype=torch.float32).view(1, F, 1, 1, 1) * noise
    if cuts:
        scene = torch.randn(S, 3, 224, 224, generator=g)
        for s in range(S):
            c = 1 + s % max(F - 1, 1)
            frames[s, c:] += scene[s] - base[s, 0]
    return frames


def measure(m, frames, rounds):
    S, F = frames.shape[:2]
    res = {}
    cands = {}
    for k in range(6, 13):
        _, st = settle_loop(m, frames[:, :4], 10.0 ** (-k / 2))
        cands[10.0 ** (-k / 2)] = float(st[:, 1:].double().mean())
    tol = min(cands, key=lambda t: abs(cands[t] - MAX_ITERS / 2))
    res["tol"] = tol
    res["tol_candidates_mean_steps_frames_1_3"] = {f"{t:.1e}": round(v, 2) for t, v in cands.items()}
    arms = {
        "A_settle_loop": lambda: settle_loop(m, frames, tol),
        "B_settle_video": lambda: m.settle_video(frames, tol, max_iters=MAX_ITERS, slots=SLOTS),
        "C_forward_loop": lambda: forward_loop(m, frames),
    }
    outs = {k: fn() for k, fn in arms.items()}                      # warm-up, and the results compared below
    (la, sa), (lb, sb) = outs["A_settle_loop"], outs["B_settle_video"]
    res["B_equals_A_bitwise"] = bool(torch.equal(la, lb) and torch.equal(sa, sb))
    steps = sa.cpu().numpy()
    res["steps_per_frame"] = [{int(a): int(b) for a, b in zip(*np.unique(steps[:, f], return_counts=True))}
                              for f in range(F)]
    res["mean_steps"] = float(steps.mean())
    res["sum_f_max_s_steps"] = int(steps.max(axis=0).sum())
    res["max_s_sum_f_steps"] = int(steps.sum(axis=1).max())
    del outs, la, lb
    secs = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            t, out = wall(fn)
            del out
            secs[k].append(t)
    res["frames_per_s"] = {k: {"median": round(S * F / statistics.median(v), 1), "min": round(S * F / max(v), 1),
                               "max": round(S * F / min(v), 1)} for k, v in secs.items()}
    res["B_over_A"] = round(statistics.median(secs["A_settle_loop"]) / statistics.median(secs["B_settle_video"]), 3)
    res["B_over_C"] = round(statistics.median(secs["C_forward_loop"]) / statistics.median(secs["B_settle_video"]), 3)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=32)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("settle_video_probe needs a CUDA device (an H100)")
    dev = torch.device("cuda:0")
    S, F = args.streams, args.frames
    res = {"card": card(), "config": f"dim=512 L=6 224/14 streams={S} frames={F} slots={SLOTS} max_iters={MAX_ITERS} "
                                     f"bf16, second MLP layers x{SECOND_LAYER_SCALE}, start init_levels"}

    torch.manual_seed(0)
    m = G.Glom(dim=512, levels=6, image_size=224, patch_size=14).to(dev).eval()
    with torch.no_grad():
        for net in (m.bottom_up, m.top_down):
            net.net[3].weight.mul_(SECOND_LAYER_SCALE)
        for cuts in (False, True):
            res["scene_cuts" if cuts else "drift"] = measure(m, make_frames(S, F, cuts).to(dev), args.rounds)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
