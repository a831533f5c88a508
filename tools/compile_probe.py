"""Eager vs torch.compile vs torch.compile(mode="reduce-overhead") at configs[1] shapes (dim 512, 6 levels, 224 / 14,
iters 12): an inference forward at batch 1 and batch 32, and a training step at batch 32 (forward with return_all and
the bench loss, compiled or not; backward and an SGD step, both inside the timed step).  Wall time per call,
synchronised, with the modes interleaved round by round; medians and spread over --rounds.  Writes nothing; the card's
name and power limit are printed with the numbers.

    python tools/compile_probe.py [--rounds 5] [--calls 20]
"""
import argparse
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import glom_pytorch_b200 as G  # noqa: E402


def timed(fn, calls):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(calls):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / calls * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    args = ap.parse_args()
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip()
    except OSError:
        smi = "nvidia-smi unavailable"
    print(f"device: {torch.cuda.get_device_name()} ({smi}), torch {torch.__version__}")
    torch.manual_seed(0)
    model = G.Glom(dim=512, levels=6, image_size=224, patch_size=14).cuda()

    def forward_case(batch):
        img = torch.randn(batch, 3, 224, 224, device="cuda")
        m = model.eval()
        modes = {"eager": m, "compile": torch.compile(m, fullgraph=True),
                 "reduce-overhead": torch.compile(m, fullgraph=True, mode="reduce-overhead")}
        fns = {k: (lambda f=f: f(img, iters=12)) for k, f in modes.items()}
        return fns

    def train_case(batch):
        img = torch.randn(batch, 3, 224, 224, device="cuda")
        m = model.train()
        opt = torch.optim.SGD(m.parameters(), lr=1e-4)

        def loss(mm, x):
            return mm(x, iters=12, return_all=True)[7, :, :, -1].square().mean()
        compiled = torch.compile(loss, fullgraph=True)

        def step(f):
            opt.zero_grad(set_to_none=True)
            f(m, img).backward()
            opt.step()
        return {"eager": lambda: step(loss), "compile": lambda: step(compiled)}

    cases = {"forward B=1": lambda: forward_case(1), "forward B=32": lambda: forward_case(32),
             "train step B=32": lambda: train_case(32)}
    for name, make in cases.items():
        with torch.set_grad_enabled(name.startswith("train")):
            fns = make()
            for fn in fns.values():                 # compile and warm up every mode first
                for _ in range(3):
                    fn()
            samples = {k: [] for k in fns}
            for _ in range(args.rounds):
                for k, fn in fns.items():
                    samples[k].append(timed(fn, args.calls))
        for k, v in samples.items():
            print(f"{name:16s} {k:16s} median {statistics.median(v):8.3f} ms/call  "
                  f"(min {min(v):.3f}, max {max(v):.3f}, {args.rounds} rounds x {args.calls} calls)")
        torch._dynamo.reset()


if __name__ == "__main__":
    main()
