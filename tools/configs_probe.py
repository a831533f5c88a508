"""Device-time the other configs on one GPU (informative; bench.py's line is configs[1])."""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import glom_pytorch_b200 as G

def timeit(fn, reps=5, warm=2):
    for _ in range(warm): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps

torch.manual_seed(0)
with torch.no_grad():
    # configs[3] per GPU: dim=1024 L=8 384/16 iters=16, batch 64 over 8 GPUs = 8 per GPU
    m = G.Glom(dim=1024, levels=8, image_size=384, patch_size=16).cuda().eval()
    img = torch.randn(8, 3, 384, 384, device="cuda")
    ms = timeit(lambda: m(img, iters=16))
    ci = 8 * 576 * 8 * 16
    fl = (16 * 1024 ** 2 * 15 / 8 + 4 * 576 * 1024) * ci
    print(f"configs[3] per GPU (d=1024 L=8 N=576 B=8 iters=16): {ms:.3f} ms -> {ci / ms * 1e3:.4g} col-iters/s, {fl / ms / 1e9:.0f} TFLOP/s")
    del m
    # configs[4]: 3-frame continuation 12 -> 10 -> 6 iterations, batch 32
    m = G.Glom(dim=512, levels=6, image_size=224, patch_size=14).cuda().eval()
    imgs = [torch.randn(32, 3, 224, 224, device="cuda") for _ in range(3)]
    def video():
        l1 = m(imgs[0], iters=12); l2 = m(imgs[1], levels=l1, iters=10); return m(imgs[2], levels=l2, iters=6)
    ms = timeit(video)
    ci = 32 * 256 * 6 * 28
    print(f"configs[4] (3-frame continuation 12->10->6, B=32): {ms:.3f} ms -> {ci / ms * 1e3:.4g} col-iters/s")
    # configs[1] with return_all
    ms = timeit(lambda: m(imgs[0], iters=12, return_all=True))
    print(f"configs[1] return_all=True: {ms:.3f} ms")
    # large batch on one GPU (configs[2] total batch on one device)
    big = torch.randn(256, 3, 224, 224, device="cuda")
    ms = timeit(lambda: m(big, iters=12), reps=2, warm=1)
    print(f"B=256 on one GPU: {ms:.3f} ms -> {256 * 256 * 6 * 12 / ms * 1e3:.4g} col-iters/s")
