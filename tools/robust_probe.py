"""API-level robustness checks on a GPU: interleaved models, varying batch, side stream, CUDA-graph capture."""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import glom_pytorch_b200 as G
torch.manual_seed(0)
dev = "cuda:0"
a = G.Glom(dim=256, levels=4, image_size=64, patch_size=8).to(dev).eval()      # n = 64
b = G.Glom(dim=512, levels=6, image_size=224, patch_size=14).to(dev).eval()    # n = 256
ok = True
def same(x, y, what):
    global ok
    e = (x - y).abs().max().item()
    print(f"{what}: max diff {e:.3e}"); ok &= e == 0.0
with torch.no_grad():
    xa = [torch.randn(B, 3, 64, 64, device=dev) for B in (1, 3, 7, 2)]
    xb = [torch.randn(B, 3, 224, 224, device=dev) for B in (2, 1, 5)]
    ra = [a(x, iters=3) for x in xa]; rb = [b(x, iters=2) for x in xb]
    # interleaved, reversed order, repeated: results must be bit-identical (deterministic engine, cached workspaces)
    for i in (3, 0, 2, 1):
        same(a(xa[i], iters=3), ra[i], f"model a batch {xa[i].shape[0]} again")
        if i < 3: same(b(xb[i], iters=2), rb[i], f"model b batch {xb[i].shape[0]} again")
    # side stream
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        y = b(xb[0], iters=2)
    torch.cuda.current_stream().wait_stream(s)
    same(y, rb[0], "side stream")
    # batch subset consistency
    same(a(xa[2][:3], iters=3), ra[2][:3], "batch subset")
    # CUDA graph capture of a forward
    try:
        static_x = xb[2].clone()
        g = torch.cuda.CUDAGraph()
        s2 = torch.cuda.Stream(); s2.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s2):
            b(static_x, iters=2)                    # eager warm-up on a side stream; the capture packs and allocates its own
        torch.cuda.current_stream().wait_stream(s2)
        with torch.cuda.graph(g):
            static_y = b(static_x, iters=2)
        static_x.copy_(xb[2]); g.replay(); torch.cuda.synchronize()
        same(static_y, rb[2], "CUDA graph replay")
    except Exception as e:
        print("CUDA graph capture not supported:", type(e).__name__, str(e)[:200])
torch.cuda.synchronize()
print("ROBUST OK" if ok else "ROBUST MISMATCH")
