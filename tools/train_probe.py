"""Training-step timing at configs[1] shapes (forward on tensor cores + fp32 CUDA-core backward)."""
import os, sys, time
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import glom_pytorch_b200 as G
B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
torch.manual_seed(0)
m = G.Glom(dim=512, levels=6, image_size=224, patch_size=14).cuda()
img = torch.randn(B, 3, 224, 224, device="cuda")
for rep in range(2):
    torch.cuda.synchronize(); t0 = time.time()
    out = m(img, iters=12, return_all=True)
    loss = out[7, :, :, -1].square().mean()
    torch.cuda.synchronize(); t1 = time.time()
    loss.backward()
    torch.cuda.synchronize(); t2 = time.time()
    print(f"B={B} fwd {1e3*(t1-t0):.1f} ms  bwd {1e3*(t2-t1):.1f} ms  loss {loss.item():.4f}  "
          f"|d init_levels| {m.init_levels.grad.norm().item():.3e}  mem {torch.cuda.max_memory_allocated()/2**30:.2f} GiB")
    m.zero_grad()
