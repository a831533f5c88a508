"""Golden GRADIENT fixtures from the live reference (autograd on CPU, fp32).  Run in the build container:

    python tests/golden/make_golden_grads.py [case ...]      (default: every case)

loss = sum(out * cot) with a seeded cotangent; gradients of every parameter, of the image and (when given) of the
carried-in `levels` are stored."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.environ.get("GLOM_REF_PATH", "/root/reference"))
sys.path.insert(0, HERE)

from glom_pytorch import Glom as RefGlom  # noqa: E402
from oracle.glom_oracle import synth_params  # noqa: E402
from cases import GRAD_CASES, grad_inputs  # noqa: E402


def main():
    torch.set_num_threads(8)
    for name in sys.argv[1:] or GRAD_CASES:
        case = GRAD_CASES[name]
        kw = dict(dim=case["dim"], levels=case["levels"], image_size=case["image_size"], patch_size=case["patch_size"],
                  consensus_self=case.get("consensus_self", False),
                  local_consensus_radius=case.get("local_consensus_radius", 0))
        model = RefGlom(**kw)
        params = synth_params(case["dim"], case["levels"], case["image_size"], case["patch_size"], seed=case["param_seed"])
        model.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=False)
        img, lv, cot = grad_inputs(case)
        img_t = torch.from_numpy(img).requires_grad_(True)
        lv_t = None if lv is None else torch.from_numpy(lv).requires_grad_(True)
        out = model(img_t, iters=case["iters"], levels=lv_t, return_all=case["return_all"])
        loss = (out * torch.from_numpy(cot)).sum()
        loss.backward()
        res = {"out": out.detach().numpy().astype(np.float32), "d_img": img_t.grad.numpy()}
        if lv_t is not None:
            res["d_levels"] = lv_t.grad.numpy()
        for k, p in model.named_parameters():
            res["d_" + k] = p.grad.numpy() if p.grad is not None else np.zeros(tuple(p.shape), np.float32)
        np.savez_compressed(os.path.join(HERE, name + ".npz"), **res)
        print(name, {k: v.shape for k, v in res.items() if k in ("out", "d_img", "d_init_levels")},
              "loss", float(loss))


if __name__ == "__main__":
    main()
