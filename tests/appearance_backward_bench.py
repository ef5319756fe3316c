"""A training step of the appearance path at 1M Gaussians with the fused float32 backward — needs a GPU.  Not a
pytest file.

    python tests/appearance_backward_bench.py [--P 1000000] [--cases 4:1,16:3] [--repeats 7] [--iters 10]

Per case M:D (tests/appearance_bench.py's inputs and timing), three timings of forward + backward to every input a
training step updates (features, Fourier features, camera embedding, MLP, xyz):
  torch_step        the torch formulation (reference_colors) and autograd
  fused_step        fused_appearance_colors with the default backward (the torch recompute)
  fused_bwd_step    fused_appearance_colors(..., fused_backward=True)
plus the fused backward kernel alone (`bwd_kernel`), the largest |fused_bwd_step - torch_step| over the gradients,
and the card's name and power limit.  One JSON line per case.
"""
import argparse
import importlib.util
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, os.path.join(ROOT, "skyfall-gs_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)
import numpy as np
import torch

from sfgs import appearance as AP

_spec = importlib.util.spec_from_file_location("appearance_bench", os.path.join(HERE, "appearance_bench.py"))
B = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(B)


def run_case(P, M, D, dev, repeats, iters):
    feats, gemb, aemb, W1, b1, W2, b2, W3, b3, xyz, campos = B.inputs(P, M, dev)
    leaves = [t.clone().requires_grad_(True) for t in (feats, gemb, aemb, W1, b1, W2, b2, W3, b3, xyz)]
    cot = torch.randn((P, 3), generator=torch.Generator(device="cpu").manual_seed(9)).to(dev)
    saved = [t.detach() for t in leaves] + [campos]
    needs = [True] * 10 + [False]

    def torch_step():
        return torch.autograd.grad(AP.reference_colors(*leaves, campos, D), leaves, cot)

    def fused_step():
        return torch.autograd.grad(AP.fused_appearance_colors(*leaves[:3], tuple(leaves[3:9]), leaves[9], campos, D),
                                   leaves, cot)

    def fused_bwd_step():
        out = AP.fused_appearance_colors(*leaves[:3], tuple(leaves[3:9]), leaves[9], campos, D, fused_backward=True)
        return torch.autograd.grad(out, leaves, cot)

    def bwd_kernel():
        return AP._bwd(saved, D, cot, needs)

    fns = {"torch_step": torch_step, "fused_step": fused_step, "fused_bwd_step": fused_bwd_step, "bwd_kernel": bwd_kernel}
    for fn in fns.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize(dev)
    times = {k: [] for k in fns}
    for _ in range(repeats):
        for k, fn in fns.items():
            times[k].append(B.timer(fn, iters))
    g_err = max(float((a - b).abs().max()) for a, b in zip(fused_bwd_step(), torch_step()))
    rec = {"P": P, "M": M, "D": D}
    for k, v in times.items():
        rec[f"{k}_ms"] = round(float(np.median(v)), 4)
        rec[f"{k}_range_ms"] = [round(float(min(v)), 4), round(float(max(v)), 4)]
    rec["fused_bwd_step_over_torch_step"] = round(rec["fused_bwd_step_ms"] / rec["torch_step_ms"], 3)
    rec["max_abs_diff_grads"] = g_err
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=1_000_000)
    ap.add_argument("--cases", default="4:1,16:3", help="comma-separated M:D pairs")
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("appearance_backward_bench.py needs a CUDA device")
    dev = torch.device("cuda:0")
    card = {"device": torch.cuda.get_device_name(dev), "power_limit_w": B.power_limit_w(0)}
    for case in a.cases.split(","):
        M, D = (int(x) for x in case.split(":"))
        print(json.dumps({**card, **run_case(a.P, M, D, dev, a.repeats, a.iters)}), flush=True)


if __name__ == "__main__":
    main()
