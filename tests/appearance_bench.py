"""The appearance path of render() at 1M Gaussians, fused against the torch formulation — needs a GPU.  Not a pytest file.

    python tests/appearance_bench.py [--P 1000000] [--cases 4:1,16:3] [--repeats 7] [--iters 10]

A case M:D has features [P, M, 3] (M = (max_sh_degree + 1)^2) at active SH degree D.  4:1 is what Skyfall-GS trains
(`--sh_degree 1 --appearance_enabled`), 16:3 the degree-3 model.  Per case, four timings:
  torch_fwd    reference_colors, the reference's statements in torch eager (no autograd graph)
  fused_fwd    fused_appearance_colors (the wgmma kernel, no autograd graph)
  torch_step   the torch formulation's forward + backward to every input a training step updates (features, Fourier
               features, camera embedding, MLP, xyz): what render() and loss.backward() spend on the appearance path
  fused_step   the same with fused_appearance_colors: fused forward, then the backward's torch recompute
Each timing is CUDA events around `--iters` calls after three warm-up calls; the four alternate inside each of
`--repeats` rounds, and the median, min and max over rounds are reported.  One JSON line per case, with the card's
name and power limit on it.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "skyfall-gs_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)
import numpy as np
import torch

from sfgs import appearance as AP


def power_limit_w(index):
    """The card's enforced power limit in watts (read-only NVML or nvidia-smi query), or None."""
    try:
        import pynvml as nv
        nv.nvmlInit()
        try:
            return nv.nvmlDeviceGetEnforcedPowerLimit(nv.nvmlDeviceGetHandleByIndex(index)) / 1000.0
        finally:
            nv.nvmlShutdown()
    except Exception:  # noqa: BLE001
        pass
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:  # noqa: BLE001
        return None


def inputs(P, M, dev):
    """Seeded inputs shaped like a GaussianModel with appearance enabled, and the six MLP tensors."""
    g = torch.Generator(device="cpu").manual_seed(3)
    feats = torch.randn(P, M, 3, generator=g) * 0.3
    feats[:, 0] += 0.6
    gemb = torch.sin(torch.randn(P, 24, generator=g) * 3)
    aemb = torch.randn(32, generator=g) * 0.5
    xyz = torch.randn(P, 3, generator=g) * 80
    campos = torch.tensor([10.0, -300.0, 120.0])
    torch.manual_seed(5)
    lin = [torch.nn.Linear(59, 128), torch.nn.Linear(128, 128), torch.nn.Linear(128, 6)]
    W = [x.detach() for l in lin for x in (l.weight, l.bias)]
    return [t.to(dev) for t in (feats, gemb, aemb, *W, xyz, campos)]


def timer(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def run_case(P, M, D, dev, repeats, iters):
    feats, gemb, aemb, W1, b1, W2, b2, W3, b3, xyz, campos = inputs(P, M, dev)
    W = (W1, b1, W2, b2, W3, b3)
    leaves = [t.clone().requires_grad_(True) for t in (feats, gemb, aemb, *W, xyz)]
    cot = torch.randn((P, 3), generator=torch.Generator(device="cpu").manual_seed(9)).to(dev)

    def torch_fwd():
        with torch.no_grad():
            return AP.reference_colors(feats, gemb, aemb, *W, xyz, campos, D)

    def fused_fwd():
        with torch.no_grad():
            return AP.fused_appearance_colors(feats, gemb, aemb, W, xyz, campos, D)

    def torch_step():
        out = AP.reference_colors(*leaves[:10], campos, D)
        return torch.autograd.grad(out, leaves, cot)

    def fused_step():
        out = AP.fused_appearance_colors(*leaves[:3], tuple(leaves[3:9]), leaves[9], campos, D)
        return torch.autograd.grad(out, leaves, cot)

    fns = {"torch_fwd": torch_fwd, "fused_fwd": fused_fwd, "torch_step": torch_step, "fused_step": fused_step}
    for fn in fns.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize(dev)
    times = {k: [] for k in fns}
    for _ in range(repeats):
        for k, fn in fns.items():
            times[k].append(timer(fn, iters))
    err = float((fused_fwd() - torch_fwd()).abs().max())
    g_err = max(float((a - b).abs().max()) for a, b in zip(fused_step(), torch_step()))
    rec = {"P": P, "M": M, "D": D}
    for k, v in times.items():
        rec[f"{k}_ms"] = round(float(np.median(v)), 4)
        rec[f"{k}_range_ms"] = [round(float(min(v)), 4), round(float(max(v)), 4)]
    rec["fwd_speedup"] = round(rec["torch_fwd_ms"] / rec["fused_fwd_ms"], 1)
    rec["step_saving_ms"] = round(rec["torch_step_ms"] - rec["fused_step_ms"], 4)
    rec["max_abs_diff_fwd"] = err
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
        sys.exit("appearance_bench.py needs a CUDA device")
    dev = torch.device("cuda:0")
    card = {"device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0)}
    for case in a.cases.split(","):
        M, D = (int(x) for x in case.split(":"))
        rec = run_case(a.P, M, D, dev, a.repeats, a.iters)
        print(json.dumps({**card, **rec}), flush=True)


if __name__ == "__main__":
    main()
