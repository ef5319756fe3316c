"""Cost of the depth distortion on the headline frame (1M Gaussians, 1920x1080, SH degree 3): the rasterizer forward
and backward with and without `depth_distortion=True`, for the default and the deterministic backward, alternated call
by call, medians of 30 of each, CUDA events around each call.  The card's name, power limit and SM clock are read in
the same run.

    python tests/depth_distortion_bench.py [--reps 30]
"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "skyfall-gs_b200"), os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)

import helpers as Hh  # noqa: E402
from sfgs import rasterizer as R  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    _, cam, D, d, _ = Hh.frame("jax004", dev)
    W, H = cam.width, cam.height
    bg = torch.zeros(3, device=dev)
    e = torch.empty(0, device=dev)
    g = torch.Generator(device=dev).manual_seed(0)
    cot = (torch.randn((3, H, W), generator=g, device=dev), torch.randn((1, H, W), generator=g, device=dev) * 0.1,
           torch.randn((3, H, W), generator=g, device=dev), torch.randn((1, H, W), generator=g, device=dev))
    g_r = torch.randn((1, H, W), generator=g, device=dev)

    def fwd(dist):
        return R.rasterize_gaussians(bg, d["means3D"], e, d["opacities"], d["scales"], d["rotations"], 1.0, e, e, e, 0,
                                     d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, 0.1, H, W, d["shs"],
                                     D, d["campos"], False, False, fuse_normalize=True, depth_distortion=dist)

    def bwd(f, dist, det):
        kw = dict(distortion_state=f[12], dL_dout_distortion=g_r) if dist else {}
        with Hh.deterministic(det):
            return R.rasterize_gaussians_backward(bg, d["means3D"], f[5], e, d["scales"], d["rotations"], e, 1.0, e,
                                                  e, d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, 0.1,
                                                  cot[0], cot[1], cot[2], cot[3], e, d["shs"], D, d["campos"], f[7],
                                                  f[0], f[8], f[9], f[4], False, norm_raw=f[10], **kw)

    def timed(fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        b.synchronize()
        return a.elapsed_time(b), out

    arms = [(dist, det) for det in (False, True) for dist in (False, True)]
    times = {(k, arm): [] for k in ("fwd", "bwd") for arm in arms}
    for _ in range(3):                                  # warm-up of every arm
        for dist, det in arms:
            bwd(fwd(dist), dist, det)
    torch.cuda.synchronize()
    for _ in range(args.reps):
        for arm in arms:
            t, f = timed(lambda: fwd(arm[0]))
            times[("fwd", arm)].append(t)
            t, _ = timed(lambda: bwd(f, *arm))
            times[("bwd", arm)].append(t)
    med = {k: float(np.median(v)) for k, v in times.items()}
    print(f"card: {card()}")
    print(f"1M Gaussians, {W}x{H}, SH degree 3, medians of {args.reps} alternated calls (ms)")
    print("| backward | stage | without | depth_distortion=True | difference |")
    print("|---|---|---|---|---|")
    for det in (False, True):
        name = "deterministic" if det else "default"
        rows = [(k, med[(k, (False, det))], med[(k, (True, det))]) for k in ("fwd", "bwd")]
        rows.append(("fwd + bwd", rows[0][1] + rows[1][1], rows[0][2] + rows[1][2]))
        for k, a, b in rows:
            print(f"| {name} | {k} | {a:.3f} | {b:.3f} | {b - a:+.3f} ({100 * (b - a) / a:+.1f} %) |")

    # where the difference goes: device time per kernel (torch.profiler, a run of its own), per forward + backward
    from torch.profiler import ProfilerActivity, profile
    n = 10
    rows = {}
    for dist in (False, True):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(n):
                bwd(fwd(dist), dist, False)
            torch.cuda.synchronize()
        for ev in prof.key_averages():
            us = getattr(ev, "device_time_total", None)
            if us is None:
                us = ev.cuda_time_total
            if us > 0:
                rows.setdefault(ev.key, {})[dist] = us / n / 1000.0
    print(f"\ndevice time per forward + default backward, torch.profiler over {n} calls of each arm (ms)")
    print("| kernel | without | depth_distortion=True |")
    print("|---|---|---|")
    tot = {False: 0.0, True: 0.0}
    for k, v in sorted(rows.items(), key=lambda kv: -max(kv[1].values())):
        for q in tot:
            tot[q] += v.get(q, 0.0)
        if max(v.values()) >= 0.005:
            name = k.replace("void ", "").replace("(anonymous namespace)::", "")
            name = name.split(">(")[0] + ">" if ">(" in name else name.split("(")[0]
            print(f"| `{name}` | {v.get(False, 0.0):.4f} | {v.get(True, 0.0):.4f} |")
    print(f"| all device work | {tot[False]:.4f} | {tot[True]:.4f} |")

if __name__ == "__main__":
    main()
