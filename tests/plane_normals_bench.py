"""Cost of plane normals: the rasterizer forward + backward with `ray_depth=True`, with and without
`plane_normals=True`, on the headline frame (1M Gaussians, 1920x1080, SH degree 3), alternated call by call, medians of
30 of each (CUDA events around each call), for the default and the deterministic backward; then the preprocess and
per-Gaussian adjoint stage times of each arm from the library's stage profiler (a separate pass: the profiler records
events around every stage).  The card's name, power limit and SM clock are read in the same run.

    python tests/plane_normals_bench.py [--reps 30]
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
from sfgs import native as N  # noqa: E402
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

    def fwd(pn):
        return R.rasterize_gaussians(bg, d["means3D"], e, d["opacities"], d["scales"], d["rotations"], 1.0, e, e, e, 0,
                                     d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, 0.1, H, W, d["shs"],
                                     D, d["campos"], False, False, fuse_normalize=True, ray_depth=True,
                                     plane_normals=pn)

    def bwd(f, pn, det):
        with Hh.deterministic(det):
            return R.rasterize_gaussians_backward(bg, d["means3D"], f[5], e, d["scales"], d["rotations"], e, 1.0, e,
                                                  e, d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, 0.1,
                                                  cot[0], cot[1], cot[2], cot[3], e, d["shs"], D, d["campos"], f[7],
                                                  f[0], f[8], f[9], f[4], False, norm_raw=f[10], ray_depth=True,
                                                  plane_normals=pn)

    def timed(fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        b.synchronize()
        return a.elapsed_time(b), out

    print(f"card: {card()}")
    arms = [(pn, det) for det in (False, True) for pn in (False, True)]
    times = {(k, arm): [] for k in ("fwd", "bwd") for arm in arms}
    for _ in range(3):                                  # warm-up of every arm
        for pn, det in arms:
            bwd(fwd(pn), pn, det)
    torch.cuda.synchronize()
    for _ in range(args.reps):
        for arm in arms:
            t, f = timed(lambda: fwd(arm[0]))
            times[("fwd", arm)].append(t)
            t, _ = timed(lambda: bwd(f, *arm))
            times[("bwd", arm)].append(t)
    med = {k: float(np.median(v)) for k, v in times.items()}
    print(f"\nheadline frame: 1M Gaussians, {W}x{H}, SH degree 3, ray_depth=True, medians of {args.reps} alternated "
          "calls (ms)")
    print("| stage | ray depth | + plane_normals | difference |")
    print("|---|---|---|---|")
    rows = [("forward", med[("fwd", (False, False))], med[("fwd", (True, False))]),
            ("default backward", med[("bwd", (False, False))], med[("bwd", (True, False))]),
            ("deterministic backward", med[("bwd", (False, True))], med[("bwd", (True, True))]),
            ("forward + default backward", med[("fwd", (False, False))] + med[("bwd", (False, False))],
             med[("fwd", (True, False))] + med[("bwd", (True, False))])]
    for k, a, b in rows:
        print(f"| {k} | {a:.3f} | {b:.3f} | {b - a:+.3f} ({100 * (b - a) / a:+.1f} %) |")

    # stage times: the profiler's per-stage event pairs, each arm in turn, one stage profile per arm
    stage = {}
    for pn in (False, True):
        stage[pn] = {k: [] for k in ("preprocess", "gauss_bwd")}
        for _ in range(args.reps):
            N.profile_enable(True)
            bwd(fwd(pn), pn, False)
            torch.cuda.synchronize()
            prof = N.profile_read()
            N.profile_enable(False)
            for k in stage[pn]:
                ms, n = prof[k]
                stage[pn][k].append(ms / max(n, 1))
    print(f"\nstage medians of {args.reps} profiled calls (ms)")
    print("| stage | ray depth | + plane_normals | difference |")
    print("|---|---|---|---|")
    for k in ("preprocess", "gauss_bwd"):
        a, b = float(np.median(stage[False][k])), float(np.median(stage[True][k]))
        print(f"| {k} | {a:.3f} | {b:.3f} | {b - a:+.3f} ({100 * (b - a) / a:+.1f} %) |")


if __name__ == "__main__":
    main()
