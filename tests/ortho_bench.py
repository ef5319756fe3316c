"""Cost of an orthographic frame next to a pinhole frame of the headline scene.

The scene is sfgs.synthetic.city_scene (1M Gaussians, SH degree 3) at 1920x1080.  The pinhole frame is the headline
camera (jax004_camera); the orthographic frame is a nadir view of the scene's centre (sfgs.ortho.nadir_camera) at the
same resolution.  Forward, backward and forward + backward are timed with CUDA events, the two cameras alternating
call by call, and the medians are reported with the card's name, power limit and clocks.

    python tests/ortho_bench.py [--reps 30] [--warmup 5] [--out ortho_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "skyfall-gs_b200"))

from sfgs import rasterizer as R  # noqa: E402
from sfgs import synthetic as S  # noqa: E402
from sfgs.ortho import nadir_camera  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")])) if r.stdout else {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--P", type=int, default=1_000_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ortho_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    W, H = 1920, 1080
    sc = S.city_scene(args.P, seed=0, sh_degree=3)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    means, scales, rots, opac, shs = (t(sc.means3D), t(sc.scales), t(sc.rotations), t(sc.opacities), t(sc.shs))
    e = torch.empty(0, device=dev)
    bg = torch.zeros(3, device=dev)
    pin = S.jax004_camera(W, H)
    res = 512.0 / W                                           # the 512-unit-wide scene across the image
    nad = nadir_camera(-256.0, 256.0, -0.5 * H * res, 0.5 * H * res, res, 200.0)
    cams = {
        "pinhole": (t(pin.viewmatrix), t(pin.projmatrix), pin.tanfovx, pin.tanfovy, t(pin.campos), False),
        "ortho": (nad.viewmatrix.to(dev), nad.projmatrix.to(dev), nad.half_width, nad.half_height,
                  torch.zeros(3, device=dev), True),
    }
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(W, H, seed=1)]

    def fwd(name):
        view, proj, tx, ty, campos, ortho = cams[name]
        return R.rasterize_gaussians(bg, means, e, opac, scales, rots, 1.0, e, e, e, 0, view, proj, tx, ty, 0.1, H, W,
                                     shs, 3, campos, False, False, ortho=ortho)

    def bwd(name, o):
        view, proj, tx, ty, campos, ortho = cams[name]
        return R.rasterize_gaussians_backward(bg, means, o[5], e, scales, rots, e, 1.0, e, e, view, proj, tx, ty, 0.1,
                                              cot[0], cot[1], cot[2], cot[3], e, shs, 3, campos, o[7], o[0], o[8],
                                              o[9], o[4], False, ortho=ortho)

    times = {n: {"fwd": [], "bwd": [], "fwd_bwd": []} for n in cams}
    visible = {}
    for i in range(args.warmup + args.reps):
        for name in (cams if i % 2 == 0 else list(cams)[::-1]):      # alternate which camera goes first
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            torch.cuda.synchronize()
            ev[0].record()
            o = fwd(name)
            ev[1].record()
            bwd(name, o)
            ev[2].record()
            torch.cuda.synchronize()
            visible[name] = (int((o[5] > 0).sum()), int(o[0]))
            if i >= args.warmup:
                times[name]["fwd"].append(ev[0].elapsed_time(ev[1]))
                times[name]["bwd"].append(ev[1].elapsed_time(ev[2]))
                times[name]["fwd_bwd"].append(ev[0].elapsed_time(ev[2]))
    res = {"gpu": gpu_info(), "P": args.P, "W": W, "H": H, "reps": args.reps,
           "visible_and_instances": visible,
           "median_ms": {n: {k: float(np.median(v)) for k, v in d.items()} for n, d in times.items()},
           "spread_ms": {n: {k: [float(np.percentile(v, 10)), float(np.percentile(v, 90))] for k, v in d.items()}
                         for n, d in times.items()}}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
