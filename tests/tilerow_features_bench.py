"""Cost of subpixel offsets and camera / focal gradients in the tile-row sharded mode, on one GPU — needs a GPU.
Not a pytest file.

    python tests/tilerow_features_bench.py [--repeats 7] [--iters 10]

Frame: bench.py's headline frame, 1M Gaussians (city scene, seed 0, SH degree 3), 1920x1080, its cotangents
(S.cotangents(W, H, seed=1)), split into 2 tile-row bands by `partition_rows` on the frame's per-row instance
histogram, with the Gaussians cut into the 2 slices of `gaussian_slices`.  One step is what both ranks of a 2-GPU
sharded frame run, one after the other on this GPU: each band's forward, each band's phase-1 blend adjoint into one
[P,16] buffer, and each slice's phase-2 per-Gaussian adjoint.  No exchange is timed: there is one GPU.
Four arms, timed alternately in one process: without offsets, with U(-0.5, 0.5) offsets, and with offsets plus the
35 (pose) or 37 (pose and focal) camera partials of phase 2.  CUDA events around `--iters` steps, `--repeats` rounds,
median / min / max over rounds.  One JSON line, with the card's name and power limit.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "skyfall-gs_b200"), os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)
import numpy as np
import torch

import helpers as Hh
from appearance_bench import power_limit_w
from sfgs import multigpu as MG
from sfgs import rasterizer as R
from sfgs import synthetic as S


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("tilerow_features_bench.py needs a CUDA device")
    dev = torch.device("cuda:0")
    P = 1_000_000
    scene, cam = S.city_scene(P, seed=0, sh_degree=3, extent=256.0), S.jax004_camera(1920, 1080)
    d = Hh.to_torch(scene, cam, dev)
    H, W = cam.height, cam.width
    bg = torch.zeros(3, device=dev)
    e = torch.empty(0, device=dev)
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(W, H, seed=1)]
    g = torch.Generator(device=dev).manual_seed(23)
    offsets = torch.rand((H, W, 2), generator=g, device=dev) - 0.5

    def fwd(band, off):
        return R.rasterize_gaussians(bg, d["means3D"], e, d["opacities"], d["scales"], d["rotations"], 1.0, e, e, e, 0,
                                     d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, 0.1, H, W, d["shs"],
                                     3, d["campos"], False, False, tile_rows=band, subpixel_offset=off)

    def bwd(f, band, off, **kw):
        return R.rasterize_gaussians_backward(bg, d["means3D"], f[5], e, d["scales"], d["rotations"], e, 1.0, e, e,
                                              d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, 0.1, cot[0],
                                              cot[1], cot[2], cot[3], e, d["shs"], 3, d["campos"], f[7], f[0], f[8],
                                              f[9], f[4], False, tile_rows=band, subpixel_offset=off, **kw)

    f0 = fwd(None, None)
    it = Hh.our_internals(dict(zip(("num_rendered", "color", "depth", "norm", "alpha", "radii", "extra", "geom",
                                    "binning", "img"), f0)), P, H, W)
    cuts = MG.partition_rows(MG.row_histogram(it["ranges"], (W + 15) // 16), 2)
    bands = [(cuts[r], cuts[r + 1]) for r in range(2)]
    sl = MG.gaussian_slices(P, 2)
    acc = torch.empty((P, 16), device=dev)
    del f0, it

    def step(off, ncam):
        fs = [fwd(b, off) for b in bands]
        acc.zero_()
        for f, b in zip(fs, bands):
            acc.add_(bwd(f, b, off, phase=1))
        cam_kw = dict(camera_grad=ncam > 0, intrinsics_grad=ncam == 37)
        return [bwd(fs[r], bands[r], off, phase=2, acc=acc[sl[r]:sl[r + 1]], gauss_range=(sl[r], sl[r + 1]), **cam_kw)
                for r in range(2)]

    arms = {"plain": (None, 0), "offsets": (offsets, 0), "offsets_cam35": (offsets, 35),
            "offsets_cam37": (offsets, 37)}

    def timed(fn):
        s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(a.iters):
            fn()
        t.record()
        t.synchronize()
        return s.elapsed_time(t) / a.iters

    for _ in range(3):                                  # warm-up of every shape the timed window uses
        for v in arms.values():
            step(*v)
    torch.cuda.synchronize(dev)
    times = {k: [] for k in arms}
    for _ in range(a.repeats):
        for k, v in arms.items():
            times[k].append(timed(lambda: step(*v)))
    rec = {"device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0), "frame": "configs1_1M_jax004",
           "P": P, "W": W, "H": H, "cuts": cuts, "slices": sl, "iters": a.iters, "repeats": a.repeats,
           "step": "2 band forwards + 2 band phase-1 adjoints + 2 slice phase-2 adjoints, one GPU, no exchange"}
    for k, v in times.items():
        rec[f"{k}_ms"] = round(float(np.median(v)), 4)
        rec[f"{k}_range_ms"] = [round(float(min(v)), 4), round(float(max(v)), 4)]
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
