"""Cost of the focal-length gradients on bench.py's headline frame — needs a GPU.  Not a pytest file.

    python tests/intrinsics_grad_bench.py [--repeats 9] [--iters 20]

Frame: 1M Gaussians (city scene, seed 0, SH degree 3), 1920x1080, bench.py's cotangents (S.cotangents(W, H, seed=1)).
Six arms of the backward, timed alternately in one process: without camera gradients, with the 35 camera terms
(sfgs_rasterize_backward_camera) and with the 37 camera and focal terms (sfgs_rasterize_backward_camera_intrinsics),
each in its default and its deterministic form.  CUDA events around `--iters` calls of one forward's backward,
`--repeats` rounds, median / min / max over rounds; plus the per-Gaussian stage (stage 8, which holds the camera
reduction) from the library's stage timer.  One JSON line, with the card's name and power limit.
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
from sfgs import native as N
from sfgs import rasterizer as R
from sfgs import synthetic as S


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=9)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("intrinsics_grad_bench.py needs a CUDA device")
    dev = torch.device("cuda:0")
    P = 1_000_000
    scene, cam = S.city_scene(P, seed=0, sh_degree=3, extent=256.0), S.jax004_camera(1920, 1080)
    d = Hh.to_torch(scene, cam, dev)
    H, W = cam.height, cam.width
    bg = torch.zeros(3, device=dev)
    e = torch.empty(0, device=dev)
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(W, H, seed=1)]
    f = R.rasterize_gaussians(bg, d["means3D"], e, d["opacities"], d["scales"], d["rotations"], 1.0, e, e, e, 0,
                              d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, 0.1, H, W, d["shs"], 3,
                              d["campos"], False, False)
    # (deterministic, camera_grad, intrinsics_grad)
    arms = {"default": (False, False, False), "camera": (False, True, False), "intrinsics": (False, True, True),
            "det_default": (True, False, False), "det_camera": (True, True, False),
            "det_intrinsics": (True, True, True)}

    def bwd(det, camera, intrinsics):
        torch.use_deterministic_algorithms(det)
        try:
            return R.rasterize_gaussians_backward(bg, d["means3D"], f[5], e, d["scales"], d["rotations"], e, 1.0, e, e,
                                                  d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, 0.1,
                                                  cot[0], cot[1], cot[2], cot[3], e, d["shs"], 3, d["campos"], f[7],
                                                  f[0], f[8], f[9], f[4], False, camera_grad=camera,
                                                  intrinsics_grad=intrinsics)
        finally:
            torch.use_deterministic_algorithms(False)

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
            bwd(*v)
    torch.cuda.synchronize(dev)
    times = {k: [] for k in arms}
    for r in range(a.repeats):
        order = list(arms.items())
        if r % 2:
            order.reverse()                             # alternate the order of the arms between rounds
        for k, v in order:
            times[k].append(timed(lambda: bwd(*v)))
    stage8 = {}
    for k, v in arms.items():
        N.profile_enable(True)
        for _ in range(a.iters):
            bwd(*v)
        torch.cuda.synchronize(dev)
        ms, n = N.profile_read()["gauss_bwd"]
        N.profile_enable(False)
        stage8[k] = round(ms / max(n, 1), 4)
    rec = {"device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0), "frame": "configs1_1M_jax004",
           "P": P, "W": W, "H": H, "R": int(f[0]), "visible": int((f[5] > 0).sum()), "iters": a.iters,
           "repeats": a.repeats}
    for k, v in times.items():
        rec[f"{k}_bwd_ms"] = round(float(np.median(v)), 4)
        rec[f"{k}_bwd_range_ms"] = [round(float(min(v)), 4), round(float(max(v)), 4)]
        rec[f"{k}_stage8_ms"] = stage8[k]
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
