"""Cost of subpixel offsets on bench.py's headline frame — needs a GPU.  Not a pytest file.

    python tests/subpixel_bench.py [--repeats 7] [--iters 20]

Frame: 1M Gaussians (city scene, seed 0, SH degree 3), 1920x1080, bench.py's cotangents (S.cotangents(W, H, seed=1)).
Three arms, timed alternately in one process: the default call, the _subpixel call with all-zero offsets, and with
U(-0.5, 0.5) offsets.  Per arm: forward, backward and forward + backward, each with CUDA events around `--iters` calls,
`--repeats` rounds, median / min / max over rounds.  Also the number of set (instance, block) reach-mask bits with and
without the dilation of the U(-0.5, 0.5) offsets: the extra (pixel, Gaussian) pairs that jitter lets through.  One JSON
line, with the card's name and power limit.
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
from sfgs import rasterizer as R
from sfgs import synthetic as S

POPCOUNT = torch.tensor([bin(i).count("1") for i in range(256)], dtype=torch.int64)


def mask_bits(f):
    """Set bits over every sorted instance's reach mask (BinningLayout: point_list, then inst_mask)."""
    hdr = f[9][:32].view(torch.int32).cpu().numpy().astype(np.uint32)
    cap = int(hdr[2]) | (int(hdr[3]) << 32)
    b = f[8]
    off = ((b.data_ptr() + 255) & ~255) - b.data_ptr() + ((cap * 4 + 255) & ~255)
    m = b[off:off + int(f[0])].long().cpu()
    return int(POPCOUNT[m].sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("subpixel_bench.py needs a CUDA device")
    dev = torch.device("cuda:0")
    P = 1_000_000
    scene, cam = S.city_scene(P, seed=0, sh_degree=3, extent=256.0), S.jax004_camera(1920, 1080)
    d = Hh.to_torch(scene, cam, dev)
    H, W = cam.height, cam.width
    bg = torch.zeros(3, device=dev)
    e = torch.empty(0, device=dev)
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(W, H, seed=1)]
    g = torch.Generator(device=dev).manual_seed(0)
    arms = {"default": None, "zero": torch.zeros((H, W, 2), device=dev),
            "uniform": torch.rand((H, W, 2), generator=g, device=dev) - 0.5}

    def fwd(off):
        return R.rasterize_gaussians(bg, d["means3D"], e, d["opacities"], d["scales"], d["rotations"], 1.0, e, e, e, 0,
                                     d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, 0.1, H, W, d["shs"], 3,
                                     d["campos"], False, False, subpixel_offset=off)

    def bwd(f, off):
        return R.rasterize_gaussians_backward(bg, d["means3D"], f[5], e, d["scales"], d["rotations"], e, 1.0, e, e,
                                              d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, 0.1, cot[0],
                                              cot[1], cot[2], cot[3], e, d["shs"], 3, d["campos"], f[7], f[0], f[8],
                                              f[9], f[4], False, subpixel_offset=off)

    def timed(fn):
        s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(a.iters):
            fn()
        t.record()
        t.synchronize()
        return s.elapsed_time(t) / a.iters

    saved = {k: fwd(v) for k, v in arms.items()}
    for _ in range(3):                                  # warm-up of every shape the timed window uses
        for k, v in arms.items():
            bwd(fwd(v), v)
    torch.cuda.synchronize(dev)
    times = {k: {"fwd": [], "bwd": [], "fwd_bwd": []} for k in arms}
    for _ in range(a.repeats):
        for k, v in arms.items():
            times[k]["fwd"].append(timed(lambda: fwd(v)))
            times[k]["bwd"].append(timed(lambda: bwd(saved[k], v)))
            times[k]["fwd_bwd"].append(timed(lambda: bwd(fwd(v), v)))
    rec = {"device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0), "frame": "configs1_1M_jax004",
           "P": P, "W": W, "H": H, "R": int(saved["default"][0]), "iters": a.iters, "repeats": a.repeats}
    for k, t in times.items():
        for s, v in t.items():
            rec[f"{k}_{s}_ms"] = round(float(np.median(v)), 4)
            rec[f"{k}_{s}_range_ms"] = [round(float(min(v)), 4), round(float(max(v)), 4)]
    rec["mask_bits_undilated"] = mask_bits(saved["default"])
    rec["mask_bits_zero_offsets"] = mask_bits(saved["zero"])
    rec["mask_bits_dilated"] = mask_bits(saved["uniform"])
    rec["offset_bound"] = [round(float(arms["uniform"][..., i].abs().max()), 6) for i in range(2)]
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
