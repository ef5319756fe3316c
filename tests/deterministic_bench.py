"""The deterministic backward against the default one on bench.py's frames — needs a GPU.  Not a pytest file.

    python tests/deterministic_bench.py [--frames configs1_1M_jax004,dense_5M_jax004] [--repeats 7] [--iters 20]

Per frame: bench.py's scene, camera and cotangents (S.cotangents(W, H, seed=1)), one forward, then the default and the
deterministic backward (torch.use_deterministic_algorithms) timed alternately: CUDA events around `--iters` calls,
`--repeats` rounds, median / min / max over rounds.  Then one profiled call of each gives the stage times
(sfgs_profile_*).  The last call of every timed deterministic round, the warm-up calls and repeats x iters further
calls are compared byte for byte with the first deterministic call; any difference fails the run.  The extra scratch of the
deterministic path is 4 P + 524 R bytes (include/sfgs.h).  One JSON line per frame, with the card's name and power limit.
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
from sfgs import synthetic as S

FRAMES = {   # bench.py's headline frame and EXTRA_FRAMES["dense_5M_jax004"]
    "configs1_1M_jax004": (1_000_000, 256.0),
    "dense_5M_jax004": (5_000_000, 256.0),
}


KEYS = ("means2D", "colors", "opacity", "means3D", "cov3D", "norm3D", "sh", "scales", "rot")


def same_bytes(a, b):
    return all(torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)) for k in KEYS)


def run_frame(name, dev, repeats, iters):
    P, extent = FRAMES[name]
    scene, cam = S.city_scene(P, seed=0, sh_degree=3, extent=extent), S.jax004_camera(1920, 1080)
    d = Hh.to_torch(scene, cam, dev)
    bg = torch.zeros(3, device=dev)
    f = Hh.run_ours_forward(d, cam, 3, bg)
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height, seed=1)]
    R = int(f["num_rendered"])
    first = None
    checked, differing = 0, 0

    def default():
        torch.use_deterministic_algorithms(False)
        return Hh.run_ours_backward(d, cam, 3, bg, f, cot)

    def ordered():
        torch.use_deterministic_algorithms(True)
        try:
            return Hh.run_ours_backward(d, cam, 3, bg, f, cot)
        finally:
            torch.use_deterministic_algorithms(False)

    def check(o):
        nonlocal checked, differing
        checked += 1
        differing += 0 if same_bytes(o, first) else 1

    def timed(fn, keep):
        """ms per call; with `keep` the last call's outputs are compared with the first deterministic call's"""
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            o = fn()
        b.record()
        b.synchronize()
        if keep:
            check(o)
        return a.elapsed_time(b) / iters

    for _ in range(3):
        default()
        o = ordered()
        first = o if first is None else first
        check(o)
    torch.cuda.synchronize(dev)
    times = {"default": [], "deterministic": []}
    for _ in range(repeats):
        times["default"].append(timed(default, False))
        times["deterministic"].append(timed(ordered, True))
    # every one of as many further deterministic calls as were timed, compared on the device
    for _ in range(repeats * iters):
        check(ordered())
    stages = {}
    for k, fn in (("default", default), ("deterministic", ordered)):
        N.profile_enable(True)
        fn()
        torch.cuda.synchronize(dev)
        stages[k] = {s: round(v[0], 4) for s, v in N.profile_read().items() if s in ("bwd_zero", "render_bwd", "gauss_bwd", "bwd_order")}
        N.profile_enable(False)
    tt = Hh.our_internals(f, P, cam.height, cam.width)["tiles_touched"]
    rec = {"frame": name, "P": P, "V": int((f["radii"] > 0).sum()), "R": R, "max_tiles_touched": int(tt.max()),
           "iters": iters, "repeats": repeats}
    for k, v in times.items():
        rec[f"{k}_ms"] = round(float(np.median(v)), 4)
        rec[f"{k}_range_ms"] = [round(float(min(v)), 4), round(float(max(v)), 4)]
    rec["ratio"] = round(rec["deterministic_ms"] / rec["default_ms"], 3)
    rec["stages_ms"] = stages
    rec["extra_scratch_bytes"] = 4 * P + 524 * R
    rec["calls_compared"] = checked
    rec["calls_differing"] = differing
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", default=",".join(FRAMES))
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("deterministic_bench.py needs a CUDA device")
    dev = torch.device("cuda:0")
    card = {"device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0)}
    bad = []
    for name in a.frames.split(","):
        rec = run_frame(name, dev, a.repeats, a.iters)
        print(json.dumps({**card, **rec}), flush=True)
        if rec["calls_differing"]:
            bad.append(name)
        torch.cuda.empty_cache()
    if bad:
        sys.exit(f"deterministic backward returned different bytes across calls on {bad}")


if __name__ == "__main__":
    main()
