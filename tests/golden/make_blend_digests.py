"""SHA-256 digests of every output of the blend kernels (forward blend and blend adjoint) on fixed inputs.

Each case runs this library's forward, whose outputs are reproducible bit for bit, and (except for the extra_attrs
cases, which are forward only) the deterministic backward under torch.use_deterministic_algorithms(True): its
phase=1 sums acc [P,16], which are the blend adjoint's per-(block, Gaussian) sums added in a fixed order with no
unordered reduction, and its full gradient tuple.  tests/test_blend_walk.py holds the blend kernels to the digests
stored in blend_digests.npz, which were recorded with this script on an H100 from the build before the forward blend
and its adjoint were moved onto one shared reach-list walk (csrc/sfgs_blend_walk.cuh):

    python tests/golden/make_blend_digests.py        # needs a CUDA device and the built library
"""
from __future__ import annotations

import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "skyfall-gs_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

FIXTURE = os.path.join(HERE, "blend_digests.npz")
FWD_OUTPUTS = ("color", "depth", "alpha", "norm", "n_contrib")
GRAD_KEYS = ("means2D", "colors", "opacity", "means3D", "cov3D", "norm3D", "sh", "scales", "rot")

# name: scene, camera, background, tile-row band, fuse_normalize, extra_attrs channels (0: none; > 0: forward only)
CASES = {
    # the 1M-Gaussian benchmark frame and the whole-scene orbit frame
    "headline": dict(scene=("city", 1_000_000, 0, 256.0), cam=("jax", 1920, 1080), bg=(0.0, 0.0, 0.0)),
    "orbit": dict(scene=("city", 1_000_000, 0, 256.0), cam=("orbit", 1920, 1080), bg=(0.0, 0.0, 0.0)),
    # one band of tile rows of a smaller city frame
    "band": dict(scene=("city", 120_000, 9, 120.0), cam=("jax", 640, 360), bg=(0.1, 0.0, 0.2), band=(3, 15)),
    # non-zero background and the fused normalisation of the normal map (and its adjoint)
    "blob_fuse": dict(scene=("blob", 6000, 31, 2.5, 0.15), cam=("simple", 320, 200), bg=(0.1, 0.2, 0.3), fuse=True),
    # few, small Gaussians: most blocks' lists are shorter than one 16-record chunk
    "short_lists": dict(scene=("blob", 400, 17, 2.5, 0.05), cam=("simple", 256, 144), bg=(0.3, 0.2, 0.1)),
    # extra_attrs at one channel and at SFGS_MAX_EXTRA channels
    "extra_1": dict(scene=("blob", 6000, 31, 2.5, 0.15), cam=("simple", 320, 200), bg=(0.1, 0.2, 0.3), ED=1),
    "extra_34": dict(scene=("blob", 6000, 31, 2.5, 0.15), cam=("simple", 320, 200), bg=(0.1, 0.2, 0.3), ED=34),
}


def case_inputs(name):
    """(scene, camera, case dict) of a case."""
    from sfgs import synthetic as S
    c = CASES[name]
    kind, P, seed, *rest = c["scene"]
    scene = S.city_scene(P, seed=seed, extent=rest[0]) if kind == "city" else \
        S.blob_scene(P, seed=seed, spread=rest[0], scale=rest[1])
    kind, W, H = c["cam"]
    cam = {"jax": lambda: S.jax004_camera(W, H), "orbit": lambda: S.orbit_camera(width=W, height=H),
           "simple": lambda: S.simple_camera(W, H)}[kind]()
    return scene, cam, c


def run_case(name, dev):
    """Forward, then (unless the case has extra_attrs) the deterministic backward: {output: tensor}.  Images are
    cropped to the band's pixel rows, the only ones the call writes."""
    import torch
    import helpers as Hh
    from sfgs import rasterizer as R
    from sfgs import synthetic as S
    scene, cam, c = case_inputs(name)
    P, H, W = scene.P, cam.height, cam.width
    d = Hh.to_torch(scene, cam, dev)
    e = torch.empty(0, device=dev)
    bg = torch.tensor(c["bg"], device=dev)
    ED, band, fuse = c.get("ED", 0), c.get("band"), c.get("fuse", False)
    extras = torch.from_numpy(np.random.default_rng(5).uniform(-1, 1, (P, ED)).astype(np.float32)).to(dev) if ED else e
    out = R.rasterize_gaussians(bg, d["means3D"], e, d["opacities"], d["scales"], d["rotations"], 1.0, e, e, extras, ED,
                                d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, 0.1, H, W, d["shs"], 3,
                                d["campos"], False, False, tile_rows=band, fuse_normalize=fuse)
    f = dict(zip(("num_rendered", "color", "depth", "norm", "alpha", "radii", "extra", "geom", "binning", "img"), out))
    f["norm_raw"] = out[10] if fuse else None
    f["n_contrib"] = Hh.our_internals(f, P, H, W)["n_contrib"].view(1, H, W)
    rows = slice(band[0] * 16, min(band[1] * 16, H)) if band is not None else slice(0, H)
    res = {k: f[k][:, rows] for k in FWD_OUTPUTS}
    if fuse:
        res["norm_raw"] = f["norm_raw"][:, rows]
    if ED:
        res["extra"] = f["extra"][:, rows]
        torch.cuda.synchronize(dev)
        return res
    cot = [torch.from_numpy(x).to(dev) for x in S.cotangents(W, H, seed=3)]
    kw = dict(tile_rows=band, norm_raw=f["norm_raw"])
    prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
    torch.use_deterministic_algorithms(True)
    try:
        res["acc"] = Hh.run_ours_backward(d, cam, 3, bg, f, cot, phase=1, **kw)
        g = Hh.run_ours_backward(d, cam, 3, bg, f, cot, **kw)
    finally:
        torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])
    res.update({f"grad_{k}": g[k] for k in GRAD_KEYS})
    torch.cuda.synchronize(dev)
    return res


def digest(t):
    return hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()


def main():
    import torch
    dev = torch.device("cuda:0")
    rec = {"device": np.array(torch.cuda.get_device_name(dev))}
    for name in CASES:
        res = run_case(name, dev)
        for k, v in res.items():
            rec[f"{name}/{k}"] = np.array(digest(v))
        nc = res["n_contrib"]
        print(f"{name}: {len(res)} outputs, n_contrib max {int(nc.max())} mean {float(nc.float().mean()):.1f}", flush=True)
    np.savez_compressed(FIXTURE, **rec)
    print("wrote", FIXTURE)


if __name__ == "__main__":
    main()
