"""SHA-256 digests of every output of the per-Gaussian adjoint (backward phase 2) on fixed inputs.

Each case runs this library's forward (deterministic and bit-exact), then the backward with phase=2 over a Gaussian
range from a seeded [P,16] blend-adjoint sum buffer `acc`.  Phase 2 is the per-Gaussian adjoint alone, with no
unordered reductions in front of it, so its eleven output arrays are reproducible bit for bit.
tests/test_gauss_bwd.py holds the kernel to the digests stored in gauss_bwd_digests.npz, which were recorded with
this script on an H100 from the build before the per-Gaussian adjoint was rewritten as a span pipeline:

    python tests/golden/make_gauss_bwd_digests.py        # needs a CUDA device and the built library
"""
from __future__ import annotations

import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "skyfall-gs_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

FIXTURE = os.path.join(HERE, "gauss_bwd_digests.npz")
OUTPUTS = ("means2D", "conic", "opacity", "colors", "depths", "means3D", "cov3D", "norm3D", "sh", "scales", "rot")
# rasterizer.rasterize_gaussians_backward allocates the fixed-width gradients as one buffer, in this order, each part
# padded to a multiple of 4 floats; conic and depths are not in its return tuple and are read from that buffer
_FLAT = (("means3D", 3), ("means2D", 3), ("colors", 3), ("depths", 1), ("conic", 4), ("opacity", 1), ("cov3D", 6),
         ("norm3D", 3), ("scales", 3), ("rot", 4))

# name: scene, camera, stored SH degree, active degree, scale_modifier, inputs (shs | colors | cov3D+norm3D), range
CASES = {
    "headline": dict(scene="city", P=1_000_000, cam="jax", stored=3, D=3, mod=1.0, kind="shs", rng=None),
    "headline_subrange": dict(scene="city", P=1_000_000, cam="jax", stored=3, D=3, mod=1.0, kind="shs",
                              rng=(12_345, 987_651)),
    "orbit": dict(scene="city", P=1_000_000, cam="orbit", stored=3, D=3, mod=1.0, kind="shs", rng=None),
    "blob_m9_mod": dict(scene="blob", P=20_001, cam="simple", stored=2, D=1, mod=0.8, kind="shs", rng=(3, 19_998)),
    "blob_colors": dict(scene="blob", P=20_001, cam="simple", stored=3, D=3, mod=1.0, kind="colors", rng=None),
    "blob_precomp": dict(scene="blob", P=20_001, cam="simple", stored=3, D=3, mod=1.0, kind="precomp", rng=(1, 20_001)),
}


def cov3d_from(scales, rotations, mod=1.0):
    """Upper triangle (xx, xy, xz, yy, yz, zz) of R S S^T R^T, as the forward computes it from scales and rotations."""
    r, x, y, z = (rotations[:, k].astype(np.float64) for k in range(4))
    R = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                  2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                  2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)
    Mm = R * (mod * scales.astype(np.float64))[:, None, :]
    Sig = Mm @ Mm.transpose(0, 2, 1)
    return np.stack([Sig[:, 0, 0], Sig[:, 0, 1], Sig[:, 0, 2], Sig[:, 1, 1], Sig[:, 1, 2], Sig[:, 2, 2]], 1).astype(np.float32)


def case_inputs(name):
    """(scene, camera, case dict, extra numpy inputs) of a case."""
    from sfgs import synthetic as S
    c = CASES[name]
    if c["scene"] == "city":
        scene = S.city_scene(c["P"], seed=0, sh_degree=c["stored"])
    else:
        scene = S.blob_scene(c["P"], seed=29, sh_degree=c["stored"])
    cam = {"jax": lambda: S.jax004_camera(1920, 1080), "orbit": lambda: S.orbit_camera(width=1920, height=1080),
           "simple": lambda: S.simple_camera(333, 211)}[c["cam"]]()
    rng = np.random.default_rng(7)
    extra = {}
    if c["kind"] == "colors":
        extra["colors"] = rng.uniform(0, 1, (scene.P, 3)).astype(np.float32)
    elif c["kind"] == "precomp":
        extra["cov3D"] = cov3d_from(scene.scales, scene.rotations, c["mod"])
        n = rng.normal(size=(scene.P, 3))
        extra["norm3D"] = (n / np.linalg.norm(n, axis=1, keepdims=True)).astype(np.float32)
    return scene, cam, c, extra


def run_phase2(name, dev):
    """Forward, then the per-Gaussian adjoint over the case's range from a seeded acc: {output: tensor of the range}."""
    import torch
    from sfgs import rasterizer as R
    scene, cam, c, extra = case_inputs(name)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    e = torch.empty(0, device=dev)
    P = scene.P
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    means3D, opac = t(scene.means3D), t(scene.opacities)
    shs = e if c["kind"] == "colors" else t(scene.shs)
    colors = t(extra["colors"]) if "colors" in extra else e
    cov3D = t(extra["cov3D"]) if "cov3D" in extra else e
    norm3D = t(extra["norm3D"]) if "norm3D" in extra else e
    scales, rots = (e, e) if c["kind"] == "precomp" else (t(scene.scales), t(scene.rotations))
    view, proj, campos = t(cam.viewmatrix), t(cam.projmatrix), t(cam.campos)
    f = R.rasterize_gaussians(bg, means3D, colors, opac, scales, rots, c["mod"], cov3D, norm3D, e, 0, view, proj,
                              cam.tanfovx, cam.tanfovy, 0.1, cam.height, cam.width, shs, c["D"], campos, False, False)
    a, b = c["rng"] if c["rng"] is not None else (0, P)
    g = torch.Generator().manual_seed(1234)
    acc = (torch.randn((P, 16), generator=g) * 0.01).to(dev)
    cot = [torch.zeros((k, cam.height, cam.width), device=dev) for k in (3, 1, 3, 1)]
    out = R.rasterize_gaussians_backward(bg, means3D, f[5], colors, scales, rots, e, c["mod"], cov3D, norm3D, view, proj,
                                         cam.tanfovx, cam.tanfovy, 0.1, cot[0], cot[1], cot[2], cot[3], e, shs, c["D"],
                                         campos, f[7], f[0], f[8], f[9], f[4], False, phase=2,
                                         acc=acc[a:b].clone(), gauss_range=(a, b))
    torch.cuda.synchronize(dev)
    ret = dict(zip(("means2D", "colors", "opacity", "means3D", "cov3D", "norm3D", "sh", "scales", "rot"), out[:9]))
    # the whole fixed-width buffer, to reach conic and depths
    flat = torch.empty(0, dtype=torch.float32, device=dev).set_(ret["means3D"].untyped_storage())
    off = 0
    for k, w in _FLAT:
        assert ret.get(k) is None or ret[k].data_ptr() == flat.data_ptr() + 4 * off, k
        ret[k] = flat[off:off + P * w].view(P, w)
        off += (P * w + 3) & ~3
    res = {k: ret[k][a:b] for k in OUTPUTS}
    res["_visible"] = int((f[5][a:b] > 0).sum().item())
    return res


def digest(t):
    return hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()


def main():
    import torch
    dev = torch.device("cuda:0")
    rec = {"device": np.array(torch.cuda.get_device_name(dev))}
    for name in CASES:
        res = run_phase2(name, dev)
        for k in OUTPUTS:
            rec[f"{name}/{k}"] = np.array(digest(res[k]))
        print(f"{name}: visible {res['_visible']}, sh {tuple(res['sh'].shape)}", flush=True)
    np.savez_compressed(FIXTURE, **rec)
    print("wrote", FIXTURE)


if __name__ == "__main__":
    main()
