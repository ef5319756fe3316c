"""The per-Gaussian adjoint (backward phase 2) on its own.

- Bit identity: for fixed inputs and a seeded [P,16] blend-adjoint sum buffer, all eleven output arrays hash to the
  digests in tests/golden/gauss_bwd_digests.npz (recorded on an H100 by tests/golden/make_gauss_bwd_digests.py).
  The cases cover the 1M-Gaussian benchmark frame, a sub-range starting at an odd Gaussian (unaligned output rows,
  acc row 0 != Gaussian 0), the whole-scene orbit frame, stored SH degree 2 (M = 9) at active degree 1 with a
  scale_modifier, precomputed colours (M = 0) and precomputed covariances and normals without scales.
- Precomputed covariances and normals against the CPU oracle, through the whole backward.
"""
import importlib.util
import os

import numpy as np
import pytest
import torch

from sfgs import synthetic as S

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _cases_module():
    spec = importlib.util.spec_from_file_location("make_gauss_bwd_digests", os.path.join(GOLD, "make_gauss_bwd_digests.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


G = _cases_module()


@pytest.mark.parametrize("case", list(G.CASES))
def test_phase2_outputs_bit_identical(cuda_device, case):
    with np.load(G.FIXTURE) as z:
        want = {k: str(z[k]) for k in z.files}
    res = G.run_phase2(case, cuda_device)
    assert res["_visible"] > 0
    bad = [k for k in G.OUTPUTS if G.digest(res[k]) != want[f"{case}/{k}"]]
    assert not bad, f"{case}: {bad} differ from the recorded digests"


def test_precomputed_cov3d_and_normals_vs_cpu_oracle(cuda_device):
    from oracle import cpu_oracle as O
    dev = cuda_device
    scene, cam = S.blob_scene(3001, seed=43), S.simple_camera(190, 150)
    rng = np.random.default_rng(8)
    cov3D = G.cov3d_from(scene.scales, scene.rotations)
    n = rng.normal(size=(scene.P, 3))
    norm3D = (n / np.linalg.norm(n, axis=1, keepdims=True)).astype(np.float32)
    bg = np.array([0.3, 0.1, 0.2], np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    from sfgs import rasterizer as R
    e = torch.empty(0, device=dev)
    means3D, opac, shs = t(scene.means3D), t(scene.opacities), t(scene.shs)
    view, proj, campos, bg_t = t(cam.viewmatrix), t(cam.projmatrix), t(cam.campos), t(bg)
    f = R.rasterize_gaussians(bg_t, means3D, e, opac, e, e, 1.0, t(cov3D), t(norm3D), e, 0, view, proj, cam.tanfovx,
                              cam.tanfovy, 0.1, cam.height, cam.width, shs, 3, campos, False, False)
    o = O.forward(scene.means3D, None, None, scene.opacities, scene.shs, 3, cam.viewmatrix, cam.projmatrix, cam.campos,
                  cam.width, cam.height, cam.tanfovx, cam.tanfovy, bg, cov3D_precomp=cov3D, norm3D_precomp=norm3D)
    assert np.array_equal(f[5].cpu().numpy(), o["radii"]) and (o["radii"] > 0).sum() > 1000
    for k, ours in (("color", f[1]), ("depth", f[2]), ("norm", f[3]), ("alpha", f[4])):
        assert np.abs(ours.cpu().numpy() - o[k]).max() <= 5e-5, k
    cot = S.cotangents(cam.width, cam.height, seed=6)
    c = [t(x) for x in cot]
    out = R.rasterize_gaussians_backward(bg_t, means3D, f[5], e, e, e, e, 1.0, t(cov3D), t(norm3D), view, proj,
                                         cam.tanfovx, cam.tanfovy, 0.1, c[0], c[1], c[2], c[3], e, shs, 3, campos,
                                         f[7], f[0], f[8], f[9], f[4], False)
    gb = dict(zip(("means2D", "colors", "opacity", "means3D", "cov3D", "norm3D", "sh", "scales", "rot"), out[:9]))
    og = O.backward(o, *cot)
    for k in ("means2D", "opacity", "means3D", "cov3D", "norm3D", "sh"):
        a, b = gb[k].cpu().numpy().astype(np.float64), og[k].astype(np.float64)
        assert np.abs(a - b).max() <= 1e-4 + 2e-4 * np.abs(b).max(), k
    assert not gb["scales"].any() and not gb["rot"].any()
