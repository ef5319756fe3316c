"""GPU tests of the two sibling ops: fused SSIM and simple-knn's distCUDA2."""
import os

import numpy as np
import pytest
import torch

import helpers as Hh

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def torch_ssim_map(a, b):
    """conv2d SSIM, the construction the reference's own test compares against (SSIM/tests/test.py:47-76)."""
    import torch.nn.functional as F
    from oracle.ssim_oracle import GAUSS
    g = torch.tensor(GAUSS, dtype=a.dtype, device=a.device)
    C = a.shape[1]
    w = (g[:, None] * g[None, :])[None, None].expand(C, 1, 11, 11).contiguous()
    mu1, mu2 = F.conv2d(a, w, padding=5, groups=C), F.conv2d(b, w, padding=5, groups=C)
    s1 = F.conv2d(a * a, w, padding=5, groups=C) - mu1 * mu1
    s2 = F.conv2d(b * b, w, padding=5, groups=C) - mu2 * mu2
    s12 = F.conv2d(a * b, w, padding=5, groups=C) - mu1 * mu2
    return ((2 * mu1 * mu2 + 1e-4) * (2 * s12 + 9e-4)) / ((mu1 * mu1 + mu2 * mu2 + 1e-4) * (s1 + s2 + 9e-4))


def test_fused_ssim_matches_golden_and_torch(cuda_device):
    from fused_ssim import fused_ssim
    dev = cuda_device
    g = np.load(os.path.join(GOLD, "ssim_ref.npz"))
    a = torch.from_numpy(g["img1"]).to(dev).requires_grad_(True)
    b = torch.from_numpy(g["img2"]).to(dev)
    v = fused_ssim(a, b)
    v.backward()
    assert abs(v.item() - float(g["mean"])) < 2e-6
    assert np.abs(a.grad.cpu().numpy() - g["grad"]).max() < 1e-7 + 1e-3 * np.abs(g["grad"]).max()
    # the reference's own test shapes (B,CH,H,W = 5,5,1080,1920 there; smaller here) and its isclose criterion
    torch.manual_seed(0)
    x = torch.rand(2, 3, 270, 333, device=dev, requires_grad=True)
    y = torch.rand(2, 3, 270, 333, device=dev)
    got = fused_ssim(x, y)
    want = torch_ssim_map(x.double(), y.double()).mean()
    assert torch.isclose(got.double(), want, rtol=1e-5, atol=1e-6)
    got.backward()
    gx = x.grad.clone()
    xd = x.detach().double().requires_grad_(True)
    torch_ssim_map(xd, y.double()).mean().backward()
    assert (gx.double() - xd.grad).abs().max().item() < 1e-9 + 1e-3 * xd.grad.abs().max().item()
    # "valid" padding crops 5 px and inference mode skips the derivative maps
    vv = fused_ssim(x.detach(), y, padding="valid", train=False)
    want_v = torch_ssim_map(x.detach().double(), y.double())[:, :, 5:-5, 5:-5].mean()
    assert torch.isclose(vv.double(), want_v, rtol=1e-5, atol=1e-6)


def test_dist_cuda2_matches_bruteforce_and_reference(cuda_device):
    from oracle import knn_oracle
    from simple_knn._C import distCUDA2
    dev = cuda_device
    rng = np.random.default_rng(3)
    clouds = {
        "uniform": rng.uniform(-5, 5, size=(20000, 3)),
        "clustered": np.concatenate([rng.normal(0, 0.05, (5000, 3)), rng.normal(3, 1.0, (5000, 3)), [[40.0, -30.0, 9.0]]]),
        "flat": np.concatenate([rng.uniform(-2, 2, (8000, 2)), np.zeros((8000, 1))], 1),
        "dupes": np.repeat(rng.uniform(0, 1, (300, 3)), 4, axis=0),
        "tiny": rng.uniform(0, 1, (5, 3)),
    }
    for name, pts in clouds.items():
        pts = pts.astype(np.float32)
        got = distCUDA2(torch.from_numpy(pts).to(dev)).cpu().numpy()
        want = knn_oracle.dist2_knn3(pts)
        assert np.allclose(got, want, rtol=2e-6, atol=1e-12), name
    from oracle import ref_cuda
    F = Hh.RefFacts("dist_cuda2")
    pts = torch.from_numpy(clouds["uniform"].astype(np.float32)).to(dev)
    # same 3-NN set; the squared distance may contract differently (1 ulp)
    F.close("uniform", distCUDA2(pts), lambda: ref_cuda.knn(pts), atol=0.0, rtol=1e-6)


def test_expf_replica_is_bit_exact(cuda_device):
    """The blend kernels evaluate expf through a hand-scheduled replica of the compiler's routine (constants pinned in
    registers, csrc/sfgs_common.cuh).  The alpha thresholds that decide n_contrib sit on its result, so it must equal
    expf() bit for bit: a dense sweep of the range the kernels use, every exponent/sign pattern, and special values."""
    from sfgs import native as N
    dev = cuda_device
    g = torch.Generator(device="cpu").manual_seed(3)
    parts = [torch.linspace(-110.0, 0.0, 8_000_001, dtype=torch.float64).float(),          # the kernels' range
             -torch.rand(4_000_000, generator=g).mul(20.0),                                 # where alpha is decided
             -torch.exp(torch.rand(2_000_000, generator=g) * 60.0 - 50.0),                  # log-uniform magnitudes
             torch.randint(-2 ** 31, 2 ** 31 - 1, (4_000_000,), generator=g, dtype=torch.int64).to(torch.int32).view(torch.float32),
             torch.tensor([0.0, -0.0, 1.0, -1.0, 88.7, 88.8, -87.3, -87.4, -103.9, -104.1, float("inf"), float("-inf"),
                           1e-45, -1e-45, 1.1754944e-38, -1.1754944e-38, 3.0e38, -3.0e38])]
    x = torch.cat(parts).to(dev)
    yr, ye = torch.empty_like(x), torch.empty_like(x)
    N.check(N.lib().sfgs_selftest_expf(x.numel(), x.data_ptr(), yr.data_ptr(), ye.data_ptr(),
                                       torch.cuda.current_stream(dev).cuda_stream), "selftest_expf")
    torch.cuda.synchronize(dev)
    ok = (yr.view(torch.int32) == ye.view(torch.int32)) | (torch.isnan(yr) & torch.isnan(ye))
    # the kernels only ever use the value for arguments <= 0 (a positive `power` is rejected before/independently)
    neg = x <= 0
    bad = (~ok) & neg
    assert int(bad.sum()) == 0, f"{int(bad.sum())} mismatches for x <= 0, e.g. x = {x[bad][:5].tolist()}"
    assert float(ok.float().mean()) > 0.999, "replica should agree with expf on (almost) every bit pattern"


def _ref_fused_ssim():
    from oracle import build_ref_torch
    return build_ref_torch.import_reference_packages()[1] if build_ref_torch.built() else None


@pytest.mark.parametrize("shape", [(5, 5, 1080, 1920), (1, 3, 1080, 1920), (2, 3, 270, 333), (1, 1, 17, 19), (1, 2, 64, 4),
                                   (1, 3, 33, 130)])
def test_fused_ssim_against_the_reference_cuda_kernel(cuda_device, shape):
    """The reference's own compiled fused-ssim (SSIM/ssim.cu, built by oracle/build_ref_torch.py with its setup.py's
    flags) as the oracle, first on its own test workload (SSIM/tests/test.py:81-83: B=5, CH=5, 1080x1920), then on
    the training shape and on sizes that are off the tile grid, odd, narrower than a tile or not 16-byte rows (the
    non-TMA load path).  The reference kernel is compiled with --use_fast_math (approximate divisions): the map agrees
    within 1e-5 (the image tolerance of the north star), and for the end-to-end value and gradient a float64 torch
    evaluation decides whose error a deviation is (ours <= 2x the reference kernel's).  Where the reference's build is
    absent, what a run on an H100 recorded stands in for it (helpers.RefFacts); the backward kernel alone, fed the
    reference's derivative maps, is then not compared (the maps themselves and the end-to-end gradient are)."""
    ref = _ref_fused_ssim()
    F = Hh.RefFacts("fused_ssim_" + "x".join(str(n) for n in shape), live=ref is not None)
    from fused_ssim import fused_ssim, fusedssim, fusedssim_backward
    dev = cuda_device
    g = torch.Generator(device="cpu").manual_seed(sum(shape))
    a = torch.rand(shape, generator=g).to(dev)
    b = (a + 0.2 * torch.randn(shape, generator=g).to(dev)).clamp(0, 1) if shape[2] > 20 else torch.rand(shape, generator=g).to(dev)
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    r = ref.fusedssim(C1, C2, a, b, True) if F.live else None
    m1, d1, e1, f1 = fusedssim(C1, C2, a, b, True)
    # the value map is O(1); the derivative maps reach ~1/C2 and dm_dmu1 is a difference of terms far larger than the
    # result (the reference sums four of them with approximate divisions), so they are compared relative to the
    # largest magnitude in the tensor
    for i, (name, x, rel) in enumerate((("ssim_map", m1, 1e-5), ("dm_dmu1", d1, 2e-5), ("dm_dsigma1_sq", e1, 2e-5),
                                        ("dm_dsigma12", f1, 2e-5))):
        tol = rel * max(1.0, F.value(name + "_absmax", lambda: float(r[i].abs().max())))
        F.close(name, x, lambda: r[i], tol)
    dL = torch.randn(shape, generator=g).to(dev)
    if F.live:
        m0, d0, e0, f0 = r
        g0 = ref.fusedssim_backward(C1, C2, a, b, dL, d0, e0, f0)
        g1 = fusedssim_backward(C1, C2, a, b, dL, d0, e0, f0)         # same derivative maps in: isolates the backward kernel
        assert float((g1 - g0).abs().max()) <= 2e-6 * max(1.0, float(g0.abs().max()))
        del r, m0, d0, e0, f0, g0, g1
    # the public entry point end to end; whose error a deviation is, is decided by a float64 torch evaluation
    x0, x1 = a.clone().requires_grad_(True), a.clone().requires_grad_(True)
    v1 = fused_ssim(x1, b)
    v1.backward()
    if F.live:
        v0 = ref.fused_ssim(x0, b)
        v0.backward()
    v0_item = F.value("value", lambda: v0.item())
    assert abs(v0_item - v1.item()) < 2e-6
    if a.numel() <= 20_000_000:
        xd = a.double().requires_grad_(True)
        vd = torch_ssim_map(xd, b.double()).mean()
        vd.backward()
        e_ours = float((x1.grad.double() - xd.grad).abs().max())
        e_ref = F.value("grad_err_vs_f64", lambda: float((x0.grad.double() - xd.grad).abs().max()))
        assert abs(v1.item() - vd.item()) <= 2 * abs(v0_item - vd.item()) + 1e-6
        assert e_ours <= 2 * e_ref + 1e-9 * float(xd.grad.abs().max()) + 1e-12, (e_ours, e_ref)
    else:
        F.close("grad", x1.grad, lambda: x0.grad, 2e-5 * F.value("grad_absmax", lambda: float(x0.grad.abs().max())) + 1e-12)
    if shape[2] > 10 and shape[3] > 10:
        v_valid = F.value("value_valid", lambda: ref.fused_ssim(a, b, padding="valid", train=False).item())
        assert abs(v_valid - fused_ssim(a, b, padding="valid", train=False).item()) < 2e-6
