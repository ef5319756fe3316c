"""The fused appearance path at every SH width a GaussianModel can store: features [P, M, 3], M = 1, 4, 9, 16.

Golden vectors: tests/golden/appearance_ref.npz holds the inputs and the M = 16 colours.  For M = 1, 4, 9 the features
are the first M coefficients of its features with the rows shifted by `row_shift`, and
tests/golden/appearance_widths_ref.npz holds the colours the reference's own EmbeddingModel + eval_sh give for them
at every degree the width holds (tests/golden/make_appearance_widths_golden.py, float32 and float64).
  * CPU: the torch formulation (the backward's recompute) equals the reference modules at every width and degree;
    the C ABI rejects widths it is not built for and degrees the width cannot hold.
  * GPU: the wgmma kernel equals the float64 reference within the bf16-split tolerance at every (M, D) pair and ragged
    P; its M = 16 colours are bit-identical to the digests recorded from the kernel before it was templated on M
    (tests/golden/make_appearance_digests.py); the autograd wrapper's gradients at M = 4 are the torch formulation's.
"""
import importlib.util
import os

import numpy as np
import pytest
import torch

GOLD_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
WIDTHS = os.path.join(GOLD_DIR, "appearance_widths_ref.npz")
M16 = os.path.join(GOLD_DIR, "appearance_ref.npz")
COLOR_ATOL = 1e-4      # split-bf16 (hi + lo) tensor-core operands, fp32 accumulation: ~2^-16 relative per product
KEYS = ("features", "gemb", "aemb", "W1", "b1", "W2", "b2", "W3", "b3", "xyz", "campos")
PAIRS = [(M, D) for M in (1, 4, 9, 16) for D in range(4) if (D + 1) ** 2 <= M]
SFGS_E_BADARG, SFGS_E_UNSUPPORTED = -2, -4


def _load(M, dev, dtype=torch.float32, tag="f64"):
    """({deg: reference colours in `tag` precision, ...}, {input: tensor}) of the fixture for width M."""
    g = np.load(M16)
    arrays = {k: g[k] for k in KEYS}
    if M != 16:
        g = np.load(WIDTHS)
        arrays["features"] = np.ascontiguousarray(np.roll(arrays["features"], int(g["row_shift"]), axis=0)[:, :M])
    want = {D: g[f"colors_deg{D}_{tag}"] for M_, D in PAIRS if M_ == M}
    return want, {k: torch.from_numpy(v).to(dev, dtype) for k, v in arrays.items()}


def _digests_module():
    spec = importlib.util.spec_from_file_location("make_appearance_digests", os.path.join(GOLD_DIR, "make_appearance_digests.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("M", [1, 4, 9])
def test_torch_formulation_matches_the_reference_modules_at_width(M):
    from sfgs.appearance import reference_colors
    want, t = _load(M, "cpu", torch.float64)
    assert t["features"].shape == (3000, M, 3)
    for D, ref in want.items():
        got = reference_colors(*(t[k] for k in KEYS), D)
        assert np.abs(got.numpy() - ref).max() < 1e-12, (M, D)
    f32, t = _load(M, "cpu", torch.float32, "f32")
    for D, ref in f32.items():
        got = reference_colors(*(t[k] for k in KEYS), D)
        assert np.abs(got.numpy() - ref).max() < 2e-6, (M, D)


def test_abi_rejects_unbuilt_widths_and_degrees_the_width_cannot_hold():
    # argument checks come before any pointer is read or any CUDA call is made
    from sfgs import native
    L = native.lib()

    def call(M, D):
        return L.sfgs_appearance_forward(8, D, M, None, None, 24, None, 32, None, None, None, None, None, None, None, None,
                                         None, None)
    for M in (0, 2, 5, 8, 15, 17, 25):
        assert call(M, 0) == SFGS_E_UNSUPPORTED, M
        assert "1, 4, 9 or 16" in native.last_error()
    for M, D in ((1, 1), (1, 3), (4, 2), (9, 3)):
        assert call(M, D) == SFGS_E_BADARG, (M, D)
        assert "(D+1)^2 <= M" in native.last_error()
    for M, D in PAIRS:                   # a supported pair gets as far as the pointer checks
        assert call(M, D) == SFGS_E_BADARG and "null pointer" in native.last_error(), (M, D)


@pytest.mark.gpu
@pytest.mark.parametrize("M,D", PAIRS)
def test_fused_appearance_matches_the_reference_modules_at_every_width(cuda_device, M, D):
    from sfgs.appearance import fused_appearance_colors
    want, t = _load(M, cuda_device)
    ref_all = want[D]
    full = None
    for P in (3000, 2999, 129, 128, 127, 1):
        sub = {k: (v[:P].contiguous() if k in ("features", "gemb", "xyz") else v) for k, v in t.items()}
        got = fused_appearance_colors(sub["features"], sub["gemb"], sub["aemb"], tuple(sub[k] for k in KEYS[3:9]),
                                      sub["xyz"], sub["campos"], D)
        assert got.shape == (P, 3)
        got = got.cpu().numpy()
        ref = ref_all[:P]
        err = np.abs(got.astype(np.float64) - ref)
        assert err.max() <= COLOR_ATOL, (M, D, P, float(err.max()))
        if P >= 2999:
            assert err.mean() <= 1e-5, (M, D, P, float(err.mean()))
        # zeros where the reference clamps (clamp_min(. + 0.5, 0)) except within the tolerance of the threshold
        assert np.all(got[ref == 0.0] <= COLOR_ATOL), (M, D, P)
        # each Gaussian's colour depends on its own row only, whatever tile and lane it lands in
        if full is None:
            full = got
        else:
            assert np.array_equal(got, full[:P]), (M, D, P)
    assert (ref_all == 0.0).any()        # the clamp at 0 is exercised by the fixture


@pytest.mark.gpu
def test_fused_appearance_m16_bit_identical_to_recorded_digests(cuda_device):
    Dg = _digests_module()
    with np.load(Dg.FIXTURE) as z:
        want = {k: str(z[k]) for k in z.files}
    bad = [D for D in Dg.DEGREES if Dg.digest(Dg.fused_colors(cuda_device, D)) != want[f"deg{D}"]]
    assert not bad, f"M = 16 colours at degrees {bad} differ from the recorded digests"


@pytest.mark.gpu
def test_fused_appearance_gradients_at_m4(cuda_device):
    from sfgs.appearance import fused_appearance_colors, reference_colors
    _, t = _load(4, cuda_device)
    leaves = {k: t[k].clone().requires_grad_(True) for k in KEYS if k != "campos"}
    out = fused_appearance_colors(leaves["features"], leaves["gemb"], leaves["aemb"], tuple(leaves[k] for k in KEYS[3:9]),
                                  leaves["xyz"], t["campos"], 1)
    w = torch.randn(out.shape, generator=torch.Generator().manual_seed(0)).to(cuda_device)
    (out * w).sum().backward()
    ref_leaves = {k: t[k].clone().requires_grad_(True) for k in KEYS if k != "campos"}
    (reference_colors(*(ref_leaves[k] for k in KEYS[:10]), t["campos"], 1) * w).sum().backward()
    for k in leaves:
        assert leaves[k].grad is not None and leaves[k].grad.shape == t[k].shape, k
        assert torch.allclose(leaves[k].grad, ref_leaves[k].grad, rtol=1e-5, atol=1e-7), k


@pytest.mark.gpu
def test_fused_appearance_rejects_bad_widths_and_degrees(cuda_device):
    from sfgs.appearance import fused_appearance_colors
    from sfgs.native import SfgsError
    _, t = _load(4, cuda_device)
    mlp = tuple(t[k] for k in KEYS[3:9])
    for M, D in ((1, 1), (4, 2), (4, 3)):
        f = t["features"][:, :M].contiguous()
        with pytest.raises(SfgsError, match=f"code {SFGS_E_BADARG}"):
            fused_appearance_colors(f, t["gemb"], t["aemb"], mlp, t["xyz"], t["campos"], D)
    f5 = torch.cat((t["features"], t["features"][:, :1]), dim=1)
    with pytest.raises(SfgsError, match=f"code {SFGS_E_UNSUPPORTED}"):
        fused_appearance_colors(f5, t["gemb"], t["aemb"], mlp, t["xyz"], t["campos"], 0)
