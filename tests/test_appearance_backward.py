"""The fused float32 backward of the appearance path: `sfgs_appearance_backward`, `fused_appearance_colors(...,
fused_backward=True)`.

Yardstick: the torch formulation (`reference_colors`) in float64 is the truth, and torch float32 sets the scale of an
acceptable float32 error.  For every gradient tensor the fused error against float64 may not exceed FACTOR times torch
float32's own error, in the worst element and in the mean, plus 1e-7 of the tensor's largest magnitude.  An
elementwise `allclose(rtol=1e-5, atol=1e-7)` against torch float32 is not attainable by any other float32 evaluation:
on the golden MLP (a multiplier head with h ~ 100 before the x0.01) torch float32 itself misses float64 by up to 14x
that tolerance in dL/dW2 and 2-3x in dL/dfeatures, measured on an H100.

  * CPU: the C ABI rejects bad widths, degrees, NULL inputs and misaligned rows before any CUDA work.
  * GPU: the float64 adjudication on the golden inputs at every (M, D) and ragged P, and at P = 262144 on seeded
    inputs with the Gaussians near a ReLU or clamp threshold removed; P = 0; bit-identical repeats at P = 1M; partial
    gradient requests are bit-identical to the all-gradients call and return None for the rest.
"""
import importlib.util
import os

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD_DIR = os.path.join(HERE, "golden")
KEYS = ("features", "gemb", "aemb", "W1", "b1", "W2", "b2", "W3", "b3", "xyz", "campos")
PAIRS = [(M, D) for M in (1, 4, 9, 16) for D in range(4) if (D + 1) ** 2 <= M]
SFGS_E_BADARG, SFGS_E_UNSUPPORTED = -2, -4


def _load(M, dev, dtype=torch.float32):
    """Inputs of the golden fixture at width M (tests/test_appearance_widths.py's construction)."""
    g = np.load(os.path.join(GOLD_DIR, "appearance_ref.npz"))
    arrays = {k: g[k] for k in KEYS}
    if M != 16:
        w = np.load(os.path.join(GOLD_DIR, "appearance_widths_ref.npz"))
        arrays["features"] = np.ascontiguousarray(np.roll(arrays["features"], int(w["row_shift"]), axis=0)[:, :M])
    return {k: torch.from_numpy(v).to(dev, dtype) for k, v in arrays.items()}


def _bench_module():
    spec = importlib.util.spec_from_file_location("appearance_bench", os.path.join(HERE, "appearance_bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _fused_grads(t, D, cot, needs=None):
    """Gradients of sum(cot * colours) through fused_appearance_colors(..., fused_backward=True); None where the
    input does not require grad."""
    from sfgs.appearance import fused_appearance_colors
    needs = needs or {k: True for k in KEYS}
    leaves = {k: t[k].detach().clone().requires_grad_(needs[k]) for k in KEYS}
    out = fused_appearance_colors(leaves["features"], leaves["gemb"], leaves["aemb"], tuple(leaves[k] for k in KEYS[3:9]),
                                  leaves["xyz"], leaves["campos"], D, fused_backward=True)
    (out * cot).sum().backward()
    return {k: leaves[k].grad for k in KEYS}


def _torch_grads(t, D, cot, dtype):
    from sfgs.appearance import reference_colors
    leaves = {k: t[k].detach().to(dtype).clone().requires_grad_(True) for k in KEYS}
    (reference_colors(*(leaves[k] for k in KEYS), D) * cot.to(dtype)).sum().backward()
    return {k: leaves[k].grad for k in KEYS}


# Bound factor on torch float32's error.  Arithmetic alone suggests 2: both are float32 evaluations of the same
# expression.  Measured on an H100 80GB HBM3 (700 W), the fused error is 0.7-3.4x torch's over these cases, the
# largest at P = 128-1000 on the weight gradients: the fused kernel sums a chunk's (>= 512) Gaussians sequentially in
# float32 per weight element before the float64 chunk sums, where cuBLAS blocks the reduction.  6 leaves a margin.
FACTOR = 6.0


def _adjudicate(fused, t, D, cot, what):
    """Fused float32 against float64, bounded by FACTOR x torch float32's error plus 1e-7 of the largest magnitude,
    in the worst element and in the mean.  Returns the largest (error - slack) / torch error seen."""
    f64, f32 = _torch_grads(t, D, cot, torch.float64), _torch_grads(t, D, cot, torch.float32)
    worst = 0.0
    for k in KEYS:
        if D == 0 and k in ("xyz", "campos"):
            assert fused[k] is None, (what, k)
            continue
        assert fused[k] is not None and fused[k].shape == t[k].shape and fused[k].dtype == torch.float32, (what, k)
        ref = f64[k]
        e_fused = (fused[k].double() - ref).abs()
        e_torch = (f32[k].double() - ref).abs()
        slack = 1e-7 * float(ref.abs().max())
        for red in (torch.max, torch.mean):
            ef, et = float(red(e_fused)), float(red(e_torch))
            worst = max(worst, (ef - slack) / max(et, 1e-300))
            assert ef <= FACTOR * et + slack, (what, k, red.__name__, ef, et)
    return worst


def test_abi_rejects_bad_arguments_before_any_cuda_work():
    # fake, never-dereferenced addresses: the checks run before any pointer is read or any CUDA call is made
    from sfgs import native
    L = native.lib()
    A = 1 << 20                                   # 16-byte aligned
    noop = native.ALLOC_FN(lambda _u, _n: None)

    def call(M, D, G=24, E=32, features=A, gemb=A, W2=A, dcol=A, alloc=noop):
        return L.sfgs_appearance_backward(8, D, M, features, gemb, G, A, E, A, A, W2, A, A, A, A, A, dcol,
                                          *([A] * 11), alloc, None, None)
    for M in (0, 2, 5, 8, 15, 17, 25):
        assert call(M, 0) == SFGS_E_UNSUPPORTED, M
        assert "appearance_backward" in native.last_error() and "1, 4, 9 or 16" in native.last_error()
    assert call(4, 1, G=23) == SFGS_E_UNSUPPORTED
    assert call(4, 1, E=16) == SFGS_E_UNSUPPORTED
    assert call(16, 4) == SFGS_E_UNSUPPORTED and call(16, -1) == SFGS_E_UNSUPPORTED
    for M, D in ((1, 1), (1, 3), (4, 2), (4, 3), (9, 3)):
        assert call(M, D) == SFGS_E_BADARG, (M, D)
        assert "(D+1)^2 <= M" in native.last_error()
    for M, D in PAIRS:
        assert call(M, D, W2=None) == SFGS_E_BADARG and "null pointer" in native.last_error(), (M, D)
        assert call(M, D, dcol=None) == SFGS_E_BADARG and "null pointer" in native.last_error(), (M, D)
        assert call(M, D, alloc=native.ALLOC_FN()) == SFGS_E_BADARG and "null pointer" in native.last_error(), (M, D)
        assert call(M, D, features=A + 4) == SFGS_E_BADARG and "16-byte aligned" in native.last_error(), (M, D)
        assert call(M, D, gemb=A + 8) == SFGS_E_BADARG and "16-byte aligned" in native.last_error(), (M, D)
    assert L.sfgs_appearance_backward(-1, 0, 1, *([A] * 2), 24, A, 32, *([A] * 20), noop, None, None) == SFGS_E_BADARG
    assert L.sfgs_appearance_backward_scratch_bytes(0) == 1024
    assert L.sfgs_appearance_backward_scratch_bytes(1_000_000) == 977 * 20876 * 4 + 1024


@pytest.mark.gpu
@pytest.mark.parametrize("M,D", PAIRS)
def test_fused_backward_against_float64_at_every_width(cuda_device, M, D):
    t = _load(M, cuda_device)
    gen = torch.Generator().manual_seed(100 * M + D)
    for P in (1, 127, 128, 129, 1000, 2999):
        sub = {k: (v[:P].contiguous() if k in ("features", "gemb", "xyz") else v) for k, v in t.items()}
        cot = torch.randn((P, 3), generator=gen).to(cuda_device)
        worst = _adjudicate(_fused_grads(sub, D, cot), sub, D, cot, (M, D, P))
        print(f"M={M} D={D} P={P}: largest (fused error - slack) / torch float32 error {worst:.2f}")


@pytest.mark.gpu
def test_fused_backward_with_no_gaussians_writes_zero_sums(cuda_device):
    t = _load(4, cuda_device)
    sub = {k: (v[:0].contiguous() if k in ("features", "gemb", "xyz") else v) for k, v in t.items()}
    got = _fused_grads(sub, 1, torch.zeros((0, 3), device=cuda_device))
    for k in KEYS:
        assert got[k].shape == sub[k].shape, k
        assert torch.count_nonzero(got[k]) == 0, k
        assert not torch.signbit(got[k]).any(), k


@pytest.mark.gpu
@pytest.mark.parametrize("M,D", [(4, 1), (16, 3)])
def test_fused_backward_float64_adjudication_at_256k(cuda_device, M, D):
    from sfgs.appearance import SH_C0, eval_sh_torch
    P = 262144
    t = dict(zip(KEYS, _bench_module().inputs(P, M, cuda_device)))
    # drop the Gaussians whose float64 ReLU inputs or clamp inputs lie within 1e-4 of a threshold, so that float32
    # evaluations cannot take a different branch than float64 and the comparison measures rounding alone
    d = {k: v.double() for k, v in t.items()}
    color = d["features"].reshape(P, -1)
    inp = torch.cat((color.clamp_max(1)[:, :3], d["gemb"], d["aemb"][None].expand(P, -1)), dim=-1)
    z1 = inp @ d["W1"].t() + d["b1"]
    z2 = torch.relu(z1) @ d["W2"].t() + d["b2"]
    out = (torch.relu(z2) @ d["W3"].t() + d["b3"]) * 0.01
    offset = torch.cat((out[:, :3] / SH_C0, torch.zeros_like(color[:, 3:])), dim=-1)
    tv = color.clamp_max(1) * out[:, 3:].repeat(1, M) + offset
    v = d["xyz"] - d["campos"][None]
    rgb = eval_sh_torch(D, tv.clamp_max(1).view(P, -1, 3).transpose(1, 2), v / v.norm(dim=1, keepdim=True)) + 0.5
    near = lambda x, at: ((x - at).abs() < 1e-4).any(dim=1)  # noqa: E731
    keep = ~(near(z1, 0) | near(z2, 0) | near(color, 1) | near(tv, 1) | near(rgb, 0))
    removed = int(P - keep.sum())
    print(f"M={M} D={D}: removed {removed} of {P} Gaussians near a threshold")
    assert removed < P // 4, removed
    sub = {k: (v[keep].contiguous() if k in ("features", "gemb", "xyz") else v) for k, v in t.items()}
    cot = torch.randn((int(keep.sum()), 3), generator=torch.Generator().manual_seed(7)).to(cuda_device)
    worst = _adjudicate(_fused_grads(sub, D, cot), sub, D, cot, (M, D, "262144"))
    print(f"M={M} D={D} P=262144: largest (fused error - slack) / torch float32 error {worst:.2f}")


@pytest.mark.gpu
def test_fused_backward_is_bit_reproducible_at_1m(cuda_device):
    t = dict(zip(KEYS, _bench_module().inputs(1_000_000, 4, cuda_device)))
    cot = torch.randn((1_000_000, 3), generator=torch.Generator().manual_seed(9)).to(cuda_device)
    a, b = _fused_grads(t, 1, cot), _fused_grads(t, 1, cot)
    for k in KEYS:
        assert torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)), k


@pytest.mark.gpu
@pytest.mark.parametrize("M,D", [(4, 1), (16, 3), (9, 0)])
def test_partial_gradient_requests_are_bit_identical(cuda_device, M, D):
    t = _load(M, cuda_device)
    cot = torch.randn((t["features"].shape[0], 3), generator=torch.Generator().manual_seed(3)).to(cuda_device)
    full = _fused_grads(t, D, cot)
    mlp = set(KEYS[3:9])
    cases = {
        "campos frozen": {k: k != "campos" for k in KEYS},
        "MLP frozen": {k: k not in mlp for k in KEYS},
        "only the MLP": {k: k in mlp for k in KEYS},
        "only xyz and campos": {k: k in ("xyz", "campos") for k in KEYS},
        "only W2": {k: k == "W2" for k in KEYS},
    }
    for name, needs in cases.items():
        if not any(needs[k] for k in KEYS if D > 0 or k not in ("xyz", "campos")):
            continue
        got = _fused_grads(t, D, cot, needs)
        for k in KEYS:
            if not needs[k] or (D == 0 and k in ("xyz", "campos")):
                assert got[k] is None, (name, k)
            else:
                assert torch.equal(got[k].view(torch.int32), full[k].view(torch.int32)), (name, k)
