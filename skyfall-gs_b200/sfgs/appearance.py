"""Fused appearance path (SURVEY.md 8f rank 2): `colors_precomp` of the --appearance_enabled branch of render().

    colors = fused_appearance_colors(features, gemb, aemb, mlp, xyz, campos, active_sh_degree)

replaces, in gaussian_renderer/__init__.py:105-118,

    colors_toned = pc.appearance_mlp(pc._embeddings, embedding_expanded, pc.get_features).clamp_max(1.0)
    colors_toned = colors_toned.view(-1, shdim, 3).transpose(1, 2).contiguous().clamp_max(1.0)
    dir_pp_normalized = ...; colors_toned = eval_sh(pc.active_sh_degree, colors_toned, dir_pp_normalized)
    colors_precomp = torch.clamp_min(colors_toned + 0.5, 0.0)

for any SH width the model stores: features [P, M, 3] with M = (max_sh_degree + 1)^2 = 1, 4, 9 or 16 (the README's
training commands use --sh_degree 1, M = 4), at any active degree D with (D + 1)^2 <= M.

Forward: one wgmma tensor-core kernel (csrc/sfgs_appearance.cu, `sfgs_appearance_forward`).

Backward, two choices:
  * default: the autograd function recomputes the same expression with torch ops (`reference_colors`, float32) and
    differentiates that, so the gradients are the torch formulation's, rounding included.  A training step then pays
    the fused forward on top of the torch forward and backward (DESIGN.md §7).
  * `fused_backward=True`: one float32 CUDA-core kernel (`sfgs_appearance_backward`) recomputes the forward and forms
    every requested gradient, deterministically (fixed-order float64 sums over Gaussians, no atomics).  Its gradients
    are float32-accurate — their error against float64 is at most 3.4x torch float32's own (measured, H100) — but they
    are not torch's bits: on
    a trained MLP (a multiplier head with h ~ 100 before the x0.01) the two float32 evaluations differ by up to ~15x
    rtol = 1e-5 / atol = 1e-7 in dL/dW2, because torch float32 itself misses float64 by that much (DESIGN.md §7).
"""
from __future__ import annotations

import torch

from . import native as N

SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
         1.445305721320277, -0.5900435899266435)


def eval_sh_torch(deg, sh, dirs):
    """Real SH evaluation, sh [..., 3, (deg+1)^2], dirs [..., 3] — the polynomial of utils/sh_utils.py:eval_sh."""
    result = SH_C0 * sh[..., 0]
    if deg > 0:
        x, y, z = dirs[..., 0:1], dirs[..., 1:2], dirs[..., 2:3]
        result = result - SH_C1 * y * sh[..., 1] + SH_C1 * z * sh[..., 2] - SH_C1 * x * sh[..., 3]
        if deg > 1:
            xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
            result = (result + SH_C2[0] * xy * sh[..., 4] + SH_C2[1] * yz * sh[..., 5]
                      + SH_C2[2] * (2.0 * zz - xx - yy) * sh[..., 6] + SH_C2[3] * xz * sh[..., 7] + SH_C2[4] * (xx - yy) * sh[..., 8])
            if deg > 2:
                result = (result + SH_C3[0] * y * (3 * xx - yy) * sh[..., 9] + SH_C3[1] * xy * z * sh[..., 10]
                          + SH_C3[2] * y * (4 * zz - xx - yy) * sh[..., 11] + SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * sh[..., 12]
                          + SH_C3[4] * x * (4 * zz - xx - yy) * sh[..., 13] + SH_C3[5] * z * (xx - yy) * sh[..., 14]
                          + SH_C3[6] * x * (xx - 3 * yy) * sh[..., 15])
    return result


def reference_colors(features, gemb, aemb, W1, b1, W2, b2, W3, b3, xyz, campos, deg):
    """The torch formulation (the reference's statements, scene/gaussian_model.py:60-69 and
    gaussian_renderer/__init__.py:107-117, written out on plain tensors)."""
    P = features.shape[0]
    color = features.reshape(P, -1).clamp_max(1.0)
    inp = torch.cat((color[:, :3], gemb, aemb[None].expand(P, -1)), dim=-1)
    h = torch.relu(inp @ W1.t() + b1)
    h = torch.relu(h @ W2.t() + b2)
    out = (h @ W3.t() + b3) * 0.01
    offset, mul = out[:, :3], out[:, 3:]
    offset = torch.cat((offset / SH_C0, torch.zeros_like(color[:, 3:])), dim=-1)
    mul = mul.repeat(1, color.shape[-1] // 3)
    toned = (color * mul + offset).clamp_max(1.0)
    toned = toned.view(P, -1, 3).transpose(1, 2).contiguous().clamp_max(1.0)
    d = xyz - campos[None]
    d = d / d.norm(dim=1, keepdim=True)
    return torch.clamp_min(eval_sh_torch(deg, toned, d) + 0.5, 0.0)


def _fwd(features, gemb, aemb, W1, b1, W2, b2, W3, b3, xyz, campos, deg):
    L = N.lib()
    P = int(features.shape[0])
    t = [x.contiguous().float() for x in (features, gemb, aemb, W1, b1, W2, b2, W3, b3, xyz, campos)]
    t = [x.clone() if x.data_ptr() % 16 else x for x in t]
    f, g, a, w1, bb1, w2, bb2, w3, bb3, xz, cp = t
    out = torch.empty((P, 3), dtype=torch.float32, device=features.device)
    with torch.cuda.device(features.device):
        N.check(L.sfgs_appearance_forward(P, int(deg), int(f.shape[1]), f.data_ptr(), g.data_ptr(), int(g.shape[1]),
                                          a.data_ptr(), int(a.numel()), w1.data_ptr(), bb1.data_ptr(), w2.data_ptr(),
                                          bb2.data_ptr(), w3.data_ptr(), bb3.data_ptr(), xz.data_ptr(), cp.data_ptr(),
                                          out.data_ptr(), torch.cuda.current_stream(features.device).cuda_stream),
                "sfgs_appearance_forward")
    return out


def _bwd(saved, deg, g, needs):
    """Gradients of the 11 inputs from the fused float32 kernel; None where `needs` is False (and for xyz and campos at
    degree 0, which do not reach the colours)."""
    L = N.lib()
    features = saved[0]
    P, dev = int(features.shape[0]), features.device
    needs = list(needs)
    if deg == 0:
        needs[9] = needs[10] = False
    t = [x.detach().contiguous().float() for x in saved] + [g.contiguous().float()]
    t = [x.clone() if x.data_ptr() % 16 else x for x in t]
    outs = [torch.empty(s.shape, dtype=torch.float32, device=dev) if n else None for s, n in zip(saved, needs)]
    ptr = [o.data_ptr() if o is not None else None for o in outs]
    f, ge, a, w1, bb1, w2, bb2, w3, bb3, xz, cp, gc = t
    arena = _Arena(dev)
    with torch.cuda.device(dev):
        N.check(L.sfgs_appearance_backward(P, int(deg), int(f.shape[1]), f.data_ptr(), ge.data_ptr(), int(ge.shape[1]),
                                           a.data_ptr(), int(a.numel()), w1.data_ptr(), bb1.data_ptr(), w2.data_ptr(),
                                           bb2.data_ptr(), w3.data_ptr(), bb3.data_ptr(), xz.data_ptr(), cp.data_ptr(),
                                           gc.data_ptr(), *ptr, arena.cb, None,
                                           torch.cuda.current_stream(dev).cuda_stream),
                "sfgs_appearance_backward")
    arena.tensor = None
    return [o.to(s.dtype) if o is not None else None for o, s in zip(outs, saved)]


class _Arena:
    """Scratch for the backward's allocator callback: the tensor lives until the call has been queued."""

    def __init__(self, device):
        self.device = device
        self.tensor = None
        self.cb = N.ALLOC_FN(self._alloc)

    def _alloc(self, _user, nbytes):
        try:
            self.tensor = torch.empty(int(nbytes), dtype=torch.uint8, device=self.device)
            return self.tensor.data_ptr()
        except Exception:  # noqa: BLE001 - must not raise through the C ABI
            return None


class _Appearance(torch.autograd.Function):
    @staticmethod
    def forward(ctx, features, gemb, aemb, W1, b1, W2, b2, W3, b3, xyz, campos, deg, fused_backward=False):
        ctx.deg = int(deg)
        ctx.fused_backward = bool(fused_backward)
        ctx.save_for_backward(features, gemb, aemb, W1, b1, W2, b2, W3, b3, xyz, campos)
        return _fwd(features, gemb, aemb, W1, b1, W2, b2, W3, b3, xyz, campos, deg)

    @staticmethod
    def backward(ctx, g):
        saved = ctx.saved_tensors
        needs = ctx.needs_input_grad[:11]
        if ctx.fused_backward:
            return tuple(_bwd(saved, ctx.deg, g, needs)) + (None, None)
        with torch.enable_grad():
            leaves = [s.detach().requires_grad_(n) for s, n in zip(saved, needs)]
            out = reference_colors(*leaves, ctx.deg)
            grads = torch.autograd.grad(out, [l for l, n in zip(leaves, needs) if n], g, allow_unused=True)
        it = iter(grads)
        return tuple(next(it) if n else None for n in needs) + (None, None)


def fused_appearance_colors(features, gemb, aemb, mlp, xyz, campos, active_sh_degree, *, fused_backward=False):
    """features [P,M,3] (pc.get_features, M = (pc.max_sh_degree + 1)^2 = 1, 4, 9 or 16), gemb [P,24]
    (pc._embeddings), aemb [32] (the camera's appearance embedding), mlp = pc.appearance_mlp.mlp (nn.Sequential
    Linear-ReLU-Linear-ReLU-Linear) or its six tensors; active_sh_degree D needs (D + 1)^2 <= M.  Another M, or a D
    the width cannot hold, raises native.SfgsError.  fused_backward=True differentiates with the fused float32
    kernel instead of the torch recompute (see the module docstring)."""
    if isinstance(mlp, (tuple, list)):
        W1, b1, W2, b2, W3, b3 = mlp
    else:
        W1, b1, W2, b2, W3, b3 = mlp[0].weight, mlp[0].bias, mlp[2].weight, mlp[2].bias, mlp[4].weight, mlp[4].bias
    return _Appearance.apply(features, gemb, aemb, W1, b1, W2, b2, W3, b3, xyz, campos, active_sh_degree,
                             fused_backward)
