"""The fused appearance forward (`sfgs_appearance_forward`) at training scale, against a per-element float64 bound.

The kernel is persistent: a grid of min(ceil(ntiles / 2), #SMs) CTAs, two warpgroups each, every warpgroup looping over
128-row tiles (`tile += gridDim.x * 2`).  With T = 2 * #SMs * 128 rows every warpgroup runs exactly one tile, so the
other fused-appearance tests (P <= 3000) never reach a second loop iteration, the reuse of a group's operand and h3
buffers across tiles, a prefetch of a tile that is then computed, or a ragged tile that is not a group's first.

Yardstick: `colour_bound` bounds |fused - float64| per colour, a priori, from the kernel's arithmetic (split-bf16
operands, fp32 tensor-core accumulation, float32 tail); the float64 truth is `reference_colors` in float64.  An element
past its bound is a defect, not rounding.

  * CPU: a torch emulation of the kernel's numeric scheme stays within the bound; one that drops the Al.Wh products
    does not.
  * GPU: every element within the bound, and the documented max <= 1e-4 / mean <= 1e-5, at P = T, T + 1,
    T + 128 #SMs + 77 for every (M, D) and at 1M and 1M + 3 for (4, 1) and (16, 3), on seeded inputs and on the golden
    MLP with tiled, perturbed golden rows; bit-identical colours when rows move by whole tiles, for prefixes and for
    repeats; no write past the P-th colour.
"""
import importlib.util
import os

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD_DIR = os.path.join(HERE, "golden")
KEYS = ("features", "gemb", "aemb", "W1", "b1", "W2", "b2", "W3", "b3", "xyz", "campos")
ROWS = ("features", "gemb", "xyz")
PAIRS = [(M, D) for M in (1, 4, 9, 16) for D in range(4) if (D + 1) ** 2 <= M]
COLOR_ATOL, COLOR_MEAN = 1e-4, 1e-5       # the bar of tests/test_appearance.py
TILE = 128
P_1M = (1_000_000, 1_000_003)

# ---- the bound ---------------------------------------------------------------------------------------------------
# Float32 unit roundoff; bf16 keeps 8 significant bits, so round-to-nearest leaves |x - bf16(x)| <= 2^-8 |x|.
U32 = 2.0 ** -24
# Split operand x = hi + lo, hi = bf16(x), lo = bf16(x - hi) (x - hi is exact in float32):
# |x - hi - lo| <= 2^-8 |x - hi| <= 2^-16 |x|.
SPLIT = 2.0 ** -16
# The kernel forms A W as Ah Wh + Ah Wl + Al Wh and drops Al Wl: |Al| <= 2^-8 (1 + 2^-8) |a|, the same for |Wl|.
DROP = 2.0 ** -16 * (1 + 2.0 ** -8) ** 2
# Tensor-core accumulation: each m64nNk16 MMA adds 16 exact products to the fp32 accumulator.  Hopper's adder is not
# an IEEE fp32 add; assume the worst plausible one: the 16 products and the accumulator aligned to the largest
# exponent and truncated to 24 bits (< 2^-23 of the largest magnitude lost per addend, 17 addends), then the sum
# rounded (2^-23).  The largest magnitude is at most the running sum of |terms|, so each MMA costs at most
# 18 * 2^-23 sum |a||w|, and a layer over K runs 3 K / 16 MMAs: 3.4 K * 2^-23, above the K * 2^-23 of an IEEE chain.
ACC_PER_MMA = 18 * 2.0 ** -23


def gamma(K):
    """Relative error, against sum_k |a_k w_k| + |b|, of one split-bf16 layer over K (padded) inputs: both operands'
    splits, the dropped Al Wl, the accumulation (the three products sum to at most (1 + 2^-7) |a w|), and float32
    roundings outside the MMA: the bias add (1) and, in layer 1, the once-per-CTA fold of the embedding columns into
    the bias (32 fmaf)."""
    return 2 * SPLIT + DROP + ACC_PER_MMA * 3 * (K // 16) * (1 + 2.0 ** -7) + 33 * U32


# eval_sh basis k (utils/sh_utils.py) as a polynomial in the unit direction: polynomial degree and the sum of the
# absolute values of its monomial coefficients (with the SH constant), which bound its change per unit change of any
# component and the size of every intermediate of its float32 evaluation.
def _sh_tables():
    from sfgs.appearance import SH_C0, SH_C1, SH_C2, SH_C3
    a = [SH_C0, SH_C1, SH_C1, SH_C1, abs(SH_C2[0]), abs(SH_C2[1]), 4 * SH_C2[2], abs(SH_C2[3]), 2 * SH_C2[4],
         4 * abs(SH_C3[0]), SH_C3[1], 6 * abs(SH_C3[2]), 8 * SH_C3[3], 6 * abs(SH_C3[4]), 2 * SH_C3[5], 4 * abs(SH_C3[6])]
    deg = [0, 1, 1, 1, 2, 2, 2, 2, 2, 3, 3, 3, 3, 3, 3, 3]
    return a, deg


# float32 direction d = v / |v|: v = xyz - campos (1 rounding), |v|^2 (3, plus 2 from v), IEEE sqrtf (halves the
# relative error, +1), IEEE 1 / r (+1), v * inv (+1): each component within 6.5 U32 of the unit vector's.
EPS_DIR = 6.5 * U32


def colour_bound(t, D, chunk=1 << 16):
    """Per-element bound [P, 3] (float64, on t's device) on |fused colour - float64 colour| for inputs t (KEYS ->
    float32 tensors, features [P, M, 3]) at active SH degree D.

    MLP: each layer's own error is eps_l <= gamma_l (|W_l| |a_{l-1}| + |b_l|) (|a| from the float64 forward, widened by
    the naive running bound below, so the kernel's own activations are covered).  It reaches the layer-3 output h
    through the float64 Jacobian:  |dh| <= eps_3 + |W3| S2 eps_2 + |W3 S2 W2| S1 eps_1, S_l = the layer's ReLU mask.
    A unit whose float64 input lies within the naive bound of zero may switch sides in the kernel; ReLU is
    1-Lipschitz, so such a unit passes its error with an unknown factor in [0, 1]: it counts in S_l, and its term of
    W3 S2 W2 is bounded in absolute value.  The naive bound e_l = gamma_l (|W_l| |a| + |b_l|) + (1 + gamma_l) |W_l| e_{l-1}
    (worst-case signs everywhere) decides which units are uncertain.

    Tail (float32, per element): mul = 0.01 (h + b3)[3:] and off = 0.01 (h + b3)[:3] / C0 carry 0.01 |dh| (/ C0) and
    3 (5) roundings of the float32 constants and operations; toned tv = min(f, 1) mul + off (DC only), two roundings;
    the clamps are 1-Lipschitz; rgb = sum_k bas_k tv_k + 0.5 by fmaf, (D + 1)^2 + 1 roundings of at most
    sum_k |bas_k tv_k| + 0.5; the basis itself is off by at most deg_k EPS_DIR + (2 deg_k + 4) U32 times its
    coefficient sum.  Second-order terms (products of two relative errors, <= 2^-12 of the first-order ones) are
    covered by a factor 1 + 2^-10."""
    from sfgs.appearance import SH_C0, eval_sh_torch
    d = {k: v.double() for k, v in t.items()}
    P, M = d["features"].shape[:2]
    dev = d["features"].device
    W1, W2, W3 = d["W1"], d["W2"], d["W3"]
    aW1, aW2, aW3 = W1.abs(), W2.abs(), W3.abs()
    g1, g2 = gamma(32), gamma(128)
    sh_a, sh_deg = _sh_tables()
    n = (D + 1) ** 2
    coef = torch.tensor(sh_a[:n], dtype=torch.float64, device=dev)
    deg = torch.tensor(sh_deg[:n], dtype=torch.float64, device=dev)
    e_bas = coef * (deg * EPS_DIR + (2 * deg + 4) * U32)
    out = []
    for r0 in range(0, P, chunk):
        color = d["features"][r0:r0 + chunk].reshape(-1, 3 * M).clamp_max(1.0)
        R = color.shape[0]
        x0 = torch.cat((color[:, :3], d["gemb"][r0:r0 + chunk], d["aemb"][None].expand(R, -1)), dim=-1)
        z1 = x0 @ W1.t() + d["b1"]
        a1 = z1.relu()
        z2 = a1 @ W2.t() + d["b2"]
        a2 = z2.relu()
        # naive running bound: local errors, then worst-case propagation through |W|
        eps1 = g1 * (x0.abs() @ aW1.t() + d["b1"].abs())
        n1 = eps1
        eps2 = g2 * ((a1 + n1) @ aW2.t() + d["b2"].abs())
        n2 = eps2 + (1 + g2) * (n1 @ aW2.t())
        eps3 = g2 * ((a2 + n2) @ aW3.t() + d["b3"].abs())
        on1, unsure1 = (z1 > n1).double(), (z1.abs() <= n1).double()
        on2, unsure2 = (z2 > n2).double(), (z2.abs() <= n2).double()
        s1, s2 = on1 + unsure1, on2 + unsure2
        J = (W3[None] * on2[:, None]) @ W2                       # [R, 6, 128]: d h / d z1 through the sure units
        dh = (eps3 + (s2 * eps2) @ aW3.t() + (J.abs() @ (s1 * eps1)[..., None])[..., 0]
              + (unsure2 * ((s1 * eps1) @ aW2.t())) @ aW3.t())
        h = a2 @ W3.t() + d["b3"]
        mul, off = 0.01 * h[:, 3:], 0.01 * h[:, :3] / SH_C0
        e_mul = 0.01 * dh[:, 3:] + 3 * U32 * mul.abs()            # one error per channel, shared by its coefficients
        e_off = 0.01 / SH_C0 * dh[:, :3] + 5 * U32 * off.abs()
        fc = color.view(R, M, 3)[:, :n]
        tv = fc * mul[:, None]
        e_round = 2 * U32 * tv.abs()
        tv[:, 0] += off
        e_round[:, 0] += 2 * U32 * off.abs()
        e_tv = fc.abs() * e_mul[:, None] + e_round
        e_tv[:, 0] += e_off
        # clamp_max(1) passes tv's error where tv + e_tv < 1, none where tv - e_tv > 1, a part of it in between
        below, unsure = (tv + e_tv < 1).double(), ((tv - 1).abs() <= e_tv).double()
        v = d["xyz"][r0:r0 + chunk] - d["campos"][None]
        bas = eval_sh_torch(D, torch.eye(n, dtype=torch.float64, device=dev).expand(R, n, n),
                            v / v.norm(dim=1, keepdim=True))[..., None]                 # [R, n, 1]: basis k
        tvc = tv.clamp_max(1.0).abs()
        e_rgb = (e_mul * ((bas * fc * below).sum(1).abs() + (bas * fc * unsure).abs().sum(1))
                 + e_off * bas[:, 0].abs() * (below[:, 0] + unsure[:, 0])
                 + (bas.abs() * e_round * (below + unsure)).sum(1)
                 + (e_bas[None, :, None] * tvc).sum(1) + (n + 1) * U32 * ((bas.abs() * tvc).sum(1) + 0.5))
        out.append((1 + 2.0 ** -10) * e_rgb)
    return torch.cat(out)


# ---- inputs ------------------------------------------------------------------------------------------------------
def _bench_module():
    spec = importlib.util.spec_from_file_location("appearance_bench", os.path.join(HERE, "appearance_bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _golden(M):
    """The golden fixture at width M (tests/test_appearance_widths.py's construction), float32 numpy arrays."""
    g = np.load(os.path.join(GOLD_DIR, "appearance_ref.npz"))
    arrays = {k: g[k] for k in KEYS}
    if M != 16:
        w = np.load(os.path.join(GOLD_DIR, "appearance_widths_ref.npz"))
        arrays["features"] = np.ascontiguousarray(np.roll(arrays["features"], int(w["row_shift"]), axis=0)[:, :M])
    return arrays


def _inputs(family, P, M, dev):
    """"bench": appearance_bench.inputs (seeded, freshly initialised MLP).  "golden": the golden MLP, embedding and
    camera, the golden rows tiled up to P with seeded perturbations, so that every row is distinct."""
    if family == "bench":
        return dict(zip(KEYS, _bench_module().inputs(P, M, dev)))
    g = _golden(M)
    idx = torch.arange(P) % g["features"].shape[0]
    gen = torch.Generator().manual_seed(1000 * M + P % 1000)
    rows = {k: torch.from_numpy(g[k])[idx] for k in ROWS}
    rows["features"] = rows["features"] * (1 + 0.02 * torch.randn(rows["features"].shape, generator=gen))
    rows["gemb"] = (rows["gemb"] + 0.02 * torch.randn(rows["gemb"].shape, generator=gen)).clamp(-1, 1)
    rows["xyz"] = rows["xyz"] + torch.randn(rows["xyz"].shape, generator=gen)
    t = {k: torch.from_numpy(g[k]) for k in KEYS if k not in ROWS}
    t.update(rows)
    return {k: t[k].contiguous().to(dev) for k in KEYS}


# ---- CPU: the bound against an emulation of the kernel's arithmetic ---------------------------------------------
def _emulate(t, D, drop_lh=False):
    """The kernel's numeric scheme in torch float32: split-bf16 operands, three products per layer (two when drop_lh:
    Al Wh missing), the embedding folded into b1 in float32, then the float32 tone map and eval_sh."""
    from sfgs.appearance import SH_C0, eval_sh_torch

    def split(x):
        hi = x.bfloat16().float()
        return hi, (x - hi).bfloat16().float()

    def layer(a, W):
        (ah, al), (wh, wl) = split(a), split(W)
        r = ah @ wh.t() + ah @ wl.t()
        return r if drop_lh else r + al @ wh.t()

    f = t["features"]
    P, M = f.shape[:2]
    color = f.reshape(P, -1).clamp_max(1.0)
    b1 = t["b1"] + t["W1"][:, 27:] @ t["aemb"]
    a = torch.relu(layer(torch.cat((color[:, :3], t["gemb"]), dim=-1), t["W1"][:, :27]) + b1)
    a = torch.relu(layer(a, t["W2"]) + t["b2"])
    h = layer(a, t["W3"]) + t["b3"]
    offset = torch.cat((h[:, :3] * 0.01 / SH_C0, torch.zeros_like(color[:, 3:])), dim=-1)
    toned = (color * (h[:, 3:] * 0.01).repeat(1, M) + offset).clamp_max(1.0).view(P, M, 3).transpose(1, 2)
    v = t["xyz"] - t["campos"][None]
    return torch.clamp_min(eval_sh_torch(D, toned, v / v.norm(dim=1, keepdim=True)) + 0.5, 0.0)


@pytest.mark.parametrize("M,D", PAIRS)
def test_bound_holds_for_the_split_bf16_emulation_and_not_without_al_wh(M, D):
    from sfgs.appearance import reference_colors
    worst = 0.0
    for family in ("golden", "bench"):
        t = ({k: torch.from_numpy(v) for k, v in _golden(M).items()} if family == "golden"
             else dict(zip(KEYS, _bench_module().inputs(4096, M, "cpu"))))
        ref = reference_colors(*(t[k].double() for k in KEYS), D)
        bound = colour_bound(t, D)
        ok = float(((_emulate(t, D).double() - ref).abs() / bound).max())
        dropped = float(((_emulate(t, D, drop_lh=True).double() - ref).abs() / bound).max())
        print(f"{family} M={M} D={D}: worst err / bound {ok:.4f} split-bf16, {dropped:.2f} without Al.Wh")
        assert ok <= 1.0, (family, ok)
        assert dropped > 1.0, (family, dropped)
        worst = max(worst, ok)
    assert worst >= 0.01, worst          # the bound is not vacuous


# ---- GPU: the fused forward past the persistent loop's first tile -----------------------------------------------
@pytest.fixture(scope="module")
def n_sm(cuda_device):
    return torch.cuda.get_device_properties(cuda_device).multi_processor_count


def _first_pass(n_sm):
    """Rows that one pass of the persistent grid covers: every warpgroup of every CTA runs one 128-row tile."""
    return 2 * n_sm * TILE


def _fused(t, D):
    from sfgs.appearance import fused_appearance_colors
    with torch.no_grad():
        return fused_appearance_colors(t["features"], t["gemb"], t["aemb"], tuple(t[k] for k in KEYS[3:9]), t["xyz"],
                                       t["campos"], D)


def _check_against_float64(t, D, what):
    """Every colour within colour_bound of the float64 truth, plus the flat bar; prints the case's numbers."""
    from sfgs.appearance import reference_colors
    got = _fused(t, D)
    ref = reference_colors(*(t[k].double() for k in KEYS), D)
    err = (got.double() - ref).abs()
    ratio = float((err / colour_bound(t, D)).max())
    emax, emean = float(err.max()), float(err.mean())
    print(f"{what}: max {emax:.3e} mean {emean:.3e} worst err / bound {ratio:.4f}")
    assert ratio <= 1.0, (what, ratio)
    assert emax <= COLOR_ATOL, (what, emax)
    assert emean <= COLOR_MEAN, (what, emean)
    clamped = got[ref == 0]
    assert clamped.numel() == 0 or float(clamped.max()) <= COLOR_ATOL, what
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["bench", "golden"])
@pytest.mark.parametrize("M,D", PAIRS)
def test_fused_forward_within_bound_past_the_first_tile(cuda_device, n_sm, family, M, D):
    T = _first_pass(n_sm)
    # T: one tile per warpgroup; T + 1: one group runs a second, one-row tile; + 128 n_sm + 77: ragged second tiles
    for P in (T, T + 1, T + TILE * n_sm + 77):
        _check_against_float64(_inputs(family, P, M, cuda_device), D, f"{family} P={P} M={M} D={D}")


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["bench", "golden"])
@pytest.mark.parametrize("M,D", [(4, 1), (16, 3)])
def test_fused_forward_within_bound_at_1m(cuda_device, family, M, D):
    for P in P_1M:
        _check_against_float64(_inputs(family, P, M, cuda_device), D, f"{family} P={P} M={M} D={D}")


# ---- GPU: bitwise invariants that expose state carried from one tile to the next ----------------------------------
def _bits(x):
    return x.contiguous().view(torch.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("M,D", [(4, 1), (16, 3)])
def test_rows_moved_by_whole_tiles_give_bit_identical_colours(cuda_device, n_sm, M, D):
    P = P_1M[1]
    t = _inputs("bench", P, M, cuda_device)
    base = _bits(_fused(t, D))
    for shift in (TILE, TILE * n_sm, TILE * (2 * n_sm + 1), TILE * n_sm + 37):
        moved = dict(t, **{k: torch.roll(t[k], shift, dims=0) for k in ROWS})
        got = _bits(torch.roll(_fused(moved, D), -shift, dims=0))
        # row i lands on row i + shift: the same lane of another tile, group, CTA and loop iteration when the shift is
        # a multiple of 128 and the row does not wrap around; wrapped rows and other shifts change the MMA row
        same_lane = slice(0, P - shift) if shift % TILE == 0 else slice(0, 0)
        assert torch.equal(got[same_lane], base[same_lane]), (M, D, shift)
        print(f"M={M} D={D} roll {shift}: rows keeping their lane bit-identical; rows changing MMA row "
              f"{'bit-identical' if torch.equal(got, base) else 'NOT bit-identical'}")


@pytest.mark.gpu
@pytest.mark.parametrize("M,D", [(4, 1), (16, 3)])
def test_prefixes_and_repeats_at_1m_are_bit_identical(cuda_device, n_sm, M, D):
    P = P_1M[0]
    t = _inputs("bench", P, M, cuda_device)
    full = _bits(_fused(t, D))
    assert torch.equal(full, _bits(_fused(t, D))), (M, D)
    T = _first_pass(n_sm)
    for Pp in (T, T + 1):
        sub = {k: (v[:Pp].contiguous() if k in ROWS else v) for k, v in t.items()}
        assert torch.equal(_bits(_fused(sub, D)), full[:Pp]), (M, D, Pp)


# ---- GPU: no write past the P-th colour ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("M,D", [(4, 1), (9, 2)])
def test_no_write_past_the_last_colour(cuda_device, n_sm, M, D):
    from sfgs import native as N
    L = N.lib()
    for P in (_first_pass(n_sm) + 1, P_1M[1]):
        t = {k: v.clone() for k, v in _inputs("golden", P, M, cuda_device).items()}      # exactly P rows
        want = _bits(_fused(t, D)).reshape(-1)
        buf = torch.full((3 * P + 3 * 256,), 0x7FA5A5A5, dtype=torch.int32, device=cuda_device)
        f, g, a, w1, b1, w2, b2, w3, b3, xz, cp = (t[k] for k in KEYS)
        with torch.cuda.device(cuda_device):
            N.check(L.sfgs_appearance_forward(P, D, M, f.data_ptr(), g.data_ptr(), int(g.shape[1]), a.data_ptr(),
                                              int(a.numel()), w1.data_ptr(), b1.data_ptr(), w2.data_ptr(),
                                              b2.data_ptr(), w3.data_ptr(), b3.data_ptr(), xz.data_ptr(),
                                              cp.data_ptr(), buf.data_ptr(),
                                              torch.cuda.current_stream(cuda_device).cuda_stream),
                    "sfgs_appearance_forward")
        torch.cuda.synchronize(cuda_device)
        assert torch.equal(buf[:3 * P], want), (M, D, P)
        assert bool((buf[3 * P:] == 0x7FA5A5A5).all()), (M, D, P)
