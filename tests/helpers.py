"""Shared helpers for the parity tests (test infrastructure)."""
from __future__ import annotations

import hashlib
import os

import numpy as np
import torch

from sfgs import synthetic as S


def to_torch(scene: S.Scene, cam: S.Camera, device):
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)  # noqa: E731
    return dict(means3D=t(scene.means3D), scales=t(scene.scales), rotations=t(scene.rotations),
                opacities=t(scene.opacities), shs=t(scene.shs), viewmatrix=t(cam.viewmatrix),
                projmatrix=t(cam.projmatrix), campos=t(cam.campos))


def run_ours_forward(d, cam, sh_degree, bg, kernel_size=0.1, scale_modifier=1.0, colors=None, debug=False,
                     extras=None):
    from sfgs import rasterizer as R
    e = torch.empty(0, device=d["means3D"].device)
    sh = e if colors is not None else d["shs"]
    col = colors if colors is not None else e
    ex, ED = (extras, int(extras.shape[1])) if extras is not None else (e, 0)
    out = R.rasterize_gaussians(bg, d["means3D"], col, d["opacities"], d["scales"], d["rotations"], scale_modifier,
                                e, e, ex, ED, d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, kernel_size,
                                cam.height, cam.width, sh, sh_degree, d["campos"], False, debug)
    keys = ("num_rendered", "color", "depth", "norm", "alpha", "radii", "extra", "geom", "binning", "img")
    return dict(zip(keys, out))


def run_ours_backward(d, cam, sh_degree, bg, fwd, cot, kernel_size=0.1, scale_modifier=1.0, colors=None, debug=False,
                      extras=None, dL_extra=None, **kw):
    from sfgs import rasterizer as R
    e = torch.empty(0, device=d["means3D"].device)
    sh = e if colors is not None else d["shs"]
    col = colors if colors is not None else e
    ex = extras if extras is not None else e
    dex = dL_extra if dL_extra is not None else e
    out = R.rasterize_gaussians_backward(bg, d["means3D"], fwd["radii"], col, d["scales"], d["rotations"], ex,
                                         scale_modifier, e, e, d["viewmatrix"], d["projmatrix"], cam.tanfovx,
                                         cam.tanfovy, kernel_size, cot[0], cot[1], cot[2], cot[3], dex, sh, sh_degree,
                                         d["campos"], fwd["geom"], fwd["num_rendered"], fwd["binning"], fwd["img"],
                                         fwd["alpha"], debug, **kw)
    if kw.get("phase") == 1:
        return out                      # the [P,16] blend-adjoint sums
    keys = ("means2D", "colors", "opacity", "means3D", "cov3D", "norm3D", "sh", "scales", "rot", "extra")
    return dict(zip(keys, out))


def run_ref_forward(d, cam, sh_degree, bg, kernel_size=0.1, scale_modifier=1.0, colors=None):
    from oracle import ref_cuda
    e = torch.empty(0, device=d["means3D"].device)
    sh = e if colors is not None else d["shs"]
    col = colors if colors is not None else e
    return ref_cuda.forward(bg, d["means3D"], col, d["opacities"], d["scales"], d["rotations"], scale_modifier, e, e,
                            e, d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, kernel_size, cam.height,
                            cam.width, sh, sh_degree, d["campos"])


def run_ref_backward(d, cam, sh_degree, bg, fwd, cot, kernel_size=0.1, scale_modifier=1.0, colors=None):
    from oracle import ref_cuda
    e = torch.empty(0, device=d["means3D"].device)
    sh = e if colors is not None else d["shs"]
    col = colors if colors is not None else e
    return ref_cuda.backward(bg, d["means3D"], fwd["radii"], col, d["scales"], d["rotations"], e, scale_modifier, e,
                             e, d["viewmatrix"], d["projmatrix"], cam.tanfovx, cam.tanfovy, kernel_size, cot[0],
                             cot[1], cot[2], cot[3], e, sh, sh_degree, d["campos"], fwd["geom"],
                             fwd["num_rendered"], fwd["binning"], fwd["img"], fwd["alpha"])


def our_internals(fwd, P, H, W):
    """Unpack this library's scratch buffers into the reference's vocabulary."""
    import ctypes as C
    from sfgs import native as N
    L = N.lib()
    dev = fwd["geom"].device
    gv, iv, bv = N.GeomView(), N.ImageView(), N.BinningView()
    N.check(L.sfgs_geom_layout(fwd["geom"].data_ptr(), P, C.byref(gv)), "geom_layout")
    N.check(L.sfgs_image_layout(fwd["img"].data_ptr(), W, H, C.byref(iv)), "image_layout")
    # the binning layout depends on the capacity THIS forward used; it is recorded in the image header (words 2,3)
    hdr = fwd["img"][:32].view(torch.int32).cpu().numpy().astype(np.uint32)
    assert fwd["img"].data_ptr() % 256 == 0
    cap = int(hdr[2]) | (int(hdr[3]) << 32)
    N.check(L.sfgs_binning_layout(fwd["binning"].data_ptr(), cap, C.byref(bv)), "binning_layout")
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    R = fwd["num_rendered"]

    def view(ptr, base_t, shape, dtype):
        off = ptr - base_t.data_ptr()
        n = int(np.prod(shape)) * torch.empty(0, dtype=dtype).element_size()
        return base_t[off:off + n].view(dtype).view(*shape).clone()

    rec = view(gv.rec, fwd["geom"], (P, 16), torch.float32)
    out = dict(rec=rec, means2D=rec[:, 0:2], conic_opacity=torch.cat([rec[:, 2:5], rec[:, 5:6]], 1),
               depths=rec[:, 6], rgb=rec[:, 8:11], norm3D=rec[:, 11:14],
               cov3D=view(gv.cov3D, fwd["geom"], (P, 6), torch.float32),
               clamped=view(gv.clamped, fwd["geom"], (P,), torch.uint8),
               tiles_touched=view(gv.tiles_touched, fwd["geom"], (P,), torch.int32),
               n_contrib=view(iv.n_contrib, fwd["img"], (H * W,), torch.int32),
               ranges=view(iv.ranges, fwd["img"], (tiles, 2), torch.int32),
               keys=view(bv.keys, fwd["binning"], (R,), torch.int64),
               point_list=view(bv.point_list, fwd["binning"], (R,), torch.int32))
    return out


def ref_style_keys(ranges, keys_depth_id):
    """Rebuild the reference's (tile << 32 | depth_bits) keys from our per-tile (depth_bits << 32 | id) keys."""
    R = keys_depth_id.shape[0]
    counts = (ranges[:, 1] - ranges[:, 0]).long()
    tile_of = torch.repeat_interleave(torch.arange(ranges.shape[0], device=ranges.device), counts)
    assert tile_of.shape[0] == R
    depth_bits = (keys_depth_id >> 32) & 0xFFFFFFFF
    return (tile_of << 32) | depth_bits


# ----------------------------------------------------------------------------- float64-adjudicated gradient parity
# Our error against the float64 values may be at most this multiple of the reference CUDA build's own error against
# them, per gradient tensor.  The bulk statistics (mean, 99.9th percentile) are held to tight factors; the worst
# single element is an extreme-value statistic of a heavy-tailed error distribution (the ill-conditioned covariance /
# rotation chain) and is compared with the worst element of the reference over several of its (non-deterministic)
# runs, with a wider factor.  Nothing is exempt: the maximum is over every element.
ADJ_FACTORS = {"mean": 1.5, "p999": 2.0, "max": 4.0}
ADJ_FLOOR = 1e-5      # north_star: 1e-5 abs on gradient tensors


def adjudicate_gradients(d, cam, sh_degree, bg, I, out_alpha, radii, cot, ours, ref, tag, kernel_size=0.1,
                         scale_modifier=1.0, colors=None, factors=None, floor=ADJ_FLOOR, ref_stats=None):
    """The gradient gate of the parity tests.

    The reference's backward is itself an approximation (float atomics in a run-dependent order, transmittance
    recovered by repeated float division), so `|ours - ref|` cannot say whose error a deviation is.  The float64
    adjudicator (oracle/adjudicator_f64.cu: the reference's algorithm in double with the float32 control flow)
    can: for every gradient tensor the error of this library against the float64 values must not exceed
    ADJ_FACTORS x the reference CUDA build's own error against them (+ the 1e-5 absolute floor of the north star)
    in the mean, at the 99.9th percentile and in the worst element.  No element is exempt.

    I: forward intermediates in the reference's vocabulary (oracle.ref_cuda.internals or helpers.our_internals).
    ref: one run of the reference's gradients, or a list of runs (every statistic: the largest over the runs).
    ours: one run of this library's gradients, or a list of runs (mean / p99.9: the largest over the runs; the worst
    element: the median over the runs — see oracle.adjudicator.error_report).
    ref_stats: instead of `ref`, the reference build's statistics per tensor as stored by RefFacts.adjudicate.
    Returns the report."""
    from oracle import adjudicator as A
    factors = factors or ADJ_FACTORS
    f64 = A.backward_f64(I, d["means3D"], radii, d["shs"], d["scales"], d["rotations"], scale_modifier,
                         d["viewmatrix"], d["projmatrix"], d["campos"], cam.tanfovx, cam.tanfovy, kernel_size,
                         sh_degree, bg, out_alpha, cot, colors_precomp=colors)
    keys = [k for k in A.GRAD_KEYS if not (colors is not None and k == "sh")]
    rep = A.error_report(ours, ref, f64, keys)
    if ref_stats is not None:
        for k in rep:
            rep[k]["ref"] = ref_stats[k]
    print(f"\n[adjudication] {tag}\n" + A.format_report(rep))
    failures = []
    for k, r in rep.items():
        for stat, factor in factors.items():
            lim = factor * r["ref"][stat] + floor
            if not r["ours"][stat] <= lim:
                failures.append(f"{k}.{stat}: ours {r['ours'][stat]:.3e} > {factor} x ref {r['ref'][stat]:.3e} + {floor}")
    assert not failures, f"{tag}: " + "; ".join(failures)
    return rep


# ----------------------------------------------------------------------------- recorded reference facts
REF_FACTS_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference")
SAMPLE = 8192          # elements of a tolerance-compared tensor kept per fact


def _canon(t):
    """Bytes that identify a tensor's values exactly: float32 as their bit patterns, everything widened to int64."""
    t = t.detach().contiguous()
    if t.dtype.is_floating_point:
        t = t.float().view(torch.int32)
    return t.to(torch.int64).cpu().numpy().tobytes() + str(tuple(t.shape)).encode()


def _sample_index(n, name):
    seed = int.from_bytes(hashlib.sha256(name.encode()).digest()[:8], "little")
    return np.sort(np.random.default_rng(seed).choice(n, size=min(n, SAMPLE), replace=False))


class RefFacts:
    """What a parity test compares against the original rasterizer, kept small enough to live in the repository.

    Live (the original's CUDA build is in oracle/_ref): every comparison runs against the original's values, and with
    SFGS_RECORD_REFERENCE=1 what it compared against is stored in tests/golden/reference/<tag>.npz.  Replay (no
    original build): the stored facts stand in for it.  A quantity compared bit for bit is stored as the SHA-256 digest
    of its values, so replay still compares it bit for bit; a quantity compared within a tolerance as its values at a
    fixed seeded sample of elements; a scalar as itself; a gradient comparison as the original build's error
    statistics against the float64 adjudicator (helpers.adjudicate_gradients)."""

    def __init__(self, tag, live=None):
        from oracle import ref_cuda
        self.tag = tag
        self.path = os.path.join(REF_FACTS_DIR, tag + ".npz")
        self.live = ref_cuda.available() if live is None else live
        self.record = self.live and os.environ.get("SFGS_RECORD_REFERENCE") == "1"
        self.facts = {}
        if not self.live:
            assert os.path.exists(self.path), f"no recorded reference facts for {tag} ({self.path})"
            with np.load(self.path) as z:
                self.facts = {k: z[k] for k in z.files}

    def _put(self, key, value):
        if self.record:
            self.facts[key] = np.asarray(value)
            os.makedirs(REF_FACTS_DIR, exist_ok=True)
            np.savez_compressed(self.path, **self.facts)

    def value(self, name, fn):
        """A number of the original's run: computed by `fn` when live, else the stored one."""
        if self.live:
            v = fn()
            self._put("value/" + name, v)
            return v
        return self.facts["value/" + name].item()

    def same(self, name, ours, ref_fn):
        """`ours` equals the original's tensor bit for bit."""
        if self.live:
            ref = ref_fn()
            ok = _canon(ours) == _canon(ref)
            self._put("same/" + name, hashlib.sha256(_canon(ref)).hexdigest())
        else:
            ok = hashlib.sha256(_canon(ours)).hexdigest() == str(self.facts["same/" + name])
        assert ok, f"{self.tag}: {name} differs from the original"

    def close(self, name, ours, ref_fn, atol, rtol=0.0):
        """|ours - original| <= atol + rtol |original| (every element live; the stored sample on replay)."""
        o = ours.detach().reshape(-1).double()
        idx = _sample_index(o.numel(), self.tag + "/" + name)
        if self.live:
            ref = ref_fn().detach().reshape(-1).double()
            self._put("close/" + name, ref[torch.from_numpy(idx).to(ref.device)].float().cpu().numpy())
        else:
            ref = torch.from_numpy(self.facts["close/" + name]).to(o.device)
            o = o[torch.from_numpy(idx).to(o.device)]
        err = float(((o - ref).abs() - rtol * ref.abs()).max()) if o.numel() else 0.0
        assert err <= atol, (self.tag, name, err, atol)

    def adjudicate(self, d, cam, sh_degree, bg, I_ours, out_alpha, radii, cot, ours, ref_fn, tag, **kw):
        """helpers.adjudicate_gradients against the original's gradient runs (`ref_fn` returns (internals, out_alpha,
        radii, list of runs)) when live; against its stored error statistics, on this library's forward intermediates
        (asserted bit-identical on indexing by the caller), on replay."""
        if self.live:
            I, alpha, rad, runs = ref_fn()
            rep = adjudicate_gradients(d, cam, sh_degree, bg, I, alpha, rad, cot, ours, runs, tag, **kw)
            for k, r in rep.items():
                for stat, v in r["ref"].items():
                    self._put(f"adj/{k}/{stat}", v)
            return rep
        stats = {}
        for key, v in self.facts.items():
            if key.startswith("adj/"):
                _, k, stat = key.split("/")
                stats.setdefault(k, {})[stat] = float(v)
        return adjudicate_gradients(d, cam, sh_degree, bg, I_ours, out_alpha, radii, cot, ours, None, tag,
                                    ref_stats=stats, **kw)
