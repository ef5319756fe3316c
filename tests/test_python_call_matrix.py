"""The rasterizer's Python layer, pinned call by call (CPU).

`test_entry_rejections.py` pins which C checks an entry runs; this pins which entry the Python layer above it reaches.
The native library is replaced by a recorder whose every function records its call and returns 5, and tensors stay on
the CPU.  For every combination of options of `sfgs.rasterizer.rasterize_gaussians[_backward]`, and for
`diff_gauss.GaussianRasterizer`, `sfgs.ortho.OrthoRasterizer` and `render_height_map`, forward and backward, the table
holds what the call did:

- each native call: the entry, its scalar arguments (`*` for a pointer, `0` for NULL), the scalar fields of
  `ForwardArgs` / `BackwardArgs` and which of their pointer fields are NULL;
- the returned tuple (and the leaves' gradients): lengths, shapes and dtypes;
- or the Python-layer rejection: its type and message.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import itertools
import types

import pytest
import torch

H, W, P = 8, 8, 4


class _Recorder:
    """A stand-in for the loaded libsfgs.so: every function records (entry, args) and returns 5."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if not name.startswith("sfgs_"):
            raise AttributeError(name)
        return lambda *a: self.calls.append(_native_record(name, a)) or 5


def _struct_record(s):
    scalars, nulls = [], []
    for name, typ in s._fields_:
        if name in ("stream",) or name.endswith("_alloc") or name.endswith("_user"):
            continue
        v = getattr(s, name)
        if typ in (C.c_int, C.c_longlong):
            scalars.append(f"{name}={v}")
        elif typ is C.c_float:
            scalars.append(f"{name}={v:.9g}")
        elif not v:
            nulls.append(name)
    return " ".join(scalars) + " null=" + ",".join(nulls)


def _native_record(name, args):
    parts = []
    for x in args[1:]:
        if x is None:
            parts.append("0")
        elif isinstance(x, float):
            parts.append(f"{x:.9g}")
        elif isinstance(x, int) and abs(x) < 1 << 16:
            parts.append(str(x))
        else:
            parts.append("*")
    return f"{name}({', '.join(parts)}) | {_struct_record(args[0]._obj)}"


def _describe(x):
    if isinstance(x, torch.Tensor):
        return f"{str(x.dtype)[6:]}{list(x.shape)}"
    if isinstance(x, (tuple, list)):
        return "(" + ", ".join(_describe(y) for y in x) + ")"
    return repr(x)


@pytest.fixture
def recorder(monkeypatch):
    from sfgs import graphs
    from sfgs import native as N
    from sfgs import rasterizer as R
    rec = _Recorder()
    monkeypatch.setattr(N, "lib", lambda: rec)
    monkeypatch.setattr(R, "_ptr", lambda t, keep: None if t is None or t.numel() == 0 else 1 << 40)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda dev=None: types.SimpleNamespace(cuda_stream=0))
    monkeypatch.setattr(graphs, "status_word", lambda dev: torch.zeros(1, dtype=torch.int32))
    monkeypatch.setattr(graphs, "resolve_capacity", lambda dev, P, W, H: 4321)
    # the layer's own checks ask for CUDA tensors; the capture cases set is_current_stream_capturing themselves
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    return rec


@contextlib.contextmanager
def _deterministic(on):
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was)


def _run(rec, fn):
    """fn()'s record: the native calls it made and what it returned, or the exception it raised."""
    rec.calls.clear()
    try:
        out = _describe(fn())
    except Exception as e:  # noqa: BLE001 - the rejection is the record
        out = f"{type(e).__name__}: {e}"
    return rec.calls + ["-> " + out]


# ----------------------------------------------------------------------------- the functional entries
def _fwd_inputs(n, F):
    f = lambda *s: torch.zeros(s)  # noqa: E731
    return dict(background=f(3), means3D=f(n, 3), colors=torch.empty(0), opacity=f(n, 1), scales=f(n, 3),
                rotations=f(n, 4), scale_modifier=1.0, cov3Ds_precomp=torch.empty(0), norm3Ds_precomp=torch.empty(0),
                extra_attrs=f(n, F) if F else torch.empty(0), attr_degree=F, viewmatrix=f(4, 4), projmatrix=f(4, 4),
                tan_fovx=0.5, tan_fovy=0.25, kernel_size=0.1, image_height=H, image_width=W, sh=f(n, 4, 3), degree=1,
                campos=f(3), prefiltered=False, debug=False)


FWD_MODES = {"plain": {}, "graph": dict(graph=True, capacity_hint=100), "ortho": dict(ortho=True),
             "q": dict(depth_quantile=0.25), "dist": dict(depth_distortion=True),
             "ortho_q": dict(ortho=True, depth_quantile=0.75), "ortho_dist": dict(ortho=True, depth_distortion=True),
             "q_dist": dict(depth_quantile=0.5, depth_distortion=True), "graph_ortho": dict(graph=True, ortho=True,
                                                                                          capacity_hint=100)}
FWD_BANDS = {"": {}, "tile_rows": dict(tile_rows=(1, 3)), "out_peers": dict(out_peers=[1 << 40, 1 << 41]),
             "empty_band": dict(tile_rows=(2, 2), out_planes=torch.zeros(8 * H * W), out_peers=[1 << 40])}


def _fwd_cases():
    for mode, band, off in itertools.product(FWD_MODES, FWD_BANDS, (False, True)):
        yield f"{mode}{'+' + band if band else ''}{'+off' if off else ''}", dict(FWD_MODES[mode], **FWD_BANDS[band], off=off)
    for mode in FWD_MODES:
        yield f"{mode}+fuse", dict(FWD_MODES[mode], fuse_normalize=True)
        yield f"{mode}+off+fuse", dict(FWD_MODES[mode], fuse_normalize=True, off=True)
        yield f"{mode}+P0", dict(FWD_MODES[mode], n=0, fuse_normalize=True)
        yield f"{mode}+extra", dict(FWD_MODES[mode], F=2)
        yield f"{mode}+debug", dict(FWD_MODES[mode], debug=True)
    yield "graph+no_capacity", dict(graph=True)
    yield "graph+tan_tensor", dict(graph=True, capacity_hint=100, tan_fovx=torch.tensor(0.5))
    yield "graph+tan_vector", dict(graph=True, capacity_hint=100, tan_fovx=torch.zeros(2))
    yield "off+bad_shape", dict(off="bad")


def _call_forward(opts):
    from sfgs import rasterizer as R
    opts = dict(opts)
    args = _fwd_inputs(opts.pop("n", P), opts.pop("F", 0))
    for k in ("debug", "tan_fovx"):
        if k in opts:
            args[k] = opts.pop(k)
    off = opts.pop("off", False)
    if off:
        opts["subpixel_offset"] = torch.zeros((H, W - 1, 2)) if off == "bad" else torch.zeros((H, W, 2))
    return lambda: R.rasterize_gaussians(*args.values(), **opts)


def _bwd_inputs(n, F):
    f = lambda *s: torch.zeros(s)  # noqa: E731
    g = f(3, H, W)
    return dict(background=f(3), means3D=f(n, 3), radii=torch.zeros(n, dtype=torch.int32), colors=torch.empty(0),
                scales=f(n, 3), rotations=f(n, 4), extra_attrs=f(n, F) if F else torch.empty(0), scale_modifier=1.0,
                cov3Ds_precomp=torch.empty(0), norm3Ds_precomp=torch.empty(0), viewmatrix=f(4, 4),
                projmatrix=f(4, 4), tan_fovx=0.5, tan_fovy=0.25, kernel_size=0.1, dL_dout_color=g,
                dL_dout_depth=g[:1], dL_dout_norm=g, dL_dout_alpha=g[:1], dL_dout_extra=f(F, H, W) if F else
                torch.empty(0), sh=f(n, 4, 3), degree=1, campos=f(3), geomBuffer=torch.zeros(8, dtype=torch.uint8),
                R=77, binningBuffer=torch.zeros(8, dtype=torch.uint8), imageBuffer=torch.zeros(8, dtype=torch.uint8),
                out_alpha=g[:1], debug=False)


BWD_MODES = {"plain": {}, "graph": dict(graph=True), "ortho": dict(ortho=True), "q": dict(q=True),
             "dist": dict(dist=True), "ortho_q": dict(ortho=True, q=True), "ortho_dist": dict(ortho=True, dist=True),
             "q_dist": dict(q=True, dist=True)}
BWD_CAMERA = {"": {}, "cam": dict(camera_grad=True), "cam_intr": dict(camera_grad=True, intrinsics_grad=True),
              "intr": dict(intrinsics_grad=True)}


def _bwd_cases():
    for (mode, phase, cam), det in zip(itertools.product(BWD_MODES, (0, 1, 2), BWD_CAMERA), itertools.cycle((False, True, True))):
        yield (f"{mode}+phase{phase}{'+' + cam if cam else ''}{'+det' if det else ''}",
               dict(BWD_MODES[mode], **BWD_CAMERA[cam], phase=phase, det=det, off=phase != 1,
                    gauss_range=(1, 3) if phase == 2 else None))
    for mode, det in itertools.product(BWD_MODES, (False, True)):
        yield f"{mode}+no_off{'+det' if det else ''}", dict(BWD_MODES[mode], det=det)
        yield f"{mode}+fuse{'+det' if det else ''}", dict(BWD_MODES[mode], det=det, fuse=True)
        yield f"{mode}+tile_rows", dict(BWD_MODES[mode], det=det, phase=1, tile_rows=(0, 0))
        yield f"{mode}+acc_peers{'+det' if det else ''}", dict(BWD_MODES[mode], det=det, phase=1,
                                                               acc_peers=[1 << 40, 1 << 41], peer_slice=1)
        yield f"{mode}+extra{'+det' if det else ''}", dict(BWD_MODES[mode], det=det, F=2)
        yield f"{mode}+P0+cam_intr", dict(BWD_MODES[mode], n=0, camera_grad=True, intrinsics_grad=True)
        yield f"{mode}+debug", dict(BWD_MODES[mode], debug=True)
    yield "plain+P0+phase2+cam", dict(n=0, phase=2, camera_grad=True)
    yield "plain+P0+phase2+cam_intr", dict(n=0, phase=2, camera_grad=True, intrinsics_grad=True)
    yield "plain+P0+phase1", dict(n=0, phase=1)
    yield "plain+phase1+acc", dict(phase=1, acc=torch.zeros((P, 16)))
    yield "plain+acc_peers+phase0", dict(acc_peers=[1 << 40])
    yield "extra+det_warn", dict(F=2, det="warn")
    yield "q+half_pair", dict(q="half")
    yield "dist+half_pair", dict(dist="half")
    yield "q+bad_pos", dict(q="bad")
    yield "dist+bad_state", dict(dist="bad")
    yield "off+bad_shape", dict(off="bad")


def _call_backward(opts):
    from sfgs import rasterizer as R
    opts = dict(opts)
    args = _bwd_inputs(opts.pop("n", P), opts.pop("F", 0))
    if "debug" in opts:
        args["debug"] = opts.pop("debug")
    det = opts.pop("det", False)
    off = opts.pop("off", False)
    if off:
        opts["subpixel_offset"] = torch.zeros((H, W - 1, 2)) if off == "bad" else torch.zeros((H, W, 2))
    if opts.pop("fuse", False):
        opts["norm_raw"] = torch.zeros((3, H, W))
    q, dist = opts.pop("q", False), opts.pop("dist", False)
    if q:
        opts["depth_q_pos"] = torch.zeros((H, W), dtype=torch.float32 if q == "bad" else torch.int32)
        if q != "half":
            opts["dL_dout_depth_q"] = torch.zeros((1, H, W))
    if dist:
        opts["distortion_state"] = torch.zeros((1 if dist == "bad" else 2, H, W))
        if dist != "half":
            opts["dL_dout_distortion"] = torch.zeros((H, W))

    def call():
        import warnings
        with _deterministic(bool(det)), warnings.catch_warnings(record=True) as w:
            if det == "warn":
                torch.use_deterministic_algorithms(True, warn_only=True)
            warnings.simplefilter("always")
            out = R.rasterize_gaussians_backward(*args.values(), **opts)
        return (out, [str(x.message)[:60] for x in w]) if w else out
    return call


# ----------------------------------------------------------------------------- the modules
def _leaves(n=P, precomp=False):
    t = lambda *s: torch.zeros(s, requires_grad=True)  # noqa: E731
    kw = dict(colors_precomp=t(n, 3)) if precomp else dict(shs=t(n, 4, 3))
    return (t(n, 3), t(n, 3), t(n, 1)), dict(kw, scales=t(n, 3), rotations=t(n, 4))


def _grads(out, leaves):
    """Backward from the sum of every float output; the leaves' gradients."""
    loss = sum(o.float().sum() for o in out if isinstance(o, torch.Tensor) and o.is_floating_point() and
               o.requires_grad)
    loss.backward()
    return out, [x.grad if isinstance(x, torch.Tensor) else x for x in leaves]


MODULE_CASES = {
    "plain": {}, "q": dict(depth_quantile=0.5), "dist": dict(depth_distortion=True),
    "q_dist": dict(depth_quantile=0.5, depth_distortion=True), "precomp": dict(precomp=True),
    "view": dict(view=True), "proj_campos": dict(proj=True, campos=True), "focal": dict(focal=True),
    "focal_x": dict(focal="x"), "focal_cpu_tensor": dict(focal="nograd"), "view_focal": dict(view=True, focal=True),
    "q_view_focal": dict(depth_quantile=0.5, view=True, focal=True), "dist_focal": dict(depth_distortion=True,
                                                                                         focal=True),
    "offset_env": dict(env_off=True), "no_fuse": dict(fuse=False), "no_fuse_q": dict(fuse=False, depth_quantile=0.5),
    "debug": dict(debug=True), "det": dict(det=True), "capture": dict(capture=True),
    "capture_view_focal": dict(capture=True, view=True, focal=True), "P0": dict(n=0, precomp=True),
    "P0_q": dict(n=0, precomp=True, depth_quantile=0.5),
    "P0_dist_focal": dict(n=0, precomp=True, depth_distortion=True, focal=True), "no_colors": dict(no_colors=True),
}


def _call_gaussian_rasterizer(opts, monkeypatch):
    import diff_gauss
    from diff_gauss import GaussianRasterizationSettings, GaussianRasterizer
    opts = dict(opts)
    n = opts.get("n", P)
    monkeypatch.setattr(diff_gauss, "FUSE_NORMALIZE", opts.get("fuse", True))
    monkeypatch.setattr(diff_gauss, "SUBPIXEL_OFFSET", bool(opts.get("env_off")))
    if opts.get("capture"):
        monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    focal = opts.get("focal")
    tx = torch.tensor(0.5, requires_grad=focal in (True, "x")) if focal else 0.5
    ty = torch.tensor(0.25, requires_grad=focal is True) if focal else 0.25
    view = torch.eye(4, requires_grad=bool(opts.get("view")))
    proj = torch.eye(4, requires_grad=bool(opts.get("proj")))
    campos = torch.zeros(3, dtype=torch.float64 if opts.get("campos") else torch.float32,
                         requires_grad=bool(opts.get("campos")))
    rs = GaussianRasterizationSettings(H, W, tx, ty, 0.1, torch.zeros((H, W, 2)), torch.zeros(3), 1.0, view, proj, 1,
                                       campos, False, bool(opts.get("debug")))
    (means, means2D, opac), kw = _leaves(n, opts.get("precomp", False))
    if opts.get("no_colors"):
        kw.pop("shs")
    r = GaussianRasterizer(rs, depth_quantile=opts.get("depth_quantile"),
                           depth_distortion=opts.get("depth_distortion", False))

    def call():
        with _deterministic(bool(opts.get("det"))):
            out = r(means, means2D, opac, **kw)
            return _grads(out, [means, means2D, opac, *kw.values(), view, proj, campos, tx, ty])
    return call


def _call_ortho_rasterizer(opts, monkeypatch):
    from sfgs.ortho import OrthoRasterizationSettings, OrthoRasterizer
    opts = dict(opts)
    n = opts.get("n", P)
    rs = OrthoRasterizationSettings(H, W, 2.5, 1.5, 0.1, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 1, False,
                                    bool(opts.get("debug")), torch.zeros((H, W, 2)) if opts.get("env_off") else None)
    (means, means2D, opac), kw = _leaves(n, opts.get("precomp", False))
    if opts.get("no_colors"):
        kw.pop("shs")
    r = OrthoRasterizer(rs, depth_quantile=opts.get("depth_quantile"),
                        depth_distortion=opts.get("depth_distortion", False))

    def call():
        with _deterministic(bool(opts.get("det"))):
            out = r(means, means2D, opac, **kw)
            return _grads(out, [means, means2D, opac, *kw.values()])
    return call


def _call_height_map(q, n):
    from sfgs.ortho import nadir_camera, render_height_map
    cam = nadir_camera(0.0, 8.0, 0.0, 8.0, 1.0, 10.0)
    (means, _, opac), kw = _leaves(n)

    shs = kw["shs"] if n else None     # P = 0: the colours render_height_map makes

    def call():
        out = render_height_map(cam, means, opac, kw["scales"], kw["rotations"], shs=shs, sh_degree=1,
                                surface_quantile=q)
        out.nan_to_num().sum().backward()
        return out, [means.grad, opac.grad, kw["scales"].grad, kw["rotations"].grad, kw["shs"].grad]
    return call


ORTHO_CASES = ("plain", "q", "dist", "q_dist", "precomp", "offset_env", "debug", "det", "P0", "P0_q", "no_colors")


def _all_records(recorder, monkeypatch):
    got = {}
    for name, opts in _fwd_cases():
        got[f"fwd:{name}"] = _run(recorder, _call_forward(opts))
    for name, opts in _bwd_cases():
        got[f"bwd:{name}"] = _run(recorder, _call_backward(opts))
    for name, opts in MODULE_CASES.items():
        with monkeypatch.context() as m:
            got[f"GaussianRasterizer:{name}"] = _run(recorder, _call_gaussian_rasterizer(opts, m))
    for name in ORTHO_CASES:
        with monkeypatch.context() as m:
            got[f"OrthoRasterizer:{name}"] = _run(recorder, _call_ortho_rasterizer(MODULE_CASES[name], m))
    for q, n in ((None, P), (0.5, P), (0.5, 0)):
        got[f"render_height_map:q={q},P={n}"] = _run(recorder, _call_height_map(q, n))
    return got


def _compact(lines):
    """The record with each struct's fields replaced by its key in STRUCTS (unknown structs stay spelled out)."""
    keys = {v: k for k, v in STRUCTS.items()}
    out = []
    for line in lines:
        call, sep, fields = line.partition(" | ")
        out.append(f"{call} | {keys.get(fields, fields)}" if sep else line)
    return out


def test_python_call_matrix(recorder, monkeypatch):
    got = {name: _compact(r) for name, r in _all_records(recorder, monkeypatch).items()}
    assert sorted(got) == sorted(EXPECTED)
    for name, want in EXPECTED.items():
        assert got[name] == want, name


# ----------------------------------------------------------------------------- the table
STRUCTS = {
    'F0': 'P=4 D=1 M=4 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 prefiltered=0 debug=0 capacity_hint=0 tile_row_begin=0 tile_row_end=0 n_out_peers=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,out_extra,out_norm_raw,out_peers',
    'F1': 'P=4 D=1 M=4 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 prefiltered=0 debug=0 capacity_hint=0 tile_row_begin=1 tile_row_end=3 n_out_peers=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,out_extra,out_norm_raw,out_peers',
    'F2': 'P=4 D=1 M=4 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 prefiltered=0 debug=0 capacity_hint=0 tile_row_begin=0 tile_row_end=0 n_out_peers=2 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,out_extra,out_norm_raw',
    'F3': 'P=4 D=1 M=4 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 prefiltered=0 debug=0 capacity_hint=0 tile_row_begin=1048576 tile_row_end=1048576 n_out_peers=1 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,out_extra,out_norm_raw',
    'F4': 'P=4 D=1 M=4 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 prefiltered=0 debug=0 capacity_hint=100 tile_row_begin=0 tile_row_end=0 n_out_peers=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,out_extra,out_norm_raw,out_peers',
    'F5': 'P=4 D=1 M=4 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 prefiltered=0 debug=0 capacity_hint=0 tile_row_begin=0 tile_row_end=0 n_out_peers=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,out_extra,out_peers',
    'F6': 'P=4 D=1 M=4 ED=2 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 prefiltered=0 debug=0 capacity_hint=0 tile_row_begin=0 tile_row_end=0 n_out_peers=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,out_norm_raw,out_peers',
    'F7': 'P=4 D=1 M=4 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 prefiltered=0 debug=1 capacity_hint=0 tile_row_begin=0 tile_row_end=0 n_out_peers=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,out_extra,out_norm_raw,out_peers',
    'F8': 'P=4 D=1 M=4 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 prefiltered=0 debug=0 capacity_hint=100 tile_row_begin=0 tile_row_end=0 n_out_peers=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,out_extra,out_peers',
    'F9': 'P=4 D=1 M=4 ED=2 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 prefiltered=0 debug=0 capacity_hint=100 tile_row_begin=0 tile_row_end=0 n_out_peers=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,out_norm_raw,out_peers',
    'F10': 'P=4 D=1 M=4 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=1 tan_fovy=1 kernel_size=0.100000001 prefiltered=0 debug=0 capacity_hint=100 tile_row_begin=0 tile_row_end=0 n_out_peers=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,out_extra,out_norm_raw,out_peers',
    'B0': 'P=4 D=1 M=4 R=77 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 debug=0 tile_row_begin=0 tile_row_end=0 phase=0 gauss_begin=0 gauss_end=0 n_peers=0 peer_slice=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,dL_dpix_extra,dL_dextra,norm_raw,acc,acc_peers',
    'B1': 'P=4 D=1 M=4 R=77 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 debug=0 tile_row_begin=0 tile_row_end=0 phase=1 gauss_begin=0 gauss_end=0 n_peers=0 peer_slice=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,dL_dpix_extra,dL_dextra,norm_raw,acc_peers',
    'B2': 'P=4 D=1 M=4 R=77 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 debug=0 tile_row_begin=0 tile_row_end=0 phase=2 gauss_begin=1 gauss_end=3 n_peers=0 peer_slice=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,dL_dpix_extra,dL_dextra,norm_raw,acc,acc_peers',
    'B3': 'P=4 D=1 M=4 R=77 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 debug=0 tile_row_begin=0 tile_row_end=0 phase=0 gauss_begin=0 gauss_end=0 n_peers=0 peer_slice=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,dL_dpix_extra,dL_dextra,acc,acc_peers',
    'B4': 'P=4 D=1 M=4 R=77 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 debug=0 tile_row_begin=1048576 tile_row_end=1048576 phase=1 gauss_begin=0 gauss_end=0 n_peers=0 peer_slice=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,dL_dpix_extra,dL_dextra,norm_raw,acc_peers',
    'B5': 'P=4 D=1 M=4 R=77 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 debug=0 tile_row_begin=0 tile_row_end=0 phase=1 gauss_begin=0 gauss_end=0 n_peers=2 peer_slice=1 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,dL_dpix_extra,dL_dextra,norm_raw,acc',
    'B6': 'P=4 D=1 M=4 R=77 ED=2 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 debug=0 tile_row_begin=0 tile_row_end=0 phase=0 gauss_begin=0 gauss_end=0 n_peers=0 peer_slice=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,norm_raw,acc,acc_peers',
    'B7': 'P=4 D=1 M=4 R=77 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 debug=1 tile_row_begin=0 tile_row_end=0 phase=0 gauss_begin=0 gauss_end=0 n_peers=0 peer_slice=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,dL_dpix_extra,dL_dextra,norm_raw,acc,acc_peers',
    'B8': 'P=4 D=1 M=4 R=5 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 debug=0 tile_row_begin=0 tile_row_end=0 phase=0 gauss_begin=0 gauss_end=0 n_peers=0 peer_slice=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,geom_buffer,binning_buffer,image_buffer,dL_dpix_extra,dL_dextra,acc,acc_peers',
    'F11': 'P=4 D=1 M=0 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 prefiltered=0 debug=0 capacity_hint=0 tile_row_begin=0 tile_row_end=0 n_out_peers=0 null=shs,cov3D_precomp,norm3D_precomp,extra_attrs,out_extra,out_peers',
    'B9': 'P=4 D=1 M=0 R=5 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 debug=0 tile_row_begin=0 tile_row_end=0 phase=0 gauss_begin=0 gauss_end=0 n_peers=0 peer_slice=0 null=shs,cov3D_precomp,norm3D_precomp,extra_attrs,geom_buffer,binning_buffer,image_buffer,dL_dpix_extra,dL_dsh,dL_dextra,acc,acc_peers',
    'B10': 'P=4 D=1 M=4 R=5 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 debug=0 tile_row_begin=0 tile_row_end=0 phase=0 gauss_begin=0 gauss_end=0 n_peers=0 peer_slice=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,geom_buffer,binning_buffer,image_buffer,dL_dpix_extra,dL_dextra,norm_raw,acc,acc_peers',
    'F12': 'P=4 D=1 M=4 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 prefiltered=0 debug=1 capacity_hint=0 tile_row_begin=0 tile_row_end=0 n_out_peers=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,out_extra,out_peers',
    'B11': 'P=4 D=1 M=4 R=5 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 debug=1 tile_row_begin=0 tile_row_end=0 phase=0 gauss_begin=0 gauss_end=0 n_peers=0 peer_slice=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,geom_buffer,binning_buffer,image_buffer,dL_dpix_extra,dL_dextra,acc,acc_peers',
    'F13': 'P=4 D=1 M=4 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 prefiltered=0 debug=0 capacity_hint=4321 tile_row_begin=0 tile_row_end=0 n_out_peers=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,out_extra,out_peers',
    'B12': 'P=4 D=1 M=4 R=4321 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=0.5 tan_fovy=0.25 kernel_size=0.100000001 debug=0 tile_row_begin=0 tile_row_end=0 phase=0 gauss_begin=0 gauss_end=0 n_peers=0 peer_slice=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,geom_buffer,binning_buffer,image_buffer,dL_dpix_extra,dL_dextra,acc,acc_peers',
    'F14': 'P=4 D=1 M=4 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=1 tan_fovy=1 kernel_size=0.100000001 prefiltered=0 debug=0 capacity_hint=4321 tile_row_begin=0 tile_row_end=0 n_out_peers=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,out_extra,out_peers',
    'B13': 'P=4 D=1 M=4 R=4321 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=1 tan_fovy=1 kernel_size=0.100000001 debug=0 tile_row_begin=0 tile_row_end=0 phase=0 gauss_begin=0 gauss_end=0 n_peers=0 peer_slice=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,geom_buffer,binning_buffer,image_buffer,dL_dpix_extra,dL_dextra,acc,acc_peers',
    'F15': 'P=4 D=1 M=4 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=2.5 tan_fovy=1.5 kernel_size=0.100000001 prefiltered=0 debug=0 capacity_hint=0 tile_row_begin=0 tile_row_end=0 n_out_peers=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,out_extra,out_peers',
    'B14': 'P=4 D=1 M=4 R=5 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=2.5 tan_fovy=1.5 kernel_size=0.100000001 debug=0 tile_row_begin=0 tile_row_end=0 phase=0 gauss_begin=0 gauss_end=0 n_peers=0 peer_slice=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,geom_buffer,binning_buffer,image_buffer,dL_dpix_extra,dL_dextra,acc,acc_peers',
    'F16': 'P=4 D=1 M=0 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=2.5 tan_fovy=1.5 kernel_size=0.100000001 prefiltered=0 debug=0 capacity_hint=0 tile_row_begin=0 tile_row_end=0 n_out_peers=0 null=shs,cov3D_precomp,norm3D_precomp,extra_attrs,out_extra,out_peers',
    'B15': 'P=4 D=1 M=0 R=5 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=2.5 tan_fovy=1.5 kernel_size=0.100000001 debug=0 tile_row_begin=0 tile_row_end=0 phase=0 gauss_begin=0 gauss_end=0 n_peers=0 peer_slice=0 null=shs,cov3D_precomp,norm3D_precomp,extra_attrs,geom_buffer,binning_buffer,image_buffer,dL_dpix_extra,dL_dsh,dL_dextra,acc,acc_peers',
    'F17': 'P=4 D=1 M=4 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=2.5 tan_fovy=1.5 kernel_size=0.100000001 prefiltered=0 debug=1 capacity_hint=0 tile_row_begin=0 tile_row_end=0 n_out_peers=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,out_extra,out_peers',
    'B16': 'P=4 D=1 M=4 R=5 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=2.5 tan_fovy=1.5 kernel_size=0.100000001 debug=1 tile_row_begin=0 tile_row_end=0 phase=0 gauss_begin=0 gauss_end=0 n_peers=0 peer_slice=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,geom_buffer,binning_buffer,image_buffer,dL_dpix_extra,dL_dextra,acc,acc_peers',
    'F18': 'P=4 D=1 M=4 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=4 tan_fovy=4 kernel_size=0.100000001 prefiltered=0 debug=0 capacity_hint=0 tile_row_begin=0 tile_row_end=0 n_out_peers=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,out_extra,out_peers',
    'B17': 'P=4 D=1 M=4 R=5 ED=0 width=8 height=8 scale_modifier=1 tan_fovx=4 tan_fovy=4 kernel_size=0.100000001 debug=0 tile_row_begin=0 tile_row_end=0 phase=0 gauss_begin=0 gauss_end=0 n_peers=0 peer_slice=0 null=colors_precomp,cov3D_precomp,norm3D_precomp,extra_attrs,geom_buffer,binning_buffer,image_buffer,dL_dpix_extra,dL_dextra,acc,acc_peers',
}

EXPECTED = {
    'fwd:plain': [
        'sfgs_rasterize_forward() | F0',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0])',
    ],
    'fwd:plain+off': [
        'sfgs_rasterize_forward_subpixel(*) | F0',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0])',
    ],
    'fwd:plain+tile_rows': [
        'sfgs_rasterize_forward() | F1',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0])',
    ],
    'fwd:plain+tile_rows+off': [
        'sfgs_rasterize_forward_subpixel(*) | F1',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0])',
    ],
    'fwd:plain+out_peers': [
        'sfgs_rasterize_forward() | F2',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0])',
    ],
    'fwd:plain+out_peers+off': [
        'sfgs_rasterize_forward_subpixel_peers(*) | F2',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0])',
    ],
    'fwd:plain+empty_band': [
        'sfgs_rasterize_forward() | F3',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0])',
    ],
    'fwd:plain+empty_band+off': [
        'sfgs_rasterize_forward_subpixel_peers(*) | F3',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0])',
    ],
    'fwd:graph': [
        'sfgs_rasterize_forward_graph(0, 0, *) | F4',
        '-> (-1, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0])',
    ],
    'fwd:graph+off': [
        'sfgs_rasterize_forward_graph(*, 0, *) | F4',
        '-> (-1, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0])',
    ],
    'fwd:graph+tile_rows': [
        '-> SfgsError: rasterize_gaussians(graph=True): tile_rows cannot be captured in a CUDA graph',
    ],
    'fwd:graph+tile_rows+off': [
        '-> SfgsError: rasterize_gaussians(graph=True): tile_rows cannot be captured in a CUDA graph',
    ],
    'fwd:graph+out_peers': [
        '-> SfgsError: rasterize_gaussians(graph=True): out_peers cannot be captured in a CUDA graph',
    ],
    'fwd:graph+out_peers+off': [
        '-> SfgsError: rasterize_gaussians(graph=True): out_peers cannot be captured in a CUDA graph',
    ],
    'fwd:graph+empty_band': [
        '-> SfgsError: rasterize_gaussians(graph=True): tile_rows, out_peers cannot be captured in a CUDA graph',
    ],
    'fwd:graph+empty_band+off': [
        '-> SfgsError: rasterize_gaussians(graph=True): tile_rows, out_peers cannot be captured in a CUDA graph',
    ],
    'fwd:ortho': [
        'sfgs_rasterize_forward_ortho(0) | F0',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0])',
    ],
    'fwd:ortho+off': [
        'sfgs_rasterize_forward_ortho(*) | F0',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0])',
    ],
    'fwd:ortho+tile_rows': [
        '-> SfgsError: rasterize_gaussians(ortho=True): tile_rows not supported with an orthographic camera',
    ],
    'fwd:ortho+tile_rows+off': [
        '-> SfgsError: rasterize_gaussians(ortho=True): tile_rows not supported with an orthographic camera',
    ],
    'fwd:ortho+out_peers': [
        '-> SfgsError: rasterize_gaussians(ortho=True): out_peers not supported with an orthographic camera',
    ],
    'fwd:ortho+out_peers+off': [
        '-> SfgsError: rasterize_gaussians(ortho=True): out_peers not supported with an orthographic camera',
    ],
    'fwd:ortho+empty_band': [
        '-> SfgsError: rasterize_gaussians(ortho=True): tile_rows, out_peers not supported with an orthographic camera',
    ],
    'fwd:ortho+empty_band+off': [
        '-> SfgsError: rasterize_gaussians(ortho=True): tile_rows, out_peers not supported with an orthographic camera',
    ],
    'fwd:q': [
        'sfgs_rasterize_forward_depth_quantile(0, 0, 0.25, *, *) | F0',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[1, 8, 8], int32[8, 8])',
    ],
    'fwd:q+off': [
        'sfgs_rasterize_forward_depth_quantile(*, 0, 0.25, *, *) | F0',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[1, 8, 8], int32[8, 8])',
    ],
    'fwd:q+tile_rows': [
        '-> SfgsError: rasterize_gaussians(depth_quantile=...): tile_rows not supported with the depth quantile',
    ],
    'fwd:q+tile_rows+off': [
        '-> SfgsError: rasterize_gaussians(depth_quantile=...): tile_rows not supported with the depth quantile',
    ],
    'fwd:q+out_peers': [
        '-> SfgsError: rasterize_gaussians(depth_quantile=...): out_peers not supported with the depth quantile',
    ],
    'fwd:q+out_peers+off': [
        '-> SfgsError: rasterize_gaussians(depth_quantile=...): out_peers not supported with the depth quantile',
    ],
    'fwd:q+empty_band': [
        '-> SfgsError: rasterize_gaussians(depth_quantile=...): tile_rows, out_peers not supported with the depth quantile',
    ],
    'fwd:q+empty_band+off': [
        '-> SfgsError: rasterize_gaussians(depth_quantile=...): tile_rows, out_peers not supported with the depth quantile',
    ],
    'fwd:dist': [
        'sfgs_rasterize_forward_distortion(0, 0, *, *) | F0',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[1, 8, 8], float32[2, 8, 8])',
    ],
    'fwd:dist+off': [
        'sfgs_rasterize_forward_distortion(*, 0, *, *) | F0',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[1, 8, 8], float32[2, 8, 8])',
    ],
    'fwd:dist+tile_rows': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): tile_rows not supported with the depth distortion',
    ],
    'fwd:dist+tile_rows+off': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): tile_rows not supported with the depth distortion',
    ],
    'fwd:dist+out_peers': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): out_peers not supported with the depth distortion',
    ],
    'fwd:dist+out_peers+off': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): out_peers not supported with the depth distortion',
    ],
    'fwd:dist+empty_band': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): tile_rows, out_peers not supported with the depth distortion',
    ],
    'fwd:dist+empty_band+off': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): tile_rows, out_peers not supported with the depth distortion',
    ],
    'fwd:ortho_q': [
        'sfgs_rasterize_forward_depth_quantile(0, 1, 0.75, *, *) | F0',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[1, 8, 8], int32[8, 8])',
    ],
    'fwd:ortho_q+off': [
        'sfgs_rasterize_forward_depth_quantile(*, 1, 0.75, *, *) | F0',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[1, 8, 8], int32[8, 8])',
    ],
    'fwd:ortho_q+tile_rows': [
        '-> SfgsError: rasterize_gaussians(depth_quantile=...): tile_rows not supported with the depth quantile',
    ],
    'fwd:ortho_q+tile_rows+off': [
        '-> SfgsError: rasterize_gaussians(depth_quantile=...): tile_rows not supported with the depth quantile',
    ],
    'fwd:ortho_q+out_peers': [
        '-> SfgsError: rasterize_gaussians(depth_quantile=...): out_peers not supported with the depth quantile',
    ],
    'fwd:ortho_q+out_peers+off': [
        '-> SfgsError: rasterize_gaussians(depth_quantile=...): out_peers not supported with the depth quantile',
    ],
    'fwd:ortho_q+empty_band': [
        '-> SfgsError: rasterize_gaussians(depth_quantile=...): tile_rows, out_peers not supported with the depth quantile',
    ],
    'fwd:ortho_q+empty_band+off': [
        '-> SfgsError: rasterize_gaussians(depth_quantile=...): tile_rows, out_peers not supported with the depth quantile',
    ],
    'fwd:ortho_dist': [
        'sfgs_rasterize_forward_distortion(0, 1, *, *) | F0',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[1, 8, 8], float32[2, 8, 8])',
    ],
    'fwd:ortho_dist+off': [
        'sfgs_rasterize_forward_distortion(*, 1, *, *) | F0',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[1, 8, 8], float32[2, 8, 8])',
    ],
    'fwd:ortho_dist+tile_rows': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): tile_rows not supported with the depth distortion',
    ],
    'fwd:ortho_dist+tile_rows+off': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): tile_rows not supported with the depth distortion',
    ],
    'fwd:ortho_dist+out_peers': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): out_peers not supported with the depth distortion',
    ],
    'fwd:ortho_dist+out_peers+off': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): out_peers not supported with the depth distortion',
    ],
    'fwd:ortho_dist+empty_band': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): tile_rows, out_peers not supported with the depth distortion',
    ],
    'fwd:ortho_dist+empty_band+off': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): tile_rows, out_peers not supported with the depth distortion',
    ],
    'fwd:q_dist': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): depth_quantile not supported with the depth distortion',
    ],
    'fwd:q_dist+off': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): depth_quantile not supported with the depth distortion',
    ],
    'fwd:q_dist+tile_rows': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): depth_quantile, tile_rows not supported with the depth distortion',
    ],
    'fwd:q_dist+tile_rows+off': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): depth_quantile, tile_rows not supported with the depth distortion',
    ],
    'fwd:q_dist+out_peers': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): depth_quantile, out_peers not supported with the depth distortion',
    ],
    'fwd:q_dist+out_peers+off': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): depth_quantile, out_peers not supported with the depth distortion',
    ],
    'fwd:q_dist+empty_band': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): depth_quantile, tile_rows, out_peers not supported with the depth distortion',
    ],
    'fwd:q_dist+empty_band+off': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): depth_quantile, tile_rows, out_peers not supported with the depth distortion',
    ],
    'fwd:graph_ortho': [
        '-> SfgsError: rasterize_gaussians(ortho=True): graph not supported with an orthographic camera',
    ],
    'fwd:graph_ortho+off': [
        '-> SfgsError: rasterize_gaussians(ortho=True): graph not supported with an orthographic camera',
    ],
    'fwd:graph_ortho+tile_rows': [
        '-> SfgsError: rasterize_gaussians(ortho=True): graph, tile_rows not supported with an orthographic camera',
    ],
    'fwd:graph_ortho+tile_rows+off': [
        '-> SfgsError: rasterize_gaussians(ortho=True): graph, tile_rows not supported with an orthographic camera',
    ],
    'fwd:graph_ortho+out_peers': [
        '-> SfgsError: rasterize_gaussians(ortho=True): graph, out_peers not supported with an orthographic camera',
    ],
    'fwd:graph_ortho+out_peers+off': [
        '-> SfgsError: rasterize_gaussians(ortho=True): graph, out_peers not supported with an orthographic camera',
    ],
    'fwd:graph_ortho+empty_band': [
        '-> SfgsError: rasterize_gaussians(ortho=True): graph, tile_rows, out_peers not supported with an orthographic camera',
    ],
    'fwd:graph_ortho+empty_band+off': [
        '-> SfgsError: rasterize_gaussians(ortho=True): graph, tile_rows, out_peers not supported with an orthographic camera',
    ],
    'fwd:plain+fuse': [
        'sfgs_rasterize_forward() | F5',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[3, 8, 8])',
    ],
    'fwd:plain+off+fuse': [
        'sfgs_rasterize_forward_subpixel(*) | F5',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[3, 8, 8])',
    ],
    'fwd:plain+P0': [
        '-> (0, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[0], float32[0], uint8[0], uint8[0], uint8[0], float32[3, 8, 8])',
    ],
    'fwd:plain+extra': [
        'sfgs_rasterize_forward() | F6',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[2, 8, 8], uint8[0], uint8[0], uint8[0])',
    ],
    'fwd:plain+debug': [
        'sfgs_rasterize_forward() | F7',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0])',
    ],
    'fwd:graph+fuse': [
        'sfgs_rasterize_forward_graph(0, 0, *) | F8',
        '-> (-1, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[3, 8, 8])',
    ],
    'fwd:graph+off+fuse': [
        'sfgs_rasterize_forward_graph(*, 0, *) | F8',
        '-> (-1, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[3, 8, 8])',
    ],
    'fwd:graph+P0': [
        '-> (0, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[0], float32[0], uint8[0], uint8[0], uint8[0], float32[3, 8, 8])',
    ],
    'fwd:graph+extra': [
        'sfgs_rasterize_forward_graph(0, 0, *) | F9',
        '-> (-1, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[2, 8, 8], uint8[0], uint8[0], uint8[0])',
    ],
    'fwd:graph+debug': [
        '-> SfgsError: rasterize_gaussians(graph=True): debug=True (it synchronises after every stage) cannot be captured in a CUDA graph',
    ],
    'fwd:ortho+fuse': [
        'sfgs_rasterize_forward_ortho(0) | F5',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[3, 8, 8])',
    ],
    'fwd:ortho+off+fuse': [
        'sfgs_rasterize_forward_ortho(*) | F5',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[3, 8, 8])',
    ],
    'fwd:ortho+P0': [
        '-> (0, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[0], float32[0], uint8[0], uint8[0], uint8[0], float32[3, 8, 8])',
    ],
    'fwd:ortho+extra': [
        'sfgs_rasterize_forward_ortho(0) | F6',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[2, 8, 8], uint8[0], uint8[0], uint8[0])',
    ],
    'fwd:ortho+debug': [
        'sfgs_rasterize_forward_ortho(0) | F7',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0])',
    ],
    'fwd:q+fuse': [
        'sfgs_rasterize_forward_depth_quantile(0, 0, 0.25, *, *) | F5',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[3, 8, 8], float32[1, 8, 8], int32[8, 8])',
    ],
    'fwd:q+off+fuse': [
        'sfgs_rasterize_forward_depth_quantile(*, 0, 0.25, *, *) | F5',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[3, 8, 8], float32[1, 8, 8], int32[8, 8])',
    ],
    'fwd:q+P0': [
        '-> (0, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[0], float32[0], uint8[0], uint8[0], uint8[0], float32[3, 8, 8], float32[1, 8, 8], int32[8, 8])',
    ],
    'fwd:q+extra': [
        '-> SfgsError: rasterize_gaussians(depth_quantile=...): extra_attrs not supported with the depth quantile',
    ],
    'fwd:q+debug': [
        'sfgs_rasterize_forward_depth_quantile(0, 0, 0.25, *, *) | F7',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[1, 8, 8], int32[8, 8])',
    ],
    'fwd:dist+fuse': [
        'sfgs_rasterize_forward_distortion(0, 0, *, *) | F5',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[3, 8, 8], float32[1, 8, 8], float32[2, 8, 8])',
    ],
    'fwd:dist+off+fuse': [
        'sfgs_rasterize_forward_distortion(*, 0, *, *) | F5',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[3, 8, 8], float32[1, 8, 8], float32[2, 8, 8])',
    ],
    'fwd:dist+P0': [
        '-> (0, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[0], float32[0], uint8[0], uint8[0], uint8[0], float32[3, 8, 8], float32[1, 8, 8], float32[2, 8, 8])',
    ],
    'fwd:dist+extra': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): extra_attrs not supported with the depth distortion',
    ],
    'fwd:dist+debug': [
        'sfgs_rasterize_forward_distortion(0, 0, *, *) | F7',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[1, 8, 8], float32[2, 8, 8])',
    ],
    'fwd:ortho_q+fuse': [
        'sfgs_rasterize_forward_depth_quantile(0, 1, 0.75, *, *) | F5',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[3, 8, 8], float32[1, 8, 8], int32[8, 8])',
    ],
    'fwd:ortho_q+off+fuse': [
        'sfgs_rasterize_forward_depth_quantile(*, 1, 0.75, *, *) | F5',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[3, 8, 8], float32[1, 8, 8], int32[8, 8])',
    ],
    'fwd:ortho_q+P0': [
        '-> (0, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[0], float32[0], uint8[0], uint8[0], uint8[0], float32[3, 8, 8], float32[1, 8, 8], int32[8, 8])',
    ],
    'fwd:ortho_q+extra': [
        '-> SfgsError: rasterize_gaussians(depth_quantile=...): extra_attrs not supported with the depth quantile',
    ],
    'fwd:ortho_q+debug': [
        'sfgs_rasterize_forward_depth_quantile(0, 1, 0.75, *, *) | F7',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[1, 8, 8], int32[8, 8])',
    ],
    'fwd:ortho_dist+fuse': [
        'sfgs_rasterize_forward_distortion(0, 1, *, *) | F5',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[3, 8, 8], float32[1, 8, 8], float32[2, 8, 8])',
    ],
    'fwd:ortho_dist+off+fuse': [
        'sfgs_rasterize_forward_distortion(*, 1, *, *) | F5',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[3, 8, 8], float32[1, 8, 8], float32[2, 8, 8])',
    ],
    'fwd:ortho_dist+P0': [
        '-> (0, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[0], float32[0], uint8[0], uint8[0], uint8[0], float32[3, 8, 8], float32[1, 8, 8], float32[2, 8, 8])',
    ],
    'fwd:ortho_dist+extra': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): extra_attrs not supported with the depth distortion',
    ],
    'fwd:ortho_dist+debug': [
        'sfgs_rasterize_forward_distortion(0, 1, *, *) | F7',
        '-> (5, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0], float32[1, 8, 8], float32[2, 8, 8])',
    ],
    'fwd:q_dist+fuse': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): depth_quantile not supported with the depth distortion',
    ],
    'fwd:q_dist+off+fuse': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): depth_quantile not supported with the depth distortion',
    ],
    'fwd:q_dist+P0': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): depth_quantile not supported with the depth distortion',
    ],
    'fwd:q_dist+extra': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): depth_quantile, extra_attrs not supported with the depth distortion',
    ],
    'fwd:q_dist+debug': [
        '-> SfgsError: rasterize_gaussians(depth_distortion=True): depth_quantile not supported with the depth distortion',
    ],
    'fwd:graph_ortho+fuse': [
        '-> SfgsError: rasterize_gaussians(ortho=True): graph not supported with an orthographic camera',
    ],
    'fwd:graph_ortho+off+fuse': [
        '-> SfgsError: rasterize_gaussians(ortho=True): graph not supported with an orthographic camera',
    ],
    'fwd:graph_ortho+P0': [
        '-> SfgsError: rasterize_gaussians(ortho=True): graph not supported with an orthographic camera',
    ],
    'fwd:graph_ortho+extra': [
        '-> SfgsError: rasterize_gaussians(ortho=True): graph not supported with an orthographic camera',
    ],
    'fwd:graph_ortho+debug': [
        '-> SfgsError: rasterize_gaussians(ortho=True): graph not supported with an orthographic camera',
    ],
    'fwd:graph+no_capacity': [
        '-> SfgsError: rasterize_gaussians(graph=True) needs capacity_hint > 0 (see sfgs.graphs.capacity)',
    ],
    'fwd:graph+tan_tensor': [
        'sfgs_rasterize_forward_graph(0, *, *) | F10',
        '-> (-1, float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], uint8[0], uint8[0], uint8[0])',
    ],
    'fwd:graph+tan_vector': [
        '-> ValueError: under graph capture tanfovx / tanfovy must be Python numbers or 0-d CUDA tensors',
    ],
    'fwd:off+bad_shape': [
        '-> ValueError: subpixel_offset must be a CUDA float32 tensor of shape (8, 8, 2), got torch.float32 (8, 7, 2) on cpu',
    ],
    'bwd:plain+phase0': [
        'sfgs_rasterize_backward_subpixel(*) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:plain+phase0+cam+det': [
        'sfgs_rasterize_backward_camera(*, 1, *) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0], float32[4, 4], float32[4, 4], float32[3])',
    ],
    'bwd:plain+phase0+cam_intr+det': [
        'sfgs_rasterize_backward_camera_intrinsics(*, 1, *) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0], float32[4, 4], float32[4, 4], float32[3], float32[], float32[])',
    ],
    'bwd:plain+phase0+intr': [
        '-> ValueError: intrinsics_grad=True needs camera_grad=True',
    ],
    'bwd:plain+phase1+det': [
        'sfgs_rasterize_backward_deterministic() | B1',
        '-> float32[4, 16]',
    ],
    'bwd:plain+phase1+cam+det': [
        'sfgs_rasterize_backward_camera(0, 1, *) | B1',
        '-> float32[4, 16]',
    ],
    'bwd:plain+phase1+cam_intr': [
        'sfgs_rasterize_backward_camera_intrinsics(0, 0, *) | B1',
        '-> float32[4, 16]',
    ],
    'bwd:plain+phase1+intr+det': [
        '-> ValueError: intrinsics_grad=True needs camera_grad=True',
    ],
    'bwd:plain+phase2+det': [
        'sfgs_rasterize_backward_deterministic_subpixel(*) | B2',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:plain+phase2+cam': [
        'sfgs_rasterize_backward_camera_partial(*, 0, 35, *) | B2',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0], float64[35])',
    ],
    'bwd:plain+phase2+cam_intr+det': [
        'sfgs_rasterize_backward_camera_partial(*, 1, 37, *) | B2',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0], float64[37])',
    ],
    'bwd:plain+phase2+intr+det': [
        '-> ValueError: intrinsics_grad=True needs camera_grad=True',
    ],
    'bwd:graph+phase0': [
        'sfgs_rasterize_backward_graph(*, 0, 0, 0, 0) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:graph+phase0+cam+det': [
        'sfgs_rasterize_backward_graph(*, 1, 0, *, 35) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0], float32[4, 4], float32[4, 4], float32[3])',
    ],
    'bwd:graph+phase0+cam_intr+det': [
        'sfgs_rasterize_backward_graph(*, 1, 0, *, 37) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0], float32[4, 4], float32[4, 4], float32[3], float32[], float32[])',
    ],
    'bwd:graph+phase0+intr': [
        '-> ValueError: intrinsics_grad=True needs camera_grad=True',
    ],
    'bwd:graph+phase1+det': [
        '-> SfgsError: rasterize_gaussians_backward(graph=True): phase=1 (the two-phase backward) cannot be captured in a CUDA graph',
    ],
    'bwd:graph+phase1+cam+det': [
        '-> SfgsError: rasterize_gaussians_backward(graph=True): phase=1 (the two-phase backward) cannot be captured in a CUDA graph',
    ],
    'bwd:graph+phase1+cam_intr': [
        '-> SfgsError: rasterize_gaussians_backward(graph=True): phase=1 (the two-phase backward) cannot be captured in a CUDA graph',
    ],
    'bwd:graph+phase1+intr+det': [
        '-> ValueError: intrinsics_grad=True needs camera_grad=True',
    ],
    'bwd:graph+phase2+det': [
        '-> SfgsError: rasterize_gaussians_backward(graph=True): phase=2 (the two-phase backward) cannot be captured in a CUDA graph',
    ],
    'bwd:graph+phase2+cam': [
        '-> SfgsError: rasterize_gaussians_backward(graph=True): phase=2 (the two-phase backward) cannot be captured in a CUDA graph',
    ],
    'bwd:graph+phase2+cam_intr+det': [
        '-> SfgsError: rasterize_gaussians_backward(graph=True): phase=2 (the two-phase backward) cannot be captured in a CUDA graph',
    ],
    'bwd:graph+phase2+intr+det': [
        '-> ValueError: intrinsics_grad=True needs camera_grad=True',
    ],
    'bwd:ortho+phase0': [
        'sfgs_rasterize_backward_ortho(*, 0) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:ortho+phase0+cam+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): camera_grad not supported with an orthographic camera',
    ],
    'bwd:ortho+phase0+cam_intr+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): camera_grad, intrinsics_grad not supported with an orthographic camera',
    ],
    'bwd:ortho+phase0+intr': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): intrinsics_grad not supported with an orthographic camera',
    ],
    'bwd:ortho+phase1+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=1 not supported with an orthographic camera',
    ],
    'bwd:ortho+phase1+cam+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=1, camera_grad not supported with an orthographic camera',
    ],
    'bwd:ortho+phase1+cam_intr': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=1, camera_grad, intrinsics_grad not supported with an orthographic camera',
    ],
    'bwd:ortho+phase1+intr+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=1, intrinsics_grad not supported with an orthographic camera',
    ],
    'bwd:ortho+phase2+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=2 not supported with an orthographic camera',
    ],
    'bwd:ortho+phase2+cam': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=2, camera_grad not supported with an orthographic camera',
    ],
    'bwd:ortho+phase2+cam_intr+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=2, camera_grad, intrinsics_grad not supported with an orthographic camera',
    ],
    'bwd:ortho+phase2+intr+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=2, intrinsics_grad not supported with an orthographic camera',
    ],
    'bwd:q+phase0': [
        'sfgs_rasterize_backward_depth_quantile(*, 0, 0, *, *, 0, 0) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:q+phase0+cam+det': [
        'sfgs_rasterize_backward_depth_quantile(*, 0, 1, *, *, *, 35) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0], float32[4, 4], float32[4, 4], float32[3])',
    ],
    'bwd:q+phase0+cam_intr+det': [
        'sfgs_rasterize_backward_depth_quantile(*, 0, 1, *, *, *, 37) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0], float32[4, 4], float32[4, 4], float32[3], float32[], float32[])',
    ],
    'bwd:q+phase0+intr': [
        '-> ValueError: intrinsics_grad=True needs camera_grad=True',
    ],
    'bwd:q+phase1+det': [
        'sfgs_rasterize_backward_depth_quantile(0, 0, 1, *, *, 0, 0) | B1',
        '-> float32[4, 16]',
    ],
    'bwd:q+phase1+cam+det': [
        'sfgs_rasterize_backward_depth_quantile(0, 0, 1, *, *, *, 35) | B1',
        '-> float32[4, 16]',
    ],
    'bwd:q+phase1+cam_intr': [
        'sfgs_rasterize_backward_depth_quantile(0, 0, 0, *, *, *, 37) | B1',
        '-> float32[4, 16]',
    ],
    'bwd:q+phase1+intr+det': [
        '-> ValueError: intrinsics_grad=True needs camera_grad=True',
    ],
    'bwd:q+phase2+det': [
        'sfgs_rasterize_backward_depth_quantile(*, 0, 1, *, *, 0, 0) | B2',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:q+phase2+cam': [
        'sfgs_rasterize_backward_depth_quantile(*, 0, 0, *, *, *, 35) | B2',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0], float32[35])',
    ],
    'bwd:q+phase2+cam_intr+det': [
        'sfgs_rasterize_backward_depth_quantile(*, 0, 1, *, *, *, 37) | B2',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0], float32[37])',
    ],
    'bwd:q+phase2+intr+det': [
        '-> ValueError: intrinsics_grad=True needs camera_grad=True',
    ],
    'bwd:dist+phase0': [
        'sfgs_rasterize_backward_distortion(*, 0, 0, *, *, 0, 0) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:dist+phase0+cam+det': [
        'sfgs_rasterize_backward_distortion(*, 0, 1, *, *, *, 35) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0], float32[4, 4], float32[4, 4], float32[3])',
    ],
    'bwd:dist+phase0+cam_intr+det': [
        'sfgs_rasterize_backward_distortion(*, 0, 1, *, *, *, 37) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0], float32[4, 4], float32[4, 4], float32[3], float32[], float32[])',
    ],
    'bwd:dist+phase0+intr': [
        '-> ValueError: intrinsics_grad=True needs camera_grad=True',
    ],
    'bwd:dist+phase1+det': [
        'sfgs_rasterize_backward_distortion(0, 0, 1, *, *, 0, 0) | B1',
        '-> float32[4, 16]',
    ],
    'bwd:dist+phase1+cam+det': [
        'sfgs_rasterize_backward_distortion(0, 0, 1, *, *, *, 35) | B1',
        '-> float32[4, 16]',
    ],
    'bwd:dist+phase1+cam_intr': [
        'sfgs_rasterize_backward_distortion(0, 0, 0, *, *, *, 37) | B1',
        '-> float32[4, 16]',
    ],
    'bwd:dist+phase1+intr+det': [
        '-> ValueError: intrinsics_grad=True needs camera_grad=True',
    ],
    'bwd:dist+phase2+det': [
        'sfgs_rasterize_backward_distortion(*, 0, 1, *, *, 0, 0) | B2',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:dist+phase2+cam': [
        'sfgs_rasterize_backward_distortion(*, 0, 0, *, *, *, 35) | B2',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0], float32[35])',
    ],
    'bwd:dist+phase2+cam_intr+det': [
        'sfgs_rasterize_backward_distortion(*, 0, 1, *, *, *, 37) | B2',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0], float32[37])',
    ],
    'bwd:dist+phase2+intr+det': [
        '-> ValueError: intrinsics_grad=True needs camera_grad=True',
    ],
    'bwd:ortho_q+phase0': [
        'sfgs_rasterize_backward_depth_quantile(*, 1, 0, *, *, 0, 0) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:ortho_q+phase0+cam+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): camera_grad not supported with an orthographic camera',
    ],
    'bwd:ortho_q+phase0+cam_intr+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): camera_grad, intrinsics_grad not supported with an orthographic camera',
    ],
    'bwd:ortho_q+phase0+intr': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): intrinsics_grad not supported with an orthographic camera',
    ],
    'bwd:ortho_q+phase1+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=1 not supported with an orthographic camera',
    ],
    'bwd:ortho_q+phase1+cam+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=1, camera_grad not supported with an orthographic camera',
    ],
    'bwd:ortho_q+phase1+cam_intr': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=1, camera_grad, intrinsics_grad not supported with an orthographic camera',
    ],
    'bwd:ortho_q+phase1+intr+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=1, intrinsics_grad not supported with an orthographic camera',
    ],
    'bwd:ortho_q+phase2+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=2 not supported with an orthographic camera',
    ],
    'bwd:ortho_q+phase2+cam': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=2, camera_grad not supported with an orthographic camera',
    ],
    'bwd:ortho_q+phase2+cam_intr+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=2, camera_grad, intrinsics_grad not supported with an orthographic camera',
    ],
    'bwd:ortho_q+phase2+intr+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=2, intrinsics_grad not supported with an orthographic camera',
    ],
    'bwd:ortho_dist+phase0': [
        'sfgs_rasterize_backward_distortion(*, 1, 0, *, *, 0, 0) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:ortho_dist+phase0+cam+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): camera_grad not supported with an orthographic camera',
    ],
    'bwd:ortho_dist+phase0+cam_intr+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): camera_grad, intrinsics_grad not supported with an orthographic camera',
    ],
    'bwd:ortho_dist+phase0+intr': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): intrinsics_grad not supported with an orthographic camera',
    ],
    'bwd:ortho_dist+phase1+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=1 not supported with an orthographic camera',
    ],
    'bwd:ortho_dist+phase1+cam+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=1, camera_grad not supported with an orthographic camera',
    ],
    'bwd:ortho_dist+phase1+cam_intr': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=1, camera_grad, intrinsics_grad not supported with an orthographic camera',
    ],
    'bwd:ortho_dist+phase1+intr+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=1, intrinsics_grad not supported with an orthographic camera',
    ],
    'bwd:ortho_dist+phase2+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=2 not supported with an orthographic camera',
    ],
    'bwd:ortho_dist+phase2+cam': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=2, camera_grad not supported with an orthographic camera',
    ],
    'bwd:ortho_dist+phase2+cam_intr+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=2, camera_grad, intrinsics_grad not supported with an orthographic camera',
    ],
    'bwd:ortho_dist+phase2+intr+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): phase=2, intrinsics_grad not supported with an orthographic camera',
    ],
    'bwd:q_dist+phase0': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): depth_q_pos not supported with the depth distortion',
    ],
    'bwd:q_dist+phase0+cam+det': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): depth_q_pos not supported with the depth distortion',
    ],
    'bwd:q_dist+phase0+cam_intr+det': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): depth_q_pos not supported with the depth distortion',
    ],
    'bwd:q_dist+phase0+intr': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): depth_q_pos not supported with the depth distortion',
    ],
    'bwd:q_dist+phase1+det': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): depth_q_pos not supported with the depth distortion',
    ],
    'bwd:q_dist+phase1+cam+det': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): depth_q_pos not supported with the depth distortion',
    ],
    'bwd:q_dist+phase1+cam_intr': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): depth_q_pos not supported with the depth distortion',
    ],
    'bwd:q_dist+phase1+intr+det': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): depth_q_pos not supported with the depth distortion',
    ],
    'bwd:q_dist+phase2+det': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): depth_q_pos not supported with the depth distortion',
    ],
    'bwd:q_dist+phase2+cam': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): depth_q_pos not supported with the depth distortion',
    ],
    'bwd:q_dist+phase2+cam_intr+det': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): depth_q_pos not supported with the depth distortion',
    ],
    'bwd:q_dist+phase2+intr+det': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): depth_q_pos not supported with the depth distortion',
    ],
    'bwd:plain+no_off': [
        'sfgs_rasterize_backward() | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:plain+fuse': [
        'sfgs_rasterize_backward() | B3',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:plain+tile_rows': [
        'sfgs_rasterize_backward_deterministic() | B4',
        '-> float32[4, 16]',
    ],
    'bwd:plain+acc_peers': [
        'sfgs_rasterize_backward() | B5',
        '-> None',
    ],
    'bwd:plain+extra': [
        'sfgs_rasterize_backward() | B6',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[4, 2])',
    ],
    'bwd:plain+P0+cam_intr': [
        '-> (float32[0, 3], float32[0, 3], float32[0, 1], float32[0, 3], float32[0, 6], float32[0, 3], float32[0, 0, 3], float32[0, 3], float32[0, 4], float32[0], float32[4, 4], float32[4, 4], float32[3], float32[], float32[])',
    ],
    'bwd:plain+debug': [
        'sfgs_rasterize_backward() | B7',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:plain+no_off+det': [
        'sfgs_rasterize_backward_deterministic() | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:plain+fuse+det': [
        'sfgs_rasterize_backward_deterministic() | B3',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:plain+acc_peers+det': [
        "-> RuntimeError: rasterize_gaussians_backward with acc_peers does not have a deterministic implementation, but you set 'torch.use_deterministic_algorithms(True)'. You can turn off determinism just for this operation, or you can use the 'warn_only=True' option, if that's acceptable for your application.",
    ],
    'bwd:plain+extra+det': [
        "-> RuntimeError: rasterize_gaussians_backward with extra_attrs does not have a deterministic implementation, but you set 'torch.use_deterministic_algorithms(True)'. You can turn off determinism just for this operation, or you can use the 'warn_only=True' option, if that's acceptable for your application.",
    ],
    'bwd:graph+no_off': [
        'sfgs_rasterize_backward_graph(0, 0, 0, 0, 0) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:graph+fuse': [
        'sfgs_rasterize_backward_graph(0, 0, 0, 0, 0) | B3',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:graph+tile_rows': [
        '-> SfgsError: rasterize_gaussians_backward(graph=True): tile_rows, phase=1 (the two-phase backward) cannot be captured in a CUDA graph',
    ],
    'bwd:graph+acc_peers': [
        '-> SfgsError: rasterize_gaussians_backward(graph=True): acc_peers, phase=1 (the two-phase backward) cannot be captured in a CUDA graph',
    ],
    'bwd:graph+extra': [
        'sfgs_rasterize_backward_graph(0, 0, 0, 0, 0) | B6',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[4, 2])',
    ],
    'bwd:graph+P0+cam_intr': [
        '-> (float32[0, 3], float32[0, 3], float32[0, 1], float32[0, 3], float32[0, 6], float32[0, 3], float32[0, 0, 3], float32[0, 3], float32[0, 4], float32[0], float32[4, 4], float32[4, 4], float32[3], float32[], float32[])',
    ],
    'bwd:graph+debug': [
        '-> SfgsError: rasterize_gaussians_backward(graph=True): debug=True (it synchronises after every stage) cannot be captured in a CUDA graph',
    ],
    'bwd:graph+no_off+det': [
        'sfgs_rasterize_backward_graph(0, 1, 0, 0, 0) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:graph+fuse+det': [
        'sfgs_rasterize_backward_graph(0, 1, 0, 0, 0) | B3',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:graph+acc_peers+det': [
        '-> SfgsError: rasterize_gaussians_backward(graph=True): acc_peers, phase=1 (the two-phase backward) cannot be captured in a CUDA graph',
    ],
    'bwd:graph+extra+det': [
        "-> RuntimeError: rasterize_gaussians_backward with extra_attrs does not have a deterministic implementation, but you set 'torch.use_deterministic_algorithms(True)'. You can turn off determinism just for this operation, or you can use the 'warn_only=True' option, if that's acceptable for your application.",
    ],
    'bwd:ortho+no_off': [
        'sfgs_rasterize_backward_ortho(0, 0) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:ortho+fuse': [
        'sfgs_rasterize_backward_ortho(0, 0) | B3',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:ortho+tile_rows': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): tile_rows, phase=1 not supported with an orthographic camera',
    ],
    'bwd:ortho+acc_peers': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): acc_peers, phase=1 not supported with an orthographic camera',
    ],
    'bwd:ortho+extra': [
        'sfgs_rasterize_backward_ortho(0, 0) | B6',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[4, 2])',
    ],
    'bwd:ortho+P0+cam_intr': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): camera_grad, intrinsics_grad not supported with an orthographic camera',
    ],
    'bwd:ortho+debug': [
        'sfgs_rasterize_backward_ortho(0, 0) | B7',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:ortho+no_off+det': [
        'sfgs_rasterize_backward_ortho(0, 1) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:ortho+fuse+det': [
        'sfgs_rasterize_backward_ortho(0, 1) | B3',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:ortho+acc_peers+det': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): acc_peers, phase=1 not supported with an orthographic camera',
    ],
    'bwd:ortho+extra+det': [
        "-> RuntimeError: rasterize_gaussians_backward with extra_attrs does not have a deterministic implementation, but you set 'torch.use_deterministic_algorithms(True)'. You can turn off determinism just for this operation, or you can use the 'warn_only=True' option, if that's acceptable for your application.",
    ],
    'bwd:q+no_off': [
        'sfgs_rasterize_backward_depth_quantile(0, 0, 0, *, *, 0, 0) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:q+fuse': [
        'sfgs_rasterize_backward_depth_quantile(0, 0, 0, *, *, 0, 0) | B3',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:q+tile_rows': [
        '-> SfgsError: rasterize_gaussians_backward(depth_q_pos=...): tile_rows not supported with the depth quantile',
    ],
    'bwd:q+acc_peers': [
        '-> SfgsError: rasterize_gaussians_backward(depth_q_pos=...): acc_peers not supported with the depth quantile',
    ],
    'bwd:q+extra': [
        '-> SfgsError: rasterize_gaussians_backward(depth_q_pos=...): extra_attrs not supported with the depth quantile',
    ],
    'bwd:q+P0+cam_intr': [
        '-> (float32[0, 3], float32[0, 3], float32[0, 1], float32[0, 3], float32[0, 6], float32[0, 3], float32[0, 0, 3], float32[0, 3], float32[0, 4], float32[0], float32[4, 4], float32[4, 4], float32[3], float32[], float32[])',
    ],
    'bwd:q+debug': [
        'sfgs_rasterize_backward_depth_quantile(0, 0, 0, *, *, 0, 0) | B7',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:q+no_off+det': [
        'sfgs_rasterize_backward_depth_quantile(0, 0, 1, *, *, 0, 0) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:q+fuse+det': [
        'sfgs_rasterize_backward_depth_quantile(0, 0, 1, *, *, 0, 0) | B3',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:q+acc_peers+det': [
        '-> SfgsError: rasterize_gaussians_backward(depth_q_pos=...): acc_peers not supported with the depth quantile',
    ],
    'bwd:q+extra+det': [
        '-> SfgsError: rasterize_gaussians_backward(depth_q_pos=...): extra_attrs not supported with the depth quantile',
    ],
    'bwd:dist+no_off': [
        'sfgs_rasterize_backward_distortion(0, 0, 0, *, *, 0, 0) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:dist+fuse': [
        'sfgs_rasterize_backward_distortion(0, 0, 0, *, *, 0, 0) | B3',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:dist+tile_rows': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): tile_rows not supported with the depth distortion',
    ],
    'bwd:dist+acc_peers': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): acc_peers not supported with the depth distortion',
    ],
    'bwd:dist+extra': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): extra_attrs not supported with the depth distortion',
    ],
    'bwd:dist+P0+cam_intr': [
        '-> (float32[0, 3], float32[0, 3], float32[0, 1], float32[0, 3], float32[0, 6], float32[0, 3], float32[0, 0, 3], float32[0, 3], float32[0, 4], float32[0], float32[4, 4], float32[4, 4], float32[3], float32[], float32[])',
    ],
    'bwd:dist+debug': [
        'sfgs_rasterize_backward_distortion(0, 0, 0, *, *, 0, 0) | B7',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:dist+no_off+det': [
        'sfgs_rasterize_backward_distortion(0, 0, 1, *, *, 0, 0) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:dist+fuse+det': [
        'sfgs_rasterize_backward_distortion(0, 0, 1, *, *, 0, 0) | B3',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:dist+acc_peers+det': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): acc_peers not supported with the depth distortion',
    ],
    'bwd:dist+extra+det': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): extra_attrs not supported with the depth distortion',
    ],
    'bwd:ortho_q+no_off': [
        'sfgs_rasterize_backward_depth_quantile(0, 1, 0, *, *, 0, 0) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:ortho_q+fuse': [
        'sfgs_rasterize_backward_depth_quantile(0, 1, 0, *, *, 0, 0) | B3',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:ortho_q+tile_rows': [
        '-> SfgsError: rasterize_gaussians_backward(depth_q_pos=...): tile_rows not supported with the depth quantile',
    ],
    'bwd:ortho_q+acc_peers': [
        '-> SfgsError: rasterize_gaussians_backward(depth_q_pos=...): acc_peers not supported with the depth quantile',
    ],
    'bwd:ortho_q+extra': [
        '-> SfgsError: rasterize_gaussians_backward(depth_q_pos=...): extra_attrs not supported with the depth quantile',
    ],
    'bwd:ortho_q+P0+cam_intr': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): camera_grad, intrinsics_grad not supported with an orthographic camera',
    ],
    'bwd:ortho_q+debug': [
        'sfgs_rasterize_backward_depth_quantile(0, 1, 0, *, *, 0, 0) | B7',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:ortho_q+no_off+det': [
        'sfgs_rasterize_backward_depth_quantile(0, 1, 1, *, *, 0, 0) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:ortho_q+fuse+det': [
        'sfgs_rasterize_backward_depth_quantile(0, 1, 1, *, *, 0, 0) | B3',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:ortho_q+acc_peers+det': [
        '-> SfgsError: rasterize_gaussians_backward(depth_q_pos=...): acc_peers not supported with the depth quantile',
    ],
    'bwd:ortho_q+extra+det': [
        '-> SfgsError: rasterize_gaussians_backward(depth_q_pos=...): extra_attrs not supported with the depth quantile',
    ],
    'bwd:ortho_dist+no_off': [
        'sfgs_rasterize_backward_distortion(0, 1, 0, *, *, 0, 0) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:ortho_dist+fuse': [
        'sfgs_rasterize_backward_distortion(0, 1, 0, *, *, 0, 0) | B3',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:ortho_dist+tile_rows': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): tile_rows not supported with the depth distortion',
    ],
    'bwd:ortho_dist+acc_peers': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): acc_peers not supported with the depth distortion',
    ],
    'bwd:ortho_dist+extra': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): extra_attrs not supported with the depth distortion',
    ],
    'bwd:ortho_dist+P0+cam_intr': [
        '-> SfgsError: rasterize_gaussians_backward(ortho=True): camera_grad, intrinsics_grad not supported with an orthographic camera',
    ],
    'bwd:ortho_dist+debug': [
        'sfgs_rasterize_backward_distortion(0, 1, 0, *, *, 0, 0) | B7',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:ortho_dist+no_off+det': [
        'sfgs_rasterize_backward_distortion(0, 1, 1, *, *, 0, 0) | B0',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:ortho_dist+fuse+det': [
        'sfgs_rasterize_backward_distortion(0, 1, 1, *, *, 0, 0) | B3',
        '-> (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[0])',
    ],
    'bwd:ortho_dist+acc_peers+det': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): acc_peers not supported with the depth distortion',
    ],
    'bwd:ortho_dist+extra+det': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): extra_attrs not supported with the depth distortion',
    ],
    'bwd:q_dist+no_off': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): depth_q_pos not supported with the depth distortion',
    ],
    'bwd:q_dist+fuse': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): depth_q_pos not supported with the depth distortion',
    ],
    'bwd:q_dist+tile_rows': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): depth_q_pos, tile_rows not supported with the depth distortion',
    ],
    'bwd:q_dist+acc_peers': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): depth_q_pos, acc_peers not supported with the depth distortion',
    ],
    'bwd:q_dist+extra': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): depth_q_pos, extra_attrs not supported with the depth distortion',
    ],
    'bwd:q_dist+P0+cam_intr': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): depth_q_pos not supported with the depth distortion',
    ],
    'bwd:q_dist+debug': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): depth_q_pos not supported with the depth distortion',
    ],
    'bwd:q_dist+no_off+det': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): depth_q_pos not supported with the depth distortion',
    ],
    'bwd:q_dist+fuse+det': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): depth_q_pos not supported with the depth distortion',
    ],
    'bwd:q_dist+acc_peers+det': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): depth_q_pos, acc_peers not supported with the depth distortion',
    ],
    'bwd:q_dist+extra+det': [
        '-> SfgsError: rasterize_gaussians_backward(distortion_state=...): depth_q_pos, extra_attrs not supported with the depth distortion',
    ],
    'bwd:plain+P0+phase2+cam': [
        '-> (float32[0, 3], float32[0, 3], float32[0, 1], float32[0, 3], float32[0, 6], float32[0, 3], float32[0, 0, 3], float32[0, 3], float32[0, 4], float32[0], float64[35])',
    ],
    'bwd:plain+P0+phase2+cam_intr': [
        '-> (float32[0, 3], float32[0, 3], float32[0, 1], float32[0, 3], float32[0, 6], float32[0, 3], float32[0, 0, 3], float32[0, 3], float32[0, 4], float32[0], float64[37])',
    ],
    'bwd:plain+P0+phase1': [
        '-> (float32[0, 3], float32[0, 3], float32[0, 1], float32[0, 3], float32[0, 6], float32[0, 3], float32[0, 0, 3], float32[0, 3], float32[0, 4], float32[0])',
    ],
    'bwd:plain+phase1+acc': [
        'sfgs_rasterize_backward() | B1',
        '-> float32[4, 16]',
    ],
    'bwd:plain+acc_peers+phase0': [
        '-> ValueError: acc_peers is a phase-1 option',
    ],
    'bwd:extra+det_warn': [
        'sfgs_rasterize_backward() | B6',
        "-> ((float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 6], float32[4, 3], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[4, 2]), ('rasterize_gaussians_backward with extra_attrs does not have '))",
    ],
    'bwd:q+half_pair': [
        '-> ValueError: depth_q_pos and dL_dout_depth_q come together',
    ],
    'bwd:dist+half_pair': [
        '-> ValueError: distortion_state and dL_dout_distortion come together',
    ],
    'bwd:q+bad_pos': [
        '-> ValueError: depth_q_pos must be a torch.int32 tensor of shape (8, 8) on cpu, got torch.float32 (8, 8) on cpu',
    ],
    'bwd:dist+bad_state': [
        '-> ValueError: distortion_state must be a torch.float32 tensor of shape (2, 8, 8) on cpu, got torch.float32 (1, 8, 8) on cpu',
    ],
    'bwd:off+bad_shape': [
        '-> ValueError: subpixel_offset must be a CUDA float32 tensor of shape (8, 8, 2), got torch.float32 (8, 7, 2) on cpu',
    ],
    'GaussianRasterizer:plain': [
        'sfgs_rasterize_forward() | F5',
        'sfgs_rasterize_backward() | B8',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4], None, None, None, 0.5, 0.25))',
    ],
    'GaussianRasterizer:q': [
        'sfgs_rasterize_forward_depth_quantile(0, 0, 0.5, *, *) | F5',
        'sfgs_rasterize_backward_depth_quantile(0, 0, 0, *, *, 0, 0) | B8',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], float32[1, 8, 8]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4], None, None, None, 0.5, 0.25))',
    ],
    'GaussianRasterizer:dist': [
        'sfgs_rasterize_forward_distortion(0, 0, *, *) | F5',
        'sfgs_rasterize_backward_distortion(0, 0, 0, *, *, 0, 0) | B8',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], float32[1, 8, 8]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4], None, None, None, 0.5, 0.25))',
    ],
    'GaussianRasterizer:q_dist': [
        '-> SfgsError: diff_gauss: depth_distortion and depth_quantile in one call are not supported; render them in two calls',
    ],
    'GaussianRasterizer:precomp': [
        'sfgs_rasterize_forward() | F11',
        'sfgs_rasterize_backward() | B9',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 3], float32[4, 4], None, None, None, 0.5, 0.25))',
    ],
    'GaussianRasterizer:view': [
        'sfgs_rasterize_forward() | F5',
        'sfgs_rasterize_backward_camera(0, 0, *) | B8',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[4, 4], None, None, 0.5, 0.25))',
    ],
    'GaussianRasterizer:proj_campos': [
        'sfgs_rasterize_forward() | F5',
        'sfgs_rasterize_backward_camera(0, 0, *) | B8',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4], None, float32[4, 4], float64[3], 0.5, 0.25))',
    ],
    'GaussianRasterizer:focal': [
        'sfgs_rasterize_forward() | F5',
        'sfgs_rasterize_backward_camera_intrinsics(0, 0, *) | B8',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4], None, None, None, float32[], float32[]))',
    ],
    'GaussianRasterizer:focal_x': [
        'sfgs_rasterize_forward() | F5',
        'sfgs_rasterize_backward_camera_intrinsics(0, 0, *) | B8',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4], None, None, None, float32[], None))',
    ],
    'GaussianRasterizer:focal_cpu_tensor': [
        'sfgs_rasterize_forward() | F5',
        'sfgs_rasterize_backward() | B8',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4], None, None, None, None, None))',
    ],
    'GaussianRasterizer:view_focal': [
        'sfgs_rasterize_forward() | F5',
        'sfgs_rasterize_backward_camera_intrinsics(0, 0, *) | B8',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[4, 4], None, None, float32[], float32[]))',
    ],
    'GaussianRasterizer:q_view_focal': [
        'sfgs_rasterize_forward_depth_quantile(0, 0, 0.5, *, *) | F5',
        'sfgs_rasterize_backward_depth_quantile(0, 0, 0, *, *, *, 37) | B8',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], float32[1, 8, 8]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[4, 4], None, None, float32[], float32[]))',
    ],
    'GaussianRasterizer:dist_focal': [
        'sfgs_rasterize_forward_distortion(0, 0, *, *) | F5',
        'sfgs_rasterize_backward_distortion(0, 0, 0, *, *, *, 37) | B8',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], float32[1, 8, 8]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4], None, None, None, float32[], float32[]))',
    ],
    'GaussianRasterizer:offset_env': [
        'sfgs_rasterize_forward_subpixel(*) | F5',
        'sfgs_rasterize_backward_subpixel(*) | B8',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4], None, None, None, 0.5, 0.25))',
    ],
    'GaussianRasterizer:no_fuse': [
        'sfgs_rasterize_forward() | F0',
        'sfgs_rasterize_backward() | B10',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4], None, None, None, 0.5, 0.25))',
    ],
    'GaussianRasterizer:no_fuse_q': [
        'sfgs_rasterize_forward_depth_quantile(0, 0, 0.5, *, *) | F0',
        'sfgs_rasterize_backward_depth_quantile(0, 0, 0, *, *, 0, 0) | B10',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], float32[1, 8, 8]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4], None, None, None, 0.5, 0.25))',
    ],
    'GaussianRasterizer:debug': [
        'sfgs_rasterize_forward() | F12',
        'sfgs_rasterize_backward() | B11',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4], None, None, None, 0.5, 0.25))',
    ],
    'GaussianRasterizer:det': [
        'sfgs_rasterize_forward() | F5',
        'sfgs_rasterize_backward_deterministic() | B8',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4], None, None, None, 0.5, 0.25))',
    ],
    'GaussianRasterizer:capture': [
        'sfgs_rasterize_forward_graph(0, 0, *) | F13',
        'sfgs_rasterize_backward_graph(0, 0, 0, 0, 0) | B12',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4], None, None, None, 0.5, 0.25))',
    ],
    'GaussianRasterizer:capture_view_focal': [
        'sfgs_rasterize_forward_graph(0, *, *) | F14',
        'sfgs_rasterize_backward_graph(0, 0, *, *, 37) | B13',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4], float32[4, 4], None, None, float32[], float32[]))',
    ],
    'GaussianRasterizer:P0': [
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[0], float32[0]), (float32[0, 3], float32[0, 3], float32[0, 1], float32[0, 3], float32[0, 3], float32[0, 4], None, None, None, 0.5, 0.25))',
    ],
    'GaussianRasterizer:P0_q': [
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[0], float32[0], float32[1, 8, 8]), (float32[0, 3], float32[0, 3], float32[0, 1], float32[0, 3], float32[0, 3], float32[0, 4], None, None, None, 0.5, 0.25))',
    ],
    'GaussianRasterizer:P0_dist_focal': [
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[0], float32[0], float32[1, 8, 8]), (float32[0, 3], float32[0, 3], float32[0, 1], float32[0, 3], float32[0, 3], float32[0, 4], None, None, None, float32[], float32[]))',
    ],
    'GaussianRasterizer:no_colors': [
        '-> Exception: Please provide excatly one of either SHs or precomputed colors!',
    ],
    'OrthoRasterizer:plain': [
        'sfgs_rasterize_forward_ortho(0) | F15',
        'sfgs_rasterize_backward_ortho(0, 0) | B14',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4]))',
    ],
    'OrthoRasterizer:q': [
        'sfgs_rasterize_forward_depth_quantile(0, 1, 0.5, *, *) | F15',
        'sfgs_rasterize_backward_depth_quantile(0, 1, 0, *, *, 0, 0) | B14',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], float32[1, 8, 8]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4]))',
    ],
    'OrthoRasterizer:dist': [
        'sfgs_rasterize_forward_distortion(0, 1, *, *) | F15',
        'sfgs_rasterize_backward_distortion(0, 1, 0, *, *, 0, 0) | B14',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0], float32[1, 8, 8]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4]))',
    ],
    'OrthoRasterizer:q_dist': [
        '-> SfgsError: OrthoRasterizer: depth_distortion and depth_quantile in one call are not supported; render them in two calls',
    ],
    'OrthoRasterizer:precomp': [
        'sfgs_rasterize_forward_ortho(0) | F16',
        'sfgs_rasterize_backward_ortho(0, 0) | B15',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 3], float32[4, 4]))',
    ],
    'OrthoRasterizer:offset_env': [
        'sfgs_rasterize_forward_ortho(*) | F15',
        'sfgs_rasterize_backward_ortho(*, 0) | B14',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4]))',
    ],
    'OrthoRasterizer:debug': [
        'sfgs_rasterize_forward_ortho(0) | F17',
        'sfgs_rasterize_backward_ortho(0, 0) | B16',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4]))',
    ],
    'OrthoRasterizer:det': [
        'sfgs_rasterize_forward_ortho(0) | F15',
        'sfgs_rasterize_backward_ortho(0, 1) | B14',
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[4], float32[0]), (float32[4, 3], float32[4, 3], float32[4, 1], float32[4, 4, 3], float32[4, 3], float32[4, 4]))',
    ],
    'OrthoRasterizer:P0': [
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[0], float32[0]), (float32[0, 3], float32[0, 3], float32[0, 1], float32[0, 3], float32[0, 3], float32[0, 4]))',
    ],
    'OrthoRasterizer:P0_q': [
        '-> ((float32[3, 8, 8], float32[1, 8, 8], float32[3, 8, 8], float32[1, 8, 8], int32[0], float32[0], float32[1, 8, 8]), (float32[0, 3], float32[0, 3], float32[0, 1], float32[0, 3], float32[0, 3], float32[0, 4]))',
    ],
    'OrthoRasterizer:no_colors': [
        '-> Exception: Please provide excatly one of either SHs or precomputed colors!',
    ],
    'render_height_map:q=None,P=4': [
        'sfgs_rasterize_forward_ortho(0) | F18',
        'sfgs_rasterize_backward_ortho(0, 0) | B17',
        '-> (float32[8, 8], (float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 4], float32[4, 4, 3]))',
    ],
    'render_height_map:q=0.5,P=4': [
        'sfgs_rasterize_forward_depth_quantile(0, 1, 0.5, *, *) | F18',
        'sfgs_rasterize_backward_depth_quantile(0, 1, 0, *, *, 0, 0) | B17',
        '-> (float32[8, 8], (float32[4, 3], float32[4, 1], float32[4, 3], float32[4, 4], float32[4, 4, 3]))',
    ],
    'render_height_map:q=0.5,P=0': [
        '-> (float32[8, 8], (float32[0, 3], float32[0, 1], float32[0, 3], float32[0, 4], None))',
    ],
}
