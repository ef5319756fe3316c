"""CUDA-graph capture of the rasterizer (sfgs_rasterize_forward_graph / sfgs_rasterize_backward_graph, sfgs.graphs).

CPU: the capture-safe entries reject what cannot be captured before any CUDA work, and the struct mirrors are those of
the eager entries.  GPU: a captured diff_gauss forward+backward replayed over several cameras equals eager calls; an
overflowed replay is reported and nothing runs past the capacity; a whole captured training step equals the eager
step."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

from helpers import deterministic
from sfgs import graphs, native
from sfgs import synthetic as S

SFGS_E_BADARG, SFGS_E_UNSUPPORTED = -2, -4


# ----------------------------------------------------------------------------- CPU
def _fwd_args():
    a = native.ForwardArgs()
    a.P, a.D, a.M, a.width, a.height = 0, 0, 0, 32, 32
    a.capacity_hint = 1024
    return a


def test_forward_graph_rejects_before_cuda_work():
    L = native.lib()
    word = C.c_uint(0)
    status = C.cast(C.pointer(word), C.c_void_p)
    a = _fwd_args()
    assert L.sfgs_rasterize_forward_graph(C.byref(a), None, None, None) == SFGS_E_BADARG
    assert "null status" in native.last_error()
    a.debug = 1
    assert L.sfgs_rasterize_forward_graph(C.byref(a), None, None, status) == SFGS_E_BADARG
    assert "debug" in native.last_error()
    a.debug, a.capacity_hint = 0, 0
    assert L.sfgs_rasterize_forward_graph(C.byref(a), None, None, status) == SFGS_E_BADARG
    assert "capacity_hint" in native.last_error()
    a.capacity_hint, a.tile_row_begin, a.tile_row_end = 1024, 0, 1
    assert L.sfgs_rasterize_forward_graph(C.byref(a), None, None, status) == SFGS_E_UNSUPPORTED
    assert "tile-row" in native.last_error()
    a.tile_row_end = 0
    peers = (C.c_void_p * 1)(None)
    a.out_peers, a.n_out_peers = C.cast(peers, C.POINTER(C.c_void_p)), 1
    assert L.sfgs_rasterize_forward_graph(C.byref(a), None, None, status) == SFGS_E_UNSUPPORTED
    assert "out_peers" in native.last_error()
    assert word.value == 0


def test_backward_graph_rejects_before_cuda_work():
    L = native.lib()
    b = native.BackwardArgs()
    b.P, b.width, b.height, b.R = 8, 32, 32, 4096
    cam_buf = (C.c_float * 37)()
    cam = C.cast(cam_buf, C.c_void_p)
    b.debug = 1
    assert L.sfgs_rasterize_backward_graph(C.byref(b), None, 0, None, None, 0) == SFGS_E_BADARG
    assert "debug" in native.last_error()
    b.debug, b.R = 0, 0
    assert L.sfgs_rasterize_backward_graph(C.byref(b), None, 0, None, None, 0) == SFGS_E_BADARG
    assert "capacity" in native.last_error()
    b.R = 4096
    assert L.sfgs_rasterize_backward_graph(C.byref(b), None, 0, None, cam, 36) == SFGS_E_BADARG
    assert "ncam" in native.last_error()
    assert L.sfgs_rasterize_backward_graph(C.byref(b), None, 0, None, None, 35) == SFGS_E_BADARG
    assert "dL_dcamera" in native.last_error()
    for phase in (1, 2):
        b.phase = phase
        assert L.sfgs_rasterize_backward_graph(C.byref(b), None, 0, None, None, 0) == SFGS_E_UNSUPPORTED
        assert "phases 1 and 2" in native.last_error()
    b.phase = 0
    peers = (C.c_void_p * 1)(None)
    b.acc_peers, b.n_peers = C.cast(peers, C.POINTER(C.c_void_p)), 1
    assert L.sfgs_rasterize_backward_graph(C.byref(b), None, 0, None, None, 0) == SFGS_E_UNSUPPORTED
    assert "acc_peers" in native.last_error()
    b.acc_peers, b.n_peers, b.tile_row_begin, b.tile_row_end = None, 0, 0, 1
    assert L.sfgs_rasterize_backward_graph(C.byref(b), None, 0, None, None, 0) == SFGS_E_UNSUPPORTED
    assert "tile-row" in native.last_error()


def test_struct_mirrors_unchanged():
    L = native.lib()
    for which, st in enumerate((native.ForwardArgs, native.BackwardArgs)):
        assert L.sfgs_sizeof(which) == C.sizeof(st)
    assert [f[0] for f in native.ForwardArgs._fields_][-2:] == ["out_peers", "n_out_peers"]
    assert [f[0] for f in native.BackwardArgs._fields_][-3:] == ["acc_peers", "n_peers", "peer_slice"]


def test_python_layer_rejects_uncapturable_options():
    from sfgs import rasterizer as R
    z = torch.zeros
    with pytest.raises(native.SfgsError, match="debug=True"):
        R.rasterize_gaussians(z(3), z(4, 3), z(0), z(4, 1), z(4, 3), z(4, 4), 1.0, z(0), z(0), z(0), 0, z(4, 4), z(4, 4),
                              1.0, 1.0, 0.1, 8, 8, z(4, 1, 3), 0, z(3), False, True, capacity_hint=64, graph=True)
    with pytest.raises(native.SfgsError, match="tile_rows"):
        R.rasterize_gaussians(z(3), z(4, 3), z(0), z(4, 1), z(4, 3), z(4, 4), 1.0, z(0), z(0), z(0), 0, z(4, 4), z(4, 4),
                              1.0, 1.0, 0.1, 8, 8, z(4, 1, 3), 0, z(3), False, False, capacity_hint=64, tile_rows=(0, 1),
                              graph=True)
    with pytest.raises(native.SfgsError, match="capacity_hint"):
        R.rasterize_gaussians(z(3), z(4, 3), z(0), z(4, 1), z(4, 3), z(4, 4), 1.0, z(0), z(0), z(0), 0, z(4, 4), z(4, 4),
                              1.0, 1.0, 0.1, 8, 8, z(4, 1, 3), 0, z(3), False, False, graph=True)
    img = z(3, 4, 4)
    for kw, what in ((dict(phase=1), "phase=1"), (dict(phase=2), "phase=2"), (dict(acc_peers=[0]), "acc_peers")):
        with pytest.raises(native.SfgsError, match=what):
            R.rasterize_gaussians_backward(z(3), z(4, 3), z(4, dtype=torch.int32), z(0), z(4, 3), z(4, 4), z(0), 1.0,
                                           z(0), z(0), z(4, 4), z(4, 4), 1.0, 1.0, 0.1, img, z(1, 4, 4), img, z(1, 4, 4),
                                           z(0), z(4, 1, 3), 0, z(3), z(1), 64, z(1), z(1), z(1, 4, 4), False, graph=True,
                                           **kw)


def test_capacity_sources():
    with pytest.raises(native.SfgsError, match="run one eager step first or set a capacity"):
        graphs.resolve_capacity("cuda:0", 12345, 17, 19)
    with graphs.capacity(777):
        assert graphs.resolve_capacity("cuda:0", 12345, 17, 19) == 777
        with graphs.capacity(5):
            assert graphs.resolve_capacity("cuda:0", 12345, 17, 19) == 5
        assert graphs.resolve_capacity("cuda:0", 12345, 17, 19) == 777
    assert graphs.estimate("cuda:0", 12345, 17, 19) is None
    assert graphs.describe(graphs.OVERFLOW | graphs.OFFSET).count(";") == 1


# ----------------------------------------------------------------------------- GPU helpers
def _t(x, dev):
    return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def _cam_tensors(cam, dev):
    return dict(view=_t(cam.viewmatrix, dev), proj=_t(cam.projmatrix, dev), campos=_t(cam.campos, dev),
                tanx=torch.tensor(cam.tanfovx, dtype=torch.float32, device=dev),
                tany=torch.tensor(cam.tanfovy, dtype=torch.float32, device=dev))


_SCENE = {}


def _city(P=1_000_000):
    if P not in _SCENE:
        _SCENE[P] = S.city_scene(P, seed=0, sh_degree=3)
    return _SCENE[P]


CAMERAS = [S.jax004_camera(), S.orbit_camera(azimuth_deg=30.0), S.orbit_camera(azimuth_deg=120.0, fov_deg=50.0),
           S.orbit_camera(azimuth_deg=250.0, fov_deg=70.0, elevation_deg=80.0)]


# ----------------------------------------------------------------------------- GPU: rasterizer replay
@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["sh", "subpixel", "precomp", "camera", "default_mode"])
def test_rasterizer_replay_equals_eager(cuda_device, variant, monkeypatch):
    import diff_gauss
    from diff_gauss import GaussianRasterizationSettings, GaussianRasterizer
    from sfgs import rasterizer as R
    dev = cuda_device
    scene = _city()
    P, H, W = scene.P, CAMERAS[0].height, CAMERAS[0].width
    assert all((c.height, c.width) == (H, W) for c in CAMERAS)
    if variant == "subpixel":
        monkeypatch.setattr(diff_gauss, "SUBPIXEL_OFFSET", True)
    g = torch.Generator(device=dev).manual_seed(7)
    means = _t(scene.means3D, dev).requires_grad_(True)
    scales, rots = _t(scene.scales, dev).requires_grad_(True), _t(scene.rotations, dev).requires_grad_(True)
    opac = _t(scene.opacities, dev).requires_grad_(True)
    shs = _t(scene.shs, dev).requires_grad_(True)
    colors = torch.rand((P, 3), device=dev, generator=g).requires_grad_(True)
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    static = _cam_tensors(CAMERAS[0], dev)
    cam_grad = variant == "camera"
    for k in static:
        static[k].requires_grad_(cam_grad)
    offset = torch.zeros((H, W, 2), device=dev)
    cot = [torch.randn(s, device=dev, generator=g) for s in ((3, H, W), (1, H, W), (3, H, W), (1, H, W))]
    leaves = [means, scales, rots, opac] + ([colors] if variant == "precomp" else [shs])
    if cam_grad:
        leaves += [static["view"], static["proj"], static["campos"], static["tanx"], static["tany"]]

    def step():
        m2d = torch.zeros((P, 3), device=dev, requires_grad=True)
        rs = GaussianRasterizationSettings(H, W, static["tanx"], static["tany"], 0.1, offset, bg, 1.0, static["view"],
                                           static["proj"], 3, static["campos"], False, False)
        kw = dict(colors_precomp=colors) if variant == "precomp" else dict(shs=shs)
        color, depth, norm, alpha, radii, _ = GaussianRasterizer(rs)(means, m2d, opac, scales=scales, rotations=rots, **kw)
        loss = sum((o * c).sum() for o, c in zip((color, depth, norm, alpha), cot))
        grads = torch.autograd.grad(loss, [m2d] + leaves)
        return (color, depth, norm, alpha, radii) + tuple(grads)

    def load(cam):
        with torch.no_grad():
            for k, v in _cam_tensors(cam, dev).items():
                static[k].copy_(v)
            offset.copy_(torch.rand((H, W, 2), device=dev, generator=g) - 0.5 if variant == "subpixel" else 0.0)

    e = torch.empty(0, device=dev)
    Rmax = 0
    for cam in CAMERAS:
        f = R.rasterize_gaussians(bg, means.detach(), e, opac.detach(), scales.detach(), rots.detach(), 1.0, e, e, e, 0,
                                  _t(cam.viewmatrix, dev), _t(cam.projmatrix, dev), cam.tanfovx, cam.tanfovy, 0.1, H, W,
                                  shs.detach(), 3, _t(cam.campos, dev), False, False)
        Rmax = max(Rmax, f[0])
    graphs.status(dev)
    with deterministic(variant != "default_mode"):
        load(CAMERAS[0])
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            step()                                   # warm-up on a side stream, as torch.cuda.graph asks
        torch.cuda.current_stream(dev).wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with graphs.capacity(Rmax + Rmax // 8 + 4096), torch.cuda.graph(graph):
            outs = step()
        for cam in CAMERAS:
            load(cam)
            graph.replay()
            replayed = [o.clone() for o in outs]
            graphs.check(dev)
            eager = step()
            torch.cuda.synchronize(dev)
            for i, (a, b) in enumerate(zip(replayed, eager)):
                # images and radii always; every gradient (means2D.grad first) when deterministic -- the default
                # backward's atomics make even two eager calls differ in the last bits
                if i < 5 or variant != "default_mode":
                    assert torch.equal(a, b), (variant, i)
                else:
                    tol = 1e-3 * float(b.abs().max()) + 1e-6
                    assert float((a - b).abs().max()) <= tol, (variant, i)


# ----------------------------------------------------------------------------- GPU: overflow
class _GuardArena:
    """Allocator target whose buffers carry a guard region filled with a known pattern behind the requested bytes."""
    GUARD = 0
    handed = []

    def __init__(self, device):
        self.device = device
        self.tensor = None
        self.cb = native.ALLOC_FN(self._alloc)

    def _alloc(self, _user, nbytes):
        try:
            buf = torch.full((int(nbytes) + self.GUARD,), 0xA5, dtype=torch.uint8, device=self.device)
            self.tensor = buf
            _GuardArena.handed.append((buf, int(nbytes)))
            return buf.data_ptr()
        except Exception:  # noqa: BLE001 - must not raise through the C ABI
            return None


@pytest.mark.gpu
def test_overflow_is_reported_and_never_run_past(cuda_device, monkeypatch):
    from sfgs import rasterizer as R
    dev = cuda_device
    scene = S.blob_scene(20000, seed=3)
    cam = S.simple_camera(320, 240)
    e = torch.empty(0, device=dev)
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    args = lambda: (bg, _t(scene.means3D, dev), e, _t(scene.opacities, dev), _t(scene.scales, dev),  # noqa: E731
                    _t(scene.rotations, dev), 1.0, e, e, e, 0, _t(cam.viewmatrix, dev), _t(cam.projmatrix, dev),
                    cam.tanfovx, cam.tanfovy, 0.1, cam.height, cam.width, _t(scene.shs, dev), scene.sh_degree,
                    _t(cam.campos, dev), False, False)
    eager = R.rasterize_gaussians(*args())
    Rtrue = eager[0]
    assert Rtrue > 1000
    # the guard is at least as large as the eager binning buffer and the deterministic scratch of the true count
    _GuardArena.GUARD = int(native.lib().sfgs_binning_bytes(2 * Rtrue)) + 524 * 2 * Rtrue + 4 * scene.P
    monkeypatch.setattr(R, "_Arena", _GuardArena)
    graphs.status(dev)
    H, W = cam.height, cam.width
    cot = [torch.rand(s, device=dev) for s in ((3, H, W), (1, H, W), (3, H, W), (1, H, W))]

    def run(capacity, det):
        _GuardArena.handed.clear()
        a = args()
        f = R.rasterize_gaussians(*a, capacity_hint=capacity, graph=True)
        with deterministic(det):
            grads = R.rasterize_gaussians_backward(bg, a[1], f[5], e, a[4], a[5], e, 1.0, e, e, a[11], a[12],
                                                   cam.tanfovx, cam.tanfovy, 0.1, *cot, e, a[18], scene.sh_degree,
                                                   a[20], f[7], capacity, f[8], f[9], f[4], False, graph=True)
        torch.cuda.synchronize(dev)
        for buf, n in _GuardArena.handed:
            assert bool((buf[n:] == 0xA5).all()), "a kernel wrote past its buffer"
        return f, grads

    for det in (False, True):
        f, grads = run(Rtrue // 2, det)
        assert graphs.status(dev) & graphs.OVERFLOW
        assert float(grads[0].abs().max()) == 0.0          # means2D gradient: only the blend adjoint forms it
    f, grads = run(Rtrue + 4096, True)
    assert graphs.status(dev) == 0
    for i in (1, 2, 3, 4, 5):
        assert torch.equal(f[i], eager[i]), i


# ----------------------------------------------------------------------------- GPU: whole training step
def _train(dev, mode, steps=20, warmup=3, appearance=False, P=400_000):
    from diff_gauss import GaussianRasterizationSettings, GaussianRasterizer
    from fused_ssim import fused_ssim
    from sfgs import densify as DN
    from sfgs.activations import fused_activations
    from sfgs.appearance import fused_appearance_colors
    scene = _city(P)
    cams = [S.orbit_camera(azimuth_deg=45.0 * k, width=960, height=540) for k in range(8)]
    H, W = cams[0].height, cams[0].width
    torch.manual_seed(0)
    rng = np.random.default_rng(1)
    xyz = _t((scene.means3D + rng.normal(0, 0.05, scene.means3D.shape)).astype(np.float32), dev).requires_grad_(True)
    scaling = torch.log(_t(scene.scales, dev)).requires_grad_(True)
    rotation = _t(scene.rotations, dev).clone().requires_grad_(True)
    opacity = torch.logit(_t(scene.opacities, dev).clamp(1e-4, 1 - 1e-4)).reshape(P, 1).clone().requires_grad_(True)
    shs = (_t(scene.shs, dev) * 0.9).requires_grad_(True)
    params = [xyz, scaling, rotation, opacity, shs]
    if appearance:
        M = 4
        feats = (_t(scene.shs, dev)[:, :M] * 0.9).contiguous().requires_grad_(True)
        gemb = (torch.randn((P, 24), device=dev) * 0.1).requires_grad_(True)
        aembs = torch.randn((8, 32), device=dev) * 0.1
        mlp = torch.nn.Sequential(torch.nn.Linear(3 + 24 + 32, 128), torch.nn.ReLU(), torch.nn.Linear(128, 128),
                                  torch.nn.ReLU(), torch.nn.Linear(128, 6)).to(dev)
        params = [xyz, scaling, rotation, opacity, feats, gemb] + list(mlp.parameters())
    filter_3D = torch.full((P, 1), 0.05, dtype=torch.float64, device=dev)
    lr = lambda v: torch.tensor(v, device=dev)  # noqa: E731
    opt = torch.optim.Adam([{"params": [p], "lr": lr(1e-3)} for p in params], eps=1e-15, capturable=True)
    bg = torch.zeros(3, device=dev)
    targets = [torch.rand((3, H, W), device=dev) for _ in cams]
    static = dict(_cam_tensors(cams[0], dev), gt=targets[0].clone(), cam_idx=torch.zeros((), dtype=torch.long, device=dev))
    z = lambda: torch.zeros(P, device=dev)  # noqa: E731
    stats = types.SimpleNamespace(max_radii2D=z(), xyz_gradient_accum=z(), xyz_gradient_accum_abs=z(),
                                  xyz_gradient_accum_abs_max=z(), denom=z())

    def load(i):
        with torch.no_grad():
            for k, v in _cam_tensors(cams[i % 8], dev).items():
                static[k].copy_(v)
            static["gt"].copy_(targets[i % 8])
            static["cam_idx"].fill_(i % 8)

    def step():
        op, sc, rot = fused_activations(opacity, scaling, rotation, filter_3D)
        m2d = torch.zeros((P, 3), device=dev, requires_grad=True)
        rs = GaussianRasterizationSettings(H, W, static["tanx"], static["tany"], 0.1, torch.zeros(1, device=dev), bg, 1.0,
                                           static["view"], static["proj"], 3, static["campos"], False, False)
        if appearance:
            aemb = aembs.index_select(0, static["cam_idx"].reshape(1))[0]   # indexing with the tensor itself syncs
            colors = fused_appearance_colors(feats, gemb, aemb, mlp, xyz, static["campos"], 1, fused_backward=True)
            out = GaussianRasterizer(rs)(xyz, m2d, op, colors_precomp=colors, scales=sc, rotations=rot)
        else:
            out = GaussianRasterizer(rs)(xyz, m2d, op, shs=shs, scales=sc, rotations=rot)
        color, radii = out[0], out[4]
        gt = static["gt"]
        loss = 0.8 * torch.nn.functional.l1_loss(color, gt) + 0.2 * (1.0 - fused_ssim(color[None], gt[None]))
        loss.backward()
        opt.step()
        vs = types.SimpleNamespace(grad=torch.nn.functional.pad(m2d.grad, (0, 1)).contiguous())
        DN.add_densification_stats(stats, vs, radii)
        return loss.detach()

    graphs.status(dev)
    with deterministic(True):
        for i in range(warmup):
            load(i)
            opt.zero_grad(set_to_none=True)
            step()
        if mode == "graph":
            opt.zero_grad(set_to_none=True)
            graph = torch.cuda.CUDAGraph()
            side = torch.cuda.Stream(dev)
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                with torch.cuda.graph(graph):
                    step()
            torch.cuda.current_stream(dev).wait_stream(side)
            for i in range(warmup, warmup + steps):
                load(i)
                for p in params:
                    p.grad.zero_()
                graph.replay()
                graphs.check(dev)
        else:
            for i in range(warmup, warmup + steps):
                load(i)
                opt.zero_grad(set_to_none=True)
                step()
    torch.cuda.synchronize(dev)
    state = [opt.state[p][k] for p in params for k in ("exp_avg", "exp_avg_sq", "step")]
    return [p.detach().clone() for p in params] + [s.clone() for s in state] + [
        getattr(stats, k).clone() for k in vars(stats)]


@pytest.mark.gpu
@pytest.mark.parametrize("appearance", [False, True], ids=["sh3", "appearance_m4"])
def test_whole_training_step_replay_equals_eager(cuda_device, appearance):
    eager = _train(cuda_device, "eager", appearance=appearance)
    replay = _train(cuda_device, "graph", appearance=appearance)
    assert len(eager) == len(replay)
    for i, (a, b) in enumerate(zip(eager, replay)):
        assert torch.equal(a, b), i
