"""The tile-row sharded mode with the rasterizer's newer options: subpixel offsets through the band forward, the fused
image all-gather (out_peers) and the fused reduce-scatter (acc_peers), and camera / focal gradients formed from the
phase-2 Gaussian slices (sfgs_rasterize_backward_camera_partial) and summed across ranks
(sfgs.multigpu.reduce_camera_gradients).

CPU: the C ABI's argument checks, and world-size-2 gloo runs of the cross-rank camera sum and of the ordered
reduce-scatter.  GPU (one device; the "peers" are local buffers): bands reassemble the one-call frame bit for bit,
per-band and peer phase-1 sums equal the one-call sums, and the slices' camera partials, added and rounded once, match
the float64 restatement within the bound the one-call camera gradients meet."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import chain_f64 as CH
import helpers as Hh
from helpers import release_cached_frames  # noqa: F401
from sfgs import multigpu as MG
from sfgs import synthetic as S

SFGS_E_BADARG, SFGS_E_UNSUPPORTED = -2, -4
GRAD_KEYS = ("means2D", "colors", "opacity", "means3D", "cov3D", "norm3D", "sh", "scales", "rot")


# ----------------------------------------------------------------------------- CPU: argument checks
def test_abi_rejections_before_cuda_work():
    """Without a device any CUDA call fails with SFGS_E_CUDA: each expected code shows the check ran first."""
    from sfgs import native as N
    L = N.lib()
    dummy = (C.c_double * 64)()
    ptr = C.cast(dummy, C.c_void_p)
    peers = (C.c_void_p * 1)(ptr)

    def bargs(**kw):
        b = N.BackwardArgs()
        b.P, b.width, b.height = 8, 32, 32
        b.scratch_alloc = N.ALLOC_FN(lambda _u, _n: None)
        for k, v in kw.items():
            setattr(b, k, v)
        return b

    slice2 = dict(phase=2, acc=ptr, gauss_begin=0, gauss_end=8)
    partial = L.sfgs_rasterize_backward_camera_partial
    cases = [
        (bargs(**slice2), None, 0, 35, None, SFGS_E_BADARG, "null dL_dcamera_partial"),
        (bargs(**slice2), None, 0, 36, ptr, SFGS_E_BADARG, "ncam"),
        (bargs(), None, 0, 35, ptr, SFGS_E_UNSUPPORTED, "phase 2 only"),
        (bargs(phase=1, acc=ptr), ptr, 0, 37, ptr, SFGS_E_UNSUPPORTED, "phase 2 only"),
        (bargs(ED=2, **slice2), None, 0, 35, ptr, SFGS_E_UNSUPPORTED, "extra_attrs"),
        (bargs(ED=2, **slice2), ptr, 1, 37, ptr, SFGS_E_UNSUPPORTED, "extra_attrs"),
    ]
    nalloc = bargs(**slice2)
    nalloc.scratch_alloc = N.ALLOC_FN()
    cases.append((nalloc, None, 0, 35, ptr, SFGS_E_BADARG, "scratch"))
    for b, off, det, ncam, dst, code, what in cases:
        assert partial(C.byref(b), off, det, ncam, dst) == code, what
        assert what in N.last_error(), (what, N.last_error())
    assert partial(None, None, 0, 35, ptr) == SFGS_E_BADARG

    # offsets with extra_attrs stay unsupported, in one phase or two; the deterministic backward has no acc_peers
    assert L.sfgs_rasterize_backward_subpixel(C.byref(bargs(ED=2, phase=1, acc=ptr)), ptr) == SFGS_E_UNSUPPORTED
    assert "extra_attrs" in N.last_error()
    pa = bargs(phase=1, n_peers=1, peer_slice=8)
    pa.acc_peers = C.cast(peers, C.POINTER(C.c_void_p))
    assert L.sfgs_rasterize_backward_deterministic_subpixel(C.byref(pa), ptr) == SFGS_E_UNSUPPORTED
    assert "acc_peers" in N.last_error()
    assert L.sfgs_rasterize_backward_deterministic(C.byref(pa)) == SFGS_E_UNSUPPORTED
    fa = N.ForwardArgs()
    fa.P, fa.width, fa.height, fa.ED = 8, 32, 32, 2
    fa.out_peers, fa.n_out_peers = C.cast(peers, C.POINTER(C.c_void_p)), 1
    assert L.sfgs_rasterize_forward_subpixel(C.byref(fa), ptr) == SFGS_E_UNSUPPORTED
    assert "extra_attrs" in N.last_error()


def test_subpixel_peers_entries_accept_peers_before_cuda_work():
    """The _subpixel_peers entries pass out_peers / acc_peers through the offset checks (the calls then fail later on
    the missing buffers, still before any CUDA work) and still reject extra_attrs; the _subpixel entries keep
    rejecting the peer pointers."""
    from sfgs import native as N
    L = N.lib()
    dummy = (C.c_float * 64)()
    ptr = C.cast(dummy, C.c_void_p)
    peers = (C.c_void_p * 1)(ptr)
    a = N.ForwardArgs()
    a.P, a.width, a.height, a.ED = 8, 32, 32, 2
    assert L.sfgs_rasterize_forward_subpixel_peers(C.byref(a), ptr) == SFGS_E_UNSUPPORTED
    assert "extra_attrs" in N.last_error()
    a.ED = 0
    a.out_peers, a.n_out_peers = C.cast(peers, C.POINTER(C.c_void_p)), 1
    assert L.sfgs_rasterize_forward_subpixel_peers(C.byref(a), ptr) == SFGS_E_BADARG and "null output" in N.last_error()
    assert L.sfgs_rasterize_forward_subpixel(C.byref(a), ptr) == SFGS_E_UNSUPPORTED
    assert "sfgs_rasterize_forward_subpixel_peers" in N.last_error()
    assert L.sfgs_rasterize_forward_subpixel_peers(None, ptr) == SFGS_E_BADARG
    b = N.BackwardArgs()
    b.P, b.width, b.height, b.ED = 8, 32, 32, 2
    assert L.sfgs_rasterize_backward_subpixel_peers(C.byref(b), ptr) == SFGS_E_UNSUPPORTED
    assert "extra_attrs" in N.last_error()
    b.ED, b.phase, b.acc = 0, 1, ptr
    b.acc_peers, b.n_peers, b.peer_slice = C.cast(peers, C.POINTER(C.c_void_p)), 1, 8
    assert L.sfgs_rasterize_backward_subpixel_peers(C.byref(b), ptr) == SFGS_E_BADARG
    assert "null scratch buffer" in N.last_error()
    assert L.sfgs_rasterize_backward_subpixel(C.byref(b), ptr) == SFGS_E_UNSUPPORTED
    assert "sfgs_rasterize_backward_subpixel_peers" in N.last_error()
    assert L.sfgs_rasterize_backward_subpixel_peers(None, ptr) == SFGS_E_BADARG


# ----------------------------------------------------------------------------- CPU: gloo world size 2
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out, received):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        res = {}
        # camera partials: entry 0 is 1 + 2^-24 on rank 0 and 2^-24 on rank 1.  Rounded once, the sum is 1 + 2^-23;
        # rounding each partial first gives 1 + 2^-24 -> 1.0 (a tie to even).
        g = torch.Generator().manual_seed(11)
        parts = [torch.randn(37, generator=g, dtype=torch.float64) * 10.0 ** torch.randint(-3, 4, (37,), generator=g)
                 for _ in range(world)]
        parts[0][0], parts[1][0] = 1.0 + 2.0 ** -24, 2.0 ** -24
        want = (parts[0] + parts[1]).float()
        assert want[0].item() == 1.0 + 2.0 ** -23 and (parts[0].float() + parts[1].float())[0].item() == 1.0
        r37 = MG.reduce_camera_gradients(parts[rank].clone())
        r35 = MG.reduce_camera_gradients(parts[rank][:35].clone())
        res["cam37"] = torch.cat([r37[0].reshape(16), r37[1].reshape(16), r37[2], r37[3].reshape(1), r37[4].reshape(1)])
        res["cam35"] = torch.cat([r35[0].reshape(16), r35[1].reshape(16), r35[2]])
        res["cam_ok"] = (len(r37) == 5 and len(r35) == 3 and r37[0].shape == (4, 4) and r37[3].shape == ()
                         and torch.equal(res["cam37"], want) and torch.equal(res["cam35"], want[:35]))
        # ordered reduce-scatter against all_reduce + slice: P = 7 over 2 ranks (ragged slices)
        P = 7
        acc = torch.randn((P, 16), generator=torch.Generator().manual_seed(100 + rank))
        mine = MG.reduce_scatter_sums(acc.clone(), ordered=True)
        full = torch.cat([acc, acc.new_zeros((1, 16))], 0)
        dist.all_reduce(full)
        res["rs_ok"] = mine.shape == (4, 16) and torch.equal(mine, full[rank * 4:(rank + 1) * 4])
        res["rs"] = mine
        out.put((rank, res))
        # the result tensors travel as file descriptors this process serves: it must outlive their unpickling
        received.wait(timeout=120)
    finally:
        dist.destroy_process_group()


def test_camera_sum_and_ordered_reduce_scatter_world2_gloo():
    ctx = mp.get_context("spawn")
    q, received = ctx.Queue(), ctx.Event()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q, received)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        res = dict(q.get(timeout=120) for _ in procs)
    finally:
        received.set()
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [0, 1]
    assert res[0]["cam_ok"] and res[1]["cam_ok"], "rank-order float64 sum rounded once"
    assert torch.equal(res[0]["cam37"], res[1]["cam37"]) and torch.equal(res[0]["cam35"], res[1]["cam35"])
    assert res[0]["rs_ok"] and res[1]["rs_ok"], "ordered reduce-scatter differs from all_reduce + slice"
    assert torch.equal(res[1]["rs"][3], torch.zeros(16))          # the row past P


# ----------------------------------------------------------------------------- GPU
def _city(dev, D=3, P=120_000, extent=120.0, seed=9):
    scene, cam = S.city_scene(P, seed=seed, sh_degree=D, extent=extent), S.jax004_camera(640, 360)
    return scene, cam, Hh.to_torch(scene, cam, dev)


def _planes(f):
    return torch.cat([f["color"], f["depth"], f["alpha"], f["norm"]], 0)     # the out_peers plane order


def _cuts(f, scene, cam, n):
    it = Hh.our_internals(f, scene.P, cam.height, cam.width)
    return MG.partition_rows(MG.row_histogram(it["ranges"], (cam.width + 15) // 16), n)


@pytest.mark.gpu
def test_bands_with_offsets_reassemble_the_frame(cuda_device):
    """Three bands with U(-0.5, 0.5) offsets, rendered into local outputs, into one "peer" frame block, and into two
    "peer" blocks that are the halves of one buffer: colour, depth, alpha, normal and n_contrib equal the one-call
    _subpixel frame bit for bit."""
    dev = cuda_device
    scene, cam, d = _city(dev)
    H, W = cam.height, cam.width
    bg = torch.tensor([0.1, 0.0, 0.2], device=dev)
    off = Hh.uniform_offsets(cam.height, cam.width, dev, 23)
    full = Hh.run_ours_forward(d, cam, 3, bg, subpixel_offset=off)
    full_nc = Hh.our_internals(full, scene.P, H, W)["n_contrib"].view(H, W)
    want = _planes(full)
    assert not torch.equal(want, _planes(Hh.run_ours_forward(d, cam, 3, bg)))          # the offsets move the samples
    cuts = _cuts(full, scene, cam, 3)
    one = torch.full((8 * H * W,), float("nan"), device=dev)
    two = torch.full((2, 8 * H * W), float("nan"), device=dev)
    total_R = 0
    for g in range(3):
        band = (cuts[g], cuts[g + 1])
        y0, y1 = MG.band_pixel_rows(cuts, g, H)
        f = Hh.run_ours_forward(d, cam, 3, bg, subpixel_offset=off, tile_rows=band)
        total_R += f["num_rendered"]
        assert torch.equal(_planes(f)[:, y0:y1], want[:, y0:y1]), g
        assert torch.equal(f["radii"], full["radii"])
        for fp in (Hh.run_ours_forward(d, cam, 3, bg, subpixel_offset=off, tile_rows=band, out_planes=one,
                                       out_peers=[one.data_ptr()]),
                   Hh.run_ours_forward(d, cam, 3, bg, subpixel_offset=off, tile_rows=band, out_planes=two[0],
                                       out_peers=[two[0].data_ptr(), two[1].data_ptr()]),
                   f):
            nc = Hh.our_internals(fp, scene.P, H, W)["n_contrib"].view(H, W)
            assert torch.equal(nc[y0:y1], full_nc[y0:y1]), g
    assert total_R == full["num_rendered"]
    torch.cuda.synchronize(dev)
    assert torch.equal(one.view(8, H, W), want)
    assert torch.equal(two[0].view(8, H, W), want) and torch.equal(two[1].view(8, H, W), want)


@pytest.mark.gpu
def test_phase1_band_and_peer_sums_with_offsets(cuda_device):
    """Per-band phase-1 sums with offsets, added, and the acc_peers forms (one peer; two peers that are the halves of
    one buffer) equal the one-call _subpixel sums within the two-phase tolerance."""
    dev = cuda_device
    scene, cam, d = _city(dev)
    bg = torch.tensor([0.1, 0.0, 0.2], device=dev)
    off = Hh.uniform_offsets(cam.height, cam.width, dev, 23)
    cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height, seed=2)]
    P = scene.P
    full = Hh.run_ours_forward(d, cam, 3, bg, subpixel_offset=off)
    ref = Hh.run_ours_backward(d, cam, 3, bg, full, cot, subpixel_offset=off, phase=1)
    tol = 1e-5 + 2e-4 * ref.abs().max().item()
    cuts = _cuts(full, scene, cam, 3)
    half = (P + 1) // 2
    acc_p = torch.zeros((P, 16), device=dev)
    acc_q = torch.zeros((2 * half, 16), device=dev)
    total = torch.zeros((P, 16), device=dev)
    for g in range(3):
        band = (cuts[g], cuts[g + 1])
        f = Hh.run_ours_forward(d, cam, 3, bg, subpixel_offset=off, tile_rows=band)
        total += Hh.run_ours_backward(d, cam, 3, bg, f, cot, subpixel_offset=off, tile_rows=band, phase=1)
        assert Hh.run_ours_backward(d, cam, 3, bg, f, cot, subpixel_offset=off, tile_rows=band, phase=1,
                                    acc_peers=[acc_p.data_ptr()], peer_slice=P) is None
        Hh.run_ours_backward(d, cam, 3, bg, f, cot, subpixel_offset=off, tile_rows=band, phase=1,
                             acc_peers=[acc_q.data_ptr(), acc_q[half:].data_ptr()], peer_slice=half)
    torch.cuda.synchronize(dev)
    for name, got in (("bands", total), ("one peer", acc_p), ("two peers", acc_q[:P])):
        assert (got - ref).abs().max().item() <= tol, name
    # the offsets matter here: the sums without them differ by far more
    plain = Hh.run_ours_backward(d, cam, 3, bg, Hh.run_ours_forward(d, cam, 3, bg), cot, phase=1)
    assert (plain - ref).abs().max().item() > 10 * tol


def _camera_case(name, jitter, dev):
    """One-call deterministic camera + focal gradients, the deterministic phase-1 sums, and the float64 / float32
    restatements on those sums, for a 200k-Gaussian city frame at 640x360."""
    def make():
        D = 3 if name == "d3" else 1
        scene, cam, d = _city(dev, D=D, P=200_000, extent=128.0, seed=4)
        colors = None
        if name == "precomp":
            colors = np.random.default_rng(5).uniform(0, 1, size=(scene.P, 3)).astype(np.float32)
            colors = torch.from_numpy(colors).to(dev)
        bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
        off = Hh.uniform_offsets(cam.height, cam.width, dev, 23) if jitter else None
        f = Hh.run_ours_forward(d, cam, D, bg, subpixel_offset=off, colors=colors)
        cot = [torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width, cam.height, seed=6)]
        one = Hh.run_ours_backward(d, cam, D, bg, f, cot, subpixel_offset=off, colors=colors, det=True,
                                   camera_grad=True, intrinsics_grad=True)
        one = torch.cat([one["view"].reshape(16), one["proj"].reshape(16), one["campos"], one["tanx"].reshape(1),
                         one["tany"].reshape(1)])
        a = Hh.restatement_inputs(f, d, cam, D, bg, cot, colors, off)

        def flat(r):
            return torch.cat([r["view"].reshape(16), r["proj"].reshape(16), r["campos"].reshape(3),
                              r["tanx"].reshape(1), r["tany"].reshape(1)]).double()
        r64, r32 = CH.chain(**a, focal=True, dtype=torch.float64), CH.chain(**a, focal=True, dtype=torch.float32)
        return (scene, cam, d, D, colors, bg, off, f, cot, a["acc"], one.double(), flat(r64), flat(r32),
                r64["abs"].double())
    return Hh.cached("case", (name, jitter), make)


@pytest.mark.gpu
@pytest.mark.parametrize("jitter", [False, True], ids=["plain", "jitter"])
@pytest.mark.parametrize("name", ["d3", "d1", "precomp"])
def test_camera_partials_of_two_slices(cuda_device, name, jitter):
    """Slices [0, 2173) and [2173, P) (the cut is not a multiple of the 96-Gaussian span): their float64 partials,
    added and rounded once, are within the camera tests' bound of the float64 restatement (twice the float32
    restatement's error, or 1e-6 of the sum of the terms' magnitudes), and so within it of the one-call gradients.
    Three deterministic repeats of each partial are byte-identical, and the ten gradient tensors of each slice are
    bit-identical to the phase-2 call without camera terms."""
    dev = cuda_device
    scene, cam, d, D, colors, bg, off, f, cot, acc, one, f64, f32, mag = _camera_case(name, jitter, dev)
    P, cut = scene.P, 2173
    tol = torch.maximum(2.0 * (f32 - f64).abs(), 1e-6 * mag)
    assert ((one - f64).abs() <= tol).all()                       # the one-call gradients meet the bound themselves
    for ncam in (35, 37):
        partials = []
        for a, b in ((0, cut), (cut, P)):
            kw = dict(phase=2, gauss_range=(a, b), colors=colors, det=True)
            runs = [Hh.run_ours_backward(d, cam, D, bg, f, cot, subpixel_offset=off, acc=acc[a:b].clone(),
                                         camera_grad=True, intrinsics_grad=ncam == 37, **kw) for _ in range(3)]
            assert len(runs[0]) == 11
            part = runs[0][10]
            assert part.dtype == torch.float64 and part.shape == (ncam,)
            for r in runs[1:]:
                assert torch.equal(r[10].view(torch.int64), part.view(torch.int64)), (ncam, a)
            plain = Hh.run_ours_backward(d, cam, D, bg, f, cot, subpixel_offset=off, acc=acc[a:b].clone(), **kw)
            for k, x in zip(GRAD_KEYS, runs[0][:9]):
                if colors is not None and k == "sh":
                    continue
                assert torch.equal(Hh.bits(x[a:b]), Hh.bits(plain[k][a:b])), (ncam, a, k)
            partials.append(part)
        got = (partials[0] + partials[1]).float().double()
        err = (got - f64[:ncam]).abs()
        print(f"\n[{name} {'jitter' if jitter else 'plain'} ncam {ncam}] max err / tol "
              f"{float((err / tol[:ncam].clamp_min(1e-300)).max()):.3f}, "
              f"max |sharded - one call| / tol {float(((got - one[:ncam]).abs() / tol[:ncam].clamp_min(1e-300)).max()):.3g}")
        assert (err <= tol[:ncam]).all(), (ncam, err, tol[:ncam])
        assert ((got - one[:ncam]).abs() <= tol[:ncam]).all(), ncam
        if colors is not None:
            assert torch.equal(got[32:35], torch.zeros(3, dtype=torch.float64, device=dev))


@pytest.mark.gpu
def test_empty_slice_writes_zero_partials(cuda_device):
    dev = cuda_device
    scene, cam, d, D, colors, bg, off, f, cot, acc, *_ = _camera_case("d3", True, dev)
    for ncam in (35, 37):
        r = Hh.run_ours_backward(d, cam, D, bg, f, cot, subpixel_offset=off, phase=2, gauss_range=(5, 5),
                                 acc=acc[5:6].clone(), camera_grad=True, intrinsics_grad=ncam == 37)
        assert torch.equal(r[10], torch.zeros(ncam, dtype=torch.float64, device=dev))
