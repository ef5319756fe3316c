"""Render-set data parallelism for the Stage-2 IDU loop (SURVEY.md 8f rank 4; BASELINE.json configs[4], rasterizer side).

One IDU episode renders num_targets x num_cams x num_samples look-at views (108 at the reference's defaults: 9 grid
targets x 6 orbit cameras x 2 samples, 1024 x 1024; train.py:360-525, utils/camera_utils.py:167-226,
arguments/__init__.py:232-256) before each view goes through FlowEdit and MoGe.  The views are independent, so the set
shards by VIEW: every rank holds the scene, renders a contiguous share of the views (forward only, fused normal
normalisation), and only the results — 8-bit colour and float depth — are gathered on rank 0.  There is no exchange
inside a frame; the single collective is the gather of finished images (backend-agnostic: NCCL on the H100s, gloo in the
CPU tests).  The diffusion / depth models themselves are out of scope (no weights, no network).
"""
from __future__ import annotations

from typing import List, Sequence

import torch
import torch.distributed as dist

from . import synthetic as S


def idu_orbit_cameras(targets: Sequence[Sequence[float]], elevation_deg: float, radius: float, num_cams: int = 6,
                      num_samples: int = 2, fov_deg: float = 60.0, size: int = 1024) -> List[S.Camera]:
    """The cameras gen_idu_orbit_camera (utils/camera_utils.py:167-226) generates for each look-at target: `num_cams`
    azimuths on a circle of the given elevation and radius, each repeated `num_samples` times, z up, square image."""
    cams = []
    for tgt in targets:
        for i in range(num_cams):
            cam = S.orbit_camera(target=tuple(tgt), elevation_deg=elevation_deg, azimuth_deg=360.0 * i / num_cams,
                                 radius=radius, fov_deg=fov_deg, width=size, height=size)
            cams.extend([cam] * num_samples)
    return cams


def idu_grid_targets(grid_width: float = 256.0, grid_height: float = 256.0, grid_size: int = 2) -> List[List[float]]:
    """(grid_size + 1)^2 look-at points on the ground plane (arguments/__init__.py:258-260: 256 x 256, size 2 -> 9)."""
    xs = [-grid_width / 2 + grid_width * i / grid_size for i in range(grid_size + 1)]
    ys = [-grid_height / 2 + grid_height * j / grid_size for j in range(grid_size + 1)]
    return [[x, y, 0.0] for y in ys for x in xs]


def partition_views(n_views: int, world: int) -> List[int]:
    """world+1 boundaries of contiguous, balanced shares (the first n_views % world ranks get one more view)."""
    base, extra = divmod(n_views, world)
    cuts = [0]
    for r in range(world):
        cuts.append(cuts[-1] + base + (1 if r < extra else 0))
    return cuts


def gather_views(color_u8: torch.Tensor, depth: torch.Tensor, cuts: Sequence[int], group=None):
    """color_u8 [n_local,3,H,W] uint8 and depth [n_local,1,H,W] float32 of this rank's views -> on every rank the full
    [n_views,...] tensors in view order (shares padded to the largest one for a single all_gather each)."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    n_max = max(cuts[r + 1] - cuts[r] for r in range(world))
    n_local = cuts[rank + 1] - cuts[rank]
    assert color_u8.shape[0] == n_local and depth.shape[0] == n_local

    def one(t):
        pad = torch.zeros((n_max,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
        pad[:n_local] = t
        out = torch.empty((world,) + tuple(pad.shape), dtype=t.dtype, device=t.device)
        dist.all_gather_into_tensor(out.view(-1), pad.view(-1), group=group)
        return torch.cat([out[r, : cuts[r + 1] - cuts[r]] for r in range(world)], 0)
    return one(color_u8), one(depth)


def upload_cameras(cams: Sequence[S.Camera], dev):
    """The episode's camera matrices as ONE device tensor [n, 35] (view 16 | proj 16 | centre 3): one copy per episode
    instead of three small synchronous copies per view."""
    import numpy as np
    if not cams:
        return torch.empty((0, 35), device=dev)
    tab = np.stack([np.concatenate([c.viewmatrix.ravel(), c.projmatrix.ravel(), c.campos]) for c in cams]).astype(np.float32)
    return torch.from_numpy(tab).to(dev)


def render_views(d, cams: Sequence[S.Camera], sh_degree: int = 3, cam_table=None):
    """Forward-only renders of `cams` (this rank's share) -> (uint8 colour [n,3,H,W], float32 depth [n,1,H,W])."""
    from . import rasterizer as R
    dev = d["means3D"].device
    e = torch.empty(0, device=dev)
    bg = torch.zeros(3, device=dev)
    if cam_table is None:
        cam_table = upload_cameras(cams, dev)
    colors, depths = [], []
    for k, cam in enumerate(cams):
        row = cam_table[k]
        f = R.rasterize_gaussians(bg, d["means3D"], e, d["opacities"], d["scales"], d["rotations"], 1.0, e, e, e, 0,
                                  row[0:16].view(4, 4), row[16:32].view(4, 4), cam.tanfovx, cam.tanfovy, 0.1, cam.height,
                                  cam.width, d["shs"], sh_degree, row[32:35], False, False)
        colors.append((f[1].clamp(0, 1) * 255.0 + 0.5).to(torch.uint8))
        depths.append(f[2])
    if not colors:
        H, W = (cams[0].height, cams[0].width) if cams else (1, 1)
        return torch.empty((0, 3, H, W), dtype=torch.uint8, device=dev), torch.empty((0, 1, H, W), device=dev)
    return torch.stack(colors), torch.stack(depths)


def run_renderset(P, rank, world, dev, repeats=3, size=1024):
    """Time one IDU episode's render set (108 views at `size`^2, jax_v1 parameters: elevation 85, radius 300, fov 60)
    sharded by view over the ranks, including the gather of the finished images.  Returns a dict (same on all ranks)."""
    import numpy as np
    scene = S.city_scene(P, seed=0, sh_degree=3)
    d = {k: torch.from_numpy(np.ascontiguousarray(getattr(scene, k))).to(dev) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
    cams = idu_orbit_cameras(idu_grid_targets(), 85.0, 300.0, num_cams=6, num_samples=2, fov_deg=60.0, size=size)
    cuts = partition_views(len(cams), world)
    mine = cams[cuts[rank]:cuts[rank + 1]]
    table = upload_cameras(mine, dev)
    render_views(d, mine[:2], cam_table=table[:2])     # warm-up (binning estimates, allocator)
    times = []
    for _ in range(repeats):
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize(dev)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        c, z = render_views(d, mine, cam_table=table)
        if world > 1:
            c, z = gather_views(c, z, cuts)
        b.record()
        torch.cuda.synchronize(dev)
        ms = torch.tensor([a.elapsed_time(b)], dtype=torch.float64, device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        times.append(float(ms.item()))
    best = min(times)
    return {"workload": f"IDU render set: {len(cams)} look-at views at {size}x{size} (9 targets x 6 cameras x 2 samples, elevation 85, "
                        f"radius 300, fov 60) of the {P}-Gaussian scene, forward only, results gathered as uint8 colour + float depth",
            "views": len(cams), "views_per_rank": [cuts[r + 1] - cuts[r] for r in range(world)], "ms_per_set": round(best, 3),
            "views_per_s": round(len(cams) / best * 1e3, 1), "Mpix_per_s": round(len(cams) * size * size / best / 1e3, 1),
            "collective": "one padded all_gather each for colour and depth (NCCL)" if world > 1 else "none",
            "timing": f"CUDA events around render + gather, max over ranks, best of {repeats}",
            "gathered": [int(c.shape[0]), int(z.shape[0])]}
