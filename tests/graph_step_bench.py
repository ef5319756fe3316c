"""The training step of tests/train_loop_bench.py, eager and as a replayed CUDA graph — needs a GPU.  Not a pytest file.

    python tests/graph_step_bench.py [--P 1000000] [--rounds 7] [--steps 20]

Step: fused activations -> diff_gauss render of one of 8 orbit views at 1920x1080 (SH 3) -> 0.8 L1 + 0.2 (1 - SSIM) ->
backward -> Adam(capturable=True, tensor learning rates) -> add_densification_stats.  A second configuration adds the
appearance path (fused_appearance_colors at M = 4, fused backward).  Reported, per configuration:
  eager_ms / replay_ms      device time per step (CUDA events around `steps` steps), median of alternating rounds;
  host_issue_ms             host clock around the enqueue of one eager step (no synchronise of our own, so it includes
                            the forward's one host wait), median over the eager rounds' steps;
  raster_eager_ms / raster_replay_ms   the rasterizer forward + backward alone (diff_gauss), eager and replayed.
Every shape is warmed up before the first timed round.  The card name and power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "skyfall-gs_b200"))
import numpy as np
import torch

from sfgs import synthetic as S


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def build(dev, P, appearance):
    from diff_gauss import GaussianRasterizationSettings, GaussianRasterizer
    from fused_ssim import fused_ssim
    from sfgs import densify as DN
    from sfgs.activations import fused_activations
    from sfgs.appearance import fused_appearance_colors
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    scene = S.city_scene(P, seed=0, sh_degree=3)
    cams = [S.orbit_camera(azimuth_deg=45.0 * k) for k in range(8)]
    H, W = cams[0].height, cams[0].width
    rng = np.random.default_rng(1)
    xyz = t((scene.means3D + rng.normal(0, 0.05, scene.means3D.shape)).astype(np.float32)).requires_grad_(True)
    scaling = torch.log(t(scene.scales)).requires_grad_(True)
    rotation = t(scene.rotations).clone().requires_grad_(True)
    opacity = torch.logit(t(scene.opacities).clamp(1e-4, 1 - 1e-4)).reshape(P, 1).clone().requires_grad_(True)
    shs = (t(scene.shs) * 0.9).requires_grad_(True)
    params = [xyz, scaling, rotation, opacity, shs]
    lrs = [1.6e-4, 5e-3, 1e-3, 5e-2, 2.5e-3]
    if appearance:
        feats = (t(scene.shs)[:, :4] * 0.9).contiguous().requires_grad_(True)
        gemb = (torch.randn((P, 24), device=dev) * 0.1).requires_grad_(True)
        aembs = torch.randn((8, 32), device=dev) * 0.1
        mlp = torch.nn.Sequential(torch.nn.Linear(59, 128), torch.nn.ReLU(), torch.nn.Linear(128, 128), torch.nn.ReLU(),
                                  torch.nn.Linear(128, 6)).to(dev)
        params = [xyz, scaling, rotation, opacity, feats, gemb] + list(mlp.parameters())
        lrs = [1.6e-4, 5e-3, 1e-3, 5e-2, 2.5e-3, 1e-3] + [1e-3] * 6
    opt = torch.optim.Adam([{"params": [p], "lr": torch.tensor(lr, device=dev)} for p, lr in zip(params, lrs)],
                           eps=1e-15, capturable=True)
    filter_3D = torch.full((P, 1), 0.05, dtype=torch.float64, device=dev)
    bg = torch.zeros(3, device=dev)
    targets = [torch.rand((3, H, W), device=dev) for _ in cams]
    camt = [dict(view=t(c.viewmatrix), proj=t(c.projmatrix), campos=t(c.campos),
                 tanx=torch.tensor(c.tanfovx, device=dev), tany=torch.tensor(c.tanfovy, device=dev)) for c in cams]
    static = {k: v.clone() for k, v in camt[0].items()}
    static["gt"], static["idx"] = targets[0].clone(), torch.zeros((), dtype=torch.long, device=dev)
    z = lambda: torch.zeros(P, device=dev)  # noqa: E731
    stats = types.SimpleNamespace(max_radii2D=z(), xyz_gradient_accum=z(), xyz_gradient_accum_abs=z(),
                                  xyz_gradient_accum_abs_max=z(), denom=z())

    def load(i):
        with torch.no_grad():
            for k, v in camt[i % 8].items():
                static[k].copy_(v)
            static["gt"].copy_(targets[i % 8])
            static["idx"].fill_(i % 8)

    def render(op, sc, rot):
        m2d = torch.zeros((P, 3), device=dev, requires_grad=True)
        rs = GaussianRasterizationSettings(H, W, static["tanx"], static["tany"], 0.1, torch.zeros(1, device=dev), bg, 1.0,
                                           static["view"], static["proj"], 3, static["campos"], False, False)
        if appearance:
            aemb = aembs.index_select(0, static["idx"].reshape(1))[0]   # indexing with the tensor itself syncs
            colors = fused_appearance_colors(feats, gemb, aemb, mlp, xyz, static["campos"], 1, fused_backward=True)
            out = GaussianRasterizer(rs)(xyz, m2d, op, colors_precomp=colors, scales=sc, rotations=rot)
        else:
            out = GaussianRasterizer(rs)(xyz, m2d, op, shs=shs, scales=sc, rotations=rot)
        return out, m2d

    def step():
        op, sc, rot = fused_activations(opacity, scaling, rotation, filter_3D)
        out, m2d = render(op, sc, rot)
        color, radii, gt = out[0], out[4], static["gt"]
        loss = 0.8 * torch.nn.functional.l1_loss(color, gt) + 0.2 * (1.0 - fused_ssim(color[None], gt[None]))
        loss.backward()
        opt.step()
        DN.add_densification_stats(stats, types.SimpleNamespace(grad=torch.nn.functional.pad(m2d.grad, (0, 1))), radii)

    cot = torch.rand((3, H, W), device=dev)

    def raster():
        with torch.no_grad():
            op, sc, rot = fused_activations(opacity, scaling, rotation, filter_3D)
        leaves = [t_.detach().requires_grad_(True) for t_ in (op, sc, rot)]
        out, m2d = render(*leaves)
        torch.autograd.grad((out[0] * cot).sum(), [m2d, xyz] + leaves)

    return opt, params, load, step, raster


def timed(fn, n, dev):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(n):
        fn(i)
    b.record()
    torch.cuda.synchronize(dev)
    return a.elapsed_time(b) / n


def measure(dev, P, appearance, rounds, steps):
    from sfgs import graphs
    opt, params, load, step, raster = build(dev, P, appearance)

    def eager_step(i):
        load(i)
        opt.zero_grad(set_to_none=True)
        step()

    for i in range(8):                      # every camera once: kernels loaded, capacity estimates in place
        eager_step(i)
        load(i)
        raster()
    graphs.status(dev)
    torch.cuda.synchronize(dev)
    opt.zero_grad(set_to_none=True)
    g_step, g_raster = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        with torch.cuda.graph(g_step):
            step()
        with torch.cuda.graph(g_raster):
            raster()
    torch.cuda.current_stream(dev).wait_stream(side)

    def replay_step(i):
        load(i)
        g_step.replay()

    def replay_raster(i):
        load(i)
        g_raster.replay()

    def eager_raster(i):
        load(i)
        raster()

    for fn in (replay_step, replay_raster, eager_step, eager_raster):
        timed(fn, 8, dev)
    graphs.check(dev)
    res = {k: [] for k in ("eager_ms", "replay_ms", "raster_eager_ms", "raster_replay_ms", "host_issue_ms")}
    for r in range(rounds):
        res["eager_ms"].append(timed(eager_step, steps, dev))
        res["replay_ms"].append(timed(replay_step, steps, dev))
        res["raster_eager_ms"].append(timed(eager_raster, steps, dev))
        res["raster_replay_ms"].append(timed(replay_raster, steps, dev))
        graphs.check(dev)
        for i in range(steps):              # host clock around the enqueue of one eager step
            load(i)
            t0 = time.perf_counter()
            opt.zero_grad(set_to_none=True)
            step()
            res["host_issue_ms"].append((time.perf_counter() - t0) * 1e3)
        torch.cuda.synchronize(dev)
    out = {k: round(statistics.median(v), 3) for k, v in res.items()}
    out["replay_speedup"] = round(out["eager_ms"] / out["replay_ms"], 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=1_000_000)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    card = _card()
    results = {"card": card, "config": f"{a.P} Gaussians, 8 orbit views 1920x1080, SH 3, L1+SSIM, Adam(capturable)"}
    results["sh3"] = measure(dev, a.P, False, a.rounds, a.steps)
    results["appearance_m4"] = measure(dev, a.P, True, a.rounds, a.steps)
    print(json.dumps(results))


if __name__ == "__main__":
    main()
