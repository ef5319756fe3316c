import os, sys
ROOT=os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "skyfall-gs_b200")); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch, numpy as np
import helpers as Hh
from sfgs import synthetic as S
dev=torch.device("cuda:0")
for tag,scene,cam in (("one", S.blob_scene(1,seed=2), S.simple_camera(32,32)), ("blob", S.blob_scene(2000,seed=3), S.simple_camera(200,136))):
    if tag=="one":
        scene.means3D[:]=0; scene.scales[:]=0.5; scene.opacities[:]=0.7
    d=Hh.to_torch(scene,cam,dev); bg=torch.tensor([0.1,0.2,0.3],device=dev)
    ref=Hh.run_ref_forward(d,cam,3,bg); our=Hh.run_ours_forward(d,cam,3,bg)
    cot=[torch.from_numpy(c).to(dev) for c in S.cotangents(cam.width,cam.height)]
    rb=Hh.run_ref_backward(d,cam,3,bg,ref,cot); ob=Hh.run_ours_backward(d,cam,3,bg,our,cot)
    for k in ("means2D","colors","opacity","means3D","cov3D","norm3D","sh","scales","rot"):
        a,b=ob[k].double().flatten(),rb[k].double().flatten()
        print(tag,k,"max|d|=%.3e max|ref|=%.3e"%((a-b).abs().max().item(), b.abs().max().item()))
    if tag=="one":
        print("ours means2D",ob["means2D"], "ref",rb["means2D"]); print("ours conic", ob["cov3D"], rb["cov3D"])
