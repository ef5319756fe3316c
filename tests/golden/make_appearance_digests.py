"""SHA-256 digests of the fused appearance colours at M = 16 on fixed inputs.

The kernel runs on tests/golden/appearance_ref.npz (M = 16, P = 3000) at every active SH degree D = 0..3.  The
split-bf16 MMAs, the fp32 epilogue and the launch geometry are deterministic, so the colours are reproducible bit for
bit.  tests/test_appearance_widths.py holds the kernel to the digests stored in appearance_m16_digests.npz, which were
recorded with this script on an H100 from the build before the kernel was templated on the SH width:

    python tests/golden/make_appearance_digests.py [OUT.npz]     # needs a CUDA device and the built library
"""
from __future__ import annotations

import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "skyfall-gs_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLD = os.path.join(HERE, "appearance_ref.npz")
FIXTURE = os.path.join(HERE, "appearance_m16_digests.npz")
DEGREES = (0, 1, 2, 3)


def fused_colors(dev, deg):
    """The fused kernel's colours [3000, 3] on appearance_ref.npz at active degree `deg`."""
    import torch
    from sfgs.appearance import fused_appearance_colors
    g = np.load(GOLD)
    t = {k: torch.from_numpy(g[k]).to(dev) for k in ("features", "gemb", "aemb", "xyz", "campos", "W1", "b1", "W2", "b2",
                                                      "W3", "b3")}
    mlp = tuple(t[k] for k in ("W1", "b1", "W2", "b2", "W3", "b3"))
    with torch.no_grad():
        out = fused_appearance_colors(t["features"], t["gemb"], t["aemb"], mlp, t["xyz"], t["campos"], deg)
    torch.cuda.synchronize(dev)
    return out


def digest(t):
    return hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()


def main():
    import torch
    dev = torch.device("cuda:0")
    out = sys.argv[1] if len(sys.argv) > 1 else FIXTURE
    rec = {"device": np.array(torch.cuda.get_device_name(dev))}
    for deg in DEGREES:
        rec[f"deg{deg}"] = np.array(digest(fused_colors(dev, deg)))
        print(f"deg {deg}: {rec[f'deg{deg}']}", flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    np.savez_compressed(out, **rec)
    print("wrote", out)


if __name__ == "__main__":
    main()
