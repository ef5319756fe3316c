"""The blend kernels (forward blend and blend adjoint, which share the reach-list walk of csrc/sfgs_blend_walk.cuh)
bit for bit: every forward output (colour, depth, alpha, normal, n_contrib; the raw normal blend with
fuse_normalize; the extra_attrs channels) and the deterministic backward's blend-adjoint sums and gradients hash to
the digests in tests/golden/blend_digests.npz (recorded on an H100 by tests/golden/make_blend_digests.py).  The cases
cover the 1M-Gaussian benchmark frame, the orbit frame, one band of tile rows, a non-zero background with the fused
normalisation, short tile lists (partial chunks) and extra_attrs at 1 and SFGS_MAX_EXTRA channels.
"""
import importlib.util
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _cases_module():
    spec = importlib.util.spec_from_file_location("make_blend_digests", os.path.join(GOLD, "make_blend_digests.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


G = _cases_module()


@pytest.mark.parametrize("case", list(G.CASES))
def test_blend_outputs_bit_identical(cuda_device, case):
    with np.load(G.FIXTURE) as z:
        want = {k[len(case) + 1:]: str(z[k]) for k in z.files if k.startswith(case + "/")}
    res = G.run_case(case, cuda_device)
    assert int(res["n_contrib"].max()) > 0
    assert set(res) == set(want)
    bad = [k for k in res if G.digest(res[k]) != want[k]]
    assert not bad, f"{case}: {bad} differ from the recorded digests"
