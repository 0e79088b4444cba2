"""Pin the oracle's photometric / geometry loss and its gradients to the unmodified reference (tests/golden/loss_edges.npz,
made by tests/golden/make_golden_loss_edges.py) on the inputs where the GPU tests of the loss backward compare the kernel with
the oracle: sharp images that saturate the L1 clamp, large motion, points behind the camera.  CPU only.

Yardstick, as in test_oracle_golden.py: the fp32 oracle does the reference's arithmetic, so its losses agree to fp32 rounding
and its gradients to a tight L2; the fp64 oracle agrees with the fp32 reference on all but a few kink pixels (|T - Iw| = 1,
the sign of T - Iw or of Dc - Dp, a bilinear cell) and within the fp32 reference's own noise on the pose gradients."""
import os

import numpy as np
import pytest
import torch

import loss_edge_inputs as E
from helpers import frac_within, rel_l2
from oracle import losses as OL

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "loss_edges.npz")


@pytest.fixture(scope="module")
def golden_edges():
    return np.load(GOLDEN)


@pytest.mark.parametrize("name", list(E.GOLDEN_SETTINGS))
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
def test_oracle_loss_and_gradients_vs_reference(golden_edges, name, dtype):
    g = golden_edges
    (tgt, refs, K, td, rd, ps, pi), n_scales, flags, pm = E.golden_setting(name)
    np.testing.assert_allclose(E.checksums((tgt, refs, K, td, rd, ps, pi)), g[f"{name}_in_checksum"], rtol=1e-6)
    cv = lambda x: x.to(dtype)  # noqa: E731
    leaf = lambda x: cv(x).requires_grad_(True)  # noqa: E731
    td, rd, ps, pi = [leaf(x) for x in td], [[leaf(x) for x in r] for r in rd], [leaf(x) for x in ps], [leaf(x) for x in pi]
    p, q = OL.compute_photo_and_geometry_loss(cv(tgt), [cv(x) for x in refs], cv(K), td, rd, ps, pi, n_scales, *flags, pm)
    (p + 0.5 * q).backward()
    fp32 = dtype == torch.float32
    np.testing.assert_allclose([float(p.detach()), float(q.detach())], g[f"{name}_loss"], rtol=2e-6 if fp32 else 1e-5, atol=1e-7)
    dense = [(f"tgt_depth_s{s}", t) for s, t in enumerate(td)]
    dense += [(f"ref_depth{i}_s{s}", t) for i, r in enumerate(rd) for s, t in enumerate(r)]
    for key, t in dense:
        mine, want = t.grad[E.SUB4], g[f"{name}_{key}"]
        if fp32:
            assert rel_l2(mine, want) < 2e-4, (key, rel_l2(mine, want))
        else:
            assert frac_within(mine, want, 1e-4) > 0.995, (key, frac_within(mine, want, 1e-4))
    for i in range(len(ps)):
        for key, t in ((f"pose{i}", ps[i]), (f"pose_inv{i}", pi[i])):
            err = rel_l2(t.grad, g[f"{name}_{key}"])
            assert err < (1e-3 if fp32 else 5e-2), (key, err)
