"""Gradients with respect to the camera intrinsics, CPU side: the fp64 oracle's d(loss)/dK against the unmodified reference's
fp32 gradient (tests/golden/intrinsics.npz, make_golden_intrinsics.py), and the C ABI of the two new entries (declared,
exported, argument errors reported without a launch)."""
import os
import re

import numpy as np
import pytest
import torch

from helpers import golden_loss_inputs, rel_l2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def golden_k():
    return np.load(os.path.join(GOLDEN, "intrinsics.npz"))


def iw2_upstream(g, B, H, W):
    """The seeded upstream gradients of the inverse_warp2 case of intrinsics.npz, checked against their stored checksums."""
    gen = torch.Generator().manual_seed(int(g["iw2_up_seed"][0]))
    ups = [torch.randn(B, c, H, W, generator=gen) for c in (3, 1, 1)]
    np.testing.assert_allclose([float(u.double().abs().sum()) for u in ups], g["iw2_up_checksum"], rtol=1e-9)
    return ups


def oracle_loss_dK(golden_warp, pm, flags, dtype=torch.float64):
    """d(1*photo + 0.5*geo)/dK of the golden loss inputs (2 references, 2 scales) through the oracle."""
    from oracle import losses as OL
    o = golden_loss_inputs(golden_warp, dtype)
    K = o[2].clone().requires_grad_(True)
    p, q = OL.compute_photo_and_geometry_loss(o[0], o[1], K, o[3], o[4], o[5], o[6], 2, *flags, pm)
    (p + 0.5 * q).backward()
    return K.grad


def oracle_iw2_dK(golden_warp, golden_k, pm, dtype=torch.float64):
    from oracle import geometry as OG
    o = golden_loss_inputs(golden_warp, dtype)
    K = o[2].clone().requires_grad_(True)
    w, _, pd, cd = OG.inverse_warp2(o[1][0], o[3][0], o[4][0][0], o[5][0], K, pm)
    ups = [u.to(dtype) for u in iw2_upstream(golden_k, *o[3][0].shape[:1], *o[3][0].shape[-2:])]
    ((w * ups[0]).sum() + (pd * ups[1]).sum() + (cd * ups[2]).sum()).backward()
    return K.grad


def test_golden_inputs_are_those_of_the_loss_golden(golden_warp, golden_k):
    np.testing.assert_array_equal(golden_k["in_checksum"], golden_warp["in_checksum"])


@pytest.mark.parametrize("pm", ["zeros", "border"])
@pytest.mark.parametrize("flags", [(1, 1, 0), (1, 1, 1)])
def test_oracle_intrinsics_gradient_of_the_losses_vs_reference(golden_warp, golden_k, pm, flags):
    """The reference's fp32 dK differs from the fp64 oracle's by its own noise only: pixels whose sampling coordinate or mask sits
    on a kink are decided differently by fp32 and fp64 (largest in 'zeros' without auto-mask, about 2e-2 here)."""
    want = golden_k[f"{pm}_loss_K{flags[0]}{flags[1]}{flags[2]}"]
    got = oracle_loss_dK(golden_warp, pm, flags)
    assert float(got.abs().max()) > 1e-3           # a live gradient, not two zeros
    assert rel_l2(want, got) < 5e-2, rel_l2(want, got)


@pytest.mark.parametrize("pm", ["zeros", "border"])
def test_oracle_intrinsics_gradient_of_inverse_warp2_vs_reference(golden_warp, golden_k, pm):
    got = oracle_iw2_dK(golden_warp, golden_k, pm)
    assert float(got.abs().max()) > 1.0
    assert rel_l2(golden_k[f"{pm}_iw2_K"], got) < 1e-4, rel_l2(golden_k[f"{pm}_iw2_K"], got)


def test_header_declares_and_library_exports_the_intrinsics_entries():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "scsfm.h")).read(), flags=re.S)
    for name in ("scsfm_pairwise_intrinsics_grad", "scsfm_inverse_warp2_intrinsics_grad"):
        assert re.search(r"\b%s\s*\(" % name, src), name
    from scsfm import lib
    L = lib.load()
    assert hasattr(L, "scsfm_pairwise_intrinsics_grad") and hasattr(L, "scsfm_inverse_warp2_intrinsics_grad")


def test_intrinsics_entries_reject_bad_arguments_without_a_launch():
    import ctypes
    from scsfm import lib
    L = lib.load()
    n0 = lib.launch_count()
    fake = ctypes.c_void_p(16)            # never dereferenced: every call below fails its argument check first
    job = (lib.PairJob * 1)(lib.PairJob(fake, fake, fake, fake, fake, None, None, None, 0, 0))
    assert L.scsfm_pairwise_intrinsics_grad(None, 0, fake, 1, fake, fake, None) == -1
    assert b"njobs" in L.scsfm_last_error()
    assert L.scsfm_pairwise_intrinsics_grad(job, lib.MAX_JOBS + 1, fake, 1, fake, fake, None) == -1
    assert L.scsfm_pairwise_intrinsics_grad(job, 1, fake, 0, fake, fake, None) == -1
    assert b"batch" in L.scsfm_last_error()
    assert L.scsfm_pairwise_intrinsics_grad(job, 1, fake, 1, fake, None, None) == -1
    assert b"grad_intrinsics" in L.scsfm_last_error()
    nopose = (lib.PairJob * 1)(lib.PairJob(fake, fake, fake, fake, None, None, None, None, 0, 0))
    assert L.scsfm_pairwise_intrinsics_grad(nopose, 1, fake, 1, fake, fake, None) == -1
    assert b"null pose" in L.scsfm_last_error()
    assert L.scsfm_inverse_warp2_intrinsics_grad(fake, fake, 1, None, fake, None) == -1
    assert b"inverse_warp2_intrinsics_grad" in L.scsfm_last_error()
    assert L.scsfm_inverse_warp2_intrinsics_grad(fake, fake, 0, fake, fake, None) == -1
    with pytest.raises(ValueError):
        lib.check(L.scsfm_inverse_warp2_intrinsics_grad(None, None, 1, None, None, None), "scsfm_inverse_warp2_intrinsics_grad")
    assert lib.launch_count() == n0
