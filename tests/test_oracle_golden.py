"""Pin the oracle (oracle/*.py) against vectors produced by the unmodified reference
(tests/golden/make_golden.py).  CPU only."""
import numpy as np
import pytest
import torch

from golden_util import det_image, det_weights
from helpers import SUB, error_pair, frac_within, golden_loss_inputs, rel_l2, t
from oracle import geometry as G
from oracle import losses as L
from oracle import nets as N


@pytest.mark.parametrize("pm", ["zeros", "border"])
def test_inverse_warp2_maps(golden_warp, pm):
    g = golden_warp
    tgt, refs, K, td, rd, ps, pi = golden_loss_inputs(g)
    w, v, pd, cd = G.inverse_warp2(refs[0], td[0], rd[0][0], ps[0], K, pm)
    w, v, pd, cd = w[SUB], v[SUB], pd[SUB], cd[SUB]
    assert torch.equal(v, t(g[f"{pm}_valid"]))
    np.testing.assert_allclose(w.numpy(), g[f"{pm}_warped"], atol=2e-5)
    np.testing.assert_allclose(pd.numpy(), g[f"{pm}_proj_depth"], atol=2e-6)
    np.testing.assert_allclose(cd.numpy(), g[f"{pm}_comp_depth"], rtol=1e-6)
    assert 0.3 < float(v.mean()) < 0.99          # some points do leave the frame


@pytest.mark.parametrize("pm", ["zeros", "border"])
@pytest.mark.parametrize("flags", [(1, 1, 1), (1, 1, 0), (0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1)])
def test_scalar_losses(golden_warp, pm, flags):
    g = golden_warp
    tgt, refs, K, td, rd, ps, pi = golden_loss_inputs(g)
    p, q = L.compute_photo_and_geometry_loss(tgt, refs, K, td, rd, ps, pi, 2, *flags, pm)
    want = g[f"{pm}_loss_{flags[0]}{flags[1]}{flags[2]}"]
    np.testing.assert_allclose([float(p), float(q)], want, rtol=2e-6, atol=1e-7)


def test_threshold_makes_geometry_zero_with_automask(golden_warp):
    # 2*64*128 pixels: with the auto-mask fewer than 10000 survive -> geometry term is the constant 0,
    # while the photometric term counts the mask three times (expand_as) and stays on.
    want = golden_warp["zeros_loss_111"]
    assert want[0] > 0


@pytest.mark.parametrize("pm", ["zeros", "border"])
@pytest.mark.parametrize("flags", [(1, 1, 0), (1, 1, 1)])
def test_gradients_fp32_and_fp64(golden_warp, pm, flags):
    g = golden_warp
    tag = f"{pm}_g{flags[0]}{flags[1]}{flags[2]}"
    for dtype, tol in ((torch.float32, 2e-4), (torch.float64, 2e-2)):
        # fp64 oracle vs fp32 reference: the reference's own fp32 noise (kink pixels) bounds the match
        tgt, refs, K, td, rd, ps, pi = golden_loss_inputs(g, dtype, requires_grad=True)
        p, q = L.compute_photo_and_geometry_loss(tgt, refs, K, td, rd, ps, pi, 2, *flags, pm)
        s = L.compute_smooth_loss(td, tgt, rd, refs)
        (p + 0.5 * q + 0.1 * s).backward()
        np.testing.assert_allclose(float(s.detach()), g[f"{tag}_smooth"][0], rtol=2e-6)
        def close(a, b):
            # fp32: same arithmetic -> tight L2.  fp64 vs the fp32 reference: all but a handful of
            # kink pixels (|T-Iw| sign, floor() cell, |Dc-Dp| sign flips) agree (SURVEY.md section 7)
            if dtype == torch.float32:
                return rel_l2(a, b) < tol
            return frac_within(a, b, 1e-4) > 0.995
        for sidx in range(2):
            assert close(td[sidx].grad[SUB], g[f"{tag}_tgt_depth_s{sidx}"])
            for i in range(2):
                assert close(rd[i][sidx].grad[SUB], g[f"{tag}_ref_depth{i}_s{sidx}"])
        for i in range(2):
            assert rel_l2(ps[i].grad, g[f"{tag}_pose{i}"]) < (1e-3 if dtype == torch.float32 else 5e-2)
            assert rel_l2(pi[i].grad, g[f"{tag}_pose_inv{i}"]) < (1e-3 if dtype == torch.float32 else 5e-2)


def test_tiny_image_below_threshold(golden_warp):
    import scsfm.synth as synth
    d = synth.loss_inputs(11, 1, 32, 48, n_ref=1, n_scales=1)
    p, q = L.compute_photo_and_geometry_loss(d["tgt_img"], d["ref_imgs"], d["intrinsics"], d["tgt_depth"],
                                             d["ref_depths"], d["poses"], d["poses_inv"], 1, 1, 1, 1, "zeros")
    assert float(p) == 0.0 and float(q) == 0.0
    assert list(golden_warp["tiny_loss"]) == [0.0, 0.0]
    s = L.compute_smooth_loss(d["tgt_depth"], d["tgt_img"], d["ref_depths"], d["ref_imgs"])
    np.testing.assert_allclose(float(s), golden_warp["tiny_smooth"][0], rtol=2e-6)


def test_pose_matrices_and_legacy_warp(golden_warp):
    g = golden_warp
    vec = t(g["pose_vec"])
    np.testing.assert_allclose(G.pose_to_matrix(vec, "euler").numpy(), g["pose_mat_euler"], atol=1e-6)
    np.testing.assert_allclose(G.pose_to_matrix(vec, "quat").numpy(), g["pose_mat_quat"], atol=1e-6)
    tgt, refs, K, td, rd, ps, pi = golden_loss_inputs(g)
    w, v = G.inverse_warp(refs[0], td[0][:, 0], ps[0], K, "euler", "zeros")
    np.testing.assert_allclose(w[SUB].numpy(), g["legacy_warped"], atol=2e-5)
    assert np.array_equal(v[SUB].numpy(), g["legacy_valid"])


def test_compute_errors(golden_warp):
    g = golden_warp
    gt, pred = error_pair()
    np.testing.assert_allclose(L.compute_errors(gt, pred, "kitti"), g["err_kitti"], rtol=1e-5)
    np.testing.assert_allclose(L.compute_errors(gt.clamp(max=12), pred, "nyu"), g["err_nyu"], rtol=1e-5)


@pytest.mark.parametrize("layers", [18, 50])
@pytest.mark.parametrize("kind", ["disp", "pose"])
def test_networks(golden_nets, layers, kind):
    g = golden_nets
    tag = f"{kind}{layers}"
    net = N.DispResNet(layers) if kind == "disp" else N.PoseResNet(layers)
    sd = net.state_dict()
    assert list(sd.keys()) == list(g[f"{tag}_keys"])
    assert ["x".join(map(str, v.shape)) for v in sd.values()] == list(g[f"{tag}_shapes"])
    net.load_state_dict(det_weights(sd))
    net.train()
    img1, img2 = det_image("img1", 2, 64, 96), det_image("img2", 2, 64, 96)
    if kind == "disp":
        outs = net(img1)
        loss = sum(((1.0 / o) * (i + 1)).mean() for i, o in enumerate(outs))
        for s, o in enumerate(outs):
            np.testing.assert_allclose(o.detach().numpy(), g[f"{tag}_out_s{s}"], rtol=2e-4, atol=2e-5)
    else:
        o = net(img1, img2)
        loss = (o * torch.arange(1, 7, dtype=o.dtype)).sum() * 100
        np.testing.assert_allclose(o.detach().numpy(), g[f"{tag}_out"], rtol=2e-4, atol=1e-7)
    loss.backward()
    np.testing.assert_allclose(float(loss), g[f"{tag}_loss"][0], rtol=1e-5)
    grads = {k: p.grad for k, p in net.named_parameters() if p.grad is not None}
    assert list(grads.keys()) == list(g[f"{tag}_grad_names"])
    norms = np.array([float(v.double().norm()) for v in grads.values()])
    np.testing.assert_allclose(norms, g[f"{tag}_grad_norms"], rtol=5e-3, atol=1e-9)
    sd2 = net.state_dict()
    rn = np.array([float(sd2[k].double().norm()) for k in g[f"{tag}_running_names"]])
    np.testing.assert_allclose(rn, g[f"{tag}_running_norms"], rtol=1e-4)
    net.eval()
    with torch.no_grad():
        e = net(img1) if kind == "disp" else net(img1, img2)
    np.testing.assert_allclose(e.numpy(), g[f"{tag}_eval_out"], rtol=2e-4, atol=2e-5)


def test_library_kernel_mode_agrees_with_the_restatement(golden_warp):
    """bench.py times the oracle with F.grid_sample / F.avg_pool2d switched in; both forms must agree."""
    g = golden_warp
    vals = []
    for fast in (False, True):
        G.USE_LIBRARY_KERNELS = fast
        try:
            tgt, refs, K, td, rd, ps, pi = golden_loss_inputs(g, requires_grad=True)
            p, q = L.compute_photo_and_geometry_loss(tgt, refs, K, td, rd, ps, pi, 2, 1, 1, 1, "zeros")
            (p + 0.5 * q).backward()
            vals.append((float(p.detach()), float(q.detach()), td[0].grad.clone(), ps[0].grad.clone()))
        finally:
            G.USE_LIBRARY_KERNELS = False
    np.testing.assert_allclose(vals[0][:2], vals[1][:2], rtol=2e-6)
    assert rel_l2(vals[0][2], vals[1][2]) < 1e-4 and rel_l2(vals[0][3], vals[1][3]) < 1e-3
