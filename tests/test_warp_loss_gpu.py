"""Parity of the fused CUDA loss path (through the reference-shaped Python API, i.e. through the C ABI)
against the oracle and the committed reference vectors.  Needs a GPU.

Tolerances (north_star: 1e-4 relative fp32):
  * scalar losses, warped images, depths: 1e-4 relative / absolute
  * masks: exact up to a handful of pixels whose coordinate sits on the validity / auto-mask kink
  * dense gradients: >= 99.5 % of elements within 1e-4 * max|g| of the fp32 reference (the rest are kink
    pixels where any independent fp32 evaluation flips a sign/floor, SURVEY.md section 7), and an L2
    error against the fp64 oracle no worse than 3x the fp32 reference's own.
"""
import numpy as np
import pytest
import torch

from helpers import SUB, error_pair, frac_within, golden_loss_inputs, rel_l2, t

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _api():
    import inverse_warp
    import loss_functions
    return inverse_warp, loss_functions


@pytest.mark.parametrize("pm", ["zeros", "border"])
def test_inverse_warp2_maps_vs_reference(golden_warp, pm):
    iw, _ = _api()
    g = golden_warp
    tgt, refs, K, td, rd, ps, pi = golden_loss_inputs(g, device=DEV)
    w, v, pd, cd = iw.inverse_warp2(refs[0], td[0], rd[0][0], ps[0], K, pm)
    w, v, pd, cd = w[SUB], v[SUB], pd[SUB], cd[SUB]
    v_ref = t(g[f"{pm}_valid"], device=DEV)
    flips = (v != v_ref)
    assert int(flips.sum()) <= 4
    keep = (~flips).float()
    np.testing.assert_allclose((w * keep).cpu().numpy(), g[f"{pm}_warped"] * keep.cpu().numpy(), atol=1e-4)
    np.testing.assert_allclose((pd * keep).cpu().numpy(), g[f"{pm}_proj_depth"] * keep.cpu().numpy(), atol=1e-5)
    np.testing.assert_allclose(cd.cpu().numpy(), g[f"{pm}_comp_depth"], rtol=1e-5)


@pytest.mark.parametrize("pm", ["zeros", "border"])
@pytest.mark.parametrize("flags", [(1, 1, 1), (1, 1, 0), (0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1)])
def test_scalar_losses_vs_reference(golden_warp, pm, flags):
    _, lf = _api()
    g = golden_warp
    tgt, refs, K, td, rd, ps, pi = golden_loss_inputs(g, device=DEV)
    p, q = lf.compute_photo_and_geometry_loss(tgt, refs, K, td, rd, ps, pi, 2, *flags, pm)
    want = g[f"{pm}_loss_{flags[0]}{flags[1]}{flags[2]}"]
    np.testing.assert_allclose([float(p), float(q)], want, rtol=1e-4, atol=1e-6)
    # single direction entry point: compute_pairwise_loss equals the oracle's
    from oracle import losses as OL
    a = lf.compute_pairwise_loss(tgt, refs[1], td[0], rd[1][0], ps[1], K, *flags, pm)
    c = golden_loss_inputs(g)
    b = OL.compute_pairwise_loss(c[0], c[1][1], c[3][0], c[4][1][0], c[5][1], c[2], *flags, pm)
    np.testing.assert_allclose([float(a[0]), float(a[1])], [float(b[0]), float(b[1])], rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("pm", ["zeros", "border"])
@pytest.mark.parametrize("flags", [(1, 1, 0), (1, 1, 1)])
def test_gradients_vs_reference_and_fp64_oracle(golden_warp, pm, flags):
    from oracle import losses as OL
    _, lf = _api()
    g = golden_warp
    tag = f"{pm}_g{flags[0]}{flags[1]}{flags[2]}"
    # CUDA path
    tgt, refs, K, td, rd, ps, pi = golden_loss_inputs(g, device=DEV, requires_grad=True)
    p, q = lf.compute_photo_and_geometry_loss(tgt, refs, K, td, rd, ps, pi, 2, *flags, pm)
    s = lf.compute_smooth_loss(td, tgt, rd, refs)
    np.testing.assert_allclose(float(s), g[f"{tag}_smooth"][0], rtol=1e-4)
    (p + 0.5 * q + 0.1 * s).backward()
    # fp64 oracle
    o = golden_loss_inputs(g, torch.float64, requires_grad=True)
    po, qo = OL.compute_photo_and_geometry_loss(o[0], o[1], o[2], o[3], o[4], o[5], o[6], 2, *flags, pm)
    so = OL.compute_smooth_loss(o[3], o[0], o[4], o[1])
    (po + 0.5 * qo + 0.1 * so).backward()

    def dense(mine, ref32, ref64):
        assert frac_within(mine.grad[SUB], ref32, 1e-4) > 0.995
        assert rel_l2(mine.grad[SUB], ref64.grad[SUB]) < 3 * rel_l2(ref32, ref64.grad[SUB]) + 1e-4

    def small(mine, ref32, ref64):
        assert rel_l2(mine.grad, ref64.grad) < 3 * rel_l2(ref32, ref64.grad) + 2e-4

    for sidx in range(2):
        dense(td[sidx], g[f"{tag}_tgt_depth_s{sidx}"], o[3][sidx])
        for i in range(2):
            dense(rd[i][sidx], g[f"{tag}_ref_depth{i}_s{sidx}"], o[4][i][sidx])
    for i in range(2):
        small(ps[i], g[f"{tag}_pose{i}"], o[5][i])
        small(pi[i], g[f"{tag}_pose_inv{i}"], o[6][i])


def test_backward_is_linear_in_upstream_gradient(golden_warp):
    _, lf = _api()
    g = golden_warp
    grads = []
    for scale in (1.0, -2.5):
        tgt, refs, K, td, rd, ps, pi = golden_loss_inputs(g, device=DEV, requires_grad=True)
        p, q = lf.compute_photo_and_geometry_loss(tgt, refs, K, td, rd, ps, pi, 1, 1, 1, 0, "zeros")
        (scale * (p + 0.5 * q)).backward()
        grads.append((td[0].grad.clone(), ps[0].grad.clone()))
    assert rel_l2(grads[1][0], -2.5 * grads[0][0]) < 1e-5
    assert rel_l2(grads[1][1], -2.5 * grads[0][1]) < 1e-4


def test_tiny_image_hits_the_10000_threshold(golden_warp):
    import scsfm.synth as synth
    _, lf = _api()
    d = synth.loss_inputs(11, 1, 32, 48, n_ref=1, n_scales=1)
    c = lambda x: x.to(DEV)  # noqa: E731
    td = [c(x).requires_grad_(True) for x in d["tgt_depth"]]
    p, q = lf.compute_photo_and_geometry_loss(c(d["tgt_img"]), [c(x) for x in d["ref_imgs"]], c(d["intrinsics"]), td,
                                              [[c(x) for x in r] for r in d["ref_depths"]], [c(x) for x in d["poses"]],
                                              [c(x) for x in d["poses_inv"]], 1, 1, 1, 1, "zeros")
    assert float(p) == 0.0 and float(q) == 0.0
    (p + q).backward()
    assert float(td[0].grad.abs().max()) == 0.0
    s = lf.compute_smooth_loss(td, c(d["tgt_img"]), [[c(x) for x in r] for r in d["ref_depths"]],
                               [c(x) for x in d["ref_imgs"]])
    np.testing.assert_allclose(float(s), golden_warp["tiny_smooth"][0], rtol=1e-4)


@pytest.mark.parametrize("shape", [(1, 50, 70), (3, 33, 97), (2, 52, 76)])
@pytest.mark.parametrize("pm", ["zeros", "border"])
def test_ragged_sizes_maps_and_grads_vs_oracle(shape, pm):
    """Sizes that are not multiples of the 32x16 tile; per-pixel maps + inverse_warp2 autograd."""
    import scsfm.synth as synth
    from oracle import geometry as OG
    from oracle import losses as OL
    from scsfm import loss_ops
    iw, lf = _api()
    B, H, W = shape
    d = synth.loss_inputs(5, B, H, W, n_ref=1, n_scales=1)
    pose = d["poses"][0] * 4
    args = (d["tgt_img"], d["ref_imgs"][0], d["tgt_depth"][0], d["ref_depths"][0][0], pose, d["intrinsics"])
    want = OL.pairwise_terms(*[a.double() for a in args], 1, 1, 1, pm)
    got = loss_ops.pairwise_maps(*[a.to(DEV) for a in args], 1, 1, 1, pm)
    flips = (got["mask"].cpu().double() != want["valid"]) | (got["valid"].cpu().double() != want["warp_valid"])
    assert int(flips.sum()) <= 4
    keep = (~flips).double()
    for k_got, k_want, tol in (("warped", "warped", 1e-4), ("proj_depth", "proj_depth", 1e-5),
                               ("comp_depth", "comp_depth", 1e-5), ("diff_depth", "diff_depth", 1e-4),
                               ("diff_img", "diff_img", 2e-4)):
        err = ((got[k_got].cpu().double() - want[k_want]).abs() * keep).max()
        assert float(err) < tol, (k_got, float(err))
    # stand-alone inverse_warp2 autograd (random upstream gradients) vs fp64 oracle
    gen = torch.Generator().manual_seed(1)
    ups = [torch.randn(B, c, H, W, generator=gen) for c in (3, 1, 1)]
    leaves_c = [a.to(DEV).requires_grad_(True) for a in (args[2], args[3], pose)]
    w, v, pd, cd = iw.inverse_warp2(args[1].to(DEV), leaves_c[0], leaves_c[1], leaves_c[2], args[5].to(DEV), pm)
    ((w * ups[0].to(DEV)).sum() + (pd * ups[1].to(DEV)).sum() + (cd * ups[2].to(DEV)).sum()).backward()
    leaves_o = [a.double().requires_grad_(True) for a in (args[2], args[3], pose)]
    w2, v2, pd2, cd2 = OG.inverse_warp2(args[1].double(), leaves_o[0], leaves_o[1], leaves_o[2], args[5].double(), pm)
    ((w2 * ups[0]).sum() + (pd2 * ups[1]).sum() + (cd2 * ups[2]).sum()).backward()
    for a, b in zip(leaves_c[:2], leaves_o[:2]):
        assert frac_within(a.grad, b.grad, 1e-4) > 0.995
    assert rel_l2(leaves_c[2].grad, leaves_o[2].grad) < 5e-3


def test_full_size_kitti_batch_vs_oracle():
    """BASELINE config 2 shape (B=4, 256x832, 2 refs): scalar losses vs the fp32 oracle on the CPU,
    plus size-independent properties."""
    import scsfm.synth as synth
    from oracle import losses as OL
    _, lf = _api()
    d = synth.loss_inputs(0, 4, 256, 832, n_ref=2, n_scales=1)
    p0, q0 = OL.compute_photo_and_geometry_loss(d["tgt_img"], d["ref_imgs"], d["intrinsics"], d["tgt_depth"],
                                                d["ref_depths"], d["poses"], d["poses_inv"], 1, 1, 1, 1, "zeros")
    s0 = OL.compute_smooth_loss(d["tgt_depth"], d["tgt_img"], d["ref_depths"], d["ref_imgs"])
    c = lambda x: x.to(DEV)  # noqa: E731
    tgt, refs, K = c(d["tgt_img"]), [c(x) for x in d["ref_imgs"]], c(d["intrinsics"])
    td = [c(x) for x in d["tgt_depth"]]
    rd = [[c(x) for x in r] for r in d["ref_depths"]]
    ps, pi = [c(x) for x in d["poses"]], [c(x) for x in d["poses_inv"]]
    p, q = lf.compute_photo_and_geometry_loss(tgt, refs, K, td, rd, ps, pi, 1, 1, 1, 1, "zeros")
    s = lf.compute_smooth_loss(td, tgt, rd, refs)
    np.testing.assert_allclose([float(p), float(q), float(s)], [float(p0), float(q0), float(s0)], rtol=1e-4)
    # property: zero motion and identical constant depth => depth inconsistency vanishes (border mode:
    # with 'zeros' the half-out-of-image taps of the (W-1)-normalised edge pixels sample 0, as in the reference)
    const = [torch.full_like(td[0], 0.7)]
    zero = [torch.zeros_like(ps[0])] * 2
    _, q_id = lf.compute_photo_and_geometry_loss(tgt, refs, K, const, [const, const], zero, zero, 1, 1, 1, 0, "border")
    assert abs(float(q_id)) < 1e-5
    # property: the sum over pair-directions is the sum of single-direction calls
    parts = [lf.compute_pairwise_loss(tgt, refs[i], td[0], rd[i][0], ps[i], K, 1, 1, 1, "zeros") for i in range(2)]
    parts += [lf.compute_pairwise_loss(refs[i], tgt, rd[i][0], td[0], pi[i], K, 1, 1, 1, "zeros") for i in range(2)]
    np.testing.assert_allclose(float(p), sum(float(x[0]) for x in parts), rtol=1e-5)
    np.testing.assert_allclose(float(q), sum(float(x[1]) for x in parts), rtol=1e-5)
    # property: smoothness is invariant to a global rescale of depth (mean normalisation)
    s2 = lf.compute_smooth_loss([td[0] * 3.0], tgt, [[r[0] * 3.0] for r in rd], refs)
    np.testing.assert_allclose(float(s2), float(s), rtol=1e-5)


SMOOTH_CASES = [
    # (B, H, W), references, upstream gradient, constant patch, which depths require a gradient (target first)
    ((1, 2, 2), 0, 1.0, False, (True,)),
    ((1, 2, 2), 2, -2.5, True, (True, False, True)),
    ((3, 3, 257), 1, 0.1, True, (True, True)),
    ((2, 37, 61), 2, -2.5, True, (True, False, True)),
    ((2, 37, 61), 2, 0.1, False, (False, True, False)),
    ((4, 256, 832), 2, 0.1, True, (True, True, True)),
    ((4, 256, 832), 0, 1.0, False, (True,)),
]


@pytest.mark.parametrize("case", SMOOTH_CASES, ids=lambda c: "B%d_%dx%d_refs%d_up%g_patch%d_grad%s" % (
    *c[0], c[1], c[2], c[3], "".join(str(int(r)) for r in c[4])))
def test_smooth_loss_value_and_depth_gradients_vs_fp64_oracle(case):
    """compute_smooth_loss against the fp64 oracle: the loss and the dense gradient of every depth that requires one.  A
    constant patch makes neighbour differences exactly 0, where the gradient of |.| is 0 in both; depths without a gradient
    get no buffer and must leave the others intact.  Bounds: fp32 sums of fp32 terms (1e-5)."""
    from oracle import losses as OL
    _, lf = _api()
    (B, H, W), n_ref, upstream, patch, need = case
    g = torch.Generator().manual_seed(B * H * W + n_ref)
    depths, imgs = [], []
    for _ in range(1 + n_ref):
        d = 0.5 + 4.0 * torch.rand(B, 1, H, W, generator=g)
        if patch:
            d[:, :, H // 3:H // 3 + 5, W // 4:W // 4 + 7] = 1.75
        depths.append(d)
        imgs.append(torch.rand(B, 3, H, W, generator=g) * 2 - 1)
    mine = [d.to(DEV).requires_grad_(r) for d, r in zip(depths, need)]
    s = lf.compute_smooth_loss([mine[0]], imgs[0].to(DEV), [[d] for d in mine[1:]], [im.to(DEV) for im in imgs[1:]])
    (upstream * s).backward()
    ref = [d.double().requires_grad_(r) for d, r in zip(depths, need)]
    so = OL.compute_smooth_loss([ref[0]], imgs[0].double(), [[d] for d in ref[1:]], [im.double() for im in imgs[1:]])
    (upstream * so).backward()
    np.testing.assert_allclose(float(s), float(so), rtol=1e-5)
    for i, (a, b) in enumerate(zip(mine, ref)):
        if not need[i]:
            assert a.grad is None
            continue
        assert rel_l2(a.grad, b.grad) < 1e-5, (i, rel_l2(a.grad, b.grad))


def test_pose_matrices_and_legacy_warp(golden_warp):
    iw, _ = _api()
    g = golden_warp
    vec = t(g["pose_vec"], device=DEV)
    np.testing.assert_allclose(iw.pose_vec2mat(vec, "euler").cpu().numpy(), g["pose_mat_euler"], atol=1e-6)
    np.testing.assert_allclose(iw.pose_vec2mat(vec, "quat").cpu().numpy(), g["pose_mat_quat"], atol=1e-6)
    vec.requires_grad_(True)
    np.testing.assert_allclose(iw.pose_vec2mat(vec).detach().cpu().numpy(), g["pose_mat_euler"], atol=1e-6)
    tgt, refs, K, td, rd, ps, pi = golden_loss_inputs(g, device=DEV)
    w, v = iw.inverse_warp(refs[0], td[0][:, 0], ps[0], K, "euler", "zeros")
    np.testing.assert_allclose(w[SUB].cpu().numpy(), g["legacy_warped"], atol=1e-4)
    assert int((v[SUB].cpu().numpy() != g["legacy_valid"]).sum()) <= 4


def test_error_behaviour_matches_reference():
    iw, lf = _api()
    img = torch.zeros(2, 3, 16, 16, device=DEV)
    depth = torch.ones(2, 1, 16, 16, device=DEV)
    pose = torch.zeros(2, 6, device=DEV)
    K = torch.eye(3, device=DEV).repeat(2, 1, 1)
    with pytest.raises(AssertionError, match="wrong size for depth"):
        iw.inverse_warp2(img, depth[:, 0], depth, pose, K)
    with pytest.raises(AssertionError, match="wrong size for pose"):
        iw.inverse_warp2(img, depth, depth, pose[:, :5], K)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        iw.inverse_warp2(img.cpu(), depth.cpu(), depth.cpu(), pose.cpu(), K.cpu())
    with pytest.raises(ValueError):
        lf.compute_photo_and_geometry_loss(img, [img], K, [depth], [[depth]], [pose], [pose], 1, 1, 1, 1, "reflection")


def test_compute_errors_and_ssim_module(golden_warp):
    from oracle import losses as OL
    _, lf = _api()
    g = golden_warp
    gt, pred = (x.to(DEV) for x in error_pair())
    np.testing.assert_allclose(lf.compute_errors(gt, pred, "kitti"), g["err_kitti"], rtol=1e-4)
    np.testing.assert_allclose(lf.compute_errors(gt.clamp(max=12), pred, "nyu"), g["err_nyu"], rtol=1e-4)
    c = golden_loss_inputs(g)
    x, y = c[0].to(DEV), c[1][0].to(DEV)
    want = OL.ssim_dissimilarity(c[0], c[1][0])
    np.testing.assert_allclose(lf.compute_ssim_loss(x, y).cpu().numpy(), want.numpy(), atol=1e-5)


def test_image_gradients_are_refused_loudly():
    """The reference propagates gradients into the images too; this implementation does not (the training path never asks for
    them).  Asking must fail with a clear message instead of silently returning no gradient."""
    iw, lf = _api()
    img = torch.rand(2, 3, 16, 16, device=DEV)
    depth = torch.ones(2, 1, 16, 16, device=DEV, requires_grad=True)
    pose = torch.zeros(2, 6, device=DEV, requires_grad=True)
    K = torch.tensor([[20.0, 0, 8], [0, 20.0, 8], [0, 0, 1]], device=DEV).repeat(2, 1, 1)
    gi = img.clone().requires_grad_(True)
    with pytest.raises(NotImplementedError, match="IMAGES"):
        iw.inverse_warp2(gi, depth, depth, pose, K)
    with pytest.raises(NotImplementedError, match="IMAGES"):
        lf.compute_photo_and_geometry_loss(gi, [img], K, [depth], [[depth]], [pose], [pose], 1, 1, 1, 0, "zeros")
    with pytest.raises(NotImplementedError, match="IMAGES"):
        lf.compute_photo_and_geometry_loss(img, [gi], K, [depth], [[depth]], [pose], [pose], 1, 1, 1, 0, "zeros")
    with pytest.raises(NotImplementedError, match="IMAGES"):
        lf.compute_smooth_loss([depth], gi, [[depth]], [img])
    # without image gradients everything works as before
    p, g = lf.compute_photo_and_geometry_loss(img, [img], K, [depth], [[depth]], [pose], [pose], 1, 1, 1, 0, "zeros")
    (p + g + lf.compute_smooth_loss([depth], img, [[depth]], [img])).backward()
    assert depth.grad is not None and pose.grad is not None
