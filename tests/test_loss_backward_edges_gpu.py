"""The fused photometric / geometry loss backward (csrc/warp_loss.cu: pairwise_bwd_kernel, geometry_backward, reduce_gM,
pose_grad_kernel, the intrinsics gradient) against the float64 oracle on the CPU, where the smooth golden inputs never go:

  * sharp images at the dataset normalisation, where |T - Iw| > 1 on a large share of the pixels (the L1 clamp's zero-gradient
    side and the clamp inside the auto-mask);
  * all 8 (ssim, mask, auto_mask) settings in both padding modes;
  * large motion (points out of view) and points behind the camera (Zr < 1e-3, where cam2pixel2's clamp cuts d/dZ);
  * 1 to 3 references x 1 to 3 scales (18 pair-directions: two launches of MAX_JOBS), a ragged size, target and reference
    depths of different resolutions at one scale, planes smaller than one 32x16 tile;
  * upstream gradients other than (1, 0.5), and calls where only some depths or poses require a gradient;
  * the shipped training configuration (B=4, 256x832, 2 references, 1 scale, (1,1,1), zeros).

Every case first asserts, from the fp64 oracle's per-pixel maps, that it exercises what it is meant to (share of saturated
pixels, share removed by the auto-mask, share out of view, pixels behind the camera, masked pixels above the 10000 threshold).

Bounds.  Losses: rtol 1e-4 against fp64.  Dense depth gradients: >= 99.9 % of the elements within 1e-4 max|g| of fp64 (plain
rel-L2 is a weak test here: a handful of pixels on a kink -- |T - Iw| = 1, a sign of T - Iw, a bilinear cell -- decide it, and
any independent fp32 evaluation flips some of them); on the quarter-resolution depths of many pair-directions, where every
element gathers the kinks of 16 pixels of each direction, the fp32 oracle itself misses up to 0.35 %, and the share of
elements outside may then be 3x that of the worse fp32 oracle.  Pose and intrinsics gradients: rel-L2 against fp64 at most 3x
the worse of two independent fp32 evaluations of the oracle (CPU, and stock PyTorch on the GPU) plus 3e-3.  The floor is
wider than the 2e-4 of the smooth golden inputs because each of these gradients sums signed contributions of every pixel: the
few kink pixels an fp32 evaluation flips move it by up to 1.9e-2 on sharp inputs (the fp32 oracle against fp64), and two
fp32 evaluations may happen to flip almost none (measured on an H100: 2.6e-3 for the kernel where both yardsticks gave
5.6e-4).  Pixels behind the camera, one by one: relative error at most 3x the worse fp32 oracle's plus 1e-2.

The oracle's gradients of the photometric and the geometry loss are computed once per set of inputs (module-scoped cache) and
combined linearly for each upstream gradient."""
import collections

import numpy as np
import pytest
import torch

import loss_edge_inputs as E
from helpers import frac_within, rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda"

Case = collections.namedtuple("Case", "B H W n_ref n_scales motion flags pm up need k_grad block ref_depth_shifts pairwise seed")


def case(B=2, H=128, W=256, n_ref=1, n_scales=1, motion="small", flags=(1, 1, 1), pm="zeros", up=(1.0, 0.5), need="all",
         k_grad=True, block=8, ref_depth_shifts=None, pairwise=False, seed=1):
    return Case(B, H, W, n_ref, n_scales, motion, flags, pm, up, need, k_grad, block, ref_depth_shifts, pairwise, seed)


SHIFTED = dict(n_ref=2, n_scales=2, ref_depth_shifts=(0, 2), seed=4)   # scale 1: target depth H/2, reference depths H/4
CASES = {}
for _pm in ("zeros", "border"):
    for _f in [(s, m, a) for s in (1, 0) for m in (1, 0) for a in (1, 0)]:
        CASES["flags%d%d%d_%s" % (*_f, _pm)] = case(flags=_f, pm=_pm)
CASES.update({
    "refs2_large_border": case(n_ref=2, motion="large", flags=(1, 1, 0), pm="border", seed=2),
    "refs1_scales3_large": case(n_scales=3, motion="large", flags=(0, 1, 0), seed=3),
    "refs3_scales3_two_chunks": case(n_ref=3, n_scales=3, flags=(1, 1, 1), seed=5),
    "ragged_52x76_scales3": case(B=5, H=52, W=76, n_ref=2, n_scales=3, flags=(1, 1, 0), pm="border", seed=6),
    "depth_shifts_differ": case(**SHIFTED),
    "tiny_3x3": case(B=4000, H=3, W=3, block=1, flags=(1, 1, 0), seed=7),
    "tiny_2x5": case(B=6000, H=2, W=5, block=1, motion="large", flags=(1, 0, 0), pm="border", seed=8),
    "tiny_5x2": case(B=6000, H=5, W=2, block=1, motion="large", flags=(0, 1, 1), seed=9),
    "upstream_1_0": case(up=(1.0, 0.0)),
    "upstream_0_1": case(up=(0.0, 1.0)),
    "upstream_-2.5_0.7": case(up=(-2.5, 0.7)),
    "grad_poses_only": case(**SHIFTED, need="poses", k_grad=False),
    "grad_tgt_depth_only": case(**SHIFTED, need="tgt", k_grad=False),
    "grad_one_ref_depth_only": case(**SHIFTED, need="ref1_s1", k_grad=False),
    "behind_camera_pairwise": case(motion="behind", flags=(1, 1, 0), pairwise=True, seed=10),
    "behind_camera_border": case(motion="behind", flags=(1, 0, 0), pm="border", seed=11),
    "shipped_4x256x832": case(B=4, H=256, W=832, n_ref=2, flags=(1, 1, 1), seed=12),
})


def _inputs(c):
    n_ref = 1 if c.pairwise else c.n_ref
    return E.loss_inputs(c.seed, c.B, c.H, c.W, n_ref, c.n_scales, c.motion, c.block, c.ref_depth_shifts)


def _names(c):
    """Names of the differentiable inputs, in the order _flat returns them."""
    if c.pairwise:
        return [("td", 0), ("rd", 0, 0), ("p", 0), ("K",)]
    return ([("td", s) for s in range(c.n_scales)] + [("rd", i, s) for i in range(c.n_ref) for s in range(c.n_scales)] +
            [("p", i) for i in range(c.n_ref)] + [("pi", i) for i in range(c.n_ref)] + [("K",)])


def _flat(td, rd, ps, pi, K, c):
    if c.pairwise:
        return [td[0], rd[0][0], ps[0], K]
    return [*td, *[x for r in rd for x in r], *ps, *pi, K]


def _loss(mod, c, tgt, refs, K, td, rd, ps, pi):
    if c.pairwise:
        return mod.compute_pairwise_loss(tgt, refs[0], td[0], rd[0][0], ps[0], K, *c.flags, c.pm)
    return mod.compute_photo_and_geometry_loss(tgt, refs, K, td, rd, ps, pi, c.n_scales, *c.flags, c.pm)


def _directions(c, tgt, refs, K, td, rd, ps, pi):
    """(tgt, ref, tgt_depth, ref_depth, pose) of every pair-direction, depths upsampled as the loss does."""
    import torch.nn.functional as F
    up = lambda x: x if x.shape[-2:] == tgt.shape[-2:] else F.interpolate(x, tgt.shape[-2:], mode="nearest")  # noqa: E731
    if c.pairwise:
        return [(tgt, refs[0], td[0], rd[0][0], ps[0])]
    out = []
    for i in range(c.n_ref):
        for s in range(c.n_scales):
            out += [(tgt, refs[i], up(td[s]), up(rd[i][s]), ps[i]), (refs[i], tgt, up(rd[i][s]), up(td[s]), pi[i])]
    return out


def _oracle_run(c, dtype, device):
    """Losses and the gradients of the photometric and of the geometry loss with respect to every differentiable input."""
    from oracle import losses as OL
    tgt, refs, K, td, rd, ps, pi = _inputs(c)
    cv = lambda x: x.to(device=device, dtype=dtype)  # noqa: E731
    leaf = lambda x: cv(x).requires_grad_(True)  # noqa: E731
    tgt, refs, K = cv(tgt), [cv(x) for x in refs], leaf(K)
    td, rd = [leaf(x) for x in td], [[leaf(x) for x in r] for r in rd]
    ps, pi = [leaf(x) for x in ps], [leaf(x) for x in pi]
    leaves = _flat(td, rd, ps, pi, K, c)
    p, q = _loss(OL, c, tgt, refs, K, td, rd, ps, pi)

    def grads(t):
        if not t.requires_grad:
            return [torch.zeros(x.shape, dtype=torch.float64) for x in leaves]
        gs = torch.autograd.grad(t, leaves, retain_graph=True, allow_unused=True)
        return [torch.zeros(x.shape, dtype=torch.float64) if g is None else g.detach().double().cpu() for g, x in zip(gs, leaves)]
    return dict(loss=(float(p.detach()), float(q.detach())), gp=grads(p), gq=grads(q))


def _regime(c):
    """Per-pixel statistics of the fp64 oracle's maps over all pair-directions."""
    from oracle import losses as OL
    tgt, refs, K, td, rd, ps, pi = _inputs(c)
    d = lambda x: x.double()  # noqa: E731
    args = (d(tgt), [d(x) for x in refs], d(K), [d(x) for x in td], [[d(x) for x in r] for r in rd], [d(x) for x in ps],
            [d(x) for x in pi])
    sat = inview = kept = n_pix = 0
    mask_min = float("inf")
    for k, (t, r, tdd, rdd, pose) in enumerate(_directions(c, *args)):
        m = OL.pairwise_terms(t, r, tdd, rdd, pose, args[2], *c.flags, c.pm)
        wv, v = m["warp_valid"], m["valid"]
        sat += float((((t - m["warped"]).abs() > 1).double() * wv).sum())
        inview += float(wv.sum())
        kept += float(v.sum())
        n_pix += wv.numel()
        mask_min = min(mask_min, float(v.sum()))
        if k == 0:
            behind = (m["comp_depth"] == 1e-3) & (v > 0)      # in-view pixels of the first direction with Zr clamped
    return dict(saturated=sat / (3 * inview), automask_removed=1 - kept / inview, out_of_view=1 - inview / n_pix,
                mask_min=mask_min, behind=int(behind.sum()), behind_pixels=behind)


@pytest.fixture(scope="module")
def oracle_cache():
    return {}


def _oracle(cache, c):
    key = c._replace(up=None, need=None, k_grad=None)
    if key not in cache:
        cache[key] = dict(regime=_regime(c), o64=_oracle_run(c, torch.float64, "cpu"), o32=_oracle_run(c, torch.float32, "cpu"),
                          o32gpu=_oracle_run(c, torch.float32, DEV))
    return cache[key]


def _needed(c, name):
    if name == ("K",):
        return c.k_grad
    if c.need == "all":
        return True
    if c.need == "poses":
        return name[0] in ("p", "pi")
    if c.need == "tgt":
        return name[0] == "td"
    assert c.need == "ref1_s1"
    return name == ("rd", 1, 1)


def _cuda_run(c, need):
    """Losses and input gradients of the CUDA path; need(name) says which inputs require a gradient."""
    import loss_functions as lf
    tgt, refs, K, td, rd, ps, pi = _inputs(c)
    d = lambda x: x.to(DEV)  # noqa: E731
    tgt, refs, K = d(tgt), [d(x) for x in refs], d(K)
    td, rd, ps, pi = [d(x) for x in td], [[d(x) for x in r] for r in rd], [d(x) for x in ps], [d(x) for x in pi]
    leaves = _flat(td, rd, ps, pi, K, c)
    for n, x in zip(_names(c), leaves):
        x.requires_grad_(need(n))
    p, q = _loss(lf, c, tgt, refs, K, td, rd, ps, pi)
    (c.up[0] * p + c.up[1] * q).backward()
    return (float(p.detach()), float(q.detach())), [None if x.grad is None else x.grad.double().cpu() for x in leaves]


@pytest.mark.parametrize("name", list(CASES))
def test_loss_backward_vs_fp64_oracle(oracle_cache, name):
    c = CASES[name]
    o = _oracle(oracle_cache, c)
    rg = o["regime"]
    # the case exercises what it is meant to
    assert rg["mask_min"] > 10000, rg["mask_min"]
    assert 0.01 <= rg["saturated"] <= 0.9, rg["saturated"]
    if c.flags[2]:
        assert 0.1 <= rg["automask_removed"] <= 0.9, rg["automask_removed"]
    if c.motion == "large":
        assert rg["out_of_view"] >= 0.05, rg["out_of_view"]
    if c.motion == "behind":
        assert rg["behind"] >= 36, rg["behind"]

    (p, q), got = _cuda_run(c, lambda n: _needed(c, n))
    np.testing.assert_allclose([p, q], o["o64"]["loss"], rtol=1e-4, atol=1e-6)
    up0, up1 = c.up
    want = {k: [up0 * a + up1 * b for a, b in zip(o[k]["gp"], o[k]["gq"])] for k in ("o64", "o32", "o32gpu")}
    report = []
    for j, n in enumerate(_names(c)):
        g, w64 = got[j], want["o64"][j]
        if not _needed(c, n):
            assert g is None, n
            continue
        if n[0] in ("td", "rd"):
            miss = 1 - frac_within(g, w64, 1e-4)
            miss32 = max(1 - frac_within(want[k][j], w64, 1e-4) for k in ("o32", "o32gpu"))
            report.append("%s outside %.5f (fp32 oracle %.5f)" % (n, miss, miss32))
            assert miss <= max(1e-3, 3 * miss32), (n, miss, miss32)
        else:
            yard = max(rel_l2(want["o32"][j], w64), rel_l2(want["o32gpu"][j], w64))
            err = rel_l2(g, w64)
            report.append("%s rel_l2 %.3g (fp32 yardstick %.3g)" % (n, err, yard))
            assert err <= 3 * yard + 3e-3, (n, err, yard)
    if c.motion == "behind":
        # the pixels behind the camera, one by one: a whole-map bound would not see them
        sel = o["regime"]["behind_pixels"]
        w64 = want["o64"][0][sel]
        err = lambda g: float(((g[sel] - w64).abs() / (w64.abs() + 1e-3 * float(w64.abs().max()))).max())  # noqa: E731
        e, e32 = err(got[0]), max(err(want[k][0]) for k in ("o32", "o32gpu"))
        report.append("behind-camera pixels: %d, max rel err %.3g (fp32 oracle %.3g)" % (int(sel.sum()), e, e32))
        assert e <= 3 * e32 + 1e-2, (e, e32)
    print(name, "; ".join(report))


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c.need != "all"])
def test_gradient_subset_equals_full_call(name):
    """Inputs that do not require a gradient get none; the others get what the call with every gradient gives them."""
    c = CASES[name]
    _, part = _cuda_run(c, lambda n: _needed(c, n))
    _, full = _cuda_run(c, lambda n: True)
    for n, a, b in zip(_names(c), part, full):
        if a is not None:
            assert rel_l2(a, b) < 1e-5, n
