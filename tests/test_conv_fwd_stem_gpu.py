"""Forward of the 7x7 stride-2 pad-3 stems (conv_stem_fwd.cu: one TMA box of a tile's input rows, the im2col operand fed to
wgmma from registers, lo(x) computed from it) against F.conv2d in fp64, with 4 and 8 (padded) input channels.  Each case
runs three ways: the automatic choice, a forced TMA tile knob (which the stems ignore) and the cp.async gather kernel
(SCSFM_TUNE_NO_TMA).  Also: BatchNorm sums over several groups, the fused eval-mode BatchNorm, the low part of the output,
scsfm_conv_reads_lo, and that a tf32x3 training step no longer splits the stem inputs.  Needs a GPU."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from helpers import rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda"

CASES = [
    # B, H, W (input)
    (2, 256, 832),          # full KITTI size: 128 x 416 output
    (2, 37, 45),            # output plane not a multiple of the 8 x 16 tile
    (3, 20, 9),             # output narrower than one tile (5 columns)
    (3, 2, 5),              # two input rows: one output row
    (2, 256, 320),          # NYU
]
WAYS = [("auto", {}), ("forced", dict(mt=1)), ("gather", dict(no_tma=1))]


def _O():
    from scsfm import nnops
    return nnops


def _inputs(B, H, W, Cin, mode, seed):
    O = _O()
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, H, W, Cin, generator=g).to(DEV)
    w = (torch.randn(64, 7, 7, Cin, generator=g) / (49 * Cin) ** 0.5).to(DEV)
    if mode == "tf32":
        O.round_tf32(x, x)
        O.round_tf32(w, w)
    return x, w


def _ref(x, w):
    y = F.conv2d(x.double().permute(0, 3, 1, 2).cpu(), w.double().permute(0, 3, 1, 2).cpu(), None, 2, 3)
    return y.permute(0, 2, 3, 1)


def _conv(O, mode, knobs, x, w, act=0, sums=None, groups=1, **kw):
    cx = O.ConvCtx(mode)
    cx.tune = O.tune(**knobs)
    w_lo = O.split_tf32(w) if cx.split else None
    return cx.conv_fwd(x, w, None, 2, 3, O.PAD_ZERO, act, sums, groups, w_lo, **kw)


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("cin", [4, 8])
@pytest.mark.parametrize("case", CASES)
def test_stem_fwd_vs_fp64(case, cin, mode):
    O = _O()
    tol = 1e-5 if mode == "tf32x3" else 1e-3
    x, w = _inputs(*case, cin, mode, 3 + sum(case) + cin)
    want = _ref(x, w)
    got = {}
    for name, knobs in WAYS:
        y = _conv(O, mode, knobs, x, w)
        y2 = _conv(O, mode, knobs, x, w)
        torch.cuda.synchronize()
        assert torch.equal(y.view(torch.int32), y2.view(torch.int32)), name        # no atomics: repeatable bit for bit
        assert rel_l2(y.cpu(), want) < tol, (name, rel_l2(y.cpu(), want))
        got[name] = y
    assert torch.equal(got["auto"], got["forced"])
    assert rel_l2(got["auto"], got["gather"]) < tol


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("cin", [4, 8])
@pytest.mark.parametrize("groups", [3, 4])
def test_stem_fwd_bn_sums(groups, cin, mode):
    """BatchNorm sums over 3 and 4 groups of images against fp64 sums of the stored output."""
    O = _O()
    B, C = 12, 64
    x, w = _inputs(B, 37, 45, cin, mode, 5 + groups + cin)
    want = _ref(x, w)
    for name, knobs in WAYS:
        sums = torch.zeros(O.BN_SLOTS, groups, C, 2, dtype=torch.float64, device=DEV)
        y = _conv(O, mode, knobs, x, w, sums=sums, groups=groups)
        assert rel_l2(y.cpu(), want) < (1e-5 if mode == "tf32x3" else 1e-3), name
        s = sums.sum(0).cpu()
        yd = y.double().cpu().reshape(groups, B // groups, -1, C)
        s1, s2 = yd.sum((1, 2)), (yd * yd).sum((1, 2))
        assert float((s[..., 0] - s1).abs().max()) <= 1e-5 * float(yd.abs().sum((1, 2)).max()), name
        assert float(((s[..., 1] - s2).abs() / s2).max()) <= 1e-5, name


class _BN:
    def __init__(self, C, seed):
        g = torch.Generator().manual_seed(seed)
        self.weight = (1 + 0.3 * torch.randn(C, generator=g)).to(DEV)
        self.bias = (0.2 * torch.randn(C, generator=g)).to(DEV)
        self.running_mean = (0.3 * torch.randn(C, generator=g)).to(DEV)
        self.running_var = (0.5 + 1.5 * torch.rand(C, generator=g)).to(DEV)


def _bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("cin", [4, 8])
def test_stem_fwd_fused_bn(cin, mode):
    """Eval-mode BatchNorm + ReLU (+ TF32 rounding in tf32) in the epilogue is bitwise the convolution followed by bn_apply,
    and the low part of the output bitwise split_tf32 of it."""
    O = _O()
    x, w = _inputs(2, 37, 45, cin, mode, 9 + cin)
    bn = _BN(64, 17)
    tab = O.BnEvalTable([bn], 1e-5)
    tab.prepare()
    sc, sh = tab.coeffs[0]
    rnd = O.ROUND_TF32 if mode == "tf32" else 0
    for name, knobs in WAYS:
        y = _conv(O, mode, knobs, x, w)
        z, _ = O.bn_apply(y, None, bn.weight, bn.bias, bn.running_mean, bn.running_var, 0.1, 1e-5, None, 1 | rnd, 1,
                          with_lo=True)
        zf = _conv(O, mode, knobs, x, w, act=O.ACT_RELU | rnd, bn_scale=sc, bn_shift=sh, with_lo=True)
        torch.cuda.synchronize()
        assert _bits(zf, z), (name, float((zf - z).abs().max()))
        assert _bits(zf._scsfm_lo, O.split_tf32(zf)), name


def test_stem_fwd_reads_no_input_low_part():
    """The stem kernel runs in split mode with in_lo NULL; the gather kernel forced by tune reads in_lo, so the same call
    is refused with an argument error (never a device fault)."""
    O = _O()
    lib = O._lib()
    x, w = _inputs(2, 37, 45, 8, "tf32x3", 21)
    w_lo = O.split_tf32(w)
    want = _ref(x, w)
    for knobs, reads in ((dict(), 0), (dict(no_tma=1), 1)):
        d = O.conv_desc(x.shape, w, 2, 3, O.PAD_ZERO, O.ACT_NONE)
        y = torch.zeros(2, 19, 23, 64, device=DEV)
        d.inp, d.out, d.w_lo, d.split, d.tune = x.data_ptr(), y.data_ptr(), w_lo.data_ptr(), 1, O.tune(**knobs)
        assert lib.scsfm_conv_reads_lo(ctypes.byref(d), O.PASS_FWD) == reads
        rc = lib.scsfm_conv2d_fwd_tc(ctypes.byref(d), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        if reads:
            assert rc == -1 and b"in_lo" in lib.scsfm_last_error()
            assert float(y.abs().max()) == 0.0
        else:
            assert rc == 0 and rel_l2(y.cpu(), want) < 1e-5


def test_training_step_splits_no_stem_input():
    """A tf32x3 training step computes no low part of a stem input (the stem forward and its TMA weight gradient compute
    lo(x) from their operands) and no lo(dy) of the stems' BatchNorm backward."""
    import models
    from scsfm import lib as L
    from scsfm import nnops as O
    from scsfm import synth
    from scsfm.trainer import Trainer
    H, W = 64, 96
    tgt, refs, K = synth.triplet(2, 2, H, W)
    args = (tgt.to(DEV), [r.to(DEV) for r in refs], K.to(DEV))
    tr = Trainer(models.DispResNet(18, False).to(DEV).train(), models.PoseResNet(18, False).to(DEV).train(), lr=1e-4,
                 with_auto_mask=0, distributed=False, conv_mode="tf32x3")
    split_shapes, bn_lo_shapes = [], []
    split0, bn0 = O.split_tf32, O.bn_backward

    def split(src, dst=None):
        split_shapes.append(tuple(src.shape))
        return split0(src, dst)

    def bn_backward(dz, z, y, saved, dgamma, dbeta, relu, want_dres, groups=1, with_lo=False):
        if with_lo:
            bn_lo_shapes.append(tuple(y.shape))
        return bn0(dz, z, y, saved, dgamma, dbeta, relu, want_dres, groups, with_lo)

    O.split_tf32 = split
    O.bn_backward = bn_backward
    L.PROF["enabled"], L.PROF["only"], L.PROF["events"] = True, {"split"}, []
    try:
        tr.step(*args)
        torch.cuda.synchronize()
        families = [e[0] for e in L.PROF["events"]]
    finally:
        O.split_tf32, O.bn_backward = split0, bn0
        L.PROF["enabled"], L.PROF["only"], L.PROF["events"] = False, None, []
    assert families.count("split") == len(split_shapes)         # every launch of the family went through split_tf32
    assert not [s for s in split_shapes if len(s) == 4 and s[1:3] == (H, W) and s[3] in (4, 8)], split_shapes
    assert not [s for s in bn_lo_shapes if s[1:] == (H // 2, W // 2, 64)], bn_lo_shapes
