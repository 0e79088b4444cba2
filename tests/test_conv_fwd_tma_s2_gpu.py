"""Stride-2 forward convolutions on the TMA kernel (conv_tma.cu: one box per row parity, read through the (row, column)
parity views of the input) against F.conv2d in fp64, each run three ways: the automatic choice, forced TMA tile
configurations (SCSFM_TUNE_MT / TW) and the cp.async gather kernel (SCSFM_TUNE_NO_TMA).  Epilogue variants: bias and
activation, residual addend, TF32 rounding, BatchNorm sums over several groups, and the fused eval-mode BatchNorm with the
low part of its output.  Needs a GPU."""
import pytest
import torch
import torch.nn.functional as F

from helpers import rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda"

CASES = [
    # B, H, W, Cin, Cout, k
    (2, 37, 45, 20, 24, 3),         # odd plane: partial tiles, the last input row / column only in the even views
    (2, 38, 46, 24, 28, 3),         # even plane, Cin and Cout below one 32-channel chunk / 16-row weight tile
    (3, 2, 3, 36, 40, 3),           # two input rows: a one-row odd view, one partial tile per image
    (2, 37, 45, 20, 24, 1),         # 1x1, odd plane
    (2, 38, 46, 64, 32, 1),
    (3, 64, 208, 64, 128, 3),       # enc layer2 first conv / downsample
    (3, 64, 208, 64, 128, 1),
    (2, 32, 104, 128, 256, 3),      # enc layer3
    (2, 32, 104, 128, 256, 1),
    (3, 16, 52, 256, 512, 3),       # enc layer4: 8 x 26 output planes
    (3, 16, 52, 256, 512, 1),
    (2, 16, 52, 512, 512, 3),       # ResNet-50 layer4: the gather kernel in split mode, unless a tile is forced
    (2, 16, 52, 1024, 2048, 1),
]
WAYS = [("auto", {}), ("tma mt1 tw16", dict(mt=1, tw_log2=4)), ("tma mt1 tw8", dict(mt=1, tw_log2=3)),
        ("tma mt2", dict(mt=2)), ("gather", dict(no_tma=1))]


def _O():
    from scsfm import nnops
    return nnops


def _inputs(case, mode, seed):
    O = _O()
    B, H, W, Cin, Cout, k = case
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, H, W, Cin, generator=g).to(DEV)
    w = (torch.randn(Cout, k, k, Cin, generator=g) / (k * k * Cin) ** 0.5).to(DEV)
    bias = (0.1 * torch.randn(Cout, generator=g)).to(DEV)
    if mode == "tf32":
        O.round_tf32(x, x)
        O.round_tf32(w, w)
    return x, w, bias


def _ref(x, w, bias, k):
    y = F.conv2d(x.double().permute(0, 3, 1, 2).cpu(), w.double().permute(0, 3, 1, 2).cpu(),
                 None if bias is None else bias.double().cpu(), 2, k // 2)
    return y.permute(0, 2, 3, 1)


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("case", CASES)
def test_conv_fwd_stride2_vs_fp64(case, mode):
    O = _O()
    k = case[5]
    # fp64 reference from the operands the kernel reads.  tf32: products of TF32 operands are exact in fp32, but the wgmma
    # accumulator adds with truncation over a whole K loop (worst on an H100: 1.04e-5, the 512 -> 512 3x3 layer, K = 4608)
    tol = 1e-5 if mode == "tf32x3" else 5e-5
    x, w, bias = _inputs(case, mode, 11 + sum(case))
    want = _ref(x, w, bias, k)
    got = {}
    for name, knobs in WAYS:
        cx = O.ConvCtx(mode)
        cx.tune = O.tune(**knobs)
        assert cx._use_tc("fwd", case[3], case[4], k, 2)
        w_lo = O.split_tf32(w) if cx.split else None
        y = cx.conv_fwd(x, w, bias, 2, k // 2, O.PAD_ZERO, O.ACT_NONE, None, 1, w_lo)
        y2 = cx.conv_fwd(x, w, bias, 2, k // 2, O.PAD_ZERO, O.ACT_NONE, None, 1, w_lo)
        torch.cuda.synchronize()
        assert torch.equal(y.view(torch.int32), y2.view(torch.int32)), name       # no atomics: repeatable bit for bit
        assert rel_l2(y.cpu(), want) < tol, (name, rel_l2(y.cpu(), want))
        got[name] = y
    for name, _ in WAYS[:-1]:
        assert rel_l2(got[name], got["gather"]) < tol, name
    # Cin >= 512 into an output plane of at most 8 x 26 pixels: the gather kernel (faster there in split mode)
    if mode == "tf32x3" and case[3] >= 512:
        assert torch.equal(got["auto"], got["gather"])


EPI_CASES = [(3, 37, 45, 20, 24, 3), (3, 16, 52, 256, 512, 1), (3, 32, 104, 128, 256, 3)]


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("case", EPI_CASES)
def test_conv_fwd_stride2_epilogues(case, mode):
    """bias + ReLU / ELU, the residual addend, ROUND_TF32 and BatchNorm sums over 3 groups (one per image), on the TMA and the
    gather kernel."""
    O = _O()
    B, k = case[0], case[5]
    # fp64 reference from the operands the kernel reads.  tf32: products of TF32 operands are exact in fp32, but the wgmma
    # accumulator adds with truncation over a whole K loop (worst on an H100: 1.04e-5, the 512 -> 512 3x3 layer, K = 4608)
    tol = 1e-5 if mode == "tf32x3" else 5e-5
    x, w, bias = _inputs(case, mode, 7 + sum(case))
    lin = _ref(x, w, bias, k)
    g = torch.Generator().manual_seed(3)
    addend = torch.randn(lin.shape, generator=g).float()
    for name, knobs in (("auto", {}), ("tma mt2", dict(mt=2)), ("gather", dict(no_tma=1))):
        cx = O.ConvCtx(mode)
        cx.tune = O.tune(**knobs)
        w_lo = O.split_tf32(w) if cx.split else None
        for act, fn in ((O.ACT_RELU, torch.relu), (O.ACT_ELU, F.elu)):
            y = cx.conv_fwd(x, w, bias, 2, k // 2, O.PAD_ZERO, act, None, 1, w_lo)
            assert rel_l2(y.cpu(), fn(lin)) < tol, (name, act)
        y = cx.conv_fwd(x, w, bias, 2, k // 2, O.PAD_ZERO, O.ACT_RELU | O.ROUND_TF32, None, 1, w_lo, addend=addend.to(DEV))
        want = torch.relu(lin + addend.double())
        # the stored result is rounded to TF32 (relative error up to 2^-11): compared with unrounded values, 1e-3 is the bound
        assert rel_l2(y.cpu(), want) < 1e-3, name
        assert rel_l2(y, cx.conv_fwd(x, w, bias, 2, k // 2, O.PAD_ZERO, O.ACT_RELU, None, 1, w_lo, addend=addend.to(DEV))) < 1e-3, name
        assert torch.equal(y.view(torch.int32) & 0x1FFF, torch.zeros_like(y.view(torch.int32))), name   # TF32 mantissa
        sums = torch.zeros(O.BN_SLOTS, 3, case[4], 2, dtype=torch.float64, device=DEV)
        y = cx.conv_fwd(x, w, bias, 2, k // 2, O.PAD_ZERO, O.ACT_NONE, sums, 3, w_lo)
        s = sums.sum(0).cpu()
        yd = y.double().cpu().reshape(3, B // 3, -1, case[4])
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
@pytest.mark.parametrize("case", EPI_CASES)
def test_conv_fwd_stride2_fused_bn(case, mode):
    """Eval-mode BatchNorm in the epilogue (with residual, ReLU, the low part of the output) is bitwise the convolution
    followed by bn_apply, and its low part bitwise split_tf32 of its output."""
    O = _O()
    k = case[5]
    x, w, _ = _inputs(case, mode, 5 + sum(case))
    bn = _BN(case[4], 17)
    tab = O.BnEvalTable([bn], 1e-5)
    tab.prepare()
    sc, sh = tab.coeffs[0]
    for name, knobs in (("auto", {}), ("tma mt2", dict(mt=2)), ("gather", dict(no_tma=1))):
        cx = O.ConvCtx(mode)
        cx.tune = O.tune(**knobs)
        w_lo = O.split_tf32(w) if cx.split else None
        y = cx.conv_fwd(x, w, None, 2, k // 2, O.PAD_ZERO, O.ACT_NONE, None, 1, w_lo)
        res = torch.randn(y.shape, generator=torch.Generator().manual_seed(1)).to(DEV)
        z, _ = O.bn_apply(y, None, bn.weight, bn.bias, bn.running_mean, bn.running_var, 0.1, 1e-5, res, 1 | O.ROUND_TF32, 1, with_lo=True)
        zf = cx.conv_fwd(x, w, None, 2, k // 2, O.PAD_ZERO, O.ACT_RELU | O.ROUND_TF32, None, 1, w_lo, bn_scale=sc, bn_shift=sh,
                         addend=res, with_lo=True)
        torch.cuda.synchronize()
        assert _bits(zf, z), (name, float((zf - z).abs().max()))
        assert _bits(zf._scsfm_lo, z._scsfm_lo), name
        assert _bits(zf._scsfm_lo, O.split_tf32(zf)), name
