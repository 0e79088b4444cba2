"""Stride-2 weight gradients on the TMA kernel (conv_wgrad_tma.cu: parity-row input views; 3x3 pad 1, 1x1 pad 0 and the 7x7 stems) against
autograd in fp64, forced through the tune word (SCSFM_TUNE_WGRAD(2)), as the automatic choice, and on the gather kernel
(SCSFM_TUNE_WGRAD(1)); both Cout tiles (SCSFM_TUNE_BN(32 | 64)) of the TMA kernel."""
import pytest
import torch
import torch.nn.functional as F

from helpers import rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda"

CASES = [
    # B, H, W, Cin, Cout, k
    (2, 37, 45, 20, 24, 3),         # odd H and W: partial 4 x 16 tiles, last input row / column only on one parity
    (2, 38, 46, 24, 28, 3),         # even H and W, Cin and Cout below one box
    (3, 2, 3, 36, 40, 3),           # two input rows: a one-row odd view, the output is one partial tile
    (6, 7, 9, 64, 128, 3),          # one tile per image: several images inside one split
    (2, 18, 62, 96, 32, 3),         # Cin 96: a half-empty second 64-channel block; Cout 32
    (3, 64, 208, 64, 128, 3),       # enc layer2 first conv
    (2, 32, 104, 128, 256, 3),      # enc layer3 first conv
    (2, 16, 52, 256, 512, 3),       # enc layer4 first conv: 4 x 3 channel-block rows x 8 Cout tiles
    (2, 37, 45, 20, 24, 1),         # 1x1, odd plane
    (3, 64, 208, 64, 128, 1),       # downsample convs
    (2, 32, 104, 128, 256, 1),
    (2, 16, 52, 256, 512, 1),
]


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("case", CASES)
def test_wgrad_tma_stride2_vs_fp64(case, mode):
    from scsfm import nnops as O
    B, H, W, Cin, Cout, k = case
    pad = k // 2
    Ho, Wo = (H + 2 * pad - k) // 2 + 1, (W + 2 * pad - k) // 2 + 1
    tol = 1e-5 if mode == "tf32x3" else 1e-3
    g = torch.Generator().manual_seed(5)
    xc = torch.randn(B, H, W, Cin, generator=g).to(DEV)
    dc = torch.randn(B, Ho, Wo, Cout, generator=g).to(DEV)
    if mode == "tf32":
        O.round_tf32(xc, xc)
        O.round_tf32(dc, dc)
    # reference from the operands the kernel sees
    w = torch.zeros(Cout, Cin, k, k, dtype=torch.float64, requires_grad=True)
    F.conv2d(xc.double().permute(0, 3, 1, 2).cpu(), w, None, 2, pad).backward(dc.double().permute(0, 3, 1, 2).cpu())
    want = w.grad
    got = {}
    for name, tune in (("tma", dict(wgrad=2)), ("tma bn32", dict(wgrad=2, bn=32)), ("tma bn64", dict(wgrad=2, bn=64)),
                       ("auto", {}), ("gather", dict(wgrad=1))):
        cx = O.ConvCtx(mode)
        cx.tune = O.tune(**tune)
        assert cx._use_tc("wgrad", Cin, Cout, k, 2)
        dw = torch.zeros(Cout, k, k, Cin, device=DEV)
        cx.conv_wgrad(xc, dc, dw, None, 2, pad, O.PAD_ZERO)
        assert rel_l2(dw.permute(0, 3, 1, 2), want) < tol, name
        got[name] = dw.clone()
        # dw accumulates: a second call doubles it
        cx.conv_wgrad(xc, dc, dw, None, 2, pad, O.PAD_ZERO)
        assert rel_l2(dw.permute(0, 3, 1, 2), 2 * want) < tol, name
    for name in ("tma", "tma bn32", "tma bn64", "auto"):
        assert rel_l2(got[name], got["gather"]) < tol, name


STEMS = [
    # B, H, W, Cin (padded), Cout
    (2, 5, 7, 8, 24),               # a plane smaller than one tile; Cout 24: a partial Cout tile
    (2, 37, 45, 4, 64),             # odd plane: partial tiles, the last input row only in the even-row view
    (2, 38, 46, 8, 64),
    (3, 64, 208, 4, 64),            # DispResNet stem (channels padded 3 -> 4)
    (2, 128, 416, 8, 64),           # PoseResNet stem (channels padded 6 -> 8)
]


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("case", STEMS)
def test_wgrad_tma_stem_vs_fp64(case, mode):
    """The 7x7 stride-2 pad-3 stems: (dx, c) on M, one accumulator.  The pad channels of the networks' operands are zero;
    the last real channel is zeroed here as they are, the gradient of every channel is still checked."""
    from scsfm import nnops as O
    B, H, W, Cin, Cout = case
    Ho, Wo = (H + 6 - 7) // 2 + 1, (W + 6 - 7) // 2 + 1
    tol = 1e-5 if mode == "tf32x3" else 1e-3
    g = torch.Generator().manual_seed(9)
    xc = torch.randn(B, H, W, Cin, generator=g)
    xc[..., -1] = 0
    xc = xc.to(DEV)
    dc = torch.randn(B, Ho, Wo, Cout, generator=g).to(DEV)
    if mode == "tf32":
        O.round_tf32(xc, xc)
        O.round_tf32(dc, dc)
    w = torch.zeros(Cout, Cin, 7, 7, dtype=torch.float64, requires_grad=True)
    F.conv2d(xc.double().permute(0, 3, 1, 2).cpu(), w, None, 2, 3).backward(dc.double().permute(0, 3, 1, 2).cpu())
    want = w.grad
    got = {}
    for name, tune in (("tma", dict(wgrad=2)), ("auto", {}), ("gather", dict(wgrad=1))):
        cx = O.ConvCtx(mode)
        cx.tune = O.tune(**tune)
        dw = torch.zeros(Cout, 7, 7, Cin, device=DEV)
        cx.conv_wgrad(xc, dc, dw, None, 2, 3, O.PAD_ZERO)
        assert rel_l2(dw.permute(0, 3, 1, 2), want) < tol, name
        got[name] = dw.clone()
        cx.conv_wgrad(xc, dc, dw, None, 2, 3, O.PAD_ZERO)
        assert rel_l2(dw.permute(0, 3, 1, 2), 2 * want) < tol, name
    for name in ("tma", "auto"):
        assert rel_l2(got[name], got["gather"]) < tol, name
