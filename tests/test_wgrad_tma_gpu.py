"""The TMA weight-gradient kernel (conv_wgrad_tma.cu: stride 1, kh, kw <= 3) against autograd in fp64, forced through the
tune word (SCSFM_TUNE_WGRAD(2)) and as the automatic choice, and against the gather kernel (SCSFM_TUNE_WGRAD(1))."""
import pytest
import torch
import torch.nn.functional as F

from helpers import rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda"

CASES = [
    # B, H, W, Cin, Cout, k, pad_mode (0 zero / 1 reflect)
    (2, 37, 45, 20, 24, 3, 0),      # partial 4 x 16 tiles in both directions, Cin and Cout below one box
    (3, 19, 21, 36, 40, 3, 1),      # reflection: interior on the TMA kernel, ring on the gather kernel
    (2, 3, 3, 64, 64, 3, 1),        # smallest plane reflection padding allows, smaller than one tile
    (6, 3, 5, 64, 128, 3, 0),       # one tile per image: several images inside one split
    (2, 10, 14, 96, 32, 3, 1),      # Cin 96: a half-empty second 64-channel block
    (2, 8, 26, 512, 256, 3, 1),     # deep decoder layer: 8 channel blocks x 4 Cout tiles
    (3, 24, 40, 64, 64, 3, 0),
    (2, 9, 13, 256, 128, 1, 0),     # 1x1 stride 1
    (2, 11, 37, 32, 16, 3, 1),      # Cin 32 -> Cout 16 (tf32: the thin fp32 kernel only takes split mode)
]


def _ref(x, w, dpre, pad_mode):
    k = w.shape[-1]
    pad = k // 2
    xr = F.pad(x, (pad,) * 4, mode="reflect") if pad_mode == 1 and pad else x
    w = w.detach().clone().requires_grad_(True)
    F.conv2d(xr, w, None, 1, 0 if pad_mode == 1 else pad).backward(dpre)
    return w.grad


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("case", CASES)
def test_wgrad_tma_vs_fp64(case, mode):
    from scsfm import nnops as O
    B, H, W, Cin, Cout, k, pad_mode = case
    pad = k // 2
    # fp64 reference from the operands the kernel reads (tf32: products of TF32 operands are exact in fp32); worst tf32
    # relative L2 of these shapes on an H100: 2.4e-6
    tol = 1e-5
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, Cin, H, W, generator=g, dtype=torch.float64)
    dpre = torch.randn(B, Cout, H, W, generator=g, dtype=torch.float64)
    xc = x.float().permute(0, 2, 3, 1).contiguous().to(DEV)
    dc = dpre.float().permute(0, 2, 3, 1).contiguous().to(DEV)
    if mode == "tf32":
        O.round_tf32(xc, xc)
        O.round_tf32(dc, dc)
    # reference from the operands the kernel sees
    want = _ref(xc.double().permute(0, 3, 1, 2).cpu(), torch.zeros(Cout, Cin, k, k, dtype=torch.float64),
                dc.double().permute(0, 3, 1, 2).cpu(), pad_mode)
    got = {}
    for name, forced in (("tma", 2), ("auto", 0), ("gather", 1)):
        cx = O.ConvCtx(mode)
        cx.tune = O.tune(wgrad=forced)
        assert cx._use_tc("wgrad", Cin, Cout, k, 1)
        dw = torch.zeros(Cout, k, k, Cin, device=DEV)
        cx.conv_wgrad(xc, dc, dw, None, 1, pad, pad_mode)
        assert rel_l2(dw.permute(0, 3, 1, 2), want) < tol, name
        got[name] = dw.clone()
        # dw accumulates: a second call doubles it
        cx.conv_wgrad(xc, dc, dw, None, 1, pad, pad_mode)
        assert rel_l2(dw.permute(0, 3, 1, 2), 2 * want) < tol, name
    assert rel_l2(got["tma"], got["gather"]) < tol
