"""scsfm_conv_plan pinned for every convolution the networks make: the layers of tools/conv_layers.py and the pose head's
256 -> 6 convolution, in the three modes and the three passes, with tune 0 and with each forcing knob.  The expected kernel
and operand flags are restated here from the routing rules (conv_plan in conv_tc.cu).  No GPU needed."""
import ctypes

import pytest

from test_conv_calls_fp64_gpu import _conv_layers_table

KNOBS = [dict(), dict(no_tma=1), dict(mt=1), dict(mt=2), dict(tw_log2=3), dict(tw_log2=4), dict(bn=64), dict(wgrad=1),
         dict(wgrad=2), dict(wgrad=3)]
POSE_HEAD = ("pose head 1x1 256->6", 16, 8, 26, 256, 6, 1, 1, 0, 0)


def _layers():
    return _conv_layers_table() + [POSE_HEAD]


def _expected(O, layer, mode, pass_, knobs):
    _, B, H, W, Cin, Cout, k, s, pad, refl = layer
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    x3, no_tma = mode == "tf32x3", knobs.get("no_tma", 0)
    forced = any(knobs.get(n, 0) for n in ("mt", "tw_log2", "bn"))
    wgrad = knobs.get("wgrad", 0)
    thin = k == 3 and s == 1 and pad == 1 and Ho >= 3 and Wo >= 3 and Cout == 16 and Cin in (16, 32)
    if pass_ == O.PASS_FWD:
        if mode == "fp32" or Cin % 4 or Cout < 16:
            return O.KERNEL_SIMT
        lo = O.PLAN_W_LO | O.PLAN_IN_LO if x3 else 0
        if not no_tma and s == 2 and k == 7 and pad == 3 and not refl and Cin in (4, 8) and Cout == 64:
            return O.KERNEL_STEM | (O.PLAN_W_LO if x3 else 0)
        tma = not no_tma and k <= 3 and Cout % 4 == 0
        if not refl and tma and not (s == 2 and x3 and Cin >= 512 and Ho * Wo <= 8 * 26 and not forced):
            return O.KERNEL_TMA | lo
        if refl and s == 1 and Ho >= 3 and Wo >= 3 and (Ho * Wo >= 64 * 208 or forced) and tma:
            return O.KERNEL_TMA_RING | lo
        return O.KERNEL_GATHER | lo
    if pass_ == O.PASS_DGRAD:
        # the forward routing on dout, zero-padded stride-1 (sub-)convolutions with at most 2 x 2 taps per stride-2 class
        if mode == "fp32" or s not in (1, 2) or Cout % 4 or Cin < 16:
            return O.KERNEL_SIMT
        flags = O.PLAN_FLIPPED | (O.PLAN_DOUT_LO | O.PLAN_W_LO if x3 else 0)
        return (O.KERNEL_TMA if not no_tma and k <= 3 else O.KERNEL_GATHER) | flags
    if mode == "fp32" or Cin % 4 or Cout % 4 or Cout < 16:
        return O.KERNEL_THIN if thin and wgrad != 1 else O.KERNEL_SIMT
    if thin and (wgrad == 3 or (wgrad == 0 and x3)):
        return O.KERNEL_THIN
    lo = O.PLAN_IN_LO | O.PLAN_DOUT_LO if x3 else 0
    stem = s == 2 and k == 7 and Cin in (4, 8)
    tma = not no_tma and (stem or k <= 3) and not (refl and (Ho < 3 or Wo < 3))
    if wgrad != 1 and tma:
        return O.KERNEL_TMA_RING | lo if refl else O.KERNEL_TMA
    return O.KERNEL_GATHER | lo


@pytest.mark.parametrize("mode", ["fp32", "tf32", "tf32x3"])
def test_plan_of_every_network_convolution(mode):
    from scsfm import nnops as O
    lib = O._lib()
    n0 = lib.scsfm_launch_count()
    checked, kernels = 0, set()
    for layer in _layers():
        _, B, H, W, Cin, Cout, k, s, pad, refl = layer
        for pass_ in (O.PASS_FWD, O.PASS_DGRAD, O.PASS_WGRAD):
            for knobs in KNOBS:
                d = O.conv_desc((B, H, W, Cin), (Cout, k, k, Cin), s, pad, O.PAD_REFLECT if refl else O.PAD_ZERO, O.ACT_NONE)
                d.mode, d.tune = O.MODES.index(mode), O.tune(**knobs)
                got, want = lib.scsfm_conv_plan(ctypes.byref(d), pass_), _expected(O, layer, mode, pass_, knobs)
                assert got == want, (layer[0], pass_, knobs, hex(got), hex(want))
                kernels.add(got & 0xff)
                checked += 1
    assert checked == len(_layers()) * 3 * len(KNOBS)
    # ConvCtx._use_tc: the tensor cores exactly where the plan picks a kernel other than the CUDA-core one in a tf32 mode
    cx = O.ConvCtx(mode)
    for _, B, H, W, Cin, Cout, k, s, pad, refl in _layers():
        for kind, pass_ in (("fwd", O.PASS_FWD), ("dgrad", O.PASS_DGRAD), ("wgrad", O.PASS_WGRAD)):
            want = mode != "fp32" and _expected(O, (None, B, H, W, Cin, Cout, k, s, pad, refl), mode, pass_, {}) & 0xff != O.KERNEL_SIMT
            assert cx._use_tc(kind, Cin, Cout, k, s) == want, (kind, Cin, Cout, k, s)
    assert kernels == ({O.KERNEL_SIMT, O.KERNEL_THIN} if mode == "fp32" else set(range(6)))
    assert lib.scsfm_launch_count() == n0


def test_plan_is_memoised_per_descriptor_key():
    """ConvCtx asks the library once per distinct call: the integer fields and the null pointers make the key."""
    from scsfm import nnops as O
    cx = O.ConvCtx("tf32x3")
    d = O.conv_desc((12, 64, 208, 64), (64, 3, 3, 64), 1, 1, O.PAD_ZERO, O.ACT_NONE)
    cx._finish(d)
    p = cx.plan(d, O.PASS_WGRAD)
    assert p == O.KERNEL_TMA and len(cx._plans) == 1
    d.inp, d.dout = 256, 512                    # other pointers: a new key
    assert cx.plan(d, O.PASS_WGRAD) == p and len(cx._plans) == 2
    d.inp, d.dout = 768, 1024                   # the same pointers null or not: the same key
    assert cx.plan(d, O.PASS_WGRAD) == p and len(cx._plans) == 2
    cx.tune = O.tune(wgrad=1)
    cx._finish(d)
    assert cx.plan(d, O.PASS_WGRAD) == O.KERNEL_GATHER | O.PLAN_IN_LO | O.PLAN_DOUT_LO and len(cx._plans) == 3
