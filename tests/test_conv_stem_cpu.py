"""CPU-side checks of scsfm_conv_plan (which low parts of its activation operands the kernel picked for a call reads in split
mode) and of the split-mode argument checks of the convolution entry points: no kernel is launched."""
import ctypes

import pytest


def _O():
    from scsfm import nnops
    return nnops


def _desc(O, x_shape, w_shape, stride, pad, pad_mode=0, **tune):
    d = O.conv_desc(x_shape, w_shape, stride, pad, pad_mode, O.ACT_NONE)
    d.tune, d.mode = O.tune(**tune), O.MODES.index("tf32x3")
    return d


STEM8 = ((16, 256, 832, 8), (64, 7, 7, 8), 2, 3)
STEM4 = ((12, 256, 832, 4), (64, 7, 7, 4), 2, 3)


def test_plan_reports_the_low_parts_each_kernel_reads():
    O = _O()
    F, D, W = O.PASS_FWD, O.PASS_DGRAD, O.PASS_WGRAD
    lo = {F: O.PLAN_IN_LO, D: O.PLAN_DOUT_LO, W: O.PLAN_IN_LO | O.PLAN_DOUT_LO}

    def q(d, pass_):
        plan = O._lib().scsfm_conv_plan(ctypes.byref(d), pass_)
        assert plan >= 0 and plan & lo[pass_] in (0, lo[pass_]), plan
        return 1 if plan & lo[pass_] else 0
    for stem in (STEM8, STEM4):
        assert q(_desc(O, *stem), F) == 0                      # stem forward: lo(x) from the A fragment
        assert q(_desc(O, *stem, no_tma=1), F) == 1            # the gather kernel reads in_lo
        assert q(_desc(O, *stem), W) == 0                      # TMA weight gradient computes both
        assert q(_desc(O, *stem, wgrad=1), W) == 1             # gather weight gradient reads both
        assert q(_desc(O, *stem), D) == 0                      # Cin < 16: the data gradient runs on the CUDA cores
    # not a stem: other channel counts or padding; the epilogue does not change the choice
    assert q(_desc(O, (2, 64, 64, 12), (64, 7, 7, 12), 2, 3), F) == 1
    assert q(_desc(O, (2, 64, 64, 8), (64, 7, 7, 8), 2, 2), F) == 1
    d = _desc(O, *STEM8)
    d.bias, d.addend = 256, 512
    assert q(d, F) == 0
    assert q(_desc(O, (2, 64, 208, 64), (64, 3, 3, 64), 1, 1), F) == 1
    assert q(_desc(O, (2, 64, 208, 64), (64, 3, 3, 64), 1, 1), W) == 0
    assert q(_desc(O, (2, 64, 208, 64), (64, 3, 3, 64), 1, 1), D) == 1
    assert q(_desc(O, (2, 64, 208, 64), (128, 3, 3, 64), 2, 1), D) == 1
    assert q(_desc(O, (2, 64, 208, 64), (64, 3, 3, 64), 1, 1, O.PAD_REFLECT), W) == 1   # ring: gather kernel


def test_plan_query_rejects_bad_arguments():
    O = _O()
    lib = O._lib()
    n0 = lib.scsfm_launch_count()
    assert lib.scsfm_conv_plan(None, O.PASS_FWD) == -1
    assert lib.scsfm_conv_plan(ctypes.byref(_desc(O, *STEM8)), 3) == -1
    assert lib.scsfm_conv_plan(ctypes.byref(_desc(O, *STEM8)), -1) == -1
    d = _desc(O, *STEM8)
    d.B = 0
    assert lib.scsfm_conv_plan(ctypes.byref(d), O.PASS_FWD) == -1 and b"conv_plan" in lib.scsfm_last_error()
    d = _desc(O, *STEM8)
    d.mode = 3
    assert lib.scsfm_conv_plan(ctypes.byref(d), O.PASS_FWD) == -1 and b"mode" in lib.scsfm_last_error()
    assert lib.scsfm_launch_count() == n0


@pytest.mark.parametrize("tune", [dict(), dict(no_tma=1)])
def test_tf32x3_forward_without_weight_low_part_is_refused(tune):
    O = _O()
    lib = O._lib()
    d = _desc(O, *STEM8, **tune)
    d.inp, d.w, d.out = 256, 640, 512                 # never dereferenced: the call is refused first
    n0 = lib.scsfm_launch_count()
    assert lib.scsfm_conv2d_fwd(ctypes.byref(d), None) == -1 and b"w_lo" in lib.scsfm_last_error()
    assert lib.scsfm_launch_count() == n0


def test_tf32x3_calls_missing_a_low_part_their_kernel_reads_are_refused():
    O = _O()
    lib = O._lib()
    n0 = lib.scsfm_launch_count()
    d = _desc(O, *STEM8, no_tma=1)                    # gather kernel: reads in_lo
    d.inp, d.w, d.out, d.w_lo = 256, 640, 512, 768
    assert lib.scsfm_conv2d_fwd(ctypes.byref(d), None) == -1 and b"in_lo" in lib.scsfm_last_error()
    d = _desc(O, *STEM8, wgrad=1)                     # gather weight gradient: reads in_lo and dout_lo
    d.inp, d.dout, d.dw = 256, 512, 768
    assert lib.scsfm_conv2d_wgrad(ctypes.byref(d), None) == -1 and b"dout_lo" in lib.scsfm_last_error()
    d = _desc(O, (2, 64, 64, 64), (64, 3, 3, 64), 1, 1)
    d.dout, d.w, d.din = 256, 512, 768
    assert lib.scsfm_conv2d_dgrad(ctypes.byref(d), None) == -1 and b"dout_lo" in lib.scsfm_last_error()
    assert lib.scsfm_launch_count() == n0
