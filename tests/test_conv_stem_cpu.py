"""CPU-side checks of scsfm_conv_reads_lo (which kernels read the low parts of their activation operands in split mode)
and of the split-mode argument checks of the tensor-core convolution entry points: no kernel is launched."""
import ctypes

import pytest


def _O():
    from scsfm import nnops
    return nnops


def _desc(O, x_shape, w_shape, stride, pad, pad_mode=0, **tune):
    d = O.conv_desc(x_shape, w_shape, stride, pad, pad_mode, O.ACT_NONE)
    d.tune = O.tune(**tune)
    return d


STEM8 = ((16, 256, 832, 8), (64, 7, 7, 8), 2, 3)
STEM4 = ((12, 256, 832, 4), (64, 7, 7, 4), 2, 3)


def test_reads_lo_answers_per_kernel():
    O = _O()
    q = O._lib().scsfm_conv_reads_lo
    F, D, W = O.PASS_FWD, O.PASS_DGRAD, O.PASS_WGRAD
    for stem in (STEM8, STEM4):
        assert q(ctypes.byref(_desc(O, *stem)), F) == 0                      # stem forward: lo(x) from the A fragment
        assert q(ctypes.byref(_desc(O, *stem, no_tma=1)), F) == 1            # the gather kernel reads in_lo
        assert q(ctypes.byref(_desc(O, *stem)), W) == 0                      # TMA weight gradient computes both
        assert q(ctypes.byref(_desc(O, *stem, wgrad=1)), W) == 1             # gather weight gradient reads both
        assert q(ctypes.byref(_desc(O, *stem)), D) == 1
    # not a stem: other channel counts or padding; the epilogue does not change the choice
    assert q(ctypes.byref(_desc(O, (2, 64, 64, 12), (64, 7, 7, 12), 2, 3)), F) == 1
    assert q(ctypes.byref(_desc(O, (2, 64, 64, 8), (64, 7, 7, 8), 2, 2)), F) == 1
    d = _desc(O, *STEM8)
    d.bias, d.addend = 256, 512
    assert q(ctypes.byref(d), F) == 0
    assert q(ctypes.byref(_desc(O, (2, 64, 208, 64), (64, 3, 3, 64), 1, 1)), F) == 1
    assert q(ctypes.byref(_desc(O, (2, 64, 208, 64), (64, 3, 3, 64), 1, 1)), W) == 0
    assert q(ctypes.byref(_desc(O, (2, 64, 208, 64), (64, 3, 3, 64), 1, 1, O.PAD_REFLECT)), W) == 1   # ring: gather kernel


def test_reads_lo_rejects_bad_arguments():
    O = _O()
    lib = O._lib()
    n0 = lib.scsfm_launch_count()
    assert lib.scsfm_conv_reads_lo(None, O.PASS_FWD) == -1
    assert lib.scsfm_conv_reads_lo(ctypes.byref(_desc(O, *STEM8)), 3) == -1
    assert lib.scsfm_conv_reads_lo(ctypes.byref(_desc(O, *STEM8)), -1) == -1
    d = _desc(O, *STEM8)
    d.B = 0
    assert lib.scsfm_conv_reads_lo(ctypes.byref(d), O.PASS_FWD) == -1 and b"conv_reads_lo" in lib.scsfm_last_error()
    assert lib.scsfm_launch_count() == n0


@pytest.mark.parametrize("tune", [dict(), dict(no_tma=1)])
def test_split_forward_without_weight_low_part_is_refused(tune):
    O = _O()
    lib = O._lib()
    d = _desc(O, *STEM8, **tune)
    d.inp, d.w, d.out, d.split = 256, 640, 512, 1     # never dereferenced: the call is refused first
    n0 = lib.scsfm_launch_count()
    assert lib.scsfm_conv2d_fwd_tc(ctypes.byref(d), None) == -1 and b"w_lo" in lib.scsfm_last_error()
    assert lib.scsfm_launch_count() == n0


def test_split_calls_missing_a_low_part_their_kernel_reads_are_refused():
    O = _O()
    lib = O._lib()
    n0 = lib.scsfm_launch_count()
    d = _desc(O, *STEM8, no_tma=1)                    # gather kernel: reads in_lo
    d.inp, d.w, d.out, d.w_lo, d.split = 256, 640, 512, 768, 1
    assert lib.scsfm_conv2d_fwd_tc(ctypes.byref(d), None) == -1 and b"in_lo" in lib.scsfm_last_error()
    d = _desc(O, *STEM8, wgrad=1)                     # gather weight gradient: reads in_lo and dout_lo
    d.inp, d.dout, d.dw, d.split = 256, 512, 768, 1
    assert lib.scsfm_conv2d_wgrad_tc(ctypes.byref(d), None) == -1 and b"dout_lo" in lib.scsfm_last_error()
    d = _desc(O, (2, 64, 64, 64), (64, 3, 3, 64), 1, 1)
    d.dout, d.w, d.din, d.split = 256, 512, 768, 1
    assert lib.scsfm_conv2d_dgrad_tc(ctypes.byref(d), None) == -1 and b"dout_lo" in lib.scsfm_last_error()
    assert lib.scsfm_launch_count() == n0
