"""CPU-side checks: the C-ABI library loads and exports every symbol include/scsfm.h declares,
and the host-side argument logic of the wrappers (no kernel launches)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "scsfm.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(scsfm_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_the_hot_path_entry_points():
    syms = _declared_symbols()
    for must in ("scsfm_pairwise_fwd", "scsfm_pairwise_bwd", "scsfm_smooth_fwd", "scsfm_smooth_bwd",
                 "scsfm_inverse_warp2_fwd", "scsfm_inverse_warp2_bwd", "scsfm_last_error", "scsfm_version"):
        assert must in syms


def test_library_exports_every_declared_symbol():
    from scsfm import lib
    if not os.path.exists(lib.LIB_PATH):
        import subprocess
        subprocess.check_call([os.path.join(ROOT, "sc-sfmlearner-release_b200", "build.sh")])
    dll = ctypes.CDLL(lib.LIB_PATH)
    missing = [s for s in _declared_symbols() if not hasattr(dll, s)]
    assert not missing, missing
    assert lib.load().scsfm_version() >= 100
    assert lib.load().scsfm_pairwise_stats_bytes(4, 4) == 4 * (8 + 48) * 8


def test_argument_errors_are_reported_without_a_gpu():
    from scsfm import lib
    L = lib.load()
    rc = L.scsfm_pairwise_fwd(None, 0, None, 1, 16, 16, 0, 0, None, None, None, None)
    assert rc == -1
    assert b"njobs" in L.scsfm_last_error()
    with pytest.raises(ValueError):
        lib.check(rc, "scsfm_pairwise_fwd")


def test_host_side_helpers():
    import torch
    from scsfm import lib, loss_ops
    assert loss_ops._shift_of(256, 256, "d") == 0
    assert loss_ops._shift_of(256, 32, "d") == 3
    with pytest.raises(ValueError):
        loss_ops._shift_of(256, 100, "d")
    assert loss_ops._flags(1, 1, 1) == 7
    assert loss_ops._flags(2, 1, 0) == 2          # the reference's `== True` test: only 1 enables a term
    assert loss_ops._flags(True, False, True) == 5
    with pytest.raises(ValueError):
        loss_ops._padding("reflection")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        lib.dev_f32(torch.zeros(1, 3, 8, 8), "x")


def test_network_operators_reject_bad_arguments_without_a_gpu():
    """Host-side checks of the network operators added for the tensor-core path (no launch happens on an error)."""
    from scsfm import lib
    from scsfm import nnops as O
    L = O._lib()
    n0 = lib.launch_count()
    assert L.scsfm_weight_flip(None, 8, 3, 3, 8, 1, 1, None, 5, None) == -1 and b"weight_flip" in L.scsfm_last_error()
    assert L.scsfm_split_tf32(None, None, 16, None) == -1 and b"split_tf32" in L.scsfm_last_error()
    assert L.scsfm_adam_step(None, None, None, None, 0, 1e-4, 0.9, 0.999, 1e-8, 0.0, 1, None, None, 0, None) == -1
    assert L.scsfm_weight_flip_batched(None, 1, 1, None) == -1
    assert L.scsfm_head_conv_dgrad(None, None, None, 1, 8, 8, 16, None) == -1
    assert L.scsfm_conv2d_fwd(None, None) == -1
    assert lib.launch_count() == n0          # nothing was launched


def test_conv_descriptor_matches_the_c_struct_and_tune_word():
    """The ctypes mirror of ScsfmConv must have the C layout (include/scsfm.h) and nnops.tune() the SCSFM_TUNE_* encoding."""
    import subprocess
    import tempfile
    from scsfm import nnops as O
    src = r'''
#include <stdio.h>
#include <stddef.h>
#include "scsfm.h"
int main(void) {
    printf("%zu %zu %zu %zu %zu %zu %zu\n", sizeof(ScsfmConv), offsetof(ScsfmConv, bn_groups), offsetof(ScsfmConv, act),
           offsetof(ScsfmConv, in_lo), offsetof(ScsfmConv, tune), offsetof(ScsfmConv, debug), offsetof(ScsfmConv, mode));
    printf("%u %u\n", SCSFM_TUNE_NO_TMA | SCSFM_TUNE_MT(2) | SCSFM_TUNE_TW(4) | SCSFM_TUNE_BN(64) | SCSFM_TUNE_WGRAD(2),
           SCSFM_TUNE_MT(1) | SCSFM_TUNE_TW(3) | SCSFM_TUNE_BN(128));
    return 0;
}'''
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", os.path.join(d, "t")])
        out = subprocess.check_output([os.path.join(d, "t")], text=True).split()
    C = O.Conv
    assert [int(v) for v in out[:7]] == [ctypes.sizeof(C), C.bn_groups.offset, C.act.offset, C.in_lo.offset, C.tune.offset, C.debug.offset,
                                         C.mode.offset]
    assert int(out[7]) == O.tune(no_tma=1, mt=2, tw_log2=4, bn=64, wgrad=2) and int(out[8]) == O.tune(mt=1, tw_log2=3, bn=128)


def test_conv_context_is_per_network_state():
    """No process-global convolution mode: every network owns its ConvCtx."""
    import models
    from scsfm import nnops as O
    a, b = models.DispResNet(18, False), models.PoseResNet(18, False)
    assert a.conv_mode == b.conv_mode == "fp32"
    a.set_conv_mode("tf32x3")
    assert a.conv_mode == "tf32x3" and b.conv_mode == "fp32" and a.ctx.split and not b.ctx.tc
    assert a.ctx.rnd() == 0 and O.ConvCtx("tf32").rnd() == O.ROUND_TF32
    with pytest.raises(ValueError):
        a.set_conv_mode("bf16")
    assert not hasattr(O, "CONFIG")

