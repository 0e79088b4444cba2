"""Thin Python layer over the network entry points of libscsfm (include/scsfm.h, "Network operators").

Tensors are torch CUDA tensors used as typed device buffers: activations NHWC `[B,H,W,C]` fp32
contiguous, conv weights `[Cout,kh,kw,Cin]`.  Every function enqueues on torch's current stream.
"""
import ctypes

import torch

from . import lib as L

PAD_ZERO, PAD_REFLECT = 0, 1
ACT_NONE, ACT_RELU, ACT_ELU, ACT_DISP = 0, 1, 2, 3
BN_SLOTS = 16      # SCSFM_BN_SLOTS: replicas of the fused BatchNorm sums
ROUND_TF32 = 0x100  # SCSFM_ROUND_TF32: store the result rounded to TF32 (operand of a tensor-core conv)
BN_FROZEN = 0x200   # SCSFM_BN_FROZEN: bn_backward with the running statistics held fixed (eval mode)
OPERAND_TF32, OPERAND_RAW, OPERAND_LO = 0, 1, 2      # SCSFM_OPERAND_*

# Arithmetic of the convolutions (a property of each network, see ConvCtx -- there is no process-global mode):
#   "fp32"    exact CUDA-core kernels everywhere
#   "tf32"    wgmma tensor-core kernels, single TF32 product (the reference's cuDNN default on a GPU; ~1e-3 per layer)
#   "tf32x3"  wgmma kernels with split-accumulate operands: hi*hi + lo*hi + hi*lo, short chains added in fp32 registers
#             (fp32-level products; the 1e-4 parity mode on the tensor cores)
MODES = ("fp32", "tf32", "tf32x3")


def tune(no_tma=0, mt=0, tw_log2=0, bn=0, wgrad=0):
    """ScsfmConv.tune word (include/scsfm.h): per-call experiment knobs of the tensor-core kernels."""
    t = 1 if no_tma else 0
    t |= (mt & 3) << 4
    t |= ((tw_log2 - 2 if tw_log2 else 0) & 3) << 6
    t |= {0: 0, 16: 1, 32: 2, 64: 3, 128: 4}[bn] << 8
    t |= (wgrad & 3) << 12
    return t


class Conv(ctypes.Structure):
    _fields_ = ([(n, ctypes.c_void_p) for n in ("inp", "w", "bias", "out", "dout", "din", "addend", "dw", "dbias",
                                                "bn_sums")] +
                [(n, ctypes.c_int) for n in ("bn_groups", "B", "Hi", "Wi", "Cin", "Ho", "Wo", "Cout", "kh", "kw",
                                             "stride", "pad", "pad_mode", "act")] +
                [(n, ctypes.c_void_p) for n in ("in_lo", "w_lo", "dout_lo")] +
                [("tune", ctypes.c_uint), ("debug", ctypes.c_void_p)] +
                [(n, ctypes.c_void_p) for n in ("bn_scale", "bn_shift", "out_lo")] +
                [("split", ctypes.c_int)])

PASS_FWD, PASS_DGRAD, PASS_WGRAD = 0, 1, 2        # SCSFM_PASS_* of scsfm_conv_reads_lo


_bound = False


def _lib():
    global _bound
    lib = L.load()
    if not _bound:
        I, P, LL, F = ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_float
        CP = ctypes.POINTER(Conv)
        for name in ("scsfm_conv2d_fwd_simt", "scsfm_conv2d_dgrad_simt", "scsfm_conv2d_wgrad_simt",
                     "scsfm_conv2d_fwd_tc", "scsfm_conv2d_dgrad_tc", "scsfm_conv2d_wgrad_tc"):
            getattr(lib, name).argtypes = [CP, P]
        lib.scsfm_conv_reads_lo.argtypes = [CP, I]
        lib.scsfm_round_tf32.argtypes = [P, P, LL, P]
        lib.scsfm_split_tf32.argtypes = [P, P, LL, P]
        lib.scsfm_weight_flip.argtypes = [P, I, I, I, I, P, I, P]
        lib.scsfm_weight_flip_s2.argtypes = [P, I, I, I, I, I, P, I, P]
        lib.scsfm_weight_flip_batched.argtypes = [P, I, I, P]
        lib.scsfm_nchw_to_nhwc.argtypes = [P, P, I, I, I, I, P, P]
        lib.scsfm_nhwc_to_nchw.argtypes = [P, I, I, I, I, P, P]
        lib.scsfm_stem_dgrad.argtypes = [P, P, I, I, I, I, P, P, P]
        lib.scsfm_head_conv_fwd.argtypes = [P, P, P, P, I, I, I, I, I, P]
        lib.scsfm_head_conv_wgrad.argtypes = [P, P, P, P, I, I, I, I, P]
        lib.scsfm_head_conv_dgrad.argtypes = [P, P, P, I, I, I, I, P]
        lib.scsfm_nchw_to_nhwc_pad.argtypes = [P, P, I, I, I, I, I, P, I, P]
        lib.scsfm_pad_channels.argtypes = [P, LL, I, I, P, I, P]
        lib.scsfm_unpad_add.argtypes = [P, LL, I, I, P, P]
        lib.scsfm_bn_prepare.argtypes = [P, I, I, LL, P, P, P, P, F, F, I, P, P]
        lib.scsfm_bn_apply.argtypes = [P, P, P, P, P, P, F, F, P, P, P, P, LL, I, I, I, P]
        lib.scsfm_bn_eval_prepare_batched.argtypes = [P, I, P]
        lib.scsfm_bn_backward.argtypes = [P, P, P, P, P, P, P, P, P, P, LL, I, I, I, P, P]
        lib.scsfm_maxpool_fwd.argtypes = [P, I, I, I, I, P, P, P]
        lib.scsfm_maxpool_bwd.argtypes = [P, P, I, I, I, I, P, I, P]
        lib.scsfm_upcat_fwd.argtypes = [P, P, I, I, I, I, I, P, P]
        lib.scsfm_fold_bwd.argtypes = [P, I, I, I, I, I, I, P, P, I, I, P, P]
        lib.scsfm_act_bwd.argtypes = [P, P, LL, I, P]
        lib.scsfm_spatial_mean_fwd.argtypes = [P, I, I, I, F, P, P]
        lib.scsfm_spatial_mean_bwd.argtypes = [P, I, I, I, F, P, P]
        lib.scsfm_adam_step.argtypes = [P, P, P, P, LL, F, F, F, F, F, I, P, P, I, P]
        lib.scsfm_adam_step_masked.argtypes = [P, P, P, P, LL, P, F, F, F, F, F, I, P, P, I, P]
        _bound = True
    return lib


def round_tf32(src, dst):
    L.launch(_lib().scsfm_round_tf32, "scsfm_round_tf32", "weight_round", 1, 8.0 * src.numel(), L.ptr(src), L.ptr(dst), src.numel(), L.stream())


def split_tf32(src, dst=None):
    """Low part of a split-accumulate operand: dst = tf32(src - trunc_tf32(src)) (ScsfmConv.in_lo / w_lo / dout_lo)."""
    if dst is None:
        dst = torch.empty_like(src)
    L.launch(_lib().scsfm_split_tf32, "scsfm_split_tf32", "split", 1, 8.0 * src.numel(), L.ptr(src), L.ptr(dst), src.numel(), L.stream())
    return dst


def lo_of(t):
    """Low part of tensor `t`, computed once per tensor object (activations and gradients are written once and then only
    read as convolution operands; the cache lives on the tensor object and dies with it)."""
    lo = getattr(t, "_scsfm_lo", None)
    if lo is None:
        lo = split_tf32(t)
        t._scsfm_lo = lo
    return lo


def empty(shape, like):
    return torch.empty(shape, device=like.device, dtype=torch.float32)


def aligned64(n):
    """n rounded up to a multiple of 64 elements: slices of a packed fp32 buffer at such offsets start on a 256-byte
    boundary (float4 loads)."""
    return (n + 63) // 64 * 64


def tc_supported(kind, Cin, Cout, kh, stride):
    """Shapes the tensor-core kernels take; everything else runs the CUDA-core kernel."""
    if kind == "fwd":
        return Cin % 4 == 0 and Cout >= 16
    if kind == "dgrad":                      # forward kernel on dout: its "Cin" is Cout, its "Cout" is Cin
        return stride in (1, 2) and Cout % 4 == 0 and Cin >= 16
    if kind == "wgrad":
        return Cin % 4 == 0 and Cout % 4 == 0 and Cout >= 16
    return False


def _s2_classes(kh, kw, pad):
    """Parity classes (py, px) of a stride-2 data gradient: taps kept = jh x jw starting at (dy_max, dx_max), step 2."""
    out = []
    for py in range(2):
        for px in range(2):
            dy_max, dx_max = kh - 1, kw - 1
            while dy_max >= 0 and ((py + pad - dy_max) & 1):
                dy_max -= 1
            while dx_max >= 0 and ((px + pad - dx_max) & 1):
                dx_max -= 1
            jh = 0 if dy_max < 0 else dy_max // 2 + 1
            jw = 0 if dx_max < 0 else dx_max // 2 + 1
            out.append((jh, jw, dy_max, dx_max))
    return out


class FlipTable:
    """Device job table of every cached flip of one context (one network's operand arena)."""

    def __init__(self, cache, device):
        self.keys = sorted(cache)
        rows, blk = [], 0
        for key in self.keys:
            ptr, (Cout, kh, kw, Cin), stride, pad, operand = key
            dst = cache[key][1].data_ptr()
            jobs = [(kh, kw, kh - 1, kw - 1)] if stride == 1 else _s2_classes(kh, kw, pad)
            for (jh, jw, dy_max, dx_max) in jobs:
                total = Cout * jh * jw * Cin
                if total > 0:
                    rows.append([ptr, dst, Cout, kh, kw, Cin, jh, jw, dy_max, dx_max, stride | (operand << 8), blk])
                    blk += ((Cout + 31) // 32) * ((Cin + 31) // 32) * jh * jw      # one block per 32x32 tile of one tap
                dst += 4 * total
        self.n_rows, self.total_blocks, self.bytes = len(rows), blk, 8.0 * sum(cache[k][1].numel() for k in self.keys)
        rows.append([0] * 11 + [blk])
        self.table = torch.tensor(rows, dtype=torch.int64).to(device)


def conv_desc(x_shape, w, stride, pad, pad_mode, act):
    """ScsfmConv of a convolution of an input of shape x_shape with weights w (a tensor, or only their shape)."""
    B, Hi, Wi, Cin = x_shape
    Cout, kh, kw, _ = w if isinstance(w, tuple) else w.shape
    w = None if isinstance(w, tuple) else w
    Ho = (Hi + 2 * pad - kh) // stride + 1
    Wo = (Wi + 2 * pad - kw) // stride + 1
    return Conv(None, L.ptr(w), None, None, None, None, None, None, None, None, 1, B, Hi, Wi, Cin, Ho, Wo, Cout, kh, kw,
                stride, pad, pad_mode, act, None, None, None, 0, None, None, None, None)


def _tag(d):
    if L.PROF["enabled"]:
        L.TAG["next"] = "B%d %dx%d C%d->%d k%d s%d -> %dx%d" % (d.B, d.Hi, d.Wi, d.Cin, d.Cout, d.kh, d.stride, d.Ho, d.Wo)


def _flops(d):
    """Algorithmic FLOPs of one conv pass: 2 * (B*Ho*Wo) * Cout * (kh*kw*Cin)."""
    return 2.0 * d.B * d.Ho * d.Wo * d.Cout * d.kh * d.kw * d.Cin


class ConvCtx:
    """Convolution context of ONE network: arithmetic mode, experiment knobs and the cache of flipped / transposed
    data-gradient weights.  Everything the convolution entry points need beyond their tensor arguments lives here (and
    travels to the C library inside the ScsfmConv descriptor), not in module-level state."""

    def __init__(self, mode="fp32"):
        if mode not in MODES:
            raise ValueError("conv mode must be one of %s, got %r" % (MODES, mode))
        self.mode = mode
        self.tune = 0                 # ScsfmConv.tune of every call made through this context (see tune())
        self.debug = None             # ScsfmConv.debug: uint64 tensor [8 * SMs] of per-role cycle counters, or None
        self._flips = {}              # (source pointer, shape, stride, pad, operand) -> (source tensor, flipped weights)
        self._table = None
        self.sums_pool = None         # fp64 scratch of the fused BatchNorm sums of this network's calls (scsfm.nets._pool)
        # Optional side stream for the weight gradients: a layer's wgrad is off the backward's critical path (only the
        # optimizer reads dW), so it can run next to the dgrad / BatchNorm chain and fill the SMs their small grids leave idle.
        # Operand tensors are kept alive until join_wgrad() so that the caching allocator cannot recycle them early.
        self.wgrad_stream = None
        self._wgrad_keep = []

    # -- mode -----------------------------------------------------------------------------------------
    @property
    def tc(self):
        return self.mode != "fp32"

    @property
    def split(self):
        return self.mode == "tf32x3"

    def rnd(self):
        """Flag to OR into act / relu arguments of kernels whose output feeds a single-product TF32 convolution."""
        return ROUND_TF32 if self.mode == "tf32" else 0

    @property
    def operand(self):
        """SCSFM_OPERAND_* of tensors prepared for the tensor cores (padded stem input / weights)."""
        return OPERAND_TF32 if self.mode == "tf32" else OPERAND_RAW

    def _use_tc(self, kind, Cin, Cout, kh, stride):
        return self.tc and tc_supported(kind, Cin, Cout, kh, stride)

    def _finish(self, d):
        d.tune = self.tune
        d.debug = self.debug.data_ptr() if self.debug is not None else None

    def _reads_lo(self, d, pass_):
        """tf32x3: does the kernel picked for descriptor d (its tune included) read the low parts of its activation
        operands?  The stem forward and the TMA / thin-layer weight gradients compute them themselves."""
        rc = _lib().scsfm_conv_reads_lo(ctypes.byref(d), pass_)
        L.check(0 if rc >= 0 else rc, "scsfm_conv_reads_lo")
        return rc == 1

    def wgrad_reads_lo(self, x_shape, w_shape, stride, pad, pad_mode=PAD_ZERO):
        """Whether conv_wgrad of this shape will read lo(x) and lo(dout): False outside tf32x3, and where its kernel
        computes them itself (a producer of dout can then skip writing lo(dout))."""
        if not (self.split and self._use_tc("wgrad", x_shape[-1], w_shape[0], w_shape[1], stride)):
            return False
        d = conv_desc(tuple(x_shape), tuple(w_shape), stride, pad, pad_mode, ACT_NONE)
        self._finish(d)
        return self._reads_lo(d, PASS_WGRAD)

    # -- flipped weights of the data gradients -----------------------------------------------------------
    def flipped_weights(self, w, stride, pad, operand):
        """[Cout,kh,kw,Cin] -> weights of the transposed conv ([Cin,kh,kw,Cout], reversed taps; for stride 2 the four
        parity-class tap subsets back to back) as operand kind `operand`.  Cached per source tensor (the entry keeps the
        source alive, so its address cannot be recycled while the entry exists); refreshed in place by refresh_flips()."""
        key = (w.data_ptr(), tuple(w.shape), stride, pad, operand)
        hit = self._flips.get(key)
        if hit is None:
            Cout, kh, kw, Cin = w.shape
            wt = empty((Cin, kh, kw, Cout), w)
            if stride == 1:
                L.launch(_lib().scsfm_weight_flip, "scsfm_weight_flip", "weight_flip", 1, 8.0 * w.numel(), L.ptr(w), Cout, kh, kw, Cin,
                         L.ptr(wt), operand, L.stream())
            else:
                L.launch(_lib().scsfm_weight_flip_s2, "scsfm_weight_flip_s2", "weight_flip", 4, 8.0 * w.numel(), L.ptr(w), Cout, kh, kw,
                         Cin, pad, L.ptr(wt), operand, L.stream())
            hit = self._flips[key] = (w, wt)
            self._table = None
        return hit[1]

    def refresh_flips(self, device):
        """The source weights have changed (optimizer step): recompute every cached flip with one launch."""
        if not self._flips:
            return
        if self._table is None:
            self._table = FlipTable(self._flips, device)
        tab = self._table
        L.launch(_lib().scsfm_weight_flip_batched, "scsfm_weight_flip_batched", "weight_flip", 1, tab.bytes, L.ptr(tab.table), tab.n_rows,
                 tab.total_blocks, L.stream())

    def invalidate(self):
        self._flips.clear()
        self._table = None

    # -- convolutions ---------------------------------------------------------------------------------------
    def conv_fwd(self, x, w, bias=None, stride=1, pad=0, pad_mode=PAD_ZERO, act=ACT_NONE, bn_sums=None, bn_groups=1, w_lo=None,
                 bn_scale=None, bn_shift=None, addend=None, with_lo=False):
        """y = act(conv(x, w) + bias); optionally accumulates per-(group, channel) sum / sum-of-squares of y.
        w_lo: low part of the weights (tf32x3 mode).
        Eval-mode BatchNorm fused into the epilogue: y = act(fmaf(conv(x, w), bn_scale, bn_shift) + addend) with the
        per-channel coefficients of bn_eval_prepare() (no bias, no bn_sums).  with_lo: also write the low part of y
        (attached to y like lo_of() would), for a following tf32x3 convolution."""
        lib = _lib()
        d = conv_desc(x.shape, w, stride, pad, pad_mode, act)
        y = empty((d.B, d.Ho, d.Wo, d.Cout), x)
        d.inp, d.bias, d.out, d.bn_sums, d.bn_groups = x.data_ptr(), bias.data_ptr() if bias is not None else None, \
            y.data_ptr(), bn_sums.data_ptr() if bn_sums is not None else None, bn_groups
        if bn_scale is not None:
            d.bn_scale, d.bn_shift = bn_scale.data_ptr(), bn_shift.data_ptr()
        if addend is not None:
            d.addend = addend.data_ptr()
        if with_lo:
            y._scsfm_lo = empty(y.shape, y)
            d.out_lo = y._scsfm_lo.data_ptr()
        tc = self._use_tc("fwd", d.Cin, d.Cout, d.kh, stride)
        if tc and self.split:
            if w_lo is None:
                raise RuntimeError("tf32x3 convolution called without the low part of its weights")
            d.w_lo, d.split = w_lo.data_ptr(), 1
        self._finish(d)
        if tc and self.split and self._reads_lo(d, PASS_FWD):
            d.in_lo = lo_of(x).data_ptr()
        _tag(d)
        fn = lib.scsfm_conv2d_fwd_tc if tc else lib.scsfm_conv2d_fwd_simt
        L.launch(fn, "scsfm_conv2d_fwd", "conv_fwd_tc" if tc else "conv_fwd_simt", 1, _flops(d), ctypes.byref(d), L.stream())
        return y

    def conv_dgrad(self, dout, w, x_shape, stride=1, pad=0, addend=None, padded_input=False, w_src=None):
        """Gradient w.r.t. the conv input.  padded_input=True returns the gradient of the reflect-PADDED input
        ([B,H+2,W+2,C], to be folded by fold_bwd) for a pad-1 reflection conv.  w: the forward operand weights
        [Cout,kh,kw,Cin]; w_src (tf32x3): the raw weights both flipped parts are derived from (defaults to w)."""
        lib = _lib()
        B, Hi, Wi, Cin = x_shape
        if padded_input:
            Hi, Wi, pad = Hi + 2, Wi + 2, 0
        d = conv_desc((B, Hi, Wi, Cin), w, stride, pad, PAD_ZERO, ACT_NONE)
        assert (d.Ho, d.Wo, d.Cout) == tuple(dout.shape[1:]), (d.Ho, d.Wo, d.Cout, dout.shape)
        din = empty((B, Hi, Wi, Cin), dout)
        d.dout, d.din, d.addend = dout.data_ptr(), din.data_ptr(), addend.data_ptr() if addend is not None else None
        tc = self._use_tc("dgrad", d.Cin, d.Cout, d.kh, stride)
        if tc:
            if self.split:
                src = w if w_src is None else w_src
                d.w = self.flipped_weights(src, stride, pad, OPERAND_RAW).data_ptr()
                d.w_lo = self.flipped_weights(src, stride, pad, OPERAND_LO).data_ptr()
                d.dout_lo, d.split = lo_of(dout).data_ptr(), 1
            else:
                d.w = self.flipped_weights(w, stride, pad, OPERAND_TF32).data_ptr()
        self._finish(d)
        _tag(d)
        fn = lib.scsfm_conv2d_dgrad_tc if tc else lib.scsfm_conv2d_dgrad_simt
        L.launch(fn, "scsfm_conv2d_dgrad", "conv_dgrad_tc" if tc else "conv_dgrad_simt", 1, _flops(d), ctypes.byref(d), L.stream())
        return din

    def conv_wgrad(self, x, dout, dw, dbias=None, stride=1, pad=0, pad_mode=PAD_ZERO):
        """dw += dout^T * gather(x); dbias += column sums of dout.  With a wgrad stream set the launch goes there (after
        everything already enqueued on the current stream); join_wgrad() must follow before dw is read."""
        lib = _lib()
        d = conv_desc(x.shape, dw, stride, pad, pad_mode, ACT_NONE)
        assert (d.Ho, d.Wo, d.Cout) == tuple(dout.shape[1:])
        d.inp, d.dout, d.dw, d.dbias = x.data_ptr(), dout.data_ptr(), dw.data_ptr(), dbias.data_ptr() if dbias is not None else None
        d.w = None
        tc = self._use_tc("wgrad", d.Cin, d.Cout, d.kh, stride)
        keep = [x, dout]
        self._finish(d)
        if tc and self.split:
            d.split = 1
            if self._reads_lo(d, PASS_WGRAD):
                x_lo, dout_lo = lo_of(x), lo_of(dout)      # (computed on the CURRENT stream: the data gradient reads them too)
                d.in_lo, d.dout_lo = x_lo.data_ptr(), dout_lo.data_ptr()
                keep += [x_lo, dout_lo]
        _tag(d)
        fn = lib.scsfm_conv2d_wgrad_tc if tc else lib.scsfm_conv2d_wgrad_simt
        with self.on_wgrad_stream(keep):
            L.launch(fn, "scsfm_conv2d_wgrad", "conv_wgrad_tc" if tc else "conv_wgrad_simt", 2 if dbias is not None else 1, _flops(d),
                     ctypes.byref(d), L.stream())

    def on_wgrad_stream(self, keep=()):
        """Context: the weight-gradient side stream, ordered after the work already enqueued on the current stream (no-op
        without a side stream)."""
        import contextlib
        if self.wgrad_stream is None:
            return contextlib.nullcontext()
        ev = torch.cuda.Event()
        ev.record()
        self.wgrad_stream.wait_event(ev)
        self._wgrad_keep.extend(keep)
        return torch.cuda.stream(self.wgrad_stream)

    def join_wgrad(self):
        """The current stream waits for every weight gradient enqueued so far; their operands may be released."""
        if self.wgrad_stream is not None:
            torch.cuda.current_stream().wait_stream(self.wgrad_stream)
        self._wgrad_keep.clear()


def head_fwd(x, w, bias, act):
    """Disparity head: 3x3 reflect conv to one channel (+ activation).  x [B,H,W,C], w [1,3,3,C] -> [B,H,W,1]."""
    B, H, W, C = x.shape
    out = empty((B, H, W, 1), x)
    L.launch(_lib().scsfm_head_conv_fwd, "scsfm_head_conv_fwd", "head_fwd", 1, 4.0 * x.numel(), L.ptr(x), L.ptr(w), L.ptr(bias), L.ptr(out),
             B, H, W, C, act, L.stream())
    return out


def head_dgrad(dpre, w, x_shape):
    """Gradient of the disparity head w.r.t. its reflection-padded input: dpre [B,H,W,1], w [1,3,3,C] -> [B,H+2,W+2,C]."""
    B, H, W, C = x_shape
    dpad = empty((B, H + 2, W + 2, C), dpre)
    L.launch(_lib().scsfm_head_conv_dgrad, "scsfm_head_conv_dgrad", "head_dgrad", 1, 4.0 * dpad.numel(), L.ptr(dpre), L.ptr(w), L.ptr(dpad),
             B, H, W, C, L.stream())
    return dpad


def head_wgrad(x, dpre, dw, dbias):
    B, H, W, C = x.shape
    L.launch(_lib().scsfm_head_conv_wgrad, "scsfm_head_conv_wgrad", "head_wgrad", 1, 4.0 * x.numel(), L.ptr(x), L.ptr(dpre), L.ptr(dw),
             L.ptr(dbias), B, H, W, C, L.stream())


def nchw_to_nhwc(a, b=None):
    B, C, H, W = a.shape
    out = empty((B, H, W, C * (2 if b is not None else 1)), a)
    L.launch(_lib().scsfm_nchw_to_nhwc, "scsfm_nchw_to_nhwc", "layout", 1, 8.0 * out.numel(), L.ptr(a), L.ptr(b), B, C, H, W, L.ptr(out), L.stream())
    return out


def nchw_to_nhwc_pad(a, b, Cpad, operand=OPERAND_TF32):
    B, C, H, W = a.shape
    out = empty((B, H, W, Cpad), a)
    L.launch(_lib().scsfm_nchw_to_nhwc_pad, "scsfm_nchw_to_nhwc_pad", "layout", 1, 8.0 * out.numel(), L.ptr(a), L.ptr(b), B, C, H, W, Cpad,
             L.ptr(out), operand, L.stream())
    return out


def pad_channels(w, Cpad, operand=OPERAND_TF32):
    """[..., C] -> [..., Cpad] zero padded, as operand kind `operand` (stem weights)."""
    C = w.shape[-1]
    out = empty(tuple(w.shape[:-1]) + (Cpad,), w)
    L.launch(_lib().scsfm_pad_channels, "scsfm_pad_channels", "weight_round", 1, 8.0 * out.numel(), L.ptr(w), w.numel() // C, C, Cpad,
             L.ptr(out), operand, L.stream())
    return out


def unpad_add_(dst, src):
    """dst[..., c] += src[..., c] for c < C."""
    C, Cpad = dst.shape[-1], src.shape[-1]
    L.launch(_lib().scsfm_unpad_add, "scsfm_unpad_add", "weight_round", 1, 12.0 * dst.numel(), L.ptr(src), dst.numel() // C, C, Cpad,
             L.ptr(dst), L.stream())


def nhwc_to_nchw(x):
    B, H, W, C = x.shape
    out = empty((B, C, H, W), x)
    L.launch(_lib().scsfm_nhwc_to_nchw, "scsfm_nhwc_to_nchw", "layout", 1, 8.0 * out.numel(), L.ptr(x), B, C, H, W, L.ptr(out), L.stream())
    return out


def stem_dgrad(dy, w, H, W, need):
    """Gradient of the input images of a 7x7 stride-2 pad-3 stem: dy [N,Ho,Wo,64] (pre-BatchNorm gradient), w [64,7,7,Cin] the fp32
    stem weights (Cin 3: one image, 6: two images concatenated on channels), `need` one flag per image.  Returns one NCHW
    [N,3,H,W] tensor per image (None where not needed)."""
    N, Cin = dy.shape[0], w.shape[-1]
    outs = [empty((N, 3, H, W), dy) if n else None for n in need]
    outs += [None] * (2 - len(outs))
    L.launch(_lib().scsfm_stem_dgrad, "scsfm_stem_dgrad", "stem_dgrad", 1, 2.0 * N * H * W * Cin * 64 * 49 / 4, L.ptr(dy), L.ptr(w),
             N, H, W, Cin, L.ptr(outs[0]), L.ptr(outs[1]), L.stream())
    return outs[:len(need)]


def bn_prepare(sums, groups, count, gamma, beta, rmean, rvar, momentum, eps, training):
    C = gamma.numel()
    saved = empty((groups, C, 4), gamma)
    L.launch(_lib().scsfm_bn_prepare, "scsfm_bn_prepare", "bn_prepare", 1, 0.0, L.ptr(sums), groups, C, count, L.ptr(gamma), L.ptr(beta), L.ptr(rmean), L.ptr(rvar),
                                    momentum, eps, 1 if training else 0, L.ptr(saved), L.stream())
    return saved


def bn_apply(y, sums, gamma, beta, rmean, rvar, momentum, eps, residual, flags, groups=1, with_lo=False):
    """z = relu?(bn(y) + residual); statistics from the fused sums (training) or the running stats (sums=None).
    Returns (z, saved) with saved[g][c] = {scale, shift, mean, invstd} for the backward.  with_lo: also produce lo(z), the
    low part the split-accumulate convolutions read (attached to z like lo_of() would)."""
    z = torch.empty_like(y)
    z_lo = torch.empty_like(y) if with_lo else None
    C = y.shape[-1]
    saved = empty((groups, C, 4), y)
    rows = y.numel() // C
    L.launch(_lib().scsfm_bn_apply, "scsfm_bn_apply", "bn_apply", 1, (12.0 if residual is not None else 8.0) * y.numel(), L.ptr(y), L.ptr(sums),
             L.ptr(gamma), L.ptr(beta), L.ptr(rmean), L.ptr(rvar), momentum, eps, L.ptr(saved), L.ptr(residual), L.ptr(z), L.ptr(z_lo), rows, C,
             groups, int(flags), L.stream())
    if with_lo:
        z._scsfm_lo = z_lo
    return z, saved


class BnEvalTable:
    """Device job table of scsfm_bn_eval_prepare_batched for a list of BatchNorm layers (objects with weight, bias,
    running_mean, running_var), and the [Cout] scale / shift arrays it fills: coeffs[i] = (scale, shift) of layer i.  The
    table bakes in every buffer address; `key` lists them so that a caller can tell when it is stale."""

    def __init__(self, bns, eps):
        import struct
        dev = bns[0].weight.device
        total = sum(2 * aligned64(bn.weight.numel()) for bn in bns)
        self.buf = torch.empty(total, device=dev, dtype=torch.float32)
        eps_bits = struct.unpack("<i", struct.pack("<f", eps))[0]
        rows, self.coeffs, off = [], [], 0
        for bn in bns:
            C = bn.weight.numel()
            sc, sh = self.buf[off:off + C], self.buf[off + aligned64(C):off + aligned64(C) + C]
            off += 2 * aligned64(C)
            self.coeffs.append((sc, sh))
            rows.append([bn.weight.data_ptr(), bn.bias.data_ptr(), bn.running_mean.data_ptr(), bn.running_var.data_ptr(),
                         sc.data_ptr(), sh.data_ptr(), C, eps_bits])
        self.key = BnEvalTable.key_of(bns)
        self.table = torch.tensor(rows, dtype=torch.int64).to(dev)
        self.n, self.bytes = len(rows), 24.0 * sum(bn.weight.numel() for bn in bns)

    @staticmethod
    def key_of(bns):
        return tuple((bn.weight.data_ptr(), bn.bias.data_ptr(), bn.running_mean.data_ptr(), bn.running_var.data_ptr()) for bn in bns)

    def prepare(self):
        """(Re)compute every layer's scale / shift from the current parameters and running statistics: one launch."""
        L.launch(_lib().scsfm_bn_eval_prepare_batched, "scsfm_bn_eval_prepare_batched", "bn_prepare", 1, self.bytes,
                 L.ptr(self.table), self.n, L.stream())


def bn_backward(dz, z, y, saved, dgamma, dbeta, relu, want_dres, groups=1, with_lo=False):
    """Returns (dy, dres).  dres (= dz gated by the ReLU) is written in place over dz when requested.  with_lo: also
    produce lo(dy) (attached to dy like lo_of() would).  relu | BN_FROZEN: frozen statistics (eval mode), one pass; dgamma and
    dbeta may then be None (no parameter gradient, no sums)."""
    C = y.shape[-1]
    rows = y.numel() // C
    dy = torch.empty_like(y)
    dy_lo = torch.empty_like(y) if with_lo else None
    work = torch.empty(groups * C * 2, device=y.device, dtype=torch.float64)
    dres = dz if want_dres else None
    frozen = int(relu) & BN_FROZEN
    L.launch(_lib().scsfm_bn_backward, "scsfm_bn_backward", "bn_bwd", 2 if frozen else 4, (20.0 if frozen else 28.0) * y.numel(), L.ptr(dz), L.ptr(z), L.ptr(y), L.ptr(saved), None, L.ptr(dy),
             L.ptr(dy_lo), L.ptr(dres), L.ptr(dgamma), L.ptr(dbeta), rows, C, groups, int(relu), L.ptr(work), L.stream())
    if with_lo:
        dy._scsfm_lo = dy_lo
    return dy, dres


def maxpool_fwd(x):
    B, H, W, C = x.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    y = empty((B, Ho, Wo, C), x)
    idx = torch.empty((B, Ho, Wo, C), device=x.device, dtype=torch.uint8)
    L.launch(_lib().scsfm_maxpool_fwd, "scsfm_maxpool_fwd", "pool", 1, 4.0 * x.numel(), L.ptr(x), B, H, W, C, L.ptr(y), L.ptr(idx), L.stream())
    return y, idx


def maxpool_bwd(dy, idx, x_shape, dx, accumulate):
    B, H, W, C = x_shape
    L.launch(_lib().scsfm_maxpool_bwd, "scsfm_maxpool_bwd", "pool", 1, 4.0 * dx.numel(), L.ptr(dy), L.ptr(idx), B, H, W, C, L.ptr(dx), 1 if accumulate else 0, L.stream())


def upcat_fwd(lo, skip):
    B, h, w, C1 = lo.shape
    C2 = skip.shape[-1] if skip is not None else 0
    out = empty((B, 2 * h, 2 * w, C1 + C2), lo)
    L.launch(_lib().scsfm_upcat_fwd, "scsfm_upcat_fwd", "upcat", 1, 8.0 * out.numel(), L.ptr(lo), L.ptr(skip), B, 2 * h, 2 * w, C1, C2, L.ptr(out), L.stream())
    return out


def fold_plain(dpad, d, act_out, act, accumulate):
    B, Hp, Wp, C = dpad.shape
    L.launch(_lib().scsfm_fold_bwd, "scsfm_fold_bwd", "fold", 1, 8.0 * d.numel(), L.ptr(dpad), B, Hp - 2, Wp - 2, C, 0, 0, L.ptr(d),
             L.ptr(act_out), act, 1 if accumulate else 0, None, L.stream())


def fold_upcat(dpad, C1, lo_act, act, with_skip=True):
    """Gradient of the upsampled part (d_lo) and, with_skip, of the skip part (d_skip; None without) of a concatenation."""
    B, Hp, Wp, Ct = dpad.shape
    H, W, C2 = Hp - 2, Wp - 2, Ct - C1
    d_lo = empty((B, H // 2, W // 2, C1), dpad)
    d_skip = empty((B, H, W, C2), dpad) if C2 > 0 and with_skip else None
    L.launch(_lib().scsfm_fold_bwd, "scsfm_fold_bwd", "fold", 2 if d_skip is not None else 1, 4.0 * dpad.numel(), L.ptr(dpad), B, H, W, C1,
             C2, 1, L.ptr(d_lo), L.ptr(lo_act), act, 0, L.ptr(d_skip), L.stream())
    return d_lo, d_skip


def act_bwd_(d, out, act):
    L.launch(_lib().scsfm_act_bwd, "scsfm_act_bwd", "elementwise", 1, 12.0 * d.numel(), L.ptr(d), L.ptr(out), d.numel(), act, L.stream())
    return d


def spatial_mean_fwd(x, scale):
    B, H, W, C = x.shape
    out = empty((B, C), x)
    L.launch(_lib().scsfm_spatial_mean_fwd, "scsfm_spatial_mean_fwd", "pose_head", 1, 4.0 * x.numel(), L.ptr(x), B, H * W, C, scale, L.ptr(out), L.stream())
    return out


def spatial_mean_bwd(dout, x_shape, scale):
    B, H, W, C = x_shape
    dx = empty(x_shape, dout)
    L.launch(_lib().scsfm_spatial_mean_bwd, "scsfm_spatial_mean_bwd", "pose_head", 1, 4.0 * dx.numel(), L.ptr(dout), B, H * W, C, scale, L.ptr(dx), L.stream())
    return dx


def adam_step(param, grad, exp_avg, exp_avg_sq, lr, beta1, beta2, eps, weight_decay, step, step_dev=None, mirror=None,
              mirror_operand=OPERAND_TF32):
    L.launch(_lib().scsfm_adam_step, "scsfm_adam_step", "adam", 1, (32.0 if mirror is not None else 28.0) * param.numel(), L.ptr(param),
             L.ptr(grad), L.ptr(exp_avg), L.ptr(exp_avg_sq), param.numel(), lr, beta1, beta2, eps, weight_decay, step, L.ptr(step_dev),
             L.ptr(mirror), mirror_operand, L.stream())


def adam_step_masked(param, grad, exp_avg, exp_avg_sq, chunk_mask, lr, beta1, beta2, eps, weight_decay, step, step_dev=None,
                     mirror=None, mirror_operand=OPERAND_TF32):
    """adam_step over the chunks of 64 floats whose chunk_mask byte (uint8 [ceil(n / 64)], see chunk_mask()) is nonzero; the
    others -- frozen parameters -- are not touched at all."""
    if chunk_mask.dtype != torch.uint8 or chunk_mask.numel() != (param.numel() + 63) // 64:
        raise ValueError("adam_step_masked: chunk_mask must be uint8 with ceil(n / 64) = %d entries" % ((param.numel() + 63) // 64))
    L.launch(_lib().scsfm_adam_step_masked, "scsfm_adam_step_masked", "adam", 1, (32.0 if mirror is not None else 28.0) * param.numel(),
             L.ptr(param), L.ptr(grad), L.ptr(exp_avg), L.ptr(exp_avg_sq), param.numel(), L.ptr(chunk_mask), lr, beta1, beta2, eps,
             weight_decay, step, L.ptr(step_dev), L.ptr(mirror), mirror_operand, L.stream())


def chunk_mask(sizes, trainable, device):
    """uint8 mask of adam_step_masked for an arena that packs tensors of `sizes` elements at aligned64 offsets: 1 on the chunks of
    the tensors flagged in `trainable`."""
    mask = torch.zeros(sum(aligned64(n) for n in sizes) // 64, dtype=torch.uint8)
    off = 0
    for n, t in zip(sizes, trainable):
        if t:
            mask[off // 64:(off + aligned64(n)) // 64] = 1
        off += aligned64(n)
    return mask.to(device)
