"""Every convolution call the training step and the fused eval forward make, replayed on seeded synthetic operands and
compared ELEMENT BY ELEMENT with the same operation in fp64.

The calls are recorded, not listed: ConvCtx.conv_fwd / conv_dgrad / conv_wgrad are wrapped at class level while one eager
Trainer.step runs at the benchmarked configuration (256x832, two references, auto-mask on; ResNet-18 at batch 4 in fp32,
tf32 and tf32x3, ResNet-50 at batch 2 in tf32x3) and while each network runs one fused eval forward.  So the replays reach
the dispatch decisions that depend on the real layer sizes and on the SM count: the reflection forward on the TMA kernel
plus the border-ring pass, the tile heuristics, the pixel-split counts of the weight gradients, s2_prefers_gather.

Each distinct call runs on three operand variants (dense randn, ReLU'd with about half exact zeros, per-channel scales
from 2^-8 to 2^8), with the tune word training used and, on the dense operands, with forced kernel choices, so that every
convolution kernel instantiation of the library is launched (CONV_KERNELS, checked by test_every_conv_kernel_launched and
pinned to the built library by test_conv_kernel_list_cpu.py).  Per output element i, with A_i the same operation on |x|
and |w| (weight gradient: |x| and |dout|), the textbook forward-error bound of a dot product:

    |got_i - ref_i| <= TAU * A_i + 2^-23 * |ref_i|

TAU is one value for fp32, tf32 (on TF32 operands, whose products are exact in fp32) and tf32x3.  A k-slice of 8 channels
of one tap dropped from the reduction moves an element by about sqrt(8) / K of A_i: 6e-4 at K = 4608, 1.5e-4 at the
ResNet-50 decoder's K = 18432, so TAU = 2e-5 sees it.  Errors spread thinly over a long reduction (a pixel tile missing
from a weight gradient over 2.5 M pixels moves its norm by ~7e-3) are caught by the relative L2 bound instead: 1e-5 in
fp32 and tf32x3.  Plain tf32 runs a whole K loop (or a whole pixel split of a weight gradient) as one wgmma accumulator
chain, and the tensor core adds into its accumulator with truncation (conv_tma.cu, TmaGeom::cpg): a bias that grows with
the chain, ~1e-5 relative L2 at K = 4608 and ~1e-4 over the 640 k-pixel stem weight gradients, so tf32 has its own,
measured, relative L2 bounds (REL_L2).  Besides: no element is left
unwritten (every buffer nnops.empty hands out during a replay is NaN-filled), the forward and the data gradient are
bitwise repeatable and each image's output depends on that image alone, and every epilogue (bias, activation, addend,
BatchNorm sums, fused eval BatchNorm, the low part of the output, TF32 rounding, accumulation into dw) matches.  Needs a GPU.
"""
import ast
import collections
import inspect
import math
import os
import re
import time

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Worst ratios measured on an H100 (80 GB HBM3, 700 W) over all replays: fp32 1.2e-6, tf32 3.4e-6, tf32x3 1.3e-6.
TAU = 2e-5              # elementwise bound, in units of A_i (see the module docstring)
REL_L2 = {"fp32": dict(fwd=1e-5, dgrad=1e-5, wgrad=1e-5), "tf32x3": dict(fwd=1e-5, dgrad=1e-5, wgrad=1e-5),
          "tf32": dict(fwd=5e-5, dgrad=5e-5, wgrad=5e-4)}       # relative L2 bounds (see the module docstring)
ULP = 2.0 ** -23

# Every convolution kernel instantiation of libscsfm.so (demangled, up to the argument list).
CONV_KERNELS = sorted(
    ["scsfm::conv_tma_kernel<%d, %d>" % (bn, mt) for bn, mt in ((16, 1), (32, 1), (64, 1), (128, 1), (16, 2), (32, 2), (64, 2))] +
    ["scsfm::conv_fwd_tc_kernel<%d, %s>" % a for a in ((16, "false"), (32, "false"), (64, "false"), (128, "false"),
                                                        (32, "true"), (64, "true"), (128, "true"))] +
    ["scsfm::conv_wgrad_tc_kernel<%d, %s>" % a for a in ((16, "false"), (32, "false"), (64, "false"), (128, "false"),
                                                          (32, "true"), (64, "true"), (128, "true"))] +
    ["scsfm::conv_wgrad_tma_kernel<%d, %s, %d, %d>" % (bn, sp, kw, s) for bn in (32, 64) for sp in ("false", "true")
     for kw, s in ((1, 1), (1, 2), (3, 1), (3, 2), (7, 2))] +
    ["scsfm::conv_stem_fwd_kernel<%d, %s>" % (c, sp) for c in (4, 8) for sp in ("false", "true")] +
    ["scsfm::conv_wgrad_thin_kernel<16, 16, 32, 2>", "scsfm::conv_wgrad_thin_kernel<32, 16, 16, 1>"] +
    ["scsfm::conv_%s_simt_kernel<%d, %d>" % (p, a, b) for p in ("fwd", "dgrad") for a, b in ((256, 16), (128, 32), (64, 64))] +
    ["scsfm::conv_wgrad_simt_kernel<%d, %d>" % ab for ab in ((16, 256), (32, 128), (64, 64))])
CONV_FAMILY = re.compile(r"^scsfm::conv_\w*kernel<")


def kernel_key(name):
    """Demangled kernel name -> its name up to the argument list, in the GNU c++filt spelling (cu++filt's "(int)16" and
    "(bool)1" become "16" and "true")."""
    name = re.sub(r"\(bool\)0", "false", re.sub(r"\(bool\)1", "true", name.replace("(int)", "")))
    name = name.split("(")[0].strip()
    return name[5:] if name.startswith("void ") else name


# ---------------------------------------------------------------------------------------------------------------------
# recording
# ---------------------------------------------------------------------------------------------------------------------
# One convolution call, by its arguments.  x: shape of the operand reduced over (forward, weight gradient: the input;
# data gradient: dout); w: weight shape [Cout,kh,kw,Cin] (weight gradient: dw); out: data gradient: x_shape, weight
# gradient: dout shape.  bias: a bias (weight gradient: dbias); bn_groups: BatchNorm sums over that many groups (0: none);
# bn_eval: the fused eval-mode BatchNorm; zero_ch: input channels that are identically zero (the channel-padded stems).
Call = collections.namedtuple("Call", "kind mode tune x w out stride pad pad_mode act bias addend bn_groups bn_eval with_lo "
                                      "padded zero_ch")
CONFIGS = [("r18-fp32", 18, "fp32", 4), ("r18-tf32", 18, "tf32", 4), ("r18-tf32x3", 18, "tf32x3", 4), ("r50-tf32x3", 50, "tf32x3", 2)]


def _zero_channels(x):
    return tuple((x.abs().amax((0, 1, 2)) == 0).nonzero().flatten().tolist())


def _describe(name, cx, a):
    base = dict(mode=cx.mode, tune=int(cx.tune), out=None, pad_mode=0, act=0, bias=False, addend=False, bn_groups=0,
                bn_eval=False, with_lo=False, padded=False, zero_ch=())
    if name == "conv_fwd":
        x, w = a["x"], a["w"]
        return Call(kind="fwd", x=tuple(x.shape), w=tuple(w.shape), stride=a["stride"], pad=a["pad"], **dict(
            base, pad_mode=a["pad_mode"], act=int(a["act"]), bias=a["bias"] is not None, addend=a["addend"] is not None,
            bn_groups=a["bn_groups"] if a["bn_sums"] is not None else 0, bn_eval=a["bn_scale"] is not None,
            with_lo=bool(a["with_lo"]), zero_ch=_zero_channels(x) if w.shape[1] == 7 else ()))
    if name == "conv_dgrad":
        assert a["w_src"] is None, "the replay builds both flipped parts from w"
        return Call(kind="dgrad", x=tuple(a["dout"].shape), w=tuple(a["w"].shape), stride=a["stride"], pad=a["pad"], **dict(
            base, out=tuple(a["x_shape"]), addend=a["addend"] is not None, padded=bool(a["padded_input"])))
    x, dw = a["x"], a["dw"]
    return Call(kind="wgrad", x=tuple(x.shape), w=tuple(dw.shape), stride=a["stride"], pad=a["pad"], **dict(
        base, out=tuple(a["dout"].shape), pad_mode=a["pad_mode"], bias=a["dbias"] is not None,
        zero_ch=_zero_channels(x) if dw.shape[1] == 7 else ()))


class _Recording:
    """Wraps the three ConvCtx entry points at class level for the duration of a with-block; restores them afterwards."""
    NAMES = ("conv_fwd", "conv_dgrad", "conv_wgrad")

    def __init__(self, calls):
        from scsfm import nnops as O
        self.O, self.calls = O, calls
        self.orig = {n: getattr(O.ConvCtx, n) for n in self.NAMES}

    def __enter__(self):
        for n, f in self.orig.items():
            setattr(self.O.ConvCtx, n, self._wrap(n, f))
        return self

    def _wrap(self, name, f):
        sig = inspect.signature(f)

        def recorded(cx, *args, **kw):
            a = sig.bind(cx, *args, **kw)
            a.apply_defaults()
            self.calls.append(_describe(name, cx, a.arguments))
            return f(cx, *args, **kw)
        return recorded

    def __exit__(self, *exc):
        for n, f in self.orig.items():
            setattr(self.O.ConvCtx, n, f)


@pytest.fixture(scope="module")
def recorded():
    """config -> the distinct convolution calls of one eager training step and one fused eval forward of each network,
    in the order they were first made."""
    import models
    from scsfm import synth
    from scsfm.trainer import Trainer
    runs = {}
    for cfg, layers, mode, batch in CONFIGS:
        tgt, refs, K = synth.triplet(1234, batch, 256, 832, 2, "kitti")
        tgt, refs, K = tgt.to(DEV), [r.to(DEV) for r in refs], K.to(DEV)
        torch.manual_seed(0)
        disp, pose = models.DispResNet(layers, False).to(DEV).train(), models.PoseResNet(layers, False).to(DEV).train()
        calls = []
        with _Recording(calls):
            tr = Trainer(disp, pose, lr=1e-4, with_auto_mask=1, distributed=False, conv_mode=mode)
            losses = [float(v) for v in tr.step(tgt, refs, K)]
            assert all(math.isfinite(v) for v in losses), (cfg, losses)
            disp.eval()
            pose.eval()
            with torch.no_grad():
                disp(tgt)
                pose(tgt, refs[0])
            torch.cuda.synchronize()
        runs[cfg] = list(dict.fromkeys(calls))
        del tr, disp, pose, tgt, refs, K
        torch.cuda.empty_cache()
    return runs


def _conv_layers_table():
    """LAYERS of tools/conv_layers.py, parsed (importing the tool would flip torch's global TF32 switches)."""
    tree = ast.parse(open(os.path.join(ROOT, "tools", "conv_layers.py")).read())
    for node in tree.body:
        if isinstance(node, ast.Assign) and any(getattr(t, "id", None) == "LAYERS" for t in node.targets):
            return ast.literal_eval(node.value)
    raise AssertionError("LAYERS not found in tools/conv_layers.py")


def test_recorded_calls_cover_conv_layers_table(recorded):
    """Every ResNet-18 layer of the per-layer tool's table is among the recorded forward calls at the batch it lists, and
    each recorded step made all three passes."""
    from scsfm import nnops as O
    fwd = {(c.x, c.w[0], c.w[1], c.stride, c.pad, c.pad_mode) for calls in recorded.values() for c in calls if c.kind == "fwd"}
    rows = [r for r in _conv_layers_table() if not r[0].startswith(("r50", "odd"))]
    assert len(rows) == 24
    missing = [r[0] for r in rows
               if ((r[1], r[2], r[3], r[4]), r[5], r[6], r[7], r[8], O.PAD_REFLECT if r[9] else O.PAD_ZERO) not in fwd]
    assert not missing, missing
    for cfg, calls in recorded.items():
        kinds = collections.Counter(c.kind for c in calls)
        assert all(kinds[k] > 0 for k in ("fwd", "dgrad", "wgrad")), (cfg, kinds)
        assert any(c.bn_eval for c in calls) and any(c.bn_groups for c in calls), cfg
        print("%s: %d distinct calls (%s)" % (cfg, len(calls), dict(kinds)))


# ---------------------------------------------------------------------------------------------------------------------
# replay
# ---------------------------------------------------------------------------------------------------------------------
VARIANTS = ("dense", "relu", "scaled")


def _ways(c):
    """(label, ScsfmConv.tune word): the tune word training used (recorded with the call), then, for the dense operands,
    forced kernel choices -- together they launch every instantiation in CONV_KERNELS."""
    from scsfm import nnops as O
    ways = [("auto" if c.tune == 0 else "recorded tune 0x%x" % c.tune, c.tune)]
    thin = c.kind == "wgrad" and c.w[0] == 16 and c.w[1] == 3 and c.stride == 1 and c.pad == 1 and c.w[3] in (16, 32)
    if c.mode == "fp32":
        forced = [("gather", dict(wgrad=1))] if thin else []
    elif c.kind == "wgrad":
        forced = [("gather", dict(wgrad=1)), ("tma bn32", dict(wgrad=2, bn=32)), ("tma bn64", dict(wgrad=2, bn=64))] + \
            ([("thin", dict(wgrad=3))] if thin else [])
    else:
        forced = [("gather", dict(no_tma=1)), ("tma 128px tw8", dict(mt=1, tw_log2=3)), ("tma 256px tw16", dict(mt=2, tw_log2=4))]
    return ways + [(label, O.tune(**knobs)) for label, knobs in forced]


class _NanEmpty:
    """nnops.empty hands out NaN-filled buffers: an element a kernel does not write stays NaN."""

    def __enter__(self):
        from scsfm import nnops as O
        self.O, self.orig = O, O.empty
        O.empty = lambda shape, like: torch.full(shape, float("nan"), device=like.device, dtype=torch.float32)

    def __exit__(self, *exc):
        self.O.empty = self.orig


def _nchw(t):
    return t.double().permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


class _Operands:
    """Seeded synthetic operands of call c, generated on the GPU and rounded / split as their producers would."""

    def __init__(self, c, variant, seed):
        from scsfm import nnops as O
        self.c, self.variant = c, variant
        self.g = torch.Generator(device=DEV).manual_seed(seed)
        self.scales = None
        Cout, kh, kw, Cin = c.w
        main = c.x                                           # the operand the variant shapes (reduced over its channels)
        self.a = self.activation(main)
        if c.kind == "wgrad":
            self.b = self.randn(c.out)                       # dout
            if c.mode == "tf32":
                O.round_tf32(self.b, self.b)
            self.w = None
        else:
            self.w = self.randn(c.w) / math.sqrt(kh * kw * Cin)
            if c.zero_ch:
                self.w[..., list(c.zero_ch)] = 0
            if c.mode == "tf32":
                O.round_tf32(self.w, self.w)
        self.w_lo = O.split_tf32(self.w) if (self.w is not None and c.mode == "tf32x3") else None
        self.bias = 0.1 * self.randn((Cout,)) if c.bias else None
        if c.kind == "fwd":
            Ho, Wo = self.out_hw()
            self.addend = self.randn((c.x[0], Ho, Wo, Cout)) if c.addend else None
            self.bn_scale = (1 + 0.3 * self.randn((Cout,))) if c.bn_eval else None
            self.bn_shift = 0.2 * self.randn((Cout,)) if c.bn_eval else None
        elif c.kind == "dgrad":
            self.addend = self.randn(c.out) if c.addend else None

    def randn(self, shape):
        return torch.randn(tuple(shape), generator=self.g, device=DEV)

    def activation(self, shape):
        from scsfm import nnops as O
        a = self.randn(shape)
        if self.variant == "relu":
            a = torch.relu_(a)
        elif self.variant == "scaled":
            if self.scales is None:
                self.scales = torch.exp2(16 * torch.rand(shape[-1], generator=self.g, device=DEV) - 8)
            a = a * self.scales
        if self.c.zero_ch:
            a[..., list(self.c.zero_ch)] = 0
        if self.c.mode == "tf32":
            O.round_tf32(a, a)
        return a

    def out_hw(self):
        c = self.c
        return ((c.x[1] + 2 * c.pad - c.w[1]) // c.stride + 1, (c.x[2] + 2 * c.pad - c.w[2]) // c.stride + 1)


def _reference(c, op):
    """(ref, A) in fp64, NHWC / [Cout,kh,kw,Cin]: the operation without epilogue on the operands, and on their magnitudes."""
    Cout, kh, kw, Cin = c.w
    if c.kind == "fwd" or c.kind == "wgrad":
        x = _nchw(op.a)
        pad = c.pad
        if c.pad_mode == 1:
            x, pad = F.pad(x, (c.pad,) * 4, mode="reflect"), 0
    if c.kind == "fwd":
        w = _nchw(op.w)
        return _nhwc(F.conv2d(x, w, None, c.stride, pad)), _nhwc(F.conv2d(x.abs(), w.abs(), None, c.stride, pad))
    if c.kind == "dgrad":
        B, H, W, C = c.out
        size, pad = ((B, C, H + 2, W + 2), 0) if c.padded else ((B, C, H, W), c.pad)
        w, d = _nchw(op.w), _nchw(op.a)
        gi = torch.nn.grad.conv2d_input
        return _nhwc(gi(size, w, d, c.stride, pad)), _nhwc(gi(size, w.abs(), d.abs(), c.stride, pad))
    d = _nchw(op.b)
    gw = torch.nn.grad.conv2d_weight
    return (_nhwc(gw(x, (Cout, Cin, kh, kw), d, c.stride, pad)), _nhwc(gw(x.abs(), (Cout, Cin, kh, kw), d.abs(), c.stride, pad)))


def _act64(v, act):
    from scsfm import nnops as O
    act &= 0xff
    if act == O.ACT_RELU:
        return torch.relu(v)
    if act == O.ACT_ELU:
        return F.elu(v)
    assert act == O.ACT_NONE, act
    return v


class _Check:
    """Worst ratio of one comparison: max_i (|got_i - ref_i| - slack_i)+ / A_i, must be <= TAU; plus relative L2 <= rel."""

    def __init__(self, rel):
        self.rel = rel
        self.items = []          # (what, ratio, rel_l2 or None, nan count)

    def elementwise(self, what, got, ref, A, slack, l2=True, delta=None, base=None):
        """l2: also bound the relative L2 error, ||got - ref|| / ||ref||, or ||delta|| / ||base|| where given (an
        accumulating output: the error of the increment relative to the increment)."""
        g = got.double()
        nan = int(torch.isnan(got).sum())
        err = ((g - ref).abs() - slack).clamp_min(0)
        ratio = float((err / A.clamp_min(1e-300)).max()) if nan == 0 else float("inf")
        rl2 = None
        if l2:
            dd, bb = (g - ref, ref) if delta is None else (delta, base)
            rl2 = float(dd.norm() / (bb.norm() + 1e-300)) if nan == 0 else float("inf")
        self.items.append((what, ratio, rl2, nan))

    def fact(self, what, ok):
        self.items.append((what, 0.0 if ok else float("inf"), None, 0))

    def failures(self):
        return [it for it in self.items if not (it[1] <= TAU and (it[2] is None or it[2] <= self.rel))]


def _run_fwd(c, op, tune, x=None, act=None, sums=True):
    from scsfm import nnops as O
    cx = O.ConvCtx(c.mode)
    cx.tune = tune
    x = op.a if x is None else x
    Cout = c.w[0]
    s = torch.zeros(O.BN_SLOTS, c.bn_groups, Cout, 2, dtype=torch.float64, device=DEV) if (c.bn_groups and sums) else None
    with _NanEmpty():
        y = cx.conv_fwd(x, op.w, op.bias, c.stride, c.pad, c.pad_mode, c.act if act is None else act, s, max(c.bn_groups, 1),
                        op.w_lo, bn_scale=op.bn_scale, bn_shift=op.bn_shift, addend=op.addend, with_lo=c.with_lo)
    return y, s


def _check_fwd(c, op, ref, A, tune, chk):
    from scsfm import nnops as O
    pre, Aw = ref, A
    if op.bias is not None:
        pre, Aw = pre + op.bias.double(), Aw + op.bias.double().abs()
    add = op.addend.double() if op.addend is not None else 0.0
    if c.bn_eval:
        sc, sh = op.bn_scale.double(), op.bn_shift.double()
        lin = sc * pre + sh + add
        bound_A = sc.abs() * Aw
        slack = 2 * ULP * ((sc * pre).abs() + sh.abs() + (add.abs() if torch.is_tensor(add) else 0.0))
    else:
        lin = pre + add
        bound_A = Aw
        slack = ULP * lin.abs()
    want = _act64(lin, c.act)
    slack = slack + ULP * want.abs()
    y, sums = _run_fwd(c, op, tune)
    y2, _ = _run_fwd(c, op, tune, sums=False)
    chk.fact("repeatable", _bits(y, y2))
    if c.with_lo:
        chk.fact("out_lo written", not bool(torch.isnan(y._scsfm_lo).any()))
        chk.fact("out_lo == split_tf32(out)", _bits(y._scsfm_lo, O.split_tf32(y)) and _bits(y._scsfm_lo, y2._scsfm_lo))
    if c.act & O.ROUND_TF32:
        plain, _ = _run_fwd(c, op, tune, act=c.act & ~O.ROUND_TF32, sums=False)
        r = torch.empty_like(plain)
        O.round_tf32(plain, r)
        chk.fact("ROUND_TF32 == round_tf32(unrounded)", _bits(y, r))
        chk.elementwise("out", plain, want, bound_A, slack)
    else:
        chk.elementwise("out", y, want, bound_A, slack)
    if sums is not None:
        G, C = c.bn_groups, c.w[0]
        s = sums.sum(0)
        yd = y.double().reshape(G, -1, C)
        chk.elementwise("bn sum", s[..., 0], yd.sum(1), yd.abs().sum(1), 0.0, l2=False)
        chk.elementwise("bn sum sq", s[..., 1], (yd * yd).sum(1), (yd * yd).sum(1), 0.0, l2=False)
    if c.x[0] > 1:
        x2 = op.a.clone()
        x2[0] = op.activation((1,) + tuple(c.x[1:]))[0]
        y3, _ = _run_fwd(c, op, tune, x=x2, sums=False)
        chk.fact("images independent", _bits(y3[1:], y[1:]))


def _run_dgrad(c, op, tune, dout=None):
    from scsfm import nnops as O
    cx = O.ConvCtx(c.mode)
    cx.tune = tune
    with _NanEmpty():
        return cx.conv_dgrad(op.a if dout is None else dout, op.w, c.out, c.stride, c.pad, op.addend, padded_input=c.padded)


def _check_dgrad(c, op, ref, A, tune, chk):
    want, Aw = ref, A
    if op.addend is not None:
        want, Aw = want + op.addend.double(), Aw + op.addend.double().abs()
    din = _run_dgrad(c, op, tune)
    chk.fact("repeatable", _bits(din, _run_dgrad(c, op, tune)))
    chk.elementwise("din", din, want, Aw, ULP * want.abs())
    if c.x[0] > 1:
        d2 = op.a.clone()
        d2[0] = op.activation((1,) + tuple(c.x[1:]))[0]
        chk.fact("images independent", _bits(_run_dgrad(c, op, tune, d2)[1:], din[1:]))


def _check_wgrad(c, op, ref, A, tune, chk):
    from scsfm import nnops as O
    cx = O.ConvCtx(c.mode)
    cx.tune = tune
    # accumulation into a nonzero starting matrix of the gradient's own magnitude
    g = torch.Generator(device=DEV).manual_seed(99)
    dw0 = torch.randn(c.w, generator=g, device=DEV) * float(ref.pow(2).mean().sqrt())
    dw = dw0.clone()
    db0 = torch.randn(c.w[0], generator=g, device=DEV) if c.bias else None
    db = db0.clone() if c.bias else None
    with _NanEmpty():
        cx.conv_wgrad(op.a, op.b, dw, db, c.stride, c.pad, c.pad_mode)
        cx.join_wgrad()
    want = ref + dw0.double()
    chk.elementwise("dw", dw, want, A + dw0.double().abs(), ULP * want.abs(), delta=dw.double() - dw0.double() - ref,
                    base=ref)
    if c.bias:
        d = op.b.double().reshape(-1, c.w[0])
        wb = d.sum(0) + db0.double()
        chk.elementwise("dbias", db, wb, d.abs().sum(0) + db0.double().abs(), ULP * wb.abs(),
                        delta=db.double() - db0.double() - d.sum(0), base=d.sum(0))


CHECK = {"fwd": _check_fwd, "dgrad": _check_dgrad, "wgrad": _check_wgrad}


def _label(c):
    s = "%s B%d %dx%d C%d->%d k%d s%d p%d%s" % (c.kind, c.x[0], c.x[1], c.x[2], c.w[3], c.w[0], c.w[1], c.stride, c.pad,
                                            " refl" if c.pad_mode == 1 else "")
    flags = [n for n, v in (("bias", c.bias), ("addend", c.addend), ("bn_sums/%d" % c.bn_groups, c.bn_groups),
                            ("bn_eval", c.bn_eval), ("out_lo", c.with_lo), ("padded", c.padded)) if v]
    if c.act & 0xff:
        flags.append("act%d" % (c.act & 0xff))
    if c.act & 0x100:
        flags.append("round")
    return s + (" [" + ",".join(flags) + "]" if flags else "")


@pytest.fixture(scope="module")
def replays(recorded):
    """Replays every recorded call; returns {"results": {(config, pass): [(label, way, variant, check items)]}, "kernels":
    names of the convolution kernels launched, "worst": {(mode, pass): [worst elementwise ratio, worst relative L2]},
    "seconds": wall time}."""
    from torch.profiler import ProfilerActivity, profile
    t0 = time.time()
    results, kernels, worst = collections.defaultdict(list), set(), collections.defaultdict(lambda: [0.0, 0.0])
    for cfg, calls in recorded.items():
        t1 = time.time()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i, c in enumerate(calls):
                for vi, variant in enumerate(VARIANTS):
                    op = _Operands(c, variant, 1000 * i + vi)
                    ref, A = _reference(c, op)
                    for way, tune in (_ways(c) if variant == "dense" else _ways(c)[:1]):
                        chk = _Check(REL_L2[c.mode][c.kind])
                        try:
                            CHECK[c.kind](c, op, ref, A, tune, chk)
                        except Exception as e:          # noqa: BLE001 -- reported with the call that raised it
                            chk.items.append(("raised %r" % e, float("inf"), None, 0))
                        results[(cfg, c.kind)].append((_label(c), way, variant, chk))
                        for what, ratio, rl2, _ in chk.items:
                            if what in ("out", "din", "dw"):
                                w = worst[(c.mode, c.kind)]
                                w[0], w[1] = max(w[0], ratio), max(w[1], rl2)
                    del op, ref, A
            torch.cuda.synchronize()
        kernels |= {kernel_key(e.key) for e in prof.key_averages()}
        torch.cuda.empty_cache()
        print("%s: %d distinct calls replayed in %.1f s" % (cfg, len(calls), time.time() - t1), flush=True)
    return {"results": results, "kernels": kernels, "worst": dict(worst), "seconds": time.time() - t0}


@pytest.mark.parametrize("kind", ["fwd", "dgrad", "wgrad"])
@pytest.mark.parametrize("cfg", [c[0] for c in CONFIGS])
def test_conv_calls_vs_fp64(replays, cfg, kind):
    rows = replays["results"][(cfg, kind)]
    assert rows, (cfg, kind)
    bad = []
    for label, way, variant, chk in rows:
        for what, ratio, rl2, nan in chk.failures():
            bad.append("%s | %s | %s | %s: ratio %.3g (tau %g) rel-L2 %s (bound %g) NaN %d" % (
                label, way, variant, what, ratio, TAU, "-" if rl2 is None else "%.3g" % rl2, chk.rel, nan))
    main = [it for _, _, _, chk in rows for it in chk.items if it[0] in ("out", "din", "dw")]
    print("%s %s: %d replays, worst elementwise ratio %.3g (tau %g), worst relative L2 %.3g" % (
        cfg, kind, len(rows), max(it[1] for it in main), TAU, max(it[2] for it in main)))
    assert not bad, "\n".join(bad[:40]) + ("\n... %d more" % (len(bad) - 40) if len(bad) > 40 else "")


def test_every_conv_kernel_launched(replays):
    """The replays launched every convolution kernel instantiation of the library."""
    launched = {k for k in replays["kernels"] if CONV_FAMILY.match(k)}
    print("replays: %.0f s; worst elementwise ratio / relative L2 per (mode, pass): %s" % (
        replays["seconds"], ", ".join("%s %s %.3g / %.3g" % (m, p, r, l2) for (m, p), (r, l2) in sorted(replays["worst"].items()))))
    assert not launched - set(CONV_KERNELS), sorted(launched - set(CONV_KERNELS))
    assert not set(CONV_KERNELS) - launched, sorted(set(CONV_KERNELS) - launched)
