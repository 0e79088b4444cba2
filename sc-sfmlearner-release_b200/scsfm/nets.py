"""DispResNet / PoseResNet executed with libscsfm kernels (forward AND hand-scheduled backward).

Module tree and parameter names reproduce the reference's `state_dict` keys exactly (reference
models/DispResNet.py, models/PoseResNet.py, models/resnet_encoder.py + torchvision ResNet; SURVEY.md
section 2.2).  Differences from a stock nn.Module network:

  * all parameters of a network live in ONE flat fp32 arena (conv weights stored channels-last, i.e.
    physically [Cout,kh,kw,Cin], still exposed with the reference's logical [Cout,Cin,kh,kw] shape), and
    all gradients in a second arena: the data-parallel allreduce and Adam each touch one buffer;
  * a whole network call is ONE autograd node: forward runs the kernel sequence and records the
    activations, backward replays the hand-written gradient kernels and accumulates parameter
    gradients straight into the gradient arena (`p.grad` are persistent views of it);
  * activations are NHWC; BatchNorm statistics are fused into the producing conv's epilogue.

There is no CPU path: calling a network on CPU tensors raises.
"""
import math

import torch
import torch.nn as nn

from . import nnops as O

BN_EPS, BN_MOMENTUM = 1e-5, 0.1
STAGE_BLOCKS = {18: (2, 2, 2, 2), 34: (3, 4, 6, 3), 50: (3, 4, 6, 3), 101: (3, 4, 23, 3), 152: (3, 8, 36, 3)}


# ------------------------------------------------------------------------------------------------
# parameter holders (names = reference state_dict keys)
# ------------------------------------------------------------------------------------------------
class ConvParams(nn.Module):
    def __init__(self, cin, cout, k, bias, init):
        super().__init__()
        w = torch.empty(cout, cin, k, k)
        if init == "kaiming_fan_out":      # torchvision ResNet.__init__ / resnet_encoder.py:34-36
            nn.init.kaiming_normal_(w, mode="fan_out", nonlinearity="relu")
        else:                              # nn.Conv2d default (DispResNet.py:37, PoseResNet.py:26-29)
            nn.init.kaiming_uniform_(w, a=math.sqrt(5))
        self.weight = nn.Parameter(w.contiguous(memory_format=torch.channels_last))
        if bias:
            bound = 1.0 / math.sqrt(cin * k * k)
            self.bias = nn.Parameter(torch.empty(cout).uniform_(-bound, bound))
        else:
            self.bias = None
        self.k = k

    def w_khwc(self):
        """[Cout,kh,kw,Cin] contiguous view of the channels-last weight (no copy)."""
        return self.weight.permute(0, 2, 3, 1)

    def w_op(self, cx):
        """Weights as the conv kernels' operand: in tf32 mode the TF32-rounded mirror of the arena, otherwise the raw
        parameters (fp32: exact kernels; tf32x3: the tensor core reads their high part)."""
        tc = getattr(self, "_tc_view", None)
        return tc if (tc is not None and cx.mode == "tf32") else self.w_khwc()

    def w_lo(self, cx):
        """tf32x3 mode: the low part of the weights (the mirror arena holds it in that mode); None otherwise."""
        return self._tc_view if cx.split else None


class BNParams(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(c))
        self.bias = nn.Parameter(torch.zeros(c))
        self.register_buffer("running_mean", torch.zeros(c))
        self.register_buffer("running_var", torch.ones(c))
        self.register_buffer("num_batches_tracked", torch.tensor(0, dtype=torch.long))


class LinearParams(nn.Module):
    """The torchvision classifier head the reference never calls but keeps in its state_dict."""

    def __init__(self, cin, cout):
        super().__init__()
        bound = 1.0 / math.sqrt(cin)
        w = torch.empty(cout, cin)
        nn.init.kaiming_uniform_(w, a=math.sqrt(5))
        self.weight = nn.Parameter(w)
        self.bias = nn.Parameter(torch.empty(cout).uniform_(-bound, bound))


class Block(nn.Module):
    """BasicBlock (expansion 1) or Bottleneck (expansion 4, stride on the 3x3)."""

    def __init__(self, cin, width, stride, bottleneck):
        super().__init__()
        self.bottleneck, self.stride = bottleneck, stride
        cout = width * (4 if bottleneck else 1)
        if bottleneck:
            self.conv1, self.bn1 = ConvParams(cin, width, 1, False, "kaiming_fan_out"), BNParams(width)
            self.conv2, self.bn2 = ConvParams(width, width, 3, False, "kaiming_fan_out"), BNParams(width)
            self.conv3, self.bn3 = ConvParams(width, cout, 1, False, "kaiming_fan_out"), BNParams(cout)
        else:
            self.conv1, self.bn1 = ConvParams(cin, width, 3, False, "kaiming_fan_out"), BNParams(width)
            self.conv2, self.bn2 = ConvParams(width, width, 3, False, "kaiming_fan_out"), BNParams(width)
        self.downsample = None
        if stride != 1 or cin != cout:
            self.downsample = nn.Sequential(ConvParams(cin, cout, 1, False, "kaiming_fan_out"), BNParams(cout))
        self.cout = cout


class Trunk(nn.Module):
    def __init__(self, num_layers, in_ch):
        super().__init__()
        bott = num_layers >= 50
        self.conv1, self.bn1 = ConvParams(in_ch, 64, 7, False, "kaiming_fan_out"), BNParams(64)
        cin = 64
        for i, (n, width) in enumerate(zip(STAGE_BLOCKS[num_layers], (64, 128, 256, 512))):
            blocks = []
            for j in range(n):
                blk = Block(cin, width, 2 if (j == 0 and i > 0) else 1, bott)
                blocks.append(blk)
                cin = blk.cout
            setattr(self, "layer%d" % (i + 1), nn.Sequential(*blocks))
        self.fc = LinearParams(cin, 1000)


class ResnetEncoder(nn.Module):
    def __init__(self, num_layers, pretrained, num_input_images=1):
        super().__init__()
        if num_layers not in STAGE_BLOCKS:
            raise ValueError("{} is not a valid number of resnet layers".format(num_layers))
        self.num_ch_enc = [64, 64, 128, 256, 512] if num_layers <= 34 else [64, 256, 512, 1024, 2048]
        self.encoder = Trunk(num_layers, 3 * num_input_images)
        if pretrained:
            self.load_imagenet(num_layers, num_input_images)

    def load_imagenet(self, num_layers, num_input_images):
        """ImageNet initialisation (reference resnet_encoder.py:40-58,70-82) from a LOCAL torchvision checkpoint
        `resnet<num_layers>-*.pth` in $SCSFM_PRETRAINED_DIR or the torch hub cache -- there is no network to download it.
        For the multi-image pose encoder the stem is replicated as cat([w] * n, 1) / n (resnet_encoder.py:56-57)."""
        import glob
        import os
        dirs = [os.environ.get("SCSFM_PRETRAINED_DIR", ""), os.path.join(torch.hub.get_dir(), "checkpoints")]
        hits = [f for d in dirs if d for f in sorted(glob.glob(os.path.join(d, "resnet%d-*.pth" % num_layers)))]
        if not hits:
            raise FileNotFoundError("no local ImageNet checkpoint resnet%d-*.pth in %s (no network access: put the torchvision "
                                    "file there, or use pretrained=False / --with-pretrain 0)" % (num_layers, [d for d in dirs if d]))
        sd = torch.load(hits[0], map_location="cpu")
        if num_input_images > 1:
            sd["conv1.weight"] = torch.cat([sd["conv1.weight"]] * num_input_images, 1) / num_input_images
        own = self.encoder.state_dict()
        for k, v in sd.items():
            if k in own and own[k].shape == v.shape:
                own[k].copy_(v)


class _ReflConv(nn.Module):      # reference Conv3x3: keys  <name>.conv.{weight,bias}
    def __init__(self, cin, cout):
        super().__init__()
        self.conv = ConvParams(int(cin), int(cout), 3, True, "default")


class _ReflConvELU(nn.Module):   # reference ConvBlock: keys  <name>.conv.conv.{weight,bias}
    def __init__(self, cin, cout):
        super().__init__()
        self.conv = _ReflConv(cin, cout)


class DepthDecoder(nn.Module):
    def __init__(self, num_ch_enc):
        super().__init__()
        dec = [16, 32, 64, 128, 256]
        mods, self.idx = [], {}
        for i in range(4, -1, -1):
            cin = num_ch_enc[-1] if i == 4 else dec[i + 1]
            self.idx[("up", i, 0)] = len(mods)
            mods.append(_ReflConvELU(cin, dec[i]))
            cin = dec[i] + (num_ch_enc[i - 1] if i > 0 else 0)
            self.idx[("up", i, 1)] = len(mods)
            mods.append(_ReflConvELU(cin, dec[i]))
        for s in range(4):
            self.idx[("disp", s)] = len(mods)
            mods.append(_ReflConv(dec[s], 1))
        self.decoder = nn.ModuleList(mods)

    def up(self, i, j):
        return self.decoder[self.idx[("up", i, j)]].conv.conv

    def disp(self, s):
        return self.decoder[self.idx[("disp", s)]].conv


class PoseDecoder(nn.Module):
    def __init__(self, num_ch_enc):
        super().__init__()
        self.net = nn.ModuleList([ConvParams(num_ch_enc[-1], 256, 1, True, "default"),
                                  ConvParams(256, 256, 3, True, "default"), ConvParams(256, 256, 3, True, "default"),
                                  ConvParams(256, 6, 1, True, "default")])


# ------------------------------------------------------------------------------------------------
# flat parameter / gradient arenas
# ------------------------------------------------------------------------------------------------
def _aligned(n, quantum=64):
    return (n + quantum - 1) // quantum * quantum


class ArenaNet(nn.Module):
    """Base class: owns the flat arenas and the single-autograd-node plumbing."""

    def __init__(self):
        super().__init__()
        self._flat = None          # fp32 [n_params] parameter arena
        self._flat_grad = None     # fp32 [n_params] gradient arena
        self._views = []           # (param, grad_view)
        self._hook = None          # dummy leaf that makes autograd schedule our backward
        self._pending = 0          # forward calls whose backward has not run yet (this step)
        self.grads_ready_callback = None
        self.ctx = O.ConvCtx("fp32")   # convolution arithmetic + flipped-weight cache of THIS network (set_conv_mode)

    @property
    def conv_mode(self):
        return self.ctx.mode

    def set_conv_mode(self, mode):
        """"fp32" (exact CUDA-core kernels), "tf32" (wgmma, single TF32 product) or "tf32x3" (wgmma with
        split-accumulate operands: fp32-level products, the parity mode on the tensor cores).  Returns self."""
        if mode != self.ctx.mode:
            pool, ws = self.ctx.sums_pool, self.ctx.wgrad_stream
            self.ctx = O.ConvCtx(mode)
            self.ctx.sums_pool, self.ctx.wgrad_stream = pool, ws
            self._tf32_version = None          # the operand mirror holds something else in every mode
        return self

    def _arena_ok(self):
        if self._flat is None:
            return False
        p0 = next(self.parameters())
        if p0.device != self._flat.device:
            return False
        off = 0
        for p in self.parameters():
            if p.data_ptr() != self._flat.data_ptr() + 4 * off:
                return False
            off += _aligned(p.numel())
        return True

    def ensure_arena(self):
        """(Re)pack every parameter into one flat buffer; called lazily so that .to(device) and
        load_state_dict() keep working the usual way."""
        if self._arena_ok():
            return
        params = list(self.parameters())
        dev = params[0].device
        if dev.type != "cuda":
            raise RuntimeError("the networks run on CUDA only (no CPU fallback): move the module with .to('cuda')")
        n = sum(_aligned(p.numel()) for p in params)      # every tensor starts on a 256-byte boundary (float4 loads)
        flat = torch.zeros(n, device=dev, dtype=torch.float32)
        gflat = torch.zeros(n, device=dev, dtype=torch.float32)
        views, off = [], 0
        for p in params:
            cnt = p.numel()
            if p.dim() == 4:
                O_, I_, kh, kw = p.shape
                dst = flat[off:off + cnt].view(O_, kh, kw, I_).permute(0, 3, 1, 2)
                gv = gflat[off:off + cnt].view(O_, kh, kw, I_).permute(0, 3, 1, 2)
            else:
                dst = flat[off:off + cnt].view(p.shape)
                gv = gflat[off:off + cnt].view(p.shape)
            dst.copy_(p.data)
            p.data = dst
            p.grad = gv
            views.append((p, gv))
            off += _aligned(cnt)
        self._flat, self._flat_grad, self._views = flat, gflat, views
        self._hook = torch.zeros(1, device=dev, requires_grad=True)
        # num_batches_tracked of all BatchNorm layers as views of one int64 tensor (one add per network call)
        bns = [m for m in self.modules() if isinstance(m, BNParams)]
        if bns:
            nbt = torch.stack([m.num_batches_tracked.to(dev) for m in bns])
            for i, m in enumerate(bns):
                m.num_batches_tracked = nbt[i]
            for m in self.modules():
                if isinstance(m, ResnetEncoder):
                    m._nbt = nbt
        # operand mirror of the parameter arena for the tensor-core kernels: the TF32-rounded parameters in tf32 mode, their
        # low parts in tf32x3 mode (refreshed at the start of a network call when stale; ArenaAdam writes it with the update)
        self._flat_tf32 = torch.zeros_like(flat)
        self._tf32_version = None
        self.ctx.invalidate()              # cached flips referred to the previous arena
        off = 0
        mods = {id(m.weight): m for m in self.modules() if isinstance(m, ConvParams)}
        for p in params:
            cnt = p.numel()
            if p.dim() == 4 and id(p) in mods:
                O_, I_, kh, kw = p.shape
                mods[id(p)]._tc_view = self._flat_tf32[off:off + cnt].view(O_, kh, kw, I_)
            off += _aligned(cnt)

    trust_adam_mirror = False      # see refresh_operand_weights
    _tf32_version = None

    def _versions(self):
        """torch version counters of the arena and of every parameter (in-place updates bump them)."""
        return (self._flat._version, sum(p._version for p, _ in self._views))

    def refresh_operand_weights(self):
        """Start of every network call: the weights may have changed since the last one (optimizer, load_state_dict)."""
        cx = self.ctx
        if cx.tc:
            # operand mirror: ArenaAdam writes it together with the parameters (and records the arena's torch
            # version counter); any other in-place change of the parameters bumps that counter -> recompute here
            # (the shortcut is opt-in -- Trainer sets trust_adam_mirror -- because writes through `.data` are invisible to
            # the version counters; without it the mirror is recomputed on every call)
            if not (self.trust_adam_mirror and self._tf32_version == self._versions()):
                if cx.split:
                    O.split_tf32(self._flat, self._flat_tf32)
                else:
                    O.round_tf32(self._flat, self._flat_tf32)
                self._tf32_version = self._versions()
            # flipped / transposed copies for the data gradients: all of them in one launch, in place
            cx.refresh_flips(self._flat.device)

    def _fused_eval(self):
        """Eval mode with autograd off: the forward runs without recording (every activation is freed once dead) and with
        BatchNorm fused into the convolution epilogues (see encoder_forward_eval)."""
        return not self.training and not torch.is_grad_enabled()

    def bn_eval_coeffs(self):
        """Eval-mode {scale, shift} of every BatchNorm layer, recomputed from the current parameters and running statistics
        by one launch; returns {id(BNParams): (scale, shift)}.  The job table is rebuilt when a buffer address changes."""
        bns = [m for m in self.modules() if isinstance(m, BNParams)]
        tab = getattr(self, "_bn_eval", None)
        if tab is None or tab.key != O.BnEvalTable.key_of(bns):
            tab = self._bn_eval = O.BnEvalTable(bns, BN_EPS)
        tab.prepare()
        return {id(bn): c for bn, c in zip(bns, tab.coeffs)}

    def _attach_grads(self):
        """Called at the start of every backward: if an optimizer dropped the gradients
        (zero_grad(set_to_none=True)) the arena is stale -> zero it and re-attach the views."""
        if self._views and self._views[0][0].grad is None:
            self._flat_grad.zero_()
        for p, gv in self._views:
            if p.grad is not gv:
                p.grad = gv

    def zero_grad(self, set_to_none=False):
        if self._flat_grad is not None:
            self._flat_grad.zero_()
            for p, gv in self._views:
                p.grad = gv
        else:
            super().zero_grad(set_to_none=set_to_none)

    def flat_params(self):
        self.ensure_arena()
        return self._flat

    def flat_grads(self):
        self.ensure_arena()
        return self._flat_grad

    @staticmethod
    def g(p):
        """Gradient buffer of a parameter in kernel layout."""
        return p.grad.permute(0, 2, 3, 1) if p.dim() == 4 else p.grad


class BackwardPlan:
    """What one network backward computes.
      bn:     flags OR-ed into every BatchNorm backward: O.BN_FROZEN when the forward ran in eval mode (it normalised with the
              running statistics, so the batch-statistics terms of the gradient are absent);
      params: parameter gradients at all -- False when no parameter of the network requires grad: then no weight-gradient,
              head-gradient or BatchNorm parameter-gradient work is issued and the gradient arena is left alone;
      dimg:   one flag per input image (DispResNet 1, PoseResNet 2): its gradient is wanted (the stem's data gradient)."""

    def __init__(self, training=True, params=True, dimg=(False, False)):
        self.bn = 0 if training else O.BN_FROZEN
        self.params = params
        self.dimg = tuple(bool(n) for n in dimg)


TRAIN_PLAN = BackwardPlan()


class _NetCall(torch.autograd.Function):
    @staticmethod
    def forward(ctx, net, hook, groups, *inputs):
        rec, outs = net._forward_impl(groups, *inputs)
        ctx.net, ctx.rec = net, rec
        ctx.set_materialize_grads(False)     # unused outputs (scales 1-3 with --num-scales 1) arrive as None
        return tuple(outs)

    @staticmethod
    def backward(ctx, *grads):
        net = ctx.net
        need = ctx.needs_input_grad[3:]
        # the BatchNorm formula follows the mode the FORWARD ran in (recorded), not net.training now
        plan = BackwardPlan(ctx.rec["training"], any(p.requires_grad for p, _ in net._views), need)
        dimgs = [None] * len(need)
        if plan.params or any(need):
            if plan.params:
                net._attach_grads()
            dimgs = net._backward_impl(ctx.rec, [None if g is None else g.contiguous() for g in grads], plan)
            net.ctx.join_wgrad()       # weight gradients enqueued on the side stream (if any) are part of this backward
        ctx.rec = None
        net._pending -= 1
        if net._pending == 0 and net.grads_ready_callback is not None:
            net.grads_ready_callback(net)
        return (None, None, None) + tuple(dimgs)


# ------------------------------------------------------------------------------------------------
# encoder execution
# ------------------------------------------------------------------------------------------------
class _SumsPool:
    """fp64 scratch for the fused BatchNorm sums of one network call: ONE fill per call instead of one torch.zeros per
    layer.  Each layer's slice is consumed by bn_apply right after the convolution that accumulates into it, so the
    pool is recycled by the next call.  It grows to the largest call seen (growth happens during the eager warm-up,
    i.e. before any CUDA-graph capture)."""

    def __init__(self):
        self.buf, self.cursor, self.need = {}, 0, 0

    def begin(self, device):
        self.need = max(self.need, self.cursor)
        buf = self.buf.get(device)
        if buf is None or buf.numel() < self.need:
            buf = self.buf[device] = torch.zeros(max(self.need, 1 << 16), device=device, dtype=torch.float64)
        elif self.cursor:
            buf[:self.cursor].zero_()
        self.cursor = 0

    def take(self, n, device):
        n = (n + 31) // 32 * 32                      # 256-byte aligned slices
        buf = self.buf.get(device)
        start, self.cursor = self.cursor, self.cursor + n
        if buf is None or self.cursor > buf.numel():
            return torch.zeros(n, device=device, dtype=torch.float64)       # first (sizing) call only
        return buf[start:start + n]


def _pool(cx):
    """The BatchNorm-sums pool of one network (lives on its ConvCtx: two networks may run concurrently on two streams, and
    a pool is sized by its own network's calls during the eager warm-up, i.e. before any CUDA-graph capture)."""
    if cx.sums_pool is None:
        cx.sums_pool = _SumsPool()
    return cx.sums_pool


def _bn_fwd(cx, y, sums, bn, training, relu, residual, groups):
    """BatchNorm over `groups` independent sample groups (one per batched network call: statistics, and the
    running-stat updates, stay per call exactly as in train.py:427-442).  num_batches_tracked of every layer is bumped
    by one add per network call (ArenaNet._nbt, see encoder_forward)."""
    return O.bn_apply(y, sums if training else None, bn.weight, bn.bias, bn.running_mean, bn.running_var, BN_MOMENTUM, BN_EPS,
                      residual, (1 if relu else 0) | cx.rnd(), groups, cx.split)


def _conv_bn(cx, x, conv, bn, stride, pad, training, relu, residual=None, groups=1):
    C = conv.weight.shape[0]
    sums = _pool(cx).take(O.BN_SLOTS * groups * C * 2, x.device) if training else None
    y = cx.conv_fwd(x, conv.w_op(cx), None, stride, pad, O.PAD_ZERO, O.ACT_NONE, sums, groups, conv.w_lo(cx))
    z, saved = _bn_fwd(cx, y, sums, bn, training, relu, residual, groups)
    return y, z, saved


def _bn_param_grads(bn, plan):
    return (bn.weight.grad, bn.bias.grad) if plan.params else (None, None)


def _conv_bn_bwd(cx, dz, z, y, saved, x, conv, bn, stride, pad, relu, want_dres, need_dx, addend=None, groups=1, plan=TRAIN_PLAN):
    """Backward through relu?(bn(conv(x)) [+res]).  Returns (dx or None, dres or None)."""
    dy, dres = O.bn_backward(dz, z, y, saved, *_bn_param_grads(bn, plan), (1 if relu else 0) | cx.rnd() | plan.bn, want_dres, groups,
                             cx.split)
    if plan.params:
        cx.conv_wgrad(x, dy, ArenaNet.g(conv.weight), None, stride, pad, O.PAD_ZERO)
    dx = cx.conv_dgrad(dy, conv.w_op(cx), x.shape, stride, pad, addend) if need_dx else None
    return dx, dres


def block_forward(cx, blk, x, training, G=1):
    r = {"x": x, "G": G}
    if blk.bottleneck:
        r["y1"], r["h1"], r["s1"] = _conv_bn(cx, x, blk.conv1, blk.bn1, 1, 0, training, True, None, G)
        r["y2"], r["h2"], r["s2"] = _conv_bn(cx, r["h1"], blk.conv2, blk.bn2, blk.stride, 1, training, True, None, G)
        last_in, last_conv, last_bn, key = r["h2"], blk.conv3, blk.bn3, "3"
        ls, lp = 1, 0
    else:
        r["y1"], r["h1"], r["s1"] = _conv_bn(cx, x, blk.conv1, blk.bn1, blk.stride, 1, training, True, None, G)
        last_in, last_conv, last_bn, key = r["h1"], blk.conv2, blk.bn2, "2"
        ls, lp = 1, 1
    sc = x
    if blk.downsample is not None:
        r["yd"], sc, r["sd"] = _conv_bn(cx, x, blk.downsample[0], blk.downsample[1], blk.stride, 0, training, False, None, G)
    C = last_conv.weight.shape[0]
    sums = _pool(cx).take(O.BN_SLOTS * G * C * 2, x.device) if training else None
    y = cx.conv_fwd(last_in, last_conv.w_op(cx), None, ls, lp, O.PAD_ZERO, O.ACT_NONE, sums, G, last_conv.w_lo(cx))
    out, saved = _bn_fwd(cx, y, sums, last_bn, training, True, sc, G)
    r["y" + key], r["s" + key], r["out"] = y, saved, out
    return r, out


def block_backward(cx, blk, r, d_out, extra_addend=None, plan=TRAIN_PLAN):
    """d_out: gradient w.r.t. the block output (consumed / overwritten).  extra_addend: gradient that reaches
    the block INPUT from elsewhere (decoder skip connection) -- folded into the dgrad epilogue chain.
    Returns gradient w.r.t. the block input."""
    x, G = r["x"], r["G"]
    if blk.bottleneck:
        dh2, dres = _conv_bn_bwd(cx, d_out, r["out"], r["y3"], r["s3"], r["h2"], blk.conv3, blk.bn3, 1, 0, True, True, True, None, G, plan)
        dh1, _ = _conv_bn_bwd(cx, dh2, r["h2"], r["y2"], r["s2"], r["h1"], blk.conv2, blk.bn2, blk.stride, 1, True, False, True, None, G,
                              plan)
        first = (dh1, r["h1"], r["y1"], r["s1"], blk.conv1, blk.bn1, 1, 0)
    else:
        dh1, dres = _conv_bn_bwd(cx, d_out, r["out"], r["y2"], r["s2"], r["h1"], blk.conv2, blk.bn2, 1, 1, True, True, True, None, G, plan)
        first = (dh1, r["h1"], r["y1"], r["s1"], blk.conv1, blk.bn1, blk.stride, 1)
    if blk.downsample is not None:
        d_sc, _ = _conv_bn_bwd(cx, dres, None, r["yd"], r["sd"], x, blk.downsample[0], blk.downsample[1], blk.stride, 0, False,
                               False, True, extra_addend, G, plan)
    else:
        d_sc = dres
        if extra_addend is not None:
            d_sc = d_sc + extra_addend          # not reached by ResNet-18/50 (skips feed downsample blocks)
    dz, z, y, s, conv, bn, st, pd = first
    dx, _ = _conv_bn_bwd(cx, dz, z, y, s, x, conv, bn, st, pd, True, False, True, d_sc, G, plan)
    return dx


def encoder_forward(cx, enc, imgs, training, G=1):
    """imgs: tuple of one (DispResNet) or two (PoseResNet, channel-concatenated) NCHW image batches."""
    t = enc.encoder
    rec = {"G": G}
    if training:
        _pool(cx).begin(imgs[0].device)
        nbt = getattr(enc, "_nbt", None)
        if nbt is not None:
            nbt.add_(G)                      # every BatchNorm layer's num_batches_tracked (views of this tensor)
        else:
            for m in enc.modules():
                if isinstance(m, BNParams):
                    m.num_batches_tracked += G
    if cx.tc:
        # 7x7 stem on the tensor cores: input channels zero-padded 3 -> 4 / 6 -> 8 (K = 49 * Cpad), weights likewise
        cpad = 4 * len(imgs)
        x_nhwc = O.nchw_to_nhwc_pad(imgs[0], imgs[1] if len(imgs) > 1 else None, cpad, cx.operand)
        w0 = O.pad_channels(t.conv1.w_khwc(), cpad, cx.operand)
        w0_lo = O.pad_channels(t.conv1.w_khwc(), cpad, O.OPERAND_LO) if cx.split else None
        C = w0.shape[0]
        sums = _pool(cx).take(O.BN_SLOTS * G * C * 2, x_nhwc.device) if training else None
        rec["y0"] = cx.conv_fwd(x_nhwc, w0, None, 2, 3, O.PAD_ZERO, O.ACT_NONE, sums, G, w0_lo)
        f0, rec["s0"] = _bn_fwd(cx, rec["y0"], sums, t.bn1, training, True, None, G)
    else:
        x_nhwc = O.nchw_to_nhwc(imgs[0], imgs[1] if len(imgs) > 1 else None)
        rec["y0"], f0, rec["s0"] = _conv_bn(cx, x_nhwc, t.conv1, t.bn1, 2, 3, training, True, None, G)
    rec["x"] = x_nhwc
    rec["f0"] = f0
    pooled, rec["pool_idx"] = O.maxpool_fwd(f0)
    feats, blocks, x = [f0], [], pooled
    for li in range(1, 5):
        for blk in getattr(t, "layer%d" % li):
            r, x = block_forward(cx, blk, x, training, G)
            blocks.append((blk, r))
        feats.append(x)
    rec["blocks"], rec["feats"] = blocks, feats
    return rec, feats


def _conv_bn_eval(cx, x, conv, bn, coeffs, stride, pad, relu, residual=None, with_lo=False):
    """relu?(bn(conv(x)) [+ residual]) in eval mode as ONE convolution: BatchNorm, residual, ReLU and TF32 rounding in its
    epilogue (bitwise conv_fwd followed by bn_apply).  with_lo: the output feeds a tensor-core convolution (tf32x3: write its
    low part too)."""
    sc, sh = coeffs[id(bn)]
    return cx.conv_fwd(x, conv.w_op(cx), None, stride, pad, O.PAD_ZERO, (O.ACT_RELU if relu else O.ACT_NONE) | cx.rnd(), None, 1,
                       conv.w_lo(cx), bn_scale=sc, bn_shift=sh, addend=residual, with_lo=with_lo and cx.split)


def block_forward_eval(cx, blk, x, coeffs):
    if blk.bottleneck:
        h1 = _conv_bn_eval(cx, x, blk.conv1, blk.bn1, coeffs, 1, 0, True, None, True)
        h2 = _conv_bn_eval(cx, h1, blk.conv2, blk.bn2, coeffs, blk.stride, 1, True, None, True)
        del h1
        last_in, last_conv, last_bn, ls, lp = h2, blk.conv3, blk.bn3, 1, 0
    else:
        h1 = _conv_bn_eval(cx, x, blk.conv1, blk.bn1, coeffs, blk.stride, 1, True, None, True)
        last_in, last_conv, last_bn, ls, lp = h1, blk.conv2, blk.bn2, 1, 1
    sc = x
    if blk.downsample is not None:
        sc = _conv_bn_eval(cx, x, blk.downsample[0], blk.downsample[1], coeffs, blk.stride, 0, False)
    return _conv_bn_eval(cx, last_in, last_conv, last_bn, coeffs, ls, lp, True, sc, True)


def encoder_forward_eval(cx, enc, imgs, coeffs):
    """encoder_forward's eval-mode features without the record: imgs as there, coeffs from ArenaNet.bn_eval_coeffs()."""
    t = enc.encoder
    if cx.tc:
        cpad = 4 * len(imgs)
        x_nhwc = O.nchw_to_nhwc_pad(imgs[0], imgs[1] if len(imgs) > 1 else None, cpad, cx.operand)
        w0 = O.pad_channels(t.conv1.w_khwc(), cpad, cx.operand)
        w0_lo = O.pad_channels(t.conv1.w_khwc(), cpad, O.OPERAND_LO) if cx.split else None
        sc, sh = coeffs[id(t.bn1)]
        f0 = cx.conv_fwd(x_nhwc, w0, None, 2, 3, O.PAD_ZERO, O.ACT_RELU | cx.rnd(), None, 1, w0_lo, bn_scale=sc, bn_shift=sh)
    else:
        x_nhwc = O.nchw_to_nhwc(imgs[0], imgs[1] if len(imgs) > 1 else None)
        f0 = _conv_bn_eval(cx, x_nhwc, t.conv1, t.bn1, coeffs, 2, 3, True)
    del x_nhwc
    x, _ = O.maxpool_fwd(f0)
    feats = [f0]
    for li in range(1, 5):
        for blk in getattr(t, "layer%d" % li):
            x = block_forward_eval(cx, blk, x, coeffs)
        feats.append(x)
    return feats


def encoder_backward(cx, enc, rec, d_feats, plan=TRAIN_PLAN):
    """d_feats[i]: gradient w.r.t. feature i coming from the decoder (None if unused).  d_feats[4] is required.
    Returns the gradients of the input images (NCHW, one per image of the forward; None where plan.dimg does not ask)."""
    t = enc.encoder
    blocks = rec["blocks"]
    # index of the last block of each layer -> the feature it produces
    ends, k = {}, 0
    for li in range(1, 5):
        k += len(getattr(t, "layer%d" % li))
        ends[k - 1] = li
    d = d_feats[4]
    for bi in range(len(blocks) - 1, -1, -1):
        blk, r = blocks[bi]
        # the INPUT of block bi is the output of block bi-1; if that is a skip feature, add the decoder's gradient
        extra = None
        if bi - 1 in ends and d_feats[ends[bi - 1]] is not None:
            extra = d_feats[ends[bi - 1]]
        d = block_backward(cx, blk, r, d, extra, plan)
    # d is now the gradient w.r.t. the max-pool output
    f0 = rec["f0"]
    if d_feats[0] is not None:
        d_f0 = d_feats[0]
        O.maxpool_bwd(d, rec["pool_idx"], f0.shape, d_f0, True)
    else:
        d_f0 = torch.empty_like(f0)
        O.maxpool_bwd(d, rec["pool_idx"], f0.shape, d_f0, False)
    x = rec["x"]
    relu = 1 | cx.rnd() | plan.bn
    if x.shape[-1] != t.conv1.weight.shape[1]:
        # padded-channel stem (tensor-core modes): weight gradient in the padded layout, then folded into the gradient arena
        # (the low part of dy is only read by that weight gradient)
        dy, _ = O.bn_backward(d_f0, f0, rec["y0"], rec["s0"], *_bn_param_grads(t.bn1, plan), relu, False, rec["G"], cx.split and plan.params)
        if plan.params:
            dw = torch.zeros(t.conv1.weight.shape[0], t.conv1.k, t.conv1.k, x.shape[-1], device=x.device, dtype=torch.float32)
            cx.conv_wgrad(x, dy, dw, None, 2, 3, O.PAD_ZERO)
            with cx.on_wgrad_stream([dw]):
                O.unpad_add_(ArenaNet.g(t.conv1.weight), dw)
    else:
        dy, _ = O.bn_backward(d_f0, f0, rec["y0"], rec["s0"], *_bn_param_grads(t.bn1, plan), relu, False, rec["G"], cx.split)
        if plan.params:
            cx.conv_wgrad(x, dy, ArenaNet.g(t.conv1.weight), None, 2, 3, O.PAD_ZERO)
    if not any(plan.dimg):
        return [None] * len(plan.dimg)
    # input images: the transposed stem convolution with the fp32 weights (not the padded / TF32 operand copies)
    return O.stem_dgrad(dy, t.conv1.w_khwc(), x.shape[1], x.shape[2], plan.dimg)


# ------------------------------------------------------------------------------------------------
# networks
# ------------------------------------------------------------------------------------------------
class DispResNet(ArenaNet):
    """models.DispResNet(num_layers=18, pretrained=True) (reference DispResNet.py:104-121)."""

    def __init__(self, num_layers=18, pretrained=True):
        super().__init__()
        self.encoder = ResnetEncoder(num_layers=num_layers, pretrained=pretrained, num_input_images=1)
        self.decoder = DepthDecoder(self.encoder.num_ch_enc)

    def init_weights(self):
        pass

    def forward(self, x):
        self.ensure_arena()
        if self._fused_eval():
            return self._forward_impl(1, x, fused=True)[1][0]
        if torch.is_grad_enabled():
            self._pending += 1
        outs = _NetCall.apply(self, self._hook, 1, x)
        return list(outs) if self.training else outs[0]

    def forward_multi(self, images):
        """Several independent network calls in ONE launch sequence: `images` is a list of [B,3,H,W] tensors;
        returns one output per image, each exactly what `self(image)` would return.  The calls are stacked on
        the batch axis (more rows per GEMM, 1/len(images) of the kernel launches) while BatchNorm statistics
        and running-stat updates stay per call, in list order (train.py:427-434 semantics)."""
        self.ensure_arena()
        if torch.is_grad_enabled():
            self._pending += 1
        G, B = len(images), images[0].shape[0]
        if self._fused_eval():
            out = self._forward_impl(G, torch.cat(list(images), 0), fused=True)[1][0]
            return [out[g * B:(g + 1) * B] for g in range(G)]
        outs = _NetCall.apply(self, self._hook, G, torch.cat(list(images), 0))
        per = [[o[g * B:(g + 1) * B] for o in outs] for g in range(G)]
        return per if self.training else [p[0] for p in per]

    # -- forward ------------------------------------------------------------------------------
    def _forward_impl(self, groups, x, fused=False):
        """fused (eval mode, autograd off): no record, BatchNorm in the convolution epilogues; returns (None, outputs)."""
        from . import lib as L
        x = L.dev_f32(x, "DispResNet input")
        self.refresh_operand_weights()
        training = self.training
        cx = self.ctx
        if fused:
            enc_rec, feats = None, encoder_forward_eval(cx, self.encoder, (x,), self.bn_eval_coeffs())
        else:
            enc_rec, feats = encoder_forward(cx, self.encoder, (x,), training, groups)
        dec = self.decoder
        rec = {"enc": enc_rec, "stages": {}, "training": training}
        cur = feats[4]
        disps = {}
        for i in range(4, -1, -1):
            c0 = dec.up(i, 0)
            a = cx.conv_fwd(cur, c0.w_op(cx), c0.bias, 1, 1, O.PAD_REFLECT, O.ACT_ELU | cx.rnd(), None, 1, c0.w_lo(cx))
            cat = O.upcat_fwd(a, feats[i - 1] if i > 0 else None)
            c1 = dec.up(i, 1)
            # (fused: b feeds the next stage's first convolution directly, so its low part is written with it)
            b = cx.conv_fwd(cat, c1.w_op(cx), c1.bias, 1, 1, O.PAD_REFLECT, O.ACT_ELU | cx.rnd(), None, 1, c1.w_lo(cx),
                            with_lo=fused and cx.split and i > 0)
            if fused:
                if i > 0:
                    feats[i - 1] = None          # the skip feature is dead once concatenated
            else:
                rec["stages"][i] = {"in0": cur, "a": a, "cat": cat, "b": b}
            del a, cat
            cur = b
            if i < 4 and (training or i == 0):
                dc = dec.disp(i)
                disps[i] = O.head_fwd(cur, dc.w_khwc(), dc.bias, O.ACT_DISP)
        rec["disps"] = disps
        order = [0, 1, 2, 3] if training else [0]
        rec["order"] = order
        # [B,H,W,1] NHWC is bit-identical to [B,1,H,W] NCHW
        return None if fused else rec, [disps[s].view(disps[s].shape[0], 1, disps[s].shape[1], disps[s].shape[2]) for s in order]

    # -- backward -----------------------------------------------------------------------------
    def _backward_impl(self, rec, grads, plan=TRAIN_PLAN):
        """Returns [gradient of the input images or None] (see encoder_backward)."""
        dec = self.decoder
        g = ArenaNet.g
        cx = self.ctx
        d_disp = {s: gr for s, gr in zip(rec["order"], grads) if gr is not None}
        d_feats = [None] * 5
        d_b = None          # gradient w.r.t. the pre-activation of up(i,1) (after folding every consumer)
        pending = None      # gradient of b_i from stage i-1's first conv, waiting for the dispconv share
        for i in range(0, 5):
            st = rec["stages"][i]
            b = st["b"]
            have = pending is not None
            d_b = pending
            if i in d_disp:
                dc = dec.disp(i)
                disp = rec["disps"][i]
                dpre = O.act_bwd_(d_disp[i].reshape(disp.shape).clone(), disp, O.ACT_DISP)
                if plan.params:
                    O.head_wgrad(b, dpre, g(dc.weight), dc.bias.grad)
                dpad = O.head_dgrad(dpre, dc.w_khwc(), b.shape)
                if not have:
                    d_b = torch.empty_like(b)
                O.fold_plain(dpad, d_b, b, O.ACT_ELU | cx.rnd(), accumulate=have)
            elif have:
                O.act_bwd_(d_b, b, O.ACT_ELU | cx.rnd())
            else:
                continue            # nothing reaches this stage (cannot happen: stage 0 always has scale 0)
            # up(i,1): b = ELU(conv(reflect_pad(cat)))
            c1 = dec.up(i, 1)
            if plan.params:
                cx.conv_wgrad(st["cat"], d_b, g(c1.weight), c1.bias.grad, 1, 1, O.PAD_REFLECT)
            dpad = cx.conv_dgrad(d_b, c1.w_op(cx), st["cat"].shape, 1, 1, None, padded_input=True)
            d_a, d_skip = O.fold_upcat(dpad, st["a"].shape[-1], st["a"], O.ACT_ELU | cx.rnd())
            if i > 0:
                d_feats[i - 1] = d_skip
            # up(i,0): a = ELU(conv(reflect_pad(in0)))
            c0 = dec.up(i, 0)
            if plan.params:
                cx.conv_wgrad(st["in0"], d_a, g(c0.weight), c0.bias.grad, 1, 1, O.PAD_REFLECT)
            dpad = cx.conv_dgrad(d_a, c0.w_op(cx), st["in0"].shape, 1, 1, None, padded_input=True)
            d_in = torch.empty_like(st["in0"])
            O.fold_plain(dpad, d_in, None, O.ACT_NONE, accumulate=False)
            if i < 4:
                pending = d_in          # = raw gradient of b_{i+1}; ELU' applied once all consumers are in
            else:
                d_feats[4] = d_in
        return encoder_backward(cx, self.encoder, rec["enc"], d_feats, plan)


class PoseResNet(ArenaNet):
    """models.PoseResNet(num_layers=18, pretrained=True) (reference PoseResNet.py:54-68)."""

    def __init__(self, num_layers=18, pretrained=True):
        super().__init__()
        self.encoder = ResnetEncoder(num_layers=num_layers, pretrained=pretrained, num_input_images=2)
        self.decoder = PoseDecoder(self.encoder.num_ch_enc)

    def init_weights(self):
        pass

    def forward(self, img1, img2):
        self.ensure_arena()
        if self._fused_eval():
            return self._forward_impl(1, img1, img2, fused=True)[1][0]
        if torch.is_grad_enabled():
            self._pending += 1
        return _NetCall.apply(self, self._hook, 1, img1, img2)[0]

    def forward_multi(self, pairs):
        """`pairs` = list of (img1, img2); one stacked launch sequence, BatchNorm per call (see DispResNet.forward_multi).
        Returns the list of [B,6] poses."""
        self.ensure_arena()
        if torch.is_grad_enabled():
            self._pending += 1
        G, B = len(pairs), pairs[0][0].shape[0]
        if self._fused_eval():
            out = self._forward_impl(G, torch.cat([a for a, _ in pairs], 0), torch.cat([b for _, b in pairs], 0), fused=True)[1][0]
            return [out[g * B:(g + 1) * B] for g in range(G)]
        out = _NetCall.apply(self, self._hook, G, torch.cat([a for a, _ in pairs], 0), torch.cat([b for _, b in pairs], 0))[0]
        return [out[g * B:(g + 1) * B] for g in range(G)]

    def _forward_impl(self, groups, img1, img2, fused=False):
        """fused (eval mode, autograd off): no record, BatchNorm in the convolution epilogues; returns (None, outputs)."""
        from . import lib as L
        img1, img2 = L.dev_f32(img1, "PoseResNet input"), L.dev_f32(img2, "PoseResNet input")
        self.refresh_operand_weights()
        cx = self.ctx
        n = self.decoder.net
        if fused:
            f4 = encoder_forward_eval(cx, self.encoder, (img1, img2), self.bn_eval_coeffs())[4]
            lo = cx.split
            s = cx.conv_fwd(f4, n[0].w_op(cx), n[0].bias, 1, 0, O.PAD_ZERO, O.ACT_RELU | cx.rnd(), None, 1, n[0].w_lo(cx), with_lo=lo)
            del f4
            p0 = cx.conv_fwd(s, n[1].w_op(cx), n[1].bias, 1, 1, O.PAD_ZERO, O.ACT_RELU | cx.rnd(), None, 1, n[1].w_lo(cx), with_lo=lo)
            del s
            p1 = cx.conv_fwd(p0, n[2].w_op(cx), n[2].bias, 1, 1, O.PAD_ZERO, O.ACT_RELU | cx.rnd(), None, 1, n[2].w_lo(cx))
            del p0
            p2 = cx.conv_fwd(p1, n[3].w_op(cx), n[3].bias, 1, 0, O.PAD_ZERO, O.ACT_NONE, None, 1, n[3].w_lo(cx))
            return None, [O.spatial_mean_fwd(p2, 0.01)]
        enc_rec, feats = encoder_forward(cx, self.encoder, (img1, img2), self.training, groups)
        rec = {"enc": enc_rec, "f4": feats[4], "training": self.training}
        rec["s"] = cx.conv_fwd(feats[4], n[0].w_op(cx), n[0].bias, 1, 0, O.PAD_ZERO, O.ACT_RELU | cx.rnd(), None, 1, n[0].w_lo(cx))
        rec["p0"] = cx.conv_fwd(rec["s"], n[1].w_op(cx), n[1].bias, 1, 1, O.PAD_ZERO, O.ACT_RELU | cx.rnd(), None, 1, n[1].w_lo(cx))
        rec["p1"] = cx.conv_fwd(rec["p0"], n[2].w_op(cx), n[2].bias, 1, 1, O.PAD_ZERO, O.ACT_RELU | cx.rnd(), None, 1, n[2].w_lo(cx))
        rec["p2"] = cx.conv_fwd(rec["p1"], n[3].w_op(cx), n[3].bias, 1, 0, O.PAD_ZERO, O.ACT_NONE, None, 1, n[3].w_lo(cx))
        return rec, [O.spatial_mean_fwd(rec["p2"], 0.01)]

    def _backward_impl(self, rec, grads, plan=TRAIN_PLAN):
        """Returns [gradient of img1 or None, gradient of img2 or None] (see encoder_backward)."""
        n = self.decoder.net
        g = ArenaNet.g
        cx = self.ctx
        d = O.spatial_mean_bwd(grads[0], rec["p2"].shape, 0.01)
        chain = [(n[3], rec["p1"], 0), (n[2], rec["p0"], 1), (n[1], rec["s"], 1), (n[0], rec["f4"], 0)]
        for k, (conv, inp, pad) in enumerate(chain):
            if plan.params:
                cx.conv_wgrad(inp, d, g(conv.weight), conv.bias.grad, 1, pad, O.PAD_ZERO)
            d = cx.conv_dgrad(d, conv.w_op(cx), inp.shape, 1, pad)
            if k < 3:
                O.act_bwd_(d, inp, O.ACT_RELU | cx.rnd())       # inp is the ReLU output of the previous conv
        return encoder_backward(cx, self.encoder, rec["enc"], [None, None, None, None, d], plan)


# ------------------------------------------------------------------------------------------------
# fused Adam over the arenas (train.py:171-178: two parameter groups, same hyper-parameters)
# ------------------------------------------------------------------------------------------------
class ArenaAdam:
    """torch.optim.Adam semantics (betas, eps 1e-8, weight decay folded into the gradient) with one kernel
    launch per network.  Parameters whose gradient stays zero (the unused fc head and, with
    --num-scales 1, the scale 1-3 disparity heads) are left unchanged exactly as Adam skips
    `grad is None` parameters in the reference -- for weight_decay == 0 (the reference's scripts); with
    weight_decay > 0 the whole arena is decayed, those unused tensors included (documented deviation).  The step counter lives on the device so that the whole
    training step can be captured in a CUDA graph."""

    def __init__(self, nets, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        self.nets = list(nets)
        self.lr, self.betas, self.eps, self.weight_decay = lr, betas, eps, weight_decay
        self.state = {}
        self._step = None

    @property
    def step_count(self):
        return 0 if self._step is None else int(self._step.item())

    def zero_grad(self, set_to_none=False):
        for n in self.nets:
            n.ensure_arena()
            n.zero_grad()

    def _ensure_state(self):
        for n in self.nets:
            n.ensure_arena()
            key = id(n)
            if key not in self.state or self.state[key][2] is not n._flat:      # first step, or the arena was re-packed
                self.state[key] = (torch.zeros_like(n._flat), torch.zeros_like(n._flat), n._flat)
        if self._step is None:
            self._step = torch.zeros(1, device=self.nets[0]._flat.device, dtype=torch.int32)

    def step(self):
        self._ensure_state()
        self._step += 1
        for n in self.nets:
            n._pending = 0     # nothing may be pending after the update (a forward whose backward never ran must not block
            #                    the next step's gradient all-reduce; Trainer additionally checks that both were issued)
            m, v, _ = self.state[id(n)]
            mirror = n._flat_tf32 if n.ctx.tc else None
            O.adam_step(n._flat, n._flat_grad, m, v, self.lr, self.betas[0], self.betas[1], self.eps, self.weight_decay,
                        0, self._step, mirror, O.OPERAND_LO if n.ctx.split else O.OPERAND_TF32)
            # the kernel writes through raw pointers (no torch version bump): with the mirror written the arena is in sync,
            # without it the next network call must re-round
            n._tf32_version = n._versions() if mirror is not None else None
        # (the TF32 mirror and the flipped dgrad weights are refreshed at the start of the next network call)

    def snapshot(self):
        """Copies of everything a step mutates (used to undo the warm-up step before CUDA-graph capture)."""
        self._ensure_state()
        snap = {"step": self._step.clone(), "nets": []}
        for n in self.nets:
            m, v, _ = self.state[id(n)]
            snap["nets"].append((n._flat.clone(), m.clone(), v.clone(), {k: b.clone() for k, b in n.named_buffers()}))
        return snap

    def restore(self, snap):
        self._step.copy_(snap["step"])
        for n, (flat, m0, v0, bufs) in zip(self.nets, snap["nets"]):
            m, v, _ = self.state[id(n)]
            n._flat.copy_(flat); m.copy_(m0); v.copy_(v0)
            for k, b in n.named_buffers():
                b.copy_(bufs[k])

    def state_dict(self):
        self._ensure_state()
        return {"step": self.step_count, "exp_avg": [self.state[id(n)][0] for n in self.nets],
                "exp_avg_sq": [self.state[id(n)][1] for n in self.nets]}
