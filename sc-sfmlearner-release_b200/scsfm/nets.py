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
import collections
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


class BNParams(nn.BatchNorm2d):
    """The reference's nn.BatchNorm2d(c): the same parameters, buffers, state_dict keys and initial values, found by
    isinstance(m, nn.BatchNorm2d), and put in eval mode per module (`m.eval()`: running statistics, none updated).  The
    network's kernels apply it, so its own forward is never called, and momentum / eps other than the reference's are refused
    (check_supported)."""

    def forward(self, x):
        raise RuntimeError("BNParams is applied by its network's kernels; it is not callable on its own")

    def check_supported(self):
        if self.momentum != BN_MOMENTUM or self.eps != BN_EPS or not self.affine or not self.track_running_stats:
            raise ValueError("BatchNorm with momentum=%r eps=%r affine=%r track_running_stats=%r: the network kernels implement "
                             "only the reference's momentum=%r eps=%r with affine parameters and running statistics"
                             % (self.momentum, self.eps, self.affine, self.track_running_stats, BN_MOMENTUM, BN_EPS))


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

    def units(self):
        """The block's convolutions as (conv, bn, stride, pad) units: the main path in forward order (every unit followed by a
        ReLU, the last one after the residual add), and the downsample unit of the shortcut or None.  Plain tuples of the
        registered submodules: nothing here is registered again."""
        if self.bottleneck:
            main = [(self.conv1, self.bn1, 1, 0), (self.conv2, self.bn2, self.stride, 1), (self.conv3, self.bn3, 1, 0)]
        else:
            main = [(self.conv1, self.bn1, self.stride, 1), (self.conv2, self.bn2, 1, 1)]
        ds = None if self.downsample is None else (self.downsample[0], self.downsample[1], self.stride, 0)
        return main, ds


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


# PoseDecoder.net[k] in forward order as (pad, activation); all four convolutions have stride 1 and a bias.
POSE_HEAD = ((0, O.ACT_RELU), (1, O.ACT_RELU), (1, O.ACT_RELU), (0, O.ACT_NONE))


def _pose_act(cx, k):
    """Activation flags of pose-head convolution k: the output of every one but the last feeds the next convolution."""
    act = POSE_HEAD[k][1]
    return act | cx.rnd() if k + 1 < len(POSE_HEAD) else act


# ------------------------------------------------------------------------------------------------
# flat parameter / gradient arenas
# ------------------------------------------------------------------------------------------------
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
            off += O.aligned64(p.numel())
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
        n = sum(O.aligned64(p.numel()) for p in params)      # every tensor starts on a 256-byte boundary (float4 loads)
        flat = torch.zeros(n, device=dev, dtype=torch.float32)
        gflat = torch.zeros(n, device=dev, dtype=torch.float32)
        # operand mirror of the parameter arena for the tensor-core kernels: the TF32-rounded parameters in tf32 mode, their
        # low parts in tf32x3 mode (refreshed at the start of a network call when stale; ArenaAdam writes it with the update)
        self._flat_tf32 = torch.zeros_like(flat)
        convs = {id(m.weight): m for m in self.modules() if isinstance(m, ConvParams)}
        views, off = [], 0
        for p in params:
            cnt = p.numel()
            if p.dim() == 4:
                O_, I_, kh, kw = p.shape
                dst = flat[off:off + cnt].view(O_, kh, kw, I_).permute(0, 3, 1, 2)
                gv = gflat[off:off + cnt].view(O_, kh, kw, I_).permute(0, 3, 1, 2)
                convs[id(p)]._tc_view = self._flat_tf32[off:off + cnt].view(O_, kh, kw, I_)
            else:
                dst = flat[off:off + cnt].view(p.shape)
                gv = gflat[off:off + cnt].view(p.shape)
            dst.copy_(p.data)
            p.data = dst
            p.grad = gv if p.requires_grad else None
            p._arena_grad = gv             # what the kernels accumulate into, whether or not p.grad exposes it
            views.append((p, gv))
            off += O.aligned64(cnt)
        self._flat, self._flat_grad, self._views = flat, gflat, views
        self._hook = torch.zeros(1, device=dev, requires_grad=True)
        # num_batches_tracked of all BatchNorm layers as views of one int64 tensor (one add per network call)
        bns = self._bns = [m for m in self.modules() if isinstance(m, BNParams)]
        if bns:
            nbt = torch.stack([m.num_batches_tracked.to(dev) for m in bns])
            for i, m in enumerate(bns):
                m.num_batches_tracked = nbt[i]
            for m in self.modules():
                if isinstance(m, ResnetEncoder):
                    m._nbt, m._nbt_bns, m._nbt_inc = nbt, bns, {}
        self._tf32_version = None
        self.ctx.invalidate()              # cached flips referred to the previous arena

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
        BatchNorm fused into the convolution epilogues (see _conv_bn)."""
        return not self.training and not torch.is_grad_enabled() and not any(bn.training for bn in self._bns)

    def _encoder_forward(self, groups, imgs, fused, plan):
        """The encoder part of a network call: fused where the whole call is, and inside a recording call whose backward does
        not reach the encoder (plan.feats[4] False) when all its BatchNorms are in eval mode -- bitwise the same features,
        no record."""
        fused = fused or (not plan.feats[4] and not any(bn.training for bn in self._bns))
        return encoder_forward(_Forward(self, groups, fused, plan), self.encoder, imgs)

    def flag_pattern(self):
        """The module flags a network call depends on: requires_grad of every parameter, the mode of every BatchNorm and of
        the network (a CUDA graph captured with one pattern is not valid for another).  Needs the packed arena."""
        return (self.training, tuple(p.requires_grad for p, _ in self._views), tuple(bn.training for bn in self._bns))

    def _call(self, inputs, groups=None):
        """One network call on `inputs`: the fused eval forward, or one autograd node.  groups=None returns the call's
        outputs; otherwise the inputs stack `groups` equal sample groups on the batch axis (BatchNorm statistics stay per
        group) and the result is one output list per group."""
        G = groups or 1
        self.ensure_arena()
        for bn in self._bns:
            bn.check_supported()
        if self._fused_eval():
            outs = self._forward_impl(G, *inputs, fused=True)[1]
        else:
            grad = torch.is_grad_enabled()
            if grad:
                self._pending += 1
            plan = BackwardPlan(self, [grad and x.requires_grad for x in inputs])
            outs = _NetCall.apply(self, self._hook, G, plan, *inputs)
        if groups is None:
            return outs
        B = inputs[0].shape[0] // G
        return [[o[g * B:(g + 1) * B] for o in outs] for g in range(G)]

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
        """Called at the start of every backward that computes parameter gradients: trainable parameters get their arena view
        as .grad, frozen ones keep None (as autograd leaves them; torch.optim then skips them).  If an optimizer dropped the
        gradients (zero_grad(set_to_none=True)) the arena is stale -> zero it; a parameter trainable again after being frozen
        starts from a zeroed slice."""
        first = next((p for p, _ in self._views if p.requires_grad), None)
        stale = first is not None and first.grad is None
        if stale:
            self._flat_grad.zero_()
        for p, gv in self._views:
            if not p.requires_grad:
                if p.grad is gv:
                    p.grad = None
            elif p.grad is not gv:
                if p.grad is None and not stale:
                    gv.zero_()
                p.grad = gv

    def zero_grad(self, set_to_none=False):
        if self._flat_grad is not None:
            self._flat_grad.zero_()
            for p, gv in self._views:
                p.grad = gv if p.requires_grad else None
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
        """Gradient buffer of a parameter (its arena slice) in kernel layout."""
        g = p._arena_grad
        return g.permute(0, 2, 3, 1) if p.dim() == 4 else g


class BackwardPlan:
    """What one network backward computes, unit by unit.  A unit is a (conv, BatchNorm) pair, a decoder convolution, a
    disparity head or a pose-head convolution, keyed by id() of its convolution module.  The plan is a pure function of module
    flags -- requires_grad of every parameter and which input images need a gradient -- decided when the forward runs, so
    that the forward knows what to record.

    A gradient w.r.t. an activation is "live" when a trainable parameter or an image needing a gradient lies upstream of it
    (at or below it in backward order).  Per unit:
      runs[u]:    the gradient w.r.t. its output is live: its backward (BatchNorm backward, weight / data gradients) runs;
      dgrad[u]:   the gradient w.r.t. its input is live: its data gradient runs;
      trains(p):  the parameter requires grad: the unit runs the weight (BatchNorm parameter) gradient it belongs to;
      feats[j]:   the gradient w.r.t. encoder feature j (stem output, layers 1-4) is live -- feats[4] False: the encoder has no
                  backward and its forward keeps no record;
      dimg:       one flag per input image (DispResNet 1, PoseResNet 2): its gradient is wanted (the stem's data gradient).
    Which BatchNorm backward a unit uses (O.BN_FROZEN for a module in eval mode) is recorded by the forward with the unit."""

    def __init__(self, net, dimg):
        self.dimg = tuple(bool(n) for n in dimg)
        self.train = {id(p) for p in net.parameters() if p.requires_grad} if torch.is_grad_enabled() else set()
        self.runs, self.dgrad = {}, {}
        t = net.encoder.encoder
        live = self._unit(t.conv1, t.bn1, any(self.dimg))
        self.feats = [live]
        for li in range(1, 5):
            for blk in getattr(t, "layer%d" % li):
                main, ds = blk.units()
                h = live
                for conv, bn, _, _ in main[:-1]:
                    h = self._unit(conv, bn, h)
                sc = live if ds is None else self._unit(ds[0], ds[1], live)
                # the last unit's backward also gates the shortcut's gradient (dres): it runs when the block output is live
                last = self._unit(main[-1][0], main[-1][1], h) or sc
                self.runs[id(main[-1][0])] = last
                live = last
            self.feats.append(live)
        if isinstance(net, DispResNet):
            cur = live
            for i in range(4, -1, -1):
                a = self._unit(net.decoder.up(i, 0), None, cur)
                cur = self._unit(net.decoder.up(i, 1), None, a or (i > 0 and self.feats[i - 1]))
                if i < 4:
                    self._unit(net.decoder.disp(i), None, cur)
        else:
            for conv in net.decoder.net:
                live = self._unit(conv, None, live)
        self.any = any(self.runs.values())       # the backward has anything to do (an image gradient makes every unit run)

    def _unit(self, conv, bn, live_in):
        """Records the unit's flags; returns whether the gradient w.r.t. its output is live."""
        out = live_in or self.trains(conv.weight) or self.trains(conv.bias) or (
            bn is not None and (self.trains(bn.weight) or self.trains(bn.bias)))
        self.runs[id(conv)], self.dgrad[id(conv)] = out, live_in
        return out

    def trains(self, p):
        return p is not None and id(p) in self.train

    def wgrad(self, conv):
        """The unit's convolution runs its weight (and bias) gradient."""
        return self.trains(conv.weight) or self.trains(conv.bias)

    def grad_of(self, p):
        """The arena slice that receives p's gradient when p is trainable, else None (the kernel skips it)."""
        return ArenaNet.g(p) if self.trains(p) else None


class _NetCall(torch.autograd.Function):
    @staticmethod
    def forward(ctx, net, hook, groups, plan, *inputs):
        rec, outs = net._forward_impl(groups, *inputs, plan=plan)
        ctx.net, ctx.rec = net, rec
        ctx.set_materialize_grads(False)     # unused outputs (scales 1-3 with --num-scales 1) arrive as None
        return tuple(outs)

    @staticmethod
    def backward(ctx, *grads):
        net = ctx.net
        need = ctx.needs_input_grad[4:]
        # the plan of the forward (what it recorded follows from it); the BatchNorm formula of every unit follows the mode its
        # module had in the FORWARD (recorded with the unit), not its mode now
        plan = ctx.rec["plan"]
        assert plan.dimg == tuple(bool(n) for n in need)
        dimgs = [None] * len(need)
        if plan.any:
            if plan.train:
                net._attach_grads()
            dimgs = net._backward_impl(ctx.rec, [None if g is None else g.contiguous() for g in grads], plan)
            net.ctx.join_wgrad()       # weight gradients enqueued on the side stream (if any) are part of this backward
        ctx.rec = None
        net._pending -= 1
        if net._pending == 0 and net.grads_ready_callback is not None:
            net.grads_ready_callback(net)
        return (None, None, None, None) + tuple(dimgs)


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


class _Forward:
    """What differs between the forwards of one network call.  Recording (coeffs None): each BatchNorm with batch statistics
    (its module in train mode) or the running ones (eval mode) over `groups` independent sample groups, and every unit whose
    backward runs (plan.runs) returns its record.  Fused (coeffs = ArenaNet.bn_eval_coeffs()): eval-mode BatchNorm in the
    convolution epilogues, no record."""

    def __init__(self, net, groups, fused, plan=None):
        self.cx, self.groups, self.plan = net.ctx, groups, plan
        self.coeffs = net.bn_eval_coeffs() if fused else None

    @property
    def fused(self):
        return self.coeffs is not None


# One conv+BatchNorm unit of the recording forward: its input x, the convolution output y, the unit output z, the
# BatchNorm's saved statistics and the flags of its backward (O.BN_FROZEN when the module was in eval mode).  z is kept only
# where a ReLU follows (the backward reads it for the ReLU's gate), so that the record does not hold the downsample's output
# until the backward.
_Unit = collections.namedtuple("_Unit", "x y z saved bn_flags")


def _conv_bn(f, x, unit, relu, residual=None, with_lo=False, w=None):
    """z = relu?(bn(conv(x)) [+ residual]) for unit (conv, bn, stride, pad); returns (z, its _Unit record or None).
    w: (operand weights, their low part) in place of the unit's own (the padded stem).
    Fused: ONE convolution with BatchNorm, residual, ReLU and TF32 rounding in its epilogue (bitwise conv_fwd followed by
    bn_apply); with_lo: z feeds a tensor-core convolution (tf32x3: write its low part too).
    Recording: BatchNorm statistics, and the running-stat updates, stay per sample group (one per batched network call,
    exactly as in train.py:427-442); bn_apply writes lo(z) in every tf32x3 call."""
    conv, bn, stride, pad = unit
    cx = f.cx
    w, w_lo = (conv.w_op(cx), conv.w_lo(cx)) if w is None else w
    if f.fused:
        sc, sh = f.coeffs[id(bn)]
        z = cx.conv_fwd(x, w, None, stride, pad, O.PAD_ZERO, (O.ACT_RELU if relu else O.ACT_NONE) | cx.rnd(), None, 1, w_lo,
                        bn_scale=sc, bn_shift=sh, addend=residual, with_lo=with_lo and cx.split)
        return z, None
    G = f.groups
    sums = _pool(cx).take(O.BN_SLOTS * G * conv.weight.shape[0] * 2, x.device) if bn.training else None
    y = cx.conv_fwd(x, w, None, stride, pad, O.PAD_ZERO, O.ACT_NONE, sums, G, w_lo)
    z, saved = O.bn_apply(y, sums, bn.weight, bn.bias, bn.running_mean, bn.running_var, BN_MOMENTUM, BN_EPS, residual,
                          (1 if relu else 0) | cx.rnd(), G, cx.split)
    if not f.plan.runs[id(conv)]:
        return z, None
    return z, _Unit(x, y, z if relu else None, saved, 0 if bn.training else O.BN_FROZEN)


def _conv_bn_bwd(cx, dz, unit, r, relu, want_dres, addend, groups, plan):
    """Backward through relu?(bn(conv(x)) [+res]) of `unit` with record `r`; `addend` is added to dx in the data gradient's
    epilogue.  Returns (dx, or None where the plan needs no data gradient; dres or None)."""
    conv, bn, stride, pad = unit
    dy, dres = O.bn_backward(dz, r.z, r.y, r.saved, plan.grad_of(bn.weight), plan.grad_of(bn.bias),
                             (1 if relu else 0) | cx.rnd() | r.bn_flags, want_dres, groups, cx.split)
    if plan.wgrad(conv):
        cx.conv_wgrad(r.x, dy, ArenaNet.g(conv.weight), None, stride, pad, O.PAD_ZERO)
    if not plan.dgrad[id(conv)]:
        return None, dres
    return cx.conv_dgrad(dy, conv.w_op(cx), r.x.shape, stride, pad, addend), dres


def block_forward(f, blk, x):
    """Returns (block output, record: (main-path unit records, downsample record or None); None in the fused forward and
    where the block's backward does not run)."""
    main, ds = blk.units()
    h, recs = x, []
    for unit in main[:-1]:
        h, r = _conv_bn(f, h, unit, True, with_lo=True)
        recs.append(r)
    # the shortcut runs between the main path's first convolution(s) and its last one
    sc, ds_rec = (x, None) if ds is None else _conv_bn(f, x, ds, False)
    out, r = _conv_bn(f, h, main[-1], True, sc, with_lo=True)
    return out, None if f.fused or r is None else (recs + [r], ds_rec)


def block_backward(cx, blk, rec, d_out, d_skip, groups, plan):
    """d_out: gradient w.r.t. the block output (consumed / overwritten).  d_skip: gradient that reaches the block INPUT from
    the decoder (skip connection) or None -- folded into the shortcut's dgrad epilogue.  Returns gradient w.r.t. the block
    input, or None where the plan stops the backward inside this block.  Units whose backward does not run (nothing upstream of
    them trains) are skipped: the main path from its first unit up, the shortcut."""
    main, ds = blk.units()
    recs, ds_rec = rec
    d, dres = _conv_bn_bwd(cx, d_out, main[-1], recs[-1], True, True, None, groups, plan)
    for k in range(len(main) - 2, 0, -1):
        if d is None:                   # main[k] and the units before it do not run
            break
        d, _ = _conv_bn_bwd(cx, d, main[k], recs[k], True, False, None, groups, plan)
    if ds is not None:
        d_sc = _conv_bn_bwd(cx, dres, ds, ds_rec, False, False, d_skip, groups, plan)[0] if plan.runs[id(ds[0])] else None
    else:
        # a skip feature is the output of a layer's last block, and the block after it opens one of layers 2-4: stride 2,
        # so it has a downsample
        assert d_skip is None, "skip-connection gradient at a block without downsample"
        d_sc = dres
    if d is None:
        return None
    dx, _ = _conv_bn_bwd(cx, d, main[0], recs[0], True, False, d_sc, groups, plan)
    return dx


def _stem_operands(cx, conv, imgs):
    """(x_nhwc, w, w_lo) of the 7x7 stem: imgs as in encoder_forward.  On the tensor cores the input channels are
    zero-padded 3 -> 4 / 6 -> 8 (K = 49 * Cpad) and the weights likewise; in fp32 mode the plain NHWC input and the
    unit's own weights."""
    if not cx.tc:
        return O.nchw_to_nhwc(imgs[0], imgs[1] if len(imgs) > 1 else None), conv.w_op(cx), conv.w_lo(cx)
    cpad = 4 * len(imgs)
    x_nhwc = O.nchw_to_nhwc_pad(imgs[0], imgs[1] if len(imgs) > 1 else None, cpad, cx.operand)
    w = O.pad_channels(conv.w_khwc(), cpad, cx.operand)
    w_lo = O.pad_channels(conv.w_khwc(), cpad, O.OPERAND_LO) if cx.split else None
    return x_nhwc, w, w_lo


def encoder_forward(f, enc, imgs):
    """imgs: tuple of one (DispResNet) or two (PoseResNet, channel-concatenated) NCHW image batches.
    Returns (record, or None in the fused forward and where the plan gives the encoder no backward; the five features)."""
    t = enc.encoder
    G = f.groups
    if not f.fused:
        _count_batches(f, enc, imgs[0].device)
    x_nhwc, w0, w0_lo = _stem_operands(f.cx, t.conv1, imgs)
    f0, stem = _conv_bn(f, x_nhwc, (t.conv1, t.bn1, 2, 3), True, w=(w0, w0_lo))
    del x_nhwc, w0, w0_lo              # dead in the fused forward (the record keeps the stem's input for the backward)
    x, pool_idx = O.maxpool_fwd(f0)
    feats, blocks = [f0], []
    for li in range(1, 5):
        for blk in getattr(t, "layer%d" % li):
            x, r = block_forward(f, blk, x)
            blocks.append((blk, r))
        feats.append(x)
    if f.fused or not f.plan.feats[4]:
        return None, feats
    return {"G": G, "stem": stem, "pool_idx": pool_idx, "blocks": blocks}, feats


def _count_batches(f, enc, device):
    """Recording forward: readies the BatchNorm-sums pool when any module uses batch statistics, and adds the call's group
    count to num_batches_tracked of every BatchNorm in train mode -- one add over the views of the encoder's one int64
    tensor; with some modules in eval mode the increment is a cached per-module tensor, so the add stays capturable in a CUDA
    graph."""
    G, bns = f.groups, enc._nbt_bns
    modes = tuple(bn.training for bn in bns)
    if not any(modes):
        return
    _pool(f.cx).begin(device)
    if all(modes):
        enc._nbt.add_(G)
        return
    key = (modes, G)
    inc = enc._nbt_inc.get(key)
    if inc is None:
        inc = enc._nbt_inc[key] = torch.tensor([G if m else 0 for m in modes], dtype=torch.long).to(enc._nbt.device)
    enc._nbt.add_(inc)


def encoder_backward(cx, enc, rec, d_feats, plan):
    """d_feats[i]: gradient w.r.t. feature i coming from the decoder (None if unused).  d_feats[4] is required.
    Returns the gradients of the input images (NCHW, one per image of the forward; None where plan.dimg does not ask).
    The backward stops where nothing upstream trains (plan.runs): the blocks before that point, and the stem, do not run."""
    t = enc.encoder
    blocks, G = rec["blocks"], rec["G"]
    # index of the last block of each layer -> the feature it produces
    ends, k = {}, 0
    for li in range(1, 5):
        k += len(getattr(t, "layer%d" % li))
        ends[k - 1] = li
    d = d_feats[4]
    for bi in range(len(blocks) - 1, -1, -1):
        blk, r = blocks[bi]
        if d is None:
            return [None] * len(plan.dimg)
        # the INPUT of block bi is the output of block bi-1; if that is a skip feature, add the decoder's gradient
        extra = None
        if bi - 1 in ends and d_feats[ends[bi - 1]] is not None:
            extra = d_feats[ends[bi - 1]]
        d = block_backward(cx, blk, r, d, extra, G, plan)
    if d is None:
        return [None] * len(plan.dimg)
    # d is now the gradient w.r.t. the max-pool output
    stem = rec["stem"]
    f0, x = stem.z, stem.x
    if d_feats[0] is not None:
        d_f0 = d_feats[0]
        O.maxpool_bwd(d, rec["pool_idx"], f0.shape, d_f0, True)
    else:
        d_f0 = torch.empty_like(f0)
        O.maxpool_bwd(d, rec["pool_idx"], f0.shape, d_f0, False)
    # lo(dy) could only be read by the stem's weight gradient (its data gradient, stem_dgrad, is exact fp32), and the TMA
    # weight-gradient kernel computes it itself
    w_shape = (t.conv1.weight.shape[0], t.conv1.k, t.conv1.k, x.shape[-1])
    wgrad = plan.wgrad(t.conv1)
    dy, _ = O.bn_backward(d_f0, f0, stem.y, stem.saved, plan.grad_of(t.bn1.weight), plan.grad_of(t.bn1.bias),
                          1 | cx.rnd() | stem.bn_flags, False, G, wgrad and cx.wgrad_reads_lo(x.shape, w_shape, 2, 3))
    if wgrad:
        if x.shape[-1] != t.conv1.weight.shape[1]:
            # padded-channel stem (tensor-core modes): weight gradient in the padded layout, then folded into the gradient arena
            dw = torch.zeros(t.conv1.weight.shape[0], t.conv1.k, t.conv1.k, x.shape[-1], device=x.device, dtype=torch.float32)
            cx.conv_wgrad(x, dy, dw, None, 2, 3, O.PAD_ZERO)
            with cx.on_wgrad_stream([dw]):
                O.unpad_add_(ArenaNet.g(t.conv1.weight), dw)
        else:
            cx.conv_wgrad(x, dy, ArenaNet.g(t.conv1.weight), None, 2, 3, O.PAD_ZERO)
    if not any(plan.dimg):
        return [None] * len(plan.dimg)
    # input images: the transposed stem convolution with the fp32 weights (not the padded / TF32 operand copies)
    return O.stem_dgrad(dy, t.conv1.w_khwc(), x.shape[1], x.shape[2], plan.dimg)


# ------------------------------------------------------------------------------------------------
# networks
# ------------------------------------------------------------------------------------------------
def _disp_side_ok(n, training_step):
    """Whether DispResNet takes an image side of n pixels.  Its encoder planes are ceil(n/2), ceil(n/4), ..., ceil(n/32), and
    each decoder stage concatenates its x2 upsampled plane with the encoder plane one level up, so ceil(n/2) is a multiple
    of 16; the first stage reflection-pads the ceil(n/32) plane by one, which needs 2 pixels: n = 0 or 31 mod 32, n >= 63,
    the sizes the reference's module runs on.  A training step also needs the disparity (2 ceil(n/2)) at the image's size:
    n a multiple of 32, n >= 64."""
    if training_step:
        return n % 32 == 0 and n >= 64
    h = (n + 1) // 2
    return h % 16 == 0 and h >= 32


def check_image_size(H, W, training_step=False):
    """Raises ValueError, naming the nearest accepted sizes, unless DispResNet takes an H x W image (its disparity is then
    2 ceil(H/2) x 2 ceil(W/2)); training_step: unless a training step takes it (_disp_side_ok)."""
    if _disp_side_ok(H, training_step) and _disp_side_ok(W, training_step):
        return

    def near(n):
        if _disp_side_ok(n, training_step):
            return [n]
        lo = next((m for m in range(n - 1, 0, -1) if _disp_side_ok(m, training_step)), None)
        hi = next(m for m in range(n + 1, n + 65) if _disp_side_ok(m, training_step))
        return [m for m in (lo, hi) if m is not None]
    sizes = sorted(((h, w) for h in near(H) for w in near(W)), key=lambda s: (abs(s[0] - H) + abs(s[1] - W), s))
    rule = ("a training step takes H and W that are multiples of 32, at least 64" if training_step else
            "DispResNet takes H and W = 0 or 31 mod 32, at least 63")
    raise ValueError("image size %dx%d: %s (nearest accepted sizes: %s)"
                     % (H, W, rule, ", ".join("%dx%d" % s for s in sizes[:4])))


class DispResNet(ArenaNet):
    """models.DispResNet(num_layers=18, pretrained=True) (reference DispResNet.py:104-121)."""

    def __init__(self, num_layers=18, pretrained=True):
        super().__init__()
        self.encoder = ResnetEncoder(num_layers=num_layers, pretrained=pretrained, num_input_images=1)
        self.decoder = DepthDecoder(self.encoder.num_ch_enc)

    def init_weights(self):
        pass

    def forward(self, x):
        check_image_size(x.shape[-2], x.shape[-1])
        outs = self._call((x,))
        return list(outs) if self.training else outs[0]

    def forward_multi(self, images):
        """Several independent network calls in ONE launch sequence: `images` is a list of [B,3,H,W] tensors;
        returns one output per image, each exactly what `self(image)` would return.  The calls are stacked on
        the batch axis (more rows per GEMM, 1/len(images) of the kernel launches) while BatchNorm statistics
        and running-stat updates stay per call, in list order (train.py:427-434 semantics)."""
        for x in images:
            check_image_size(x.shape[-2], x.shape[-1])
        per = self._call((torch.cat(list(images), 0),), len(images))
        return per if self.training else [p[0] for p in per]

    # -- forward ------------------------------------------------------------------------------
    def _forward_impl(self, groups, x, fused=False, plan=None):
        """fused (eval mode, autograd off): no record, BatchNorm in the convolution epilogues; returns (None, outputs).
        Recording: plan (BackwardPlan) says which units' backward will run."""
        from . import lib as L
        x = L.dev_f32(x, "DispResNet input")
        self.refresh_operand_weights()
        training = self.training
        cx = self.ctx
        enc_rec, feats = self._encoder_forward(groups, (x,), fused, plan)
        dec = self.decoder
        rec = {"enc": enc_rec, "stages": {}, "plan": plan}
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
    def _backward_impl(self, rec, grads, plan):
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
            c1, c0 = dec.up(i, 1), dec.up(i, 0)
            live = plan.runs[id(c1)]        # the gradient w.r.t. b is needed (pending is set only then)
            have = pending is not None
            d_b, pending = pending, None
            if i in d_disp and (live or plan.wgrad(dec.disp(i))):
                dc = dec.disp(i)
                disp = rec["disps"][i]
                dpre = O.act_bwd_(d_disp[i].reshape(disp.shape).clone(), disp, O.ACT_DISP)
                if plan.wgrad(dc):
                    O.head_wgrad(b, dpre, g(dc.weight), g(dc.bias))
                if not live:
                    continue
                dpad = O.head_dgrad(dpre, dc.w_khwc(), b.shape)
                if not have:
                    d_b = torch.empty_like(b)
                O.fold_plain(dpad, d_b, b, O.ACT_ELU | cx.rnd(), accumulate=have)
            elif have:
                O.act_bwd_(d_b, b, O.ACT_ELU | cx.rnd())
            else:
                continue            # nothing reaches this stage, or nothing upstream of it trains
            # up(i,1): b = ELU(conv(reflect_pad(cat)))
            if plan.wgrad(c1):
                cx.conv_wgrad(st["cat"], d_b, g(c1.weight), plan.grad_of(c1.bias), 1, 1, O.PAD_REFLECT)
            if not plan.dgrad[id(c1)]:
                continue
            dpad = cx.conv_dgrad(d_b, c1.w_op(cx), st["cat"].shape, 1, 1, None, padded_input=True)
            d_a, d_skip = O.fold_upcat(dpad, st["a"].shape[-1], st["a"], O.ACT_ELU | cx.rnd(), with_skip=i > 0 and plan.feats[i - 1])
            if i > 0:
                d_feats[i - 1] = d_skip
            # up(i,0): a = ELU(conv(reflect_pad(in0)))
            if plan.wgrad(c0):
                cx.conv_wgrad(st["in0"], d_a, g(c0.weight), plan.grad_of(c0.bias), 1, 1, O.PAD_REFLECT)
            if not plan.dgrad[id(c0)]:
                continue
            dpad = cx.conv_dgrad(d_a, c0.w_op(cx), st["in0"].shape, 1, 1, None, padded_input=True)
            d_in = torch.empty_like(st["in0"])
            O.fold_plain(dpad, d_in, None, O.ACT_NONE, accumulate=False)
            if i < 4:
                pending = d_in          # = raw gradient of b_{i+1}; ELU' applied once all consumers are in
            else:
                d_feats[4] = d_in
        if not plan.feats[4]:
            return [None] * len(plan.dimg)
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
        return self._call((img1, img2))[0]

    def forward_multi(self, pairs):
        """`pairs` = list of (img1, img2); one stacked launch sequence, BatchNorm per call (see DispResNet.forward_multi).
        Returns the list of [B,6] poses."""
        per = self._call((torch.cat([a for a, _ in pairs], 0), torch.cat([b for _, b in pairs], 0)), len(pairs))
        return [p[0] for p in per]

    def _forward_impl(self, groups, img1, img2, fused=False, plan=None):
        """fused (eval mode, autograd off): no record, BatchNorm in the convolution epilogues; returns (None, outputs).
        Recording: plan (BackwardPlan) says which units' backward will run."""
        from . import lib as L
        img1, img2 = L.dev_f32(img1, "PoseResNet input"), L.dev_f32(img2, "PoseResNet input")
        self.refresh_operand_weights()
        cx = self.ctx
        enc_rec, feats = self._encoder_forward(groups, (img1, img2), fused, plan)
        x = feats[4]
        del feats                       # the fused forward frees f0-f3 here
        head = None if fused else [x]   # recording: the input of every head convolution, then the head's output
        for k, (pad, _) in enumerate(POSE_HEAD):
            conv = self.decoder.net[k]
            # (fused, tf32x3: the inputs of the two 3x3 convolutions are written with their low part; the last convolution,
            # 256 -> 6 channels, runs on the CUDA cores and reads none)
            x = cx.conv_fwd(x, conv.w_op(cx), conv.bias, 1, pad, O.PAD_ZERO, _pose_act(cx, k), None, 1, conv.w_lo(cx),
                            with_lo=fused and cx.split and k < 2)
            if head is not None:
                head.append(x)
        rec = None if fused else {"enc": enc_rec, "head": head, "plan": plan}
        return rec, [O.spatial_mean_fwd(x, 0.01)]

    def _backward_impl(self, rec, grads, plan):
        """Returns [gradient of img1 or None, gradient of img2 or None] (see encoder_backward)."""
        cx = self.ctx
        head = rec["head"]
        d = O.spatial_mean_bwd(grads[0], head[-1].shape, 0.01)
        for k in range(len(POSE_HEAD) - 1, -1, -1):
            conv, pad, inp = self.decoder.net[k], POSE_HEAD[k][0], head[k]
            if plan.wgrad(conv):
                cx.conv_wgrad(inp, d, ArenaNet.g(conv.weight), plan.grad_of(conv.bias), 1, pad, O.PAD_ZERO)
            if not plan.dgrad[id(conv)]:
                return [None] * len(plan.dimg)
            d = cx.conv_dgrad(d, conv.w_op(cx), inp.shape, 1, pad)
            if k > 0:
                O.act_bwd_(d, inp, _pose_act(cx, k - 1))       # inp is the output of convolution k - 1
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
    training step can be captured in a CUDA graph.  Frozen parameters (requires_grad False, whose .grad the networks keep
    None) are skipped as torch.optim.Adam skips them: a network with any of them is updated by the masked kernel, which does
    not touch their values, moments or operand mirror, weight decay included."""

    def __init__(self, nets, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        self.nets = list(nets)
        self.lr, self.betas, self.eps, self.weight_decay = lr, betas, eps, weight_decay
        self.state = {}
        self._step = None
        self._masks = {}           # id(net) -> (arena, requires_grad pattern, chunk mask on the device)

    def _chunk_mask(self, n):
        """None when every parameter of network n is trainable, else its adam_step_masked chunk mask (rebuilt when the
        pattern or the arena changes; the warm-up step before a CUDA-graph capture builds it)."""
        flags = tuple(p.requires_grad for p, _ in n._views)
        if all(flags):
            return None
        hit = self._masks.get(id(n))
        if hit is None or hit[0] is not n._flat or hit[1] != flags:
            hit = self._masks[id(n)] = (n._flat, flags, O.chunk_mask([p.numel() for p, _ in n._views], flags, n._flat.device))
        return hit[2]

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
            operand = O.OPERAND_LO if n.ctx.split else O.OPERAND_TF32
            mask = self._chunk_mask(n)
            if mask is None:
                O.adam_step(n._flat, n._flat_grad, m, v, self.lr, self.betas[0], self.betas[1], self.eps, self.weight_decay,
                            0, self._step, mirror, operand)
            else:
                O.adam_step_masked(n._flat, n._flat_grad, m, v, mask, self.lr, self.betas[0], self.betas[1], self.eps,
                                   self.weight_decay, 0, self._step, mirror, operand)
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

    def load_state_dict(self, sd):
        """Load what state_dict() returns, in place: the moments and the device step counter keep their addresses (a captured
        step and the camera's Adam hold them).  A different number of networks, or a moment arena whose length is not its
        network's parameter arena's, raises ValueError before anything is copied."""
        self._ensure_state()
        for what in ("exp_avg", "exp_avg_sq"):
            if len(sd[what]) != len(self.nets):
                raise ValueError("optimizer state: %s holds %d networks, this ArenaAdam updates %d"
                                 % (what, len(sd[what]), len(self.nets)))
            for i, (n, src) in enumerate(zip(self.nets, sd[what])):
                if tuple(src.shape) != tuple(n._flat.shape):
                    raise ValueError("optimizer state: %s of network %d (%s) has shape %s, its parameter arena %s"
                                     % (what, i, type(n).__name__, tuple(src.shape), tuple(n._flat.shape)))
        for n, m0, v0 in zip(self.nets, sd["exp_avg"], sd["exp_avg_sq"]):
            m, v, _ = self.state[id(n)]
            m.copy_(m0)
            v.copy_(v0)
        self._step.fill_(int(sd["step"]))
