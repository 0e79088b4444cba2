"""The memory-bound network kernels one by one against fp64 references: TF32 operand helpers, layout / stem operands,
BatchNorm, max-pool, upsample+concat and the reflection-pad folds, activation gradients, the disparity and pose heads and
Adam (csrc/nn_ops.cu, csrc/heads.cu).  Needs a GPU.

Every kernel is called through the scsfm.nnops wrappers the networks use.  Inputs are built on the CPU, rounded to fp32,
and the fp64 reference is computed from those fp32 values, so the only differences left are the kernel's own fp32
rounding.  Bounds are therefore fp32-noise bounds: bitwise for copies and operand rounding, otherwise <= 1e-5 relative
(the reason for each is next to it).  `_close` checks every element against the largest magnitude of the reference and
the relative L2 error against the same bound.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import Adam64, assert_adam_change, rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda"
GRID_STRIDE = 132 * 32 * 256      # elements beyond which the elementwise kernels' capped grid has to stride


def _ops():
    from scsfm import nnops
    return nnops


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def f32(v):
    """A scalar as the kernels receive it (a C float)."""
    return float(np.float32(v))


def _np(t):
    return t.detach().float().cpu().numpy()


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _same_bits(got, want, what=""):
    g, w = _bits(_np(got) if torch.is_tensor(got) else got), _bits(_np(want) if torch.is_tensor(want) else want)
    bad = np.flatnonzero(g.ravel() != w.ravel())
    assert g.shape == w.shape and bad.size == 0, "%s: %d elements differ, first at %s: %08x != %08x" % (
        what, bad.size, bad[:1], g.ravel()[bad[0]] if bad.size else 0, w.ravel()[bad[0]] if bad.size else 0)


def _close(got, want, tol, what=""):
    got = torch.as_tensor(got).detach().double().cpu()
    want = torch.as_tensor(want).detach().double().cpu()
    assert got.shape == want.shape, (what, got.shape, want.shape)
    err, scale = float((got - want).abs().max()), float(want.abs().max())
    assert err <= tol * scale, "%s: max error %.3g > %g * max|ref| (%.3g)" % (what, err, tol, scale)
    assert rel_l2(got, want) <= tol, "%s: rel-L2 %.3g > %g" % (what, rel_l2(got, want), tol)


def _tf32_close(got, want, tol, what=""):
    """A TF32-rounded result: low 13 bits clear and within half a TF32 ulp (2^-11 relative) of the reference, plus the fp32
    noise `tol` of the unrounded computation."""
    g = _np(got)
    assert not (_bits(g) & 0x1FFF).any(), what + ": not a TF32 value"
    w = torch.as_tensor(want).detach().double().cpu().numpy()
    assert (np.abs(g - w) <= 2.0 ** -11 * np.abs(w) + tol * np.abs(w).max()).all(), what


def nh(t):
    """NCHW (CPU, any dtype) -> NHWC fp32 on the device."""
    return t.detach().float().permute(0, 2, 3, 1).contiguous().to(DEV)


def nc(t):
    """NHWC device tensor -> NCHW fp64 on the CPU."""
    return t.detach().permute(0, 3, 1, 2).double().cpu()


# ----- reference of the TF32 operand helpers ----------------------------------------------------------------
def rna_tf32(x):
    """cvt.rna.tf32.f32 on finite fp32 values: round to nearest with ties away from zero, low 13 bits cleared.  Adding
    half a TF32 ulp to the magnitude bits rounds the magnitude half-up (sign-magnitude format), carrying into the exponent."""
    u = _bits(x).astype(np.uint64)
    return ((u + 0x1000) & 0xFFFFE000).astype(np.uint32).view(np.float32)


def lo_tf32(x):
    """Low part of a split-accumulate operand: rna(x - trunc13(x)); the subtraction is exact in fp32."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    hi = (_bits(x) & np.uint32(0xFFFFE000)).view(np.float32)
    return rna_tf32(x - hi)


# bit patterns where rounding goes wrong: +-0, denormals (incl. ties and a round-up into the smallest normal), exact ties
# (low 13 bits = 0x1000) with even and odd kept bit, just below / above a tie, a tie that carries into the exponent
_TF32_SPECIAL = np.array([0x00000000, 0x80000000, 0x00000001, 0x80000FFF, 0x00001000, 0x00003000, 0x807FF000, 0x007FFFFF,
                          0x3F800FFF, 0x3F801001, 0xBF803000, 0x3FFFF000, 0x4B7FF000, 0x00FFF000, 0x3F801000, 0xBF801000],
                         dtype=np.uint32)


def _tf32_values(n, seed):
    rng = np.random.default_rng(seed)
    exp = rng.integers(0, 254, n, dtype=np.uint32)          # denormals .. 2^126: rounding never overflows to inf
    bits = (rng.integers(0, 2, n, dtype=np.uint32) << 31) | (exp << 23) | rng.integers(0, 1 << 23, n, dtype=np.uint32)
    bits[::7] = (bits[::7] & np.uint32(0xFFFFE000)) | np.uint32(0x1000)          # many exact ties
    k = min(n, _TF32_SPECIAL.size)
    bits[n - k:] = _TF32_SPECIAL[_TF32_SPECIAL.size - k:]                          # the tail (n % 4 != 0) gets the edge cases
    if n > 2 * k:
        bits[:k] = _TF32_SPECIAL[:k]
    return bits.view(np.float32)


@pytest.mark.parametrize("n", [1, 3, 5, 1027, 4 * GRID_STRIDE + 4099])
def test_round_and_split_tf32_bitwise(n):
    """round_tf32 / split_tf32 against the bit-level reference; n % 4 != 0 runs split_tf32's scalar tail, the largest n
    the grid-stride loops of both.  Exact: the hardware conversion is specified bit for bit."""
    O = _ops()
    x = _tf32_values(n, n)
    xc = torch.from_numpy(x.copy()).to(DEV)
    out = torch.full_like(xc, float("nan"))          # sentinel: an element the kernel skips stays NaN
    O.round_tf32(xc, out)
    _same_bits(out, rna_tf32(x), "round_tf32")
    lo = torch.full_like(xc, float("nan"))
    O.split_tf32(xc, lo)
    _same_bits(lo, lo_tf32(x), "split_tf32")
    # hi + lo reproduces x to 2^-21 relative (the split-accumulate premise), wherever the remainder is not denormal
    hi = (_bits(x) & np.uint32(0xFFFFE000)).view(np.float32).astype(np.float64)
    big = np.abs(x) >= 2.0 ** -100
    assert (np.abs(hi + _np(lo).astype(np.float64) - x) <= 2.0 ** -21 * np.abs(x))[big].all()


def _flip_ref(w, stride, pad, operand):
    """Flipped weights of the data gradient restated: w [Cout,kh,kw,Cin] -> [Cin,kh,kw,Cout] with reversed taps at stride 1;
    at stride 2 the four output-parity classes (py, px) back to back, class (py, px) holding the kernel rows dy with
    py + pad - dy even (and columns likewise), each from the last one down, in the same layout."""
    w = {0: rna_tf32, 1: lambda a: a, 2: lo_tf32}[operand](w)
    kh, kw = w.shape[1:3]
    if stride == 1:
        return np.ascontiguousarray(w[:, ::-1, ::-1].transpose(3, 1, 2, 0)).ravel()
    parts = []
    for py in range(2):
        for px in range(2):
            rows = [dy for dy in range(kh - 1, -1, -1) if (py + pad - dy) % 2 == 0]
            cols = [dx for dx in range(kw - 1, -1, -1) if (px + pad - dx) % 2 == 0]
            parts.append(w[:, rows][:, :, cols].transpose(3, 1, 2, 0).ravel())
    return np.concatenate(parts)


def test_weight_flips_match_their_restatement():
    """Every flipped layout bit for bit: strides 1 and 2, k = 1, 3, 7, pad 0, 1, 3, the three operand kinds, from the first
    flip (one launch per weight) and from the batched refresh of all of them (one launch) after the weights changed.
    Cout and Cin are not multiples of the 32 x 32 tiles."""
    O = _ops()
    cx = O.ConvCtx("tf32x3")
    g = torch.Generator().manual_seed(3)
    cases = [(s, k, pad, op) for s in (1, 2) for k in (1, 3, 7) for pad in (0, 1, 3) for op in (0, 1, 2)]
    ws = {k: torch.randn(40, k, k, 36, generator=g).to(DEV) for k in (1, 3, 7)}
    got = {c: cx.flipped_weights(ws[c[1]], c[0], c[2], c[3]) for c in cases}
    for rnd in range(2):
        torch.cuda.synchronize()
        for (s, k, pad, op), wt in got.items():
            want = _flip_ref(ws[k].cpu().numpy(), s, pad, op)
            assert wt.shape == (36, k, k, 40)
            _same_bits(wt.flatten(), want, "flip s%d k%d pad%d operand %d %s" % (s, k, pad, op, ("first", "refresh")[rnd]))
        for w in ws.values():
            w.copy_(torch.randn(w.shape, generator=g))
        cx.refresh_flips(DEV)
    assert len(cx._flips) == len(cases) and cx._table.n_rows == len(cases)


def test_split_tf32_refuses_unaligned_buffers():
    """split_tf32 reads and writes float4: a buffer offset by one float is refused before any launch."""
    from scsfm import lib as L
    O = _ops()
    buf = torch.arange(64, dtype=torch.float32, device=DEV)
    out = torch.full((64,), float("nan"), device=DEV)
    before = L.launch_count()
    with pytest.raises(ValueError, match="16-byte aligned"):
        O.split_tf32(buf[1:33], out[:32])
    with pytest.raises(ValueError, match="16-byte aligned"):
        O.split_tf32(buf[:32], out[1:33])
    torch.cuda.synchronize()
    assert L.launch_count() == before
    assert bool(torch.isnan(out).all())


# ----- layout and stem operands ----------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(1, 3, 2, 2), (2, 3, 37, 61), (4, 3, 256, 832)])
def test_layout_copies_bitwise(shape):
    O = _ops()
    g = _gen(1)
    a, b = torch.randn(shape, generator=g), torch.randn(shape, generator=g)
    ad, bd = a.to(DEV), b.to(DEV)
    _same_bits(O.nchw_to_nhwc(ad), a.permute(0, 2, 3, 1), "nchw_to_nhwc, one source")
    _same_bits(O.nchw_to_nhwc(ad, bd), torch.cat([a, b], 1).permute(0, 2, 3, 1), "nchw_to_nhwc, two sources")
    for C in (1, 3, 16):
        x = torch.randn(shape[0], shape[2], shape[3], C, generator=g)
        _same_bits(O.nhwc_to_nchw(x.to(DEV)), x.permute(0, 3, 1, 2), "nhwc_to_nchw C=%d" % C)


_OPERAND_REF = {0: rna_tf32, 1: lambda x: np.asarray(x, np.float32), 2: lo_tf32}      # SCSFM_OPERAND_TF32 / RAW / LO


@pytest.mark.parametrize("operand", [0, 1, 2])
def test_stem_operands_bitwise(operand):
    """Padded stem input (C=3 -> 4, two images 6 -> 8) and padded stem weights, as each operand kind; pad channels are +0."""
    O = _ops()
    g = _gen(2)
    ref = _OPERAND_REF[operand]
    for nsrc, Cpad in ((1, 4), (2, 8)):
        a, b = torch.randn(2, 3, 19, 26, generator=g), torch.randn(2, 3, 19, 26, generator=g)
        srcs = torch.cat([a, b], 1) if nsrc == 2 else a
        out = O.nchw_to_nhwc_pad(a.to(DEV), b.to(DEV) if nsrc == 2 else None, Cpad, operand)
        want = np.zeros((2, 19, 26, Cpad), np.float32)
        want[..., :3 * nsrc] = ref(srcs.permute(0, 2, 3, 1).numpy())
        _same_bits(out, want, "nchw_to_nhwc_pad x%d" % nsrc)
    for C, Cpad in ((3, 4), (6, 8)):
        w = torch.randn(64, 7, 7, C, generator=g) * 0.05
        out = O.pad_channels(w.to(DEV), Cpad, operand)
        want = np.zeros((64, 7, 7, Cpad), np.float32)
        want[..., :C] = ref(w.numpy())
        _same_bits(out, want, "pad_channels %d -> %d" % (C, Cpad))


def test_unpad_add_accumulates_and_stays_in_bounds():
    """dst += src[..., :C]: one fp32 add per element (bitwise), the pad channels of src are not read into dst, and the
    memory after dst is not written."""
    O = _ops()
    g = _gen(3)
    for C, Cpad in ((3, 4), (6, 8)):
        n = 64 * 7 * 7 * C
        arena = torch.randn(n + 37, generator=g)
        src = torch.randn(64, 7, 7, Cpad, generator=g)
        src[..., C:] = 1e30                                       # would show up if the pad channels were added
        dev = arena.to(DEV)
        O.unpad_add_(dev[:n].view(64, 7, 7, C), src.to(DEV))
        want = arena.clone()
        want[:n] = (arena[:n].view(64, 7, 7, C) + src[..., :C]).reshape(-1)
        _same_bits(dev, want, "unpad_add_ %d/%d" % (C, Cpad))


# ----- BatchNorm ----------------------------------------------------------------------------------------------------
BN_EPS, BN_MOM = f32(1e-5), f32(0.1)        # as the kernels receive them
BN_CASES = [
    # C, groups, rows per group, relu, residual, ROUND_TF32, with_lo
    (64, 1, 100_003, True, True, False, True),       # many row chunks; rows_per_cta does not divide the rows
    (64, 4, 25_013, True, False, True, False),
    (64, 3, 5, True, False, False, False),           # fewer rows than row lanes
    (128, 3, 7, False, True, False, False),
    (256, 3, 20_011, False, False, False, True),
    (256, 4, 3, True, True, True, False),
    (512, 4, 832, True, True, False, True),          # ResNet-18 layer4 at 256x832, B=4 per network call
    (1024, 3, 3328, True, False, True, False),       # ResNet-50 layer3
    (2048, 4, 832, False, False, False, True),       # ResNet-50 layer4 downsample: two channel slabs, no ReLU
    (2048, 1, 832, True, True, True, False),
    (1028, 3, 97, True, True, False, True),          # a partial second slab (1028 / 4 = 257 float4 columns)
    (1028, 1, 4, False, False, True, False),
]


def _bn_sums(y64, G, C, slots):
    """The fused sums the convolution epilogue leaves: per group and channel {sum y, sum y^2} in fp64, spread over `slots`
    replicas (row r of a group lands in slot r % slots)."""
    R = y64.shape[0] // G
    slot = torch.arange(R) % slots
    sums = torch.zeros(slots, G, C, 2, dtype=torch.float64)
    for g in range(G):
        yg = y64[g * R:(g + 1) * R]
        sums[:, g, :, 0] = torch.zeros(slots, C, dtype=torch.float64).index_add_(0, slot, yg)
        sums[:, g, :, 1] = torch.zeros(slots, C, dtype=torch.float64).index_add_(0, slot, yg * yg)
    return sums


def _bn_saved_ref(y64, G, gamma, beta):
    R = y64.shape[0] // G
    out = []
    for g in range(G):
        yg = y64[g * R:(g + 1) * R]
        mean, var = yg.mean(0), yg.var(0, unbiased=False)
        invstd = 1.0 / torch.sqrt(var + BN_EPS)
        out.append(torch.stack([gamma * invstd, beta - mean * gamma * invstd, mean, invstd], 1))
    return torch.stack(out)


@pytest.mark.parametrize("case", BN_CASES, ids=lambda c: "C%d_G%d_R%d_relu%d_res%d_rnd%d_lo%d" % c)
def test_batchnorm_vs_fp64(case):
    O = _ops()
    C, G, R, relu, residual, rnd, with_lo = case
    g = _gen(C + G + R)
    rows = G * R
    # per-channel offsets and spreads, per-group drift: the statistics differ per channel and per group
    y = (torch.randn(rows, C, generator=g) * (0.5 + torch.rand(C, generator=g)) + torch.randn(C, generator=g)
         + 0.3 * torch.randn(G, 1, C, generator=g).repeat_interleave(R, 0).view(rows, C)).float()
    res = torch.randn(rows, C, generator=g).float() if residual else None
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).float()
    beta = (0.2 * torch.randn(C, generator=g)).float()
    rm0, rv0 = (0.1 * torch.randn(C, generator=g)).float(), (0.5 + torch.rand(C, generator=g)).float()
    dz = torch.randn(rows, C, generator=g).float()
    dg0, db0 = torch.randn(C, generator=g).float(), torch.randn(C, generator=g).float()

    # fp64 reference: F.batch_norm per group, G sequential calls updating the running statistics (nn.BatchNorm2d)
    y64 = y.double().requires_grad_(True)
    gm64, bt64 = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    rm, rv = rm0.double(), rv0.double()
    pre = torch.cat([F.batch_norm(y64[i * R:(i + 1) * R], rm, rv, gm64, bt64, True, BN_MOM, BN_EPS) for i in range(G)])
    if residual:
        pre = pre + res.double()
    z_ref = F.relu(pre) if relu else pre
    saved_ref = _bn_saved_ref(y64.detach(), G, gm64.detach(), bt64.detach())

    flags = (1 if relu else 0) | (O.ROUND_TF32 if rnd else 0)
    sums = _bn_sums(y.double(), G, C, O.BN_SLOTS).to(DEV)
    yc, rc, gc, bc = y.to(DEV), res.to(DEV) if residual else None, gamma.to(DEV), beta.to(DEV)
    rmc, rvc = rm0.to(DEV), rv0.to(DEV)
    z, saved = O.bn_apply(yc, sums, gc, bc, rmc, rvc, BN_MOM, BN_EPS, rc, flags, G, with_lo)
    # z: one fma + one add per element after fp32 scale / shift (2e-6 covers the rounding of shift = beta - mean*scale)
    z_plain = z
    if rnd:
        # the same call without rounding: the rounded output is exactly rna() of it (the rounding is the last operation)
        z_plain, _ = O.bn_apply(yc, sums, gc, bc, rm0.to(DEV), rv0.to(DEV), BN_MOM, BN_EPS, rc, flags & ~O.ROUND_TF32, G)
        _same_bits(z, rna_tf32(_np(z_plain)), "z = rna(z unrounded)")
        _tf32_close(z, z_ref, 2e-6, "z (TF32)")
    _close(z_plain, z_ref, 2e-6, "z")
    # saved {scale, shift, mean, invstd}: fp32 values of fp64 statistics, a few roundings
    for k, name in enumerate(("scale", "shift", "mean", "invstd")):
        _close(saved[..., k], saved_ref[..., k], 1e-6, "saved " + name)
    # running statistics: G fp32 updates of the same formula (1e-6: a few roundings per update)
    _close(rmc, rm, 1e-6, "running mean")
    _close(rvc, rv, 1e-6, "running var")
    if with_lo:
        _same_bits(z._scsfm_lo, lo_tf32(_np(z)), "lo(z)")

    # bn_prepare (in the ABI, not used by the networks) computes the same statistics as bn_apply
    rmp, rvp = rm0.to(DEV), rv0.to(DEV)
    saved_p = O.bn_prepare(sums, G, R, gc, bc, rmp, rvp, BN_MOM, BN_EPS, True)
    for k, name in enumerate(("scale", "shift", "mean", "invstd")):
        _close(saved_p[..., k], saved_ref[..., k], 1e-6, "bn_prepare saved " + name)
    _close(rmp, rm, 1e-6, "bn_prepare running mean")
    _close(rvp, rv, 1e-6, "bn_prepare running var")

    # backward.  The ReLU gate is the kernel's own z: closed where z is exactly 0 (PyTorch's ReLU backward passes the
    # gradient only where the output is > 0), so a pre-activation within fp32 noise of 0 cannot flip it in one of the two.
    gate = z.cpu() > 0 if relu else torch.ones(rows, C, dtype=torch.bool)
    dpre = torch.where(gate, dz.double(), 0.0)          # +0 where closed, as the kernel writes it
    pre.backward(dpre)
    dzc = dz.to(DEV)
    dgc, dbc = dg0.to(DEV), db0.to(DEV)
    dy, dres = O.bn_backward(dzc, z, yc, saved, dgc, dbc, flags, residual, G, with_lo)
    # dy: two fp32 means over the group and one fma chain per element
    if rnd:
        _tf32_close(dy, y64.grad, 1e-5, "dy (TF32)")
    else:
        _close(dy, y64.grad, 1e-5, "dy")
    if residual:
        assert dres is dzc
        _same_bits(dres, dpre, "dres (gated dz, written over dz)")
    else:
        _same_bits(dzc, dz, "dz untouched without a residual")
    # dgamma / dbeta: fp32 partial sums over <= a few hundred rows, fp64 across CTAs and groups, then one fp32 +=
    _close(dgc, dg0.double() + gm64.grad, 1e-5, "dgamma (+=)")
    _close(dbc, db0.double() + bt64.grad, 1e-5, "dbeta (+=)")
    if with_lo:
        _same_bits(dy._scsfm_lo, lo_tf32(_np(dy)), "lo(dy)")

    # eval: the running statistics (those the training call left), which stay untouched
    rm_e, rv_e = rmc.clone(), rvc.clone()
    ze, saved_e = O.bn_apply(yc, None, gc, bc, rmc, rvc, BN_MOM, BN_EPS, rc, flags & ~O.ROUND_TF32, G)
    _same_bits(rmc, rm_e, "eval leaves the running mean")
    _same_bits(rvc, rv_e, "eval leaves the running var")
    want = F.batch_norm(y.double(), rm_e.double().cpu(), rv_e.double().cpu(), gamma.double(), beta.double(), False, BN_MOM, BN_EPS)
    if residual:
        want = want + res.double()
    _close(ze, F.relu(want) if relu else want, 2e-6, "eval z")
    for grp in range(G):
        _same_bits(saved_e[grp, :, 2], rm_e, "eval saved mean")
    saved_pe = O.bn_prepare(None, G, R, gc, bc, rmc, rvc, BN_MOM, BN_EPS, False)
    for k in range(4):
        _close(saved_pe[..., k], saved_e[..., k], 1e-6, "bn_prepare eval saved")


# ----- max-pool 3x3 / 2, pad 1 ----------------------------------------------------------------------------------
POOL_CASES = [(1, 4, 2, 2), (2, 4, 3, 3), (2, 64, 2, 5), (1, 4, 3, 8), (2, 4, 7, 10), (2, 64, 9, 13), (1, 64, 128, 416)]


def _pool_input(kind, shape, g):
    if kind == "relu":                      # post-ReLU: about half exact zeros, all-zero windows
        return F.relu(torch.randn(shape, generator=g, dtype=torch.float64)).float()
    return torch.randint(-2, 3, shape, generator=g).float()       # small integers: ties in most windows


def _tap_to_flat(idx, H, W):
    """The kernel's tap index (dy*3+dx of the window) -> PyTorch's flat input index h*W + w, NCHW."""
    k = idx.permute(0, 3, 1, 2).long().cpu()
    Ho, Wo = k.shape[2], k.shape[3]
    ho = torch.arange(Ho).view(1, 1, Ho, 1)
    wo = torch.arange(Wo).view(1, 1, 1, Wo)
    return (2 * ho + k // 3 - 1) * W + (2 * wo + k % 3 - 1)


@pytest.mark.parametrize("kind", ["relu", "int"])
@pytest.mark.parametrize("shape", POOL_CASES, ids=lambda s: "B%dC%d_%dx%d" % s)
def test_maxpool_vs_fp64(shape, kind):
    """Values are copies (bitwise) and the argmax is PyTorch's: the first maximum in scan order."""
    O = _ops()
    B, C, H, W = shape
    g = _gen(H * W + C)
    x = _pool_input(kind, (B, C, H, W), g)
    x64 = x.double().requires_grad_(True)
    p, ind = F.max_pool2d(x64, 3, 2, 1, return_indices=True)
    xc = nh(x)
    y, idx = O.maxpool_fwd(xc)
    _same_bits(nc(y), p.detach(), "max-pool values")
    assert torch.equal(_tap_to_flat(idx, H, W), ind), "max-pool argmax differs from PyTorch's"
    dp = torch.randn(p.shape, generator=g).float()
    p.backward(dp.double())
    for acc in (False, True):
        init = torch.randn(B, H, W, C, generator=g) if acc else torch.full((B, H, W, C), float("nan"))
        dx = init.to(DEV)
        O.maxpool_bwd(nh(dp), idx, xc.shape, dx, acc)
        want = x64.grad + (init.permute(0, 3, 1, 2).double() if acc else 0)
        _close(nc(dx), want, 1e-6, "max-pool backward acc=%d" % acc)      # <= 4 fp32 adds per element


def test_maxpool_nan_propagates_like_pytorch():
    O = _ops()
    g = _gen(5)
    x = torch.randn(2, 4, 5, 6, generator=g)
    x[0, 1, 1, 2] = float("nan")
    x[1, 3, 4, 5] = float("nan")
    p, ind = F.max_pool2d(x.double(), 3, 2, 1, return_indices=True)
    y, idx = O.maxpool_fwd(nh(x))
    got = nc(y)
    assert torch.equal(torch.isnan(got), torch.isnan(p)) and int(torch.isnan(p).sum()) >= 2
    keep = ~torch.isnan(p)
    assert torch.equal(got[keep], p[keep])
    assert torch.equal(_tap_to_flat(idx, 5, 6), ind)


# ----- nearest x2 upsample + concat, reflection-pad folds --------------------------------------------------------
UPCAT_STAGES = [(256, 256), (128, 128), (64, 64), (32, 64), (16, 0), (256, 1024), (128, 512), (64, 256)]


@pytest.mark.parametrize("C1,C2", UPCAT_STAGES)
def test_upcat_fwd_bitwise(C1, C2):
    O = _ops()
    g = _gen(C1 + C2)
    lo = torch.randn(2, C1, 3, 5, generator=g)
    sk = torch.randn(2, C2, 6, 10, generator=g) if C2 else None
    out = O.upcat_fwd(nh(lo), nh(sk) if C2 else None)
    up = F.interpolate(lo, scale_factor=2, mode="nearest")
    _same_bits(nc(out), torch.cat([up, sk], 1) if C2 else up, "upcat")


def _elu_pair(shape, g):
    """A pre-activation with exact zeros (the ELU kink) and its fp32 ELU output."""
    x = torch.randn(shape, generator=g).float()
    x.view(-1)[::11] = 0.0
    x64 = x.double().requires_grad_(True)
    return x64, F.elu(x64)


@pytest.mark.parametrize("act", ["elu", "elu_round"])
@pytest.mark.parametrize("C1,C2", [(16, 0), (32, 64), (8, 12)])
@pytest.mark.parametrize("plane", [(2, 2), (4, 4), (4, 6), (64, 208)], ids=lambda p: "%dx%d" % p)
def test_fold_upcat_vs_autograd(plane, C1, C2, act):
    """Gradient of reflect_pad(cat(upsample(elu(lo)), skip)) back to lo's pre-activation and to skip.  On 2x2 and 4x4
    planes both mirror rows coincide with or neighbour the 2x2 upsample cells."""
    O = _ops()
    H, W = plane
    g = _gen(H * W + C1 + C2)
    B = 2
    lo64, a64 = _elu_pair((B, C1, H // 2, W // 2), g)
    sk64 = torch.randn(B, C2, H, W, generator=g).float().double().requires_grad_(True)
    up = F.interpolate(a64, scale_factor=2, mode="nearest")
    padded = F.pad(torch.cat([up, sk64], 1) if C2 else up, (1, 1, 1, 1), mode="reflect")
    dpad = torch.randn(padded.shape, generator=g).float()
    padded.backward(dpad.double())
    flag = O.ACT_ELU | (O.ROUND_TF32 if act == "elu_round" else 0)
    d_lo, d_sk = O.fold_upcat(nh(dpad), C1, nh(a64), flag)
    if act == "elu_round":
        d_plain, _ = O.fold_upcat(nh(dpad), C1, nh(a64), O.ACT_ELU)
        _same_bits(d_lo, rna_tf32(_np(d_plain)), "d_lo = rna(d_lo unrounded)")
        _tf32_close(nc(d_lo), lo64.grad, 1e-6, "d_lo (TF32)")
        d_lo = d_plain
    # <= 16 fp32 adds and one multiply by elu' = a + 1 (the fp32 ELU output carries its own rounding)
    _close(nc(d_lo), lo64.grad, 1e-6, "d_lo")
    if C2:
        _close(nc(d_sk), sk64.grad, 1e-6, "d_skip")         # <= 4 fp32 adds
    else:
        assert d_sk is None


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("act", ["none", "elu", "elu_round"])
@pytest.mark.parametrize("plane", [(2, 2), (3, 3), (4, 6), (5, 8), (33, 64)], ids=lambda p: "%dx%d" % p)
def test_fold_plain_vs_autograd(plane, act, accumulate):
    """d (+)= fold(dpad), then times act'(out).  On 2x2 / 3x3 planes the two mirror rows (and columns) coincide with or
    neighbour each other."""
    O = _ops()
    H, W = plane
    for C in (4, 16):
        g = _gen(H * W * C + accumulate)
        B = 2
        if act == "none":
            x64 = torch.randn(B, C, H, W, generator=g).float().double().requires_grad_(True)
            a64 = x64
        else:
            x64, a64 = _elu_pair((B, C, H, W), g)
        padded = F.pad(a64, (1, 1, 1, 1), mode="reflect")
        dpad = torch.randn(padded.shape, generator=g).float()
        d0 = torch.randn(B, C, H, W, generator=g).float()
        loss = (padded * dpad.double()).sum() + ((a64 * d0.double()).sum() if accumulate else 0)
        loss.backward()
        flag = {"none": O.ACT_NONE, "elu": O.ACT_ELU, "elu_round": O.ACT_ELU | O.ROUND_TF32}[act]

        def run(f):
            d = nh(d0) if accumulate else torch.full((B, H, W, C), float("nan"), device=DEV)
            O.fold_plain(nh(dpad), d, None if act == "none" else nh(a64), f, accumulate)
            return d
        d = run(flag)
        if act == "elu_round":
            d_plain = run(O.ACT_ELU)
            _same_bits(d, rna_tf32(_np(d_plain)), "d = rna(d unrounded)")
            _tf32_close(nc(d), x64.grad, 1e-6, "fold_plain (TF32)")
            d = d_plain
        _close(nc(d), x64.grad, 1e-6, "fold_plain C=%d" % C)       # <= 5 fp32 adds and one multiply


# ----- activation gradients ---------------------------------------------------------------------------------------
def _act_ref(x64, act):
    if act == "relu":
        return F.relu(x64)
    if act == "elu":
        return F.elu(x64)
    return 10 * torch.sigmoid(x64) + 0.01


@pytest.mark.parametrize("rnd", [False, True])
@pytest.mark.parametrize("act", ["relu", "elu", "disp"])
def test_act_bwd_vs_autograd(act, rnd):
    """d *= act'(out), from the activation output; pre-activations include exact zeros (the ReLU / ELU kinks: ReLU passes
    nothing there, ELU passes 1) and values within 1e-30 of them."""
    O = _ops()
    g = _gen(11)
    n = GRID_STRIDE + 18_883
    x = (2 * torch.randn(n, generator=g)).float()
    x[:4096] = 0.0
    x[4096:4352] = 1e-30
    x[4352:4608] = -1e-30
    x64 = x.double().requires_grad_(True)
    out = _act_ref(x64, act)
    d = torch.randn(n, generator=g).float()
    out.backward(d.double())
    code = {"relu": O.ACT_RELU, "elu": O.ACT_ELU, "disp": O.ACT_DISP}[act]
    outc = out.detach().float().to(DEV)
    got = O.act_bwd_(d.to(DEV), outc, code | (O.ROUND_TF32 if rnd else 0))
    if rnd:
        plain = O.act_bwd_(d.to(DEV), outc, code)
        _same_bits(got, rna_tf32(_np(plain)), "act_bwd = rna(act_bwd unrounded)")
        _tf32_close(got, x64.grad, 1e-6, "act_bwd (TF32)")
        got = plain
    # one product with act'(out) evaluated from the fp32 output (DISP: 10 s (1 - s), s = (out - 0.01) / 10)
    _close(got, x64.grad, 1e-6, "act_bwd " + act)
    if act == "relu":
        assert float(got[:4096].abs().max()) == 0.0
    if act == "elu":
        _same_bits(got[:4096], d[:4096], "ELU gradient at 0 is exactly 1")


# ----- disparity heads --------------------------------------------------------------------------------------------
def _head_ref(x, w, b, act, chunk=1):
    """F.conv2d on the reflection-padded input in fp64 (x NCHW fp32, w [1,3,3,C]); batch chunks bound the im2col memory."""
    wt = w.double().permute(0, 3, 1, 2)
    outs = []
    for i in range(0, x.shape[0], chunk):
        pre = F.conv2d(F.pad(x[i:i + chunk].double(), (1, 1, 1, 1), mode="reflect"), wt, b.double() if b is not None else None)
        outs.append(10 * torch.sigmoid(pre) + 0.01 if act else pre)
    return torch.cat(outs)


@pytest.mark.parametrize("plane", [(1, 2, 2), (2, 3, 5), (3, 7, 11)], ids=lambda p: "B%d_%dx%d" % p)
@pytest.mark.parametrize("C", [4, 8, 16, 32, 64, 128])
def test_head_fwd_vs_fp64(C, plane):
    """Every template instance; 3x7x11 = 231 pixels is not a multiple of the pixels per CTA (256 / (C/4))."""
    O = _ops()
    B, H, W = plane
    g = _gen(C * H * W)
    x = torch.randn(B, C, H, W, generator=g)
    w = torch.randn(1, 3, 3, C, generator=g) / (9 * C) ** 0.5
    b = torch.randn(1, generator=g)
    for bias in (b, None):
        for act in (O.ACT_DISP, O.ACT_NONE):
            out = O.head_fwd(nh(x), w.to(DEV), bias.to(DEV) if bias is not None else None, act)
            # an fp32 dot product of 9*C terms, then expf: well inside 1e-5
            _close(nc(out), _head_ref(x, w, bias, act == O.ACT_DISP), 1e-5, "head_fwd bias=%s act=%d" % (bias is not None, act))


def test_head_fwd_full_size():
    """The stacked forward_multi batch at 256x832 (12 images, C=16): the grid is capped, so every CTA strides."""
    O = _ops()
    g = _gen(12)
    x = torch.rand(12, 16, 256, 832, generator=g) * 2 - 0.5
    w = torch.randn(1, 3, 3, 16, generator=g) / 12.0
    b = torch.randn(1, generator=g)
    out = O.head_fwd(nh(x), w.to(DEV), b.to(DEV), O.ACT_DISP)
    _close(nc(out), _head_ref(x, w, b, True), 1e-5, "head_fwd 12x256x832")


HEAD_WGRAD_CASES = [(16, (2, 5, 7)), (32, (2, 5, 7)), (64, (1, 2, 2)), (128, (2, 5, 7)),
                    (96, (2, 33, 47)),          # C/4 = 24 does not divide 256: 16 idle threads per CTA
                    (1024, (2, 40, 52)),        # one pixel lane per CTA
                    (32, (4, 128, 416)),
                    (16, (12, 256, 832))]       # full size: the grid is capped at 528 CTAs


def _case_id(C, plane):
    return "C%d_%s" % (C, "x".join(map(str, plane)))


@pytest.mark.parametrize("C,plane", HEAD_WGRAD_CASES, ids=[_case_id(*c) for c in HEAD_WGRAD_CASES])
def test_head_wgrad_vs_fp64(C, plane):
    O = _ops()
    B, H, W = plane
    g = _gen(C + H)
    x = torch.rand(B, C, H, W, generator=g) * 2 - 0.5
    dpre = torch.randn(B, 1, H, W, generator=g)
    dw0, db0 = torch.randn(1, 3, 3, C, generator=g), torch.randn(1, generator=g)
    w64 = torch.zeros(1, C, 3, 3, dtype=torch.float64, requires_grad=True)
    b64 = torch.zeros(1, dtype=torch.float64, requires_grad=True)
    for i in range(0, B, 2):          # leaf gradients accumulate over the chunks
        F.conv2d(F.pad(x[i:i + 2].double(), (1, 1, 1, 1), mode="reflect"), w64, b64).backward(dpre[i:i + 2].double())
    dw, db = dw0.to(DEV), db0.to(DEV)
    O.head_wgrad(nh(x), nh(dpre), dw, db)
    # fp32 sums: per pixel lane (<= ~100 pixels), over the CTA's lanes, then fp32 atomics over <= 528 CTAs
    _close(dw.cpu(), dw0.double() + w64.grad.permute(0, 2, 3, 1), 1e-5, "head dw (+=)")
    _close(db.cpu(), db0.double() + b64.grad, 1e-5, "head dbias (+=)")


HEAD_DGRAD_CASES = [(16, (2, 2, 2)), (16, (1, 3, 3)), (64, (2, 5, 9)), (32, (2, 64, 208))]


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("C,plane", HEAD_DGRAD_CASES, ids=[_case_id(*c) for c in HEAD_DGRAD_CASES])
def test_head_dgrad_and_fold_vs_autograd(C, plane, accumulate):
    """The decoder's disparity-head backward: head_dgrad to the padded input, then fold_plain(ELU) onto the pre-activation
    of the ELU that fed the head (accumulating onto the gradient another consumer left)."""
    O = _ops()
    B, H, W = plane
    g = _gen(C * H + accumulate)
    x64, b64 = _elu_pair((B, C, H, W), g)
    w = torch.randn(1, 3, 3, C, generator=g) / (9 * C) ** 0.5
    dpre = torch.randn(B, 1, H, W, generator=g)
    d0 = torch.randn(B, C, H, W, generator=g)
    padded = F.pad(b64, (1, 1, 1, 1), mode="reflect")
    padded.retain_grad()
    out = F.conv2d(padded, w.double().permute(0, 3, 1, 2))
    ((out * dpre.double()).sum() + ((b64 * d0.double()).sum() if accumulate else 0)).backward()
    dpad = O.head_dgrad(nh(dpre), w.to(DEV), (B, H, W, C))
    _close(nc(dpad), padded.grad, 1e-6, "head_dgrad")                   # <= 9 fp32 fmas
    d = nh(d0) if accumulate else torch.empty(B, H, W, C, device=DEV)
    O.fold_plain(dpad, d, nh(b64), O.ACT_ELU, accumulate)
    _close(nc(d), x64.grad, 1e-6, "head dgrad + fold")


# ----- pose head --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,C,H,W", [(1, 6, 1, 1), (16, 6, 1, 1), (3, 5, 8, 26), (16, 6, 8, 26), (2, 6, 20, 30), (16, 6, 20, 30)])
def test_spatial_mean_vs_fp64(B, C, H, W):
    """0.01 * mean over the plane and its gradient; HW = 600 is more pixels than one CTA has threads."""
    O = _ops()
    g = _gen(B * H * W + C)
    x = torch.randn(B, C, H, W, generator=g) + torch.randn(1, C, 1, 1, generator=g)
    x64 = x.double().requires_grad_(True)
    out = 0.01 * x64.mean((2, 3))
    dout = torch.randn(B, C, generator=g)
    out.backward(dout.double())
    got = O.spatial_mean_fwd(nh(x), 0.01)
    _close(got.cpu(), out.detach(), 1e-6, "spatial_mean_fwd")          # fp32 block sum of <= 600 values
    dx = O.spatial_mean_bwd(dout.to(DEV), (B, H, W, C), 0.01)
    _close(nc(dx), x64.grad, 1e-6, "spatial_mean_bwd")                 # two roundings per element


# ----- Adam -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("wd", [0.0, 1e-2])
def test_adam_vs_torch_optim_fp64(wd):
    """Five steps against torch.optim.Adam in fp64 from the same fp32 start, compared per step on the parameter CHANGE.
    Entries with |g| ~ 1e-9 (where eps dominates the denominator) and exact-zero gradients are included; n exceeds the
    capped grid so the grid-stride loop runs."""
    O = _ops()
    g = _gen(int(wd * 1e4))
    n = GRID_STRIDE + 18_877
    lr, b1, b2, eps = f32(1e-3), f32(0.9), f32(0.999), f32(1e-8)      # the fp32 values the kernel receives
    wdf = f32(wd)
    p0 = (0.05 * torch.randn(n, generator=g)).float()
    mag = torch.tensor([1.0, 1e-3, 1e-9])[torch.randint(0, 3, (n,), generator=g)]
    zero = torch.zeros(n, dtype=torch.bool)
    zero[torch.randperm(n, generator=g)[:5000]] = True
    grads = []
    for _ in range(5):
        gr = (torch.randn(n, generator=g) * mag).float()
        gr[zero] = 0.0
        grads.append(gr)

    adam64 = Adam64(p0, lr, (b1, b2), eps, wdf)
    p = p0.to(DEV)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    # the same steps with the step count on the device and an operand mirror (TF32, then LO)
    runs = [(p0.to(DEV), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV), torch.empty(n, device=DEV), op)
            for op in (O.OPERAND_TF32, O.OPERAND_LO)]
    step_dev = torch.zeros(1, dtype=torch.int32, device=DEV)
    for step, gr in enumerate(grads, 1):
        want, size = adam64.step(gr)
        before = p.double().cpu()
        grc = gr.to(DEV)
        O.adam_step(p, grc, m, v, lr, b1, b2, eps, wdf, step)
        after = p.double().cpu()
        assert_adam_change(after - before, want, size, after, gr, "step %d" % step)
        if wd == 0.0:
            _same_bits(p.cpu()[zero], p0[zero], "zero gradient leaves the parameter")
            assert float(m.cpu()[zero].abs().max()) == 0.0 and float(v.cpu()[zero].abs().max()) == 0.0
        step_dev.fill_(step)
        for (pd, md, vd, mirror, op) in runs:
            O.adam_step(pd, grc, md, vd, lr, b1, b2, eps, wdf, 0, step_dev, mirror, op)
            _same_bits(pd, p, "device step count: parameters")
            _same_bits(md, m, "device step count: m")
            _same_bits(vd, v, "device step count: v")
            ref = torch.empty_like(p)
            if op == O.OPERAND_TF32:
                O.round_tf32(p, ref)
            else:
                O.split_tf32(p, ref)
            _same_bits(mirror, ref, "operand mirror %d" % op)
