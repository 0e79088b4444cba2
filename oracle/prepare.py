"""CPU oracle for the training-set preparation kernels (csrc/prepare.cu).  TEST INFRASTRUCTURE ONLY.

resize_bilinear_u8  PIL.Image.fromarray(img).resize((w, h), Image.BILINEAR): what scipy.misc.imresize(img, (h, w)) did to a
                    uint8 RGB frame in the reference's loaders (kitti_raw_loader.py:224, kitti_odom_loader.py:57,
                    cityscapes_loader.py:119).  Pillow's src/libImaging/Resample.c, the algorithm oracle/augment.py restates
                    for BICUBIC, with the filter and its support as parameters (`resample_coeffs`).
depth_map           generate_depth_map (kitti_raw_loader.py:243-300) by the rule the kernel implements: float32(z) of the
                    last point on a pixel; for every sub2ind key with >= 2 points, float32(min z) of the key at the pixel of
                    its first point; negative values to 0.  The projection is evaluated left to right in fp64, as the kernel
                    does (the reference's np.dot goes through BLAS, whose summation order may differ in the last bit).
"""
import numpy as np

PRECISION_BITS = 32 - 8 - 2


def bilinear(x):
    """Resample.c bilinear_filter."""
    x = abs(x)
    return 1.0 - x if x < 1.0 else 0.0


def bicubic(x):
    """Resample.c bicubic_filter, a = -0.5."""
    a = -0.5
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


FILTERS = {"bilinear": (bilinear, 1.0), "bicubic": (bicubic, 2.0)}


def resample_coeffs(in_size, out_size, filt="bilinear"):
    """Resample.c precompute_coeffs + normalize_coeffs_8bpc for the box (0, in_size) and the named filter: per output
    coordinate the first input coordinate, the tap count and the integer taps (2 * ceil(support) + 1 columns)."""
    fn, base_support = FILTERS[filt]
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = base_support * filterscale
    ksize = int(np.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), np.int32)
    kk = np.zeros((out_size, ksize), np.int32)
    ss = 1.0 / filterscale
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = [fn((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for v in w:
            ww += v
        for x in range(xmax):
            k = w[x] / ww if ww != 0.0 else w[x]
            kk[xx, x] = int(-0.5 + k * (1 << PRECISION_BITS)) if k < 0 else int(0.5 + k * (1 << PRECISION_BITS))
        bounds[xx] = (xmin, xmax)
    return bounds, kk


def _pass(src, bounds, kk, axis):
    """One fixed-point pass along `axis` (1: columns, 0: rows) of an int64 H x W x C array -> uint8."""
    out_n = len(bounds)
    shape = list(src.shape)
    shape[axis] = out_n
    out = np.zeros(shape, np.uint8)
    for j in range(out_n):
        x0, n = bounds[j]
        acc = np.full(src.shape[:axis] + src.shape[axis + 1:], 1 << (PRECISION_BITS - 1), np.int64)
        for i in range(n):
            acc += np.take(src, x0 + i, axis=axis) * int(kk[j, i])
        sl = [slice(None)] * 3
        sl[axis] = j
        out[tuple(sl)] = np.clip(acc >> PRECISION_BITS, 0, 255)
    return out


def resize_u8(img, out_w, out_h, filt="bilinear"):
    """Image.fromarray(img).resize((out_w, out_h), filter) for an H x W x C uint8 array: horizontal pass into an 8-bit
    intermediate, then the vertical pass; a pass whose size does not change is skipped (ImagingResampleInner)."""
    img = np.asarray(img, np.uint8)
    H, W, _ = img.shape
    out = img.copy()
    if out_w != W:
        out = _pass(out.astype(np.int64), *resample_coeffs(W, out_w, filt), axis=1)
    if out_h != H:
        out = _pass(out.astype(np.int64), *resample_coeffs(H, out_h, filt), axis=0)
    return out


def resize_bilinear_u8(img, out_w, out_h):
    return resize_u8(img, out_w, out_h, "bilinear")


def project(velo, P):
    """Kept points (x >= 0) of an N x 4 float32 cloud -> (px, py, z) float64, px / py before the bounds test."""
    velo = np.asarray(velo, np.float32).reshape(-1, 4)
    velo = velo[velo[:, 0] >= 0]
    x, y, z = (velo[:, i].astype(np.float64) for i in range(3))
    u = [((P[r, 0] * x + P[r, 1] * y) + P[r, 2] * z) + P[r, 3] for r in range(3)]
    return np.round(u[0] / u[2]) - 1, np.round(u[1] / u[2]) - 1, u[2]


def depth_map(velo, P, Hd, Wd):
    """The Hd x Wd float32 depth map of one cloud (velo: N x 4 float32, P: 3 x 4 float64 P_velo2im)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        px, py, z = project(velo, np.asarray(P, np.float64))
        keep = (px >= 0) & (py >= 0) & (px < Wd) & (py < Hd)
    px, py, z = px[keep].astype(np.int64), py[keep].astype(np.int64), z[keep]
    depth = np.zeros((Hd, Wd), np.float32)
    depth[py, px] = z.astype(np.float32)                       # (a) repeated indices: the last point wins
    key = py * (Wd - 1) + px - 1
    order = np.argsort(key, kind="stable")                     # points of one key in file order
    uniq, first, counts = np.unique(key[order], return_index=True, return_counts=True)
    zmin = np.minimum.reduceat(z[order], first) if len(order) else np.zeros(0)
    dup = counts >= 2
    head = order[first[dup]]                                   # (b) the key's first point, in file order
    depth[py[head], px[head]] = zmin[dup].astype(np.float32)
    depth[depth < 0] = 0                                       # (c)
    return depth
