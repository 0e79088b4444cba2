"""Oracle: TSDF fusion and marching cubes over a dense voxel array, in fp64 numpy (restates include/scsfm.h, "Dense
reconstruction", the semantics scsfm.fusion.TSDFVolume implements on bricks).

TEST INFRASTRUCTURE -- see oracle/__init__.py.  Arrays are indexed [i, j, k] (x, y, z); voxel (i, j, k) has its centre at
lo + (ijk + 0.5) v.  The marching-cubes table is scsfm/mc_tables.py, the one the kernels use.
"""
import numpy as np

from scsfm.mc_tables import CORNERS, EDGES, TRI_TABLE

PIXEL_EPS = 1e-4          # pixels: a voxel this close to a pixel-rounding boundary may round either way in fp32
BAND_EPS = 1e-5           # of trunc: a voxel this close to the edge of the band may fall either side in fp32


class Grid:
    """A dense volume of shape (nx, ny, nz) at lo with voxel size v: tsdf, w, rgb in fp64, all zero."""

    def __init__(self, lo, v, shape):
        self.lo, self.v, self.shape = np.asarray(lo, np.float64), float(v), tuple(shape)
        self.tsdf = np.zeros(shape)
        self.w = np.zeros(shape)
        self.rgb = np.zeros(shape + (3,))

    def centres(self):
        ijk = np.stack(np.meshgrid(*[np.arange(n) for n in self.shape], indexing="ij"), -1).astype(np.float64)
        return self.lo + (ijk + 0.5) * self.v


def integrate(grid, depth, K, cam_to_world, trunc, max_depth, color=None):
    """Apply one frame to every voxel of `grid` in place.  depth [H,W], K [3,3], cam_to_world [4,4], color [H,W,3] uint8 or
    None.  Returns (updated, ambiguous): boolean arrays of the grid's shape, the voxels this frame updated and those whose
    decision lies within PIXEL_EPS px of a pixel-rounding boundary or BAND_EPS * trunc of the band's edge."""
    depth = np.asarray(depth, np.float64)
    H, W = depth.shape
    inv = np.linalg.inv(np.asarray(cam_to_world, np.float64))
    pc = grid.centres() @ inv[:3, :3].T + inv[:3, 3]
    z = pc[..., 2]
    front = z > 0
    zs = np.where(front, z, 1.0)
    u = K[0][0] * pc[..., 0] / zs + K[0][2]
    v = K[1][1] * pc[..., 1] / zs + K[1][2]

    def update(fu, fv):
        inside = front & (fu >= 0) & (fu < W) & (fv >= 0) & (fv < H)
        iu, iv = np.where(inside, fu, 0).astype(np.int64), np.where(inside, fv, 0).astype(np.int64)
        d = np.where(inside, depth[iv, iu], np.nan)
        valid = inside & np.isfinite(d) & (d > 0) & (d <= max_depth)
        sdf = np.where(valid, d - z, np.inf)
        return valid & (np.abs(sdf) <= trunc), valid, sdf, iu, iv

    fu, fv = np.floor(u + 0.5), np.floor(v + 0.5)
    upd, valid, sdf, iu, iv = update(fu, fv)
    # the pixel on the other side of a rounding boundary the voxel lies next to: ambiguous when either pixel updates it
    near_u = np.abs(u + 0.5 - np.rint(u + 0.5)) < PIXEL_EPS
    near_v = np.abs(v + 0.5 - np.rint(v + 0.5)) < PIXEL_EPS
    au = np.where(u + 0.5 - fu < 0.5, fu - 1, fu + 1)
    av = np.where(v + 0.5 - fv < 0.5, fv - 1, fv + 1)
    either = upd | update(np.where(near_u, au, fu), np.where(near_v, av, fv))[0] | update(np.where(near_u, au, fu), fv)[0] | \
        update(fu, np.where(near_v, av, fv))[0]
    ambiguous = ((near_u | near_v) & either) | (valid & (np.abs(np.abs(sdf) - trunc) < BAND_EPS * trunc))
    w = grid.w[upd]
    grid.tsdf[upd] = (grid.tsdf[upd] * w + sdf[upd] / trunc) / (w + 1)
    if color is not None:
        c = np.asarray(color, np.float64)[iv[upd], iu[upd]]
        grid.rgb[upd] = (grid.rgb[upd] * w[:, None] + c) / (w[:, None] + 1)
    grid.w[upd] = w + 1
    return upd, ambiguous


def marching_cubes(tsdf, w, rgb, lo, v):
    """Marching cubes over the cells whose 8 corners have w > 0.  Returns (tris, verts): tris int64 [T,3] of edge keys (the
    lower voxel's linear index (k ny + j) nx + i, times 3, plus the axis), verts {key: (position fp64 [3], colour uint8 [3])}
    with position lo + (ijk + 0.5 + t e_axis) v and colour rint(rgb0 + t (rgb1 - rgb0)), t = tsdf0 / (tsdf0 - tsdf1) from the
    lower voxel, in fp64 from the stored values."""
    tsdf, w, rgb = np.asarray(tsdf, np.float64), np.asarray(w, np.float64), np.asarray(rgb, np.float64)
    lo = np.asarray(lo, np.float64)
    nx, ny, nz = tsdf.shape
    cx, cy, cz = nx - 1, ny - 1, nz - 1
    if min(cx, cy, cz) <= 0:
        return np.zeros((0, 3), np.int64), {}
    ok = np.ones((cx, cy, cz), bool)
    config = np.zeros((cx, cy, cz), np.int64)
    for c, (a, b, e) in enumerate(CORNERS):
        sl = (slice(a, a + cx), slice(b, b + cy), slice(e, e + cz))
        ok &= w[sl] > 0
        config |= (tsdf[sl] < 0).astype(np.int64) << c
    table = np.asarray(TRI_TABLE, np.int64)
    ci, cj, ck = np.nonzero(ok)
    rows = table[config[ci, cj, ck]]
    ntri = (rows >= 0).sum(1) // 3
    tris, verts = [], {}
    corner = np.asarray(CORNERS, np.int64)
    for q in range(5):
        m = ntri > q
        tri = []
        for s in range(3):
            e = rows[m, 3 * q + s]
            a, b = np.asarray(EDGES, np.int64)[e].T
            lower = np.where(corner[a].sum(1) < corner[b].sum(1), a, b)
            upper = np.where(lower == a, b, a)
            axis = np.argmax(corner[upper] != corner[lower], axis=1)
            li = np.stack([ci[m], cj[m], ck[m]], 1) + corner[lower]
            ui = np.stack([ci[m], cj[m], ck[m]], 1) + corner[upper]
            key = ((li[:, 2] * ny + li[:, 1]) * nx + li[:, 0]) * 3 + axis
            s0 = tsdf[li[:, 0], li[:, 1], li[:, 2]]
            s1 = tsdf[ui[:, 0], ui[:, 1], ui[:, 2]]
            t = s0 / (s0 - s1)
            g = li + 0.5
            g[np.arange(len(g)), axis] += t
            pos = lo + g * v
            c0 = rgb[li[:, 0], li[:, 1], li[:, 2]]
            c1 = rgb[ui[:, 0], ui[:, 1], ui[:, 2]]
            col = np.clip(np.rint(c0 + t[:, None] * (c1 - c0)), 0, 255).astype(np.uint8)
            for kk, p, cc in zip(key.tolist(), pos, col):
                verts[kk] = (p, cc)
            tri.append(key)
        if m.any():
            tris.append(np.stack(tri, 1))
    return (np.concatenate(tris) if tris else np.zeros((0, 3), np.int64)), verts


def euler_characteristic(faces):
    """V - E + F of a triangle mesh given as vertex-id triples."""
    faces = np.asarray(faces)
    e = np.sort(np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]]), axis=1)
    return len(np.unique(faces)) - len(np.unique(e, axis=0)) + len(faces)


def canonical_triangles(tris):
    """Triangles as a sorted array of rotation-normalised triples (the smallest key first, orientation kept)."""
    tris = np.asarray(tris, np.int64).reshape(-1, 3)
    r = np.argmin(tris, axis=1)
    idx = (r[:, None] + np.arange(3)[None]) % 3
    t = np.take_along_axis(tris, idx, 1)
    return t[np.lexsort(t.T[::-1])]
