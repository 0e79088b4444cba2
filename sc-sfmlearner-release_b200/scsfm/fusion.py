"""A truncated signed distance field on the device: depth maps and poses fused into a volume, and the volume meshed.

TSDFVolume is the only code that knows the brick layout (include/scsfm.h, "Dense reconstruction").  The box [lo, hi) is
split into bricks of 8^3 voxels; a dense coarse index holds one brick id per 8^3 cell, and the brick pool grows by doubling
as frames reach new cells.  Depth is in the network's units (1 / disp) and poses are camera-to-world in the same scale.

    vol = TSDFVolume(lo, hi, voxel_size=0.2)
    vol.integrate(depth, K, cam_to_world, color)     # frames applied to each voxel in order, 16 per pass over the voxels
    verts, faces, colors = vol.mesh()
"""
import ctypes
import math

import numpy as np
import torch

from . import lib
from .mc_tables import TRI_TABLE

BRICK = 8
FIELDS = 5                     # tsdf, w, r, g, b
MAX_FRAMES = 16
MAX_CELLS = 2 ** 31 - 1


class Frame(ctypes.Structure):
    _fields_ = [("depth", ctypes.c_void_p), ("color", ctypes.c_void_p), ("R_wc", ctypes.c_float * 9), ("t_wc", ctypes.c_float * 3),
                ("R_cw", ctypes.c_float * 9), ("t_cw", ctypes.c_float * 3), ("fx", ctypes.c_float), ("fy", ctypes.c_float),
                ("cx", ctypes.c_float), ("cy", ctypes.c_float)]


class Volume(ctypes.Structure):
    _fields_ = [("lo_d", ctypes.c_double * 3), ("voxel_d", ctypes.c_double), ("lo", ctypes.c_float * 3), ("voxel", ctypes.c_float),
                ("trunc", ctypes.c_float), ("max_depth", ctypes.c_float), ("nb", ctypes.c_int * 3)]


def _bind():
    L = lib.load()
    if not getattr(L, "_fusion_bound", False):
        P, I, FP, VP = ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(Frame), ctypes.POINTER(Volume)
        L.scsfm_fusion_alloc.argtypes = [FP, I, I, I, VP, P, P, I, P, P, I, P]
        L.scsfm_fusion_integrate.argtypes = [FP, I, I, I, VP, P, P, I, P, P]
        L.scsfm_fusion_sample.argtypes = [VP, P, P, P, ctypes.c_longlong, P, P]
        L.scsfm_fusion_mesh_count.argtypes = [VP, P, P, P, I, P, P, P]
        L.scsfm_fusion_mesh_emit.argtypes = [VP, P, P, P, I, P, P, P, P, P, P]
        L._fusion_bound = True
    return L


def _vec3(x, name):
    a = np.asarray(x, dtype=np.float64)
    if a.shape != (3,) or not np.all(np.isfinite(a)):
        raise ValueError("%s must be three finite numbers, got %r" % (name, x))
    return a


def _positive(x, name):
    if isinstance(x, bool) or not isinstance(x, (int, float)) or not math.isfinite(x) or x <= 0:
        raise ValueError("%s must be a positive finite number, got %r" % (name, x))
    return float(x)


def _host64(x, name):
    if isinstance(x, torch.Tensor):
        x = x.detach().cpu().numpy()
    a = np.asarray(x)
    if a.dtype.kind not in "fiu":
        raise TypeError("%s must hold real numbers, got %s" % (name, a.dtype))
    return a.astype(np.float64)


class TSDFVolume:
    """TSDF over the box [lo, hi) with voxels of `voxel_size` (hi is rounded up to whole bricks), truncation `trunc` (4 voxels
    by default) and depths above `max_depth` ignored.  CUDA only."""
    _INITIAL_BRICKS = 4096     # first pool size; the pool doubles whenever the frames need more

    def __init__(self, lo, hi, voxel_size, trunc=None, max_depth=80.0, device="cuda"):
        lo, hi = _vec3(lo, "lo"), _vec3(hi, "hi")
        v = _positive(voxel_size, "voxel_size")
        self.trunc = 4.0 * v if trunc is None else _positive(trunc, "trunc")
        self.max_depth = _positive(max_depth, "max_depth")
        if not np.all(hi > lo):
            raise ValueError("hi must exceed lo on every axis, got lo %s hi %s" % (lo.tolist(), hi.tolist()))
        dev = torch.device(device)
        if dev.type != "cuda":
            raise ValueError("device must be a CUDA device: the volume has no CPU implementation, got %s" % device)
        nb = np.maximum(np.ceil((hi - lo) / (BRICK * v) - 1e-9), 1).astype(np.int64)   # a box of whole bricks stays as given
        cells = int(np.prod(nb))
        if cells > MAX_CELLS:
            fit = v * (cells / MAX_CELLS) ** (1.0 / 3.0) * 1.01
            raise ValueError("a box of %.6g x %.6g x %.6g at voxel size %g needs %d x %d x %d = %d bricks in the coarse index, more "
                             "than 2^31 - 1; a voxel size of %.3g or more fits" % (tuple(hi - lo) + (v,) + tuple(nb) + (cells, fit)))
        self.voxel_size, self.lo, self.nb = v, lo, nb
        self.hi = lo + nb * BRICK * v
        self._vol = Volume((ctypes.c_double * 3)(*lo), v, (ctypes.c_float * 3)(*lo), v, self.trunc, self.max_depth,
                           (ctypes.c_int * 3)(*(int(n) for n in nb)))
        self.device = dev = dev if dev.index is not None else torch.device("cuda", torch.cuda.current_device())
        self._index = torch.full((cells,), -1, dtype=torch.int32, device=dev)
        self._stamp = torch.zeros(cells, dtype=torch.int32, device=dev)
        self._counters = torch.zeros(2, dtype=torch.int32, device=dev)
        self._pool = torch.zeros(self._INITIAL_BRICKS, FIELDS, BRICK ** 3, dtype=torch.float32, device=dev)
        self._touched = torch.empty(self._INITIAL_BRICKS, dtype=torch.int32, device=dev)
        self._tri = torch.tensor(TRI_TABLE, dtype=torch.int8, device=dev)
        self._epoch = 0
        self._bricks = 0
        self.brick_visits = 0      # bricks integrated, summed over the passes (one pass per 16 frames)

    @property
    def num_bricks(self):
        """Bricks allocated so far."""
        return self._bricks

    @property
    def dims(self):
        """Voxels along x, y, z."""
        return tuple(int(n) * BRICK for n in self.nb)

    def memory_bytes(self):
        """Device bytes the volume holds (coarse index, stamps and brick pool)."""
        return sum(t.numel() * t.element_size() for t in (self._index, self._stamp, self._pool, self._touched, self._counters))

    # ----- integration ------------------------------------------------------------------------------------------------------
    def _check_frames(self, depth, K, cam_to_world, color):
        if not isinstance(depth, torch.Tensor):
            raise TypeError("depth must be a torch tensor, got %s" % type(depth).__name__)
        if depth.dim() == 4 and depth.shape[1] == 1:
            depth = depth[:, 0]
        if depth.dim() != 3:
            raise ValueError("depth must be [B,H,W] or [B,1,H,W], got %s" % list(depth.shape))
        if depth.device != self.device:
            raise ValueError("depth must be on %s, got %s" % (self.device, depth.device))
        if depth.dtype != torch.float32:
            raise TypeError("depth must be float32, got %s" % depth.dtype)
        B, H, W = depth.shape
        K = _host64(K, "K")
        if K.shape == (3, 3):
            K = np.broadcast_to(K, (B, 3, 3))
        if K.shape != (B, 3, 3):
            raise ValueError("K must be [3,3] or [%d,3,3], got %s" % (B, list(K.shape)))
        if not np.all(np.isfinite(K)) or np.any(K[:, 0, 0] <= 0) or np.any(K[:, 1, 1] <= 0):
            raise ValueError("K must be finite with positive focal lengths")
        T = _host64(cam_to_world, "cam_to_world")
        if T.shape != (B, 4, 4):
            raise ValueError("cam_to_world must be [%d,4,4], got %s" % (B, list(T.shape)))
        if not np.all(np.isfinite(T)):
            raise ValueError("cam_to_world must be finite")
        if color is not None:
            if not isinstance(color, torch.Tensor):
                raise TypeError("color must be a torch tensor, got %s" % type(color).__name__)
            if color.dtype != torch.uint8:
                raise TypeError("color must be uint8, got %s" % color.dtype)
            if tuple(color.shape) != (B, H, W, 3):
                raise ValueError("color must be [%d,%d,%d,3], got %s" % (B, H, W, list(color.shape)))
            if color.device != self.device:
                raise ValueError("color must be on %s, got %s" % (self.device, color.device))
            color = color.contiguous()
        return depth.contiguous(), K, T, color

    @staticmethod
    def _frame(depth, color, K, T):
        inv = np.linalg.inv(T)
        R_wc, t_wc = inv[:3, :3], inv[:3, 3]
        return Frame(depth.data_ptr(), color.data_ptr() if color is not None else None,
                     (ctypes.c_float * 9)(*R_wc.reshape(-1)), (ctypes.c_float * 3)(*t_wc),
                     (ctypes.c_float * 9)(*T[:3, :3].reshape(-1)), (ctypes.c_float * 3)(*T[:3, 3]),
                     K[0, 0], K[1, 1], K[0, 2], K[1, 2])

    def integrate(self, depth, K, cam_to_world, color=None):
        """Fuse B frames: depth [B,H,W] or [B,1,H,W] float32 on the volume's device, K [3,3] or [B,3,3], cam_to_world [B,4,4]
        (KITTI-format poses, any float type, on any device), optional color [B,H,W,3] uint8 on the device.  Frames are applied
        to every voxel in the order given; without colour the voxels' rgb stay as they are."""
        depth, K, T, color = self._check_frames(depth, K, cam_to_world, color)
        B, H, W = depth.shape
        for f0 in range(0, B, MAX_FRAMES):
            frames = self._frames(depth, K, T, color, f0, min(MAX_FRAMES, B - f0))
            self._apply(frames, H, W, self._allocate(frames, H, W))
        return self

    def _frames(self, depth, K, T, color, f0, n):
        """The ctypes records of frames f0 .. f0 + n - 1 (checked inputs)."""
        return (Frame * n)(*[self._frame(depth[f], None if color is None else color[f], K[f], T[f]) for f in range(f0, f0 + n)])

    def _allocate(self, frames, H, W):
        """One pass's allocation: bricks for every cell the frames can update, the pool grown to hold them, and the pass's
        cells listed in self._touched; returns their count (one host read of the device counters)."""
        L = _bind()
        while True:
            self._epoch += 1
            self._counters[1].zero_()
            lib.check(L.scsfm_fusion_alloc(frames, len(frames), H, W, ctypes.byref(self._vol), lib.ptr(self._index),
                                           lib.ptr(self._stamp), self._epoch, lib.ptr(self._counters), lib.ptr(self._touched),
                                           self._touched.numel(), lib.stream()), "scsfm_fusion_alloc")
            bricks, touched = (int(x) for x in self._counters.cpu())
            self._grow(bricks)
            if touched <= self._touched.numel():
                break
            self._touched = torch.empty(_doubled(self._touched.numel(), touched), dtype=torch.int32, device=self.device)
        self._bricks = bricks
        return touched

    def _listed(self, touched):
        """int32 [touched]: the cells of the last pass _allocate listed."""
        return self._touched[:touched]

    def _apply(self, frames, H, W, touched):
        """One pass's integration of the frames into the `touched` cells _allocate listed."""
        self.brick_visits += touched
        lib.check(_bind().scsfm_fusion_integrate(frames, len(frames), H, W, ctypes.byref(self._vol), lib.ptr(self._index),
                                                 lib.ptr(self._touched), touched, lib.ptr(self._pool), lib.stream()),
                  "scsfm_fusion_integrate")

    def _grow(self, bricks):
        cap = self._pool.shape[0]
        if bricks <= cap:
            return
        pool = torch.zeros(_doubled(cap, bricks), FIELDS, BRICK ** 3, dtype=torch.float32, device=self.device)
        pool[:cap].copy_(self._pool)
        self._pool = pool

    # ----- reading ---------------------------------------------------------------------------------------------------------
    def sample(self, ijk):
        """(tsdf, weight, rgb) of voxels ijk int64 [N,3] (device tensor): fp32 [N], [N], [N,3]; voxels in no brick or outside the
        box read all zeros (w = 0)."""
        if not isinstance(ijk, torch.Tensor):
            raise TypeError("ijk must be a torch tensor, got %s" % type(ijk).__name__)
        if ijk.dtype != torch.int64:
            raise TypeError("ijk must be int64, got %s" % ijk.dtype)
        if ijk.dim() != 2 or ijk.shape[1] != 3:
            raise ValueError("ijk must be [N,3], got %s" % list(ijk.shape))
        if ijk.device != self.device:
            raise ValueError("ijk must be on %s, got %s" % (self.device, ijk.device))
        ijk = ijk.contiguous()
        out = torch.empty(ijk.shape[0], FIELDS, dtype=torch.float32, device=self.device)
        lib.check(_bind().scsfm_fusion_sample(ctypes.byref(self._vol), lib.ptr(self._index), lib.ptr(self._pool), lib.ptr(ijk),
                                              ijk.shape[0], lib.ptr(out), lib.stream()), "scsfm_fusion_sample")
        return out[:, 0], out[:, 1], out[:, 2:]

    def brick_voxels(self):
        """int64 [num_bricks * 512, 3]: the indices of every voxel in an allocated brick, brick by brick."""
        return self._cell_voxels(self._cells())

    def _cell_voxels(self, cells):
        """int64 [len(cells) * 512, 3]: the voxel indices of the cells' bricks, in the pool's order within a brick."""
        cells = cells.long()
        nx, ny = int(self.nb[0]), int(self.nb[1])
        b = torch.stack([cells % nx, (cells // nx) % ny, cells // (nx * ny)], 1) * BRICK
        t = torch.arange(BRICK ** 3, device=self.device)
        local = torch.stack([t % 8, (t // 8) % 8, t // 64], 1)
        return (b[:, None, :] + local[None]).reshape(-1, 3)

    def _cell_fields(self, cells):
        """fp32 [5, len(cells) * 512] copy of tsdf, w, r, g, b of the cells' bricks, voxels in _cell_voxels' order."""
        return self._pool[self._index[cells.long()].long()].permute(1, 0, 2).reshape(FIELDS, -1)

    def _set_cell_fields(self, cells, fields):
        """Write back fields [5, len(cells) * 512] as _cell_fields returns them."""
        self._pool[self._index[cells.long()].long()] = fields.reshape(FIELDS, -1, BRICK ** 3).permute(1, 0, 2)

    def _cells(self):
        return torch.nonzero(self._index >= 0).flatten().to(torch.int32)

    def mesh(self, with_keys=False):
        """Marching cubes over the allocated bricks: (verts float32 [V,3] in world units, faces int64 [F,3], colors uint8 [V,3]),
        vertices welded across cells and bricks (one per edge of the voxel grid), ordered by edge key.  with_keys=True also
        returns the keys int64 [V] (the edge's lower voxel's linear index (k ny + j) nx + i, times 3, plus the axis)."""
        L, s = _bind(), lib.stream()
        cells = self._cells()
        n = cells.numel()
        dev = self.device
        empty = (torch.zeros(0, 3, dtype=torch.float32, device=dev), torch.zeros(0, 3, dtype=torch.int64, device=dev),
                 torch.zeros(0, 3, dtype=torch.uint8, device=dev))
        if n == 0:
            return empty + (torch.zeros(0, dtype=torch.int64, device=dev),) if with_keys else empty
        counts = torch.empty(n * BRICK ** 3, dtype=torch.int32, device=dev)
        lib.check(L.scsfm_fusion_mesh_count(ctypes.byref(self._vol), lib.ptr(self._index), lib.ptr(self._pool), lib.ptr(cells), n,
                                            lib.ptr(self._tri), lib.ptr(counts), s), "scsfm_fusion_mesh_count")
        ends = torch.cumsum(counts, 0, dtype=torch.int64)
        total = int(ends[-1])
        if total == 0:
            return empty + (torch.zeros(0, dtype=torch.int64, device=dev),) if with_keys else empty
        offsets = ends - counts
        keys = torch.empty(total * 3, dtype=torch.int64, device=dev)
        pos = torch.empty(total * 3, 3, dtype=torch.float32, device=dev)
        col = torch.empty(total * 3, 3, dtype=torch.uint8, device=dev)
        lib.check(L.scsfm_fusion_mesh_emit(ctypes.byref(self._vol), lib.ptr(self._index), lib.ptr(self._pool), lib.ptr(cells), n,
                                           lib.ptr(self._tri), lib.ptr(offsets), lib.ptr(keys), lib.ptr(pos), lib.ptr(col), s),
                  "scsfm_fusion_mesh_emit")
        uniq, inv = torch.unique(keys, return_inverse=True)
        verts = torch.empty(uniq.numel(), 3, dtype=torch.float32, device=dev)
        colors = torch.empty(uniq.numel(), 3, dtype=torch.uint8, device=dev)
        verts[inv] = pos              # every copy of a vertex holds the same bits
        colors[inv] = col
        out = (verts, inv.view(-1, 3), colors)
        return out + (uniq,) if with_keys else out


def _doubled(cap, need):
    while cap < need:
        cap *= 2
    return cap
