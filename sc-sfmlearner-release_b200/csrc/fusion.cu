// Dense reconstruction: frames of depth (and colour) fused into a truncated signed distance field on a two-level grid, and
// the field meshed by marching cubes (scsfm/fusion.py owns the memory and the layout; include/scsfm.h states the semantics).
//
// Layout.  The volume's box holds nb[0] x nb[1] x nb[2] bricks of 8^3 voxels.  index[cell] (cell = (bz * nb1 + by) * nb0 + bx)
// is the cell's brick id or -1 (-2 for the moment between claiming a cell and publishing its id).  Brick b's voxels are
// pool[b][field][512], fields tsdf, w, r, g, b (fp32), voxel (x, y, z) of the brick at x + 8 y + 64 z.
//
//  * fusion_alloc_kernel: one thread per pixel of each frame.  A valid depth d puts every voxel that pixel can update inside
//    the frustum piece between depths max(d - trunc, 0) and d + trunc over the pixel's square; the thread claims every brick
//    that meets the world-space box of that piece's 8 corners (grown by a small margin for fp32 rounding) and lists each
//    brick once per batch through a per-cell stamp.
//  * fusion_integrate_kernel: one CTA per listed brick, one thread per voxel; the voxel stays in registers while the thread
//    applies the batch's frames in order (their matrices are kernel parameters, in the constant bank), then it is written
//    back once.  The voxel traffic, 40 bytes per voxel per batch, is the kernel's cost; the depth maps stay in L2.
//  * fusion_mesh_kernel: one CTA per allocated brick, one thread per cell (the cube whose lowest corner is the voxel); corner
//    voxels in neighbouring bricks are read through the index.  Pass 0 counts each cell's triangles, pass 1 writes them
//    at the cell's offset of the exclusive scan: three edge keys, vertex positions and colours per triangle.
#include "common.cuh"

namespace scsfm {

constexpr int BRICK_VOXELS = 512;
constexpr int ALLOC_THREADS = 256;

struct FusionFrames {
    ScsfmFusionFrame f[SCSFM_FUSION_MAX_FRAMES];
};

__device__ __forceinline__ long long cell_of(const ScsfmFusionVolume& v, int bx, int by, int bz) {
    return ((long long)bz * v.nb[1] + by) * v.nb[0] + bx;
}

__global__ void __launch_bounds__(ALLOC_THREADS)
fusion_alloc_kernel(const __grid_constant__ FusionFrames fr, int H, int W, const __grid_constant__ ScsfmFusionVolume vol,
                    int* __restrict__ index, int* __restrict__ stamp, int epoch, int* __restrict__ counters,
                    int* __restrict__ touched, int touched_cap) {
    const long long p = (long long)blockIdx.x * ALLOC_THREADS + threadIdx.x;
    if (p >= (long long)H * W) return;
    const ScsfmFusionFrame& F = fr.f[blockIdx.y];
    const float d = __ldg(F.depth + p);
    if (!(d > 0.f && d <= vol.max_depth)) return;
    const int py = (int)(p / W), px = (int)(p - (long long)py * W);
    const float zs[2] = {fmaxf(d - vol.trunc, 0.f), d + vol.trunc};
    float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const float u = px + ((c & 1) ? 0.5f : -0.5f), v = py + ((c & 2) ? 0.5f : -0.5f), z = zs[c >> 2];
        const float xc = (u - F.cx) / F.fx * z, yc = (v - F.cy) / F.fy * z;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float w = F.R_cw[3 * a] * xc + F.R_cw[3 * a + 1] * yc + F.R_cw[3 * a + 2] * z + F.t_cw[a];
            mn[a] = fminf(mn[a], w);
            mx[a] = fmaxf(mx[a], w);
        }
    }
    const float bs = 8.f * vol.voxel, margin = 0.05f * vol.voxel;
    int lo[3], hi[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float l = floorf((mn[a] - margin - vol.lo[a]) / bs), h = floorf((mx[a] + margin - vol.lo[a]) / bs);
        if (!(h >= 0.f && l < (float)vol.nb[a])) return;        // outside the box (or NaN)
        lo[a] = l < 0.f ? 0 : (int)l;
        hi[a] = h >= (float)vol.nb[a] ? vol.nb[a] - 1 : (int)h;
    }
    for (int bz = lo[2]; bz <= hi[2]; ++bz)
        for (int by = lo[1]; by <= hi[1]; ++by)
            for (int bx = lo[0]; bx <= hi[0]; ++bx) {
                const long long cell = cell_of(vol, bx, by, bz);
                if (*(volatile int*)(index + cell) == -1 && atomicCAS(index + cell, -1, -2) == -1)
                    atomicExch(index + cell, atomicAdd(counters, 1));
                if (*(volatile int*)(stamp + cell) != epoch && atomicExch(stamp + cell, epoch) != epoch) {
                    const int s = atomicAdd(counters + 1, 1);
                    if (s < touched_cap) touched[s] = (int)cell;
                }
            }
}

__global__ void __launch_bounds__(BRICK_VOXELS)
fusion_integrate_kernel(const __grid_constant__ FusionFrames fr, int F, int H, int W, const __grid_constant__ ScsfmFusionVolume vol,
                        const int* __restrict__ index, const int* __restrict__ touched, float* __restrict__ pool) {
    const int cell = touched[blockIdx.x];
    const int id = index[cell];
    const int t = threadIdx.x;
    const long long bx = cell % vol.nb[0], by = (cell / vol.nb[0]) % vol.nb[1], bz = cell / ((long long)vol.nb[0] * vol.nb[1]);
    const float v = vol.voxel;
    // voxel indices in 64-bit, as voxel_at computes them: an axis may hold up to 2^31 - 1 bricks
    const float pw[3] = {vol.lo[0] + ((float)(bx * 8 + (t & 7)) + 0.5f) * v, vol.lo[1] + ((float)(by * 8 + ((t >> 3) & 7)) + 0.5f) * v,
                         vol.lo[2] + ((float)(bz * 8 + (t >> 6)) + 0.5f) * v};
    float* P = pool + (size_t)id * 5 * BRICK_VOXELS + t;
    float tsdf = P[0], w = P[BRICK_VOXELS], r = P[2 * BRICK_VOXELS], g = P[3 * BRICK_VOXELS], b = P[4 * BRICK_VOXELS];
    const float w0 = w;
    for (int f = 0; f < F; ++f) {
        const ScsfmFusionFrame& Fr = fr.f[f];
        const float x = Fr.R_wc[0] * pw[0] + Fr.R_wc[1] * pw[1] + Fr.R_wc[2] * pw[2] + Fr.t_wc[0];
        const float y = Fr.R_wc[3] * pw[0] + Fr.R_wc[4] * pw[1] + Fr.R_wc[5] * pw[2] + Fr.t_wc[1];
        const float z = Fr.R_wc[6] * pw[0] + Fr.R_wc[7] * pw[1] + Fr.R_wc[8] * pw[2] + Fr.t_wc[2];
        if (!(z > 0.f)) continue;
        const float iu = floorf(Fr.fx * x / z + Fr.cx + 0.5f), iv = floorf(Fr.fy * y / z + Fr.cy + 0.5f);
        if (!(iu >= 0.f && iu < (float)W && iv >= 0.f && iv < (float)H)) continue;
        const int pix = (int)iv * W + (int)iu;
        const float d = __ldg(Fr.depth + pix);
        if (!(d > 0.f && d <= vol.max_depth)) continue;
        const float sdf = d - z;
        if (!(fabsf(sdf) <= vol.trunc)) continue;
        const float wn = w + 1.f;
        tsdf = (tsdf * w + sdf / vol.trunc) / wn;
        if (Fr.color) {
            const unsigned char* c = Fr.color + (size_t)pix * 3;
            r = (r * w + (float)c[0]) / wn;
            g = (g * w + (float)c[1]) / wn;
            b = (b * w + (float)c[2]) / wn;
        }
        w = wn;
    }
    if (w != w0) {
        P[0] = tsdf;
        P[BRICK_VOXELS] = w;
        P[2 * BRICK_VOXELS] = r;
        P[3 * BRICK_VOXELS] = g;
        P[4 * BRICK_VOXELS] = b;
    }
}

// the pool address of voxel (i, j, k), or null when it is outside the box or in no brick
__device__ __forceinline__ const float* voxel_at(const ScsfmFusionVolume& vol, const int* __restrict__ index,
                                                 const float* __restrict__ pool, long long i, long long j, long long k) {
    if (i < 0 || j < 0 || k < 0 || i >= 8LL * vol.nb[0] || j >= 8LL * vol.nb[1] || k >= 8LL * vol.nb[2]) return nullptr;
    const int id = __ldg(index + cell_of(vol, (int)(i >> 3), (int)(j >> 3), (int)(k >> 3)));
    if (id < 0) return nullptr;
    return pool + (size_t)id * 5 * BRICK_VOXELS + ((k & 7) * 64 + (j & 7) * 8 + (i & 7));
}

__global__ void fusion_sample_kernel(const __grid_constant__ ScsfmFusionVolume vol, const int* __restrict__ index,
                                     const float* __restrict__ pool, const long long* __restrict__ ijk, long long n,
                                     float* __restrict__ out) {
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n) return;
    const float* P = voxel_at(vol, index, pool, ijk[3 * q], ijk[3 * q + 1], ijk[3 * q + 2]);
#pragma unroll
    for (int f = 0; f < 5; ++f) out[5 * q + f] = P ? P[f * BRICK_VOXELS] : 0.f;
}

__constant__ signed char c_corner[8][3] = {{0, 0, 0}, {1, 0, 0}, {1, 1, 0}, {0, 1, 0}, {0, 0, 1}, {1, 0, 1}, {1, 1, 1}, {0, 1, 1}};
__constant__ signed char c_edge[12][2] = {{0, 1}, {1, 2}, {2, 3}, {3, 0}, {4, 5}, {5, 6}, {6, 7}, {7, 4}, {0, 4}, {1, 5}, {2, 6}, {3, 7}};

// pass 0: counts[brick slot * 512 + voxel] = triangles of the cell; pass 1: writes them at offsets[...] (triangles)
__global__ void __launch_bounds__(BRICK_VOXELS)
fusion_mesh_kernel(int pass, const __grid_constant__ ScsfmFusionVolume vol, const int* __restrict__ index,
                   const float* __restrict__ pool, const int* __restrict__ cells, const signed char* __restrict__ tri_table,
                   int* __restrict__ counts, const long long* __restrict__ offsets, long long* __restrict__ keys,
                   float* __restrict__ verts, unsigned char* __restrict__ colors) {
    __shared__ signed char tab[256 * 16];
    for (int i = threadIdx.x; i < 256 * 16; i += BRICK_VOXELS) tab[i] = tri_table[i];
    __syncthreads();
    const int cell = cells[blockIdx.x];
    const int t = threadIdx.x;
    const long long i0 = (long long)(cell % vol.nb[0]) * 8 + (t & 7), j0 = (long long)((cell / vol.nb[0]) % vol.nb[1]) * 8 + ((t >> 3) & 7),
                    k0 = (long long)(cell / ((long long)vol.nb[0] * vol.nb[1])) * 8 + (t >> 6);
    const float* P[8];
    int config = 0;
    bool ok = true;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        P[c] = voxel_at(vol, index, pool, i0 + c_corner[c][0], j0 + c_corner[c][1], k0 + c_corner[c][2]);
        if (!P[c] || !(P[c][BRICK_VOXELS] > 0.f)) {
            ok = false;
            break;
        }
        if (P[c][0] < 0.f) config |= 1 << c;
    }
    const signed char* row = tab + (ok ? config : 0) * 16;
    int n = 0;
    while (n < 5 && row[3 * n] >= 0) ++n;
    const long long slot = (long long)blockIdx.x * BRICK_VOXELS + t;
    if (pass == 0) {
        counts[slot] = n;
        return;
    }
    const long long base = offsets[slot] * 3;
    const long long nx = 8LL * vol.nb[0], ny = 8LL * vol.nb[1];
    for (int q = 0; q < 3 * n; ++q) {
        const int e = row[q];
        const int a = c_edge[e][0], b = c_edge[e][1];
        // corner 0 of the edge is its lower voxel, so the cells sharing an edge compute the same vertex bit for bit
        const int lo = (c_corner[a][0] + c_corner[a][1] + c_corner[a][2] < c_corner[b][0] + c_corner[b][1] + c_corner[b][2]) ? a : b;
        const int hi = lo == a ? b : a;
        const int axis = c_corner[hi][0] != c_corner[lo][0] ? 0 : (c_corner[hi][1] != c_corner[lo][1] ? 1 : 2);
        const long long li = i0 + c_corner[lo][0], lj = j0 + c_corner[lo][1], lk = k0 + c_corner[lo][2];
        keys[base + q] = ((lk * ny + lj) * nx + li) * 3 + axis;
        const double s0 = P[lo][0], s1 = P[hi][0];
        const double tt = __ddiv_rn(s0, __dsub_rn(s0, s1));
        const long long ijk[3] = {li, lj, lk};
#pragma unroll
        for (int x = 0; x < 3; ++x) {
            const double g = __dadd_rn((double)ijk[x], 0.5);
            const double pos = __dadd_rn(vol.lo_d[x], __dmul_rn(x == axis ? __dadd_rn(g, tt) : g, vol.voxel_d));
            verts[(base + q) * 3 + x] = (float)pos;
            const double c0 = P[lo][(2 + x) * BRICK_VOXELS], c1 = P[hi][(2 + x) * BRICK_VOXELS];
            const double c = rint(__dadd_rn(c0, __dmul_rn(tt, __dsub_rn(c1, c0))));
            colors[(base + q) * 3 + x] = (unsigned char)(c < 0.0 ? 0.0 : (c > 255.0 ? 255.0 : c));
        }
    }
}

int check_volume(const ScsfmFusionVolume* vol, const char* what) {
    SCSFM_CHECK_ARG(vol, "%s: null volume", what);
    SCSFM_CHECK_ARG(vol->nb[0] > 0 && vol->nb[1] > 0 && vol->nb[2] > 0, "%s: brick counts must be positive, got %d x %d x %d",
                    what, vol->nb[0], vol->nb[1], vol->nb[2]);
    const long long cells = (long long)vol->nb[0] * vol->nb[1] * vol->nb[2];
    SCSFM_CHECK_ARG(cells < (1LL << 31), "%s: %d x %d x %d = %lld bricks in the coarse index, more than 2^31 - 1", what, vol->nb[0],
                    vol->nb[1], vol->nb[2], cells);
    SCSFM_CHECK_ARG(vol->voxel > 0.f && vol->trunc > 0.f && vol->max_depth > 0.f,
                    "%s: voxel size, truncation and max depth must be positive, got %g %g %g", what, vol->voxel, vol->trunc,
                    vol->max_depth);
    return SCSFM_OK;
}

int check_frames(const ScsfmFusionFrame* frames, int F, int H, int W, const char* what) {
    SCSFM_CHECK_ARG(frames, "%s: null frames", what);
    SCSFM_CHECK_ARG(F > 0 && F <= SCSFM_FUSION_MAX_FRAMES, "%s: frame count must be 1..%d, got %d", what, SCSFM_FUSION_MAX_FRAMES, F);
    SCSFM_CHECK_ARG(H > 0 && W > 0, "%s: image size must be positive, got %d x %d", what, H, W);
    for (int f = 0; f < F; ++f) SCSFM_CHECK_ARG(frames[f].depth, "%s: frame %d has a null depth map", what, f);
    return SCSFM_OK;
}

}  // namespace scsfm

using namespace scsfm;

extern "C" int scsfm_fusion_alloc(const ScsfmFusionFrame* frames, int F, int H, int W, const ScsfmFusionVolume* vol, int* index,
                                  int* stamp, int epoch, int* counters, int* touched, int touched_cap, void* stream) {
    int rc = check_frames(frames, F, H, W, "fusion_alloc");
    if (rc == SCSFM_OK) rc = check_volume(vol, "fusion_alloc");
    if (rc != SCSFM_OK) return rc;
    SCSFM_CHECK_ARG(index && stamp && counters && touched, "fusion_alloc: null pointer (index, stamp, counters and touched are "
                    "required)");
    SCSFM_CHECK_ARG(epoch > 0 && touched_cap > 0, "fusion_alloc: epoch and touched capacity must be positive, got %d %d", epoch,
                    touched_cap);
    FusionFrames fr;
    for (int f = 0; f < F; ++f) fr.f[f] = frames[f];
    const dim3 grid((unsigned)(((long long)H * W + ALLOC_THREADS - 1) / ALLOC_THREADS), F);
    fusion_alloc_kernel<<<grid, ALLOC_THREADS, 0, (cudaStream_t)stream>>>(fr, H, W, *vol, index, stamp, epoch, counters, touched,
                                                                          touched_cap);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_fusion_integrate(const ScsfmFusionFrame* frames, int F, int H, int W, const ScsfmFusionVolume* vol,
                                      const int* index, const int* touched, int n_touched, float* pool, void* stream) {
    int rc = check_frames(frames, F, H, W, "fusion_integrate");
    if (rc == SCSFM_OK) rc = check_volume(vol, "fusion_integrate");
    if (rc != SCSFM_OK) return rc;
    SCSFM_CHECK_ARG(index && touched && pool, "fusion_integrate: null pointer (index, touched and pool are required)");
    SCSFM_CHECK_ARG(n_touched >= 0, "fusion_integrate: negative brick count %d", n_touched);
    if (n_touched == 0) return SCSFM_OK;
    FusionFrames fr;
    for (int f = 0; f < F; ++f) fr.f[f] = frames[f];
    fusion_integrate_kernel<<<n_touched, BRICK_VOXELS, 0, (cudaStream_t)stream>>>(fr, F, H, W, *vol, index, touched, pool);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_fusion_sample(const ScsfmFusionVolume* vol, const int* index, const float* pool, const long long* ijk,
                                   long long n, float* out, void* stream) {
    int rc = check_volume(vol, "fusion_sample");
    if (rc != SCSFM_OK) return rc;
    SCSFM_CHECK_ARG(index && pool && ijk && out, "fusion_sample: null pointer (index, pool, ijk and out are required)");
    SCSFM_CHECK_ARG(n >= 0, "fusion_sample: negative voxel count %lld", n);
    if (n == 0) return SCSFM_OK;
    fusion_sample_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(*vol, index, pool, ijk, n, out);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_fusion_mesh_count(const ScsfmFusionVolume* vol, const int* index, const float* pool, const int* cells,
                                       int n_bricks, const signed char* tri_table, int* counts, void* stream) {
    int rc = check_volume(vol, "fusion_mesh_count");
    if (rc != SCSFM_OK) return rc;
    SCSFM_CHECK_ARG(index && pool && cells && tri_table && counts, "fusion_mesh_count: null pointer (index, pool, cells, tri_table "
                    "and counts are required)");
    SCSFM_CHECK_ARG(n_bricks > 0, "fusion_mesh_count: brick count must be positive, got %d", n_bricks);
    fusion_mesh_kernel<<<n_bricks, BRICK_VOXELS, 0, (cudaStream_t)stream>>>(0, *vol, index, pool, cells, tri_table, counts, nullptr,
                                                                            nullptr, nullptr, nullptr);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_fusion_mesh_emit(const ScsfmFusionVolume* vol, const int* index, const float* pool, const int* cells,
                                      int n_bricks, const signed char* tri_table, const long long* offsets, long long* keys,
                                      float* verts, unsigned char* colors, void* stream) {
    int rc = check_volume(vol, "fusion_mesh_emit");
    if (rc != SCSFM_OK) return rc;
    SCSFM_CHECK_ARG(index && pool && cells && tri_table && offsets && keys && verts && colors,
                    "fusion_mesh_emit: null pointer (index, pool, cells, tri_table, offsets, keys, verts and colors are required)");
    SCSFM_CHECK_ARG(n_bricks > 0, "fusion_mesh_emit: brick count must be positive, got %d", n_bricks);
    fusion_mesh_kernel<<<n_bricks, BRICK_VOXELS, 0, (cudaStream_t)stream>>>(1, *vol, index, pool, cells, tri_table, nullptr, offsets,
                                                                            keys, verts, colors);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}
