// Training-set preparation on the device (data/prepare_train_data.py, scsfm/prepare.py).  The host decodes PNGs and reads the
// Velodyne .bin files; two kernel families do the per-frame arithmetic, bit for bit what the reference's tool computed:
//
//  * resize_bilinear_u8: PIL.Image.resize((w, h), Image.BILINEAR) on uint8 HWC RGB frames (what scipy.misc.imresize did),
//    Pillow's src/libImaging/Resample.c: triangle filter of support max(in/out, 1), coefficients from precompute_coeffs in
//    double with every operation explicitly rounded (__dmul_rn, ...: no FMA contraction), normalised and rounded to 22-bit
//    fixed point with the sign-aware rounding of normalize_coeffs_8bpc, horizontal pass into an 8-bit intermediate, then the
//    vertical pass.  A pass whose axis keeps its size is skipped, as Pillow skips it.  The tap count grows with the
//    downscale: 5 for 1242 -> 832, 7 for 2048 -> 832.
//  * velo_depth: the reference's generate_depth_map (kitti_raw_loader.py) for a batch of clouds in CSR layout.  For every
//    point with x >= 0: u = P_velo2im [x y z 1] in fp64 in a fixed order, px = rint(u0/u2) - 1, py = rint(u1/u2) - 1 (half to
//    even, like np.round), kept inside the Wd x Hd map.  Per pixel the map holds (a) float32(z) of the LAST point on it
//    (numpy's repeated-index assignment), except that (b) for every key with >= 2 points the pixel of the key's FIRST point
//    gets float32(min z) of the key; keys are py * (Wd - 1) + px - 1 (the reference's sub2ind), so pixel (y, Wd-1) and
//    pixel (y+1, 0) share one; (c) negative values become 0.  Per-pixel atomics (count, first and last point, min z as an
//    order-preserving integer) and a resolve pass that reads the row-edge partner: the result does not depend on thread order.
#include "common.cuh"

namespace scsfm {

constexpr int PREP_PRECISION_BITS = 32 - 8 - 2;
constexpr int PREP_MAX_TAPS = 63;            // 2 * ceil(support) + 1: downscales of up to 31x

// Resample.c bilinear_filter
__device__ __forceinline__ double prep_triangle(double x) {
    if (x < 0.0) x = -x;
    return x < 1.0 ? __dsub_rn(1.0, x) : 0.0;
}

// One output coordinate of one axis: coef[j] = {xmin, n, k_0 .. k_{ksize-1}} (precompute_coeffs + normalize_coeffs_8bpc,
// box (0, in_size)).  The unnormalised weights are kept in the integer slots as doubles would not fit: two passes instead.
__global__ void prep_coeffs_kernel(int in_size, int out_size, int ksize, int* __restrict__ coef) {
    const int xx = blockIdx.x * blockDim.x + threadIdx.x;
    if (xx >= out_size) return;
    const double scale = __ddiv_rn((double)in_size, (double)out_size);
    const double filterscale = scale > 1.0 ? scale : 1.0;
    const double support = filterscale;                        // bilinear support 1.0 * filterscale
    const double ss = __ddiv_rn(1.0, filterscale);
    const double center = __dmul_rn(__dadd_rn((double)xx, 0.5), scale);
    int xmin = __double2int_rz(__dadd_rn(__dsub_rn(center, support), 0.5));
    if (xmin < 0) xmin = 0;
    int xmax = __double2int_rz(__dadd_rn(__dadd_rn(center, support), 0.5));
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    if (xmax > ksize) xmax = ksize;                            // (cannot happen: ksize = 2 * ceil(support) + 1)
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x)
        ww = __dadd_rn(ww, prep_triangle(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + xmin), center), 0.5), ss)));
    int* o = coef + (size_t)xx * (ksize + 2);
    o[0] = xmin;
    o[1] = xmax;
    for (int x = 0; x < ksize; ++x) {
        int k = 0;
        if (x < xmax) {
            const double w = prep_triangle(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + xmin), center), 0.5), ss));
            const double v = ww != 0.0 ? __ddiv_rn(w, ww) : w;
            const double s = __dmul_rn(v, (double)(1 << PREP_PRECISION_BITS));
            k = v < 0 ? __double2int_rz(__dadd_rn(-0.5, s)) : __double2int_rz(__dadd_rn(0.5, s));
        }
        o[2 + x] = k;
    }
}

__device__ __forceinline__ unsigned char prep_clip8(int v) {
    v >>= PREP_PRECISION_BITS;
    return (unsigned char)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// One pass of the separable resample over B frames of [rows][cols][3] uint8.  Horizontal (vertical == false): out is
// [B][rows][out_n][3], taps run along the columns.  Vertical: out is [B][out_n][cols][3], taps run along the rows.
// One thread per output pixel (three channels); grid: (x blocks, y, B).
template <bool VERTICAL>
__global__ void __launch_bounds__(256)
prep_resample_kernel(const unsigned char* __restrict__ in, int rows, int cols, int out_n, const int* __restrict__ coef, int ksize,
                     unsigned char* __restrict__ out) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    const int b = blockIdx.z;
    const int out_cols = VERTICAL ? cols : out_n;
    if (x >= out_cols) return;
    const int* k = coef + (size_t)(VERTICAL ? y : x) * (ksize + 2);
    const int first = k[0], n = k[1];
    const unsigned char* src = in + (size_t)b * rows * cols * 3;
    int acc[3] = {1 << (PREP_PRECISION_BITS - 1), 1 << (PREP_PRECISION_BITS - 1), 1 << (PREP_PRECISION_BITS - 1)};
    for (int i = 0; i < n; ++i) {
        const unsigned char* px = VERTICAL ? src + ((size_t)(first + i) * cols + x) * 3 : src + ((size_t)y * cols + first + i) * 3;
        const int w = k[2 + i];
        acc[0] += (int)__ldg(px) * w;
        acc[1] += (int)__ldg(px + 1) * w;
        acc[2] += (int)__ldg(px + 2) * w;
    }
    unsigned char* o = out + (((size_t)b * (VERTICAL ? out_n : rows) + y) * out_cols + x) * 3;
    o[0] = prep_clip8(acc[0]);
    o[1] = prep_clip8(acc[1]);
    o[2] = prep_clip8(acc[2]);
}

// ----- Velodyne -> depth map ------------------------------------------------------------------------------------------------

// per-pixel workspace: count, first point, last point, min float32(z) as an order-preserving key
struct DepthCell {
    int count, first, last;
    unsigned int minz;
};

__device__ __forceinline__ unsigned int f32_order_key(float f) {
    const unsigned int u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float f32_from_order_key(unsigned int k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// u = P [x y z 1] with the products and sums rounded one by one, left to right; false if the point is dropped
__device__ __forceinline__ bool velo_project(const float* __restrict__ pt, const double* __restrict__ P, int Hd, int Wd, int* pix,
                                             double* z) {
    const float xf = pt[0];
    if (!(xf >= 0.f)) return false;                             // velo[velo[:, 0] >= 0]
    const double x = (double)xf, y = (double)pt[1], zz = (double)pt[2];
    double u[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const double* p = P + 4 * r;
        u[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(p[0], x), __dmul_rn(p[1], y)), __dmul_rn(p[2], zz)), p[3]);
    }
    const double px = rint(__ddiv_rn(u[0], u[2])) - 1.0;       // integers: the subtraction is exact
    const double py = rint(__ddiv_rn(u[1], u[2])) - 1.0;
    if (!(px >= 0.0 && py >= 0.0 && px < (double)Wd && py < (double)Hd)) return false;   // NaN and inf fall out here
    *pix = (int)py * Wd + (int)px;
    *z = u[2];
    return true;
}

__global__ void velo_init_kernel(DepthCell* __restrict__ cells, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) cells[i] = DepthCell{0, 0x7fffffff, -1, 0xffffffffu};
}

// one thread per point; grid: (point blocks, frames)
__global__ void __launch_bounds__(256)
velo_scatter_kernel(const float* __restrict__ points, const long long* __restrict__ offsets, const double* __restrict__ P, int Hd, int Wd,
                    DepthCell* __restrict__ cells) {
    const int b = blockIdx.y;
    const long long p0 = offsets[b], np = offsets[b + 1] - p0;
    const double* Pb = P + 12 * b;
    DepthCell* cb = cells + (size_t)b * Hd * Wd;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < np; i += (long long)gridDim.x * blockDim.x) {
        int pix;
        double z;
        if (!velo_project(points + 4 * (p0 + i), Pb, Hd, Wd, &pix, &z)) continue;
        DepthCell* c = cb + pix;
        atomicAdd(&c->count, 1);
        atomicMin(&c->first, (int)i);
        atomicMax(&c->last, (int)i);
        atomicMin(&c->minz, f32_order_key((float)z));
    }
}

// one thread per pixel; grid: (pixel blocks, frames)
__global__ void __launch_bounds__(256)
velo_resolve_kernel(const float* __restrict__ points, const long long* __restrict__ offsets, const double* __restrict__ P, int Hd, int Wd,
                    const DepthCell* __restrict__ cells, float* __restrict__ depth) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Hd * Wd) return;
    const DepthCell* cb = cells + (size_t)b * Hd * Wd;
    const DepthCell c = cb[i];
    float v = 0.f;
    if (c.count > 0) {
        int pix;
        double z = 0.0;
        velo_project(points + 4 * (offsets[b] + c.last), P + 12 * b, Hd, Wd, &pix, &z);   // (a) the last point on the pixel
        v = (float)z;
        // the row-edge partner that shares this pixel's key: (y, Wd-1) <-> (y+1, 0)
        const int x = i % Wd, y = i / Wd;
        int partner = -1;
        if (x == Wd - 1 && y + 1 < Hd) partner = i + 1;
        else if (x == 0 && y > 0) partner = i - 1;
        int count = c.count, first_other = 0x7fffffff;
        unsigned int minz = c.minz;
        if (partner >= 0) {
            const DepthCell q = cb[partner];
            count += q.count;
            first_other = q.first;
            minz = min(minz, q.minz);
        }
        if (count >= 2 && c.first < first_other) v = f32_from_order_key(minz);   // (b) the key's first point is here
        if (v < 0.f) v = 0.f;                                                      // (c)
    }
    depth[(size_t)b * Hd * Wd + i] = v;
}

}  // namespace scsfm

using namespace scsfm;

static int prep_taps(int in_size, int out_size) {
    const double scale = (double)in_size / (double)out_size;
    const double support = scale > 1.0 ? scale : 1.0;
    return (int)ceil(support) * 2 + 1;
}

extern "C" size_t scsfm_resize_bilinear_workspace_bytes(int B, int H, int W, int out_h, int out_w) {
    if (B <= 0 || H <= 0 || W <= 0 || out_h <= 0 || out_w <= 0) return 0;
    size_t coef = ((size_t)out_w * (prep_taps(W, out_w) + 2) + (size_t)out_h * (prep_taps(H, out_h) + 2)) * sizeof(int);
    coef = (coef + 255) & ~(size_t)255;
    const size_t tmp = (W != out_w && H != out_h) ? (size_t)B * H * out_w * 3 : 0;
    return coef + tmp;
}

extern "C" int scsfm_resize_bilinear_u8(const unsigned char* in, int B, int H, int W, int out_h, int out_w, unsigned char* out,
                                        void* workspace, size_t workspace_bytes, void* stream) {
    SCSFM_CHECK_ARG(in && out, "resize_bilinear_u8: null pointer");
    SCSFM_CHECK_ARG(B > 0 && H > 0 && W > 0 && out_h > 0 && out_w > 0, "resize_bilinear_u8: bad geometry");
    SCSFM_CHECK_ARG(B <= 65535 && H <= 65535 && out_h <= 65535, "resize_bilinear_u8: too many frames / rows for one launch");
    const int kx = prep_taps(W, out_w), ky = prep_taps(H, out_h);
    SCSFM_CHECK_ARG(kx <= PREP_MAX_TAPS && ky <= PREP_MAX_TAPS, "resize_bilinear_u8: downscale by more than 31x");
    SCSFM_CHECK_ARG(workspace_bytes >= scsfm_resize_bilinear_workspace_bytes(B, H, W, out_h, out_w),
                    "resize_bilinear_u8: workspace too small (scsfm_resize_bilinear_workspace_bytes)");
    SCSFM_CHECK_ARG(workspace && (reinterpret_cast<uintptr_t>(workspace) & 15) == 0, "resize_bilinear_u8: workspace must be 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    const bool need_h = W != out_w, need_v = H != out_h;
    if (!need_h && !need_v) {                                   // Pillow returns a copy
        SCSFM_CHECK_CUDA(cudaMemcpyAsync(out, in, (size_t)B * H * W * 3, cudaMemcpyDeviceToDevice, st));
        return SCSFM_OK;
    }
    int* cx = static_cast<int*>(workspace);
    int* cy = cx + (size_t)out_w * (kx + 2);
    size_t coef = ((size_t)out_w * (kx + 2) + (size_t)out_h * (ky + 2)) * sizeof(int);
    coef = (coef + 255) & ~(size_t)255;
    unsigned char* tmp = static_cast<unsigned char*>(workspace) + coef;
    if (need_h) {
        prep_coeffs_kernel<<<(out_w + 127) / 128, 128, 0, st>>>(W, out_w, kx, cx);
        SCSFM_CHECK_LAUNCH();
    }
    if (need_v) {
        prep_coeffs_kernel<<<(out_h + 127) / 128, 128, 0, st>>>(H, out_h, ky, cy);
        SCSFM_CHECK_LAUNCH();
    }
    if (need_h) {
        unsigned char* dst = need_v ? tmp : out;
        prep_resample_kernel<false><<<dim3((out_w + 255) / 256, H, B), 256, 0, st>>>(in, H, W, out_w, cx, kx, dst);
        SCSFM_CHECK_LAUNCH();
    }
    if (need_v) {
        const unsigned char* src = need_h ? tmp : in;
        prep_resample_kernel<true><<<dim3((out_w + 255) / 256, out_h, B), 256, 0, st>>>(src, H, out_w, out_h, cy, ky, out);
        SCSFM_CHECK_LAUNCH();
    }
    return SCSFM_OK;
}

extern "C" size_t scsfm_velo_depth_workspace_bytes(int B, int Hd, int Wd) {
    if (B <= 0 || Hd <= 0 || Wd <= 0) return 0;
    return (size_t)B * Hd * Wd * sizeof(DepthCell);
}

extern "C" int scsfm_velo_depth(const float* points, const long long* offsets, const long long* offsets_host, const double* P, int B,
                                int Hd, int Wd, float* depth, void* workspace, size_t workspace_bytes, void* stream) {
    SCSFM_CHECK_ARG(offsets && offsets_host && P && depth, "velo_depth: null pointer");
    SCSFM_CHECK_ARG(B > 0 && B <= 65535 && Hd > 0 && Wd >= 2, "velo_depth: bad geometry (B in 1..65535, Hd >= 1, Wd >= 2)");
    SCSFM_CHECK_ARG(points || offsets_host[B] == 0, "velo_depth: null points");
    SCSFM_CHECK_ARG((long long)Hd * Wd <= (1ll << 30), "velo_depth: depth map too large");
    long long max_pts = 0;
    for (int b = 0; b < B; ++b) {
        const long long n = offsets_host[b + 1] - offsets_host[b];
        SCSFM_CHECK_ARG(offsets_host[0] == 0 && n >= 0, "velo_depth: offsets must start at 0 and not decrease");
        SCSFM_CHECK_ARG(n < 0x7fffffffll, "velo_depth: more than 2^31 - 1 points in one frame");
        if (n > max_pts) max_pts = n;
    }
    SCSFM_CHECK_ARG(workspace_bytes >= scsfm_velo_depth_workspace_bytes(B, Hd, Wd), "velo_depth: workspace too small (scsfm_velo_depth_workspace_bytes)");
    SCSFM_CHECK_ARG(workspace && (reinterpret_cast<uintptr_t>(workspace) & 15) == 0, "velo_depth: workspace must be 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    DepthCell* cells = static_cast<DepthCell*>(workspace);
    const long long n_cells = (long long)B * Hd * Wd;
    velo_init_kernel<<<(unsigned)((n_cells + 255) / 256), 256, 0, st>>>(cells, n_cells);
    SCSFM_CHECK_LAUNCH();
    if (max_pts > 0) {
        const long long blocks = (max_pts + 255) / 256;
        velo_scatter_kernel<<<dim3((unsigned)(blocks < 1024 ? blocks : 1024), B), 256, 0, st>>>(points, offsets, P, Hd, Wd, cells);
        SCSFM_CHECK_LAUNCH();
    }
    velo_resolve_kernel<<<dim3((Hd * Wd + 255) / 256, B), 256, 0, st>>>(points, offsets, P, Hd, Wd, cells, depth);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}
