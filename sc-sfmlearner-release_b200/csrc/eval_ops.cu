// Validation metrics of the depth network (reference loss_functions.py:163-205, `compute_errors`): per image the Garg /
// NYU crop + depth-range mask, median scaling of the prediction (torch.median = the LOWER median, element (n-1)/2 of the
// sorted masked values), then abs_diff, abs_rel, sq_rel and the three threshold accuracies.
//
// The reference does this with boolean-mask gathers, two sorts and ~20 elementwise kernels per image; here one CTA per
// (image, tensor) finds the exact median with a 4-pass radix select on the (positive) float bit patterns and a second
// kernel accumulates the six sums -- no host synchronisation, no temporaries.  HBM-bound: 2 x 4 passes + 1 pass over
// 8 B/pixel.
//
// scsfm_eval_depth restates the reference's offline evaluation (eval_depth.py:32-56,159-227) for a chunk of images whose
// ground truths differ in size: one CTA per image compacts the masked (gt, resized prediction) pairs into workspace, takes
// the two numpy medians with the same radix select on 32- or 64-bit keys, and reduces the seven error metrics in fp64.
#include <math.h>
#include <vector>

#include "nn_common.cuh"

namespace scsfm {

constexpr int EV_THREADS = 1024;

struct EvalGeom {
    int B, H, W, y1, y2, x1, x2;
    float max_depth;
};

// Exact key of rank `rank` (0-based, ascending) among the keys key(i, k) yields for i in [0, count), most significant byte
// first: a histogram of the next byte of the keys that share the prefix found so far picks one byte per pass (4 passes for 32-bit
// keys, 8 for 64-bit).  key(i, k) returns false for an element that does not take part.  Every thread of the block calls it;
// the result is returned to all of them.  hist: 256 shared counters; s_prefix / s_rank: shared scalars.
template <int NT, typename U, typename KeyFn>
__device__ U radix_select(int count, unsigned rank, KeyFn key, unsigned* hist, U* s_prefix, unsigned* s_rank) {
    constexpr int BITS = 8 * (int)sizeof(U);
    const int tid = threadIdx.x;
    __syncthreads();                                   // s_prefix may still be read by a previous call
    if (tid == 0) {
        *s_prefix = 0;
        *s_rank = rank;
    }
    for (int shift = BITS - 8; shift >= 0; shift -= 8) {
        for (int i = tid; i < 256; i += NT) hist[i] = 0;
        __syncthreads();
        const U prefix = *s_prefix;
        const U mask = shift == BITS - 8 ? U(0) : (~U(0) << (shift + 8));
        for (int i = tid; i < count; i += NT) {
            U u;
            if (key(i, u) && (u & mask) == prefix) atomicAdd(&hist[(unsigned)(u >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (tid == 0) {
            unsigned r = *s_rank, acc = 0;
            int d = 0;
            for (; d < 256; ++d) {
                if (acc + hist[d] > r) break;
                acc += hist[d];
            }
            *s_rank = r - acc;
            *s_prefix = prefix | ((U)d << shift);
        }
        __syncthreads();
    }
    return *s_prefix;
}

__device__ __forceinline__ bool eval_keep(const EvalGeom& g, int pix, float gt) {
    const int y = pix / g.W, x = pix - y * g.W;
    return y >= g.y1 && y < g.y2 && x >= g.x1 && x < g.x2 && gt > 0.1f && gt < g.max_depth;
}

// grid (B, 2): blockIdx.y = 0 -> median of the masked ground truth, 1 -> of the masked, clamped prediction.
// med[b][which] = value of rank (n - 1) / 2 (NaN when the mask is empty), cnt[b] = n.
__global__ void __launch_bounds__(EV_THREADS)
eval_median_kernel(const float* __restrict__ gt, const float* __restrict__ pred, EvalGeom g, float* __restrict__ med, int* __restrict__ cnt) {
    __shared__ unsigned hist[256];
    __shared__ unsigned s_prefix, s_rank, s_count;
    const int b = blockIdx.x, which = blockIdx.y, tid = threadIdx.x;
    const int HW = g.H * g.W;
    const float* gi = gt + (size_t)b * HW;
    const float* pi = pred + (size_t)b * HW;
    // count the masked pixels
    if (tid == 0) s_count = 0;
    __syncthreads();
    unsigned local = 0;
    for (int i = tid; i < HW; i += EV_THREADS) local += eval_keep(g, i, __ldg(gi + i)) ? 1u : 0u;
    local = __reduce_add_sync(0xffffffffu, local);
    if ((tid & 31) == 0 && local) atomicAdd(&s_count, local);
    __syncthreads();
    const unsigned n = s_count;
    if (n == 0) {
        if (tid == 0) {
            med[b * 2 + which] = __int_as_float(0x7fc00000);
            if (which == 0) cnt[b] = 0;
        }
        return;
    }
    if (tid == 0 && which == 0) cnt[b] = (int)n;
    const unsigned u = radix_select<EV_THREADS>(HW, (n - 1) / 2, [&](int i, unsigned& key) {      // torch.median: lower median
        const float gv = __ldg(gi + i);
        if (!eval_keep(g, i, gv)) return false;
        key = __float_as_uint(which == 0 ? gv : fminf(fmaxf(__ldg(pi + i), 1e-3f), g.max_depth));
        return true;
    }, hist, &s_prefix, &s_rank);
    if (tid == 0) med[b * 2 + which] = __uint_as_float(u);
}

// grid B: out[b][0..5] = abs_diff, abs_rel, sq_rel, a1, a2, a3 (means over the image's masked pixels), out[b][6..7] = medians
__global__ void __launch_bounds__(EV_THREADS)
eval_metrics_kernel(const float* __restrict__ gt, const float* __restrict__ pred, EvalGeom g, const float* __restrict__ med,
                    const int* __restrict__ cnt, float* __restrict__ out) {
    __shared__ double red[32][6];
    const int b = blockIdx.x, tid = threadIdx.x;
    const int HW = g.H * g.W;
    const float mg = med[b * 2], mp = med[b * 2 + 1];
    double s[6] = {0, 0, 0, 0, 0, 0};
    for (int i = tid; i < HW; i += EV_THREADS) {
        const float vg = __ldg(gt + (size_t)b * HW + i);
        if (!eval_keep(g, i, vg)) continue;
        float vp = fminf(fmaxf(__ldg(pred + (size_t)b * HW + i), 1e-3f), g.max_depth);
        vp = __fdiv_rn(__fmul_rn(vp, mg), mp);                         // valid_pred * median(gt) / median(pred), in that order
        const float th = fmaxf(__fdiv_rn(vg, vp), __fdiv_rn(vp, vg));
        const float e = fabsf(vg - vp);
        s[0] += e;
        s[1] += __fdiv_rn(e, vg);
        s[2] += __fdiv_rn(__fmul_rn(vg - vp, vg - vp), vg);
        s[3] += th < 1.25f ? 1.0 : 0.0;
        s[4] += th < 1.25f * 1.25f ? 1.0 : 0.0;
        s[5] += th < 1.25f * 1.25f * 1.25f ? 1.0 : 0.0;
    }
#pragma unroll
    for (int k = 0; k < 6; ++k) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s[k] += __shfl_xor_sync(0xffffffffu, s[k], o);
        if ((tid & 31) == 0) red[tid >> 5][k] = s[k];
    }
    __syncthreads();
    if (tid < 6) {
        double t = 0;
        for (int w = 0; w < EV_THREADS / 32; ++w) t += red[w][tid];
        const int n = cnt[b];
        out[b * 8 + tid] = n > 0 ? (float)(t / n) : __int_as_float(0x7fc00000);
    }
    if (tid == 6) out[b * 8 + 6] = mg;
    if (tid == 7) out[b * 8 + 7] = mp;
}


// ---- scsfm_eval_depth -------------------------------------------------------------------------------------------------
constexpr int ED_THREADS = 512;
constexpr int ED_WARPS = ED_THREADS / 32;

struct EvalDepthImg {          // device copy of ScsfmEvalDepthImage plus the image's slice of the pair workspace
    long long gt_off, work_off;
    int H, W, y1, y2, x1, x2;
};

// Order-preserving unsigned keys of floats (a larger key is a larger value; the inverse gives the value back).
__device__ __forceinline__ unsigned okey(float v) {
    const unsigned u = __float_as_uint(v);
    return (u >> 31) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ unsigned long long okey(double v) {
    const unsigned long long u = (unsigned long long)__double_as_longlong(v);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ float okey_value(unsigned k) { return __uint_as_float((k >> 31) ? (k & 0x7fffffffu) : ~k); }
__device__ __forceinline__ double okey_value(unsigned long long k) {
    return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

// One axis of cv2.resize INTER_LINEAR: source index (d + 0.5) * (n_in / n_out) - 0.5, clamped at both edges, fp64 weights.
struct LinearTap {
    int i0, i1;
    double w0, w1;
};
__device__ __forceinline__ LinearTap linear_tap(int d, double scale, int n_in) {
    const double f = __dadd_rn(__dmul_rn((double)d + 0.5, scale), -0.5);
    const double fl = floor(f);
    int i = (int)fl;
    double a = __dadd_rn(f, -fl);
    if (i < 0) { i = 0; a = 0.0; }
    if (i >= n_in - 1) { i = n_in - 1; a = 0.0; }
    return {i, min(i + 1, n_in - 1), __dadd_rn(1.0, -a), a};
}

// 1 / (1 / (p + 1e-6) + 1e-6) at the source pixel, the inverse-depth map the reference resizes
__device__ __forceinline__ double inv_depth(const double* __restrict__ p, int idx) { return __ddiv_rn(1.0, __dadd_rn(__ldg(p + idx), 1e-6)); }

// The reference's prediction at ground-truth pixel (y, x): inverse depth resized to H x W (horizontal pass first, then
// vertical, each sample a rounded product sum: the numpy restatement's order), then inverted again.
__device__ __forceinline__ double resized_depth(const double* __restrict__ p, int h, int w, int H, int W, int y, int x) {
    const LinearTap ty = linear_tap(y, __ddiv_rn((double)h, (double)H), h);
    const LinearTap tx = linear_tap(x, __ddiv_rn((double)w, (double)W), w);
    const int r0 = ty.i0 * w, r1 = ty.i1 * w;
    const double v0 = __dadd_rn(__dmul_rn(inv_depth(p, r0 + tx.i0), tx.w0), __dmul_rn(inv_depth(p, r0 + tx.i1), tx.w1));
    const double v1 = __dadd_rn(__dmul_rn(inv_depth(p, r1 + tx.i0), tx.w0), __dmul_rn(inv_depth(p, r1 + tx.i1), tx.w1));
    const double v = __dadd_rn(__dmul_rn(v0, ty.w0), __dmul_rn(v1, ty.w1));
    return __ddiv_rn(1.0, __dadd_rn(v, 1e-6));
}

template <typename T> struct GtKey;
template <> struct GtKey<float> { using U = unsigned; };
template <> struct GtKey<double> { using U = unsigned long long; };

// numpy's median of the n keys key(i, k): ranks (n-1)/2 and n/2 averaged.  The upper middle is one pass after the select:
// the lower middle itself if more than n/2 keys are <= it (ties), else the smallest key above it.
template <typename V, typename KeyFn>
__device__ V numpy_median(int n, KeyFn key, unsigned* hist, void* s_scratch, unsigned* s_rank, unsigned* s_cnt) {
    using U = decltype(okey(V(0)));
    U* s_u = reinterpret_cast<U*>(s_scratch);
    const U lo = radix_select<ED_THREADS>(n, (unsigned)(n - 1) / 2, key, hist, s_u, s_rank);
    if (n & 1) return okey_value(lo);
    __syncthreads();                                   // every thread has read lo out of s_u
    if (threadIdx.x == 0) {
        *s_cnt = 0;
        *s_u = ~U(0);
    }
    __syncthreads();
    unsigned le = 0;
    U above = ~U(0);
    for (int i = threadIdx.x; i < n; i += ED_THREADS) {
        U k;
        key(i, k);
        if (k <= lo) ++le;
        else if (k < above) above = k;
    }
    le = __reduce_add_sync(0xffffffffu, le);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const U t = __shfl_xor_sync(0xffffffffu, above, o);
        above = t < above ? t : above;
    }
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(s_cnt, le);
        atomicMin(s_u, above);
    }
    __syncthreads();
    const U hi = *s_cnt > (unsigned)n / 2 ? lo : *s_u;
    const V a = okey_value(lo), b = okey_value(hi);
    return (a + b) * V(0.5);                          // (a + b) rounded in V, then / 2 (exact): numpy's mean of the two
}

// grid = images of the chunk, one CTA each.  out[img][12] = {n, median(gt), median(pred), ratio, abs_rel, sq_rel, rmse,
// rmse_log, log10, a1, a2, a3}.
template <typename T>
__global__ void __launch_bounds__(ED_THREADS)
eval_depth_kernel(const double* __restrict__ pred, int h, int w, const T* __restrict__ gt, const EvalDepthImg* __restrict__ imgs,
                  double min_depth, double max_depth, double2* __restrict__ work, double* __restrict__ out) {
    using UG = typename GtKey<T>::U;
    __shared__ unsigned hist[256];
    __shared__ unsigned long long s_u;
    __shared__ unsigned s_rank, s_cnt;
    __shared__ unsigned s_warp[2][ED_WARPS];
    __shared__ double s_red[ED_WARPS][8];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const EvalDepthImg im = imgs[blockIdx.x];
    const T* g = gt + im.gt_off;
    const double* p = pred + (size_t)blockIdx.x * h * w;
    double2* pairs = work + im.work_off;
    double* o = out + (size_t)blockIdx.x * 12;
    const T lo_t = (T)min_depth, hi_t = (T)max_depth;  // the mask compares in the ground truth's dtype (numpy: float32 vs a Python float)

    // 1. compact the masked pixels of the crop, in raster order, as (gt, resized prediction) pairs
    const int cw = im.x2 - im.x1;
    const int area = (im.y2 - im.y1) * cw;
    int n = 0;
    for (int t0 = 0, tile = 0; t0 < area; t0 += ED_THREADS, ++tile) {
        const int i = t0 + tid;
        int y = 0, x = 0;
        T gv = 0;
        bool keep = false;
        if (i < area) {
            y = im.y1 + i / cw;
            x = im.x1 + i % cw;
            gv = __ldg(g + (size_t)y * im.W + x);
            keep = gv > lo_t && gv < hi_t;
        }
        const unsigned ball = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) s_warp[tile & 1][wid] = __popc(ball);
        __syncthreads();                               // double-buffered counts: one barrier per tile
        int base = n, total = 0;
        for (int k = 0; k < ED_WARPS; ++k) {
            const int c = (int)s_warp[tile & 1][k];
            base += k < wid ? c : 0;
            total += c;
        }
        if (keep)
            pairs[base + __popc(ball & ((1u << lane) - 1u))] = make_double2((double)gv, resized_depth(p, h, w, im.H, im.W, y, x));
        n += total;
    }
    __syncthreads();                                   // the pairs are visible to the whole block
    if (n == 0) {
        if (tid < 12) o[tid] = tid == 0 ? 0.0 : __longlong_as_double(0x7ff8000000000000ll);
        return;
    }

    // 2. medians: numpy's, in the ground truth's dtype for the ground truth, in fp64 for the prediction
    const T med_g = numpy_median<T>(n, [&](int i, UG& k) { k = okey((T)pairs[i].x); return true; }, hist, &s_u, &s_rank, &s_cnt);
    const double med_p = numpy_median<double>(n, [&](int i, unsigned long long& k) { k = okey(pairs[i].y); return true; }, hist, &s_u,
                                              &s_rank, &s_cnt);
    const double ratio = __ddiv_rn((double)med_g, med_p);

    // 3. metrics of the scaled, clamped prediction (compute_depth_errors); logs of the ground truth in its dtype
    double s[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = tid; i < n; i += ED_THREADS) {
        const double2 q = pairs[i];
        const T gt_t = (T)q.x;
        const double gd = q.x;
        double pv = __dmul_rn(q.y, ratio);
        if (pv < min_depth) pv = min_depth;
        if (pv > max_depth) pv = max_depth;
        const double th = fmax(__ddiv_rn(gd, pv), __ddiv_rn(pv, gd));
        const double d = __dadd_rn(gd, -pv), d2 = __dmul_rn(d, d);
        const double l = __dadd_rn((double)log(gt_t), -log(pv));
        s[0] += __ddiv_rn(fabs(d), gd);
        s[1] += __ddiv_rn(d2, gd);
        s[2] += d2;
        s[3] += __dmul_rn(l, l);
        s[4] += fabs(__dadd_rn((double)log10(gt_t), -log10(pv)));
        s[5] += th < 1.25 ? 1.0 : 0.0;
        s[6] += th < 1.25 * 1.25 ? 1.0 : 0.0;
        s[7] += th < 1.25 * 1.25 * 1.25 ? 1.0 : 0.0;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) s[k] += __shfl_xor_sync(0xffffffffu, s[k], off);
        if (lane == 0) s_red[wid][k] = s[k];
    }
    __syncthreads();
    if (tid < 8) {
        double t = 0;
        for (int k = 0; k < ED_WARPS; ++k) t += s_red[k][tid];
        const double mean = __ddiv_rn(t, (double)n);
        o[4 + tid] = (tid == 2 || tid == 3) ? sqrt(mean) : mean;
    }
    if (tid == 8) {
        o[0] = (double)n;
        o[1] = (double)med_g;
        o[2] = med_p;
        o[3] = ratio;
    }
}

}  // namespace scsfm

using namespace scsfm;

// gt, pred [B,H,W]; crop rows [y1,y2) x columns [x1,x2); work: 2*B floats + B ints; out [B][8]
extern "C" int scsfm_compute_errors(const float* gt, const float* pred, int B, int H, int W, int y1, int y2, int x1, int x2,
                                    float max_depth, void* work, float* out, void* stream) {
    SCSFM_CHECK_ARG(gt && pred && work && out && B > 0 && H > 0 && W > 0, "compute_errors: bad arguments");
    SCSFM_CHECK_ARG(0 <= y1 && y1 <= y2 && y2 <= H && 0 <= x1 && x1 <= x2 && x2 <= W && max_depth > 0.1f, "compute_errors: bad crop / depth range");
    EvalGeom g{B, H, W, y1, y2, x1, x2, max_depth};
    float* med = reinterpret_cast<float*>(work);
    int* cnt = reinterpret_cast<int*>(med + 2 * B);
    cudaStream_t st = (cudaStream_t)stream;
    eval_median_kernel<<<dim3(B, 2), EV_THREADS, 0, st>>>(gt, pred, g, med, cnt);
    SCSFM_CHECK_LAUNCH();
    eval_metrics_kernel<<<B, EV_THREADS, 0, st>>>(gt, pred, g, med, cnt, out);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

static size_t eval_depth_desc_bytes(int n) { return ((size_t)n * sizeof(EvalDepthImg) + 255) & ~(size_t)255; }

extern "C" size_t scsfm_eval_depth_workspace_bytes(const ScsfmEvalDepthImage* images_host, int n) {
    if (!images_host || n <= 0) return 0;
    size_t pairs = 0;
    for (int i = 0; i < n; ++i) {
        const ScsfmEvalDepthImage& d = images_host[i];
        if (d.y2 > d.y1 && d.x2 > d.x1) pairs += (size_t)(d.y2 - d.y1) * (size_t)(d.x2 - d.x1);
    }
    return eval_depth_desc_bytes(n) + pairs * sizeof(double2);
}

extern "C" int scsfm_eval_depth(const double* pred, int n_img, int h, int w, const void* gt, int gt_dtype, long long gt_elems,
                                const ScsfmEvalDepthImage* images_host, double min_depth, double max_depth, void* workspace,
                                size_t workspace_bytes, double* out, void* stream) {
    SCSFM_CHECK_ARG(pred && gt && images_host && workspace && out, "eval_depth: null pointer");
    SCSFM_CHECK_ARG(n_img > 0 && h > 0 && w > 0 && gt_elems > 0, "eval_depth: non-positive size (n_img %d, h %d, w %d, gt_elems %lld)",
                    n_img, h, w, gt_elems);
    SCSFM_CHECK_ARG(gt_dtype == SCSFM_EVAL_GT_F32 || gt_dtype == SCSFM_EVAL_GT_F64, "eval_depth: gt_dtype must be SCSFM_EVAL_GT_F32 or _F64");
    SCSFM_CHECK_ARG(min_depth < max_depth, "eval_depth: min_depth must be below max_depth");
    std::vector<EvalDepthImg> dev(n_img);
    long long off = 0;
    for (int i = 0; i < n_img; ++i) {
        const ScsfmEvalDepthImage& d = images_host[i];
        SCSFM_CHECK_ARG(d.H > 0 && d.W > 0 && (long long)d.H * d.W <= (1ll << 31) - 1, "eval_depth: image %d has a bad size %dx%d", i, d.H, d.W);
        SCSFM_CHECK_ARG(d.gt_offset >= 0 && d.gt_offset + (long long)d.H * d.W <= gt_elems, "eval_depth: image %d lies outside the ground-truth buffer", i);
        SCSFM_CHECK_ARG(0 <= d.y1 && d.y1 <= d.y2 && d.y2 <= d.H && 0 <= d.x1 && d.x1 <= d.x2 && d.x2 <= d.W,
                        "eval_depth: crop [%d,%d)x[%d,%d) of image %d lies outside its %dx%d image", d.y1, d.y2, d.x1, d.x2, i, d.H, d.W);
        dev[i] = EvalDepthImg{d.gt_offset, off, d.H, d.W, d.y1, d.y2, d.x1, d.x2};
        off += (long long)(d.y2 - d.y1) * (d.x2 - d.x1);
    }
    const size_t need = eval_depth_desc_bytes(n_img) + (size_t)off * sizeof(double2);
    SCSFM_CHECK_ARG(workspace_bytes >= need, "eval_depth: workspace of %zu bytes, %zu needed (scsfm_eval_depth_workspace_bytes)", workspace_bytes, need);
    SCSFM_CHECK_ARG(((uintptr_t)workspace & 15) == 0, "eval_depth: workspace must be 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    EvalDepthImg* imgs = reinterpret_cast<EvalDepthImg*>(workspace);
    double2* pairs = reinterpret_cast<double2*>(reinterpret_cast<char*>(workspace) + eval_depth_desc_bytes(n_img));
    // pageable source: the copy has been staged when cudaMemcpyAsync returns, so `dev` may go out of scope
    SCSFM_CHECK_CUDA(cudaMemcpyAsync(imgs, dev.data(), n_img * sizeof(EvalDepthImg), cudaMemcpyHostToDevice, st));
    if (gt_dtype == SCSFM_EVAL_GT_F32)
        eval_depth_kernel<float><<<n_img, ED_THREADS, 0, st>>>(pred, h, w, static_cast<const float*>(gt), imgs, min_depth, max_depth, pairs, out);
    else
        eval_depth_kernel<double><<<n_img, ED_THREADS, 0, st>>>(pred, h, w, static_cast<const double*>(gt), imgs, min_depth, max_depth, pairs, out);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}
