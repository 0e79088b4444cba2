// Disparity heads: 3x3 reflection-padded convolution with ONE output channel + 10*sigmoid+0.01
// (reference DispResNet.py:79-82,98), forward and weight gradient.  A GEMM with N = 1 wastes a tensor-core or SIMT
// tile; these are HBM/L1-bound streaming kernels in exact fp32.
#include "nn_common.cuh"

namespace scsfm {

constexpr int HT = 256;

// out[p] = act(bias + sum_{tap,c} in[refl(p + tap)][c] * w[tap][c]).
// TPP = C/4 threads per pixel, one float4 channel group each: a warp reads 32 consecutive float4 = 512 contiguous bytes per
// tap (one thread per pixel made every LDG.128 touch 16 cache lines: 4x the L1 wavefronts), then a shuffle tree adds the
// channel groups of a pixel.
template <int TPP>
__global__ void __launch_bounds__(HT)
head_fwd_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias, float* __restrict__ out,
                int B, int H, int W, int act) {
    constexpr int C = 4 * TPP;
    __shared__ float4 sw[9 * TPP];        // [9][C]
    for (int i = threadIdx.x; i < 9 * TPP; i += HT) sw[i] = __ldg(reinterpret_cast<const float4*>(w) + i);
    __syncthreads();
    const long long total = (long long)B * H * W;
    const int c4 = threadIdx.x % TPP;
    const float b0 = bias ? __ldg(bias) : 0.f;
    constexpr int PPB = HT / TPP;         // pixels per block and iteration
    for (long long p0 = blockIdx.x * (long long)PPB; p0 < total; p0 += (long long)gridDim.x * PPB) {
        const long long p = p0 + threadIdx.x / TPP;
        const bool ok = p < total;
        const long long pc = ok ? p : total - 1;
        const int x = (int)(pc % W);
        const long long t = pc / W;
        const int y = (int)(t % H), b = (int)(t / H);
        float4 acc4 = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int dy = -1; dy <= 1; ++dy) {
            const int yy = reflect_index(y + dy, H);
#pragma unroll
            for (int dx = -1; dx <= 1; ++dx) {
                const int xx = reflect_index(x + dx, W);
                const float4 a = __ldg(reinterpret_cast<const float4*>(in + (((size_t)b * H + yy) * W + xx) * C) + c4);
                const float4 k = sw[((dy + 1) * 3 + dx + 1) * TPP + c4];
                acc4.x = fmaf(a.x, k.x, acc4.x); acc4.y = fmaf(a.y, k.y, acc4.y); acc4.z = fmaf(a.z, k.z, acc4.z); acc4.w = fmaf(a.w, k.w, acc4.w);
            }
        }
        float acc = (acc4.x + acc4.y) + (acc4.z + acc4.w);
#pragma unroll
        for (int o = TPP / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (c4 == 0 && ok) {
            acc += b0;
            if ((act & 0xff) == ACT_DISP) acc = 10.0f * (1.0f / (1.0f + expf(-acc))) + 0.01f;
            out[p] = acc;
        }
    }
}

// dw[tap][c] += sum_p dpre[p] * in[refl(p + tap)][c];  dbias += sum_p dpre[p]
// thread = (pixel lane, 4-channel chunk): 9 float4 accumulators, grid-stride over pixels, block reduction, atomics.
__global__ void __launch_bounds__(HT)
head_wgrad_kernel(const float* __restrict__ in, const float* __restrict__ dpre, float* __restrict__ dw, float* __restrict__ dbias,
                  int B, int H, int W, int C) {
    const int C4 = C >> 2;
    const int c4 = threadIdx.x % C4, pl = threadIdx.x / C4, lanes = HT / C4;
    float4 acc[9];
#pragma unroll
    for (int t = 0; t < 9; ++t) acc[t] = make_float4(0.f, 0.f, 0.f, 0.f);
    float gsum = 0.f;
    const long long total = (long long)B * H * W;
    if (pl < lanes) {
        for (long long p = (long long)blockIdx.x * lanes + pl; p < total; p += (long long)gridDim.x * lanes) {
            const float g = __ldg(dpre + p);
            const int x = (int)(p % W);
            const long long t2 = p / W;
            const int y = (int)(t2 % H), b = (int)(t2 / H);
            gsum += g;
#pragma unroll
            for (int dy = -1; dy <= 1; ++dy) {
                const int yy = reflect_index(y + dy, H);
#pragma unroll
                for (int dx = -1; dx <= 1; ++dx) {
                    const int xx = reflect_index(x + dx, W);
                    const float4 a = __ldg(reinterpret_cast<const float4*>(in + (((size_t)b * H + yy) * W + xx) * C) + c4);
                    float4& r = acc[(dy + 1) * 3 + dx + 1];
                    r.x = fmaf(g, a.x, r.x); r.y = fmaf(g, a.y, r.y); r.z = fmaf(g, a.z, r.z); r.w = fmaf(g, a.w, r.w);
                }
            }
        }
    }
    // reduce over the pixel lanes of the block: one (tap, channel) column at a time through shared memory
    __shared__ float4 red[HT];
    for (int t = 0; t < 9; ++t) {
        __syncthreads();
        red[threadIdx.x] = pl < lanes ? acc[t] : make_float4(0.f, 0.f, 0.f, 0.f);
        __syncthreads();
        if (threadIdx.x < C4) {
            float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int l = 0; l < lanes; ++l) {
                const float4 v = red[l * C4 + threadIdx.x];
                s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
            }
            float* d = dw + t * C + 4 * threadIdx.x;
            red_add(d, s.x); red_add(d + 1, s.y); red_add(d + 2, s.z); red_add(d + 3, s.w);
        }
    }
    if (dbias != nullptr) {
        __syncthreads();
        float* rf = reinterpret_cast<float*>(red);
        rf[threadIdx.x] = (c4 == 0 && pl < lanes) ? gsum : 0.f;
        __syncthreads();
        if (threadIdx.x == 0) {
            float s = 0.f;
            for (int i = 0; i < HT; ++i) s += rf[i];
            red_add(dbias, s);
        }
    }
}

// Gradient w.r.t. the reflection-PADDED input of the head: dpad[b][qy][qx][c] = sum_{dy,dx} dpre[b][qy-dy][qx-dx] * w[dy][dx][c]
// over the taps whose source pixel exists ([B,H+2,W+2,C], folded onto the unpadded tensor by scsfm_fold_bwd).
// thread = (padded pixel, 4-channel chunk); 9 broadcast loads of dpre, one 16-byte store: write-bandwidth bound.
__global__ void __launch_bounds__(HT)
head_dgrad_kernel(const float* __restrict__ dpre, const float* __restrict__ w, float* __restrict__ dpad, int B, int H, int W, int C) {
    extern __shared__ float sw[];        // [9][C]
    for (int i = threadIdx.x; i < 9 * C; i += HT) sw[i] = w[i];
    __syncthreads();
    const int C4 = C >> 2, Hp = H + 2, Wp = W + 2;
    const long long total = (long long)B * Hp * Wp * C4;
    for (long long i = blockIdx.x * (long long)HT + threadIdx.x; i < total; i += (long long)gridDim.x * HT) {
        const int c4 = (int)(i % C4);
        long long t = i / C4;
        const int qx = (int)(t % Wp); t /= Wp;
        const int qy = (int)(t % Hp);
        const int b = (int)(t / Hp);
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int dy = 0; dy < 3; ++dy) {
            const int y = qy - dy;
#pragma unroll
            for (int dx = 0; dx < 3; ++dx) {
                const int x = qx - dx;
                if ((unsigned)y < (unsigned)H && (unsigned)x < (unsigned)W) {
                    const float g = __ldg(dpre + ((size_t)b * H + y) * W + x);
                    const float4 k = *reinterpret_cast<const float4*>(sw + (dy * 3 + dx) * C + 4 * c4);
                    acc.x = fmaf(g, k.x, acc.x); acc.y = fmaf(g, k.y, acc.y); acc.z = fmaf(g, k.z, acc.z); acc.w = fmaf(g, k.w, acc.w);
                }
            }
        }
        *reinterpret_cast<float4*>(dpad + i * 4) = acc;
    }
}

}  // namespace scsfm

using namespace scsfm;

extern "C" int scsfm_head_conv_fwd(const float* in, const float* w, const float* bias, float* out, int B, int H, int W, int C, int act,
                                   void* stream) {
    SCSFM_CHECK_ARG(in && w && out && B > 0 && H >= 2 && W >= 2, "head_conv_fwd: bad arguments");
    SCSFM_CHECK_ARG(C == 4 || C == 8 || C == 16 || C == 32 || C == 64 || C == 128, "head_conv_fwd: C must be 4, 8, 16, 32, 64 or 128 (got %d)", C);
    const long long total = (long long)B * H * W;
    const int ppb = HT / (C / 4);
    long long g = (total + ppb - 1) / ppb;
    if (g > 132 * 16) g = 132 * 16;
    cudaStream_t st = (cudaStream_t)stream;
    switch (C / 4) {
        case 1: head_fwd_kernel<1><<<(int)g, HT, 0, st>>>(in, w, bias, out, B, H, W, act); break;
        case 2: head_fwd_kernel<2><<<(int)g, HT, 0, st>>>(in, w, bias, out, B, H, W, act); break;
        case 4: head_fwd_kernel<4><<<(int)g, HT, 0, st>>>(in, w, bias, out, B, H, W, act); break;
        case 8: head_fwd_kernel<8><<<(int)g, HT, 0, st>>>(in, w, bias, out, B, H, W, act); break;
        case 16: head_fwd_kernel<16><<<(int)g, HT, 0, st>>>(in, w, bias, out, B, H, W, act); break;
        default: head_fwd_kernel<32><<<(int)g, HT, 0, st>>>(in, w, bias, out, B, H, W, act); break;
    }
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_head_conv_wgrad(const float* in, const float* dpre, float* dw, float* dbias, int B, int H, int W, int C, void* stream) {
    SCSFM_CHECK_ARG(in && dpre && dw && B > 0 && H >= 2 && W >= 2 && C >= 4 && (C & 3) == 0 && C <= 1024, "head_conv_wgrad: bad arguments");
    const int lanes = HT / (C / 4);
    const long long total = (long long)B * H * W;
    long long g = (total + (long long)lanes * 64 - 1) / ((long long)lanes * 64);     // >= 64 pixels per lane
    if (g > 132 * 4) g = 132 * 4;
    if (g < 1) g = 1;
    head_wgrad_kernel<<<(int)g, HT, 0, (cudaStream_t)stream>>>(in, dpre, dw, dbias, B, H, W, C);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_head_conv_dgrad(const float* dpre, const float* w, float* dpad, int B, int H, int W, int C, void* stream) {
    SCSFM_CHECK_ARG(dpre && w && dpad && B > 0 && H >= 2 && W >= 2 && C >= 4 && (C & 3) == 0 && C <= 1024, "head_conv_dgrad: bad arguments");
    const long long total = (long long)B * (H + 2) * (W + 2) * (C / 4);
    long long g = (total + HT - 1) / HT;
    if (g > 132 * 32) g = 132 * 32;
    head_dgrad_kernel<<<(int)g, HT, 9 * C * sizeof(float), (cudaStream_t)stream>>>(dpre, w, dpad, B, H, W, C);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}
