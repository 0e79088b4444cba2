// Gradient of the network's input images through the 7x7 stride-2 pad-3 stem convolution (resnet_encoder.py:93, conv1 of
// torchvision's ResNet): the transposed convolution of the stem's pre-BatchNorm gradient dy, written straight into the NCHW
// image layout.  This is what autograd gives the reference's input tensors; the training step never asks for it.
//
// Gather formulation by output parity class: input pixel (h, w) receives tap (ky, kx) from dy[(h + 3 - ky) / 2][(w + 3 - kx) / 2]
// only when h + 3 - ky and w + 3 - kx are even, so the pixels of one parity class (h & 1, w & 1) share one set of 4 or 3 tap
// rows times 4 or 3 tap columns.  A CTA works on one class of one image, so its taps, its weights (staged in shared memory,
// at most 16 of the 49 taps) and its loop trip counts are uniform.  Every output element is owned by one group of 8 lanes: no
// atomics, the result does not depend on scheduling.  Exact fp32 FMAs in every convolution mode.
//
// Thread layout: a group of 8 lanes owns P class rows of one class column; lane cg of the group sums output channels
// 4cg..4cg+3 and 32+4cg..32+4cg+3 (float4 loads: the group reads two full 128-byte rows of dy), and the 8 partial sums are
// added by a shuffle butterfly at the end.  The P rows of a thread need P + NTY - 1 dy rows per tap column (consecutive class
// rows under consecutive tap rows hit overlapping dy rows), which are loaded once into registers.
#include "nn_common.cuh"

namespace scsfm {
namespace {

constexpr int SK = 7, SPAD = 3, SCO = 64;   // stem kernel size, padding, output channels
constexpr int SNT = 256;                    // 8 warps: 4 along the class columns, 2 along the class rows
constexpr int S_TJ = 16;                    // class columns per CTA (4 per warp)
constexpr int S_MAXTAP = 16;                // taps of the largest parity class (4 x 4)

template <int CIN> struct StemRows { static constexpr int P = CIN == 3 ? 8 : 4; };   // class rows per thread

template <int CIN, int P, int NTY>
__device__ __forceinline__ void stem_dgrad_taps(const float* __restrict__ dy, const float* __restrict__ ws, int n, int Ho, int Wo,
                                                int i0, int j, int oyA, int oxA, int ntx, int cg, float (&acc)[P][CIN]) {
    constexpr int NR = P + NTY - 1;
    // tap row a (ky = ky0 + 2a) of class row i0 + p reads dy row i0 + p + oyA - a = hbase + (p - a + NTY - 1)
    const int hbase = i0 + oyA - (NTY - 1);
    for (int b = 0; b < ntx; ++b) {
        const int wo = j + oxA - b;             // tap column b (kx = kx0 + 2b)
        if (wo < 0 || wo >= Wo) continue;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int co0 = 4 * cg + 32 * half;
            float4 R[NR];
#pragma unroll
            for (int r = 0; r < NR; ++r) {
                const int ho = hbase + r;
                R[r] = (ho >= 0 && ho < Ho) ? __ldg(reinterpret_cast<const float4*>(dy + (((size_t)n * Ho + ho) * Wo + wo) * SCO + co0))
                                            : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int a = 0; a < NTY; ++a) {
                const float4* wp = reinterpret_cast<const float4*>(ws + ((a * ntx + b) * SCO + co0) * CIN);
                float wv[4 * CIN];                  // [output channel co0 + q][input channel c]
#pragma unroll
                for (int k = 0; k < CIN; ++k) {
                    const float4 v = wp[k];
                    wv[4 * k] = v.x; wv[4 * k + 1] = v.y; wv[4 * k + 2] = v.z; wv[4 * k + 3] = v.w;
                }
#pragma unroll
                for (int p = 0; p < P; ++p) {
                    const float4 d = R[p - a + NTY - 1];
#pragma unroll
                    for (int c = 0; c < CIN; ++c) {
                        float s = acc[p][c];
                        s = fmaf(d.x, wv[c], s);
                        s = fmaf(d.y, wv[CIN + c], s);
                        s = fmaf(d.z, wv[2 * CIN + c], s);
                        s = fmaf(d.w, wv[3 * CIN + c], s);
                        acc[p][c] = s;
                    }
                }
            }
        }
    }
}

// grid (ceil(ceil(W/2) / S_TJ), ceil(ceil(H/2) / (2P)), N * 4): blockIdx.z = image * 4 + parity class (py * 2 + px)
template <int CIN>
__global__ void __launch_bounds__(SNT, 2)
stem_dgrad_kernel(const float* __restrict__ dy, const float* __restrict__ w, int H, int W, int Ho, int Wo, float* __restrict__ out1,
                  float* __restrict__ out2) {
    constexpr int P = StemRows<CIN>::P;
    __shared__ __align__(16) float ws[S_MAXTAP * SCO * CIN];    // [tap row a][tap column b][co][c] of this class
    const int cls = blockIdx.z & 3, n = blockIdx.z >> 2;
    const int py = cls >> 1, px = cls & 1;
    const int ky0 = (py + SPAD) & 1, kx0 = (px + SPAD) & 1;     // first tap of the class; then every second one
    const int nty = ky0 ? 3 : 4, ntx = kx0 ? 3 : 4;
    const int nw = nty * ntx * SCO * CIN;
    for (int e = threadIdx.x; e < nw; e += SNT) {
        const int c = e % CIN, t = e / CIN;
        const int co = t % SCO, tap = t / SCO;
        const int a = tap / ntx, b = tap - a * ntx;
        ws[e] = __ldg(w + ((co * SK + ky0 + 2 * a) * SK + kx0 + 2 * b) * CIN + c);
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int cg = lane & 7;
    const int j = blockIdx.x * S_TJ + (warp & 3) * 4 + (lane >> 3);     // class column
    const int i0 = (blockIdx.y * 2 + (warp >> 2)) * P;                   // first class row
    const int oyA = (py + SPAD - ky0) >> 1, oxA = (px + SPAD - kx0) >> 1;
    float acc[P][CIN];
#pragma unroll
    for (int p = 0; p < P; ++p)
#pragma unroll
        for (int c = 0; c < CIN; ++c) acc[p][c] = 0.f;
    if (nty == 4) stem_dgrad_taps<CIN, P, 4>(dy, ws, n, Ho, Wo, i0, j, oyA, oxA, ntx, cg, acc);
    else stem_dgrad_taps<CIN, P, 3>(dy, ws, n, Ho, Wo, i0, j, oyA, oxA, ntx, cg, acc);
    // the 8 lanes of a group hold partial sums over disjoint output channels
#pragma unroll
    for (int p = 0; p < P; ++p)
#pragma unroll
        for (int c = 0; c < CIN; ++c) {
            float v = acc[p][c];
            v += __shfl_xor_sync(0xffffffffu, v, 1);
            v += __shfl_xor_sync(0xffffffffu, v, 2);
            v += __shfl_xor_sync(0xffffffffu, v, 4);
            acc[p][c] = v;
        }
    const int Hc = (H - py + 1) >> 1, Wc = (W - px + 1) >> 1;
    if (cg != 0 || j >= Wc) return;
    const int x = 2 * j + px;
#pragma unroll
    for (int p = 0; p < P; ++p) {
        const int i = i0 + p;
        if (i >= Hc) break;
        const size_t pix = (size_t)(2 * i + py) * W + x;
#pragma unroll
        for (int c = 0; c < CIN; ++c) {
            float* o = c < 3 ? out1 : out2;
            if (o) o[((size_t)n * 3 + (c < 3 ? c : c - 3)) * H * W + pix] = acc[p][c];
        }
    }
}

}  // namespace
}  // namespace scsfm

using namespace scsfm;

extern "C" int scsfm_stem_dgrad(const float* dy, const float* w, int N, int H, int W, int Cin, float* dimg1, float* dimg2, void* stream) {
    SCSFM_CHECK_ARG(dy && w && N > 0 && H > 0 && W > 0 && (Cin == 3 || Cin == 6) && (dimg1 || dimg2) && (Cin == 6 || !dimg2),
                    "stem_dgrad: bad arguments");
    SCSFM_CHECK_ARG((reinterpret_cast<uintptr_t>(dy) & 15) == 0, "stem_dgrad: dy must be 16-byte aligned");
    SCSFM_CHECK_ARG(N <= 65535 / 4, "stem_dgrad: batch too large");
    const int Ho = (H + 2 * SPAD - SK) / 2 + 1, Wo = (W + 2 * SPAD - SK) / 2 + 1;
    const int P = Cin == 3 ? StemRows<3>::P : StemRows<6>::P;
    const dim3 grid((unsigned)(((W + 1) / 2 + S_TJ - 1) / S_TJ), (unsigned)(((H + 1) / 2 + 2 * P - 1) / (2 * P)), (unsigned)(N * 4));
    if (Cin == 3) stem_dgrad_kernel<3><<<grid, SNT, 0, (cudaStream_t)stream>>>(dy, w, H, W, Ho, Wo, dimg1, dimg2);
    else stem_dgrad_kernel<6><<<grid, SNT, 0, (cudaStream_t)stream>>>(dy, w, H, W, Ho, Wo, dimg1, dimg2);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}
