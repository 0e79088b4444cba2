// Generic fp32 implicit-GEMM convolution on CUDA cores: forward, data gradient, weight gradient.
//
// This is the exact-fp32 ("parity") path for every conv shape of DispResNet / PoseResNet
// (SURVEY.md appendix A) and the production path for the layers that are too thin for the
// tensor-core kernels (7x7 stem with Cin 3/6, Cout 1/6 heads).  Activations are NHWC, weights
// [Cout][kh][kw][Cin] (K-major), so the GEMM K index runs over (tap, channel) with channels
// contiguous: every operand fetch is a 16-byte load.
//
//   forward : C[M=B*Ho*Wo, N=Cout]   = A[M, K=kh*kw*Cin] (gathered input)  x  W^T
//   dgrad   : C[M=B*Hi*Wi, N=Cin]    = A[M, K=kh*kw*Cout] (gathered dout)  x  W (re-indexed)
//   wgrad   : C[M=Cout,    N=kh*kw*Cin] = dout^T  x  A (gathered input), split over K=B*Ho*Wo
//
// Replaces cuDNN conv fwd/dgrad/wgrad reached from reference resnet_encoder.py:90-96,
// DispResNet.py:37,41 and PoseResNet.py:26-29 (rows K1, K3, K5 of SURVEY.md section 2.3): bias,
// ReLU/ELU/sigmoid-disparity, reflection padding and BatchNorm partial statistics are fused.
#include "nn_common.cuh"

namespace scsfm {

constexpr int BK = 16;
constexpr int CT = 256;   // threads per CTA

// ----- shared inner product ------------------------------------------------------------------
template <int BM, int BN>
__device__ __forceinline__ void mma_tile(const float (*As)[BM + 4], const float (*Bs)[BN + 4], int ty, int tx,
                                         float (&acc)[4][4]) {
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
        const float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
        const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
        const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
}

__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// Gather 4 consecutive channels of the input feature map for output pixel (b, ho, wo) and K index kg
// (tap-major, channel-minor).  Handles zero / reflection padding and ragged K / Cin.
struct GatherIn {
    const float* in;
    int Hi, Wi, C, kw, stride, pad, pad_mode, K;
    __device__ __forceinline__ float4 load(int b, int ho, int wo, int kg, bool row_ok) const {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (!row_ok || kg >= K) return v;
        if ((C & 3) == 0) {
            const int tap = kg / C, c = kg - tap * C;
            const int dy = tap / kw, dx = tap - dy * kw;
            int hi = ho * stride + dy - pad, wi = wo * stride + dx - pad;
            if (pad_mode == PADMODE_REFLECT) {
                hi = reflect_index(hi, Hi);
                wi = reflect_index(wi, Wi);
            } else if (hi < 0 || hi >= Hi || wi < 0 || wi >= Wi) {
                return v;
            }
            return ld4(in + (((size_t)b * Hi + hi) * Wi + wi) * C + c);
        }
        float e[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            e[j] = 0.f;
            const int k = kg + j;
            if (k < K) {
                const int tap = k / C, c = k - tap * C;
                const int dy = tap / kw, dx = tap - dy * kw;
                int hi = ho * stride + dy - pad, wi = wo * stride + dx - pad;
                bool ok = true;
                if (pad_mode == PADMODE_REFLECT) {
                    hi = reflect_index(hi, Hi);
                    wi = reflect_index(wi, Wi);
                } else {
                    ok = hi >= 0 && hi < Hi && wi >= 0 && wi < Wi;
                }
                if (ok) e[j] = __ldg(in + (((size_t)b * Hi + hi) * Wi + wi) * C + c);
            }
        }
        return make_float4(e[0], e[1], e[2], e[3]);
    }
};

__device__ __forceinline__ float apply_act(float v, int act) {
    switch (act & 0xff) {
        case ACT_RELU: return fmaxf(v, 0.f);
        case ACT_ELU: return v > 0.f ? v : expm1f(v);
        case ACT_DISP: return 10.0f * (1.0f / (1.0f + expf(-v))) + 0.01f;   // alpha*sigmoid+beta, DispResNet.py:98
        default: return v;
    }
}

// ----- forward -------------------------------------------------------------------------------
template <int BM, int BN>
__global__ void __launch_bounds__(CT)
conv_fwd_simt_kernel(ScsfmConv p) {
    __shared__ __align__(16) float As[BK][BM + 4];
    __shared__ __align__(16) float Bs[BK][BN + 4];
    __shared__ double s_stat[2][BN];
    const int tid = threadIdx.x, tx = tid % (BN / 4), ty = tid / (BN / 4);
    const int M = p.B * p.Ho * p.Wo, N = p.Cout, K = p.kh * p.kw * p.Cin;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const GatherIn ga{p.in, p.Hi, p.Wi, p.Cin, p.kw, p.stride, p.pad, p.pad_mode, K};

    constexpr int A_IT = BM * BK / 4 / CT, B_IT = (BN * BK / 4 + CT - 1) / CT;
    int a_b[A_IT], a_ho[A_IT], a_wo[A_IT];
    bool a_ok[A_IT];
#pragma unroll
    for (int i = 0; i < A_IT; ++i) {
        const int r = (tid + i * CT) / 4, m = m0 + r;
        a_ok[i] = m < M;
        const int mm = a_ok[i] ? m : 0;
        a_b[i] = mm / (p.Ho * p.Wo);
        const int rem = mm - a_b[i] * p.Ho * p.Wo;
        a_ho[i] = rem / p.Wo;
        a_wo[i] = rem - a_ho[i] * p.Wo;
    }
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    float4 ra[A_IT], rb[B_IT];
    auto fetch = [&](int kt) {
#pragma unroll
        for (int i = 0; i < A_IT; ++i) {
            const int kq = ((tid + i * CT) & 3) * 4;
            ra[i] = ga.load(a_b[i], a_ho[i], a_wo[i], kt * BK + kq, a_ok[i]);
        }
#pragma unroll
        for (int i = 0; i < B_IT; ++i) {
            const int idx = tid + i * CT;
            rb[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (idx < BN * BK / 4) {
                const int n = n0 + idx / 4, kg = kt * BK + (idx & 3) * 4;
                if (n < N && kg < K) {
                    const float* w = p.w + (size_t)n * K + kg;
                    if ((K & 3) == 0) rb[i] = ld4(w);
                    else rb[i] = make_float4(__ldg(w), kg + 1 < K ? __ldg(w + 1) : 0.f, kg + 2 < K ? __ldg(w + 2) : 0.f,
                                             kg + 3 < K ? __ldg(w + 3) : 0.f);
                }
            }
        }
    };
    auto stash = [&]() {
#pragma unroll
        for (int i = 0; i < A_IT; ++i) {
            const int idx = tid + i * CT, r = idx / 4, kq = (idx & 3) * 4;
            As[kq + 0][r] = ra[i].x; As[kq + 1][r] = ra[i].y; As[kq + 2][r] = ra[i].z; As[kq + 3][r] = ra[i].w;
        }
#pragma unroll
        for (int i = 0; i < B_IT; ++i) {
            const int idx = tid + i * CT;
            if (idx < BN * BK / 4) {
                const int n = idx / 4, kq = (idx & 3) * 4;
                Bs[kq + 0][n] = rb[i].x; Bs[kq + 1][n] = rb[i].y; Bs[kq + 2][n] = rb[i].z; Bs[kq + 3][n] = rb[i].w;
            }
        }
    };
    const int KT = (K + BK - 1) / BK;
    fetch(0);
    for (int kt = 0; kt < KT; ++kt) {
        stash();
        __syncthreads();
        if (kt + 1 < KT) fetch(kt + 1);
        mma_tile<BM, BN>(As, Bs, ty, tx, acc);
        __syncthreads();
    }

    // epilogue: bias or eval-mode BatchNorm, residual addend, activation, store (+ low part), optional BatchNorm partial sums
    // (per group of samples)
    double csum[4] = {0.0, 0.0, 0.0, 0.0}, csq[4] = {0.0, 0.0, 0.0, 0.0};   // fp64: see conv_tc.cu (variance cancellation)
    const int groups = p.bn_groups > 0 ? p.bn_groups : 1;
    const int rows_per_group = (p.B / groups) * p.Ho * p.Wo;
    const bool want_stats = p.bn_sums != nullptr;
    const bool uniform_group = want_stats && (m0 / rows_per_group) == ((min(m0 + BM, M) - 1) / rows_per_group);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + ty * 4 + i;
        if (m >= M) continue;
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            float x = acc[i][j];
            if (n < N) {
                if (p.bias) x += __ldg(p.bias + n);
                if (p.bn_scale) x = fmaf(x, __ldg(p.bn_scale + n), __ldg(p.bn_shift + n));
                if (p.addend) x += __ldg(p.addend + (size_t)m * N + n);
                x = apply_act(x, p.act);
                if (p.act & ROUND_TF32) x = tf32_round(x);
                if (want_stats) {
                    if (uniform_group) { csum[j] += (double)x; csq[j] += (double)x * (double)x; }
                    else {
                        double* d = p.bn_sums + (((size_t)(blockIdx.x % SCSFM_BN_SLOTS) * groups + m / rows_per_group) * N + n) * 2;
                        atomicAdd(d, (double)x);
                        atomicAdd(d + 1, (double)x * x);
                    }
                }
            }
            v[j] = x;
        }
        float* o = p.out + (size_t)m * N + n0 + tx * 4;
        if ((N & 3) == 0 && n0 + tx * 4 + 3 < N) *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
        else
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (n0 + tx * 4 + j < N) o[j] = v[j];
        if (p.out_lo)
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (n0 + tx * 4 + j < N) p.out_lo[(size_t)m * N + n0 + tx * 4 + j] = tf32_lo(v[j]);
    }
    if (want_stats && uniform_group) {
        if (tid < BN) { s_stat[0][tid] = 0.0; s_stat[1][tid] = 0.0; }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            atomicAdd(&s_stat[0][tx * 4 + j], csum[j]);
            atomicAdd(&s_stat[1][tx * 4 + j], csq[j]);
        }
        __syncthreads();
        if (tid < BN && n0 + tid < N) {
            double* d = p.bn_sums + (((size_t)(blockIdx.x % SCSFM_BN_SLOTS) * groups + m0 / rows_per_group) * N + n0 + tid) * 2;
            atomicAdd(d, s_stat[0][tid]);
            atomicAdd(d + 1, s_stat[1][tid]);
        }
    }
}

// ----- data gradient -------------------------------------------------------------------------
// d_in[b,hi,wi,c] = sum_{dy,dx,o} dout[b,(hi+pad-dy)/s,(wi+pad-dx)/s,o] * w[o,dy,dx,c]  (+ addend)
// For reflection-padded convs the caller asks for the gradient of the PADDED input (Hi+2 x Wi+2,
// pad = 0); nn_ops' fold kernel then folds the border back.
template <int BM, int BN>
__global__ void __launch_bounds__(CT)
conv_dgrad_simt_kernel(ScsfmConv p) {
    __shared__ __align__(16) float As[BK][BM + 4];
    __shared__ __align__(16) float Bs[BK][BN + 4];
    const int tid = threadIdx.x, tx = tid % (BN / 4), ty = tid / (BN / 4);
    const int M = p.B * p.Hi * p.Wi, N = p.Cin, T = p.kh * p.kw, K = T * p.Cout;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    constexpr int A_IT = BM * BK / 4 / CT, B_IT = (BN * BK / 4 + CT - 1) / CT;
    int a_b[A_IT], a_hi[A_IT], a_wi[A_IT];
    bool a_ok[A_IT];
#pragma unroll
    for (int i = 0; i < A_IT; ++i) {
        const int r = (tid + i * CT) / 4, m = m0 + r;
        a_ok[i] = m < M;
        const int mm = a_ok[i] ? m : 0;
        a_b[i] = mm / (p.Hi * p.Wi);
        const int rem = mm - a_b[i] * p.Hi * p.Wi;
        a_hi[i] = rem / p.Wi;
        a_wi[i] = rem - a_hi[i] * p.Wi;
    }
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    float4 ra[A_IT], rb[B_IT];
    const bool c4 = (p.Cout & 3) == 0, n4ok = (N & 3) == 0;
    auto fetch = [&](int kt) {
#pragma unroll
        for (int i = 0; i < A_IT; ++i) {
            const int kg = kt * BK + ((tid + i * CT) & 3) * 4;
            float e[4] = {0.f, 0.f, 0.f, 0.f};
            if (a_ok[i]) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int k = kg + (c4 ? 0 : j);
                    if (k < K) {
                        const int tap = k / p.Cout, o = k - tap * p.Cout;
                        const int dy = tap / p.kw, dx = tap - dy * p.kw;
                        const int tyy = a_hi[i] + p.pad - dy, txx = a_wi[i] + p.pad - dx;
                        if (tyy >= 0 && txx >= 0 && tyy % p.stride == 0 && txx % p.stride == 0) {
                            const int ho = tyy / p.stride, wo = txx / p.stride;
                            if (ho < p.Ho && wo < p.Wo) {
                                const float* src = p.dout + (((size_t)a_b[i] * p.Ho + ho) * p.Wo + wo) * p.Cout + o;
                                if (c4) {
                                    const float4 t4 = ld4(src);
                                    e[0] = t4.x; e[1] = t4.y; e[2] = t4.z; e[3] = t4.w;
                                } else {
                                    e[j] = __ldg(src);
                                }
                            }
                        }
                    }
                    if (c4) break;
                }
            }
            ra[i] = make_float4(e[0], e[1], e[2], e[3]);
        }
#pragma unroll
        for (int i = 0; i < B_IT; ++i) {
            const int idx = tid + i * CT;
            rb[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (idx < BN * BK / 4) {
                const int kk = idx / (BN / 4), nq = (idx % (BN / 4)) * 4, k = kt * BK + kk, n = n0 + nq;
                if (k < K && n < N) {
                    const int tap = k / p.Cout, o = k - tap * p.Cout;
                    const float* w = p.w + ((size_t)o * T + tap) * N + n;
                    if (n4ok) rb[i] = ld4(w);
                    else rb[i] = make_float4(__ldg(w), n + 1 < N ? __ldg(w + 1) : 0.f, n + 2 < N ? __ldg(w + 2) : 0.f,
                                             n + 3 < N ? __ldg(w + 3) : 0.f);
                }
            }
        }
    };
    auto stash = [&]() {
#pragma unroll
        for (int i = 0; i < A_IT; ++i) {
            const int idx = tid + i * CT, r = idx / 4, kq = (idx & 3) * 4;
            As[kq + 0][r] = ra[i].x; As[kq + 1][r] = ra[i].y; As[kq + 2][r] = ra[i].z; As[kq + 3][r] = ra[i].w;
        }
#pragma unroll
        for (int i = 0; i < B_IT; ++i) {
            const int idx = tid + i * CT;
            if (idx < BN * BK / 4) {
                const int kk = idx / (BN / 4), nq = (idx % (BN / 4)) * 4;
                *reinterpret_cast<float4*>(&Bs[kk][nq]) = rb[i];
            }
        }
    };
    const int KT = (K + BK - 1) / BK;
    fetch(0);
    for (int kt = 0; kt < KT; ++kt) {
        stash();
        __syncthreads();
        if (kt + 1 < KT) fetch(kt + 1);
        mma_tile<BM, BN>(As, Bs, ty, tx, acc);
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + ty * 4 + i;
        if (m >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            if (n < N) {
                float v = acc[i][j];
                if (p.addend) v += __ldg(p.addend + (size_t)m * N + n);
                p.din[(size_t)m * N + n] = v;
            }
        }
    }
}

// ----- weight gradient -----------------------------------------------------------------------
// dw[o,dy,dx,c] += sum_{b,ho,wo} dout[b,ho,wo,o] * in[b, ho*s+dy-pad, wo*s+dx-pad, c]   (split-K, atomics)
template <int BM, int BN>
__global__ void __launch_bounds__(CT)
conv_wgrad_simt_kernel(ScsfmConv p, int k_per_split) {
    __shared__ __align__(16) float As[BK][BM + 4];
    __shared__ __align__(16) float Bs[BK][BN + 4];
    const int tid = threadIdx.x, tx = tid % (BN / 4), ty = tid / (BN / 4);
    const int M = p.Cout, N = p.kh * p.kw * p.Cin, Kall = p.B * p.Ho * p.Wo;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const int k_begin = blockIdx.z * k_per_split, k_end = min(Kall, k_begin + k_per_split);
    constexpr int A_IT = (BM * BK / 4 + CT - 1) / CT, B_IT = (BN * BK / 4 + CT - 1) / CT;
    const GatherIn gb{p.in, p.Hi, p.Wi, p.Cin, p.kw, p.stride, p.pad, p.pad_mode, N};
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    float4 ra[A_IT], rb[B_IT];
    const bool m4ok = (M & 3) == 0;
    auto fetch = [&](int kbase) {
#pragma unroll
        for (int i = 0; i < A_IT; ++i) {
            const int idx = tid + i * CT;
            ra[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (idx < BM * BK / 4) {
                const int kk = idx / (BM / 4), mq = (idx % (BM / 4)) * 4, k = kbase + kk, m = m0 + mq;
                if (k < k_end && m < M) {
                    const float* s = p.dout + (size_t)k * M + m;
                    if (m4ok) ra[i] = ld4(s);
                    else ra[i] = make_float4(__ldg(s), m + 1 < M ? __ldg(s + 1) : 0.f, m + 2 < M ? __ldg(s + 2) : 0.f,
                                             m + 3 < M ? __ldg(s + 3) : 0.f);
                }
            }
        }
#pragma unroll
        for (int i = 0; i < B_IT; ++i) {
            const int idx = tid + i * CT;
            rb[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (idx < BN * BK / 4) {
                const int kk = idx / (BN / 4), nq = (idx % (BN / 4)) * 4, k = kbase + kk;
                if (k < k_end) {
                    const int b = k / (p.Ho * p.Wo), rem = k - b * p.Ho * p.Wo, ho = rem / p.Wo, wo = rem - ho * p.Wo;
                    rb[i] = gb.load(b, ho, wo, n0 + nq, true);
                }
            }
        }
    };
    auto stash = [&]() {
#pragma unroll
        for (int i = 0; i < A_IT; ++i) {
            const int idx = tid + i * CT;
            if (idx < BM * BK / 4) *reinterpret_cast<float4*>(&As[idx / (BM / 4)][(idx % (BM / 4)) * 4]) = ra[i];
        }
#pragma unroll
        for (int i = 0; i < B_IT; ++i) {
            const int idx = tid + i * CT;
            if (idx < BN * BK / 4) *reinterpret_cast<float4*>(&Bs[idx / (BN / 4)][(idx % (BN / 4)) * 4]) = rb[i];
        }
    };
    if (k_begin >= k_end) return;
    fetch(k_begin);
    for (int kb = k_begin; kb < k_end; kb += BK) {
        stash();
        __syncthreads();
        if (kb + BK < k_end) fetch(kb + BK);
        mma_tile<BM, BN>(As, Bs, ty, tx, acc);
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + ty * 4 + i;
        if (m >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            if (n < N) red_add(p.dw + (size_t)m * N + n, acc[i][j]);
        }
    }
}

// per-channel sum of dout (bias gradient), accumulated into dbias.  dout is streamed as float4; the grid stride is a multiple of
// the float4 groups per row, so a thread always owns the same four channels: register accumulation, one shared-memory
// reduction per block, one red.add per (block, channel).  C % 4 == 0 and C / 4 a power of two <= 64 (else the scalar variant).
__global__ void __launch_bounds__(CT)
bias_grad_vec_kernel(const float* __restrict__ dout, long long nvec, int gpr, float* __restrict__ dbias) {
    __shared__ float4 s[CT];
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4* src = reinterpret_cast<const float4*>(dout);
    for (long long i = blockIdx.x * (long long)CT + threadIdx.x; i < nvec; i += (long long)gridDim.x * CT) {
        const float4 v = __ldg(src + i);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    s[threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.x < gpr) {              // thread t owns channel group t % gpr (CT % gpr == 0)
        float4 t = s[threadIdx.x];
        for (int j = threadIdx.x + gpr; j < CT; j += gpr) { t.x += s[j].x; t.y += s[j].y; t.z += s[j].z; t.w += s[j].w; }
        float* d = dbias + 4 * threadIdx.x;
        red_add(d, t.x); red_add(d + 1, t.y); red_add(d + 2, t.z); red_add(d + 3, t.w);
    }
}

__global__ void __launch_bounds__(CT)
bias_grad_kernel(const float* __restrict__ dout, int rows, int C, float* __restrict__ dbias, int rows_per_cta) {
    // thread layout: tid % cpad -> channel, tid / cpad -> row lane
    const int c = blockIdx.y * 64 + (threadIdx.x & 63);
    const int lane_rows = CT / 64, rl = threadIdx.x >> 6;
    const int r0 = blockIdx.x * rows_per_cta, r1 = min(rows, r0 + rows_per_cta);
    float acc = 0.f;
    if (c < C)
        for (int r = r0 + rl; r < r1; r += lane_rows) acc += __ldg(dout + (size_t)r * C + c);
    __shared__ float s[CT];
    s[threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.x < 64 && c < C) {
        float v = s[threadIdx.x] + s[threadIdx.x + 64] + s[threadIdx.x + 128] + s[threadIdx.x + 192];
        red_add(dbias + c, v);
    }
}

bool conv_wgrad_thin_eligible(const ScsfmConv& p);                       // conv_wgrad_thin.cu
int launch_conv_wgrad_thin(const ScsfmConv& p, cudaStream_t st);

// host-side launcher shared with the tensor-core weight gradient (conv_tc.cu)
int launch_bias_grad(const float* dout, int rows, int C, float* dbias, cudaStream_t st) {
    const int gpr = C / 4;
    if ((C & 3) == 0 && gpr <= 64 && (gpr & (gpr - 1)) == 0 && (reinterpret_cast<uintptr_t>(dout) & 15) == 0) {
        const long long nvec = (long long)rows * gpr;
        long long ctas = (nvec + 8 * CT - 1) / (8 * CT);          // >= 8 float4 per thread
        if (ctas > 132 * 8) ctas = 132 * 8;
        if (ctas < 1) ctas = 1;
        bias_grad_vec_kernel<<<(int)ctas, CT, 0, st>>>(dout, nvec, gpr, dbias);
        SCSFM_CHECK_LAUNCH();
        return SCSFM_OK;
    }
    int ctas = (rows + 2047) / 2048;
    if (ctas > 592) ctas = 592;
    const int rpc = (rows + ctas - 1) / ctas;
    bias_grad_kernel<<<dim3((rows + rpc - 1) / rpc, (C + 63) / 64), CT, 0, st>>>(dout, rows, C, dbias, rpc);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

}  // namespace scsfm

using namespace scsfm;

static int check_conv(const ScsfmConv* p, const char* who) {
    SCSFM_CHECK_ARG(p != nullptr, "%s: null descriptor", who);
    SCSFM_CHECK_ARG(p->B > 0 && p->Hi > 0 && p->Wi > 0 && p->Cin > 0 && p->Ho > 0 && p->Wo > 0 && p->Cout > 0 && p->kh > 0 &&
                        p->kw > 0 && p->stride > 0 && p->pad >= 0, "%s: bad geometry", who);
    SCSFM_CHECK_ARG((long long)p->B * p->Hi * p->Wi * (long long)p->Cin < (1LL << 40), "%s: tensor too large", who);
    return SCSFM_OK;
}

extern "C" int scsfm_conv2d_fwd_simt(const ScsfmConv* p, void* stream) {
    if (int rc = check_conv(p, "conv2d_fwd")) return rc;
    SCSFM_CHECK_ARG(p->in && p->w && p->out, "conv2d_fwd: null tensor");
    SCSFM_CHECK_ARG(p->Ho == (p->Hi + 2 * p->pad - p->kh) / p->stride + 1 && p->Wo == (p->Wi + 2 * p->pad - p->kw) / p->stride + 1,
                    "conv2d_fwd: output size does not match geometry");
    SCSFM_CHECK_ARG(p->pad_mode != PADMODE_REFLECT || (p->pad < p->Hi && p->pad < p->Wi && p->pad <= 1), "conv2d_fwd: reflect pad must be 1");
    SCSFM_CHECK_ARG((p->bn_scale == nullptr) == (p->bn_shift == nullptr), "conv2d_fwd: bn_scale and bn_shift go together");
    SCSFM_CHECK_ARG(p->bn_scale == nullptr || (p->bias == nullptr && p->bn_sums == nullptr),
                    "conv2d_fwd: the eval-mode BatchNorm epilogue excludes bias and bn_sums");
    cudaStream_t st = (cudaStream_t)stream;
    const int M = p->B * p->Ho * p->Wo, N = p->Cout;
    if (N <= 16) conv_fwd_simt_kernel<256, 16><<<dim3((M + 255) / 256, (N + 15) / 16), CT, 0, st>>>(*p);
    else if (N <= 32) conv_fwd_simt_kernel<128, 32><<<dim3((M + 127) / 128, (N + 31) / 32), CT, 0, st>>>(*p);
    else conv_fwd_simt_kernel<64, 64><<<dim3((M + 63) / 64, (N + 63) / 64), CT, 0, st>>>(*p);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_conv2d_dgrad_simt(const ScsfmConv* p, void* stream) {
    if (int rc = check_conv(p, "conv2d_dgrad")) return rc;
    SCSFM_CHECK_ARG(p->dout && p->w && p->din, "conv2d_dgrad: null tensor");
    cudaStream_t st = (cudaStream_t)stream;
    const int M = p->B * p->Hi * p->Wi, N = p->Cin;
    if (N <= 16) conv_dgrad_simt_kernel<256, 16><<<dim3((M + 255) / 256, (N + 15) / 16), CT, 0, st>>>(*p);
    else if (N <= 32) conv_dgrad_simt_kernel<128, 32><<<dim3((M + 127) / 128, (N + 31) / 32), CT, 0, st>>>(*p);
    else conv_dgrad_simt_kernel<64, 64><<<dim3((M + 63) / 64, (N + 63) / 64), CT, 0, st>>>(*p);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_conv2d_wgrad_simt(const ScsfmConv* p, void* stream) {
    if (int rc = check_conv(p, "conv2d_wgrad")) return rc;
    SCSFM_CHECK_ARG(p->dout && p->in && p->dw, "conv2d_wgrad: null tensor");
    cudaStream_t st = (cudaStream_t)stream;
    const int M = p->Cout, N = p->kh * p->kw * p->Cin, Kall = p->B * p->Ho * p->Wo;
    if (conv_wgrad_thin_eligible(*p) && ((p->tune >> 12) & 3u) != 1u) {       // thin decoder layers: direct kernel (conv_wgrad_thin.cu)
        if (int rc = launch_conv_wgrad_thin(*p, st)) return rc;
        if (p->dbias) return launch_bias_grad(p->dout, Kall, M, p->dbias, st);
        return SCSFM_OK;
    }
    auto plan = [&](int bm, int bn, dim3& grid, int& kps) {
        const int tiles = ((M + bm - 1) / bm) * ((N + bn - 1) / bn);
        int splits = (132 * 4 + tiles - 1) / tiles;
        const int max_splits = (Kall + 511) / 512;
        if (splits > max_splits) splits = max_splits;
        if (splits < 1) splits = 1;
        kps = ((Kall + splits - 1) / splits + BK - 1) / BK * BK;
        grid = dim3((M + bm - 1) / bm, (N + bn - 1) / bn, (Kall + kps - 1) / kps);
    };
    dim3 grid;
    int kps;
    if (M <= 16) { plan(16, 256, grid, kps); conv_wgrad_simt_kernel<16, 256><<<grid, CT, 0, st>>>(*p, kps); }
    else if (M <= 32) { plan(32, 128, grid, kps); conv_wgrad_simt_kernel<32, 128><<<grid, CT, 0, st>>>(*p, kps); }
    else { plan(64, 64, grid, kps); conv_wgrad_simt_kernel<64, 64><<<grid, CT, 0, st>>>(*p, kps); }
    SCSFM_CHECK_LAUNCH();
    if (p->dbias) return launch_bias_grad(p->dout, Kall, M, p->dbias, st);
    return SCSFM_OK;
}
