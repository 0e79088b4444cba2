// HBM-bound network operators around the convolutions: layout change, BatchNorm apply / backward,
// max-pool, nearest-upsample + concat, reflection-pad gradient fold, activation gradients, the pose
// head's spatial mean and Adam.  All NHWC fp32, float4 accesses where the channel count allows.
//
// Replaces ATen/cuDNN kernels reached from reference resnet_encoder.py:87-97 (bn, relu, maxpool),
// DispResNet.py:34,47,95 (ReflectionPad2d, interpolate, cat), PoseResNet.py:47-49 and
// train.py:176-178,280-282 (Adam) -- rows K2-K5, K11 of SURVEY.md section 2.3.
#include "nn_common.cuh"

namespace scsfm {

constexpr int NT = 256;

static inline int grid_for(long long n, int per_cta = NT) {
    long long g = (n + per_cta - 1) / per_cta;
    if (g > 132LL * 32) g = 132 * 32;   // grid-stride beyond 32 CTAs per SM
    return (int)(g < 1 ? 1 : g);
}

// ----- layout ---------------------------------------------------------------------------------
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ a, const float* __restrict__ b, int B, int C, int HW,
                                    float* __restrict__ out) {
    const int nsrc = b ? 2 : 1, Ct = C * nsrc;
    const long long total = (long long)B * HW * Ct;
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
        const int c = (int)(i % Ct);
        const long long px = i / Ct;
        const int bb = (int)(px / HW), p = (int)(px - (long long)bb * HW);
        const float* src = c < C ? a : b;
        const int cc = c < C ? c : c - C;
        out[i] = __ldg(src + ((size_t)bb * C + cc) * HW + p);
    }
}

// [B,C,H,W] (x1 or x2 sources) -> NHWC with the channel count padded to Cpad (zeros): the 7x7 stems run on the tensor
// cores with Cin 3 -> 4 / 6 -> 8
__global__ void nchw_to_nhwc_pad_kernel(const float* __restrict__ a, const float* __restrict__ b, int B, int C, int HW, int Cpad,
                                        float* __restrict__ out, int operand) {
    const int Ct = C * (b ? 2 : 1);
    const long long total = (long long)B * HW * Cpad;
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
        const int c = (int)(i % Cpad);
        const long long px = i / Cpad;
        const int bb = (int)(px / HW), p = (int)(px - (long long)bb * HW);
        float v = 0.f;
        if (c < Ct) {
            const float* src = c < C ? a : b;
            const int cc = c < C ? c : c - C;
            v = tc_operand(__ldg(src + ((size_t)bb * C + cc) * HW + p), operand);
        }
        out[i] = v;
    }
}

// rows of C floats -> rows of Cpad floats (zero padded, TF32 rounded): stem weights [64*49][3] -> [64*49][4]
__global__ void pad_channels_kernel(const float* __restrict__ src, long long rows, int C, int Cpad, float* __restrict__ dst, int operand) {
    const long long total = rows * Cpad;
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
        const int c = (int)(i % Cpad);
        const long long r = i / Cpad;
        dst[i] = c < C ? tc_operand(__ldg(src + r * C + c), operand) : 0.f;
    }
}

// dst[r][c] += src[r][c] for c < C (src rows have Cpad floats): padded stem weight gradient -> gradient arena
__global__ void unpad_add_kernel(const float* __restrict__ src, long long rows, int C, int Cpad, float* __restrict__ dst) {
    const long long total = rows * C;
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
        const int c = (int)(i % C);
        const long long r = i / C;
        dst[i] += __ldg(src + r * Cpad + c);
    }
}

__global__ void nhwc_to_nchw_kernel(const float* __restrict__ in, int B, int C, int HW, float* __restrict__ out) {
    const long long total = (long long)B * HW * C;
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
        const int p = (int)(i % HW);
        const long long bc = i / HW;
        const int c = (int)(bc % C), bb = (int)(bc / C);
        out[i] = __ldg(in + ((size_t)bb * HW + p) * C + c);
    }
}

// ----- BatchNorm --------------------------------------------------------------------------------
// saved[g][c] = {scale, shift, mean, invstd}
__global__ void bn_prepare_kernel(const double* __restrict__ sums, int G, int C, double count, const float* __restrict__ gamma,
                                  const float* __restrict__ beta, float* __restrict__ rmean, float* __restrict__ rvar,
                                  float momentum, float eps, int training, float* __restrict__ saved) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    const float g = gamma[c], bt = beta[c];
    if (training) {
        float rm = rmean[c], rv = rvar[c];
        for (int grp = 0; grp < G; ++grp) {
            double s = 0.0, q = 0.0;
            for (int slot = 0; slot < SCSFM_BN_SLOTS; ++slot) {
                s += sums[(((size_t)slot * G + grp) * C + c) * 2];
                q += sums[(((size_t)slot * G + grp) * C + c) * 2 + 1];
            }
            const double mean = s / count;
            double var = q / count - mean * mean;
            if (var < 0) var = 0;
            const float invstd = (float)(1.0 / sqrt(var + (double)eps));
            float* o = saved + ((size_t)grp * C + c) * 4;
            o[0] = g * invstd;
            o[1] = bt - (float)mean * g * invstd;
            o[2] = (float)mean;
            o[3] = invstd;
            // running statistics: one update per network call, in call order (nn.BatchNorm2d, momentum 0.1)
            const double unbiased = count > 1 ? var * count / (count - 1) : var;
            rm = (1.f - momentum) * rm + momentum * (float)mean;
            rv = (1.f - momentum) * rv + momentum * (float)unbiased;
        }
        rmean[c] = rm;
        rvar[c] = rv;
    } else {
        const float invstd = 1.0f / sqrtf(rvar[c] + eps);
        for (int grp = 0; grp < G; ++grp) {
            float* o = saved + ((size_t)grp * C + c) * 4;
            o[0] = g * invstd;
            o[1] = bt - rmean[c] * g * invstd;
            o[2] = rmean[c];
            o[3] = invstd;
        }
    }
}

// Per-channel affine of BatchNorm: shared by bn_apply_kernel (both modes) and the eval-mode prepare of the fused convolution
// epilogue, so that the two cannot diverge (the fused eval forward is bitwise the conv followed by bn_apply).
__device__ __forceinline__ float bn_eval_invstd(float running_var, float eps) { return 1.0f / sqrtf(running_var + eps); }
__device__ __forceinline__ void bn_affine(float gamma, float beta, float mean, float invstd, float& scale, float& shift) {
    scale = gamma * invstd;
    shift = beta - mean * scale;
}

// table rows {gamma, beta, running_mean, running_var, scale, shift, C, eps bits}; one CTA per layer
__global__ void __launch_bounds__(NT) bn_eval_prepare_batched_kernel(const long long* __restrict__ table) {
    const long long* e = table + (size_t)blockIdx.x * 8;
    const float* gamma = reinterpret_cast<const float*>(e[0]);
    const float* beta = reinterpret_cast<const float*>(e[1]);
    const float* rmean = reinterpret_cast<const float*>(e[2]);
    const float* rvar = reinterpret_cast<const float*>(e[3]);
    float* scale = reinterpret_cast<float*>(e[4]);
    float* shift = reinterpret_cast<float*>(e[5]);
    const int C = (int)e[6];
    const float eps = __int_as_float((int)e[7]);
    for (int c = threadIdx.x; c < C; c += NT) {
        float sc, sh;
        bn_affine(gamma[c], beta[c], rmean[c], bn_eval_invstd(rvar[c], eps), sc, sh);
        scale[c] = sc;
        shift[c] = sh;
    }
}

// z = relu?(y*scale + shift + residual), with scale/shift derived IN the kernel from the fused batch sums (training) or
// taken from `saved` (eval).  Grid (row chunks, groups, channel slabs); a thread owns 4 consecutive channels and walks
// rows, so there is no per-element index arithmetic: pure float4 streaming.  The first row-chunk CTA of every
// (group, slab) writes saved[g][c] = {scale, shift, mean, invstd}; CTA (0,0,slab) also updates the running statistics
// for all groups in call order.
__global__ void __launch_bounds__(NT)
bn_apply_kernel(const float* __restrict__ y, const double* __restrict__ sums, const float* __restrict__ gamma,
                const float* __restrict__ beta, float* __restrict__ rmean, float* __restrict__ rvar, float momentum, float eps,
                int training, float* __restrict__ saved, const float* __restrict__ res, float* __restrict__ z, float* __restrict__ z_lo,
                long long rows_per_group, int C, int G, int flags, int rows_per_cta) {
    const int g = blockIdx.y;
    const int slab4 = min(C >> 2, NT);
    const int col4 = blockIdx.z * slab4 + (threadIdx.x % slab4);
    const int row_lanes = NT / slab4, rl = threadIdx.x / slab4;
    const int c = col4 * 4;
    // per-CTA statistics: one thread per channel of the slab (not one per row lane), shared through smem
    __shared__ float s_sc[4 * NT], s_sh[4 * NT];
    const double count = (double)rows_per_group;
    const int slab_c0 = blockIdx.z * slab4 * 4, slab_cn = min(slab4 * 4, C - slab_c0);
    for (int cc = threadIdx.x; cc < slab_cn; cc += NT) {
        const int ch = slab_c0 + cc;
        float mean, invstd;
        if (training) {
            double s1 = 0.0, s2 = 0.0;
            for (int slot = 0; slot < SCSFM_BN_SLOTS; ++slot) {
                s1 += sums[(((size_t)slot * G + g) * C + ch) * 2];
                s2 += sums[(((size_t)slot * G + g) * C + ch) * 2 + 1];
            }
            const double m = s1 / count;
            double var = s2 / count - m * m;
            if (var < 0) var = 0;
            mean = (float)m;
            invstd = (float)(1.0 / sqrt(var + (double)eps));
        } else {
            mean = rmean[ch];
            invstd = bn_eval_invstd(rvar[ch], eps);
        }
        float scale, shift;
        bn_affine(gamma[ch], beta[ch], mean, invstd, scale, shift);
        s_sc[cc] = scale;
        s_sh[cc] = shift;
        if (blockIdx.x == 0) {
            float* o = saved + ((size_t)g * C + ch) * 4;
            o[0] = scale; o[1] = shift; o[2] = mean; o[3] = invstd;
        }
    }
    __syncthreads();
    if (c >= C || rl >= row_lanes) return;
    float sc[4], sh[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        sc[j] = s_sc[c - slab_c0 + j];
        sh[j] = s_sh[c - slab_c0 + j];
    }
    if (training && blockIdx.x == 0 && blockIdx.y == 0 && rl == 0) {
        // running statistics: one update per network call, in call order (nn.BatchNorm2d, momentum 0.1, unbiased variance)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float rm = rmean[c + j], rv = rvar[c + j];
            for (int grp = 0; grp < G; ++grp) {
                double s1 = 0.0, s2 = 0.0;
                for (int slot = 0; slot < SCSFM_BN_SLOTS; ++slot) {
                    s1 += sums[(((size_t)slot * G + grp) * C + c + j) * 2];
                    s2 += sums[(((size_t)slot * G + grp) * C + c + j) * 2 + 1];
                }
                const double m = s1 / count;
                double var = s2 / count - m * m;
                if (var < 0) var = 0;
                const double unbiased = count > 1 ? var * count / (count - 1) : var;
                rm = (1.f - momentum) * rm + momentum * (float)m;
                rv = (1.f - momentum) * rv + momentum * (float)unbiased;
            }
            rmean[c + j] = rm;
            rvar[c + j] = rv;
        }
    }
    const long long r0 = (long long)g * rows_per_group + (long long)blockIdx.x * rows_per_cta;
    const long long r1 = min((long long)(g + 1) * rows_per_group, r0 + rows_per_cta);
    const bool relu = flags & 1, rnd = flags & ROUND_TF32;
    for (long long r = r0 + rl; r < r1; r += row_lanes) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(y + r * C + c));
        float o[4] = {fmaf(v.x, sc[0], sh[0]), fmaf(v.y, sc[1], sh[1]), fmaf(v.z, sc[2], sh[2]), fmaf(v.w, sc[3], sh[3])};
        if (res) {
            const float4 rr = __ldg(reinterpret_cast<const float4*>(res + r * C + c));
            o[0] += rr.x; o[1] += rr.y; o[2] += rr.z; o[3] += rr.w;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (relu) o[j] = fmaxf(o[j], 0.f);
            if (rnd) o[j] = tf32_round(o[j]);
        }
        *reinterpret_cast<float4*>(z + r * C + c) = make_float4(o[0], o[1], o[2], o[3]);
        // split-accumulate mode: the low part of the tensor-core operand, produced with the tensor itself
        if (z_lo) *reinterpret_cast<float4*>(z_lo + r * C + c) = make_float4(tf32_lo(o[0]), tf32_lo(o[1]), tf32_lo(o[2]), tf32_lo(o[3]));
    }
}

// pass 1: work[g][c] = { sum dz', sum dz' * xhat }  (dz' = dz gated by relu)
// One CTA = a chunk of rows x a slab of up to 1024 channels; every thread owns 4 consecutive channels
// (float4 loads, a row of the slab is one contiguous segment) and strides over the chunk's rows.
__global__ void __launch_bounds__(NT)
bn_bwd_reduce_kernel(const float* __restrict__ dz, const float* __restrict__ z, const float* __restrict__ y,
                     const float* __restrict__ saved, long long rows_per_group, int C, int relu, int rows_per_cta,
                     double* __restrict__ work) {
    const int g = blockIdx.y;
    const int slab4 = min(C >> 2, NT);                    // float4 columns handled by this CTA
    const int col4 = blockIdx.z * slab4 + (threadIdx.x % slab4);
    const int row_lanes = NT / slab4, rl = threadIdx.x / slab4;
    const int c = col4 * 4;
    const long long r0 = (long long)g * rows_per_group + (long long)blockIdx.x * rows_per_cta;
    const long long r1 = min((long long)(g + 1) * rows_per_group, r0 + rows_per_cta);
    float s0[4] = {0.f, 0.f, 0.f, 0.f}, s1[4] = {0.f, 0.f, 0.f, 0.f};
    const bool active = c < C && rl < row_lanes;
    if (active) {
        float mean[4], invstd[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            mean[j] = saved[((size_t)g * C + c + j) * 4 + 2];
            invstd[j] = saved[((size_t)g * C + c + j) * 4 + 3];
        }
        for (long long r = r0 + rl; r < r1; r += row_lanes) {
            const float4 d4 = __ldg(reinterpret_cast<const float4*>(dz + r * C + c));
            const float4 y4 = __ldg(reinterpret_cast<const float4*>(y + r * C + c));
            float d[4] = {d4.x, d4.y, d4.z, d4.w};
            const float yy[4] = {y4.x, y4.y, y4.z, y4.w};
            if (relu & 1) {
                const float4 z4 = __ldg(reinterpret_cast<const float4*>(z + r * C + c));
                if (!(z4.x > 0.f)) d[0] = 0.f;
                if (!(z4.y > 0.f)) d[1] = 0.f;
                if (!(z4.z > 0.f)) d[2] = 0.f;
                if (!(z4.w > 0.f)) d[3] = 0.f;
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                s0[j] += d[j];
                s1[j] += d[j] * ((yy[j] - mean[j]) * invstd[j]);
            }
        }
    }
    __shared__ float sh[8][NT];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        sh[j][threadIdx.x] = s0[j];
        sh[4 + j][threadIdx.x] = s1[j];
    }
    __syncthreads();
    if (threadIdx.x < slab4 && c < C) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float a = 0.f, b = 0.f;
            for (int l = 0; l < row_lanes; ++l) {
                a += sh[j][l * slab4 + threadIdx.x];
                b += sh[4 + j][l * slab4 + threadIdx.x];
            }
            atomicAdd(work + ((size_t)g * C + c + j) * 2, (double)a);
            atomicAdd(work + ((size_t)g * C + c + j) * 2 + 1, (double)b);
        }
    }
}

// pass 2: dy = gamma*invstd*(dz' - mean(dz') - xhat*mean(dz' xhat)); dres = dz'.  Same grid / thread layout as pass 1.
__global__ void __launch_bounds__(NT)
bn_bwd_apply_kernel(const float* __restrict__ dz, const float* __restrict__ z, const float* __restrict__ y,
                    const float* __restrict__ saved, const double* __restrict__ work, float* __restrict__ dy, float* __restrict__ dy_lo,
                    float* __restrict__ dres, long long rows_per_group, int C, int relu, int rows_per_cta) {
    const int g = blockIdx.y;
    const int slab4 = min(C >> 2, NT);
    const int col4 = blockIdx.z * slab4 + (threadIdx.x % slab4);
    const int row_lanes = NT / slab4, rl = threadIdx.x / slab4;
    const int c = col4 * 4;
    if (c >= C || rl >= row_lanes) return;
    const float inv_n = 1.0f / (float)rows_per_group;
    float sc[4], mean[4], invstd[4], m1[4], m2[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float* sv = saved + ((size_t)g * C + c + j) * 4;
        sc[j] = sv[0]; mean[j] = sv[2]; invstd[j] = sv[3];
        m1[j] = (float)work[((size_t)g * C + c + j) * 2] * inv_n;
        m2[j] = (float)work[((size_t)g * C + c + j) * 2 + 1] * inv_n;
    }
    const long long r0 = (long long)g * rows_per_group + (long long)blockIdx.x * rows_per_cta;
    const long long r1 = min((long long)(g + 1) * rows_per_group, r0 + rows_per_cta);
    const bool gate = relu & 1, rnd = relu & ROUND_TF32;
    for (long long r = r0 + rl; r < r1; r += row_lanes) {
        const float4 d4 = __ldg(reinterpret_cast<const float4*>(dz + r * C + c));
        const float4 y4 = __ldg(reinterpret_cast<const float4*>(y + r * C + c));
        float d[4] = {d4.x, d4.y, d4.z, d4.w};
        const float yy[4] = {y4.x, y4.y, y4.z, y4.w};
        if (gate) {
            const float4 z4 = __ldg(reinterpret_cast<const float4*>(z + r * C + c));
            if (!(z4.x > 0.f)) d[0] = 0.f;
            if (!(z4.y > 0.f)) d[1] = 0.f;
            if (!(z4.z > 0.f)) d[2] = 0.f;
            if (!(z4.w > 0.f)) d[3] = 0.f;
        }
        float o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float xhat = (yy[j] - mean[j]) * invstd[j];
            o[j] = sc[j] * (d[j] - m1[j] - xhat * m2[j]);
            if (rnd) o[j] = tf32_round(o[j]);
        }
        if (dres) *reinterpret_cast<float4*>(dres + r * C + c) = make_float4(d[0], d[1], d[2], d[3]);
        *reinterpret_cast<float4*>(dy + r * C + c) = make_float4(o[0], o[1], o[2], o[3]);
        if (dy_lo) *reinterpret_cast<float4*>(dy_lo + r * C + c) = make_float4(tf32_lo(o[0]), tf32_lo(o[1]), tf32_lo(o[2]), tf32_lo(o[3]));
    }
}

// Frozen statistics (eval mode: `saved` holds the running-statistics {scale, shift, mean, invstd}): dy = scale*dz' and dres = dz'
// need no batch reduction, so one pass does the apply and, when `work` is given, the parameter-gradient sums
// work[g][c] = { sum dz', sum dz' * xhat } (xhat from the running mean / invstd).  Grid / thread layout of bn_bwd_reduce_kernel.
__global__ void __launch_bounds__(NT)
bn_bwd_frozen_kernel(const float* __restrict__ dz, const float* __restrict__ z, const float* __restrict__ y,
                     const float* __restrict__ saved, float* __restrict__ dy, float* __restrict__ dy_lo, float* __restrict__ dres,
                     long long rows_per_group, int C, int relu, int rows_per_cta, double* __restrict__ work) {
    const int g = blockIdx.y;
    const int slab4 = min(C >> 2, NT);
    const int col4 = blockIdx.z * slab4 + (threadIdx.x % slab4);
    const int row_lanes = NT / slab4, rl = threadIdx.x / slab4;
    const int c = col4 * 4;
    const long long r0 = (long long)g * rows_per_group + (long long)blockIdx.x * rows_per_cta;
    const long long r1 = min((long long)(g + 1) * rows_per_group, r0 + rows_per_cta);
    float s0[4] = {0.f, 0.f, 0.f, 0.f}, s1[4] = {0.f, 0.f, 0.f, 0.f};
    const bool active = c < C && rl < row_lanes;
    if (active) {
        float sc[4], mean[4], invstd[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float* sv = saved + ((size_t)g * C + c + j) * 4;
            sc[j] = sv[0]; mean[j] = sv[2]; invstd[j] = sv[3];
        }
        const bool gate = relu & 1, rnd = relu & ROUND_TF32;
        for (long long r = r0 + rl; r < r1; r += row_lanes) {
            const float4 d4 = __ldg(reinterpret_cast<const float4*>(dz + r * C + c));
            float d[4] = {d4.x, d4.y, d4.z, d4.w};
            if (gate) {
                const float4 z4 = __ldg(reinterpret_cast<const float4*>(z + r * C + c));
                if (!(z4.x > 0.f)) d[0] = 0.f;
                if (!(z4.y > 0.f)) d[1] = 0.f;
                if (!(z4.z > 0.f)) d[2] = 0.f;
                if (!(z4.w > 0.f)) d[3] = 0.f;
            }
            float o[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                o[j] = sc[j] * d[j];
                if (rnd) o[j] = tf32_round(o[j]);
            }
            if (dres) *reinterpret_cast<float4*>(dres + r * C + c) = make_float4(d[0], d[1], d[2], d[3]);
            *reinterpret_cast<float4*>(dy + r * C + c) = make_float4(o[0], o[1], o[2], o[3]);
            if (dy_lo) *reinterpret_cast<float4*>(dy_lo + r * C + c) = make_float4(tf32_lo(o[0]), tf32_lo(o[1]), tf32_lo(o[2]), tf32_lo(o[3]));
            if (work) {
                const float4 y4 = __ldg(reinterpret_cast<const float4*>(y + r * C + c));
                const float yy[4] = {y4.x, y4.y, y4.z, y4.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    s0[j] += d[j];
                    s1[j] += d[j] * ((yy[j] - mean[j]) * invstd[j]);
                }
            }
        }
    }
    if (!work) return;
    __shared__ float sh[8][NT];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        sh[j][threadIdx.x] = s0[j];
        sh[4 + j][threadIdx.x] = s1[j];
    }
    __syncthreads();
    if (threadIdx.x < slab4 && c < C) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float a = 0.f, b = 0.f;
            for (int l = 0; l < row_lanes; ++l) {
                a += sh[j][l * slab4 + threadIdx.x];
                b += sh[4 + j][l * slab4 + threadIdx.x];
            }
            atomicAdd(work + ((size_t)g * C + c + j) * 2, (double)a);
            atomicAdd(work + ((size_t)g * C + c + j) * 2 + 1, (double)b);
        }
    }
}

__global__ void bn_param_grad_kernel(const double* __restrict__ work, int G, int C, float* __restrict__ dgamma,
                                     float* __restrict__ dbeta) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double a = 0, b = 0;
    for (int g = 0; g < G; ++g) {
        a += work[((size_t)g * C + c) * 2];
        b += work[((size_t)g * C + c) * 2 + 1];
    }
    if (dbeta) dbeta[c] += (float)a;
    if (dgamma) dgamma[c] += (float)b;
}

// ----- max-pool 3x3 stride 2 pad 1 --------------------------------------------------------------
__global__ void maxpool_fwd_kernel(const float* __restrict__ x, int B, int H, int W, int C, int Ho, int Wo,
                                   float* __restrict__ y, unsigned char* __restrict__ idx) {
    const int C4 = C >> 2;
    const long long total = (long long)B * Ho * Wo * C4;
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
        const int c = (int)(i % C4) * 4;
        long long t = i / C4;
        const int wo = (int)(t % Wo); t /= Wo;
        const int ho = (int)(t % Ho);
        const int b = (int)(t / Ho);
        float best[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
        unsigned char bi[4] = {0, 0, 0, 0};
#pragma unroll
        for (int dy = 0; dy < 3; ++dy) {
            const int h = ho * 2 + dy - 1;
            if (h < 0 || h >= H) continue;
#pragma unroll
            for (int dx = 0; dx < 3; ++dx) {
                const int w = wo * 2 + dx - 1;
                if (w < 0 || w >= W) continue;
                const float4 v = __ldg(reinterpret_cast<const float4*>(x + (((size_t)b * H + h) * W + w) * C + c));
                const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (vv[j] > best[j] || vv[j] != vv[j]) { best[j] = vv[j]; bi[j] = (unsigned char)(dy * 3 + dx); }
            }
        }
        reinterpret_cast<float4*>(y)[i] = make_float4(best[0], best[1], best[2], best[3]);
        reinterpret_cast<uchar4*>(idx)[i] = make_uchar4(bi[0], bi[1], bi[2], bi[3]);
    }
}

__global__ void maxpool_bwd_kernel(const float* __restrict__ dy, const unsigned char* __restrict__ idx, int B, int H, int W,
                                   int C, int Ho, int Wo, float* __restrict__ dx, int accumulate) {
    const int C4 = C >> 2;
    const long long total = (long long)B * H * W * C4;
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
        const int c = (int)(i % C4) * 4;
        long long t = i / C4;
        const int w = (int)(t % W); t /= W;
        const int h = (int)(t % H);
        const int b = (int)(t / H);
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        // output windows that contain (h, w): ho in {(h+1)/2 - 1 .. (h+1)/2}, tap dy = h + 1 - 2*ho
        for (int ho = (h + 1) / 2 - 1; ho <= (h + 1) / 2; ++ho) {
            const int dyy = h + 1 - 2 * ho;
            if (ho < 0 || ho >= Ho || dyy < 0 || dyy > 2) continue;
            for (int wo = (w + 1) / 2 - 1; wo <= (w + 1) / 2; ++wo) {
                const int dxx = w + 1 - 2 * wo;
                if (wo < 0 || wo >= Wo || dxx < 0 || dxx > 2) continue;
                const size_t o = (((size_t)b * Ho + ho) * Wo + wo) * C + c;
                const uchar4 k = *reinterpret_cast<const uchar4*>(idx + o);
                const float4 g = __ldg(reinterpret_cast<const float4*>(dy + o));
                const unsigned char me = (unsigned char)(dyy * 3 + dxx);
                if (k.x == me) acc[0] += g.x;
                if (k.y == me) acc[1] += g.y;
                if (k.z == me) acc[2] += g.z;
                if (k.w == me) acc[3] += g.w;
            }
        }
        float4* dst = reinterpret_cast<float4*>(dx) + i;
        if (accumulate) {
            const float4 old = *dst;
            acc[0] += old.x; acc[1] += old.y; acc[2] += old.z; acc[3] += old.w;
        }
        *dst = make_float4(acc[0], acc[1], acc[2], acc[3]);
    }
}

// ----- nearest x2 upsample + channel concat -----------------------------------------------------
__global__ void upcat_fwd_kernel(const float* __restrict__ lo, const float* __restrict__ skip, int B, int H, int W, int C1,
                                 int C2, float* __restrict__ out) {
    const int Ct4 = (C1 + C2) >> 2, C14 = C1 >> 2;
    const long long total = (long long)B * H * W * Ct4;
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
        const int c4 = (int)(i % Ct4);
        long long t = i / Ct4;
        const int w = (int)(t % W); t /= W;
        const int h = (int)(t % H);
        const int b = (int)(t / H);
        float4 v;
        if (c4 < C14) v = __ldg(reinterpret_cast<const float4*>(lo + (((size_t)b * (H / 2) + h / 2) * (W / 2) + w / 2) * C1) + c4);
        else v = __ldg(reinterpret_cast<const float4*>(skip + (((size_t)b * H + h) * W + w) * C2) + (c4 - C14));
        reinterpret_cast<float4*>(out)[i] = v;
    }
}

__device__ __forceinline__ float act_grad(float out, int act) {
    switch (act & 0xff) {
        case ACT_RELU: return out > 0.f ? 1.f : 0.f;
        case ACT_ELU: return out > 0.f ? 1.f : out + 1.f;          // d/dx elu = exp(x) = elu(x)+1 for x<=0
        case ACT_DISP: { const float s = (out - 0.01f) * 0.1f; return 10.f * s * (1.f - s); }
        default: return 1.f;
    }
}

// gradient of the reflect-padded tensor folded back onto pixel (h, w): the pixel itself plus the mirrored
// border entries (pad row -1 mirrors row 1, pad row H mirrors row H-2; same for columns)
__device__ __forceinline__ float4 fold_at(const float* __restrict__ dpad, int b, int h, int w, int H, int W, int Ct, int c) {
    const int Hp = H + 2, Wp = W + 2;
    int ys[3], xs[3], ny = 0, nx = 0;
    ys[ny++] = h + 1;
    if (h == 1) ys[ny++] = 0;
    if (h == H - 2) ys[ny++] = H + 1;
    xs[nx++] = w + 1;
    if (w == 1) xs[nx++] = 0;
    if (w == W - 2) xs[nx++] = W + 1;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int iy = 0; iy < ny; ++iy)
        for (int ix = 0; ix < nx; ++ix) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(dpad + (((size_t)b * Hp + ys[iy]) * Wp + xs[ix]) * Ct + c));
            a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
        }
    return a;
}

// plain fold: d[b,h,w,c] (+)= fold(dpad); then *= act'(act_out)
__global__ void fold_plain_kernel(const float* __restrict__ dpad, int B, int H, int W, int C, float* __restrict__ d,
                                  const float* __restrict__ act_out, int act, int accumulate) {
    const int C4 = C >> 2;
    const long long total = (long long)B * H * W * C4;
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
        const int c = (int)(i % C4) * 4;
        long long t = i / C4;
        const int w = (int)(t % W); t /= W;
        const int h = (int)(t % H);
        const int b = (int)(t / H);
        float4 a = fold_at(dpad, b, h, w, H, W, C, c);
        float4* dst = reinterpret_cast<float4*>(d) + i;
        if (accumulate) { const float4 o = *dst; a.x += o.x; a.y += o.y; a.z += o.z; a.w += o.w; }
        if ((act & 0xff) != ACT_NONE) {
            const float4 q = __ldg(reinterpret_cast<const float4*>(act_out) + i);
            a.x *= act_grad(q.x, act); a.y *= act_grad(q.y, act); a.z *= act_grad(q.z, act); a.w *= act_grad(q.w, act);
        }
        if (act & ROUND_TF32) { a.x = tf32_round(a.x); a.y = tf32_round(a.y); a.z = tf32_round(a.z); a.w = tf32_round(a.w); }
        *dst = a;
    }
}

// upsample+concat fold, low-resolution part: d_lo[b,h2,w2,c] = sum_{2x2} fold(dpad)[.., c] * act'(lo_act)
__global__ void fold_up_lo_kernel(const float* __restrict__ dpad, int B, int H, int W, int C1, int Ct, float* __restrict__ d_lo,
                                  const float* __restrict__ lo_act, int act) {
    const int C4 = C1 >> 2, H2 = H / 2, W2 = W / 2;
    const long long total = (long long)B * H2 * W2 * C4;
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
        const int c = (int)(i % C4) * 4;
        long long t = i / C4;
        const int w2 = (int)(t % W2); t /= W2;
        const int h2 = (int)(t % H2);
        const int b = (int)(t / H2);
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) {
                const float4 v = fold_at(dpad, b, 2 * h2 + dy, 2 * w2 + dx, H, W, Ct, c);
                a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
            }
        if ((act & 0xff) != ACT_NONE) {
            const float4 q = __ldg(reinterpret_cast<const float4*>(lo_act) + i);
            a.x *= act_grad(q.x, act); a.y *= act_grad(q.y, act); a.z *= act_grad(q.z, act); a.w *= act_grad(q.w, act);
        }
        if (act & ROUND_TF32) { a.x = tf32_round(a.x); a.y = tf32_round(a.y); a.z = tf32_round(a.z); a.w = tf32_round(a.w); }
        reinterpret_cast<float4*>(d_lo)[i] = a;
    }
}

// upsample+concat fold, skip part: d_skip[b,h,w,c] = fold(dpad)[.., C1 + c]   (each skip feeds one conv)
__global__ void fold_up_skip_kernel(const float* __restrict__ dpad, int B, int H, int W, int C1, int C2, float* __restrict__ d_skip) {
    const int C4 = C2 >> 2;
    const long long total = (long long)B * H * W * C4;
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
        const int c = (int)(i % C4) * 4;
        long long t = i / C4;
        const int w = (int)(t % W); t /= W;
        const int h = (int)(t % H);
        const int b = (int)(t / H);
        const float4 a = fold_at(dpad, b, h, w, H, W, C1 + C2, C1 + c);
        reinterpret_cast<float4*>(d_skip)[i] = a;
    }
}

__global__ void act_bwd_kernel(float* __restrict__ d, const float* __restrict__ out, long long n, int act) {
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < n; i += (long long)gridDim.x * NT)
        d[i] = maybe_round(d[i] * act_grad(__ldg(out + i), act), act & ROUND_TF32);
}

// ----- pose head --------------------------------------------------------------------------------
__global__ void spatial_mean_fwd_kernel(const float* __restrict__ x, int HW, int C, float scale, float* __restrict__ out) {
    // one CTA per (b, c)
    __shared__ float red[32];
    const int b = blockIdx.x / C, c = blockIdx.x % C;
    float acc = 0.f;
    for (int p = threadIdx.x; p < HW; p += blockDim.x) acc += __ldg(x + ((size_t)b * HW + p) * C + c);
    acc = block_sum<NT / 32>(acc, red);
    if (threadIdx.x == 0) out[blockIdx.x] = scale * (acc / (float)HW);
}

__global__ void spatial_mean_bwd_kernel(const float* __restrict__ dout, int B, int HW, int C, float scale, float* __restrict__ dx) {
    const long long total = (long long)B * HW * C;
    const float k = scale / (float)HW;
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
        const int c = (int)(i % C);
        const int b = (int)(i / ((long long)HW * C));
        dx[i] = __ldg(dout + b * C + c) * k;
    }
}

// ----- TF32 rounding of a whole buffer (weights, once per optimizer step) ----------------------------
__global__ void round_tf32_kernel(const float* __restrict__ in, float* __restrict__ out, long long n) {
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < n; i += (long long)gridDim.x * NT) out[i] = tf32_round(__ldg(in + i));
}

// ----- low part of a split-accumulate operand: lo = tf32(x - trunc_tf32(x)), 16 bytes per thread and iteration ---------
__global__ void __launch_bounds__(NT) split_tf32_kernel(const float* __restrict__ in, float* __restrict__ lo, long long n4, long long n) {
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < n4; i += (long long)gridDim.x * NT) {
        const float4 x = __ldg(reinterpret_cast<const float4*>(in) + i);
        reinterpret_cast<float4*>(lo)[i] = make_float4(tf32_lo(x.x), tf32_lo(x.y), tf32_lo(x.z), tf32_lo(x.w));
    }
    if (blockIdx.x == 0 && threadIdx.x < (int)(n - 4 * n4)) lo[4 * n4 + threadIdx.x] = tf32_lo(__ldg(in + 4 * n4 + threadIdx.x));
}

// ----- Adam ---------------------------------------------------------------------------------------
// torch.optim.Adam (non-amsgrad): m = b1 m + (1-b1) g ; v = b2 v + (1-b2) g^2 ;
// p -= lr/bc1 * m / (sqrt(v)/sqrt(bc2) + eps).  The step count may live on the device so that a captured
// CUDA graph of the training step stays valid across replays.
struct AdamCoeffs {
    float step_size, bc2_sqrt;
};

__device__ __forceinline__ AdamCoeffs adam_coeffs(float lr, float b1, float b2, int step_host, const int* __restrict__ step_dev) {
    const int step = step_dev ? *step_dev : step_host;
    const float bc1 = 1.0f - powf(b1, (float)step);
    return AdamCoeffs{lr / bc1, sqrtf(1.0f - powf(b2, (float)step))};
}

// the update of element i: shared by the whole-arena and the masked kernel, so both give the same bits
__device__ __forceinline__ void adam_update(long long i, float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                            float* __restrict__ v, float b1, float b2, float eps, float wd, AdamCoeffs c,
                                            float* __restrict__ mirror, int mirror_operand) {
    float gr = g[i];
    const float pp = p[i];
    if (wd != 0.f) gr += wd * pp;
    const float mm = b1 * m[i] + (1.f - b1) * gr;
    const float vv = b2 * v[i] + (1.f - b2) * gr * gr;
    m[i] = mm;
    v[i] = vv;
    const float pn = pp - c.step_size * (mm / (sqrtf(vv) / c.bc2_sqrt + eps));
    p[i] = pn;
    if (mirror != nullptr) mirror[i] = tc_operand(pn, mirror_operand);      // operand mirror of the tensor-core convolutions
}

__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                            long long n, float lr, float b1, float b2, float eps, float wd, int step_host,
                            const int* __restrict__ step_dev, float* __restrict__ mirror, int mirror_operand) {
    const AdamCoeffs c = adam_coeffs(lr, b1, b2, step_host, step_dev);
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < n; i += (long long)gridDim.x * NT)
        adam_update(i, p, g, m, v, b1, b2, eps, wd, c, mirror, mirror_operand);
}

// Frozen parameters (torch.optim.Adam skips `grad is None`): chunk_mask[i / 64] == 0 leaves element i's parameter, moments and
// operand mirror untouched.  Every parameter of an arena starts on a 64-float boundary, so a chunk never straddles two of them.
__global__ void adam_masked_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                   long long n, const unsigned char* __restrict__ chunk_mask, float lr, float b1, float b2, float eps,
                                   float wd, int step_host, const int* __restrict__ step_dev, float* __restrict__ mirror,
                                   int mirror_operand) {
    const AdamCoeffs c = adam_coeffs(lr, b1, b2, step_host, step_dev);
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < n; i += (long long)gridDim.x * NT)
        if (__ldg(chunk_mask + (i >> 6))) adam_update(i, p, g, m, v, b1, b2, eps, wd, c, mirror, mirror_operand);
}

}  // namespace scsfm

using namespace scsfm;
#define ST ((cudaStream_t)stream)

extern "C" int scsfm_nchw_to_nhwc(const float* a, const float* b, int B, int C, int H, int W, float* out, void* stream) {
    SCSFM_CHECK_ARG(a && out && B > 0 && C > 0 && H > 0 && W > 0, "nchw_to_nhwc: bad arguments");
    const long long n = (long long)B * H * W * C * (b ? 2 : 1);
    nchw_to_nhwc_kernel<<<grid_for(n), NT, 0, ST>>>(a, b, B, C, H * W, out);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_nchw_to_nhwc_pad(const float* a, const float* b, int B, int C, int H, int W, int Cpad, float* out, int operand, void* stream) {
    SCSFM_CHECK_ARG(a && out && B > 0 && C > 0 && H > 0 && W > 0 && Cpad >= C * (b ? 2 : 1) && operand >= 0 && operand <= 2, "nchw_to_nhwc_pad: bad arguments");
    nchw_to_nhwc_pad_kernel<<<grid_for((long long)B * H * W * Cpad), NT, 0, ST>>>(a, b, B, C, H * W, Cpad, out, operand);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_pad_channels(const float* src, long long rows, int C, int Cpad, float* dst, int operand, void* stream) {
    SCSFM_CHECK_ARG(src && dst && rows > 0 && C > 0 && Cpad >= C && operand >= 0 && operand <= 2, "pad_channels: bad arguments");
    pad_channels_kernel<<<grid_for(rows * Cpad), NT, 0, ST>>>(src, rows, C, Cpad, dst, operand);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_unpad_add(const float* src, long long rows, int C, int Cpad, float* dst, void* stream) {
    SCSFM_CHECK_ARG(src && dst && rows > 0 && C > 0 && Cpad >= C, "unpad_add: bad arguments");
    unpad_add_kernel<<<grid_for(rows * C), NT, 0, ST>>>(src, rows, C, Cpad, dst);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_nhwc_to_nchw(const float* in, int B, int C, int H, int W, float* out, void* stream) {
    SCSFM_CHECK_ARG(in && out && B > 0 && C > 0 && H > 0 && W > 0, "nhwc_to_nchw: bad arguments");
    nhwc_to_nchw_kernel<<<grid_for((long long)B * H * W * C), NT, 0, ST>>>(in, B, C, H * W, out);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_bn_prepare(const double* sums, int groups, int C, long long count_per_group, const float* gamma,
                                const float* beta, float* running_mean, float* running_var, float momentum, float eps,
                                int training, float* saved, void* stream) {
    SCSFM_CHECK_ARG(gamma && beta && running_mean && running_var && saved && groups > 0 && C > 0, "bn_prepare: bad arguments");
    SCSFM_CHECK_ARG(!training || (sums && count_per_group > 0), "bn_prepare: training mode needs batch sums");
    bn_prepare_kernel<<<(C + 127) / 128, 128, 0, ST>>>(sums, groups, C, (double)count_per_group, gamma, beta, running_mean,
                                                       running_var, momentum, eps, training, saved);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

static void bn_grid(long long rpg, int C, int groups, dim3& grid, int& rpc) {
    const int slab4 = (C / 4) < NT ? (C / 4) : NT;
    const int slabs = (C / 4 + slab4 - 1) / slab4;
    const int row_lanes = NT / slab4;
    long long want = (132LL * 6 + (long long)groups * slabs - 1) / ((long long)groups * slabs);
    long long max_chunks = (rpg + 4LL * row_lanes - 1) / (4LL * row_lanes);
    if (want > max_chunks) want = max_chunks;
    if (want < 1) want = 1;
    rpc = (int)((rpg + want - 1) / want);
    grid = dim3((unsigned)((rpg + rpc - 1) / rpc), groups, slabs);
}

// z = relu?(bn(y) + residual).  Training: statistics from the fused sums (also writes `saved`, updates running stats);
// eval (sums == NULL): running statistics.
extern "C" int scsfm_bn_apply(const float* y, const double* sums, const float* gamma, const float* beta, float* running_mean,
                              float* running_var, float momentum, float eps, float* saved, const float* residual, float* z,
                              float* z_lo, long long rows, int C, int groups, int flags, void* stream) {
    SCSFM_CHECK_ARG(y && gamma && beta && running_mean && running_var && saved && z && rows > 0 && C > 0 && (C & 3) == 0 && groups > 0 &&
                        rows % groups == 0, "bn_apply: bad arguments");
    dim3 grid;
    int rpc;
    bn_grid(rows / groups, C, groups, grid, rpc);
    bn_apply_kernel<<<grid, NT, 0, ST>>>(y, sums, gamma, beta, running_mean, running_var, momentum, eps, sums != nullptr, saved, residual, z, z_lo,
                                         rows / groups, C, groups, flags, rpc);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_bn_eval_prepare_batched(const long long* table, int n_layers, void* stream) {
    SCSFM_CHECK_ARG(table != nullptr && n_layers > 0, "bn_eval_prepare_batched: bad arguments");
    bn_eval_prepare_batched_kernel<<<n_layers, NT, 0, ST>>>(table);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_bn_backward(const float* dz, const float* z, const float* y, const float* saved, const float* gamma,
                                 float* dy, float* dy_lo, float* dres, float* dgamma, float* dbeta, long long rows, int C, int groups,
                                 int relu, double* work, void* stream) {
    (void)gamma;
    SCSFM_CHECK_ARG(dz && y && saved && dy && work && rows > 0 && C > 0 && (C & 3) == 0 && groups > 0 && rows % groups == 0,
                    "bn_backward: bad arguments");
    SCSFM_CHECK_ARG(!(relu & 1) || z, "bn_backward: relu gate needs z");
    const long long rpg = rows / groups;
    const bool param_grads = dgamma || dbeta;
    const int slab4 = (C / 4) < NT ? (C / 4) : NT;
    const int slabs = (C / 4 + slab4 - 1) / slab4;
    const int row_lanes = NT / slab4;
    // enough CTAs to fill the machine (4 per SM), at least 8 rows per row-lane per CTA
    long long want = (132LL * 4 + (long long)groups * slabs - 1) / ((long long)groups * slabs);
    long long max_chunks = (rpg + 8LL * row_lanes - 1) / (8LL * row_lanes);
    if (want > max_chunks) want = max_chunks;
    if (want < 1) want = 1;
    const int rpc = (int)((rpg + want - 1) / want);
    if (relu & SCSFM_BN_FROZEN) {
        // running statistics: one pass, and the sums only when a parameter gradient is wanted
        if (param_grads) SCSFM_CHECK_CUDA(cudaMemsetAsync(work, 0, (size_t)groups * C * 2 * sizeof(double), ST));
        bn_bwd_frozen_kernel<<<dim3((unsigned)((rpg + rpc - 1) / rpc), groups, slabs), NT, 0, ST>>>(dz, z, y, saved, dy, dy_lo, dres, rpg, C,
                                                                                                  relu, rpc, param_grads ? work : nullptr);
        SCSFM_CHECK_LAUNCH();
        if (param_grads) {
            bn_param_grad_kernel<<<(C + 127) / 128, 128, 0, ST>>>(work, groups, C, dgamma, dbeta);
            SCSFM_CHECK_LAUNCH();
        }
        return SCSFM_OK;
    }
    SCSFM_CHECK_CUDA(cudaMemsetAsync(work, 0, (size_t)groups * C * 2 * sizeof(double), ST));
    bn_bwd_reduce_kernel<<<dim3((unsigned)((rpg + rpc - 1) / rpc), groups, slabs), NT, 0, ST>>>(dz, z, y, saved, rpg, C, relu, rpc, work);
    SCSFM_CHECK_LAUNCH();
    {
        dim3 grid2;
        int rpc2;
        bn_grid(rpg, C, groups, grid2, rpc2);
        bn_bwd_apply_kernel<<<grid2, NT, 0, ST>>>(dz, z, y, saved, work, dy, dy_lo, dres, rpg, C, relu, rpc2);
    }
    SCSFM_CHECK_LAUNCH();
    if (dgamma || dbeta) {
        bn_param_grad_kernel<<<(C + 127) / 128, 128, 0, ST>>>(work, groups, C, dgamma, dbeta);
        SCSFM_CHECK_LAUNCH();
    }
    return SCSFM_OK;
}

extern "C" int scsfm_maxpool_fwd(const float* x, int B, int H, int W, int C, float* y, unsigned char* idx, void* stream) {
    SCSFM_CHECK_ARG(x && y && idx && B > 0 && H > 1 && W > 1 && C > 0 && (C & 3) == 0, "maxpool_fwd: bad arguments");
    const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
    maxpool_fwd_kernel<<<grid_for((long long)B * Ho * Wo * (C / 4)), NT, 0, ST>>>(x, B, H, W, C, Ho, Wo, y, idx);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_maxpool_bwd(const float* dy, const unsigned char* idx, int B, int H, int W, int C, float* dx, int accumulate,
                                 void* stream) {
    SCSFM_CHECK_ARG(dy && idx && dx && B > 0 && H > 1 && W > 1 && C > 0 && (C & 3) == 0, "maxpool_bwd: bad arguments");
    const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
    maxpool_bwd_kernel<<<grid_for((long long)B * H * W * (C / 4)), NT, 0, ST>>>(dy, idx, B, H, W, C, Ho, Wo, dx, accumulate);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_upcat_fwd(const float* lo, const float* skip, int B, int H, int W, int C1, int C2, float* out, void* stream) {
    SCSFM_CHECK_ARG(lo && out && B > 0 && H > 0 && W > 0 && (H & 1) == 0 && (W & 1) == 0 && C1 > 0 && (C1 & 3) == 0 && C2 >= 0 &&
                        (C2 & 3) == 0 && (C2 == 0 || skip), "upcat_fwd: bad arguments");
    upcat_fwd_kernel<<<grid_for((long long)B * H * W * ((C1 + C2) / 4)), NT, 0, ST>>>(lo, skip, B, H, W, C1, C2, out);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_fold_bwd(const float* dpad, int B, int H, int W, int C1, int C2, int upsample, float* d_lo,
                              const float* lo_act, int act, int accumulate, float* d_skip, void* stream) {
    SCSFM_CHECK_ARG(dpad && d_lo && B > 0 && H >= 2 && W >= 2 && C1 > 0 && (C1 & 3) == 0 && C2 >= 0 && (C2 & 3) == 0, "fold_bwd: bad arguments");
    SCSFM_CHECK_ARG((act & 0xff) == ACT_NONE || lo_act, "fold_bwd: activation gradient needs the activation output");
    if (!upsample) {
        SCSFM_CHECK_ARG(C2 == 0, "fold_bwd: concat without upsample is not used by the decoder");
        fold_plain_kernel<<<grid_for((long long)B * H * W * (C1 / 4)), NT, 0, ST>>>(dpad, B, H, W, C1, d_lo, lo_act, act, accumulate);
        SCSFM_CHECK_LAUNCH();
        return SCSFM_OK;
    }
    SCSFM_CHECK_ARG((H & 1) == 0 && (W & 1) == 0, "fold_bwd: bad upsample geometry");
    fold_up_lo_kernel<<<grid_for((long long)B * (H / 2) * (W / 2) * (C1 / 4)), NT, 0, ST>>>(dpad, B, H, W, C1, C1 + C2, d_lo, lo_act, act);
    SCSFM_CHECK_LAUNCH();
    if (C2 > 0 && d_skip) {
        fold_up_skip_kernel<<<grid_for((long long)B * H * W * (C2 / 4)), NT, 0, ST>>>(dpad, B, H, W, C1, C2, d_skip);
        SCSFM_CHECK_LAUNCH();
    }
    return SCSFM_OK;
}

extern "C" int scsfm_act_bwd(float* d, const float* out, long long n, int act, void* stream) {
    SCSFM_CHECK_ARG(d && out && n > 0, "act_bwd: bad arguments");
    act_bwd_kernel<<<grid_for(n), NT, 0, ST>>>(d, out, n, act);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_spatial_mean_fwd(const float* x, int B, int HW, int C, float scale, float* out, void* stream) {
    SCSFM_CHECK_ARG(x && out && B > 0 && HW > 0 && C > 0, "spatial_mean_fwd: bad arguments");
    spatial_mean_fwd_kernel<<<B * C, NT, 0, ST>>>(x, HW, C, scale, out);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_spatial_mean_bwd(const float* dout, int B, int HW, int C, float scale, float* dx, void* stream) {
    SCSFM_CHECK_ARG(dout && dx && B > 0 && HW > 0 && C > 0, "spatial_mean_bwd: bad arguments");
    spatial_mean_bwd_kernel<<<grid_for((long long)B * HW * C), NT, 0, ST>>>(dout, B, HW, C, scale, dx);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_round_tf32(const float* in, float* out, long long n, void* stream) {
    SCSFM_CHECK_ARG(in && out && n > 0, "round_tf32: bad arguments");
    round_tf32_kernel<<<grid_for(n), NT, 0, ST>>>(in, out, n);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_split_tf32(const float* in, float* lo, long long n, void* stream) {
    SCSFM_CHECK_ARG(in && lo && n > 0, "split_tf32: bad arguments");
    SCSFM_CHECK_ARG(((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(lo)) & 15) == 0, "split_tf32: buffers must be 16-byte aligned");
    const long long n4 = n / 4;
    split_tf32_kernel<<<grid_for(n4 > 0 ? n4 : 1), NT, 0, ST>>>(in, lo, n4, n);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n, float lr,
                               float beta1, float beta2, float eps, float weight_decay, int step, const int* step_dev,
                               float* mirror, int mirror_operand, void* stream) {
    SCSFM_CHECK_ARG(param && grad && exp_avg && exp_avg_sq && n > 0 && (step >= 1 || step_dev), "adam_step: bad arguments");
    SCSFM_CHECK_ARG(mirror_operand == SCSFM_OPERAND_TF32 || mirror_operand == SCSFM_OPERAND_LO, "adam_step: bad mirror operand kind");
    adam_kernel<<<grid_for(n), NT, 0, ST>>>(param, grad, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps, weight_decay, step, step_dev, mirror,
                                            mirror_operand);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_adam_step_masked(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n,
                                      const unsigned char* chunk_mask, float lr, float beta1, float beta2, float eps,
                                      float weight_decay, int step, const int* step_dev, float* mirror, int mirror_operand,
                                      void* stream) {
    SCSFM_CHECK_ARG(param && grad && exp_avg && exp_avg_sq && chunk_mask && n > 0 && (step >= 1 || step_dev),
                    "adam_step_masked: bad arguments");
    SCSFM_CHECK_ARG(mirror_operand == SCSFM_OPERAND_TF32 || mirror_operand == SCSFM_OPERAND_LO, "adam_step_masked: bad mirror operand kind");
    adam_masked_kernel<<<grid_for(n), NT, 0, ST>>>(param, grad, exp_avg, exp_avg_sq, n, chunk_mask, lr, beta1, beta2, eps, weight_decay,
                                                   step, step_dev, mirror, mirror_operand);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}
