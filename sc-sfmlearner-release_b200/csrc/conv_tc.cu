// Implicit-GEMM convolution on the Hopper tensor cores (wgmma, tf32 operands, fp32 accumulation in registers).
//
//   C[M = B*Ho*Wo, N = Cout] = A[M, K = kh*kw*Cin] (im2col gather of the NHWC input) x W[N, K]^T
//
// CTA = one 64 x BN output tile, 8 warps:
//   warps 0-3  producers: gather 64 x 32-float A slices (any stride / zero or reflection padding) with 16-byte cp.async
//              into the 128B-swizzled K-major layout the wgmma descriptors expect (completion on the stage's "full"
//              mbarrier); thread 0 also issues the BN x 32 weight slice as one TMA box
//   warps 4-7  one consumer warpgroup: 4 x wgmma (M64 x BN x K8) per stage, accumulators in registers, stage released
//              on its "empty" mbarrier once the wgmma that read it have retired
//   afterwards all 8 warps are the epilogue (accumulator tile through shared memory -> bias / activation / residual
//   addend / BatchNorm partial sums -> 16B stores).
// A software gather is used instead of TMA-im2col because the same loader folds in reflection padding and the
// transposed-convolution view used for the data gradient.
//
// dgrad (stride 1) is the same kernel run on dout with flipped/transposed weights (weight_flip_kernel below);
// for reflection-padded layers it returns the gradient of the padded tensor (pad' = 2), folded afterwards.
//
// Replaces cuDNN implicit-GEMM fwd/dgrad (SURVEY.md row K1) for every layer with Cin % 4 == 0.
#include <stdlib.h>

#include "conv_tc.cuh"

namespace scsfm {

// Consumer warpgroup of the gather kernels: waits for each stage, runs its 4 wgmma (K = 8 each) into the chain accumulator
// `part`, releases the stage once those wgmma have retired, and adds `part` into `acc` (fp32, round-to-nearest) at the end
// of every chain of `chain` k-blocks.  A stage is [GBM rows][32 floats] of A followed by [BN rows][32 floats] of B.
template <int BN, int STAGES, int A_BYTES, int B_BYTES>
__device__ __forceinline__ void gather_consume(float (&acc)[BN / 2], uint8_t* sA, uint8_t* sB, uint64_t* bar_full, uint64_t* bar_empty,
                                               int total, int chain) {
    float part[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    // One chain per outer iteration.  Every wgmma sits on the same straight-line path and the only wgmma_wait<0> follows
    // the inner loop: a wait that depends on a per-iteration branch makes ptxas serialise the wgmma (C7518).
    for (int it0 = 0; it0 < total; it0 += chain) {
        const int it1 = min(total, it0 + chain);
        for (int it = it0; it < it1; ++it) {
            const int s = it % STAGES;
            tc::mbar_wait(bar_full + s, (it / STAGES) & 1);
            tc::fence_proxy_async();                     // cp.async / st.shared (generic proxy) writes -> wgmma (async proxy) reads
            const uint32_t a_addr = tc::smem_u32(sA + s * A_BYTES), b_addr = tc::smem_u32(sB + s * B_BYTES);
            tc::reg_fence(part);
            tc::wgmma_fence();
#pragma unroll
            for (int j = 0; j < TBK / 8; ++j)
                tc::wgmma_tf32<BN>(part, tc::make_desc_sw128(a_addr + j * 32), tc::make_desc_sw128(b_addr + j * 32), (it == it0 && j == 0) ? 0u : 1u);
            tc::wgmma_commit();
            tc::wgmma_wait<1>();                         // the previous stage's group has retired
            if (it > it0) tc::mbar_arrive(bar_empty + (it - 1) % STAGES);
        }
        tc::wgmma_wait<0>();
        tc::reg_fence(part);
        tc::mbar_arrive(bar_empty + (it1 - 1) % STAGES);
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
    }
}

// STACK = true (split mode, Cout <= BN / 2): the weight tile holds W in rows [0, BN/2) and lo(W) in rows [BN/2, BN), so the two
// passes lo(in) and in give all four products (accumulator columns n and BN/2 + n are added in the epilogue): 2 passes, not 3.
template <int BN, bool STACK = false>
__global__ void __launch_bounds__(FW_THREADS)
conv_fwd_tc_kernel(ScsfmConv p, TcView v, const __grid_constant__ CUtensorMap wmap, const __grid_constant__ CUtensorMap wmap_lo) {
    using Cfg = TcCfg<BN>;
    constexpr int STAGES = Cfg::STAGES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sA = smem;
    uint8_t* sB = smem + STAGES * A_STAGE_BYTES;
    uint64_t* bar_full = reinterpret_cast<uint64_t*>(smem + (Cfg::OPERANDS > Cfg::EPI ? Cfg::OPERANDS : Cfg::EPI));
    uint64_t* bar_empty = bar_full + STAGES;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int rows_per_img = v.border ? border_count(p.Ho, p.Wo) : p.Ho * p.Wo;
    const int M = p.B * rows_per_img, N = p.Cout, K = v.kh * v.kw * p.Cin;
    const int m0 = blockIdx.x * GBM, n0 = blockIdx.y * BN;
    const int KB = (K + TBK - 1) / TBK;
    // split-accumulate passes over the whole K range (ScsfmConv.in_lo / w_lo): raw x raw, lo(in) x raw(w), raw(in) x lo(w)
    const int npass = STACK ? 2 : 1 + (p.in_lo != nullptr ? 1 : 0) + (p.w_lo != nullptr ? 1 : 0);
    const int chain = npass > 1 ? CHAIN_KB : KB * npass;

    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) {
            tc::mbar_init(bar_full + s, FW_PWARPS * 32 + 1);      // cp.async arrivals (activations) + 1 expect_tx arrival (weights, TMA)
            tc::mbar_init(bar_empty + s, 128);                    // every thread of the consumer warpgroup
        }
        tc::fence_barrier_init();
        tc::tma_prefetch_desc(&wmap);
        if (p.w_lo != nullptr) tc::tma_prefetch_desc(&wmap_lo);
    }
    __syncthreads();
    float acc[BN / 2];

    if (warp < FW_PWARPS) {
        // ------------------------------------------------------------------ producers
        // Per k-block every thread fetches 4 A chunks (16 B each); the BN x 32 weight slice is one TMA box.  The loop is software-pipelined:
        // the loads of k-block kb+1 are in flight while k-block kb is written to shared memory, all addressing is
        // 32-bit offset arithmetic and out-of-image taps are handled without branches (clamped address + select).
        constexpr int ROWS = GBM / (FW_PWARPS * 4);    // A rows per thread (4): rows r0 + 16*i
        const int c = tid & 7;               // 16-byte chunk column inside the 128-byte row
        const int r0 = tid >> 3;             // 0..15
        const int cs = c ^ (r0 & 7);         // 128B swizzle: chunk ^= row % 8 (rows r0+16i share row % 8)
        const bool reflect = p.pad_mode == PADMODE_REFLECT;
        int hi0[ROWS], wi0[ROWS], rbase[ROWS];   // first-tap input coordinates and the image offset of each row
#pragma unroll
        for (int i = 0; i < ROWS; ++i) {
            const int m = m0 + r0 + 16 * i;
            if (m < M) {
                const int b = m / rows_per_img, rem = m - b * rows_per_img;
                int ho, wo;
                if (v.border) border_pixel(rem, p.Ho, p.Wo, ho, wo);
                else { ho = rem / p.Wo; wo = rem - ho * p.Wo; }
                hi0[i] = ho * v.in_stride + v.oy0;
                wi0[i] = wo * v.in_stride + v.ox0;
                rbase[i] = b * p.Hi * p.Wi * p.Cin;
            } else {
                hi0[i] = -(1 << 28);          // always out of range -> zero rows
                wi0[i] = -(1 << 28);
                rbase[i] = 0;
            }
        }
        const uint32_t a_smem = tc::smem_u32(sA) + (uint32_t)(r0 * 128 + cs * 16);
        const uint32_t b_smem = tc::smem_u32(sB);
        int kc, dy, dx, ch;
        // Asynchronous copies (cp.async / LDGSTS, 16 B, zero-fill for out-of-image taps): no register staging, so the
        // loads of all pipeline stages are in flight at once; the stage's "full" mbarrier gets this thread's arrival
        // when its copies have landed (cp.async.mbarrier.arrive.noinc).  The consumers issue fence.proxy.async after
        // waiting on the barrier to order these generic-proxy writes before the tensor core's async-proxy reads.
        // Row offsets / validity only change with the tap, i.e. every Cin/32 k-blocks: they are cached in between.
        int aoff[ROWS];
        uint32_t okm = 0;
        int it = 0;                                  // k-block counter across the passes: stage = it % STAGES
        for (int q = 0; q < npass; ++q) {
        const int ps = (q + 1) % npass;              // low-part passes first (added while the accumulators are small), raw x raw last
        const float* a_base = (ps == 1 && p.in_lo != nullptr) ? p.in_lo : p.in;
        const CUtensorMap* wm = (ps == npass - 1 && ps > 0 && p.w_lo != nullptr) ? &wmap_lo : &wmap;
        kc = 4 * c;
        {
            const int tap = kc / p.Cin;
            ch = kc - tap * p.Cin;
            dy = tap / v.kw;
            dx = tap - dy * v.kw;
        }
        int cur_dy = -1, cur_dx = -1;
        for (int kb = 0; kb < KB; ++kb, ++it) {
            const int s = it % STAGES;
            const uint32_t ph = (it / STAGES) & 1;
            if (lane == 0) tc::mbar_wait(bar_empty + s, ph ^ 1);
            __syncwarp();
            const uint32_t a_st = a_smem + (uint32_t)(s * A_STAGE_BYTES);
            if (tid == 0) {
                // weights: TMA box (32 K-columns x BN rows) straight into the 128B-swizzled stage; rows / columns beyond
                // Cout / K are zero-filled by the hardware and still count towards the expected bytes
                tc::mbar_arrive_expect_tx(bar_full + s, (uint32_t)Cfg::B_STAGE_BYTES);
                if (STACK) {
                    tc::tma_load_2d(b_smem + (uint32_t)(s * Cfg::B_STAGE_BYTES), &wmap, kb * TBK, 0, bar_full + s);
                    tc::tma_load_2d(b_smem + (uint32_t)(s * Cfg::B_STAGE_BYTES + (BN / 2) * 128), &wmap_lo, kb * TBK, 0, bar_full + s);
                } else {
                    tc::tma_load_2d(b_smem + (uint32_t)(s * Cfg::B_STAGE_BYTES), wm, kb * TBK, n0, bar_full + s);
                }
            }
            if (dy != cur_dy || dx != cur_dx) {
                cur_dy = dy; cur_dx = dx;
                okm = 0;
#pragma unroll
                for (int i = 0; i < ROWS; ++i) {
                    int hi = hi0[i] + dy, wi = wi0[i] + dx;
                    bool ok;
                    if (reflect) {
                        ok = hi0[i] > -(1 << 27);
                        hi = reflect_index(hi, p.Hi);
                        wi = reflect_index(wi, p.Wi);
                    } else {
                        ok = (unsigned)hi < (unsigned)p.Hi && (unsigned)wi < (unsigned)p.Wi;
                    }
                    aoff[i] = ok ? rbase[i] + (hi * p.Wi + wi) * p.Cin : 0;
                    okm |= (ok ? 1u : 0u) << i;
                }
            }
            const bool kok = kc < K;
#pragma unroll
            for (int i = 0; i < ROWS; ++i) {
                const bool ok = kok && ((okm >> i) & 1u);
                tc::cp_async_16(a_st + i * 2048, a_base + (ok ? aoff[i] + ch : 0), ok ? 16u : 0u);
            }
            tc::cp_async_arrive_noinc(bar_full + s);
            // advance this thread's K index by one k-block
            kc += TBK;
            ch += TBK;
            while (ch >= p.Cin) {
                ch -= p.Cin;
                if (++dx == v.kw) { dx = 0; ++dy; }
            }
        }
        }
    } else {
        // ------------------------------------------------------------------ consumer warpgroup (warps 4-7)
        gather_consume<BN, STAGES, A_STAGE_BYTES, Cfg::B_STAGE_BYTES>(acc, sA, sB, bar_full, bar_empty, KB * npass, chain);
    }

    // ------------------------------------------------------------------ epilogue (all 8 warps)
    // every wgmma has retired and every cp.async / TMA write has landed: the operand ring is free for the accumulator tile
    __syncthreads();
    constexpr int TS = BN + 1;                                // tile row stride (odd: conflict-free column reads)
    float* T = reinterpret_cast<float*>(smem);
    if (warp >= FW_PWARPS) {
        const int t = tid - FW_PWARPS * 32;
        const int r = 16 * (t >> 5) + ((t & 31) >> 2), c = 2 * (t & 3);
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
            T[r * TS + 8 * i + c] = acc[4 * i];
            T[r * TS + 8 * i + c + 1] = acc[4 * i + 1];
            T[(r + 8) * TS + 8 * i + c] = acc[4 * i + 2];
            T[(r + 8) * TS + 8 * i + c + 1] = acc[4 * i + 3];
        }
    }
    __syncthreads();
    {
        const int quarter = warp & 1, half = warp >> 1;      // 32-row group of the tile / which quarter of the column chunks
        const int m = m0 + quarter * 32 + lane;
        const bool row_ok = m < M;
        size_t out_row = (size_t)m;          // row of the output / addend tensors
        if (row_ok && (v.out_sy != 1 || v.out_sx != 1 || v.border)) {
            const int b = m / rows_per_img, rem = m - b * rows_per_img;
            int ho, wo;
            if (v.border) border_pixel(rem, p.Ho, p.Wo, ho, wo);
            else { ho = rem / p.Wo; wo = rem - ho * p.Wo; }
            out_row = ((size_t)b * v.out_H + (ho * v.out_sy + v.out_oy)) * v.out_W + (wo * v.out_sx + v.out_ox);
        }
        float* stage = T + GBM * TS + warp * (32 * 33);
        constexpr int CREAL = STACK ? BN / 2 : BN;                // accumulator columns holding output channels
        constexpr int CW = CREAL < 32 ? CREAL : 32;
        constexpr int NCH = CREAL / CW;                           // column chunks of real output channels
        const float* trow = T + (quarter * 32 + lane) * TS;
#pragma unroll 1
        for (int cc = half; cc < NCH; cc += (FW_PWARPS + 4) / 2) {
            float r[32];
#pragma unroll
            for (int j = 0; j < CW; ++j) r[j] = trow[cc * CW + j];
            if (STACK) {                                          // + the lo(W) products in columns BN/2 further on (fp32, RN)
#pragma unroll
                for (int j = 0; j < CW; ++j) r[j] += trow[BN / 2 + cc * CW + j];
            }
            float v[32];
#pragma unroll
            for (int j = 0; j < CW; ++j) {
                const int n = n0 + cc * CW + j;
                float x = r[j];
                if (row_ok && n < N) {
                    if (p.bias) x += __ldg(p.bias + n);
                    if (p.bn_scale) x = fmaf(x, __ldg(p.bn_scale + n), __ldg(p.bn_shift + n));    // eval-mode BatchNorm
                    if (p.addend) x += __ldg(p.addend + out_row * N + n);
                    x = apply_act(x, p.act);
                    if (p.act & ROUND_TF32) x = tf32_round(x);
                } else {
                    x = 0.f;
                }
                v[j] = x;
            }
            if (row_ok) {
                float* o = p.out + out_row * N + n0 + cc * CW;
                if ((N & 3) == 0) {
#pragma unroll
                    for (int j = 0; j < CW; j += 4)
                        if (n0 + cc * CW + j < N) *reinterpret_cast<float4*>(o + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
                } else {
#pragma unroll
                    for (int j = 0; j < CW; ++j)
                        if (n0 + cc * CW + j < N) o[j] = v[j];
                }
                if (p.out_lo != nullptr) {                        // low part of the split-accumulate operand (N % 4 == 0)
                    float* ol = p.out_lo + out_row * N + n0 + cc * CW;
#pragma unroll
                    for (int j = 0; j < CW; j += 4)
                        if (n0 + cc * CW + j < N)
                            *reinterpret_cast<float4*>(ol + j) = make_float4(tf32_lo(v[j]), tf32_lo(v[j + 1]), tf32_lo(v[j + 2]), tf32_lo(v[j + 3]));
                }
            }
            if (p.bn_sums != nullptr) {
                // column sums over the warp's 32 rows through a padded smem transpose, then fp64 atomics into one of
                // SCSFM_BN_SLOTS replicas (spreads the per-address serialisation at L2)
#pragma unroll
                for (int j = 0; j < CW; ++j) stage[lane * 33 + j] = v[j];
                __syncwarp();
                if (lane < CW) {
                    // a tile may straddle BatchNorm groups (network calls batched into one launch): walk the warp's
                    // 32 rows and flush the column sums whenever the group changes
                    const int groups = p.bn_groups > 0 ? p.bn_groups : 1;
                    const int rows_per_group = (p.B / groups) * rows_per_img;
                    const int row_base = m0 + quarter * 32;
                    const int n = n0 + cc * CW + lane;
                    int g_cur = row_base / rows_per_group;
                    int next_edge = (g_cur + 1) * rows_per_group - row_base;      // first row index of the next group
                    // fp64 accumulation: var = E[x^2] - mean^2 cancels catastrophically when |mean| >> std, so the
                    // partial sums must not carry fp32 rounding (a handful of DFMA per output value: negligible here)
                    double s1 = 0.0, s2 = 0.0;
                    for (int rr = 0; rr <= 32; ++rr) {
                        if (rr == 32 || rr == next_edge) {
                            if (n < N && g_cur < groups && (s1 != 0.0 || s2 != 0.0)) {
                                double* d = p.bn_sums + (((size_t)(blockIdx.x % SCSFM_BN_SLOTS) * groups + g_cur) * N + n) * 2;
                                atomicAdd(d, s1);
                                atomicAdd(d + 1, s2);
                            }
                            if (rr == 32) break;
                            s1 = 0.0; s2 = 0.0;
                            ++g_cur;
                            next_edge += rows_per_group;
                        }
                        const double t = (double)stage[rr * 33 + lane];
                        s1 += t;
                        s2 += t * t;
                    }
                }
                __syncwarp();
            }
        }
    }
}

// w [Co][kh][kw][Ci] -> wt [Ci][jh][jw][Co] with wt[c][jy][jx][o] = w[o][dy_max - step*jy][dx_max - step*jx][c]:
// the (TF32-rounded) weights of the transposed conv.  step 1, d*_max = k-1: the full flipped kernel (stride-1 dgrad);
// step 2: the taps of one output-parity class of a stride-2 dgrad.
__global__ void weight_flip_kernel(const float* __restrict__ w, int Co, int kh, int kw, int Ci, int jh, int jw, int dy_max,
                                   int dx_max, int step, float* __restrict__ wt, int operand) {
    const long long total = (long long)Co * jh * jw * Ci;
    for (long long i = blockIdx.x * 256LL + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
        const int o = (int)(i % Co);
        long long t2 = i / Co;
        const int jx = (int)(t2 % jw); t2 /= jw;
        const int jy = (int)(t2 % jh);
        const int c = (int)(t2 / jh);
        const int dy = dy_max - step * jy, dx = dx_max - step * jx;
        wt[i] = tc_operand(__ldg(w + (((size_t)o * kh + dy) * kw + dx) * Ci + c), operand);
    }
}


// ---------------------------------------------------------------------------------------------------------
// weight gradient on the tensor cores:  dW^T[(tap,c), o] += sum_pix  in[pix (+) tap, c] * dout[pix, o]
//   GEMM  M = kh*kw*Cin (gathered input),  N = Cout (dout),  K = B*Ho*Wo pixels, split over gridDim.z; partial tiles are
//   added into dw with fp32 atomics.
// Both tensors are channel-contiguous ("MN-major" for this GEMM), but wgmma takes 32-bit operands only K-major.  So the
// producers load 16-byte channel vectors into registers and store them transposed into the 128B-swizzled K-major stage
// ([row = (tap,c) or o][32 pixels]); lane = pixel, so every scalar store of a warp hits 32 different banks.
// ---------------------------------------------------------------------------------------------------------
template <int BN>
struct WgCfg {
    static constexpr int STAGES = 4;
    static constexpr int A_BYTES = GBM * 128;           // 64 (tap,c) rows x 32 pixels
    static constexpr int B_BYTES = BN * 128;            // BN output channels x 32 pixels
    static constexpr size_t SMEM = 1024 + (size_t)STAGES * (A_BYTES + B_BYTES) + 256;
};

// STACK = true (split mode, Cout <= BN / 2): the N-side tile holds dout in rows [0, BN/2) and lo(dout) in [BN/2, BN), so the two
// passes lo(in) and in give all four products (columns o and BN/2 + o are both added into dw[o]): 2 passes instead of 3.
// border = 1: the pixels (K) are only the 2*(Ho+Wo)-4 image-border pixels per image (border_pixel), the reflection-padded
// ring that the TMA weight-gradient kernel leaves out.
template <int BN, bool STACK = false>
__global__ void __launch_bounds__(FW_THREADS)
conv_wgrad_tc_kernel(ScsfmConv p, int pix_per_split, int border) {
    using Cfg = WgCfg<BN>;
    constexpr int STAGES = Cfg::STAGES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sA = smem;
    uint8_t* sB = smem + STAGES * Cfg::A_BYTES;
    uint64_t* bar_full = reinterpret_cast<uint64_t*>(sB + STAGES * Cfg::B_BYTES);
    uint64_t* bar_empty = bar_full + STAGES;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int HWo = border ? border_count(p.Ho, p.Wo) : p.Ho * p.Wo;
    const int Mtot = p.kh * p.kw * p.Cin, N = p.Cout, npix = p.B * HWo;
    const int m0 = blockIdx.x * GBM, n0 = blockIdx.y * BN;
    const int pix_begin = blockIdx.z * pix_per_split, pix_end = min(npix, pix_begin + pix_per_split);
    const int KB = (pix_end - pix_begin + 31) / 32;
    if (KB <= 0) return;
    // split-accumulate passes over the CTA's pixel range (ScsfmConv.in_lo / dout_lo): raw x raw, lo(in) x raw(dout), raw(in) x lo(dout)
    const int npass = STACK ? 2 : 1 + (p.in_lo != nullptr ? 1 : 0) + (p.dout_lo != nullptr ? 1 : 0);
    const int chain = npass > 1 ? CHAIN_KB : KB * npass;

    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) {
            tc::mbar_init(bar_full + s, FW_PWARPS * 32);
            tc::mbar_init(bar_empty + s, 128);
        }
        tc::fence_barrier_init();
    }
    __syncthreads();

    if (warp < FW_PWARPS) {
        // ------------------------------------------------------------------ producers
        // Thread (warp w, lane l) handles pixel l of every 32-pixel k-block: A channel chunks w, w + 4, ... (4 (tap,c) rows
        // each) and B chunks the same way.  The pixel's coordinates advance by 32 per k-block.
        constexpr int A_IT = GBM / 4 / FW_PWARPS;            // A chunks per thread and k-block (4)
        constexpr int B_IT = BN / 4 / FW_PWARPS;             // B chunks per thread and k-block (1 .. 8)
        const bool reflect = p.pad_mode == PADMODE_REFLECT;
        int a_dy[A_IT], a_dx[A_IT], a_ch[A_IT];
#pragma unroll
        for (int i = 0; i < A_IT; ++i) {
            const int mm = m0 + 4 * (warp + FW_PWARPS * i);
            a_ch[i] = -1;                                    // -1: rows beyond M
            a_dy[i] = a_dx[i] = 0;
            if (mm < Mtot) {
                const int tap = mm / p.Cin;
                a_ch[i] = mm - tap * p.Cin;
                a_dy[i] = tap / p.kw - p.pad;
                a_dx[i] = tap - (tap / p.kw) * p.kw - p.pad;
            }
        }
        const uint32_t a_smem = tc::smem_u32(sA), b_smem = tc::smem_u32(sB);
        // Software-pipelined: the global loads of k-block it+1 are in flight while this thread waits for k-block it's stage
        // and stores it transposed.  (fq, fpx, fb, fho, fwo) is the position of the next k-block to fetch, across the
        // passes (low-part passes first: added while the sums are small; raw x raw last).
        int fq = 0, fkb = 0, fpx = pix_begin + lane, fb, fho, fwo, frow;   // frow: dout row of the pixel
        auto locate = [&]() {
            const int rem = fpx - (fb = fpx / HWo) * HWo;
            if (border) {
                border_pixel(rem, p.Ho, p.Wo, fho, fwo);
                frow = (fb * p.Ho + fho) * p.Wo + fwo;
            } else {
                fho = rem / p.Wo;
                fwo = rem - fho * p.Wo;
                frow = fpx;
            }
        };
        locate();
        auto fetch = [&](float4 (&va)[A_IT], float4 (&vb)[B_IT]) {
            const int ps = (fq + 1) % npass;
            const float* a_base = (ps == 1 && p.in_lo != nullptr) ? p.in_lo : p.in;
            const float* b_main = STACK ? p.dout : ((ps == npass - 1 && ps > 0 && p.dout_lo != nullptr) ? p.dout_lo : p.dout);
            const bool px_ok = fpx < pix_end;
#pragma unroll
            for (int i = 0; i < A_IT; ++i) {
                int hi = fho * p.stride + a_dy[i], wi = fwo * p.stride + a_dx[i];
                bool ok = px_ok && a_ch[i] >= 0;
                if (reflect) { hi = reflect_index(hi, p.Hi); wi = reflect_index(wi, p.Wi); }
                else ok = ok && (unsigned)hi < (unsigned)p.Hi && (unsigned)wi < (unsigned)p.Wi;
                va[i] = ok ? __ldg(reinterpret_cast<const float4*>(a_base + ((size_t)(fb * p.Hi + hi) * p.Wi + wi) * p.Cin + a_ch[i]))
                           : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int i = 0; i < B_IT; ++i) {
                const int col = 4 * (warp + FW_PWARPS * i);      // first tile row (output channel column) of this chunk
                const bool lo_half = STACK && col >= BN / 2;     // stacked: rows >= BN/2 read lo(dout) at channel col - BN/2
                const int nn = STACK ? col - (lo_half ? BN / 2 : 0) : n0 + col;
                const bool ok = px_ok && nn < N;
                const float* bb = lo_half ? p.dout_lo : b_main;
                vb[i] = ok ? __ldg(reinterpret_cast<const float4*>(bb + (size_t)frow * N + nn)) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
            // advance to the next k-block: 32 pixels further, or the first k-block of the next pass
            if (++fkb == KB) {
                fkb = 0;
                ++fq;
                fpx = pix_begin + lane;
                locate();
            } else if (border) {
                fpx += 32;
                locate();
            } else {
                fpx += 32;
                frow = fpx;
                fwo += 32;
                while (fwo >= p.Wo) { fwo -= p.Wo; if (++fho == p.Ho) { fho = 0; ++fb; } }
            }
        };
        const int total = KB * npass;
        float4 va[A_IT], vb[B_IT];
        fetch(va, vb);
        for (int it = 0; it < total; ++it) {
            float4 na[A_IT], nb[B_IT];
            if (it + 1 < total) fetch(na, nb);
            const int s = it % STAGES;
            tc::mbar_wait(bar_empty + s, ((it / STAGES) & 1) ^ 1);
            const uint32_t a_st = a_smem + (uint32_t)(s * Cfg::A_BYTES), b_st = b_smem + (uint32_t)(s * Cfg::B_BYTES);
#pragma unroll
            for (int i = 0; i < A_IT; ++i) {
                const int r = 4 * (warp + FW_PWARPS * i);
                tc::st_shared_f32(a_st + tc::sw128_offset(r, lane), va[i].x);
                tc::st_shared_f32(a_st + tc::sw128_offset(r + 1, lane), va[i].y);
                tc::st_shared_f32(a_st + tc::sw128_offset(r + 2, lane), va[i].z);
                tc::st_shared_f32(a_st + tc::sw128_offset(r + 3, lane), va[i].w);
            }
#pragma unroll
            for (int i = 0; i < B_IT; ++i) {
                const int r = 4 * (warp + FW_PWARPS * i);
                tc::st_shared_f32(b_st + tc::sw128_offset(r, lane), vb[i].x);
                tc::st_shared_f32(b_st + tc::sw128_offset(r + 1, lane), vb[i].y);
                tc::st_shared_f32(b_st + tc::sw128_offset(r + 2, lane), vb[i].z);
                tc::st_shared_f32(b_st + tc::sw128_offset(r + 3, lane), vb[i].w);
            }
            tc::fence_proxy_async();                         // generic-proxy stores -> wgmma (async proxy) reads
            tc::mbar_arrive(bar_full + s);
#pragma unroll
            for (int i = 0; i < A_IT; ++i) va[i] = na[i];
#pragma unroll
            for (int i = 0; i < B_IT; ++i) vb[i] = nb[i];
        }
    } else {
        // ------------------------------------------------------------------ consumer warpgroup: dw[o][mm] += D[mm][o]
        float acc[BN / 2];
        gather_consume<BN, STAGES, Cfg::A_BYTES, Cfg::B_BYTES>(acc, sA, sB, bar_full, bar_empty, KB * npass, chain);
        const int t = tid - FW_PWARPS * 32;
        const int r = m0 + 16 * (t >> 5) + ((t & 31) >> 2), c = 2 * (t & 3);
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int row = r + 8 * (e >> 1), col = 8 * i + c + (e & 1);
                const int o = STACK ? (col >= BN / 2 ? col - BN / 2 : col) : n0 + col;
                if (row < Mtot && o < N) red_add(p.dw + (size_t)o * Mtot + row, acc[4 * i + e]);
            }
        }
    }
}

CUresult encode_tiled(CUtensorMap* map, CUtensorMapDataType dtype, cuuint32_t rank, void* gaddr, const cuuint64_t* gdim,
                      const cuuint64_t* gstride, const cuuint32_t* box, const cuuint32_t* estr, CUtensorMapInterleave il,
                      CUtensorMapSwizzle sw, CUtensorMapL2promotion l2, CUtensorMapFloatOOBfill oob) {
    using Fn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                            const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static const Fn fn = []() -> Fn {                   // C++11 thread-safe one-time initialisation
        void* sym = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) != cudaSuccess || sym == nullptr ||
            qres != cudaDriverEntryPointSuccess)
            return nullptr;
        return reinterpret_cast<Fn>(sym);
    }();
    if (fn == nullptr) return CUDA_ERROR_NOT_FOUND;
    return fn(map, dtype, rank, gaddr, gdim, gstride, box, estr, il, sw, l2, oob);
}

int encode_nhwc(CUtensorMap* map, const float* base, int B, int rows, int cols, int C, long long col_step, long long row_step,
                long long img_step, int box_c, int box_w, int box_h, CUtensorMapSwizzle sw) {
    const cuuint64_t gdim[4] = {(cuuint64_t)C, (cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)B};
    const cuuint64_t gstride[3] = {(cuuint64_t)col_step * 4, (cuuint64_t)row_step * 4, (cuuint64_t)img_step * 4};
    const cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    const CUresult r = encode_tiled(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(base), gdim, gstride, box, estr,
                                    CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled(activations %d x %d x %d x %d view) failed with CUresult %d", B, rows, cols, C, (int)r);
        return SCSFM_ERR_CUDA;
    }
    return SCSFM_OK;
}

int encode_weights(CUtensorMap* map, const float* w, int Cout, int K, int box_rows) {
    const cuuint64_t gdim[2] = {(cuuint64_t)K, (cuuint64_t)Cout};
    const cuuint64_t gstride[1] = {(cuuint64_t)K * sizeof(float)};
    const cuuint32_t box[2] = {(cuuint32_t)TBK, (cuuint32_t)box_rows};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = encode_tiled(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(w), gdim, gstride, box, estr,
                                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled(weights %d x %d) failed with CUresult %d", Cout, K, (int)r);
        return SCSFM_ERR_CUDA;
    }
    return SCSFM_OK;
}

int sm_count() {
    static const int n = [] {                           // C++11 thread-safe one-time initialisation
        int dev = 0, v = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) return 132;
        return v;
    }();
    return n;
}

int launch_bias_grad(const float* dout, int rows, int C, float* dbias, cudaStream_t st);   // conv_simt.cu

template <int BN, bool STACK = false>
static int launch_wgrad_tc(const ScsfmConv& p, int border, cudaStream_t st) {
    using Cfg = WgCfg<BN>;
    static const cudaError_t attr_rc = cudaFuncSetAttribute(conv_wgrad_tc_kernel<BN, STACK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM);
    SCSFM_CHECK_CUDA(attr_rc);
    const int Mtot = p.kh * p.kw * p.Cin, npix = p.B * (border ? border_count(p.Ho, p.Wo) : p.Ho * p.Wo);
    const int mt = (Mtot + GBM - 1) / GBM, nt = STACK ? 1 : (p.Cout + BN - 1) / BN;
    // Three CTAs' worth of pixel splits per SM although only one BN = 128 CTA is resident at a time (171-174 registers x
    // 256 threads): the extra split-K CTAs queue behind it and fill the SM as the earlier ones drain.  Measured on H100
    // over the layers of tools/conv_layers.py with every tf32x3 weight gradient on this kernel: 20.0 ms with this count,
    // 28.6 ms with exactly one resident wave.
    int splits = (sm_count() * 3 + mt * nt - 1) / (mt * nt);
    const int max_splits = (npix + 1023) / 1024;             // at least 32 k-blocks per CTA
    if (splits > max_splits) splits = max_splits;
    if (splits < 1) splits = 1;
    const int pps = ((npix + splits - 1) / splits + 31) / 32 * 32;
    dim3 grid(mt, nt, (npix + pps - 1) / pps);
    conv_wgrad_tc_kernel<BN, STACK><<<grid, FW_THREADS, Cfg::SMEM, st>>>(p, pps, border);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

static TcView plain_view(const ScsfmConv& p) {
    return TcView{p.kh, p.kw, -p.pad, -p.pad, p.stride, 1, 0, 1, 0, p.Ho, p.Wo};
}

template <int BN, bool STACK = false>
static int launch_fwd_tc(const ScsfmConv& p, const TcView& v, cudaStream_t st) {
    using Cfg = TcCfg<BN>;
    static const cudaError_t attr_rc = cudaFuncSetAttribute(conv_fwd_tc_kernel<BN, STACK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM);
    SCSFM_CHECK_CUDA(attr_rc);
    const int M = p.B * (v.border ? border_count(p.Ho, p.Wo) : p.Ho * p.Wo);
    // the kernel reads wmap_lo only when p.w_lo is set (STACK is chosen for split mode only)
    const int K = v.kh * v.kw * p.Cin, rows = STACK ? BN / 2 : BN;
    CUtensorMap wmap, wmap_lo = {};
    if (int rc = encode_weights(&wmap, p.w, p.Cout, K, rows)) return rc;
    if (int rc = p.w_lo != nullptr ? encode_weights(&wmap_lo, p.w_lo, p.Cout, K, rows) : SCSFM_OK) return rc;
    dim3 grid((M + GBM - 1) / GBM, STACK ? 1 : (p.Cout + BN - 1) / BN);
    conv_fwd_tc_kernel<BN, STACK><<<grid, FW_THREADS, Cfg::SMEM, st>>>(p, v, wmap, wmap_lo);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

}  // namespace scsfm

using namespace scsfm;

// Weight-gradient kernel for *p: 1 the gather kernel, 2 the TMA kernel (and the gather kernel on the ring of a reflection-
// padded layer), 3 the thin-layer fp32 kernel.  SCSFM_TUNE_WGRAD: 0 auto, 1 the gather kernel, 2 the TMA kernel (the
// gather kernel where it does not apply), 3 the thin-layer kernel.
static int wgrad_kernel(const ScsfmConv& p) {
    const bool split = p.split || (p.in_lo != nullptr && p.dout_lo != nullptr);
    int kernel = (int)((p.tune >> 12) & 3u);
    if (kernel == 3 && !conv_wgrad_thin_eligible(p)) kernel = 0;
    // the 16-output-channel decoder layers in split mode read four tensors and use 16 of the MMA's columns: the fp32 FMA
    // kernel reads two and is exact per product (conv_wgrad_thin.cu)
    if (kernel == 0 && (split || p.in_lo != nullptr || p.dout_lo != nullptr) && conv_wgrad_thin_eligible(p)) kernel = 3;
    if ((kernel == 0 || kernel == 2) && conv_wgrad_tma_eligible(p) && (split || (p.in_lo == nullptr && p.dout_lo == nullptr))) return 2;
    return kernel == 3 ? 3 : 1;
}

// split mode: does the kernel the dispatcher picks for *p read the low parts of its activation operands?  The stem forward
// kernel and the TMA / thin weight-gradient kernels compute or do not need them; the gather kernels and the TMA forward
// read them, as does the gather pass over the ring of a reflection-padded weight gradient.
static bool conv_reads_lo(const ScsfmConv& p, int pass) {
    if (pass == SCSFM_PASS_FWD) return !conv_stem_eligible(p);
    if (pass == SCSFM_PASS_WGRAD) {
        ScsfmConv q = p;
        q.split = 1;
        const int k = wgrad_kernel(q);
        return k == 1 || (k == 2 && p.pad_mode == PADMODE_REFLECT);
    }
    return true;
}

extern "C" int scsfm_conv_reads_lo(const ScsfmConv* p, int pass) {
    SCSFM_CHECK_ARG(p != nullptr && pass >= SCSFM_PASS_FWD && pass <= SCSFM_PASS_WGRAD, "conv_reads_lo: bad arguments");
    SCSFM_CHECK_ARG(p->B > 0 && p->Hi > 0 && p->Wi > 0 && p->Cin > 0 && p->Cout > 0 && p->kh > 0 && p->kw > 0 && p->stride > 0 && p->pad >= 0,
                    "conv_reads_lo: bad geometry");
    return conv_reads_lo(*p, pass) ? 1 : 0;
}

// cp.async gather kernel: any stride / padding mode / border-only rows
static int tc_dispatch_gather(const ScsfmConv& p, const TcView& v, cudaStream_t st) {
    const int N = p.Cout;
    if (p.in_lo != nullptr && p.w_lo != nullptr && N <= 64) {       // split mode, thin: W / lo(W) stacked on the N side
        if (N <= 16) return launch_fwd_tc<32, true>(p, v, st);
        if (N <= 32) return launch_fwd_tc<64, true>(p, v, st);
        return launch_fwd_tc<128, true>(p, v, st);
    }
    if (N <= 16) return launch_fwd_tc<16>(p, v, st);
    if (N <= 32 || N % 64 != 0) return launch_fwd_tc<32>(p, v, st);
    if (N <= 64 || N % 128 != 0) return launch_fwd_tc<64>(p, v, st);
    // prefer more CTAs when the M extent is small (deep layers at 8x26 / 16x52)
    const int M = p.B * (v.border ? border_count(p.Ho, p.Wo) : p.Ho * p.Wo);
    if (((M + GBM - 1) / GBM) * (N / 128) < sm_count()) return launch_fwd_tc<64>(p, v, st);
    return launch_fwd_tc<128>(p, v, st);
}

// Stride-2 forwards the gather kernel runs faster than the TMA kernel (tools/conv_layers.py --only s2 --tune mt=1
// --compare no_tma=1, H100): in split mode, Cin >= 512 into output planes of at most 8 x 26 pixels (the ResNet-50 layer4
// 3x3 512 -> 512 and 1x1 1024 -> 2048).  Two 128-pixel tiles per image leave most SMs idle through a long K loop, where
// the gather kernel's 64-pixel tiles give twice the CTAs.  The ResNet-18 layer4 (Cin 256) and every tf32 shape are at
// least as fast on the TMA kernel.
static bool s2_prefers_gather(const ScsfmConv& p, const TcView& v) {
    return v.in_stride == 2 && p.in_lo != nullptr && p.Cin >= 512 && p.Ho * p.Wo <= 8 * 26 && !conv_tma_forced(p);
}

static int tc_dispatch(const ScsfmConv& p, const TcView& v, cudaStream_t st) {
    if (conv_stem_eligible(p)) return launch_conv_stem_fwd(p, st);      // (a data gradient's sub-convolutions have stride 1)
    if (p.pad_mode == PADMODE_ZERO && conv_tma_eligible(p, v) && !s2_prefers_gather(p, v)) return launch_conv_tma(p, v, st);
    if (p.pad_mode == PADMODE_REFLECT && v.in_stride == 1 && p.bn_sums == nullptr && p.Ho >= 3 && p.Wo >= 3 &&
        (p.Ho * p.Wo >= 64 * 208 || conv_tma_forced(p)) && conv_tma_eligible(p, v)) {
        // reflection padding only changes the outermost ring of output pixels: run the TMA kernel with zero padding
        // (interior exact), then recompute the 2*(Ho+Wo)-4 border pixels per image with the reflecting gather kernel.
        // Measured on H100 (tools/conv_layers.py --only dec --compare mt=1, tf32x3): pays off from 64x208 upwards; below
        // that the ring is too large a share of the image and the gather kernel alone is as fast or faster (8x26:
        // x0.63, 16x52: x0.95; at 32x104 the split was x1.14, not yet taken: tf32 unmeasured).
        ScsfmConv q = p;
        q.pad_mode = PADMODE_ZERO;
        if (int rc = launch_conv_tma(q, v, st)) return rc;
        TcView bv = v;
        bv.border = 1;
        return tc_dispatch_gather(p, bv, st);
    }
    return tc_dispatch_gather(p, v, st);
}

static int check_tc(const ScsfmConv* p, const char* who) {
    SCSFM_CHECK_ARG(p != nullptr && p->in && p->w && p->out, "%s: null tensor", who);
    SCSFM_CHECK_ARG(p->B > 0 && p->Hi > 0 && p->Wi > 0 && p->Cin > 0 && p->Cout > 0 && p->kh > 0 && p->kw > 0 && p->stride > 0 && p->pad >= 0,
                    "%s: bad geometry", who);
    SCSFM_CHECK_ARG((p->Cin & 3) == 0, "%s: the tensor-core kernel needs Cin %% 4 == 0 (got %d); use the CUDA-core kernel", who, p->Cin);
    SCSFM_CHECK_ARG(p->Ho == (p->Hi + 2 * p->pad - p->kh) / p->stride + 1 && p->Wo == (p->Wi + 2 * p->pad - p->kw) / p->stride + 1,
                    "%s: output size does not match geometry", who);
    SCSFM_CHECK_ARG(p->pad_mode != PADMODE_REFLECT || p->pad == 1, "%s: reflect pad must be 1", who);
    if (p->bn_sums) {
        const int g = p->bn_groups > 0 ? p->bn_groups : 1;
        SCSFM_CHECK_ARG(p->B % g == 0, "%s: batch not divisible by the number of BatchNorm groups", who);
    }
    SCSFM_CHECK_ARG((p->bn_scale == nullptr) == (p->bn_shift == nullptr), "%s: bn_scale and bn_shift go together", who);
    SCSFM_CHECK_ARG(p->bn_scale == nullptr || (p->bias == nullptr && p->bn_sums == nullptr),
                    "%s: the eval-mode BatchNorm epilogue excludes bias and bn_sums", who);
    SCSFM_CHECK_ARG(p->out_lo == nullptr || ((p->Cout & 3) == 0 && (reinterpret_cast<uintptr_t>(p->out_lo) & 15) == 0),
                    "%s: out_lo needs Cout %% 4 == 0 and 16-byte alignment", who);
    SCSFM_CHECK_ARG(((reinterpret_cast<uintptr_t>(p->bn_scale) | reinterpret_cast<uintptr_t>(p->bn_shift)) & 7) == 0,
                    "%s: bn_scale / bn_shift must be 8-byte aligned", who);
    return SCSFM_OK;
}

extern "C" int scsfm_conv2d_fwd_tc(const ScsfmConv* p, void* stream) {
    if (int rc = check_tc(p, "conv2d_fwd_tc")) return rc;
    if (p->split) {
        SCSFM_CHECK_ARG(p->w_lo != nullptr, "conv2d_fwd_tc: split mode needs w_lo");
        SCSFM_CHECK_ARG(p->in_lo != nullptr || !conv_reads_lo(*p, SCSFM_PASS_FWD),
                        "conv2d_fwd_tc: the kernel chosen for this call reads in_lo, which was not passed (scsfm_conv_reads_lo)");
    }
    return tc_dispatch(*p, plain_view(*p), (cudaStream_t)stream);
}

extern "C" int scsfm_weight_flip(const float* w, int Cout, int kh, int kw, int Cin, float* wt, int operand, void* stream) {
    SCSFM_CHECK_ARG(w && wt && Cout > 0 && kh > 0 && kw > 0 && Cin > 0 && operand >= 0 && operand <= 2, "weight_flip: bad arguments");
    const long long total = (long long)Cout * kh * kw * Cin;
    int grid = (int)((total + 255) / 256);
    if (grid > sm_count() * 16) grid = sm_count() * 16;
    weight_flip_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(w, Cout, kh, kw, Cin, kh, kw, kh - 1, kw - 1, 1, wt, operand);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

// All flips of a network in ONE launch.  table = n rows of 12 int64: {src pointer, dst pointer, Co, kh, kw, Ci, jh, jw,
// dy_max, dx_max, step, first block}; a row is one weight_flip_kernel job (a stride-2 layer contributes one row per parity
// class with taps) and owns blocks [first block, next row's first block); row n is a sentinel holding the total.
// Each block transposes one 32 (Cout) x 32 (Cin) tile of one tap through shared memory: reads coalesced along Cin, writes
// coalesced along Cout.  A row owns ceil(Co/32) * ceil(Ci/32) * jh * jw blocks.
__global__ void __launch_bounds__(256)
weight_flip_batched_kernel(const long long* __restrict__ table, int n) {
    __shared__ int s_row;
    __shared__ float tile[32][33];
    if (threadIdx.x == 0) {
        int lo = 0, hi = n;                       // last row with first block <= blockIdx.x
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (table[mid * 12 + 11] <= (long long)blockIdx.x) lo = mid; else hi = mid;
        }
        s_row = lo;
    }
    __syncthreads();
    const long long* e = table + s_row * 12;
    const float* w = reinterpret_cast<const float*>(e[0]);
    float* wt = reinterpret_cast<float*>(e[1]);
    const int Co = (int)e[2], kh = (int)e[3], kw = (int)e[4], Ci = (int)e[5], jh = (int)e[6], jw = (int)e[7];
    const int dy_max = (int)e[8], dx_max = (int)e[9], step = (int)(e[10] & 0xff), operand = (int)(e[10] >> 8);
    const int tco = (Co + 31) >> 5, tci = (Ci + 31) >> 5;
    int t = (int)((long long)blockIdx.x - e[11]);
    const int to = t % tco; t /= tco;
    const int tc = t % tci; t /= tci;
    const int jy = t / jw, jx = t - jy * jw;
    const int dy = dy_max - step * jy, dx = dx_max - step * jx;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int o = to * 32 + ty + 8 * k, c = tc * 32 + tx;
        if (o < Co && c < Ci) tile[ty + 8 * k][tx] = tc_operand(__ldg(w + (((size_t)o * kh + dy) * kw + dx) * Ci + c), operand);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int c = tc * 32 + ty + 8 * k, o = to * 32 + tx;
        if (c < Ci && o < Co) wt[(((size_t)c * jh + jy) * jw + jx) * Co + o] = tile[tx][ty + 8 * k];
    }
}

extern "C" int scsfm_weight_flip_batched(const long long* table, int n_rows, int total_blocks, void* stream) {
    SCSFM_CHECK_ARG(table != nullptr && n_rows > 0 && total_blocks > 0, "weight_flip_batched: bad arguments");
    weight_flip_batched_kernel<<<total_blocks, 256, 0, (cudaStream_t)stream>>>(table, n_rows);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

// Output-parity class (py, px) of a stride-2 data gradient: the kernel rows dy_max, dy_max - 2, ... (jh of them) and
// columns dx_max, dx_max - 2, ... (jw) reach it; jh or jw = 0: no tap does.
struct S2Class {
    int jh, jw, dy_max, dx_max;
};
static S2Class s2_class(int kh, int kw, int pad, int py, int px) {
    S2Class k{0, 0, kh - 1, kw - 1};
    while (k.dy_max >= 0 && ((py + pad - k.dy_max) & 1)) --k.dy_max;
    while (k.dx_max >= 0 && ((px + pad - k.dx_max) & 1)) --k.dx_max;
    k.jh = k.dy_max < 0 ? 0 : k.dy_max / 2 + 1;
    k.jw = k.dx_max < 0 ? 0 : k.dx_max / 2 + 1;
    return k;
}

// Stride-2 data gradient: wt4 receives the four parity-class weight sets back to back (class order (py,px) =
// (0,0),(0,1),(1,0),(1,1)); total size = Cin*kh*kw*Cout floats, the same as the full flipped kernel.
extern "C" int scsfm_weight_flip_s2(const float* w, int Cout, int kh, int kw, int Cin, int pad, float* wt4, int operand, void* stream) {
    SCSFM_CHECK_ARG(w && wt4 && Cout > 0 && kh > 0 && kw > 0 && Cin > 0 && pad >= 0 && operand >= 0 && operand <= 2, "weight_flip_s2: bad arguments");
    size_t off = 0;
    for (int py = 0; py < 2; ++py)
        for (int px = 0; px < 2; ++px) {
            const S2Class k = s2_class(kh, kw, pad, py, px);
            const long long total = (long long)Cout * k.jh * k.jw * Cin;
            if (total > 0) {
                int grid = (int)((total + 255) / 256);
                if (grid > sm_count() * 16) grid = sm_count() * 16;
                weight_flip_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(w, Cout, kh, kw, Cin, k.jh, k.jw, k.dy_max, k.dx_max, 2, wt4 + off,
                                                                           operand);
                SCSFM_CHECK_LAUNCH();
            }
            off += (size_t)total;
        }
    return SCSFM_OK;
}

// stride-1 data gradient = forward kernel on dout with the flipped weights `wt` ([Cin][kh][kw][Cout], from
// scsfm_weight_flip) passed in p->w; p->din [B,Hi,Wi,Cin] (+ p->addend).
extern "C" int scsfm_conv2d_dgrad_tc(const ScsfmConv* p, void* stream) {
    SCSFM_CHECK_ARG(p != nullptr && p->dout && p->w && p->din, "conv2d_dgrad_tc: null tensor");
    SCSFM_CHECK_ARG(p->stride == 1 || p->stride == 2, "conv2d_dgrad_tc: stride must be 1 or 2");
    SCSFM_CHECK_ARG(!p->split || (p->dout_lo != nullptr && p->w_lo != nullptr), "conv2d_dgrad_tc: split mode needs dout_lo and w_lo");
    SCSFM_CHECK_ARG(p->kh == p->kw && p->kh - 1 - p->pad >= 0, "conv2d_dgrad_tc: square kernels only");
    cudaStream_t st = (cudaStream_t)stream;
    ScsfmConv q = *p;
    q.in = p->dout; q.in_lo = p->dout_lo; q.out = p->din; q.bias = nullptr; q.bn_sums = nullptr; q.act = SCSFM_ACT_NONE;
    q.bn_scale = nullptr; q.bn_shift = nullptr; q.out_lo = nullptr;
    q.dout_lo = nullptr;                       // (w_lo: the flipped low-part weights, laid out like w)
    q.Hi = p->Ho; q.Wi = p->Wo; q.Cin = p->Cout;
    q.Cout = p->Cin; q.pad_mode = SCSFM_PADMODE_ZERO;
    if (p->stride == 1) {
        q.Ho = p->Hi; q.Wo = p->Wi;
        q.pad = p->kh - 1 - p->pad;
        if (int rc = check_tc(&q, "conv2d_dgrad_tc")) return rc;
        return tc_dispatch(q, plain_view(q), st);
    }
    // stride 2: p->w holds the four parity-class weight sets of scsfm_weight_flip_s2
    SCSFM_CHECK_ARG((q.Cin & 3) == 0, "conv2d_dgrad_tc: needs Cout %% 4 == 0");
    q.stride = 1;
    bool covered_all = true;
    for (int py = 0; py < 2; ++py)
        for (int px = 0; px < 2; ++px) {
            const S2Class k = s2_class(p->kh, p->kw, p->pad, py, px);
            const int Hs = (p->Hi - py + 1) / 2, Ws = (p->Wi - px + 1) / 2;
            if ((k.jh == 0 || k.jw == 0) && Hs > 0 && Ws > 0) covered_all = false;
        }
    if (!covered_all) {
        // parity classes without taps (1x1 stride 2): their gradient is the addend alone (or zero).  Enqueued before the
        // sub-convolutions, which write the other classes' pixels of din.
        const size_t bytes = (size_t)p->B * p->Hi * p->Wi * p->Cin * sizeof(float);
        if (p->addend) SCSFM_CHECK_CUDA(cudaMemcpyAsync(p->din, p->addend, bytes, cudaMemcpyDeviceToDevice, st));
        else SCSFM_CHECK_CUDA(cudaMemsetAsync(p->din, 0, bytes, st));
    }
    size_t woff = 0;
    for (int py = 0; py < 2; ++py)
        for (int px = 0; px < 2; ++px) {
            const S2Class k = s2_class(p->kh, p->kw, p->pad, py, px);
            const int Hs = (p->Hi - py + 1) / 2, Ws = (p->Wi - px + 1) / 2;
            if (k.jh > 0 && k.jw > 0 && Hs > 0 && Ws > 0) {
                ScsfmConv r = q;
                r.w = p->w + woff;
                r.w_lo = p->w_lo ? p->w_lo + woff : nullptr;
                r.Ho = Hs; r.Wo = Ws; r.kh = k.jh; r.kw = k.jw;
                // input (dout) row of output hy and tap jy: hy + (py + pad - dy_max)/2 + jy
                TcView v{k.jh, k.jw, (py + p->pad - k.dy_max) / 2, (px + p->pad - k.dx_max) / 2, 1, 2, py, 2, px, p->Hi, p->Wi};
                if (int rc = tc_dispatch(r, v, st)) return rc;
            }
            woff += (size_t)p->Cout * k.jh * k.jw * p->Cin;
        }
    return SCSFM_OK;
}

// cp.async gather weight-gradient kernel: any stride / padding mode (whatever the TMA kernel does not take); border = 1:
// the image-border ring pixels only
static int wgrad_gather(const ScsfmConv& p, int border, cudaStream_t st) {
    const bool split = p.in_lo != nullptr && p.dout_lo != nullptr;
    if (split && p.Cout <= 16) return launch_wgrad_tc<32, true>(p, border, st);
    if (split && p.Cout <= 32) return launch_wgrad_tc<64, true>(p, border, st);
    if (split && p.Cout <= 64) return launch_wgrad_tc<128, true>(p, border, st);
    if (p.Cout <= 16) return launch_wgrad_tc<16>(p, border, st);
    if (p.Cout <= 32) return launch_wgrad_tc<32>(p, border, st);
    if (p.Cout <= 64) return launch_wgrad_tc<64>(p, border, st);
    return launch_wgrad_tc<128>(p, border, st);
}

// dw [Cout,kh,kw,Cin] += dout^T x gather(in); dbias += column sums of dout.  Needs Cin % 4 == 0 and Cout % 4 == 0.
extern "C" int scsfm_conv2d_wgrad_tc(const ScsfmConv* p, void* stream) {
    SCSFM_CHECK_ARG(p != nullptr && p->in && p->dout && p->dw, "conv2d_wgrad_tc: null tensor");
    SCSFM_CHECK_ARG(p->B > 0 && p->Hi > 0 && p->Wi > 0 && p->Cin > 0 && p->Cout > 0 && p->kh > 0 && p->kw > 0 && p->stride > 0 && p->pad >= 0,
                    "conv2d_wgrad_tc: bad geometry");
    SCSFM_CHECK_ARG((p->Cin & 3) == 0 && (p->Cout & 3) == 0, "conv2d_wgrad_tc: needs Cin %% 4 == 0 and Cout %% 4 == 0");
    SCSFM_CHECK_ARG(p->pad_mode != PADMODE_REFLECT || p->pad == 1, "conv2d_wgrad_tc: reflect pad must be 1");
    SCSFM_CHECK_ARG((long long)p->B * p->Ho * p->Wo < (1LL << 31), "conv2d_wgrad_tc: too many pixels");
    SCSFM_CHECK_ARG(!p->split || (p->in_lo != nullptr && p->dout_lo != nullptr) || !conv_reads_lo(*p, SCSFM_PASS_WGRAD),
                    "conv2d_wgrad_tc: the kernel chosen for this call reads in_lo and dout_lo, which were not passed (scsfm_conv_reads_lo)");
    cudaStream_t st = (cudaStream_t)stream;
    int rc;
    const int kernel = wgrad_kernel(*p);
    if (kernel == 2) {
        // reflection padding: the TMA kernel takes the interior with zero padding, the gather kernel the border ring
        if ((rc = launch_conv_wgrad_tma(*p, st))) return rc;
        rc = p->pad_mode == PADMODE_REFLECT ? wgrad_gather(*p, 1, st) : SCSFM_OK;
    } else if (kernel == 3) {
        rc = launch_conv_wgrad_thin(*p, st);
    } else {
        rc = wgrad_gather(*p, 0, st);
    }
    if (rc) return rc;
    if (p->dbias) return launch_bias_grad(p->dout, p->B * p->Ho * p->Wo, p->Cout, p->dbias, st);
    return SCSFM_OK;
}
