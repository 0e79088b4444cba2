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
// dgrad (stride 1) is the same kernel run on dout with flipped/transposed weights (weight_flip_tiles_kernel below);
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

// cp.async gather kernel: any stride / padding mode / border-only rows
static int launch_gather(const ScsfmConv& p, const TcView& v, bool stacked, cudaStream_t st) {
    const int N = p.Cout;
    if (stacked) {                                                  // split mode, thin: W / lo(W) stacked on the N side
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

// cp.async gather weight-gradient kernel: any stride / padding mode (whatever the TMA kernel does not take); border = 1:
// the image-border ring pixels only
static int launch_wgrad_gather(const ScsfmConv& p, bool stacked, int border, cudaStream_t st) {
    if (stacked) {                                                  // split mode, thin: dout / lo(dout) stacked on the N side
        if (p.Cout <= 16) return launch_wgrad_tc<32, true>(p, border, st);
        if (p.Cout <= 32) return launch_wgrad_tc<64, true>(p, border, st);
        return launch_wgrad_tc<128, true>(p, border, st);
    }
    if (p.Cout <= 16) return launch_wgrad_tc<16>(p, border, st);
    if (p.Cout <= 32) return launch_wgrad_tc<32>(p, border, st);
    if (p.Cout <= 64) return launch_wgrad_tc<64>(p, border, st);
    return launch_wgrad_tc<128>(p, border, st);
}

// Output-parity class (py, px) of a stride-2 data gradient: the kernel rows dy_max, dy_max - 2, ... (jh of them) and
// columns dx_max, dx_max - 2, ... (jw) reach it; jh or jw = 0: no tap does.  The four classes partition the taps.
struct S2Class {
    int jh, jw, dy_max, dx_max;
};
__host__ __device__ static S2Class s2_class(int kh, int kw, int pad, int py, int px) {
    S2Class k{0, 0, kh - 1, kw - 1};
    while (k.dy_max >= 0 && ((py + pad - k.dy_max) & 1)) --k.dy_max;
    while (k.dx_max >= 0 && ((px + pad - k.dx_max) & 1)) --k.dx_max;
    k.jh = k.dy_max < 0 ? 0 : k.dy_max / 2 + 1;
    k.jw = k.dx_max < 0 ? 0 : k.dx_max / 2 + 1;
    return k;
}

// The data gradient of p as forward convolutions on dout with the flipped weights (p.w / p.w_lo from scsfm_weight_flip)
// into din, part cls seen through v: at stride 1 one convolution (cls 0), at stride 2 the stride-1 sub-convolution of
// output-parity class cls = 2 py + px (its weights follow the earlier classes' in the flipped set).  r.kh * r.kw = 0: no tap
// reaches the part; r.Ho * r.Wo = 0: din has no pixel in it.
static void dgrad_part(const ScsfmConv& p, int cls, ScsfmConv& r, TcView& v) {
    r = p;
    r.in = p.dout; r.in_lo = p.dout_lo; r.out = p.din; r.bias = nullptr; r.bn_sums = nullptr; r.act = SCSFM_ACT_NONE;
    r.bn_scale = nullptr; r.bn_shift = nullptr; r.out_lo = nullptr; r.dout_lo = nullptr;     // w_lo: laid out like w
    r.Hi = p.Ho; r.Wi = p.Wo; r.Cin = p.Cout; r.Cout = p.Cin; r.pad_mode = SCSFM_PADMODE_ZERO; r.stride = 1;
    if (p.stride == 1) {
        r.Ho = cls == 0 ? p.Hi : 0; r.Wo = p.Wi; r.pad = p.kh - 1 - p.pad;
        v = plain_view(r);
        return;
    }
    const int py = cls >> 1, px = cls & 1;
    size_t woff = 0;
    for (int c = 0; c < cls; ++c) {
        const S2Class k = s2_class(p.kh, p.kw, p.pad, c >> 1, c & 1);
        woff += (size_t)p.Cout * k.jh * k.jw * p.Cin;
    }
    const S2Class k = s2_class(p.kh, p.kw, p.pad, py, px);
    r.w = p.w != nullptr ? p.w + woff : nullptr;
    r.w_lo = p.w_lo != nullptr ? p.w_lo + woff : nullptr;
    r.Ho = (p.Hi - py + 1) / 2; r.Wo = (p.Wi - px + 1) / 2; r.kh = k.jh; r.kw = k.jw;
    // input (dout) row of output hy and tap jy: hy + (py + pad - dy_max)/2 + jy
    v = TcView{k.jh, k.jw, (py + p.pad - k.dy_max) / 2, (px + p.pad - k.dx_max) / 2, 1, 2, py, 2, px, p.Hi, p.Wi};
}

// ---------------------------------------------------------------------------------------------------------
// Routing: which kernel runs a call and which operands it reads.  conv_plan is the only place these rules live; the
// entry points below validate for, and launch, what it picks.
// ---------------------------------------------------------------------------------------------------------
struct ConvPlan {
    int kernel;          // SCSFM_KERNEL_*
    unsigned reads;      // SCSFM_PLAN_* operand flags
    bool stacked;        // split mode, Cout <= 64: the gather kernel (and the ring pass) stacks W and lo(W) (weight
                         // gradient: dout and lo(dout)) on the N side of one tile, 2 passes instead of 3
};

// Stride-2 forwards the gather kernel runs faster than the TMA kernel (tools/conv_layers.py --only s2 --tune mt=1
// --compare no_tma=1, H100): in split mode, Cin >= 512 into output planes of at most 8 x 26 pixels (the ResNet-50 layer4
// 3x3 512 -> 512 and 1x1 1024 -> 2048).  Two 128-pixel tiles per image leave most SMs idle through a long K loop, where
// the gather kernel's 64-pixel tiles give twice the CTAs.  The ResNet-18 layer4 (Cin 256) and every tf32 shape are at
// least as fast on the TMA kernel.
static bool s2_prefers_gather(const ScsfmConv& p, const TcView& v) {
    return v.in_stride == 2 && p.mode == SCSFM_MODE_TF32X3 && p.Cin >= 512 && p.Ho * p.Wo <= 8 * 26 && !conv_tma_forced(p);
}

// Tensor-core forward (sub-)convolution p seen through v: the stem kernel, the TMA kernel, the TMA kernel plus the gather
// kernel over the border ring, or the gather kernel.
static ConvPlan route_tc(const ScsfmConv& p, const TcView& v) {
    const bool split = p.mode == SCSFM_MODE_TF32X3;
    ConvPlan r{SCSFM_KERNEL_GATHER, split ? SCSFM_PLAN_IN_LO | SCSFM_PLAN_W_LO : 0u, split && p.Cout <= 64};
    if (conv_stem_eligible(p)) {                    // (a data gradient's sub-convolutions have stride 1)
        r.kernel = SCSFM_KERNEL_STEM;
        r.reads &= ~(unsigned)SCSFM_PLAN_IN_LO;     // lo(in) comes from the A fragment
    } else if (p.pad_mode == PADMODE_ZERO && conv_tma_eligible(p, v) && !s2_prefers_gather(p, v)) {
        r.kernel = SCSFM_KERNEL_TMA;
    } else if (p.pad_mode == PADMODE_REFLECT && v.in_stride == 1 && p.bn_sums == nullptr && p.Ho >= 3 && p.Wo >= 3 &&
               (p.Ho * p.Wo >= 64 * 208 || conv_tma_forced(p)) && conv_tma_eligible(p, v)) {
        // reflection padding only changes the outermost ring of output pixels: run the TMA kernel with zero padding
        // (interior exact), then recompute the 2*(Ho+Wo)-4 border pixels per image with the reflecting gather kernel.
        // Measured on H100 (tools/conv_layers.py --only dec --compare mt=1, tf32x3): pays off from 64x208 upwards; below
        // that the ring is too large a share of the image and the gather kernel alone is as fast or faster (8x26:
        // x0.63, 16x52: x0.95; at 32x104 the split was x1.14, not yet taken: tf32 unmeasured).
        r.kernel = SCSFM_KERNEL_TMA_RING;
    }
    return r;
}

// The kernel that runs call p of `pass` and the operands it reads (include/scsfm.h, scsfm_conv_plan).
static ConvPlan conv_plan(const ScsfmConv& p, int pass) {
    const bool tc = p.mode != SCSFM_MODE_FP32, split = p.mode == SCSFM_MODE_TF32X3;
    const ConvPlan simt{SCSFM_KERNEL_SIMT, 0u, false};
    if (pass == SCSFM_PASS_FWD) {
        if (!tc || (p.Cin & 3) != 0 || p.Cout < 16) return simt;
        return route_tc(p, plain_view(p));
    }
    if (pass == SCSFM_PASS_DGRAD) {
        // the forward routing on dout, per part (dgrad_part); reported: the part with the most taps (at stride 2 the others
        // take the same kernel unless kh or kw > 3)
        if (!tc || (p.stride != 1 && p.stride != 2) || (p.Cout & 3) != 0 || p.Cin < 16) return simt;
        ConvPlan r{SCSFM_KERNEL_GATHER, 0u, false};
        for (int cls = 0, taps = 0; cls < 4; ++cls) {
            ScsfmConv q;
            TcView v;
            dgrad_part(p, cls, q, v);
            if (q.kh * q.kw > taps && q.Ho > 0 && q.Wo > 0) {
                taps = q.kh * q.kw;
                r = route_tc(q, v);
            }
        }
        r.reads = (split ? SCSFM_PLAN_DOUT_LO | SCSFM_PLAN_W_LO : 0u) | SCSFM_PLAN_FLIPPED;
        return r;
    }
    // weight gradient.  SCSFM_TUNE_WGRAD: 0 auto, 1 the gather kernel (CUDA cores: the generic kernel), 2 the TMA kernel
    // (the gather kernel where it does not apply), 3 the thin-layer kernel (auto where it does not apply)
    const unsigned knob = (p.tune >> 12) & 3u;
    const bool thin = conv_wgrad_thin_eligible(p);
    const ConvPlan thin_plan{SCSFM_KERNEL_THIN, 0u, false};
    if (!tc || (p.Cin & 3) != 0 || (p.Cout & 3) != 0 || p.Cout < 16) return thin && knob != 1u ? thin_plan : simt;
    // the 16-output-channel decoder layers in split mode read four tensors and use 16 of the MMA's columns: the fp32 FMA
    // kernel reads two and is exact per product (conv_wgrad_thin.cu)
    if (thin && (knob == 3u || (knob == 0u && split))) return thin_plan;
    const unsigned lo = split ? SCSFM_PLAN_IN_LO | SCSFM_PLAN_DOUT_LO : 0u;
    if (knob != 1u && conv_wgrad_tma_eligible(p)) {
        // the TMA kernel computes the low parts itself; under reflection padding it takes the interior pixels with zero
        // padding and the gather kernel, which reads them, the border ring
        if (p.pad_mode == PADMODE_REFLECT) return ConvPlan{SCSFM_KERNEL_TMA_RING, lo, split && p.Cout <= 64};
        return ConvPlan{SCSFM_KERNEL_TMA, 0u, false};
    }
    return ConvPlan{SCSFM_KERNEL_GATHER, lo, split && p.Cout <= 64};
}

// Launches the kernel route_tc picked for the forward (sub-)convolution p seen through v.
static int launch_route(const ScsfmConv& p, const TcView& v, const ConvPlan& r, cudaStream_t st) {
    switch (r.kernel) {
        case SCSFM_KERNEL_STEM: return launch_conv_stem_fwd(p, st);
        case SCSFM_KERNEL_TMA: return launch_conv_tma(p, v, st);
        case SCSFM_KERNEL_TMA_RING: {
            ScsfmConv q = p;                        // the interior: zero padding
            q.pad_mode = PADMODE_ZERO;
            if (int rc = launch_conv_tma(q, v, st)) return rc;
            TcView ring = v;
            ring.border = 1;
            return launch_gather(p, ring, r.stacked, st);
        }
        default: return launch_gather(p, v, r.stacked, st);
    }
}

static int check_desc(const ScsfmConv* p, const char* who) {
    SCSFM_CHECK_ARG(p != nullptr, "%s: null descriptor", who);
    SCSFM_CHECK_ARG(p->B > 0 && p->Hi > 0 && p->Wi > 0 && p->Cin > 0 && p->Ho > 0 && p->Wo > 0 && p->Cout > 0 && p->kh > 0 &&
                        p->kw > 0 && p->stride > 0 && p->pad >= 0, "%s: bad geometry", who);
    SCSFM_CHECK_ARG(p->mode >= SCSFM_MODE_FP32 && p->mode <= SCSFM_MODE_TF32X3, "%s: bad mode %d", who, p->mode);
    return SCSFM_OK;
}

// Plans call *p of `pass` and validates it for the kernel picked; q receives the descriptor the kernels see (the low parts
// the kernel does not read dropped: the tensor-core kernels count their passes from the low-part pointers).
static int plan_call(const ScsfmConv* p, int pass, const char* who, ConvPlan& r, ScsfmConv& q) {
    if (int rc = check_desc(p, who)) return rc;
    r = conv_plan(*p, pass);
    const bool simt = r.kernel == SCSFM_KERNEL_SIMT;
    SCSFM_CHECK_ARG(pass == SCSFM_PASS_FWD ? p->in && p->w && p->out : pass == SCSFM_PASS_DGRAD ? p->dout && p->w && p->din : p->in && p->dout && p->dw,
                    "%s: null tensor", who);
    SCSFM_CHECK_ARG((long long)p->B * p->Hi * p->Wi * (long long)p->Cin < (1LL << 40), "%s: tensor too large", who);
    SCSFM_CHECK_ARG(p->Ho == (p->Hi + 2 * p->pad - p->kh) / p->stride + 1 && p->Wo == (p->Wi + 2 * p->pad - p->kw) / p->stride + 1,
                    "%s: output size does not match geometry", who);
    if (pass == SCSFM_PASS_FWD) {
        SCSFM_CHECK_ARG((p->bn_scale == nullptr) == (p->bn_shift == nullptr), "%s: bn_scale and bn_shift go together", who);
        SCSFM_CHECK_ARG(p->bn_scale == nullptr || (p->bias == nullptr && p->bn_sums == nullptr),
                        "%s: the eval-mode BatchNorm epilogue excludes bias and bn_sums", who);
        if (simt) {
            SCSFM_CHECK_ARG(p->pad_mode != PADMODE_REFLECT || (p->pad < p->Hi && p->pad < p->Wi && p->pad <= 1), "%s: reflect pad must be 1", who);
        } else {
            SCSFM_CHECK_ARG(p->pad_mode != PADMODE_REFLECT || p->pad == 1, "%s: reflect pad must be 1", who);
            SCSFM_CHECK_ARG(p->bn_sums == nullptr || p->B % (p->bn_groups > 0 ? p->bn_groups : 1) == 0,
                            "%s: batch not divisible by the number of BatchNorm groups", who);
            SCSFM_CHECK_ARG(p->out_lo == nullptr || ((p->Cout & 3) == 0 && (reinterpret_cast<uintptr_t>(p->out_lo) & 15) == 0),
                            "%s: out_lo needs Cout %% 4 == 0 and 16-byte alignment", who);
            SCSFM_CHECK_ARG(((reinterpret_cast<uintptr_t>(p->bn_scale) | reinterpret_cast<uintptr_t>(p->bn_shift)) & 7) == 0,
                            "%s: bn_scale / bn_shift must be 8-byte aligned", who);
        }
    }
    if (pass == SCSFM_PASS_DGRAD && !simt)
        SCSFM_CHECK_ARG(p->kh == p->kw && p->kh - 1 - p->pad >= 0, "%s: square kernels only", who);
    if (pass == SCSFM_PASS_WGRAD && !simt) {
        SCSFM_CHECK_ARG(p->pad_mode != PADMODE_REFLECT || p->pad == 1, "%s: reflect pad must be 1", who);
        SCSFM_CHECK_ARG((long long)p->B * p->Ho * p->Wo < (1LL << 31), "%s: too many pixels", who);
    }
    const unsigned missing = r.reads & ~((p->in_lo ? SCSFM_PLAN_IN_LO : 0u) | (p->dout_lo ? SCSFM_PLAN_DOUT_LO : 0u) |
                                         (p->w_lo ? SCSFM_PLAN_W_LO : 0u) | SCSFM_PLAN_FLIPPED);
    SCSFM_CHECK_ARG(missing == 0, "%s: the kernel chosen for this call reads low parts that were not passed:%s%s%s (scsfm_conv_plan)", who,
                    (missing & SCSFM_PLAN_W_LO) ? " w_lo" : "", (missing & SCSFM_PLAN_IN_LO) ? " in_lo" : "",
                    (missing & SCSFM_PLAN_DOUT_LO) ? " dout_lo" : "");
    q = *p;
    if (!(r.reads & SCSFM_PLAN_IN_LO)) q.in_lo = nullptr;
    if (!(r.reads & SCSFM_PLAN_DOUT_LO)) q.dout_lo = nullptr;
    if (!(r.reads & SCSFM_PLAN_W_LO)) q.w_lo = nullptr;
    return SCSFM_OK;
}

extern "C" int scsfm_conv_plan(const ScsfmConv* p, int pass) {
    SCSFM_CHECK_ARG(pass >= SCSFM_PASS_FWD && pass <= SCSFM_PASS_WGRAD, "conv_plan: bad pass %d", pass);
    if (int rc = check_desc(p, "conv_plan")) return rc;
    const ConvPlan r = conv_plan(*p, pass);
    return r.kernel | (int)r.reads;
}

extern "C" int scsfm_conv2d_fwd(const ScsfmConv* p, void* stream) {
    ConvPlan r;
    ScsfmConv q;
    if (int rc = plan_call(p, SCSFM_PASS_FWD, "conv2d_fwd", r, q)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    return r.kernel == SCSFM_KERNEL_SIMT ? launch_fwd_simt(q, st) : launch_route(q, plain_view(q), r, st);
}

// Tensor cores: the forward kernels on dout with the flipped weights in p->w / p->w_lo; p->din [B,Hi,Wi,Cin] (+ p->addend).
extern "C" int scsfm_conv2d_dgrad(const ScsfmConv* p, void* stream) {
    ConvPlan r;
    ScsfmConv q;
    if (int rc = plan_call(p, SCSFM_PASS_DGRAD, "conv2d_dgrad", r, q)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (r.kernel == SCSFM_KERNEL_SIMT) return launch_dgrad_simt(q, st);
    ScsfmConv f;
    TcView v;
    bool covered_all = true;
    for (int cls = 0; cls < 4; ++cls) {
        dgrad_part(q, cls, f, v);
        if (f.kh * f.kw == 0 && f.Ho > 0 && f.Wo > 0) covered_all = false;
    }
    if (!covered_all) {
        // stride-2 parity classes without taps (1x1 stride 2): their gradient is the addend alone (or zero).  Enqueued
        // before the sub-convolutions, which write the other classes' pixels of din.
        const size_t bytes = (size_t)q.B * q.Hi * q.Wi * q.Cin * sizeof(float);
        if (q.addend) SCSFM_CHECK_CUDA(cudaMemcpyAsync(q.din, q.addend, bytes, cudaMemcpyDeviceToDevice, st));
        else SCSFM_CHECK_CUDA(cudaMemsetAsync(q.din, 0, bytes, st));
    }
    for (int cls = 0; cls < 4; ++cls) {
        dgrad_part(q, cls, f, v);
        if (f.kh * f.kw > 0 && f.Ho > 0 && f.Wo > 0)
            if (int rc = launch_route(f, v, route_tc(f, v), st)) return rc;
    }
    return SCSFM_OK;
}

// dw [Cout,kh,kw,Cin] += dout^T x gather(in); dbias += column sums of dout.
extern "C" int scsfm_conv2d_wgrad(const ScsfmConv* p, void* stream) {
    ConvPlan r;
    ScsfmConv q;
    if (int rc = plan_call(p, SCSFM_PASS_WGRAD, "conv2d_wgrad", r, q)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    int rc;
    if (r.kernel == SCSFM_KERNEL_SIMT) rc = launch_wgrad_simt(q, st);
    else if (r.kernel == SCSFM_KERNEL_THIN) rc = launch_conv_wgrad_thin(q, st);
    else if (r.kernel == SCSFM_KERNEL_GATHER) rc = launch_wgrad_gather(q, r.stacked, 0, st);
    else if ((rc = launch_conv_wgrad_tma(q, st)) == SCSFM_OK && r.kernel == SCSFM_KERNEL_TMA_RING)
        rc = launch_wgrad_gather(q, r.stacked, 1, st);
    if (rc) return rc;
    if (q.dbias) return launch_bias_grad(q.dout, q.B * q.Ho * q.Wo, q.Cout, q.dbias, st);
    return SCSFM_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Flipped / transposed weights of the tensor-core data gradient: w [Co][kh][kw][Ci] -> the weights of the transposed
// convolution, as operand kind `operand`.  Stride 1: wt[c][jy][jx][o] = w[o][kh-1-jy][kw-1-jx][c].  Stride 2: the four
// parity classes back to back in the order (py,px) = (0,0),(0,1),(1,0),(1,1), class k as [Ci][jh][jw][Co] with
// wt[c][jy][jx][o] = w[o][dy_max - 2 jy][dx_max - 2 jx][c]; Ci*kh*kw*Co floats in total either way.
// A job owns ceil(Co/32) * ceil(Ci/32) * kh * kw blocks; each transposes one 32 (Cout) x 32 (Cin) tile of one tap through
// shared memory: reads coalesced along Cin, writes coalesced along Cout.
// ---------------------------------------------------------------------------------------------------------
constexpr int FLIP_ROW = 10;         // table row: {src, dst, Co, kh, kw, Ci, stride, pad, operand, first block}

struct FlipJob {
    const float* w;
    float* wt;
    int Co, kh, kw, Ci, stride, pad, operand;
};

// table == nullptr: the blocks of `job`; else the job of each block is the table row whose first block is the last one
// <= blockIdx.x (row n: a sentinel holding the total).
__global__ void __launch_bounds__(256)
weight_flip_tiles_kernel(FlipJob job, const long long* __restrict__ table, int n) {
    __shared__ int s_row;
    __shared__ float tile[32][33];
    long long t = blockIdx.x;
    if (table != nullptr) {
        if (threadIdx.x == 0) {
            int lo = 0, hi = n;
            while (hi - lo > 1) {
                const int mid = (lo + hi) >> 1;
                if (table[mid * FLIP_ROW + 9] <= t) lo = mid; else hi = mid;
            }
            s_row = lo;
        }
        __syncthreads();
        const long long* e = table + s_row * FLIP_ROW;
        job = FlipJob{reinterpret_cast<const float*>(e[0]), reinterpret_cast<float*>(e[1]), (int)e[2], (int)e[3], (int)e[4],
                      (int)e[5], (int)e[6], (int)e[7], (int)e[8]};
        t -= e[9];
    }
    const int Co = job.Co, kh = job.kh, kw = job.kw, Ci = job.Ci;
    const int tco = (Co + 31) >> 5, tci = (Ci + 31) >> 5;
    const int to = (int)(t % tco), tc = (int)(t / tco % tci);
    int u = (int)(t / tco / tci);                 // tap of the block, counted over the classes in order
    S2Class k{kh, kw, kh - 1, kw - 1};
    size_t off = 0;                               // the class's offset in wt
    if (job.stride == 2) {
        for (int cls = 0;; ++cls) {
            k = s2_class(kh, kw, job.pad, cls >> 1, cls & 1);
            if (u < k.jh * k.jw) break;
            u -= k.jh * k.jw;
            off += (size_t)Co * k.jh * k.jw * Ci;
        }
    }
    const int jy = u / k.jw, jx = u - jy * k.jw;
    const int dy = k.dy_max - job.stride * jy, dx = k.dx_max - job.stride * jx;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int o = to * 32 + ty + 8 * i, c = tc * 32 + tx;
        if (o < Co && c < Ci) tile[ty + 8 * i][tx] = tc_operand(__ldg(job.w + (((size_t)o * kh + dy) * kw + dx) * Ci + c), job.operand);
    }
    __syncthreads();
    float* wt = job.wt + off;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int c = tc * 32 + ty + 8 * i, o = to * 32 + tx;
        if (c < Ci && o < Co) wt[(((size_t)c * k.jh + jy) * k.jw + jx) * Co + o] = tile[tx][ty + 8 * i];
    }
}

extern "C" int scsfm_weight_flip(const float* w, int Cout, int kh, int kw, int Cin, int stride, int pad, float* wt, int operand,
                                 void* stream) {
    SCSFM_CHECK_ARG(w && wt && Cout > 0 && kh > 0 && kw > 0 && Cin > 0 && (stride == 1 || stride == 2) && pad >= 0 && operand >= 0 &&
                        operand <= 2, "weight_flip: bad arguments");
    const long long blocks = (long long)((Cout + 31) / 32) * ((Cin + 31) / 32) * kh * kw;
    SCSFM_CHECK_ARG(blocks < (1LL << 31), "weight_flip: too large");
    weight_flip_tiles_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(FlipJob{w, wt, Cout, kh, kw, Cin, stride, pad, operand}, nullptr, 0);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_weight_flip_batched(const long long* table, int n_rows, int total_blocks, void* stream) {
    SCSFM_CHECK_ARG(table != nullptr && n_rows > 0 && total_blocks > 0, "weight_flip_batched: bad arguments");
    weight_flip_tiles_kernel<<<total_blocks, 256, 0, (cudaStream_t)stream>>>(FlipJob{}, table, n_rows);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}
