// Weight gradient of stride-1 and stride-2 convolutions with kh, kw <= 3 and of the 7x7 stride-2 stems on the tensor
// cores, fed by TMA:
//
//   dW^T[(tap, c), o] += sum_pix  in[pix (+) tap, c] * dout[pix, o]        (GEMM: M = (tap, c), N = o, K = pixels)
//
// Versus the gather kernel of conv_tc.cu (producers transpose both operands through registers, every 64-row M tile of
// (tap, channel) re-reads its input and dout):
//  * a CTA owns one kernel row dy, 64 input channels and a BN-wide Cout tile, and walks a range of 4 x 16-pixel output
//    tiles.  Per tile and stage ONE 4-D TMA box per 32 channels brings the 4 x (S * 15 + kw) input patch (out-of-bounds
//    elements zero-filled = zero padding); the kw taps of the row are address offsets into it.  At stride 2 the box
//    reads a parity-row view of the input (row stride doubled, base on the even or odd row), so the 4 input rows of
//    kernel row dy, 2 y0 + dy - pad + {0, 2, 4, 6}, are one box; tap dx of output column px is patch column 2 px + dx.
//    The dout tile of the same pixels also arrives by TMA;
//  * the input is the wgmma A operand and comes from registers: wgmma takes 32-bit operands from shared memory only
//    K-major (K = pixels here) and both tensors are channel-contiguous, but a register fragment is free of that layout.
//    Each consumer thread loads its 4 fragment values per K8 slice with ld.shared straight from the 128B-swizzled patch.
//    The 4 pixels a quad of lanes reads must lie 2 patch columns (256 bytes) apart to be free of bank conflicts for
//    every tap: inside a K8 slice of 8 output pixels, k = 0..3 are the even pixels and k = 4..7 the odd ones at
//    stride 1, and the pixels in order at stride 2 (even pixels first would put them 512 bytes apart there);
//  * dout (the B operand) is transposed once per stage into the K-major 128B-swizzled layout, with the same pixel order,
//    by three transposer warps; all kw taps and both consumer warpgroups share that copy;
//  * split mode (tf32x3): lo(dout) is computed during the transpose and lo(in) from the A fragment (tf32_lo): bit-identical
//    to the stored low parts, which this kernel never reads;
//  * reflection padding: the kernel runs with zero padding and zeroes the dout rows of the image's outer ring of output
//    pixels; the 2 (Ho + Wo) - 4 ring pixels per image then go through the gather kernel (border view).
//
//   warps 0-7   two consumer warpgroups; warpgroup g multiplies the K8 slices [4g, 4g + 4) of every 64-pixel stage
//   warp 8      lane 0: TMA producer (input boxes + dout boxes per stage)
//   warps 9-11  dout transposers
// Split-K over pixel tiles: every warpgroup adds its kw x 64 x BN partial sums into dw with fp32 atomics (dw += ...).
#include <stdlib.h>

#include "conv_tc.cuh"

namespace scsfm {

constexpr int WT_TH = 4, WT_TW = 16;                 // output-pixel tile: 4 rows x 16 columns = 64 pixels = 8 K8 slices
constexpr int WT_PIX = WT_TH * WT_TW;
constexpr int WT_CK = 64;                            // input channels per CTA (= wgmma M)
constexpr int WT_THREADS = 384;
constexpr int WT_MAX_STAGES = 3;                     // pipeline depth where shared memory allows it (WtCfg::STAGES)
constexpr int WT_PRODUCER_REGS = 56, WT_CONSUMER_REGS = 224;   // setmaxnreg: 128 x 56 + 256 x 224 <= 64 K registers

template <int BN, bool SPLIT, int KW, int S>
struct WtCfg {
    static constexpr bool STEM = KW == 7;                                            // 7x7 stem, 4 or 8 channels
    static constexpr int PW = S * (WT_TW - 1) + KW;                                  // patch width (input columns)
    static constexpr int PATCH = ((WT_TH * PW * (STEM ? 32 : 128) + 1023) / 1024) * 1024;   // one input box (32 / <= 8 channels)
    static constexpr int RAW = WT_PIX * 128;                                         // one 32-channel dout box
    static constexpr int BT = (WT_PIX / 32) * BN * 128;                              // transposed dout [kb][BN rows][32 px]
    static constexpr int STAGE = 2 * PATCH + (BN / 32) * RAW + (SPLIT ? 2 : 1) * BT;
    // 3 stages where they fit into the 227 KB an SM gives one CTA; the 33-column stride-2 patch leaves 2 at BN = 64
    static constexpr int STAGES = 2048 + WT_MAX_STAGES * STAGE <= 227 * 1024 ? WT_MAX_STAGES : 2;
    static constexpr size_t SMEM = 1024 + 1024 + (size_t)STAGES * STAGE;
};

struct WtGeom {
    int tiles_x, tiles_y, n_tiles;      // output tiles per image row / column, tiles in total
    int tiles_per_cta;
    int reflect;
};

__device__ __forceinline__ void setmaxnreg_dec(void) { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(WT_PRODUCER_REGS)); }
__device__ __forceinline__ void setmaxnreg_inc(void) { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(WT_CONSUMER_REGS)); }

__device__ __forceinline__ uint32_t ld_shared_u32(uint32_t saddr) {
    uint32_t v;
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(saddr));
    return v;
}

// KW: taps per kernel row (1 or 3; a 2-wide kernel runs as KW = 3 with the third tap's sums discarded).  S: stride.
// KW = 7: the 7x7 stride-2 stems with Cin = 4 or 8 (padded) channels.  A kernel row times the channels is only 28 or 56
// rows, so the stem puts (dx, c) on M, m = dx * Cin + c, with one accumulator: the box holds the 4 x 37 x Cin patch
// unswizzled ([row][column][c]), and row m of pixel px reads patch element (2 px) * Cin + m of its row, i.e. the M index
// is contiguous in shared memory.
// amap: the input (S = 1) or its even-row view (S = 2); amap_odd: the odd-row view (S = 2 only).
template <int BN, bool SPLIT, int KW, int S>
__global__ void __launch_bounds__(WT_THREADS, 1)
conv_wgrad_tma_kernel(ScsfmConv p, WtGeom g, const __grid_constant__ CUtensorMap amap, const __grid_constant__ CUtensorMap amap_odd,
                      const __grid_constant__ CUtensorMap dmap) {
    using Cfg = WtCfg<BN, SPLIT, KW, S>;
    constexpr int PW = Cfg::PW, WT_STAGES = Cfg::STAGES;
    constexpr bool STEM = Cfg::STEM;
    constexpr int NA = STEM ? 1 : KW;                // accumulators: one per tap, one in all for the stem
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bar_full = reinterpret_cast<uint64_t*>(smem);        // TMA bytes landed
    uint64_t* bar_ready = bar_full + WT_STAGES;                     // dout transposed
    uint64_t* bar_empty = bar_ready + WT_STAGES;                    // consumers done with the stage
    const uint32_t ring = tc::smem_u32(smem + 1024);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int dy = blockIdx.x % p.kh, c0 = (blockIdx.x / p.kh) * WT_CK, n0 = blockIdx.y * BN;
    const int t_begin = blockIdx.z * g.tiles_per_cta, t_end = min(g.n_tiles, t_begin + g.tiles_per_cta);
    const int ntile = t_end - t_begin;
    if (ntile <= 0) return;
    const int in_boxes = c0 + 32 < p.Cin ? 2 : 1;

    if (tid == 0) {
        for (int s = 0; s < WT_STAGES; ++s) {
            tc::mbar_init(bar_full + s, 1);
            tc::mbar_init(bar_ready + s, 96);
            tc::mbar_init(bar_empty + s, 256);
        }
        tc::fence_barrier_init();
    }
    __syncthreads();

    auto tile_origin = [&](int t, int& b, int& y0, int& x0) {
        const int tx = t % g.tiles_x;
        t /= g.tiles_x;
        y0 = (t % g.tiles_y) * WT_TH;
        b = t / g.tiles_y;
        x0 = tx * WT_TW;
    };

    if (warp >= 8) {
        setmaxnreg_dec();
        if (warp == 8) {
            // ------------------------------------------------------------------ TMA producer
            if (lane == 0) {
                // stride 2: input row 2 (y0 + r) + dy - pad = 2 (y0 + r + (rr - par) / 2) + par with rr = dy - pad, par = rr & 1
                const int rr = dy - p.pad, par = rr & 1;
                const CUtensorMap* in_map = S == 2 && par ? &amap_odd : &amap;
                const int row_off = S == 2 ? (rr - par) / 2 : rr;
                tc::tma_prefetch_desc(in_map);
                tc::tma_prefetch_desc(&dmap);
                const uint32_t tx_bytes = (uint32_t)(in_boxes * WT_TH * PW * (STEM ? 4 * p.Cin : 128) + (BN / 32) * Cfg::RAW);
                for (int it = 0; it < ntile; ++it) {
                    const int s = it % WT_STAGES;
                    tc::mbar_wait(bar_empty + s, ((it / WT_STAGES) & 1) ^ 1);
                    int b, y0, x0;
                    tile_origin(t_begin + it, b, y0, x0);
                    const uint32_t st = ring + (uint32_t)(s * Cfg::STAGE);
                    tc::mbar_arrive_expect_tx(bar_full + s, tx_bytes);
                    for (int q = 0; q < in_boxes; ++q)
                        tc::tma_load_4d(st + q * Cfg::PATCH, in_map, c0 + 32 * q, S * x0 - p.pad, y0 + row_off, b, bar_full + s);
                    for (int q = 0; q < BN / 32; ++q)
                        tc::tma_load_4d(st + 2 * Cfg::PATCH + q * Cfg::RAW, &dmap, n0 + 32 * q, x0, y0, b, bar_full + s);
                }
            }
            __syncwarp();
        } else {
            // ------------------------------------------------------------------ dout transposers (warps 9-11)
            // unit = (32-pixel k-block kb, 4-channel chunk oc): lane = pixel; one 16-byte load, 4 (8) scalar stores into
            // row 4 oc + i, column = position of the pixel in its K8 slice (stride 1: even pixels first).  The loads of 8
            // consecutive lanes hit 8 different swizzled chunks; the stores of a warp fill one 128-byte row.
            const int kcol = S == 2 ? lane : 8 * (lane >> 3) + ((lane & 7) >> 1) + 4 * (lane & 1);
            for (int it = 0; it < ntile; ++it) {
                const int s = it % WT_STAGES;
                tc::mbar_wait(bar_full + s, (it / WT_STAGES) & 1);
                int b, y0, x0;
                tile_origin(t_begin + it, b, y0, x0);
                const uint32_t st = ring + (uint32_t)(s * Cfg::STAGE);
                const uint32_t raw = st + 2 * Cfg::PATCH, bhi = raw + (BN / 32) * Cfg::RAW, blo = bhi + Cfg::BT;
                for (int u = warp - 9; u < (WT_PIX / 32) * (BN / 4); u += 3) {
                    const int kb = u / (BN / 4), oc = u - kb * (BN / 4);
                    const int px = 32 * kb + lane;
                    const int y = y0 + px / WT_TW, x = x0 + px % WT_TW;
                    float4 v;
                    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                                 : "r"(raw + (uint32_t)((oc >> 3) * Cfg::RAW + px * 128 + ((((oc & 7) ^ px) & 7) << 4))));
                    if (g.reflect && (y == 0 || x == 0 || y == p.Ho - 1 || x == p.Wo - 1)) v = make_float4(0.f, 0.f, 0.f, 0.f);
                    const uint32_t o_hi = bhi + (uint32_t)(kb * BN * 128);
                    tc::st_shared_f32(o_hi + tc::sw128_offset(4 * oc, kcol), v.x);
                    tc::st_shared_f32(o_hi + tc::sw128_offset(4 * oc + 1, kcol), v.y);
                    tc::st_shared_f32(o_hi + tc::sw128_offset(4 * oc + 2, kcol), v.z);
                    tc::st_shared_f32(o_hi + tc::sw128_offset(4 * oc + 3, kcol), v.w);
                    if (SPLIT) {
                        const uint32_t o_lo = blo + (uint32_t)(kb * BN * 128);
                        tc::st_shared_f32(o_lo + tc::sw128_offset(4 * oc, kcol), tf32_lo(v.x));
                        tc::st_shared_f32(o_lo + tc::sw128_offset(4 * oc + 1, kcol), tf32_lo(v.y));
                        tc::st_shared_f32(o_lo + tc::sw128_offset(4 * oc + 2, kcol), tf32_lo(v.z));
                        tc::st_shared_f32(o_lo + tc::sw128_offset(4 * oc + 3, kcol), tf32_lo(v.w));
                    }
                }
                tc::fence_proxy_async();                  // generic-proxy stores -> wgmma (async proxy) reads
                tc::mbar_arrive(bar_ready + s);
            }
        }
        return;
    }

    // ------------------------------------------------------------------ consumer warpgroups (warps 0-7)
    setmaxnreg_inc();
    const int wg = warp >> 2, w = warp & 3;
    const int gq = lane >> 2, tq = lane & 3;
    // fragment rows 16 w + gq (+ 8) = channels; patch box (w >> 1), channel inside the box cc (+ 8)
    const int cc = 16 * (w & 1) + gq;
    const int m_rows = STEM ? 7 * p.Cin : p.Cin;      // stem: rows m = dx * Cin + c
    const bool w_ok = c0 + 16 * w < m_rows;           // warps whose 16 rows all lie beyond M load zeros
    float acc[NA][BN / 2];
#pragma unroll
    for (int dx = 0; dx < NA; ++dx)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[dx][i] = 0.f;
    float part[BN / 2];
    for (int it = 0; it < ntile; ++it) {
        const int s = it % WT_STAGES;
        const uint32_t ph = (it / WT_STAGES) & 1;
        tc::mbar_wait(bar_full + s, ph);              // the input patch (read with ld.shared)
        tc::mbar_wait(bar_ready + s, ph);             // the transposed dout (read by wgmma)
        const uint32_t st = ring + (uint32_t)(s * Cfg::STAGE);
        const uint32_t patch = st + (uint32_t)((w >> 1) * Cfg::PATCH);
        const uint32_t bhi = st + 2 * Cfg::PATCH + (BN / 32) * Cfg::RAW, blo = bhi + Cfg::BT;
#pragma unroll
        for (int dx = 0; dx < NA; ++dx) {
            // SPLIT: two chains of 2 K8 slices x 3 products (6 wgmma) per tap, low-part products first, each added into acc
            // in fp32 registers.  TF32: 4 slices of one product straight into acc.
#pragma unroll
            for (int h = 0; h < (SPLIT ? 2 : 1); ++h) {
                constexpr int NS = SPLIT ? 2 : 4;
                uint32_t ahi[NS][4], alo[NS][4];
#pragma unroll
                for (int j = 0; j < NS; ++j) {
                    const int sl = 4 * wg + NS * h + j;                  // K8 slice of the stage: row sl / 2, columns 8 (sl % 2) + 0..7
                    const int pbase = (sl >> 1) * PW + S * (8 * (sl & 1)) + dx + 2 * tq;
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        // a0: (g, t), a1: (g+8, t), a2: (g, t+4), a3: (g+8, t+4); k = t + 4 (e / 2) is pixel 2 t + e / 2
                        // (stride 1) or pixel t + 4 (e / 2) at patch column 2 t + 8 (e / 2) (stride 2)
                        if (STEM) {
                            const int m = 16 * w + gq + 8 * (e & 1), px = 8 * (sl & 1) + tq + 4 * (e >> 1);
                            ahi[j][e] = m < m_rows ? ld_shared_u32(st + (uint32_t)((((sl >> 1) * PW + 2 * px) * p.Cin + m) * 4)) : 0u;
                        } else {
                            const int pp = pbase + (S == 2 ? 8 : 1) * (e >> 1), ch = cc + 8 * (e & 1);
                            ahi[j][e] = w_ok ? ld_shared_u32(patch + tc::sw128_offset(pp, ch)) : 0u;
                        }
                        if (SPLIT) alo[j][e] = __float_as_uint(tf32_lo(__uint_as_float(ahi[j][e])));
                    }
                }
                if (SPLIT) {
                    tc::reg_fence(part);
                    tc::wgmma_fence();
#pragma unroll
                    for (int j = 0; j < NS; ++j) {
                        const int sl = 4 * wg + NS * h + j;
                        const uint32_t boff = (uint32_t)((sl >> 2) * BN * 128 + (sl & 3) * 32);
                        tc::wgmma_tf32_rs<BN>(part, alo[j], tc::make_desc_sw128(bhi + boff), j == 0 ? 0u : 1u);
                        tc::wgmma_tf32_rs<BN>(part, ahi[j], tc::make_desc_sw128(blo + boff), 1u);
                    }
#pragma unroll
                    for (int j = 0; j < NS; ++j) {
                        const int sl = 4 * wg + NS * h + j;
                        const uint32_t boff = (uint32_t)((sl >> 2) * BN * 128 + (sl & 3) * 32);
                        tc::wgmma_tf32_rs<BN>(part, ahi[j], tc::make_desc_sw128(bhi + boff), 1u);
                    }
                    tc::wgmma_commit();
                    tc::wgmma_wait<0>();
                    tc::reg_fence(part);
#pragma unroll
                    for (int i = 0; i < BN / 2; ++i) acc[dx][i] += part[i];
                } else {
                    tc::reg_fence(acc[dx]);
                    tc::wgmma_fence();
#pragma unroll
                    for (int j = 0; j < NS; ++j) {
                        const int sl = 4 * wg + j;
                        const uint32_t boff = (uint32_t)((sl >> 2) * BN * 128 + (sl & 3) * 32);
                        tc::wgmma_tf32_rs<BN>(acc[dx], ahi[j], tc::make_desc_sw128(bhi + boff), 1u);
                    }
                    tc::wgmma_commit();
                    tc::wgmma_wait<0>();
                    tc::reg_fence(acc[dx]);
                }
            }
        }
        tc::mbar_arrive(bar_empty + s);
    }
    // dw[o][dy][dx][c] += acc[dx][4 i + e] (row 16 w + gq + 8 (e / 2) = channel, column 8 i + 2 tq + (e % 2) = o); the
    // stem's row m = dx * Cin + c is the same offset inside dw[o][dy]
    const int kwr = p.kw;
    if (STEM) {
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int m = 16 * w + gq + 8 * (e >> 1), o = n0 + 8 * i + 2 * tq + (e & 1);
                if (m < m_rows && o < p.Cout) red_add(p.dw + ((size_t)o * p.kh + dy) * m_rows + m, acc[0][4 * i + e]);
            }
        }
        return;
    }
#pragma unroll
    for (int dx = 0; dx < NA; ++dx) {
        if (dx >= kwr) break;
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int c = c0 + 16 * w + gq + 8 * (e >> 1), o = n0 + 8 * i + 2 * tq + (e & 1);
                if (c < p.Cin && o < p.Cout) red_add(p.dw + (((size_t)o * p.kh + dy) * kwr + dx) * p.Cin + c, acc[dx][4 * i + e]);
            }
        }
    }
}

bool conv_wgrad_tma_eligible(const ScsfmConv& p) {
    if (p.tune & SCSFM_TUNE_NO_TMA) return false;
    const bool stem = p.stride == 2 && p.kh == 7 && p.kw == 7 && (p.Cin == 4 || p.Cin == 8);
    if (!stem && ((p.stride != 1 && p.stride != 2) || p.kh > 3 || p.kw > 3)) return false;
    if ((p.Cin & 3) != 0 || (p.Cout & 3) != 0) return false;        // 16-byte TMA rows
    if (p.pad_mode == PADMODE_REFLECT && (p.stride != 1 || p.Ho < 3 || p.Wo < 3)) return false;   // the border view needs distinct rings
    if (p.stride == 2 && p.Hi < 2) return false;                    // the odd-row view needs one row
    return true;
}

static int sm_count() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    }
    return n;
}

// rows: rows of the view; row_step: image rows per view row (2: a parity-row view based on base's row), H: image rows
static int encode_nhwc(CUtensorMap* map, const float* base, int B, int H, int W, int C, int box_w, int box_h, int rows, int row_step,
                       int box_c = TBK, CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_128B) {
    const cuuint64_t gdim[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)rows, (cuuint64_t)B};
    const cuuint64_t gstride[3] = {(cuuint64_t)C * 4, (cuuint64_t)row_step * W * C * 4, (cuuint64_t)H * W * C * 4};
    const cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    const CUresult r = encode_tiled(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(base), gdim, gstride, box, estr,
                                    CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled(%d x %d x %d x %d) failed with CUresult %d", B, H, W, C, (int)r);
        return SCSFM_ERR_CUDA;
    }
    return SCSFM_OK;
}

template <int BN, bool SPLIT, int KW, int S>
static int launch_wgrad_tma_cfg(const ScsfmConv& p, cudaStream_t st) {
    using Cfg = WtCfg<BN, SPLIT, KW, S>;
    static const cudaError_t attr_rc =
        cudaFuncSetAttribute(conv_wgrad_tma_kernel<BN, SPLIT, KW, S>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM);
    SCSFM_CHECK_CUDA(attr_rc);
    CUtensorMap amap, amap_odd, dmap;
    if (S == 1) {
        if (int rc = encode_nhwc(&amap, p.in, p.B, p.Hi, p.Wi, p.Cin, Cfg::PW, WT_TH, p.Hi, 1)) return rc;
        amap_odd = amap;
    } else {
        // the stem's box is all Cin (<= 8) channels, unswizzled
        const int box_c = Cfg::STEM ? p.Cin : TBK;
        const CUtensorMapSwizzle sw = Cfg::STEM ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B;
        if (int rc = encode_nhwc(&amap, p.in, p.B, p.Hi, p.Wi, p.Cin, Cfg::PW, WT_TH, (p.Hi + 1) / 2, 2, box_c, sw)) return rc;
        if (int rc = encode_nhwc(&amap_odd, p.in + (size_t)p.Wi * p.Cin, p.B, p.Hi, p.Wi, p.Cin, Cfg::PW, WT_TH, p.Hi / 2, 2, box_c, sw))
            return rc;
    }
    if (int rc = encode_nhwc(&dmap, p.dout, p.B, p.Ho, p.Wo, p.Cout, WT_TW, WT_TH, p.Ho, 1)) return rc;
    WtGeom g;
    g.tiles_x = (p.Wo + WT_TW - 1) / WT_TW;
    g.tiles_y = (p.Ho + WT_TH - 1) / WT_TH;
    g.n_tiles = g.tiles_x * g.tiles_y * p.B;
    g.reflect = p.pad_mode == PADMODE_REFLECT;
    const int mt = ((p.Cin + WT_CK - 1) / WT_CK) * p.kh, nt = (p.Cout + BN - 1) / BN;
    // one resident CTA per SM (shared memory): one wave of pixel splits, each of at least 8 tiles.  Rounded down: a
    // split count rounded up can put up to mt * nt - 1 CTAs (e.g. 1 of the 7x7 stem's 133 on 132 SMs) into a second
    // wave of full-length CTAs
    int splits = sm_count() / (mt * nt);
    const int max_splits = (g.n_tiles + 7) / 8;
    if (splits > max_splits) splits = max_splits;
    if (splits < 1) splits = 1;
    g.tiles_per_cta = (g.n_tiles + splits - 1) / splits;
    dim3 grid(mt, nt, (g.n_tiles + g.tiles_per_cta - 1) / g.tiles_per_cta);
    conv_wgrad_tma_kernel<BN, SPLIT, KW, S><<<grid, WT_THREADS, Cfg::SMEM, st>>>(p, g, amap, amap_odd, dmap);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

template <int BN, bool SPLIT>
static int launch_wgrad_tma_bn(const ScsfmConv& p, cudaStream_t st) {
    if (p.stride == 2 && p.kw == 7) return launch_wgrad_tma_cfg<BN, SPLIT, 7, 2>(p, st);
    if (p.stride == 2) return p.kw == 1 ? launch_wgrad_tma_cfg<BN, SPLIT, 1, 2>(p, st) : launch_wgrad_tma_cfg<BN, SPLIT, 3, 2>(p, st);
    return p.kw == 1 ? launch_wgrad_tma_cfg<BN, SPLIT, 1, 1>(p, st) : launch_wgrad_tma_cfg<BN, SPLIT, 3, 1>(p, st);
}

// Zero-padded pass over every pixel (reflection padding: interior pixels only, the caller adds the ring).  Split mode is
// taken from p.split or from p.in_lo / p.dout_lo being set; the kernel recomputes the low parts rather than reading them.
// SCSFM_TUNE_BN(32 | 64) picks the Cout tile (default: 32 for Cout <= 32, else 64).
int launch_conv_wgrad_tma(const ScsfmConv& p, cudaStream_t st) {
    const bool split = p.split || (p.in_lo != nullptr && p.dout_lo != nullptr);
    const unsigned bn_knob = (p.tune >> 8) & 7u;
    const bool bn32 = bn_knob == 2 || (bn_knob != 3 && p.Cout <= 32);
    if (bn32) return split ? launch_wgrad_tma_bn<32, true>(p, st) : launch_wgrad_tma_bn<32, false>(p, st);
    return split ? launch_wgrad_tma_bn<64, true>(p, st) : launch_wgrad_tma_bn<64, false>(p, st);
}

}  // namespace scsfm
