// Weight gradient of stride-1 and stride-2 convolutions with kh, kw <= 3 and of the 7x7 stride-2 stems on the tensor
// cores, fed by TMA:
//
//   dW^T[(tap, c), o] += sum_pix  in[pix (+) tap, c] * dout[pix, o]        (GEMM: M = (tap, c), N = o, K = pixels)
//
// Versus the gather kernel of conv_tc.cu (producers transpose both operands through registers, every 64-row M tile of
// (tap, channel) re-reads its input and dout):
//  * a unit of work is one kernel row dy, 64 input channels and a BN-wide Cout tile; a tile is 64 output pixels, 4 x 16
//    or 8 x 8 per call (the shape with the smaller padded output area, 4 x 16 on a tie).  Per tile and stage ONE 4-D TMA
//    box per 32 channels brings the TH x (S * (TW - 1) + kw) input patch (out-of-bounds elements zero-filled = zero
//    padding); the kw taps of the row are address offsets into it.  At stride 2 the box reads a parity-row view of the
//    input (row stride doubled, base on the even or odd row), so the TH input rows of kernel row dy,
//    2 y0 + dy - pad + {0, 2, 4, ...}, are one box; tap dx of output column px is patch column 2 px + dx.  The dout tile
//    of the same pixels also arrives by TMA;
//  * stream-K schedule: the (unit, tile) iterations are one flat unit-major range, units in (dy, channel block, Cout
//    tile) order, split evenly over one persistent wave of CTAs.  A CTA whose range crosses into the next unit adds its
//    sums into dw and starts again from zero; the stage ring runs on across units.  CTAs of different kernel rows sweep
//    the same pixel tiles at about the same time and share the input in L2;
//  * the input is the wgmma A operand and comes from registers: wgmma takes 32-bit operands from shared memory only
//    K-major (K = pixels here) and both tensors are channel-contiguous, but a register fragment is free of that layout.
//    Each consumer thread loads its 4 fragment values per K8 slice with ld.shared straight from the 128B-swizzled patch.
//    The 4 pixels a quad of lanes reads must lie 2 patch columns (256 bytes) apart to be free of bank conflicts for
//    every tap: inside a K8 slice of 8 output pixels (half a 4 x 16 tile row, or one 8 x 8 tile row), k = 0..3 are the
//    even pixels and k = 4..7 the odd ones at stride 1, and the pixels in order at stride 2 (even pixels first would put
//    them 512 bytes apart there);
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
// Split-K over pixel tiles: at the end of each unit of its range every warpgroup adds its kw x 64 x BN partial sums into
// dw with fp32 atomics (dw += ...).
#include <limits.h>
#include <stdlib.h>

#include <algorithm>

#include "conv_tc.cuh"

namespace scsfm {

constexpr int WT_PIX = 64;                           // output pixels per tile (4 x 16 or 8 x 8) = 8 K8 slices
constexpr int WT_CK = 64;                            // input channels per unit (= wgmma M)
constexpr int WT_THREADS = 384;
constexpr int WT_MAX_STAGES = 3;                     // pipeline depth where shared memory allows it (WtCfg::STAGES)
constexpr int WT_PRODUCER_REGS = 56, WT_CONSUMER_REGS = 224;   // setmaxnreg: 128 x 56 + 256 x 224 <= 64 K registers

template <int BN, bool SPLIT, int KW, int S>
struct WtCfg {
    static constexpr bool STEM = KW == 7;                                            // 7x7 stem, 4 or 8 channels
    // input columns x rows of the patch of a 4 x 16 and of an 8 x 8 tile; a box slot holds the larger
    static constexpr int LINES_416 = 4 * (S * 15 + KW), LINES_88 = 8 * (S * 7 + KW);
    static constexpr int LINES = LINES_416 > LINES_88 ? LINES_416 : LINES_88;
    static constexpr int PATCH = ((LINES * (STEM ? 32 : 128) + 1023) / 1024) * 1024;  // one input box (32 / <= 8 channels)
    static constexpr int RAW = WT_PIX * 128;                                         // one 32-channel dout box
    static constexpr int BT = (WT_PIX / 32) * BN * 128;                              // transposed dout [kb][BN rows][32 px]
    static constexpr int STAGE = 2 * PATCH + (BN / 32) * RAW + (SPLIT ? 2 : 1) * BT;
    // 3 stages where they fit into the 227 KB an SM gives one CTA; the stride-2 patches leave 2 at BN = 64
    static constexpr int STAGES = 2048 + WT_MAX_STAGES * STAGE <= 227 * 1024 ? WT_MAX_STAGES : 2;
    static constexpr size_t SMEM = 1024 + 1024 + (size_t)STAGES * STAGE;
};

struct WtGeom {
    int th, tw, pw;                     // output-pixel tile (th x tw = WT_PIX, tw = 16 or 8) and its input patch width
    int tiles_x, tiles_y, n_tiles;      // output tiles per image row / column, tiles in total
    int units, iters;                   // units (dy fastest, then the channel block, then the Cout tile); units x n_tiles
    int split_tiles;                    // 0: stream-K.  > 0: split grid, CTA unit + units * k takes tiles
                                        // [k, k + 1) * split_tiles of its unit (SCSFM_TUNE_WT_SPLIT_GRID)
    int reflect;
};

// The flat (unit, tile) iterations [f0, f1) of this CTA.  Stream-K: an even share of the range per CTA, so the tile
// counts of two CTAs differ by at most one.
__device__ __forceinline__ void wt_range(const WtGeom& g, int& f0, int& f1) {
    const int c = blockIdx.x;
    if (g.split_tiles) {
        const int u = c % g.units, k = c / g.units;
        f0 = u * g.n_tiles + k * g.split_tiles;
        f1 = u * g.n_tiles + min(g.n_tiles, (k + 1) * g.split_tiles);
    } else {
        f0 = (int)((long long)c * g.iters / gridDim.x);
        f1 = (int)((long long)(c + 1) * g.iters / gridDim.x);
    }
}

// unit u -> kernel row dy, first input channel c0, first output channel n0
template <int BN>
__device__ __forceinline__ void wt_unit(const ScsfmConv& p, int u, int& dy, int& c0, int& n0) {
    const int cb = (p.Cin + WT_CK - 1) / WT_CK;
    dy = u % p.kh;
    u /= p.kh;
    c0 = (u % cb) * WT_CK;
    n0 = (u / cb) * BN;
}

__device__ __forceinline__ void setmaxnreg_dec(void) { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(WT_PRODUCER_REGS)); }
__device__ __forceinline__ void setmaxnreg_inc(void) { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(WT_CONSUMER_REGS)); }

__device__ __forceinline__ uint32_t ld_shared_u32(uint32_t saddr) {
    uint32_t v;
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(saddr));
    return v;
}

// KW: taps per kernel row (1 or 3; a 2-wide kernel runs as KW = 3 with the third tap's sums discarded).  S: stride.
// KW = 7: the 7x7 stride-2 stems with Cin = 4 or 8 (padded) channels.  A kernel row times the channels is only 28 or 56
// rows, so the stem puts (dx, c) on M, m = dx * Cin + c, with one accumulator: the box holds the 4 x 37 (8 x 21) x Cin
// patch unswizzled ([row][column][c]), and row m of pixel px reads patch element (2 px) * Cin + m of its row, i.e. the M index
// is contiguous in shared memory.
// amap: the input (S = 1) or its even-row view (S = 2); amap_odd: the odd-row view (S = 2 only).
template <int BN, bool SPLIT, int KW, int S>
__global__ void __launch_bounds__(WT_THREADS, 1)
conv_wgrad_tma_kernel(ScsfmConv p, WtGeom g, const __grid_constant__ CUtensorMap amap, const __grid_constant__ CUtensorMap amap_odd,
                      const __grid_constant__ CUtensorMap dmap) {
    using Cfg = WtCfg<BN, SPLIT, KW, S>;
    constexpr int WT_STAGES = Cfg::STAGES;
    constexpr bool STEM = Cfg::STEM;
    constexpr int NA = STEM ? 1 : KW;                // accumulators: one per tap, one in all for the stem
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bar_full = reinterpret_cast<uint64_t*>(smem);        // TMA bytes landed
    uint64_t* bar_ready = bar_full + WT_STAGES;                     // dout transposed
    uint64_t* bar_empty = bar_ready + WT_STAGES;                    // consumers done with the stage
    const uint32_t ring = tc::smem_u32(smem + 1024);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int pw = g.pw;

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
        y0 = (t % g.tiles_y) * g.th;
        b = t / g.tiles_y;
        x0 = tx * g.tw;
    };

    if (warp >= 8) {
        setmaxnreg_dec();
        if (warp == 8) {
            // ------------------------------------------------------------------ TMA producer
            if (lane == 0) {
                tc::tma_prefetch_desc(&amap);
                if (S == 2) tc::tma_prefetch_desc(&amap_odd);
                tc::tma_prefetch_desc(&dmap);
                int f0, f1;
                wt_range(g, f0, f1);
                for (int f = f0, it = 0; f < f1; ++f, ++it) {
                    const int s = it % WT_STAGES;
                    const int u = f / g.n_tiles;
                    int dy, c0, n0, b, y0, x0;
                    wt_unit<BN>(p, u, dy, c0, n0);
                    tile_origin(f - u * g.n_tiles, b, y0, x0);
                    // stride 2: input row 2 (y0 + r) + dy - pad = 2 (y0 + r + (rr - par) / 2) + par with rr = dy - pad, par = rr & 1
                    const int rr = dy - p.pad, par = rr & 1;
                    const CUtensorMap* in_map = S == 2 && par ? &amap_odd : &amap;
                    const int row_off = S == 2 ? (rr - par) / 2 : rr;
                    const int in_boxes = c0 + 32 < p.Cin ? 2 : 1;
                    const uint32_t tx_bytes = (uint32_t)(in_boxes * g.th * pw * (STEM ? 4 * p.Cin : 128) + (BN / 32) * Cfg::RAW);
                    tc::mbar_wait(bar_empty + s, ((it / WT_STAGES) & 1) ^ 1);
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
            int f0, f1;
            wt_range(g, f0, f1);
            for (int f = f0, it = 0; f < f1; ++f, ++it) {
                const int s = it % WT_STAGES;
                tc::mbar_wait(bar_full + s, (it / WT_STAGES) & 1);
                int b, y0, x0;
                tile_origin(f % g.n_tiles, b, y0, x0);
                const uint32_t st = ring + (uint32_t)(s * Cfg::STAGE);
                const uint32_t raw = st + 2 * Cfg::PATCH, bhi = raw + (BN / 32) * Cfg::RAW, blo = bhi + Cfg::BT;
                for (int u = warp - 9; u < (WT_PIX / 32) * (BN / 4); u += 3) {
                    const int kb = u / (BN / 4), oc = u - kb * (BN / 4);
                    const int px = 32 * kb + lane;
                    const int y = y0 + px / g.tw, x = x0 + px % g.tw;
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
    // K8 slice sl of a tile: tile row sl >> rs, columns 8 (sl & rs) + 0..7 (rs = 1: 4 x 16 tile, 0: 8 x 8)
    const int rs = g.tw == 16 ? 1 : 0;
    float acc[NA][BN / 2];
    float part[BN / 2];
    unsigned long long* dbg = DRAIN_COUNTERS ? p.debug : nullptr;   // optional per-CTA cycle counters (ScsfmConv.debug)
    long long t_full = 0, t_drain = 0;
    const long long t_start = DRAIN_COUNTERS ? clock64() : 0;
    // the units of the range; the stage index it runs on across them
    int f0, f1;
    wt_range(g, f0, f1);
    for (int it = 0; f0 + it < f1;) {
        const int u = (f0 + it) / g.n_tiles, it_end = min(f1, (u + 1) * g.n_tiles) - f0;
        bool w_ok;                                    // warps whose 16 rows all lie beyond M load zeros
        {
            int dy, c0, n0;
            wt_unit<BN>(p, u, dy, c0, n0);
            w_ok = c0 + 16 * w < m_rows;
        }
#pragma unroll
        for (int dx = 0; dx < NA; ++dx)
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[dx][i] = 0.f;
        for (; it < it_end; ++it) {
            const int s = it % WT_STAGES;
            const uint32_t ph = (it / WT_STAGES) & 1;
            const long long t0 = dbg ? clock64() : 0;
            tc::mbar_wait(bar_full + s, ph);              // the input patch (read with ld.shared)
            tc::mbar_wait(bar_ready + s, ph);             // the transposed dout (read by wgmma)
            if (dbg) t_full += clock64() - t0;
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
                        const int sl = 4 * wg + NS * h + j;                  // K8 slice of the stage
                        const int pbase = (sl >> rs) * pw + S * (8 * (sl & rs)) + dx + 2 * tq;
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            // a0: (g, t), a1: (g+8, t), a2: (g, t+4), a3: (g+8, t+4); k = t + 4 (e / 2) is pixel 2 t + e / 2
                            // (stride 1) or pixel t + 4 (e / 2) at patch column 2 t + 8 (e / 2) (stride 2)
                            if (STEM) {
                                const int m = 16 * w + gq + 8 * (e & 1), col = pbase + 8 * (e >> 1);   // dx = 0: col = 2 px
                                ahi[j][e] = m < m_rows ? ld_shared_u32(st + (uint32_t)((col * p.Cin + m) * 4)) : 0u;
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
                        const long long t1 = dbg ? clock64() : 0;
                        tc::wgmma_wait<0>();
                        tc::reg_fence(part);
#pragma unroll
                        for (int i = 0; i < BN / 2; ++i) acc[dx][i] += part[i];
                        if (dbg) t_drain += clock64() - t1;
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
        // end of the unit or of the range: dw[o][dy][dx][c] += acc[dx][4 i + e] (row 16 w + gq + 8 (e / 2) =
        // channel, column 8 i + 2 tq + (e % 2) = o); the next unit starts from zero.  The stem's row m = dx * Cin + c
        // is the same offset inside dw[o][dy]
        int dy, c0, n0;
        wt_unit<BN>(p, u, dy, c0, n0);
        if (STEM) {
#pragma unroll
            for (int i = 0; i < BN / 8; ++i) {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int m = 16 * w + gq + 8 * (e >> 1), o = n0 + 8 * i + 2 * tq + (e & 1);
                    if (m < m_rows && o < p.Cout) red_add(p.dw + ((size_t)o * p.kh + dy) * m_rows + m, acc[0][4 * i + e]);
                }
            }
        } else {
            const int kwr = p.kw;
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
    }
    if (p.debug && tid == 0) {
        // slot 7: tiles of this CTA.  With the drain counters, as in conv_tma_kernel: 2 wait for a full stage, 3 chain
        // drains (wgmma_wait), 4 consumer total.  One row per CTA of the grid
        p.debug[blockIdx.x * 8 + 7] = (unsigned long long)(f1 - f0);
        if (dbg) {
            dbg[blockIdx.x * 8 + 2] = (unsigned long long)t_full;
            dbg[blockIdx.x * 8 + 3] = (unsigned long long)t_drain;
            dbg[blockIdx.x * 8 + 4] = (unsigned long long)(clock64() - t_start);
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

template <int BN, bool SPLIT, int KW, int S>
static int launch_wgrad_tma_cfg(const ScsfmConv& p, cudaStream_t st) {
    using Cfg = WtCfg<BN, SPLIT, KW, S>;
    static const cudaError_t attr_rc =
        cudaFuncSetAttribute(conv_wgrad_tma_kernel<BN, SPLIT, KW, S>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM);
    SCSFM_CHECK_CUDA(attr_rc);
    WtGeom g;
    // the pixel tile with the smaller padded output area (52 columns: 7 x 8 = 56 instead of 4 x 16 = 64), 4 x 16 on a tie
    const unsigned tile_knob = (p.tune >> 14) & 3u;
    const long long pad416 = (long long)((p.Ho + 3) / 4 * 4) * ((p.Wo + 15) / 16 * 16);
    const long long pad88 = (long long)((p.Ho + 7) / 8 * 8) * ((p.Wo + 7) / 8 * 8);
    g.tw = tile_knob == 1 ? 16 : tile_knob == 2 ? 8 : pad88 < pad416 ? 8 : 16;
    g.th = WT_PIX / g.tw;
    g.pw = S * (g.tw - 1) + KW;
    CUtensorMap amap, amap_odd, dmap;
    const long long row = (long long)p.Wi * p.Cin, img = row * p.Hi;
    if (S == 1) {
        if (int rc = encode_nhwc(&amap, p.in, p.B, p.Hi, p.Wi, p.Cin, p.Cin, row, img, TBK, g.pw, g.th, CU_TENSOR_MAP_SWIZZLE_128B))
            return rc;
        amap_odd = amap;
    } else {
        // the even and the odd input rows; the stem's box is all Cin (<= 8) channels, unswizzled
        const int box_c = Cfg::STEM ? p.Cin : TBK;
        const CUtensorMapSwizzle sw = Cfg::STEM ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B;
        if (int rc = encode_nhwc(&amap, p.in, p.B, (p.Hi + 1) / 2, p.Wi, p.Cin, p.Cin, 2 * row, img, box_c, g.pw, g.th, sw)) return rc;
        if (int rc = encode_nhwc(&amap_odd, p.in + row, p.B, p.Hi / 2, p.Wi, p.Cin, p.Cin, 2 * row, img, box_c, g.pw, g.th, sw)) return rc;
    }
    if (int rc = encode_nhwc(&dmap, p.dout, p.B, p.Ho, p.Wo, p.Cout, p.Cout, (long long)p.Wo * p.Cout, (long long)p.Ho * p.Wo * p.Cout, TBK,
                             g.tw, g.th, CU_TENSOR_MAP_SWIZZLE_128B))
        return rc;
    g.tiles_x = (p.Wo + g.tw - 1) / g.tw;
    g.tiles_y = (p.Ho + g.th - 1) / g.th;
    g.n_tiles = g.tiles_x * g.tiles_y * p.B;
    g.reflect = p.pad_mode == PADMODE_REFLECT;
    g.units = ((p.Cin + WT_CK - 1) / WT_CK) * p.kh * ((p.Cout + BN - 1) / BN);
    const long long iters = (long long)g.units * g.n_tiles;
    if (iters > INT_MAX) return SCSFM_ERR_ARG;          // the flat iteration index is an int
    g.iters = (int)iters;
    int ctas;
    if (p.tune & SCSFM_TUNE_WT_SPLIT_GRID) {
        // one CTA per (unit, pixel split), splits rounded down to one wave, each of at least 8 tiles: rounded up, up to
        // units - 1 CTAs (e.g. 1 of the 7x7 stem's 133 on 132 SMs) would form a second wave of full-length CTAs
        int splits = sm_count() / g.units;
        const int max_splits = (g.n_tiles + 7) / 8;
        if (splits > max_splits) splits = max_splits;
        if (splits < 1) splits = 1;
        g.split_tiles = (g.n_tiles + splits - 1) / splits;
        ctas = g.units * ((g.n_tiles + g.split_tiles - 1) / g.split_tiles);
    } else {
        // stream-K: one persistent wave (one resident CTA per SM: shared memory) sharing the flat range evenly, at least
        // 8 tiles per CTA
        g.split_tiles = 0;
        ctas = (int)std::min<long long>(sm_count(), (iters + 7) / 8);
    }
    conv_wgrad_tma_kernel<BN, SPLIT, KW, S><<<ctas, WT_THREADS, Cfg::SMEM, st>>>(p, g, amap, amap_odd, dmap);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

template <int BN, bool SPLIT>
static int launch_wgrad_tma_bn(const ScsfmConv& p, cudaStream_t st) {
    if (p.stride == 2 && p.kw == 7) return launch_wgrad_tma_cfg<BN, SPLIT, 7, 2>(p, st);
    if (p.stride == 2) return p.kw == 1 ? launch_wgrad_tma_cfg<BN, SPLIT, 1, 2>(p, st) : launch_wgrad_tma_cfg<BN, SPLIT, 3, 2>(p, st);
    return p.kw == 1 ? launch_wgrad_tma_cfg<BN, SPLIT, 1, 1>(p, st) : launch_wgrad_tma_cfg<BN, SPLIT, 3, 1>(p, st);
}

// Zero-padded pass over every pixel (reflection padding: interior pixels only, the caller adds the ring).  In tf32x3 mode
// the kernel recomputes the low parts rather than reading them.
// SCSFM_TUNE_BN(32 | 64) picks the Cout tile (default: 32 for Cout <= 32, else 64), SCSFM_TUNE_WT_TILE(16 | 8) the pixel
// tile and SCSFM_TUNE_WT_SPLIT_GRID the split grid instead of stream-K; none of them changes the plan.
int launch_conv_wgrad_tma(const ScsfmConv& p, cudaStream_t st) {
    const bool split = p.mode == SCSFM_MODE_TF32X3;
    const unsigned bn_knob = (p.tune >> 8) & 7u;
    const bool bn32 = bn_knob == 2 || (bn_knob != 3 && p.Cout <= 32);
    if (bn32) return split ? launch_wgrad_tma_bn<32, true>(p, st) : launch_wgrad_tma_bn<32, false>(p, st);
    return split ? launch_wgrad_tma_bn<64, true>(p, st) : launch_wgrad_tma_bn<64, false>(p, st);
}

}  // namespace scsfm
