// Stride-1 and stride-2 convolution on the tensor cores: persistent CTAs, TMA halo-patch producer, two consumer
// warpgroups (wgmma, tf32 operands, fp32 accumulation in registers).
//
//   D[pixels (M = 64 per wgmma), Cout tile (N = BNW)] = im2col(x)[pixels, K] x W[Cout, K]^T
//
// Versus the cp.async kernel of conv_tc.cu (one 64 x 32-float im2col slice gathered per (tap, channel chunk), one CTA per
// 64-pixel tile):
//  * the output tile is a 2-D patch of ONE image (MT*TH rows x TW columns, TH*TW = 128, TW in {8, 16}); per (channel
//    chunk, dx) ONE 4-D tiled TMA load brings the (MT*TH + kh - 1) x TW x 32-channel input patch in the 128B-swizzled
//    K-major layout the wgmma descriptors expect.  TW is a multiple of 8, so the operand of tap row dy is the SAME patch
//    shifted by dy*TW rows = dy*TW*128 bytes (a multiple of the 1024-byte swizzle atom): the kh vertical taps reuse one
//    load.  Zero padding is the TMA's out-of-bounds fill; channels beyond Cin in the last 32-wide chunk are zero-filled
//    the same way (the matching weight columns then multiply zeros) and all-zero K8 slices are not issued at all;
//  * stride 2: the input is read through (row parity, column parity) views (row and column strides doubled, base on
//    the even or odd row / column), where a tap is again a plain shift.  Taps of the same row parity share one box
//    (3x3 pad 1: dy = 0 and 2 the odd rows, MT*TH + 1 of them; dy = 1 the MT*TH even rows), so a stage is one
//    (channel chunk, dx, row parity) box with its taps' weights, sized for the larger box (TmaGeom);
//  * one CTA per SM walks the (tile, Cout tile) work list; the shared-memory stage ring and the mbarrier phases run
//    across tiles, so the producer prefetches the next tile's patches while the current one is multiplied and stored;
//  * the accumulator comes out pixel-major (a thread holds 2 consecutive channels of a pixel per fragment), so the
//    epilogue writes NHWC straight from registers: bias or eval-mode BatchNorm / residual addend / activation / TF32
//    rounding / low part / BatchNorm sums.
//
//   warps 0-7   two consumer warpgroups; warpgroup g owns the pixels [64 MT g, 64 MT (g + 1)) of the tile
//   warp 8      lane 0: TMA producer (1 activation box + its taps' weight boxes per stage, mbarrier expect_tx); warps
//               9-11 only complete the producer warpgroup, whose registers setmaxnreg hands to the consumers
//
// Used for: forward of every stride-1 layer and of the zero-padded stride-2 layers with kh, kw <= 3 (s2_prefers_gather in
// conv_tc.cu keeps the shapes measured faster on the gather kernel there; reflection-padded stride-1 layers run it with zero padding and the cp.async kernel then recomputes the 2*(H+W)-4 border pixels per
// image, see tc_dispatch in conv_tc.cu), stride-1 data gradients, and the four parity-class sub-convolutions of
// stride-2 data gradients.
#include <stdlib.h>
#include <string.h>

#include "conv_tc.cuh"

namespace scsfm {

constexpr int TMA_CWARPS = 8;
// a whole producer warpgroup (warp 8 issues, 9-11 idle): registers are handed out per warpgroup, so with 9 warps the
// consumers would get 65536 / 384 = 168 each anyway; setmaxnreg moves the producer group's share to the consumers
constexpr int TMA_THREADS = (TMA_CWARPS + 4) * 32;
constexpr int TMA_PRODUCER_REGS = 40, TMA_CONSUMER_REGS = 232;   // 128 x 40 + 256 x 232 <= 64 K registers
constexpr int TMA_MAX_KH = 3;
constexpr int TMA_MAX_STAGES = 8;
constexpr int TMA_SMEM_MAX = 232448;                         // 227 KB: the most one CTA may opt into on sm_90

struct TmaGeom {
    int tw_log2;             // TW = 1 << tw_log2 (3 or 4), TH = 128 >> tw_log2
    int tiles_x, tiles_y;    // pixel tiles per image
    int n_tiles, num_work;   // Cout tiles; work items = B * tiles_y * tiles_x * n_tiles (Cout tile fastest)
    int stages;              // shared-memory ring depth
    int a_bytes, stage_bytes;
    // Activation boxes: one stage = one (channel chunk, dx, box).  Box i reads the row-parity view box_py[i] (stride 1:
    // the input itself) from view row y0 + box_y[i], box_rows[i] rows, and serves the kernel rows tap_dy[box_tap0[i] + j]
    // (j < box_ntap[i]), tap j shifted by tap_shift[...] * TW pixels; stage weight slot j holds that tap.  Column tap dx
    // reads the column-parity view col_px[dx] from view column x0 + col_x[dx].  Stride 1: one box of MT*TH + kh - 1
    // rows; stride 2 (3x3 pad 1): the odd rows (dy = 0, 2: MT*TH + 1 rows) and the even rows (dy = 1: MT*TH rows).
    int nbox;
    int box_py[2], box_y[2], box_rows[2], box_tap0[2], box_ntap[2];
    int tap_dy[TMA_MAX_KH], tap_shift[TMA_MAX_KH];
    int col_px[TMA_MAX_KH], col_x[TMA_MAX_KH];
    // split-accumulate passes per (channel chunk, dx): pass i multiplies (activations: lo if a_lo bit i else raw) by
    // (weights: lo if w_lo bit i else raw); plain TF32 = one pass with both masks 0
    int npass, a_lo, w_lo;
    // accumulation chunks: channel chunks whose passes the producer issues together (low parts first).  In split mode the
    // consumers also add every stage's wgmma into the running sum in fp32 registers (round-to-nearest): the tensor core adds
    // into its accumulator with truncation, a systematic bias that grows with the chain.  Plain TF32: one chain per tile.
    int cpg;
    unsigned long long* dbg; // optional per-CTA cycle counters (ScsfmConv.debug), 8 per CTA; NULL = off
};

// a[py * 2 + px]: the activations seen through the (row parity py, column parity px) view (stride 2; stride 1 uses a[0]
// only), a_lo the same for the low part; w, w_lo the weight matrix [Cout][K]
struct TmaMaps {
    CUtensorMap a[4], a_lo[4], w, w_lo;
};

// BNW: Cout tile = weight rows kept in shared memory = N of the wgmma (16/32/64/128).
// MT: 128-pixel sub-tiles stacked vertically; each consumer warpgroup runs MT wgmma of M = 64 per K8 slice.
template <int BNW, int MT>
__global__ void __launch_bounds__(TMA_THREADS, 1)
conv_tma_kernel(ScsfmConv p, TcView v, TmaGeom g, const __grid_constant__ TmaMaps maps) {
    constexpr int W_TILE = BNW * 128;                        // one tap: BNW rows x 32 floats
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bar_full = reinterpret_cast<uint64_t*>(smem);
    uint64_t* bar_empty = bar_full + TMA_MAX_STAGES;
    uint8_t* ring = smem + 1024;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int TW = 1 << g.tw_log2, TH = TBM >> g.tw_log2;
    const int N = p.Cout;
    const int chunks = (p.Cin + TBK - 1) / TBK;

    if (tid == 0) {
        for (int s = 0; s < g.stages; ++s) {
            tc::mbar_init(bar_full + s, 1);              // the producer's expect_tx arrival; TMA completes the bytes
            tc::mbar_init(bar_empty + s, TMA_CWARPS * 32);   // every consumer thread, once the wgmma that read the stage retired
        }
        tc::fence_barrier_init();
    }
    __syncthreads();
    const uint32_t ring_base = tc::smem_u32(ring);

    if (warp >= TMA_CWARPS) {
        // ------------------------------------------------------------------ TMA producer
        tc::setmaxnreg_dec<TMA_PRODUCER_REGS>();
        if (warp == TMA_CWARPS && lane == 0) {
            for (int i = 0; i < g.nbox; ++i)
                for (int dx = 0; dx < v.kw; ++dx) {
                    const int mi = g.box_py[i] * 2 + g.col_px[dx];
                    tc::tma_prefetch_desc(&maps.a[mi]);
                    if (g.a_lo) tc::tma_prefetch_desc(&maps.a_lo[mi]);
                }
            tc::tma_prefetch_desc(&maps.w);
            if (g.w_lo) tc::tma_prefetch_desc(&maps.w_lo);
            int s = 0;
            uint32_t ph = 0;
            long long t_wait = 0;
            const long long t_begin = clock64();
            for (int w = blockIdx.x; w < g.num_work; w += gridDim.x) {
                int t = w / g.n_tiles;
                const int n0 = (w - t * g.n_tiles) * BNW;
                const int tx = t % g.tiles_x; t /= g.tiles_x;
                const int ty = t % g.tiles_y;
                const int b = t / g.tiles_y;
                const int y0 = ty * (MT * TH), x0 = tx * TW;
                // one accumulation chain = cpg channel chunks; inside a chain the low-part passes run FIRST (their sums are
                // 2^-11 of the main term: added while the accumulator is still small they lose nothing to its truncation),
                // the raw x raw pass last
                for (int ck0 = 0; ck0 < chunks; ck0 += g.cpg)
                for (int q = 0; q < g.npass; ++q) {
                    const int ps = (q + 1) % g.npass;
                    const CUtensorMap* am = ((g.a_lo >> ps) & 1) ? maps.a_lo : maps.a;
                    const CUtensorMap* wm = ((g.w_lo >> ps) & 1) ? &maps.w_lo : &maps.w;
                    for (int ck = ck0; ck < min(chunks, ck0 + g.cpg); ++ck) {
                        for (int dx = 0; dx < v.kw; ++dx) {
                            for (int bx = 0; bx < g.nbox; ++bx) {
                                const long long t0 = g.dbg ? clock64() : 0;
                                tc::mbar_wait(bar_empty + s, ph ^ 1);
                                if (g.dbg) t_wait += clock64() - t0;
                                const uint32_t st = ring_base + (uint32_t)(s * g.stage_bytes);
                                const int nt = g.box_ntap[bx];
                                tc::mbar_arrive_expect_tx(bar_full + s, (uint32_t)(g.box_rows[bx] * TW * 128 + nt * W_TILE));
                                tc::tma_load_4d(st, am + g.box_py[bx] * 2 + g.col_px[dx], ck * TBK, x0 + g.col_x[dx], y0 + g.box_y[bx], b,
                                                bar_full + s);
                                for (int j = 0; j < nt; ++j) {
                                    const int dy = g.tap_dy[g.box_tap0[bx] + j];
                                    tc::tma_load_2d(st + (uint32_t)(g.a_bytes + j * W_TILE), wm, (dy * v.kw + dx) * p.Cin + ck * TBK, n0, bar_full + s);
                                }
                                if (++s == g.stages) { s = 0; ph ^= 1; }
                            }
                        }
                    }
                }
            }
            if (g.dbg) {
                g.dbg[blockIdx.x * 8 + 0] = (unsigned long long)t_wait;
                g.dbg[blockIdx.x * 8 + 1] = (unsigned long long)(clock64() - t_begin);
            }
        }
        __syncwarp();
    } else {
        // ------------------------------------------------------------------ consumer warpgroups (warps 0-7)
        tc::setmaxnreg_inc<TMA_CONSUMER_REGS>();
        const int wg = warp >> 2, t = tid & 127;
        const int fr = 16 * (t >> 5) + ((t & 31) >> 2), fc = 2 * (t & 3);   // fragment row / column of d[0]
        const int groups = p.bn_groups > 0 ? p.bn_groups : 1;
        const int act = p.act & 0xff;
        const bool round = (p.act & ROUND_TF32) != 0;
        const long long img_step = (long long)v.out_H * v.out_W * N;       // elements between images
        const int row_step = v.out_sy * v.out_W * N;                        // ... between tile rows
        const int px_step = v.out_sx * N;                                   // ... between tile columns
        float acc[MT][BNW / 2], part[MT][BNW / 2];
        int s = 0;
        uint32_t ph = 0;
        int pend = -1;
        int items = 0;                                   // work items of this CTA (debug slot 7)
        long long t_full = 0;
        const long long t_begin = clock64();
        for (int w = blockIdx.x; w < g.num_work; w += gridDim.x, ++items) {
            int tt = w / g.n_tiles;
            const int n0 = (w - tt * g.n_tiles) * BNW;
            const int tx = tt % g.tiles_x; tt /= g.tiles_x;
            const int ty = tt % g.tiles_y;
            const int b = tt / g.tiles_y;
            const int y0 = ty * (MT * TH), x0 = tx * TW;
#pragma unroll
            for (int mb = 0; mb < MT; ++mb)
#pragma unroll
                for (int i = 0; i < BNW / 2; ++i) acc[mb][i] = 0.f;
            for (int ck0 = 0; ck0 < chunks; ck0 += g.cpg) {          // one accumulation chain (same loop nest as the producer)
                bool first = true;
                for (int q = 0; q < g.npass; ++q) {
                    for (int ck = ck0; ck < min(chunks, ck0 + g.cpg); ++ck) {
                        const int rem = p.Cin - ck * TBK;
                        const int k8 = rem >= TBK ? TBK / 8 : (rem + 7) / 8;           // K8 slices holding real channels
                        for (int dxb = 0; dxb < v.kw * g.nbox; ++dxb) {
                            const int bx = dxb % g.nbox;
                            const long long t0 = g.dbg ? clock64() : 0;
                            tc::mbar_wait(bar_full + s, ph);
                            if (g.dbg) t_full += clock64() - t0;
                            const uint32_t x_addr = ring_base + (uint32_t)(s * g.stage_bytes);
                            const uint32_t w_addr = x_addr + (uint32_t)g.a_bytes;
#pragma unroll
                            for (int mb = 0; mb < MT; ++mb) tc::reg_fence(part[mb]);
                            tc::wgmma_fence();
                            for (int j = 0; j < g.box_ntap[bx]; ++j) {
                                const int shift = g.tap_shift[g.box_tap0[bx] + j];
                                for (int q8 = 0; q8 < k8; ++q8) {
                                    const uint64_t dw = tc::make_desc_sw128(w_addr + (uint32_t)(j * W_TILE + q8 * 32));
#pragma unroll
                                    for (int mb = 0; mb < MT; ++mb) {
                                        const uint32_t a = x_addr + (uint32_t)((shift * TW + 64 * (wg * MT + mb)) * 128 + q8 * 32);
                                        tc::wgmma_tf32<BNW>(part[mb], tc::make_desc_sw128(a), dw, first ? 0u : 1u);
                                    }
                                    first = false;
                                }
                            }
                            tc::wgmma_commit();
                            if (g.npass > 1) {
                                // split mode: every stage is a chain of its own (kh * k8 <= 12 wgmma), added in fp32 registers
                                tc::wgmma_wait<0>();
#pragma unroll
                                for (int mb = 0; mb < MT; ++mb) {
                                    tc::reg_fence(part[mb]);
#pragma unroll
                                    for (int i = 0; i < BNW / 2; ++i) acc[mb][i] += part[mb][i];
                                }
                                tc::mbar_arrive(bar_empty + s);
                                first = true;
                            } else {
                                tc::wgmma_wait<1>();         // the previous stage's group has retired
                                if (pend >= 0) tc::mbar_arrive(bar_empty + pend);
                                pend = s;
                            }
                            if (++s == g.stages) { s = 0; ph ^= 1; }
                        }
                    }
                }
                if (pend >= 0) {
                    tc::wgmma_wait<0>();
#pragma unroll
                    for (int mb = 0; mb < MT; ++mb) {
                        tc::reg_fence(part[mb]);
#pragma unroll
                        for (int i = 0; i < BNW / 2; ++i) acc[mb][i] += part[mb][i];
                    }
                    tc::mbar_arrive(bar_empty + pend);
                    pend = -1;
                }
            }
            // ---- epilogue straight from the registers: fragment i of sub-tile mb holds channels n0 + 8i + fc (+1) of the
            // pixels fr and fr + 8 of the warpgroup's 64-pixel block
            const int cv = min(BNW, N - n0);                     // real channels of this Cout tile (multiple of 4)
            float bs1[BNW / 4], bs2[BNW / 4];
#pragma unroll
            for (int i = 0; i < BNW / 4; ++i) { bs1[i] = 0.f; bs2[i] = 0.f; }
            const long long tile_off = (long long)b * img_step + (long long)(y0 * v.out_sy + v.out_oy) * (v.out_W * N) +
                                       (long long)(x0 * v.out_sx + v.out_ox) * N + n0;
            // channel pair outermost: its bias / BatchNorm coefficients are loaded once and stay live for 2 * MT pixels only
#pragma unroll
            for (int i = 0; i < BNW / 8; ++i) {
                const int c = 8 * i + fc;
                if (c >= cv) continue;
                float2 bb = make_float2(0.f, 0.f), sc = make_float2(0.f, 0.f), sh = make_float2(0.f, 0.f);
                if (p.bias != nullptr) bb = __ldg(reinterpret_cast<const float2*>(p.bias + n0 + c));
                if (p.bn_scale != nullptr) {
                    sc = __ldg(reinterpret_cast<const float2*>(p.bn_scale + n0 + c));
                    sh = __ldg(reinterpret_cast<const float2*>(p.bn_shift + n0 + c));
                }
#pragma unroll
                for (int mb = 0; mb < MT; ++mb) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int l = 64 * (wg * MT + mb) + fr + 8 * h;       // pixel index inside the tile
                        const int row = l >> g.tw_log2, col = l & (TW - 1);
                        if (y0 + row >= p.Ho || x0 + col >= p.Wo) continue;
                        const long long off = tile_off + (long long)row * row_step + (long long)col * px_step;
                        float2 x = make_float2(acc[mb][4 * i + 2 * h], acc[mb][4 * i + 2 * h + 1]);
                        if (p.bias != nullptr) { x.x += bb.x; x.y += bb.y; }
                        if (p.bn_scale != nullptr) { x.x = fmaf(x.x, sc.x, sh.x); x.y = fmaf(x.y, sc.y, sh.y); }   // eval-mode BatchNorm (bn_apply's arithmetic)
                        if (p.addend != nullptr) {
                            const float2 a = __ldg(reinterpret_cast<const float2*>(p.addend + off + c));
                            x.x += a.x; x.y += a.y;
                        }
                        if (act != ACT_NONE) { x.x = tc_act(x.x, act); x.y = tc_act(x.y, act); }
                        if (round) { x.x = tf32_round(x.x); x.y = tf32_round(x.y); }
                        *reinterpret_cast<float2*>(p.out + off + c) = x;
                        if (p.out_lo != nullptr) *reinterpret_cast<float2*>(p.out_lo + off + c) = make_float2(tf32_lo(x.x), tf32_lo(x.y));
                        bs1[2 * i] += x.x; bs1[2 * i + 1] += x.y;
                        bs2[2 * i] += x.x * x.x; bs2[2 * i + 1] += x.y * x.y;
                    }
                }
            }
            if (p.bn_sums != nullptr) {
                // lanes with the same lane % 4 own the same channels: butterfly them together, then one fp64 atomic pair per
                // (warp, channel).  The tile lies in one image, hence in one BatchNorm group.
#pragma unroll
                for (int o = 4; o < 32; o <<= 1) {
#pragma unroll
                    for (int i = 0; i < BNW / 4; ++i) {
                        bs1[i] += __shfl_xor_sync(0xffffffffu, bs1[i], o);
                        bs2[i] += __shfl_xor_sync(0xffffffffu, bs2[i], o);
                    }
                }
                if (lane < 4) {
                    const int grp = b / (p.B / groups);
                    double* d = p.bn_sums + (((size_t)(w % SCSFM_BN_SLOTS) * groups + grp) * N + n0) * 2;
#pragma unroll
                    for (int i = 0; i < BNW / 8; ++i) {
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int c = 8 * i + fc + e;
                            if (c < cv) {
                                atomicAdd(d + 2 * c, (double)bs1[2 * i + e]);
                                atomicAdd(d + 2 * c + 1, (double)bs2[2 * i + e]);
                            }
                        }
                    }
                }
            }
        }
        if (g.dbg && tid == 0) {
            g.dbg[blockIdx.x * 8 + 2] = (unsigned long long)t_full;
            g.dbg[blockIdx.x * 8 + 4] = (unsigned long long)(clock64() - t_begin);
            g.dbg[blockIdx.x * 8 + 7] = (unsigned long long)items;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
// per-call knobs (ScsfmConv.tune, include/scsfm.h): no process-global state
static int tune_mt(const ScsfmConv& p) { return (int)((p.tune >> 4) & 3u); }
static int tune_tw(const ScsfmConv& p) { const int t = (int)((p.tune >> 6) & 3u); return t ? t + 2 : 0; }
static int tune_bn(const ScsfmConv& p) { const int t = (int)((p.tune >> 8) & 15u); return t ? 8 << t : 0; }

bool conv_tma_eligible(const ScsfmConv& p, const TcView& v) {
    if ((p.tune & SCSFM_TUNE_NO_TMA) || v.border) return false;
    if (v.kh > TMA_MAX_KH || v.kw > TMA_MAX_KH || v.kh < 1 || v.kw < 1) return false;
    if (v.in_stride != 1 && (v.in_stride != 2 || p.Hi < 2 || p.Wi < 2)) return false;   // stride 2: every parity view non-empty
    if ((p.Cin & 3) != 0 || (p.Cout & 3) != 0) return false;      // 16-byte TMA rows / float4 epilogue
    if (p.bn_sums && p.B % (p.bn_groups > 0 ? p.bn_groups : 1) != 0) return false;
    return true;
}

bool conv_tma_forced(const ScsfmConv& p) { return tune_mt(p) != 0 || tune_bn(p) != 0 || tune_tw(p) != 0; }

static int sm_count() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    }
    return n;
}

template <int BNW, int MT>
static int launch_tma_cfg(const ScsfmConv& p, const TcView& v, int tw_log2, cudaStream_t st) {
    // one-time opt-in to 227 KB of dynamic shared memory (C++11 thread-safe static initialisation)
    static const cudaError_t attr_rc = cudaFuncSetAttribute(conv_tma_kernel<BNW, MT>, cudaFuncAttributeMaxDynamicSharedMemorySize, TMA_SMEM_MAX);
    SCSFM_CHECK_CUDA(attr_rc);
    const int TW = 1 << tw_log2, TH = TBM >> tw_log2;
    TmaGeom g;
    g.tw_log2 = tw_log2;
    g.tiles_x = (p.Wo + TW - 1) / TW;
    g.tiles_y = (p.Ho + MT * TH - 1) / (MT * TH);
    g.n_tiles = (p.Cout + BNW - 1) / BNW;
    g.num_work = g.tiles_x * g.tiles_y * p.B * g.n_tiles;
    // input row of output row ho and tap dy: S ho + oy0 + dy = S (ho + off) + par, par = (oy0 + dy) mod S; the taps of one
    // row parity share one box, starting at the smallest off, and lie (off - that) rows further into it
    const int S = v.in_stride;
    g.nbox = 0;
    for (int dy = 0; dy < v.kh; ++dy) {
        const int par = (v.oy0 + dy) & (S - 1), off = (v.oy0 + dy - par) / S;
        int i = 0;
        while (i < g.nbox && g.box_py[i] != par) ++i;
        if (i == g.nbox) { g.box_py[i] = par; g.box_y[i] = off; g.box_ntap[i] = 0; ++g.nbox; }
        ++g.box_ntap[i];
    }
    for (int i = 0, t = 0; i < g.nbox; ++i) {
        g.box_tap0[i] = t;
        int last = g.box_y[i];
        for (int dy = 0; dy < v.kh; ++dy) {
            const int par = (v.oy0 + dy) & (S - 1), off = (v.oy0 + dy - par) / S;
            if (par != g.box_py[i]) continue;
            g.tap_dy[t] = dy;
            g.tap_shift[t++] = off - g.box_y[i];
            last = off;
        }
        g.box_rows[i] = MT * TH + last - g.box_y[i];
    }
    for (int dx = 0; dx < v.kw; ++dx) {
        g.col_px[dx] = (v.ox0 + dx) & (S - 1);
        g.col_x[dx] = (v.ox0 + dx - g.col_px[dx]) / S;
    }
    int max_rows = 0, max_taps = 0;
    for (int i = 0; i < g.nbox; ++i) {
        max_rows = g.box_rows[i] > max_rows ? g.box_rows[i] : max_rows;
        max_taps = g.box_ntap[i] > max_taps ? g.box_ntap[i] : max_taps;
    }
    g.a_bytes = (max_rows * TW * 128 + 1023) / 1024 * 1024;
    g.stage_bytes = g.a_bytes + max_taps * BNW * 128;
    const int fixed = 1024 + 1024;                          // 1024 alignment slack + 1024 barrier block
    g.stages = (TMA_SMEM_MAX - fixed) / g.stage_bytes;
    if (g.stages > TMA_MAX_STAGES) g.stages = TMA_MAX_STAGES;
    if (g.stages < 2) {
        set_error("conv_tma: stage of %d bytes does not fit twice in shared memory", g.stage_bytes);
        return SCSFM_ERR_ARG;
    }
    g.dbg = p.debug;
    // split-accumulate passes: raw x raw, then lo(activations) x raw(weights), then raw(activations) x lo(weights)
    g.npass = 1; g.a_lo = 0; g.w_lo = 0;
    if (p.in_lo != nullptr) { g.a_lo |= 1 << g.npass; ++g.npass; }
    if (p.w_lo != nullptr) { g.w_lo |= 1 << g.npass; ++g.npass; }
    {
        const int chunks = (p.Cin + TBK - 1) / TBK;
        const int mma_per_chunk = v.kw * g.npass * v.kh * (TBK / 8);
        // split mode: chains of ~100 wgmma; plain TF32 (operand rounding 3e-4 dominates): one chain per tile
        g.cpg = g.npass > 1 ? (96 + mma_per_chunk - 1) / mma_per_chunk : chunks;
        if (g.cpg < 1) g.cpg = 1;
    }
    const size_t smem = (size_t)fixed + (size_t)g.stages * g.stage_bytes;
    TmaMaps maps;
    memset(&maps, 0, sizeof(maps));
    for (int lo = 0; lo < 2; ++lo) {
        const float* base = lo ? p.in_lo : p.in;
        if (base == nullptr) continue;
        for (int i = 0; i < g.nbox; ++i)
            for (int dx = 0; dx < v.kw; ++dx) {
                // activations [B][Hi][Wi][Cin] (Cin contiguous), seen through the (py, px) parity view at stride 2: every
                // S-th row and column from row py, column px; box = 32 channels x TW x box_rows x 1, 128B swizzle
                const int py = g.box_py[i], px = g.col_px[dx];
                CUtensorMap& m = (lo ? maps.a_lo : maps.a)[py * 2 + px];
                const cuuint64_t gdim[4] = {(cuuint64_t)p.Cin, (cuuint64_t)((p.Wi - px + S - 1) / S), (cuuint64_t)((p.Hi - py + S - 1) / S),
                                            (cuuint64_t)p.B};
                const cuuint64_t gstride[3] = {(cuuint64_t)S * p.Cin * 4, (cuuint64_t)S * p.Wi * p.Cin * 4, (cuuint64_t)p.Hi * p.Wi * p.Cin * 4};
                const cuuint32_t box[4] = {(cuuint32_t)TBK, (cuuint32_t)TW, (cuuint32_t)g.box_rows[i], 1};
                const cuuint32_t estr[4] = {1, 1, 1, 1};
                const CUresult r = encode_tiled(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(base + ((size_t)py * p.Wi + px) * p.Cin),
                                                gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                                CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
                if (r != CUDA_SUCCESS) {
                    set_error("cuTensorMapEncodeTiled(activations %d x %d x %d x %d, view %d/%d) failed with CUresult %d", p.B, p.Hi, p.Wi,
                              p.Cin, py, px, (int)r);
                    return SCSFM_ERR_CUDA;
                }
            }
    }
    for (int lo = 0; lo < 2; ++lo) {
        const float* base = lo ? p.w_lo : p.w;
        CUtensorMap& wmap_ = lo ? maps.w_lo : maps.w;
        if (base == nullptr) continue;
        // weights [Cout][K] (K contiguous); box = 32 columns x BNW rows (rows past Cout are zero-filled)
        const int K = v.kh * v.kw * p.Cin;
        const cuuint64_t gdim[2] = {(cuuint64_t)K, (cuuint64_t)p.Cout};
        const cuuint64_t gstride[1] = {(cuuint64_t)K * sizeof(float)};
        const cuuint32_t box[2] = {(cuuint32_t)TBK, (cuuint32_t)BNW};
        const cuuint32_t estr[2] = {1, 1};
        const CUresult r = encode_tiled(&wmap_, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), gdim, gstride, box, estr,
                                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) {
            set_error("cuTensorMapEncodeTiled(weights %d x %d) failed with CUresult %d", p.Cout, K, (int)r);
            return SCSFM_ERR_CUDA;
        }
    }
    int ctas = sm_count();
    if (ctas > g.num_work) ctas = g.num_work;
    conv_tma_kernel<BNW, MT><<<ctas, TMA_THREADS, smem, st>>>(p, v, g, maps);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

int launch_conv_tma(const ScsfmConv& p, const TcView& v, cudaStream_t st) {
    const int N = p.Cout;
    // weight rows kept in shared memory (= wgmma N): the smallest of 16/32/64/128 covering Cout (Cout > 128: 128-row tiles)
    int bnw;
    if (N <= 16) bnw = 16;
    else if (N <= 32) bnw = 32;
    else if (N <= 64) bnw = 64;
    else bnw = 128;
    // Pixel tile: 1 or 2 stacked 128-pixel sub-tiles, TW = 8 or 16: minimise the number of waves of the persistent CTAs,
    // then the padded area (halo rows included), then prefer the smaller tile.  256-pixel tiles hold 2 x BNW / 2
    // accumulators plus as many chain registers per consumer thread, so they are built for BNW <= 64 only (the heuristic
    // picks them for Cout <= 64; forced on a wider layer they run over 64-channel Cout tiles).
    const int nsm = sm_count();
    const long nt = (N + TBM - 1) / TBM;
    int best_mt = 1, best_tw = 4;
    double best_cost = -1.0;
    for (int mt = 1; mt <= (bnw <= 64 ? 2 : 1); ++mt)
        for (int twl = 4; twl >= 3; --twl) {
            const int tw = 1 << twl, th = mt * (TBM >> twl);
            const long ty = (p.Ho + th - 1) / th, tx = (p.Wo + tw - 1) / tw;
            const long work = ty * tx * p.B * nt;
            const long waves = (work + nsm - 1) / nsm;
            const double halo = (double)(v.kh - 1) / v.in_stride;          // extra rows per tile, in output rows
            const double area = (double)ty * (th + halo) * (double)(tx * tw) / ((double)p.Ho * p.Wo);     // >= 1
            const double cost = (double)waves + 0.05 * area + 0.01 * mt;
            if (best_cost < 0 || cost < best_cost) { best_cost = cost; best_mt = mt; best_tw = twl; }
        }
    if (tune_mt(p)) best_mt = tune_mt(p);
    if (tune_tw(p)) best_tw = tune_tw(p);
    if (tune_bn(p)) bnw = tune_bn(p) < bnw ? bnw : tune_bn(p);       // never fewer rows than the Cout tile needs
    if (best_mt == 2 && bnw > 64) {
        // a forced 256-pixel tile on a wide layer: it runs over Cout tiles of 64 channels (the register budget of its
        // 2 x 64-row accumulators); a forced wider weight tile cannot be combined with it
        if (tune_bn(p) > 64) {
            set_error("conv_tma: 256-pixel tiles take weight tiles of at most 64 rows (%d requested)", tune_bn(p));
            return SCSFM_ERR_ARG;
        }
        bnw = 64;
    }
    if (best_mt == 1) {
        switch (bnw) {
            case 16: return launch_tma_cfg<16, 1>(p, v, best_tw, st);
            case 32: return launch_tma_cfg<32, 1>(p, v, best_tw, st);
            case 64: return launch_tma_cfg<64, 1>(p, v, best_tw, st);
            default: return launch_tma_cfg<128, 1>(p, v, best_tw, st);
        }
    }
    switch (bnw) {
        case 16: return launch_tma_cfg<16, 2>(p, v, best_tw, st);
        case 32: return launch_tma_cfg<32, 2>(p, v, best_tw, st);
        default: return launch_tma_cfg<64, 2>(p, v, best_tw, st);
    }
}

}  // namespace scsfm

