// Forward of the 7x7 stride-2 pad-3 stems (Cin = 4 or 8 after channel padding, Cout = 64) on the tensor cores:
//
//   D[pixels (M = 64 per wgmma), Cout] = im2col(x)[pixels, K = (dy, dx, c)] x W[Cout, K]^T
//
// Why a kernel of its own: a kernel row of the stem is only 28 or 56 K values and its input has 4 or 8 channels, so the
// 32-channel 128B-swizzled boxes of conv_tma.cu do not fit it, and the cp.async gather kernel fetches every input pixel
// ~12 times (49 taps / stride^2), re-stages the weights for every 64-pixel tile and, in split mode, gathers lo(x) as well.
//  * persistent CTAs, one per SM, walk 8 x 16-pixel output tiles of one image.  Per tile the producer issues ONE
//    unswizzled TMA box of all 2 * 8 + 5 = 21 input rows it needs (out-of-bounds rows / columns zero-filled: the zero
//    padding); every tap is an address offset into it, so each input byte crosses L2 -> SMEM 21 / 8 ~ 2.6 times;
//  * the im2col operand is the wgmma A operand from registers: for one kernel row dy, (dx, c) is contiguous in an NHWC
//    input row, which no shared-memory descriptor layout for 32-bit wgmma operands expresses;
//  * the weights stay resident in shared memory for the CTA's life (128B-swizzled K-major B operand, loaded once);
//  * split mode (tf32x3): lo(x) is computed from the A fragment (tf32_lo: bit-identical to the stored low part, which is
//    never read), W and lo(W) are stacked on the N side: a CTA owns 32 output channels, B rows [0, 32) hold W and [32, 64)
//    lo(W), so the two wgmma lo(x) x [W | lo(W)] and x x [W | lo(W)] give all four products (columns c and 32 + c are
//    added in the epilogue).  A CTA pair covers the 64 channels of a tile, reading its box twice.  Plain TF32: one
//    product, all 64 channels per CTA;
//  * accumulation: one chain of wgmma per kernel row (7 or 4 K8 slices; split mode low parts first), started from zero
//    and added into the running sum in fp32 registers (the tensor core truncates as it accumulates);
//  * epilogue from registers (NHWC), that of conv_tma.cu: bias or eval-mode BatchNorm (bn_scale / bn_shift), residual
//    addend, activation, TF32 rounding, low part, BatchNorm sums.  The choice of kernel does not depend on the epilogue, so
//    a fused eval-mode layer stays bitwise the plain convolution followed by bn_apply.
//
// Operand geometry.  The box is viewed as rows of 32-byte units: output pixel px of a tile row owns unit px, and K8 slice
// j of a kernel row reads unit px + u(j) of box b(j):
//   Cin 4: one box of input columns 2 x0 - 3 .. 2 x0 + 34 (38 columns = 19 units of two columns x 4 channels); slice j
//          holds taps dx = 2j, 2j + 1 (u = j).  Slice 3 holds dx = 6 and a phantom dx = 7: its input column lies inside
//          the box (finite values, zero where outside the image) and its weights are zero;
//   Cin 8: the input seen through its column-parity views (column stride doubled): box 0 the odd columns from view
//          column x0 - 2, box 1 the even columns from x0 - 1, 19 units of one column x 8 channels each; slice j = dx
//          reads box j % 2 at u = j / 2.
// Inside a slice K is permuted so that the two values of a thread's A fragment row are adjacent: k = q and k = q + 4
// (q = lane % 4) are the unit's words 2q and 2q + 1, read with ONE ld.shared.v2; the resident weights are written in the
// same order.  Bank conflicts: a 64-bit load is served per half-warp; lanes 0-15 (g = lane / 4 = 0..3, q = 0..3) read
// units px + u .. px + u + 3 of one box row at byte 8q: 128 consecutive bytes, i.e. all 32 banks once, for every slice,
// row and box.  Lanes 16-31 likewise.  Conflict-free by construction.
//
//   warps 0-7   two consumer warpgroups; warpgroup g owns tile rows 4g .. 4g + 3, warp w of it row 4g + w (16 pixels)
//   warp 8      lane 0: TMA producer; warps 9-11 only complete the producer warpgroup (setmaxnreg hands its registers over)
#include <string.h>

#include "conv_tc.cuh"

namespace scsfm {

constexpr int ST_TH = 8, ST_TW = 16;                     // output tile: 8 rows x 16 columns (two warpgroups of 64 pixels)
constexpr int ST_ROWS = 2 * ST_TH + 5;                   // input rows of a tile
constexpr int ST_UNITS = ST_TW + 3;                      // 32-byte units per box row
constexpr int ST_BOX = ST_ROWS * ST_UNITS * 32;          // bytes one box delivers
constexpr int ST_BOX_PITCH = (ST_BOX + 1023) / 1024 * 1024;
constexpr int ST_THREADS = 384;
constexpr int ST_PRODUCER_REGS = 40, ST_CONSUMER_REGS = 232;
constexpr int ST_MAX_STAGES = 8;
constexpr int ST_SMEM_MAX = 232448;

template <int CIN>
struct StemCfg {
    static constexpr int NSL = CIN == 8 ? 7 : 4;                 // K8 slices per kernel row
    static constexpr int NBOX = CIN == 8 ? 2 : 1;
    static constexpr int KCH = (7 * NSL + 3) / 4;                // 32-wide K chunks of the resident weights
    static constexpr int W_BYTES = KCH * 64 * 128;               // [chunk][64 rows][32 floats], 128B swizzle
    static constexpr int STAGE = NBOX * ST_BOX_PITCH;
};

struct StemGeom {
    int tiles_x, tiles_y, num_tiles;
    int stages;
};

__device__ __forceinline__ float2 ld_shared_v2(uint32_t saddr) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(saddr));
    return v;
}

// map0 / map1: Cin 4 the input and (unused) the input again; Cin 8 the odd-column and the even-column view
template <int CIN, bool SPLIT>
__global__ void __launch_bounds__(ST_THREADS, 1)
conv_stem_fwd_kernel(ScsfmConv p, StemGeom g, const __grid_constant__ CUtensorMap map0, const __grid_constant__ CUtensorMap map1) {
    using Cfg = StemCfg<CIN>;
    constexpr int NSL = Cfg::NSL;
    constexpr int CO = SPLIT ? 32 : 64;                          // output channels of this CTA
    constexpr int HALVES = SPLIT ? 2 : 1;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bar_full = reinterpret_cast<uint64_t*>(smem);
    uint64_t* bar_empty = bar_full + ST_MAX_STAGES;
    const uint32_t wsm = tc::smem_u32(smem + 1024);
    const uint32_t ring = wsm + (uint32_t)Cfg::W_BYTES;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int n0 = (blockIdx.x % HALVES) * CO;
    const int t_first = blockIdx.x / HALVES, t_step = gridDim.x / HALVES;

    if (tid == 0) {
        for (int s = 0; s < g.stages; ++s) {
            tc::mbar_init(bar_full + s, 1);
            tc::mbar_init(bar_empty + s, 256);
        }
        tc::fence_barrier_init();
    }
    // resident weights: B row n (Cout n0 + n; split mode: rows 32.. hold lo(W) of n0 + n - 32), K index k = 8 s + kq of
    // slice s = dy * NSL + j holds unit word kq < 4 ? 2 kq : 2 kq - 7 of the slice
    for (int i = tid; i < 64 * Cfg::KCH * 32; i += ST_THREADS) {
        const int n = i / (Cfg::KCH * 32), k = i - n * (Cfg::KCH * 32);
        const int s = k >> 3, kq = k & 7;
        const int dy = s / NSL, j = s - dy * NSL;
        const int word = kq < 4 ? 2 * kq : 2 * kq - 7;
        const int dx = CIN == 8 ? j : 2 * j + (word >> 2), c = CIN == 8 ? word : (word & 3);
        float v = 0.f;
        if (dy < 7 && dx < 7) {
            const float* src = SPLIT && n >= 32 ? p.w_lo : p.w;
            const int o = n0 + (SPLIT ? (n & 31) : n);
            v = __ldg(src + ((o * 7 + dy) * 7 + dx) * CIN + c);
        }
        tc::st_shared_f32(wsm + (uint32_t)((k >> 5) * 64 * 128) + tc::sw128_offset(n, k & 31), v);
    }
    tc::fence_proxy_async();                             // generic-proxy stores -> wgmma (async proxy) reads
    __syncthreads();

    if (warp >= 8) {
        // ------------------------------------------------------------------ TMA producer
        tc::setmaxnreg_dec<ST_PRODUCER_REGS>();
        if (warp == 8 && lane == 0) {
            tc::tma_prefetch_desc(&map0);
            if (CIN == 8) tc::tma_prefetch_desc(&map1);
            int s = 0;
            uint32_t ph = 0;
            for (int t = t_first; t < g.num_tiles; t += t_step) {
                const int tx = t % g.tiles_x, ty = (t / g.tiles_x) % g.tiles_y, b = t / (g.tiles_x * g.tiles_y);
                const int x0 = tx * ST_TW, iy = 2 * ty * ST_TH - 3;
                tc::mbar_wait(bar_empty + s, ph ^ 1);
                const uint32_t st = ring + (uint32_t)(s * Cfg::STAGE);
                tc::mbar_arrive_expect_tx(bar_full + s, (uint32_t)(Cfg::NBOX * ST_BOX));
                if (CIN == 8) {
                    tc::tma_load_4d(st, &map0, 0, x0 - 2, iy, b, bar_full + s);
                    tc::tma_load_4d(st + ST_BOX_PITCH, &map1, 0, x0 - 1, iy, b, bar_full + s);
                } else {
                    tc::tma_load_4d(st, &map0, 0, 2 * x0 - 3, iy, b, bar_full + s);
                }
                if (++s == g.stages) { s = 0; ph ^= 1; }
            }
        }
        __syncwarp();
    } else {
        // ------------------------------------------------------------------ consumer warpgroups (warps 0-7)
        tc::setmaxnreg_inc<ST_CONSUMER_REGS>();
        const int r = warp, gq = lane >> 2, tq = lane & 3;         // tile row r = 4 * warpgroup + warp in it
        const int groups = p.bn_groups > 0 ? p.bn_groups : 1;
        const int act = p.act & 0xff;
        const bool round = (p.act & ROUND_TF32) != 0;
        float acc[32], part[32];
        int s = 0;
        uint32_t ph = 0;
        for (int t = t_first; t < g.num_tiles; t += t_step) {
            const int tx = t % g.tiles_x, ty = (t / g.tiles_x) % g.tiles_y, b = t / (g.tiles_x * g.tiles_y);
            const int x0 = tx * ST_TW, y0 = ty * ST_TH;
#pragma unroll
            for (int i = 0; i < 32; ++i) acc[i] = 0.f;
            tc::mbar_wait(bar_full + s, ph);
            // this thread's unit of slice 0, kernel row 0 (box row 2 r + dy, unit gq; pixel gq + 8 is 8 units further)
            const uint32_t a_base = ring + (uint32_t)(s * Cfg::STAGE + (2 * r * ST_UNITS + gq) * 32 + 8 * tq);
#pragma unroll 1
            for (int dy = 0; dy < 7; ++dy) {
                uint32_t ahi[NSL][4], alo[NSL][4];
#pragma unroll
                for (int j = 0; j < NSL; ++j) {
                    const int box = CIN == 8 ? (j & 1) : 0, u = CIN == 8 ? (j >> 1) : j;
                    const uint32_t ad = a_base + (uint32_t)(box * ST_BOX_PITCH + (dy * ST_UNITS + u) * 32);
                    const float2 v0 = ld_shared_v2(ad), v1 = ld_shared_v2(ad + 8 * 32);
                    ahi[j][0] = __float_as_uint(v0.x);
                    ahi[j][1] = __float_as_uint(v1.x);
                    ahi[j][2] = __float_as_uint(v0.y);
                    ahi[j][3] = __float_as_uint(v1.y);
                    if (SPLIT) {
#pragma unroll
                        for (int e = 0; e < 4; ++e) alo[j][e] = __float_as_uint(tf32_lo(__uint_as_float(ahi[j][e])));
                    }
                }
                if (dy == 6) tc::mbar_arrive(bar_empty + s);    // the box has been read into registers
                tc::reg_fence(part);
                tc::wgmma_fence();
                if (SPLIT) {
#pragma unroll
                    for (int j = 0; j < NSL; ++j) {
                        const int sl = dy * NSL + j;
                        tc::wgmma_tf32_rs<64>(part, alo[j], tc::make_desc_sw128(wsm + (uint32_t)((sl >> 2) * 64 * 128 + (sl & 3) * 32)),
                                              j == 0 ? 0u : 1u);
                    }
                }
#pragma unroll
                for (int j = 0; j < NSL; ++j) {
                    const int sl = dy * NSL + j;
                    tc::wgmma_tf32_rs<64>(part, ahi[j], tc::make_desc_sw128(wsm + (uint32_t)((sl >> 2) * 64 * 128 + (sl & 3) * 32)),
                                          (SPLIT || j > 0) ? 1u : 0u);
                }
                tc::wgmma_commit();
                tc::wgmma_wait<0>();
                tc::reg_fence(part);
#pragma unroll
                for (int i = 0; i < 32; ++i) acc[i] += part[i];
            }
            if (++s == g.stages) { s = 0; ph ^= 1; }

            // ---- epilogue: fragment i holds channels 8 i + 2 tq (+1) of pixels gq and gq + 8 of tile row r; in split
            // mode channel c of the CTA is column c (x W) plus column 32 + c (x lo(W))
            float bs1[CO / 4], bs2[CO / 4];
#pragma unroll
            for (int i = 0; i < CO / 4; ++i) { bs1[i] = 0.f; bs2[i] = 0.f; }
            const int oy = y0 + r;
#pragma unroll
            for (int i = 0; i < CO / 8; ++i) {
                const int c = n0 + 8 * i + 2 * tq;
                float2 bb = make_float2(0.f, 0.f), sc = make_float2(0.f, 0.f), sh = make_float2(0.f, 0.f);
                if (p.bias != nullptr) bb = __ldg(reinterpret_cast<const float2*>(p.bias + c));
                if (p.bn_scale != nullptr) {
                    sc = __ldg(reinterpret_cast<const float2*>(p.bn_scale + c));
                    sh = __ldg(reinterpret_cast<const float2*>(p.bn_shift + c));
                }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int ox = x0 + gq + 8 * h;
                    if (oy >= p.Ho || ox >= p.Wo) continue;
                    float2 x = make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
                    if (SPLIT) { x.x += acc[16 + 4 * i + 2 * h]; x.y += acc[16 + 4 * i + 2 * h + 1]; }
                    const long long off = (((long long)b * p.Ho + oy) * p.Wo + ox) * 64 + c;
                    if (p.bias != nullptr) { x.x += bb.x; x.y += bb.y; }
                    if (p.bn_scale != nullptr) { x.x = fmaf(x.x, sc.x, sh.x); x.y = fmaf(x.y, sc.y, sh.y); }   // bn_apply's arithmetic
                    if (p.addend != nullptr) {
                        const float2 a = __ldg(reinterpret_cast<const float2*>(p.addend + off));
                        x.x += a.x; x.y += a.y;
                    }
                    if (act != ACT_NONE) { x.x = tc_act(x.x, act); x.y = tc_act(x.y, act); }
                    if (round) { x.x = tf32_round(x.x); x.y = tf32_round(x.y); }
                    *reinterpret_cast<float2*>(p.out + off) = x;
                    if (p.out_lo != nullptr) *reinterpret_cast<float2*>(p.out_lo + off) = make_float2(tf32_lo(x.x), tf32_lo(x.y));
                    bs1[2 * i] += x.x; bs1[2 * i + 1] += x.y;
                    bs2[2 * i] += x.x * x.x; bs2[2 * i + 1] += x.y * x.y;
                }
            }
            if (p.bn_sums != nullptr) {
                // lanes with the same tq own the same channels: butterfly over gq, then one fp64 atomic pair per (warp, channel)
#pragma unroll
                for (int o = 4; o < 32; o <<= 1) {
#pragma unroll
                    for (int i = 0; i < CO / 4; ++i) {
                        bs1[i] += __shfl_xor_sync(0xffffffffu, bs1[i], o);
                        bs2[i] += __shfl_xor_sync(0xffffffffu, bs2[i], o);
                    }
                }
                if (lane < 4) {
                    const int grp = b / (p.B / groups);
                    double* d = p.bn_sums + ((size_t)(t % SCSFM_BN_SLOTS) * groups + grp) * 64 * 2;
#pragma unroll
                    for (int i = 0; i < CO / 8; ++i) {
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int c = n0 + 8 * i + 2 * tq + e;
                            atomicAdd(d + 2 * c, (double)bs1[2 * i + e]);
                            atomicAdd(d + 2 * c + 1, (double)bs2[2 * i + e]);
                        }
                    }
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
bool conv_stem_eligible(const ScsfmConv& p) {
    if (p.tune & SCSFM_TUNE_NO_TMA) return false;
    if (p.stride != 2 || p.kh != 7 || p.kw != 7 || p.pad != 3 || p.pad_mode != PADMODE_ZERO) return false;
    if ((p.Cin != 4 && p.Cin != 8) || p.Cout != 64) return false;
    if (p.Cin == 8 && p.Wi < 2) return false;                       // the odd-column view needs one column
    if (p.in_lo != nullptr && p.w_lo == nullptr) return false;      // lo(x) x W alone is no mode of this kernel
    if (p.bn_sums && p.B % (p.bn_groups > 0 ? p.bn_groups : 1) != 0) return false;
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

static int encode_box(CUtensorMap* m, const float* base, const ScsfmConv& p, int view_cols, int col_step, int box_cols) {
    const cuuint64_t gdim[4] = {(cuuint64_t)p.Cin, (cuuint64_t)view_cols, (cuuint64_t)p.Hi, (cuuint64_t)p.B};
    const cuuint64_t gstride[3] = {(cuuint64_t)col_step * p.Cin * 4, (cuuint64_t)p.Wi * p.Cin * 4, (cuuint64_t)p.Hi * p.Wi * p.Cin * 4};
    const cuuint32_t box[4] = {(cuuint32_t)p.Cin, (cuuint32_t)box_cols, (cuuint32_t)ST_ROWS, 1};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    const CUresult r = encode_tiled(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(base), gdim, gstride, box, estr,
                                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled(stem input %d x %d x %d x %d) failed with CUresult %d", p.B, p.Hi, p.Wi, p.Cin, (int)r);
        return SCSFM_ERR_CUDA;
    }
    return SCSFM_OK;
}

template <int CIN, bool SPLIT>
static int launch_stem_cfg(const ScsfmConv& p, cudaStream_t st) {
    using Cfg = StemCfg<CIN>;
    static const cudaError_t attr_rc = cudaFuncSetAttribute(conv_stem_fwd_kernel<CIN, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, ST_SMEM_MAX);
    SCSFM_CHECK_CUDA(attr_rc);
    StemGeom g;
    g.tiles_x = (p.Wo + ST_TW - 1) / ST_TW;
    g.tiles_y = (p.Ho + ST_TH - 1) / ST_TH;
    g.num_tiles = g.tiles_x * g.tiles_y * p.B;
    const int fixed = 1024 + 1024 + Cfg::W_BYTES;              // alignment slack + barrier block + resident weights
    g.stages = (ST_SMEM_MAX - fixed) / Cfg::STAGE;
    if (g.stages > ST_MAX_STAGES) g.stages = ST_MAX_STAGES;
    CUtensorMap map0, map1;
    if (CIN == 8) {
        // odd input columns (view column v = input column 2 v + 1) and even ones (2 v)
        if (int rc = encode_box(&map0, p.in + CIN, p, p.Wi / 2, 2, ST_UNITS)) return rc;
        if (int rc = encode_box(&map1, p.in, p, (p.Wi + 1) / 2, 2, ST_UNITS)) return rc;
    } else {
        if (int rc = encode_box(&map0, p.in, p, p.Wi, 1, 2 * ST_UNITS)) return rc;
        map1 = map0;
    }
    constexpr int HALVES = SPLIT ? 2 : 1;
    int ctas = sm_count() / HALVES;
    if (ctas > g.num_tiles) ctas = g.num_tiles;
    const size_t smem = (size_t)fixed + (size_t)g.stages * Cfg::STAGE;
    conv_stem_fwd_kernel<CIN, SPLIT><<<ctas * HALVES, ST_THREADS, smem, st>>>(p, g, map0, map1);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

int launch_conv_stem_fwd(const ScsfmConv& p, cudaStream_t st) {
    const bool split = p.split || p.w_lo != nullptr;
    if (p.Cin == 8) return split ? launch_stem_cfg<8, true>(p, st) : launch_stem_cfg<8, false>(p, st);
    return split ? launch_stem_cfg<4, true>(p, st) : launch_stem_cfg<4, false>(p, st);
}

}  // namespace scsfm
