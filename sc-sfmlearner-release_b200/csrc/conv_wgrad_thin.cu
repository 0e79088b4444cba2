// Weight gradient of the thin 3x3 decoder layers (Cout = 16, Cin in {16, 32}: SC-SfMLearner's upconv(0,0) / upconv(0,1) at
// half / full resolution) on the fp32 FMA pipes.
//
// Why not the tensor cores: with pixels as the K dimension (8 per tf32 MMA) and only 16 output channels per MMA, the
// instruction count -- not the math -- bounds these layers, and the split-accumulate passes read four tensors
// (x, lo(x), dout, lo(dout)).  The layer is only 11.8 GFLOP: plain fp32 FMAs need neither the low
// parts (half the bytes) nor the passes, and are exact per product.
//
//   dW[o][dy][dx][c] += sum over the pixels (b, y, x)   dout[b, y, x, o] * in[b, y + dy - 1, x + dx - 1, c]
//
//  * a CTA walks a contiguous range of TH x TW pixel tiles; a tile's input patch with its one-pixel halo
//    ((TH+2) x (TW+2) x Cin, zero-filled or mirrored at the image border) and its dout tile are staged in shared memory by
//    16-byte cp.async, double-buffered (the next tile lands while this one is multiplied);
//  * thread = (pixel set s, tap row dy, channel group cg, output group og): it owns the 4 (o) x 4 (c) x 3 (dx) = 48 sums
//    of its (dy, cg, og) and walks the rows s, s + NSETS, .. of the tile left to right with a sliding three-pixel window:
//    per pixel ONE new float4 of x and one float4 of dout feed 48 FMAs.  The eight lanes of a quarter warp share dy and the
//    pixel, so every shared-memory read is a broadcast of <= 64 contiguous bytes;
//  * sums are kept per tile and added into the thread's totals after every tile (short fp32 chains), the NSETS pixel sets
//    are added up through shared memory and one partial dW per CTA goes out with red.global.add.v4.f32.
#include "conv_tc.cuh"

namespace scsfm {

template <int CIN, int COUT, int TW_>
struct ThinCfg {
    static constexpr int TH = 8, TW = TW_;
    static constexpr int OG = COUT / 4, CG = CIN / 4;
    static constexpr int ROLES = 3 * CG * OG;               // (dy, cg, og)
    static constexpr int NSETS = 4;                         // pixel sets: rows s, s + 4 of a tile
    static constexpr int THREADS = ROLES * NSETS;
    static constexpr int XROW = (TW + 2) * CIN;             // floats per halo row
    static constexpr int X_FLOATS = (TH + 2) * XROW;
    static constexpr int D_FLOATS = TH * TW * COUT;
    static constexpr int BUF_FLOATS = X_FLOATS + D_FLOATS;
    static constexpr int RED_FLOATS = (NSETS - 1) * 48 * ROLES;
    static constexpr size_t SMEM = 2 * (size_t)BUF_FLOATS * 4;
    static_assert(RED_FLOATS <= 2 * BUF_FLOATS, "the cross-set reduction reuses the tile buffers");
    static_assert(TW % 8 == 0 && TH % NSETS == 0 && ROLES % 8 == 0, "tile / role shape");
};

__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <int CIN, int COUT, int TW, int MINB>
__global__ void __launch_bounds__(ThinCfg<CIN, COUT, TW>::THREADS, MINB)
conv_wgrad_thin_kernel(ScsfmConv p, int tiles_x, int tiles_y, int tiles_total, int tiles_per_cta) {
    using Cfg = ThinCfg<CIN, COUT, TW>;
    constexpr int TH = Cfg::TH, THREADS = Cfg::THREADS, C4 = CIN / 4, O4 = COUT / 4;
    extern __shared__ __align__(16) float smem[];           // indexed (never turned into a generic pointer): the reads stay LDS.128

    const int tid = threadIdx.x;
    const int set = tid / Cfg::ROLES, role = tid - set * Cfg::ROLES;
    const int dy = role / (Cfg::CG * Cfg::OG), cg = (role / Cfg::OG) % Cfg::CG, og = role % Cfg::OG;
    const int H = p.Ho, W = p.Wo;                            // 3x3, stride 1, pad 1: input and output planes coincide
    const bool reflect = p.pad_mode == PADMODE_REFLECT;
    const int t_begin = blockIdx.x * tiles_per_cta, t_end = min(tiles_total, t_begin + tiles_per_cta);
    if (t_begin >= t_end) return;

    auto load_tile = [&](int t, int boff) {
        int q = t;
        const int tx = q % tiles_x; q /= tiles_x;
        const int ty = q % tiles_y;
        const int b = q / tiles_y;
        const int y0 = ty * TH, x0 = tx * TW;
        const uint32_t sx = tc::smem_u32(smem) + (uint32_t)boff * 4u, sd = sx + (uint32_t)Cfg::X_FLOATS * 4u;
        // input patch with halo: [row][column][CIN]
        constexpr int XCH = (TH + 2) * (TW + 2) * C4;
        for (int i = tid; i < XCH; i += THREADS) {
            const int ch = i % C4, px = i / C4;
            const int cx = px % (TW + 2), r = px / (TW + 2);
            int hy = y0 - 1 + r, hx = x0 - 1 + cx;
            bool ok;
            if (reflect) {
                // rows / columns further out than the mirrored ring only meet dout = 0 (partial tiles): zero-fill
                ok = hy <= H && hx <= W;
                hy = reflect_index(hy, H);
                hx = reflect_index(hx, W);
            } else ok = (unsigned)hy < (unsigned)H && (unsigned)hx < (unsigned)W;
            const float* src = ok ? p.in + (((size_t)b * H + hy) * W + hx) * CIN + 4 * ch : p.in;
            tc::cp_async_16(sx + (uint32_t)i * 16u, src, ok ? 16u : 0u);
        }
        // dout tile: [row][column][COUT], zero outside the image
        constexpr int DCH = TH * TW * O4;
        for (int i = tid; i < DCH; i += THREADS) {
            const int ch = i % O4, px = i / O4;
            const int xx = px % TW, r = px / TW;
            const int y = y0 + r, x = x0 + xx;
            const bool ok = y < H && x < W;
            const float* src = ok ? p.dout + (((size_t)b * H + y) * W + x) * COUT + 4 * ch : p.dout;
            tc::cp_async_16(sd + (uint32_t)i * 16u, src, ok ? 16u : 0u);
        }
        cp_async_commit();
    };

    float acc[3][4][4];
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[a][i][j] = 0.f;

    load_tile(t_begin, 0);
    for (int t = t_begin; t < t_end; ++t) {
        const int boff = ((t - t_begin) & 1) * Cfg::BUF_FLOATS;
        if (t + 1 < t_end) {
            load_tile(t + 1, Cfg::BUF_FLOATS - boff);
            cp_async_wait<1>();
        } else cp_async_wait<0>();
        __syncthreads();

        float ta[3][4][4];
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) ta[a][i][j] = 0.f;
#pragma unroll 1
        for (int r = set; r < TH; r += Cfg::NSETS) {
            const int xrow = boff + (r + dy) * Cfg::XROW + 4 * cg;                     // float index; pixel stride CIN
            const int drow = boff + Cfg::X_FLOATS + r * TW * COUT + 4 * og;            // pixel stride COUT
            float4 w0 = *reinterpret_cast<const float4*>(smem + xrow), w1 = *reinterpret_cast<const float4*>(smem + xrow + CIN);
#pragma unroll 1
            for (int xo = 0; xo < TW; xo += 8) {
#pragma unroll
                for (int xi = 0; xi < 8; ++xi) {
                    const int xx = xo + xi;
                    const float4 w2 = *reinterpret_cast<const float4*>(smem + xrow + (xx + 2) * CIN);
                    const float4 d = *reinterpret_cast<const float4*>(smem + drow + xx * COUT);
                    const float dv[4] = {d.x, d.y, d.z, d.w};
                    const float wa[3][4] = {{w0.x, w0.y, w0.z, w0.w}, {w1.x, w1.y, w1.z, w1.w}, {w2.x, w2.y, w2.z, w2.w}};
#pragma unroll
                    for (int a = 0; a < 3; ++a)
#pragma unroll
                        for (int i = 0; i < 4; ++i)
#pragma unroll
                            for (int j = 0; j < 4; ++j) ta[a][i][j] = fmaf(dv[i], wa[a][j], ta[a][i][j]);
                    w0 = w1;
                    w1 = w2;
                }
            }
        }
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[a][i][j] += ta[a][i][j];
        __syncthreads();                     // every thread is done with buf before the tile after next lands in it
    }

    // add up the pixel sets (shared memory, [set - 1][k][role]: consecutive lanes -> consecutive words), then one partial dW per CTA
    float* red = smem;
    if (set > 0) {
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) red[((set - 1) * 48 + (a * 16 + i * 4 + j)) * Cfg::ROLES + role] = acc[a][i][j];
    }
    __syncthreads();
    if (set == 0) {
#pragma unroll 1
        for (int s = 0; s < Cfg::NSETS - 1; ++s)
#pragma unroll
            for (int a = 0; a < 3; ++a)
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc[a][i][j] += red[(s * 48 + (a * 16 + i * 4 + j)) * Cfg::ROLES + role];
        const int Mtot = 9 * CIN;
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                float* dst = p.dw + (size_t)(4 * og + i) * Mtot + (size_t)(dy * 3 + a) * CIN + 4 * cg;
                asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(acc[a][i][0]), "f"(acc[a][i][1]), "f"(acc[a][i][2]),
                             "f"(acc[a][i][3])
                             : "memory");
            }
    }
}

bool conv_wgrad_thin_eligible(const ScsfmConv& p) {
    return p.kh == 3 && p.kw == 3 && p.stride == 1 && p.pad == 1 && (p.pad_mode == PADMODE_ZERO || p.pad_mode == PADMODE_REFLECT) &&
           p.Ho == p.Hi && p.Wo == p.Wi && p.Ho >= 3 && p.Wo >= 3 && p.Cout == 16 && (p.Cin == 16 || p.Cin == 32);
}

template <int CIN, int COUT, int TW, int MINB>
static int launch_thin(const ScsfmConv& p, cudaStream_t st) {
    using Cfg = ThinCfg<CIN, COUT, TW>;
    static const cudaError_t attr_rc =
        cudaFuncSetAttribute(conv_wgrad_thin_kernel<CIN, COUT, TW, MINB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM);
    SCSFM_CHECK_CUDA(attr_rc);
    const int tiles_x = (p.Wo + TW - 1) / TW, tiles_y = (p.Ho + Cfg::TH - 1) / Cfg::TH;
    const long long total = (long long)p.B * tiles_y * tiles_x;
    SCSFM_CHECK_ARG(total < (1LL << 31), "conv_wgrad_thin: too many tiles");
    int nsm = 132;
    {
        int dev = 0, v = 0;
        if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && v > 0) nsm = v;
    }
    int ctas = nsm * MINB;
    if (ctas > total) ctas = (int)total;
    const int per = (int)((total + ctas - 1) / ctas);
    ctas = (int)((total + per - 1) / per);
    conv_wgrad_thin_kernel<CIN, COUT, TW, MINB><<<ctas, Cfg::THREADS, Cfg::SMEM, st>>>(p, tiles_x, tiles_y, (int)total, per);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

int launch_conv_wgrad_thin(const ScsfmConv& p, cudaStream_t st) {
    if (!conv_wgrad_thin_eligible(p)) {
        set_error("conv_wgrad_thin: needs a 3x3 stride-1 pad-1 layer with Cout = 16 and Cin in {16, 32} (got %d -> %d, k%d s%d p%d)", p.Cin,
                  p.Cout, p.kh, p.stride, p.pad);
        return SCSFM_ERR_ARG;
    }
    if (p.Cin == 16) return launch_thin<16, 16, 32, 2>(p, st);
    return launch_thin<32, 16, 16, 1>(p, st);
}

}  // namespace scsfm
