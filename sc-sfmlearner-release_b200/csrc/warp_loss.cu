// K8: fused pairwise photometric + geometry-consistency loss, forward and backward.
//
// One launch covers njobs pair-directions x B samples x image tiles.  Per tile the forward
//   pixel2cam -> pose transform -> cam2pixel2 -> bilinear sample (image + depth) -> clamp|T-Iw| ->
//   depth inconsistency -> auto-mask -> 3x3 SSIM on reflect-padded tiles -> (1-diff_depth) weight
//   -> masked sums
// replaces ~180 ATen ops of reference loss_functions.py:95-129 / inverse_warp.py:230-269 (SURVEY.md
// section 3.2).  Nothing but the input images/depths is read from HBM (32 B/pixel) and only
// per-job sums are written; the backward recomputes the forward per tile (44 B/pixel).
//
// HBM-bound kernel: CUDA cores, coalesced row loads, L1/L2-served gathers, shared-memory tile with
// halo for the SSIM stencil, warp-shuffle + one fp64 atomic per CTA for the reductions.
#include "warp_geom.cuh"

namespace scsfm {

constexpr int TW = 32;                 // tile width  (one warp = one 128-byte row segment)
constexpr int TH = 16;                 // tile height
constexpr int NTHREADS = 256;
constexpr int E1W = TW + 2, E1H = TH + 2, E1N = E1W * E1H;  // tile + 1-pixel halo
constexpr int E2W = TW + 4, E2H = TH + 4, E2N = E2W * E2H;  // tile + 2-pixel halo (backward)
constexpr int STATS_PER_JOB = 8;       // doubles: S_photo, N_mask, S_geo, scale_photo, scale_geo, photo, geo, -
constexpr float SSIM_C1 = 0.01f * 0.01f;
constexpr float SSIM_C2 = 0.03f * 0.03f;
constexpr double MIN_MASK_SUM = 10000.0;

struct PairJobs {
    ScsfmPairJob j[SCSFM_MAX_JOBS];
};

// ---------------------------------------------------------------------------------------------
// per-pixel photometric pieces shared by forward and backward
// ---------------------------------------------------------------------------------------------
struct SsimStats {
    float mux, muy, n1, n2, d1, d2;
};

// 3x3 box statistics around (ey, ex) of the smem tiles sx (target) / sy (warped), pitch `pitch`.
__device__ __forceinline__ SsimStats ssim_stats(const float* sx, const float* sy, int ey, int ex, int pitch) {
    float sumx = 0.f, sumy = 0.f, sxx = 0.f, syy = 0.f, sxy = 0.f;
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
        for (int dx = -1; dx <= 1; ++dx) {
            const float a = sx[(ey + dy) * pitch + ex + dx];
            const float b = sy[(ey + dy) * pitch + ex + dx];
            sumx += a;
            sumy += b;
            sxx += a * a;
            syy += b * b;
            sxy += a * b;
        }
    SsimStats s;
    const float k = 1.0f / 9.0f;
    s.mux = sumx * k;
    s.muy = sumy * k;
    const float vx = sxx * k - s.mux * s.mux;
    const float vy = syy * k - s.muy * s.muy;
    const float cxy = sxy * k - s.mux * s.muy;
    s.n1 = 2.0f * s.mux * s.muy + SSIM_C1;
    s.n2 = 2.0f * cxy + SSIM_C2;
    s.d1 = s.mux * s.mux + s.muy * s.muy + SSIM_C1;
    s.d2 = vx + vy + SSIM_C2;
    return s;
}

__device__ __forceinline__ float ssim_value(const SsimStats& s) {
    const float r = (1.0f - (s.n1 * s.n2) / (s.d1 * s.d2)) * 0.5f;
    return fminf(fmaxf(r, 0.0f), 1.0f);
}

__device__ __forceinline__ float clamp01(float v) { return fminf(fmaxf(v, 0.0f), 1.0f); }

__device__ __forceinline__ float depth_inconsistency(float Z, float Dp) {
    return clamp01(fabsf(Z - Dp) / (Z + Dp));
}

// ---------------------------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NTHREADS)
pairwise_fwd_kernel(PairJobs jobs, const float* __restrict__ Kmat, int B, int H, int W, int flags, int padding,
                    double* __restrict__ stats, ScsfmPairMaps maps) {
    __shared__ WarpCtx ctx;
    __shared__ float sT[3][E1N];
    __shared__ float sI[3][E1N];
    __shared__ float s_dd[TW * TH];
    __shared__ float s_m[TW * TH];
    __shared__ float s_red[3][NTHREADS / 32];

    const int job = blockIdx.z / B, b = blockIdx.z % B;
    const ScsfmPairJob& J = jobs.j[job];
    const int x0 = blockIdx.x * TW, y0 = blockIdx.y * TH;
    const int HW = H * W;
    const int tid = threadIdx.x;
    if (tid == 0) make_warp_ctx(Kmat + b * 9, J.pose + b * 6, ctx);
    __syncthreads();

    const float* tgt = J.tgt_img + (size_t)b * 3 * HW;
    const float* ref = J.ref_img + (size_t)b * 3 * HW;
    const int ts = J.tgt_shift, rs = J.ref_shift;
    const float* tdep = J.tgt_depth + (size_t)b * (H >> ts) * (W >> ts);
    const float* rdep = J.ref_depth + (size_t)b * (H >> rs) * (W >> rs);
    const bool automask = flags & SCSFM_WITH_AUTO_MASK;
    const bool write_maps = (job == 0);

    // phase A: warp every pixel of the tile + halo (halo pixels through the reflection of the SSIM pad)
    for (int e = tid; e < E1N; e += NTHREADS) {
        const int ey = e / E1W, ex = e - ey * E1W;
        const int gy = y0 + ey - 1, gx = x0 + ex - 1;
        float t0 = 0.f, t1 = 0.f, t2 = 0.f, w0 = 0.f, w1 = 0.f, w2 = 0.f;
        if (gy >= -1 && gy <= H && gx >= -1 && gx <= W) {
            const int py = reflect_index(gy, H), px = reflect_index(gx, W);
            const int p = py * W + px;
            t0 = __ldg(tgt + p);
            t1 = __ldg(tgt + HW + p);
            t2 = __ldg(tgt + 2 * HW + p);
            const float D = __ldg(tdep + (py >> ts) * (W >> ts) + (px >> ts));
            const Geom g = project_pixel(ctx, D, px, py, H, W, padding);
            w0 = blend(g, gather_taps(g, ref, W, 0));
            w1 = blend(g, gather_taps(g, ref + HW, W, 0));
            w2 = blend(g, gather_taps(g, ref + 2 * HW, W, 0));
            const bool interior = ey >= 1 && ey <= TH && ex >= 1 && ex <= TW && gy < H && gx < W;
            if (interior) {
                const float Dp = blend(g, gather_taps(g, rdep, W, rs));
                const float dd = depth_inconsistency(g.Z, Dp);
                float m = g.valid ? 1.0f : 0.0f;
                if (automask) {
                    const float l = (clamp01(fabsf(t0 - w0)) + clamp01(fabsf(t1 - w1)) + clamp01(fabsf(t2 - w2))) / 3.0f;
                    const float s = (fabsf(t0 - __ldg(ref + p)) + fabsf(t1 - __ldg(ref + HW + p)) +
                                     fabsf(t2 - __ldg(ref + 2 * HW + p))) / 3.0f;
                    m = (l < s) ? m : 0.0f;
                }
                const int ii = (ey - 1) * TW + (ex - 1);
                s_dd[ii] = dd;
                s_m[ii] = m;
                if (write_maps) {
                    const size_t q = (size_t)b * HW + p;
                    if (maps.warped) {
                        maps.warped[(size_t)b * 3 * HW + p] = w0;
                        maps.warped[(size_t)b * 3 * HW + HW + p] = w1;
                        maps.warped[(size_t)b * 3 * HW + 2 * HW + p] = w2;
                    }
                    if (maps.valid) maps.valid[q] = g.valid ? 1.0f : 0.0f;
                    if (maps.proj_depth) maps.proj_depth[q] = Dp;
                    if (maps.comp_depth) maps.comp_depth[q] = g.Z;
                    if (maps.mask) maps.mask[q] = m;
                    if (maps.diff_depth) maps.diff_depth[q] = dd;
                }
            }
        }
        sT[0][e] = t0; sT[1][e] = t1; sT[2][e] = t2;
        sI[0][e] = w0; sI[1][e] = w1; sI[2][e] = w2;
    }
    __syncthreads();

    // phase B: photometric map and masked sums for the tile interior
    float acc_photo = 0.f, acc_mask = 0.f, acc_geo = 0.f;
    for (int ii = tid; ii < TW * TH; ii += NTHREADS) {
        const int iy = ii / TW, ixx = ii - iy * TW;
        const int gy = y0 + iy, gx = x0 + ixx;
        if (gy >= H || gx >= W) continue;
        const int e = (iy + 1) * E1W + ixx + 1;
        const float dd = s_dd[ii], m = s_m[ii];
        const float wgt = (flags & SCSFM_WITH_MASK) ? (1.0f - dd) : 1.0f;
        float qsum = 0.f;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float q = clamp01(fabsf(sT[c][e] - sI[c][e]));
            if (flags & SCSFM_WITH_SSIM) {
                const SsimStats s = ssim_stats(sT[c], sI[c], iy + 1, ixx + 1, E1W);
                q = 0.15f * q + 0.85f * ssim_value(s);
            }
            q *= wgt;
            qsum += q;
            if (write_maps && maps.diff_img) maps.diff_img[((size_t)b * 3 + c) * HW + gy * W + gx] = q;
        }
        acc_photo += qsum * m;
        acc_mask += m;
        acc_geo += dd * m;
    }
    acc_photo = warp_sum(acc_photo);
    acc_mask = warp_sum(acc_mask);
    acc_geo = warp_sum(acc_geo);
    const int lane = tid & 31, wid = tid >> 5;
    if (lane == 0) { s_red[0][wid] = acc_photo; s_red[1][wid] = acc_mask; s_red[2][wid] = acc_geo; }
    __syncthreads();
    if (tid < 3) {
        float v = 0.f;
#pragma unroll
        for (int w = 0; w < NTHREADS / 32; ++w) v += s_red[tid][w];
        atomicAdd(stats + job * STATS_PER_JOB + tid, (double)v);
    }
}

// mean_on_mask (loss_functions.py:123-129) for both terms of every job + the sum over jobs
// (loss_functions.py:89-90).  Also stores the 1/sum(mask) scales the backward needs.
// grad_scale multiplies the stored backward scales only (exact-global data-parallel mode: the sums were all-reduced over the
// ranks, every rank back-propagates its own pixels' share of the GLOBAL loss and the averaged gradient all-reduce divides by
// the number of ranks again).
__global__ void pairwise_finalize_kernel(double* stats, int njobs, float* __restrict__ loss_out, double grad_scale) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    double photo = 0.0, geo = 0.0;
    for (int j = 0; j < njobs; ++j) {
        double* s = stats + j * STATS_PER_JOB;
        const double n3 = 3.0 * s[1], n1 = s[1];
        // the reference evaluates sum(diff*mask)/sum(mask) in fp32
        const double sp = n3 > MIN_MASK_SUM ? 1.0 / n3 : 0.0;
        const double sg = n1 > MIN_MASK_SUM ? 1.0 / n1 : 0.0;
        s[3] = sp * grad_scale;
        s[4] = sg * grad_scale;
        s[5] = s[0] * sp;
        s[6] = s[2] * sg;
        photo += (double)(float)s[5];
        geo += (double)(float)s[6];
    }
    loss_out[0] = (float)photo;
    loss_out[1] = (float)geo;
}

// ---------------------------------------------------------------------------------------------
// backward
// ---------------------------------------------------------------------------------------------
// Accumulates d(proj matrix) (12 values) of one pixel given d(X), d(Y), d(Zr).
struct GeomGrad {
    float gM[12];
    float gD;
};

// Back half shared with the stand-alone inverse_warp2 backward: given dL/dIw[3], dL/dDp (sampled
// depth) and dL/dZ (computed depth), push through the bilinear sampling (scatter into the source
// depth gradient), the projection and the back-projection.
__device__ __forceinline__ GeomGrad geometry_backward(const WarpCtx& ctx, const Geom& g, const float* __restrict__ ref,
                                                      const float* __restrict__ rdep, float* __restrict__ g_rdep,
                                                      int H, int W, int HW, int rs, float dI0, float dI1, float dI2,
                                                      float dDp, float dZ) {
    float gix = 0.f, giy = 0.f, a, bb;
    {
        const Taps t = gather_taps(g, ref, W, 0);
        blend_grad(g, t, a, bb);
        gix += dI0 * a; giy += dI0 * bb;
    }
    {
        const Taps t = gather_taps(g, ref + HW, W, 0);
        blend_grad(g, t, a, bb);
        gix += dI1 * a; giy += dI1 * bb;
    }
    {
        const Taps t = gather_taps(g, ref + 2 * HW, W, 0);
        blend_grad(g, t, a, bb);
        gix += dI2 * a; giy += dI2 * bb;
    }
    if (rdep != nullptr) {
        const Taps t = gather_taps(g, rdep, W, rs);
        blend_grad(g, t, a, bb);
        gix += dDp * a; giy += dDp * bb;
        if (g_rdep != nullptr && dDp != 0.0f) {
            const int ws = W >> rs;
            const float ax = 1.0f - g.fx, ay = 1.0f - g.fy;
            const int xa = g.x0 >> rs, xb = (g.x0 + 1) >> rs, ya = g.y0 >> rs, yb = (g.y0 + 1) >> rs;
            if (g.in_y0 && g.in_x0) red_add(g_rdep + ya * ws + xa, dDp * ax * ay);
            if (g.in_y0 && g.in_x1) red_add(g_rdep + ya * ws + xb, dDp * g.fx * ay);
            if (g.in_y1 && g.in_x0) red_add(g_rdep + yb * ws + xa, dDp * ax * g.fy);
            if (g.in_y1 && g.in_x1) red_add(g_rdep + yb * ws + xb, dDp * g.fx * g.fy);
        }
    }
    // ix = ((xn + 1) W - 1) / 2 ; xn = 2 (X/Z) / (W-1) - 1
    const float gxn = g.gradx ? gix * (0.5f * (float)W) : 0.0f;
    const float gyn = g.grady ? giy * (0.5f * (float)H) : 0.0f;
    const float kx = 2.0f / ((float)(W - 1) * g.Z), ky = 2.0f / ((float)(H - 1) * g.Z);
    const float gX = gxn * kx, gY = gyn * ky;
    float gZ = dZ - (gX * g.X + gY * g.Y) / g.Z;
    if (!(g.Zr >= 1e-3f)) gZ = 0.0f;   // clamp(min=1e-3) passes gradient only where Zr >= 1e-3
    GeomGrad r;
    r.gM[0] = gX * g.camx; r.gM[1] = gX * g.camy; r.gM[2] = gX * g.camz; r.gM[3] = gX;
    r.gM[4] = gY * g.camx; r.gM[5] = gY * g.camy; r.gM[6] = gY * g.camz; r.gM[7] = gY;
    r.gM[8] = gZ * g.camx; r.gM[9] = gZ * g.camy; r.gM[10] = gZ * g.camz; r.gM[11] = gZ;
    const float gcx = ctx.m[0] * gX + ctx.m[4] * gY + ctx.m[8] * gZ;
    const float gcy = ctx.m[1] * gX + ctx.m[5] * gY + ctx.m[9] * gZ;
    const float gcz = ctx.m[2] * gX + ctx.m[6] * gY + ctx.m[10] * gZ;
    r.gD = gcx * g.rayx + gcy * g.rayy + gcz * g.rayz;
    return r;
}

// Block-reduce 12 per-thread values and add them to dst[12] (fp64 atomics, one per CTA and entry).
__device__ __forceinline__ void reduce_gM(float (&acc)[12], float (*s_part)[12], double* __restrict__ dst) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < 12; ++k) {
        const float v = warp_sum(acc[k]);
        if (lane == 0) s_part[wid][k] = v;
    }
    __syncthreads();
    if (threadIdx.x < 12) {
        float v = 0.f;
#pragma unroll
        for (int w = 0; w < NTHREADS / 32; ++w) v += s_part[w][threadIdx.x];
        if (v != 0.0f) atomicAdd(dst + threadIdx.x, (double)v);
    }
}

__global__ void __launch_bounds__(NTHREADS)
pairwise_bwd_kernel(PairJobs jobs, const float* __restrict__ Kmat, int B, int H, int W, int flags, int padding,
                    const double* __restrict__ stats, double* __restrict__ gM_all,
                    const float* __restrict__ grad_out) {
    __shared__ WarpCtx ctx;
    __shared__ float sT[3][E2N];
    __shared__ float sI[3][E2N];
    __shared__ float s_gq[E1N];     // upstream gradient of the photometric map (same for 3 channels)
    __shared__ float s_w[E1N];      // (1 - diff_depth) weight or 1
    __shared__ float s_A[3][E1N];   // dL/d(mu_y)  of the SSIM window centred on the pixel
    __shared__ float s_B[3][E1N];   // 2 dL/d(E[yy])
    __shared__ float s_C[3][E1N];   // dL/d(E[xy])
    __shared__ float s_q[E1N];      // sum_c (0.15 l1 + 0.85 ssim) at the pixel (for the (1-dd) weight gradient)
    __shared__ float s_part[NTHREADS / 32][12];

    const int job = blockIdx.z / B, b = blockIdx.z % B;
    const ScsfmPairJob& J = jobs.j[job];
    const int x0 = blockIdx.x * TW, y0 = blockIdx.y * TH;
    const int HW = H * W;
    const int tid = threadIdx.x;
    if (tid == 0) make_warp_ctx(Kmat + b * 9, J.pose + b * 6, ctx);
    __syncthreads();

    const double* st = stats + job * STATS_PER_JOB;
    const float gphoto = grad_out[0] * (float)st[3];   // d(loss)/d(S_photo)
    const float ggeo = grad_out[1] * (float)st[4];     // d(loss)/d(S_geo)
    const float* tgt = J.tgt_img + (size_t)b * 3 * HW;
    const float* ref = J.ref_img + (size_t)b * 3 * HW;
    const int ts = J.tgt_shift, rs = J.ref_shift;
    const float* tdep = J.tgt_depth + (size_t)b * (H >> ts) * (W >> ts);
    const float* rdep = J.ref_depth + (size_t)b * (H >> rs) * (W >> rs);
    float* g_tdep = J.grad_tgt_depth ? J.grad_tgt_depth + (size_t)b * (H >> ts) * (W >> ts) : nullptr;
    float* g_rdep = J.grad_ref_depth ? J.grad_ref_depth + (size_t)b * (H >> rs) * (W >> rs) : nullptr;
    const bool automask = flags & SCSFM_WITH_AUTO_MASK;
    const bool with_ssim = flags & SCSFM_WITH_SSIM;
    const bool with_mask = flags & SCSFM_WITH_MASK;

    // phase A: target + warped image on the 2-halo tile; mask / weights on the 1-halo tile
    for (int e = tid; e < E2N; e += NTHREADS) {
        const int ey = e / E2W, ex = e - ey * E2W;
        const int gy = y0 + ey - 2, gx = x0 + ex - 2;
        float t0 = 0.f, t1 = 0.f, t2 = 0.f, w0 = 0.f, w1 = 0.f, w2 = 0.f;
        const bool in_e1 = ey >= 1 && ey <= TH + 2 && ex >= 1 && ex <= TW + 2;
        const int e1 = (ey - 1) * E1W + (ex - 1);
        float gq = 0.f, wgt = 1.f;
        if (gy >= -1 && gy <= H && gx >= -1 && gx <= W) {
            const int py = reflect_index(gy, H), px = reflect_index(gx, W);
            const int p = py * W + px;
            t0 = __ldg(tgt + p);
            t1 = __ldg(tgt + HW + p);
            t2 = __ldg(tgt + 2 * HW + p);
            const float D = __ldg(tdep + (py >> ts) * (W >> ts) + (px >> ts));
            const Geom g = project_pixel(ctx, D, px, py, H, W, padding);
            w0 = blend(g, gather_taps(g, ref, W, 0));
            w1 = blend(g, gather_taps(g, ref + HW, W, 0));
            w2 = blend(g, gather_taps(g, ref + 2 * HW, W, 0));
            if (in_e1 && gy >= 0 && gy < H && gx >= 0 && gx < W) {
                float m = g.valid ? 1.0f : 0.0f;
                if (automask) {
                    const float l = (clamp01(fabsf(t0 - w0)) + clamp01(fabsf(t1 - w1)) + clamp01(fabsf(t2 - w2))) / 3.0f;
                    const float s = (fabsf(t0 - __ldg(ref + p)) + fabsf(t1 - __ldg(ref + HW + p)) +
                                     fabsf(t2 - __ldg(ref + 2 * HW + p))) / 3.0f;
                    m = (l < s) ? m : 0.0f;
                }
                gq = gphoto * m;
                if (with_mask) {
                    const float Dp = blend(g, gather_taps(g, rdep, W, rs));
                    wgt = 1.0f - depth_inconsistency(g.Z, Dp);
                }
            }
        }
        sT[0][e] = t0; sT[1][e] = t1; sT[2][e] = t2;
        sI[0][e] = w0; sI[1][e] = w1; sI[2][e] = w2;
        if (in_e1) { s_gq[e1] = gq; s_w[e1] = wgt; }
    }
    __syncthreads();

    // phase B: per-pixel SSIM window coefficients on the 1-halo tile
    for (int e1 = tid; e1 < E1N; e1 += NTHREADS) {
        const int ey = e1 / E1W, ex = e1 - ey * E1W;
        const int e2 = (ey + 1) * E2W + ex + 1;
        const float gq = s_gq[e1], wgt = s_w[e1];
        float qs = 0.f;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float A = 0.f, Bc = 0.f, Cc = 0.f;
            float q = clamp01(fabsf(sT[c][e2] - sI[c][e2]));
            if (with_ssim) {
                const SsimStats s = ssim_stats(sT[c], sI[c], ey + 1, ex + 1, E2W);
                const float n = s.n1 * s.n2, d = s.d1 * s.d2;
                const float raw = (1.0f - n / d) * 0.5f;
                q = 0.15f * q + 0.85f * clamp01(raw);
                if (gq != 0.0f && raw >= 0.0f && raw <= 1.0f) {
                    const float gs = gq * 0.85f * wgt * (-0.5f);     // dL/d(n/d)
                    const float inv_d = 1.0f / d;
                    const float dn_dmu = 2.0f * s.mux * (s.n2 - s.n1);
                    const float dd_dmu = 2.0f * s.muy * (s.d2 - s.d1);
                    A = gs * (dn_dmu * d - n * dd_dmu) * inv_d * inv_d;
                    Bc = 2.0f * gs * (-n * s.d1) * inv_d * inv_d;
                    Cc = gs * 2.0f * s.n1 * inv_d;
                }
            }
            qs += q;
            s_A[c][e1] = A; s_B[c][e1] = Bc; s_C[c][e1] = Cc;
        }
        s_q[e1] = qs;
    }
    __syncthreads();

    // phase C: gradient of every interior pixel
    float acc[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) acc[k] = 0.f;
    for (int ii = tid; ii < TW * TH; ii += NTHREADS) {
        const int iy = ii / TW, ixx = ii - iy * TW;
        const int gy = y0 + iy, gx = x0 + ixx;
        if (gy >= H || gx >= W) continue;
        const int e1 = (iy + 1) * E1W + ixx + 1, e2 = (iy + 2) * E2W + ixx + 2;
        const int p = gy * W + gx;
        const float gq = s_gq[e1], wgt = s_w[e1];
        const float D = __ldg(tdep + (gy >> ts) * (W >> ts) + (gx >> ts));
        const Geom g = project_pixel(ctx, D, gx, gy, H, W, padding);
        const float Dp = blend(g, gather_taps(g, rdep, W, rs));
        // mask (needed for the geometry term; gq already carries it for the photometric term)
        float m = g.valid ? 1.0f : 0.0f;
        if (automask) {
            const float l = (clamp01(fabsf(sT[0][e2] - sI[0][e2])) + clamp01(fabsf(sT[1][e2] - sI[1][e2])) +
                             clamp01(fabsf(sT[2][e2] - sI[2][e2]))) / 3.0f;
            const float s = (fabsf(sT[0][e2] - __ldg(ref + p)) + fabsf(sT[1][e2] - __ldg(ref + HW + p)) +
                             fabsf(sT[2][e2] - __ldg(ref + 2 * HW + p))) / 3.0f;
            m = (l < s) ? m : 0.0f;
        }
        float dI[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            // L1 part: d clamp(|T - Iw|, 0, 1) / dIw = -sign(T - Iw) where |T - Iw| <= 1
            const float diff = sT[c][e2] - sI[c][e2];
            const float gl1 = gq * wgt * (with_ssim ? 0.15f : 1.0f);
            float v = (fabsf(diff) <= 1.0f) ? (diff > 0.f ? -gl1 : (diff < 0.f ? gl1 : 0.f)) : 0.f;
            if (with_ssim) {
                // transposed 3x3 stencil with the multiplicities of the reflection pad
                float sa = 0.f, sb = 0.f, sc = 0.f;
#pragma unroll
                for (int dy = -1; dy <= 1; ++dy) {
                    const int qy = gy + dy;
                    if (qy < 0 || qy >= H) continue;
                    const float my = 1.0f + ((gy == 1 && qy == 0) ? 1.0f : 0.0f) + ((gy == H - 2 && qy == H - 1) ? 1.0f : 0.0f);
#pragma unroll
                    for (int dx = -1; dx <= 1; ++dx) {
                        const int qx = gx + dx;
                        if (qx < 0 || qx >= W) continue;
                        const float mx = 1.0f + ((gx == 1 && qx == 0) ? 1.0f : 0.0f) + ((gx == W - 2 && qx == W - 1) ? 1.0f : 0.0f);
                        const int q1 = e1 + dy * E1W + dx;
                        const float mult = my * mx;
                        sa += mult * s_A[c][q1];
                        sb += mult * s_B[c][q1];
                        sc += mult * s_C[c][q1];
                    }
                }
                v += (sa + sI[c][e2] * sb + sT[c][e2] * sc) * (1.0f / 9.0f);
            }
            dI[c] = v;
        }
        // diff_depth = clamp(|Z - Dp| / (Z + Dp), 0, 1)
        float g_dd = ggeo * m;
        if (with_mask) g_dd -= gq * s_q[e1];
        float dZ = 0.f, dDp = 0.f;
        {
            const float u = g.Z - Dp, v = g.Z + Dp;
            const float r = fabsf(u) / v;
            if (r >= 0.0f && r <= 1.0f && g_dd != 0.0f) {
                const float sg = u > 0.f ? 1.f : (u < 0.f ? -1.f : 0.f);
                const float common = fabsf(u) / (v * v);
                dZ = g_dd * (sg / v - common);
                dDp = g_dd * (-sg / v - common);
            }
        }
        const GeomGrad gg = geometry_backward(ctx, g, ref, rdep, g_rdep, H, W, HW, rs, dI[0], dI[1], dI[2], dDp, dZ);
#pragma unroll
        for (int k = 0; k < 12; ++k) acc[k] += gg.gM[k];
        if (g_tdep != nullptr && gg.gD != 0.0f) red_add(g_tdep + (gy >> ts) * (W >> ts) + (gx >> ts), gg.gD);
    }
    reduce_gM(acc, s_part, gM_all + ((size_t)job * B + b) * 12);
}

// d(K [R|t]) -> d(pose): translation directly, rotation through d(Rx Ry Rz)/d(angle).
__device__ inline void pose_grad_from_gM(const float* __restrict__ K, const float* __restrict__ pose, const double* gM,
                                         float* __restrict__ gpose) {
    double gT[12];
    for (int k = 0; k < 3; ++k)
        for (int c = 0; c < 4; ++c) gT[k * 4 + c] = (double)K[0 * 3 + k] * gM[c] + (double)K[1 * 3 + k] * gM[4 + c] + (double)K[2 * 3 + k] * gM[8 + c];
    const double rx = pose[3], ry = pose[4], rz = pose[5];
    const double sx = sin(rx), cx = cos(rx), sy = sin(ry), cy = cos(ry), sz = sin(rz), cz = cos(rz);
    const double Rx[9] = {1, 0, 0, 0, cx, -sx, 0, sx, cx}, Ry[9] = {cy, 0, sy, 0, 1, 0, -sy, 0, cy}, Rz[9] = {cz, -sz, 0, sz, cz, 0, 0, 0, 1};
    const double dRx[9] = {0, 0, 0, 0, -sx, -cx, 0, cx, -sx}, dRy[9] = {-sy, 0, cy, 0, 0, 0, -cy, 0, -sy}, dRz[9] = {-sz, -cz, 0, cz, -sz, 0, 0, 0, 0};
    auto mm = [](const double* a, const double* b, double* o) {
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) o[i * 3 + j] = a[i * 3] * b[j] + a[i * 3 + 1] * b[3 + j] + a[i * 3 + 2] * b[6 + j];
    };
    auto dot = [&](const double* d) {
        double s = 0;
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) s += d[i * 3 + j] * gT[i * 4 + j];
        return s;
    };
    double t1[9], t2[9];
    mm(dRx, Ry, t1); mm(t1, Rz, t2); const double grx = dot(t2);
    mm(Rx, dRy, t1); mm(t1, Rz, t2); const double gry = dot(t2);
    mm(Rx, Ry, t1); mm(t1, dRz, t2); const double grz = dot(t2);
    // atomics: several jobs (scales) may share one pose gradient buffer
    atomicAdd(gpose + 0, (float)gT[3]);
    atomicAdd(gpose + 1, (float)gT[7]);
    atomicAdd(gpose + 2, (float)gT[11]);
    atomicAdd(gpose + 3, (float)grx);
    atomicAdd(gpose + 4, (float)gry);
    atomicAdd(gpose + 5, (float)grz);
}

__global__ void pose_grad_kernel(PairJobs jobs, int njobs, const float* __restrict__ Kmat, int B, const double* __restrict__ gM_all) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= njobs * B) return;
    const int job = i / B, b = i % B;
    if (jobs.j[job].grad_pose == nullptr) return;
    pose_grad_from_gM(Kmat + b * 9, jobs.j[job].pose + b * 6, gM_all + (size_t)i * 12, jobs.j[job].grad_pose + b * 6);
}

// ---------------------------------------------------------------------------------------------
// stand-alone inverse_warp2 (reference inverse_warp.py:230-269)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NTHREADS)
inverse_warp2_fwd_kernel(const float* __restrict__ img, const float* __restrict__ depth, const float* __restrict__ ref_depth,
                         const float* __restrict__ pose, const float* __restrict__ Kmat, int H, int W, int padding,
                         float* __restrict__ warped, float* __restrict__ valid, float* __restrict__ proj_depth,
                         float* __restrict__ comp_depth) {
    __shared__ WarpCtx ctx;
    const int b = blockIdx.y, HW = H * W;
    if (threadIdx.x == 0) make_warp_ctx(Kmat + b * 9, pose + b * 6, ctx);
    __syncthreads();
    const int p = blockIdx.x * NTHREADS + threadIdx.x;
    if (p >= HW) return;
    const int y = p / W, x = p - y * W;
    const Geom g = project_pixel(ctx, depth[(size_t)b * HW + p], x, y, H, W, padding);
    const float* ref = img + (size_t)b * 3 * HW;
    if (warped) {
        warped[(size_t)b * 3 * HW + p] = blend(g, gather_taps(g, ref, W, 0));
        warped[(size_t)b * 3 * HW + HW + p] = blend(g, gather_taps(g, ref + HW, W, 0));
        warped[(size_t)b * 3 * HW + 2 * HW + p] = blend(g, gather_taps(g, ref + 2 * HW, W, 0));
    }
    if (valid) valid[(size_t)b * HW + p] = g.valid ? 1.0f : 0.0f;
    if (proj_depth) proj_depth[(size_t)b * HW + p] = blend(g, gather_taps(g, ref_depth + (size_t)b * HW, W, 0));
    if (comp_depth) comp_depth[(size_t)b * HW + p] = g.Z;
}

__global__ void __launch_bounds__(NTHREADS)
inverse_warp2_bwd_kernel(const float* __restrict__ img, const float* __restrict__ depth, const float* __restrict__ ref_depth,
                         const float* __restrict__ pose, const float* __restrict__ Kmat, int H, int W, int padding,
                         const float* __restrict__ g_warped, const float* __restrict__ g_proj, const float* __restrict__ g_comp,
                         float* __restrict__ g_depth, float* __restrict__ g_ref_depth, double* __restrict__ gM_all) {
    __shared__ WarpCtx ctx;
    __shared__ float s_part[NTHREADS / 32][12];
    const int b = blockIdx.y, HW = H * W;
    if (threadIdx.x == 0) make_warp_ctx(Kmat + b * 9, pose + b * 6, ctx);
    __syncthreads();
    float acc[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) acc[k] = 0.f;
    const int p = blockIdx.x * NTHREADS + threadIdx.x;
    if (p < HW) {
        const int y = p / W, x = p - y * W;
        const Geom g = project_pixel(ctx, depth[(size_t)b * HW + p], x, y, H, W, padding);
        const float d0 = g_warped ? g_warped[(size_t)b * 3 * HW + p] : 0.f;
        const float d1 = g_warped ? g_warped[(size_t)b * 3 * HW + HW + p] : 0.f;
        const float d2 = g_warped ? g_warped[(size_t)b * 3 * HW + 2 * HW + p] : 0.f;
        const float dDp = g_proj ? g_proj[(size_t)b * HW + p] : 0.f;
        const float dZ = g_comp ? g_comp[(size_t)b * HW + p] : 0.f;
        const GeomGrad gg = geometry_backward(ctx, g, img + (size_t)b * 3 * HW, ref_depth + (size_t)b * HW,
                                              g_ref_depth ? g_ref_depth + (size_t)b * HW : nullptr, H, W, HW, 0, d0, d1, d2, dDp, dZ);
#pragma unroll
        for (int k = 0; k < 12; ++k) acc[k] = gg.gM[k];
        if (g_depth) red_add(g_depth + (size_t)b * HW + p, gg.gD);
    }
    reduce_gM(acc, s_part, gM_all + (size_t)b * 12);
}

__global__ void inverse_warp2_pose_grad_kernel(const float* __restrict__ pose, const float* __restrict__ Kmat, int B,
                                               const double* __restrict__ gM_all, float* __restrict__ g_pose) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    pose_grad_from_gM(Kmat + b * 9, pose + b * 6, gM_all + (size_t)b * 12, g_pose + b * 6);
}

// ---------------------------------------------------------------------------------------------
// intrinsics gradient (camera self-calibration), from the same d(K [R|t]) sums as the pose gradient
// ---------------------------------------------------------------------------------------------
// Entry (r, c) of d(loss)/dK for one (job, sample), in fp64.  Per pixel c_px = K^-1 (D pix) and P = M3 c_px + m4 with
// M = [M3 | m4] = K [R|t]; gM = sum_px dL/dP [c_px^T 1].  K enters twice (reference inverse_warp.py:253,258):
//   through M:     gM3 R^T + gm4 t^T
//   through K^-1:  -K^-T (dL/dK^-1) K^-T with dL/dK^-1 = M3^T sum_px dL/dP (D pix)^T = M3^T gM3 K^T,  i.e.  -K^-T R^T K^T gM3
// The two terms cancel to a large part (exactly at R = I, t = 0), hence fp64 throughout.  K^-1 is the general 3x3 inverse.
__device__ inline double intrinsics_grad_entry(const float* __restrict__ Kf, const float* __restrict__ pose, const double* gM,
                                               int r, int c) {
    double k[9];
    for (int i = 0; i < 9; ++i) k[i] = Kf[i];
    const double A = k[4] * k[8] - k[5] * k[7], Bc = k[5] * k[6] - k[3] * k[8], C = k[3] * k[7] - k[4] * k[6];
    const double inv = 1.0 / (k[0] * A + k[1] * Bc + k[2] * C);
    const double kinv[9] = {A * inv, (k[2] * k[7] - k[1] * k[8]) * inv, (k[1] * k[5] - k[2] * k[4]) * inv,
                            Bc * inv, (k[0] * k[8] - k[2] * k[6]) * inv, (k[2] * k[3] - k[0] * k[5]) * inv,
                            C * inv, (k[1] * k[6] - k[0] * k[7]) * inv, (k[0] * k[4] - k[1] * k[3]) * inv};
    const double sx = sin((double)pose[3]), cx = cos((double)pose[3]), sy = sin((double)pose[4]), cy = cos((double)pose[4]);
    const double sz = sin((double)pose[5]), cz = cos((double)pose[5]);
    const double R[9] = {cy * cz, -cy * sz, sy,
                         cx * sz + sx * sy * cz, cx * cz - sx * sy * sz, -sx * cy,
                         sx * sz - cx * sy * cz, sx * cz + cx * sy * sz, cx * cy};
    // through M = K [R|t]
    double through_m = gM[r * 4 + 3] * (double)pose[c];
    for (int j = 0; j < 3; ++j) through_m += gM[r * 4 + j] * R[c * 3 + j];
    // column c of K^T gM3, then of R^T K^T gM3, then entry r of K^-T R^T K^T gM3
    double a[3], bcol[3];
    for (int j = 0; j < 3; ++j) a[j] = k[0 * 3 + j] * gM[0 * 4 + c] + k[1 * 3 + j] * gM[1 * 4 + c] + k[2 * 3 + j] * gM[2 * 4 + c];
    for (int i = 0; i < 3; ++i) bcol[i] = R[0 * 3 + i] * a[0] + R[1 * 3 + i] * a[1] + R[2 * 3 + i] * a[2];
    const double through_kinv = kinv[0 * 3 + r] * bcol[0] + kinv[1 * 3 + r] * bcol[1] + kinv[2 * 3 + r] * bcol[2];
    return through_m - through_kinv;
}

// One thread per (sample, entry of K): sums the jobs in their order and adds the result into grad_K (no atomics: the chunks of
// one backward are launched one after the other on one stream).
__global__ void pairwise_intrinsics_grad_kernel(PairJobs jobs, int njobs, const float* __restrict__ Kmat, int B,
                                                const double* __restrict__ gM_all, float* __restrict__ grad_K) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * 9) return;
    const int b = i / 9, e = i - b * 9;
    double s = 0.0;
    for (int job = 0; job < njobs; ++job)
        s += intrinsics_grad_entry(Kmat + b * 9, jobs.j[job].pose + b * 6, gM_all + ((size_t)job * B + b) * 12, e / 3, e % 3);
    grad_K[i] += (float)s;
}

__global__ void inverse_warp2_intrinsics_grad_kernel(const float* __restrict__ pose, const float* __restrict__ Kmat, int B,
                                                     const double* __restrict__ gM_all, float* __restrict__ grad_K) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * 9) return;
    const int b = i / 9, e = i - b * 9;
    grad_K[i] += (float)intrinsics_grad_entry(Kmat + b * 9, pose + b * 6, gM_all + (size_t)b * 12, e / 3, e % 3);
}

__global__ void pose_vec2mat_kernel(const float* __restrict__ vec, int B, int mode, float* __restrict__ out) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const float* v = vec + b * 6;
    float R[9];
    if (mode == 0) {
        euler_to_matrix(v[3], v[4], v[5], R);
    } else {
        // quat2mat (reference inverse_warp.py:115-136): (1, q) normalised
        const float n = sqrtf(1.0f + v[3] * v[3] + v[4] * v[4] + v[5] * v[5]);
        const float w = 1.0f / n, x = v[3] / n, y = v[4] / n, z = v[5] / n;
        R[0] = w * w + x * x - y * y - z * z; R[1] = 2 * x * y - 2 * w * z;         R[2] = 2 * w * y + 2 * x * z;
        R[3] = 2 * w * z + 2 * x * y;         R[4] = w * w - x * x + y * y - z * z; R[5] = 2 * y * z - 2 * w * x;
        R[6] = 2 * x * z - 2 * w * y;         R[7] = 2 * w * x + 2 * y * z;         R[8] = w * w - x * x - y * y + z * z;
    }
    float* o = out + b * 12;
    for (int r = 0; r < 3; ++r) {
        o[r * 4 + 0] = R[r * 3 + 0]; o[r * 4 + 1] = R[r * 3 + 1]; o[r * 4 + 2] = R[r * 3 + 2]; o[r * 4 + 3] = v[r];
    }
}

}  // namespace scsfm

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
using namespace scsfm;

static int check_jobs(const ScsfmPairJob* jobs, int njobs, int B, int H, int W) {
    SCSFM_CHECK_ARG(jobs != nullptr && njobs >= 1 && njobs <= SCSFM_MAX_JOBS, "pairwise: njobs must be in [1,%d], got %d", SCSFM_MAX_JOBS, njobs);
    SCSFM_CHECK_ARG(B >= 1 && H >= 2 && W >= 2, "pairwise: wrong size B=%d H=%d W=%d", B, H, W);
    SCSFM_CHECK_ARG((long long)njobs * B <= 65535, "pairwise: njobs*B too large");
    for (int i = 0; i < njobs; ++i) {
        const ScsfmPairJob& j = jobs[i];
        SCSFM_CHECK_ARG(j.tgt_img && j.ref_img && j.tgt_depth && j.ref_depth && j.pose, "pairwise: job %d has a null input", i);
        SCSFM_CHECK_ARG(j.tgt_shift >= 0 && j.tgt_shift < 8 && j.ref_shift >= 0 && j.ref_shift < 8, "pairwise: job %d bad depth shift", i);
        SCSFM_CHECK_ARG(H % (1 << j.tgt_shift) == 0 && W % (1 << j.tgt_shift) == 0 && H % (1 << j.ref_shift) == 0 && W % (1 << j.ref_shift) == 0,
                        "pairwise: job %d image size not divisible by the depth scale", i);
    }
    return SCSFM_OK;
}

extern "C" size_t scsfm_pairwise_stats_bytes(int njobs, int B) {
    return (size_t)njobs * (STATS_PER_JOB + 12 * (size_t)B) * sizeof(double);
}

extern "C" int scsfm_pairwise_fwd(const ScsfmPairJob* jobs_host, int njobs, const float* intrinsics, int B, int H, int W,
                                  int flags, int padding_mode, void* stats, float* loss_out, const ScsfmPairMaps* maps_host,
                                  void* stream) {
    if (int rc = check_jobs(jobs_host, njobs, B, H, W)) return rc;
    SCSFM_CHECK_ARG(intrinsics && stats && loss_out, "pairwise_fwd: null intrinsics/stats/loss_out");
    SCSFM_CHECK_ARG(padding_mode == SCSFM_PAD_ZEROS || padding_mode == SCSFM_PAD_BORDER, "pairwise_fwd: bad padding_mode %d", padding_mode);
    cudaStream_t st = (cudaStream_t)stream;
    PairJobs pj;
    memset(&pj, 0, sizeof(pj));
    for (int i = 0; i < njobs; ++i) pj.j[i] = jobs_host[i];
    ScsfmPairMaps maps;
    memset(&maps, 0, sizeof(maps));
    if (maps_host) maps = *maps_host;
    SCSFM_CHECK_CUDA(cudaMemsetAsync(stats, 0, scsfm_pairwise_stats_bytes(njobs, B), st));
    dim3 grid((W + TW - 1) / TW, (H + TH - 1) / TH, njobs * B);
    pairwise_fwd_kernel<<<grid, NTHREADS, 0, st>>>(pj, intrinsics, B, H, W, flags, padding_mode, (double*)stats, maps);
    SCSFM_CHECK_LAUNCH();
    if (!(flags & SCSFM_DEFER_FINALIZE)) {
        pairwise_finalize_kernel<<<1, 32, 0, st>>>((double*)stats, njobs, loss_out, 1.0);
        SCSFM_CHECK_LAUNCH();
    }
    return SCSFM_OK;
}

// Second half of scsfm_pairwise_fwd when it was called with SCSFM_DEFER_FINALIZE: the caller may add the first
// scsfm_pairwise_sums_count(njobs) doubles of `stats` (per job {sum photo, sum mask, sum geometry, ...}) over the ranks of a
// data-parallel job in between, which makes mean_on_mask (loss_functions.py:123-129) and its 10000-pixel threshold act on the
// GLOBAL batch exactly as the reference's DataParallel gather does.
extern "C" int scsfm_pairwise_finalize(void* stats, int njobs, float grad_scale, float* loss_out, void* stream) {
    SCSFM_CHECK_ARG(stats && loss_out && njobs >= 1 && njobs <= SCSFM_MAX_JOBS && grad_scale > 0.f, "pairwise_finalize: bad arguments");
    pairwise_finalize_kernel<<<1, 32, 0, (cudaStream_t)stream>>>((double*)stats, njobs, loss_out, (double)grad_scale);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_pairwise_sums_count(int njobs) { return njobs * STATS_PER_JOB; }

extern "C" int scsfm_pairwise_bwd(const ScsfmPairJob* jobs_host, int njobs, const float* intrinsics, int B, int H, int W,
                                  int flags, int padding_mode, void* stats, const float* grad_out, void* stream) {
    if (int rc = check_jobs(jobs_host, njobs, B, H, W)) return rc;
    SCSFM_CHECK_ARG(intrinsics && stats && grad_out, "pairwise_bwd: null intrinsics/stats/grad_out");
    cudaStream_t st = (cudaStream_t)stream;
    PairJobs pj;
    memset(&pj, 0, sizeof(pj));
    for (int i = 0; i < njobs; ++i) pj.j[i] = jobs_host[i];
    double* gM = (double*)stats + (size_t)njobs * STATS_PER_JOB;
    SCSFM_CHECK_CUDA(cudaMemsetAsync(gM, 0, (size_t)njobs * B * 12 * sizeof(double), st));
    dim3 grid((W + TW - 1) / TW, (H + TH - 1) / TH, njobs * B);
    pairwise_bwd_kernel<<<grid, NTHREADS, 0, st>>>(pj, intrinsics, B, H, W, flags, padding_mode, (const double*)stats, gM, grad_out);
    SCSFM_CHECK_LAUNCH();
    pose_grad_kernel<<<(njobs * B + 63) / 64, 64, 0, st>>>(pj, njobs, intrinsics, B, gM);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_inverse_warp2_fwd(const float* img, const float* depth, const float* ref_depth, const float* pose,
                                       const float* intrinsics, int B, int H, int W, int padding_mode, float* warped,
                                       float* valid, float* proj_depth, float* comp_depth, void* stream) {
    SCSFM_CHECK_ARG(img && depth && ref_depth && pose && intrinsics, "inverse_warp2_fwd: null input");
    SCSFM_CHECK_ARG(B >= 1 && B <= 65535 && H >= 2 && W >= 2, "inverse_warp2_fwd: wrong size B=%d H=%d W=%d", B, H, W);
    SCSFM_CHECK_ARG(padding_mode == SCSFM_PAD_ZEROS || padding_mode == SCSFM_PAD_BORDER, "inverse_warp2_fwd: bad padding_mode %d", padding_mode);
    dim3 grid((H * W + NTHREADS - 1) / NTHREADS, B);
    inverse_warp2_fwd_kernel<<<grid, NTHREADS, 0, (cudaStream_t)stream>>>(img, depth, ref_depth, pose, intrinsics, H, W, padding_mode,
                                                                        warped, valid, proj_depth, comp_depth);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_inverse_warp2_bwd(const float* img, const float* depth, const float* ref_depth, const float* pose,
                                       const float* intrinsics, int B, int H, int W, int padding_mode,
                                       const float* grad_warped, const float* grad_proj_depth, const float* grad_comp_depth,
                                       float* grad_depth, float* grad_ref_depth, float* grad_pose, void* scratch, void* stream) {
    SCSFM_CHECK_ARG(img && depth && ref_depth && pose && intrinsics && scratch, "inverse_warp2_bwd: null input");
    SCSFM_CHECK_ARG(B >= 1 && B <= 65535 && H >= 2 && W >= 2, "inverse_warp2_bwd: wrong size B=%d H=%d W=%d", B, H, W);
    cudaStream_t st = (cudaStream_t)stream;
    SCSFM_CHECK_CUDA(cudaMemsetAsync(scratch, 0, (size_t)B * 12 * sizeof(double), st));
    dim3 grid((H * W + NTHREADS - 1) / NTHREADS, B);
    inverse_warp2_bwd_kernel<<<grid, NTHREADS, 0, st>>>(img, depth, ref_depth, pose, intrinsics, H, W, padding_mode, grad_warped,
                                                      grad_proj_depth, grad_comp_depth, grad_depth, grad_ref_depth, (double*)scratch);
    SCSFM_CHECK_LAUNCH();
    if (grad_pose) {
        inverse_warp2_pose_grad_kernel<<<(B + 63) / 64, 64, 0, st>>>(pose, intrinsics, B, (const double*)scratch, grad_pose);
        SCSFM_CHECK_LAUNCH();
    }
    return SCSFM_OK;
}

extern "C" int scsfm_pairwise_intrinsics_grad(const ScsfmPairJob* jobs_host, int njobs, const float* intrinsics, int B,
                                              const void* stats, float* grad_intrinsics, void* stream) {
    SCSFM_CHECK_ARG(jobs_host != nullptr && njobs >= 1 && njobs <= SCSFM_MAX_JOBS,
                    "pairwise_intrinsics_grad: njobs must be in [1,%d], got %d", SCSFM_MAX_JOBS, njobs);
    SCSFM_CHECK_ARG(B >= 1 && (long long)njobs * B <= 65535, "pairwise_intrinsics_grad: wrong batch size B=%d", B);
    SCSFM_CHECK_ARG(intrinsics && stats && grad_intrinsics, "pairwise_intrinsics_grad: null intrinsics/stats/grad_intrinsics");
    PairJobs pj;
    memset(&pj, 0, sizeof(pj));
    for (int i = 0; i < njobs; ++i) {
        SCSFM_CHECK_ARG(jobs_host[i].pose != nullptr, "pairwise_intrinsics_grad: job %d has a null pose", i);
        pj.j[i] = jobs_host[i];
    }
    const double* gM = (const double*)stats + (size_t)njobs * STATS_PER_JOB;
    pairwise_intrinsics_grad_kernel<<<(B * 9 + 127) / 128, 128, 0, (cudaStream_t)stream>>>(pj, njobs, intrinsics, B, gM,
                                                                                            grad_intrinsics);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_inverse_warp2_intrinsics_grad(const float* pose, const float* intrinsics, int B, const void* scratch,
                                                   float* grad_intrinsics, void* stream) {
    SCSFM_CHECK_ARG(pose && intrinsics && scratch && grad_intrinsics, "inverse_warp2_intrinsics_grad: null input");
    SCSFM_CHECK_ARG(B >= 1 && B <= 65535, "inverse_warp2_intrinsics_grad: wrong batch size B=%d", B);
    inverse_warp2_intrinsics_grad_kernel<<<(B * 9 + 127) / 128, 128, 0, (cudaStream_t)stream>>>(pose, intrinsics, B,
                                                                                                 (const double*)scratch, grad_intrinsics);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_pose_vec2mat(const float* vec, int B, int rotation_mode, float* out, void* stream) {
    SCSFM_CHECK_ARG(vec && out && B >= 1, "pose_vec2mat: bad arguments");
    SCSFM_CHECK_ARG(rotation_mode == 0 || rotation_mode == 1, "pose_vec2mat: rotation_mode must be 0 (euler) or 1 (quat)");
    pose_vec2mat_kernel<<<(B + 63) / 64, 64, 0, (cudaStream_t)stream>>>(vec, B, rotation_mode, out);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}
