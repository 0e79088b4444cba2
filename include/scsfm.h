/*
 * scsfm.h -- C ABI of libscsfm.so: hand-written sm_90a kernels for the SC-SfMLearner
 * training hot path (SURVEY.md section 8).
 *
 * The reference (JiawangBian/SC-SfMLearner-Release) is pure Python and has no FFI of its
 * own; every entry point below names the reference function (file:line under
 * /root/reference) whose device work it replaces.  Conventions:
 *   - extern "C", plain pointers and sizes; no torch types cross this boundary.
 *   - every pointer is DEVICE memory owned by the caller unless the name ends in _host;
 *     the library keeps no pointer past return and allocates no persistent memory.
 *   - tensors are contiguous fp32; images/depths are NCHW exactly as the reference's
 *     Python API passes them (train.py:254-266).
 *   - every call enqueues work on `stream` (a cudaStream_t passed as void*) and returns
 *     without synchronising; return 0 on success, negative on error;
 *     scsfm_last_error() gives a thread-local message.
 */
#ifndef SCSFM_H_
#define SCSFM_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SCSFM_OK 0
#define SCSFM_ERR_ARG (-1)
#define SCSFM_ERR_CUDA (-2)

#define SCSFM_MAX_JOBS 16

/* flags of the pairwise loss (reference loss_functions.py:95, int flags compared with == True) */
#define SCSFM_WITH_SSIM 1
#define SCSFM_WITH_MASK 2
#define SCSFM_WITH_AUTO_MASK 4
/* scsfm_pairwise_fwd only: accumulate the masked sums but do not turn them into losses yet (scsfm_pairwise_finalize does) */
#define SCSFM_DEFER_FINALIZE 0x100
/* padding_mode of F.grid_sample (reference inverse_warp.py:262,267) */
#define SCSFM_PAD_ZEROS 0
#define SCSFM_PAD_BORDER 1

const char* scsfm_last_error(void);
int scsfm_version(void);
/* Number of CUDA kernels this library has launched so far in the process (every launch site counts itself):
 * bench.py reports the difference over its timed region as "gpu_launches". */
long long scsfm_launch_count(void);

/* One pair-direction of compute_photo_and_geometry_loss (reference loss_functions.py:84-87):
 * warp `ref_*` into the view of `tgt_*`.  Depth maps may be coarser than the image by a power
 * of two (the reference nearest-upsamples them first, loss_functions.py:77-82): element (y,x)
 * of the full-resolution map is depth[(y >> shift) * (W >> shift) + (x >> shift)]. */
typedef struct ScsfmPairJob {
    const float* tgt_img;    /* [B,3,H,W] */
    const float* ref_img;    /* [B,3,H,W] */
    const float* tgt_depth;  /* [B,1,H>>tgt_shift,W>>tgt_shift] */
    const float* ref_depth;  /* [B,1,H>>ref_shift,W>>ref_shift] */
    const float* pose;       /* [B,6] tx,ty,tz,rx,ry,rz (euler) */
    float* grad_tgt_depth;   /* backward only: accumulated into (atomic +=), same shape as tgt_depth */
    float* grad_ref_depth;   /* backward only: accumulated into (atomic +=) */
    float* grad_pose;        /* backward only: [B,6], accumulated into (+=) */
    int tgt_shift;
    int ref_shift;
} ScsfmPairJob;

/* Optional per-pixel outputs of job 0 (the four returns of inverse_warp2, reference
 * inverse_warp.py:230-269, plus the final mask/diff maps of loss_functions.py:99-113).
 * Any pointer may be NULL. */
typedef struct ScsfmPairMaps {
    float* warped;       /* [B,3,H,W] projected_img */
    float* valid;        /* [B,1,H,W] valid_mask of inverse_warp2 (before auto-mask) */
    float* proj_depth;   /* [B,1,H,W] projected_depth */
    float* comp_depth;   /* [B,1,H,W] computed_depth */
    float* mask;         /* [B,1,H,W] valid mask after the auto-mask */
    float* diff_img;     /* [B,3,H,W] final photometric map */
    float* diff_depth;   /* [B,1,H,W] */
} ScsfmPairMaps;

/* Bytes of the `stats` buffer needed by scsfm_pairwise_fwd/bwd for njobs jobs and batch B. */
size_t scsfm_pairwise_stats_bytes(int njobs, int B);

/* Fused pixel2cam -> pose -> cam2pixel2 -> bilinear sample -> L1 + SSIM -> depth consistency ->
 * auto-mask -> masked sums, for njobs pair-directions in one launch.
 * Replaces compute_pairwise_loss + inverse_warp2 (+ SSIM.forward, mean_on_mask):
 * reference loss_functions.py:95-129, :11-42; inverse_warp.py:29-44,77-112,139-154,194-269.
 *   intrinsics [B,3,3]; flags = SCSFM_WITH_*; padding_mode = SCSFM_PAD_*.
 *   stats: scratch of scsfm_pairwise_stats_bytes() bytes, kept by the caller for the backward.
 *   loss_out[2]: (photo_loss, geometry_loss) summed over the jobs (loss_functions.py:89-90).
 *   maps: optional per-pixel outputs for job 0 (NULL for none). */
int scsfm_pairwise_fwd(const ScsfmPairJob* jobs_host, int njobs, const float* intrinsics, int B, int H, int W,
                       int flags, int padding_mode, void* stats, float* loss_out, const ScsfmPairMaps* maps_host,
                       void* stream);

/* Second half of scsfm_pairwise_fwd(flags | SCSFM_DEFER_FINALIZE): mean_on_mask of every job (loss_functions.py:123-129) from
 * the sums in stats[0 .. scsfm_pairwise_sums_count(njobs)) (doubles).  A data-parallel caller all-reduces (SUM) exactly that
 * range over the ranks in between, so that the ratio of sums and the 10000-pixel threshold act on the GLOBAL batch as under the
 * reference's DataParallel gather (train.py:168-169); grad_scale (= number of ranks, 1 otherwise) multiplies the backward
 * scales because the gradient all-reduce that follows averages over the ranks. */
int scsfm_pairwise_finalize(void* stats, int njobs, float grad_scale, float* loss_out, void* stream);
int scsfm_pairwise_sums_count(int njobs);

/* Backward of scsfm_pairwise_fwd: given d(loss)/d(photo) and d(loss)/d(geometry) (device scalars
 * grad_out[2]) accumulates gradients into jobs[i].grad_tgt_depth / grad_ref_depth / grad_pose.
 * Hand-written replacement for autograd through reference loss_functions.py:95-129 and
 * inverse_warp.py:230-269 (grid_sampler_2d_backward scatter, bmm/inverse backward). */
int scsfm_pairwise_bwd(const ScsfmPairJob* jobs_host, int njobs, const float* intrinsics, int B, int H, int W,
                       int flags, int padding_mode, void* stats, const float* grad_out, void* stream);

/* Forward of inverse_warp2 alone (reference inverse_warp.py:230-269): the four maps, no loss. */
int scsfm_inverse_warp2_fwd(const float* img, const float* depth, const float* ref_depth, const float* pose,
                            const float* intrinsics, int B, int H, int W, int padding_mode, float* warped,
                            float* valid, float* proj_depth, float* comp_depth, void* stream);

/* Backward of inverse_warp2 alone: grads of the three differentiable maps -> depth, ref_depth, pose
 * (all accumulated into). grad_* inputs may be NULL (treated as zero). */
int scsfm_inverse_warp2_bwd(const float* img, const float* depth, const float* ref_depth, const float* pose,
                            const float* intrinsics, int B, int H, int W, int padding_mode,
                            const float* grad_warped, const float* grad_proj_depth, const float* grad_comp_depth,
                            float* grad_depth, float* grad_ref_depth, float* grad_pose, void* scratch_12B_doubles,
                            void* stream);

/* Gradients with respect to the camera intrinsics (learned / self-calibrated K; reference inverse_warp.py:253,258 differentiate
 * K through intrinsics.inverse() and intrinsics @ pose_mat).  Both run after the matching backward on the same stream and read
 * the per-(job, sample) sums d(loss)/d(K [R|t]) it left behind; d(loss)/dK follows from them in closed form, in fp64, with no
 * per-pixel work.  The result is ADDED into grad_intrinsics [B,3,3] (fp32); one thread per entry sums the jobs in order, so
 * the result is deterministic given the sums.
 *   scsfm_pairwise_intrinsics_grad: after scsfm_pairwise_bwd, with the same jobs, intrinsics and stats.
 *   scsfm_inverse_warp2_intrinsics_grad: after scsfm_inverse_warp2_bwd, with the same pose, intrinsics and scratch. */
int scsfm_pairwise_intrinsics_grad(const ScsfmPairJob* jobs_host, int njobs, const float* intrinsics, int B, const void* stats,
                                   float* grad_intrinsics, void* stream);
int scsfm_inverse_warp2_intrinsics_grad(const float* pose, const float* intrinsics, int B, const void* scratch_12B_doubles,
                                        float* grad_intrinsics, void* stream);

/* pose_vec2mat (reference inverse_warp.py:139-154): [B,6] -> [B,3,4]; rotation_mode 0 = euler, 1 = quat. */
int scsfm_pose_vec2mat(const float* vec, int B, int rotation_mode, float* out, void* stream);

/* One image of compute_smooth_loss (reference loss_functions.py:132-159). */
typedef struct ScsfmSmoothJob {
    const float* depth;   /* [B,1,H,W] (the reference passes scale-0 depth, called "disp" there) */
    const float* img;     /* [B,3,H,W] */
    float* grad_depth;    /* backward only, accumulated into (atomic +=) */
} ScsfmSmoothJob;

size_t scsfm_smooth_stats_bytes(int njobs, int B);

/* Edge-aware smoothness of the mean-normalised map, summed over njobs images
 * (get_smooth_loss, reference loss_functions.py:133-152). loss_out[1]. */
int scsfm_smooth_fwd(const ScsfmSmoothJob* jobs_host, int njobs, int B, int H, int W, void* stats, float* loss_out,
                     void* stream);
int scsfm_smooth_bwd(const ScsfmSmoothJob* jobs_host, int njobs, int B, int H, int W, void* stats,
                     const float* grad_out, void* stream);


/* ------------------------------------------------------------------------------------------------
 * Network operators (DispResNet / PoseResNet forward + backward).  Activations are NHWC fp32,
 * conv weights [Cout][kh][kw][Cin] (the reference's OIHW parameters stored channels-last).
 * These replace the cuDNN / ATen kernels PyTorch launches for reference models/resnet_encoder.py:87-97,
 * models/DispResNet.py:13-47,85-101 and models/PoseResNet.py:35-51 (rows K1-K5 of SURVEY.md 2.3).
 * ---------------------------------------------------------------------------------------------- */
#define SCSFM_PADMODE_ZERO 0
#define SCSFM_PADMODE_REFLECT 1   /* nn.ReflectionPad2d(1), DispResNet.py:34 */
#define SCSFM_ACT_NONE 0
#define SCSFM_ACT_RELU 1
#define SCSFM_ACT_ELU 2           /* nn.ELU, DispResNet.py:20 */
#define SCSFM_ACT_DISP 3          /* 10*sigmoid(x)+0.01, DispResNet.py:98 */
#define SCSFM_BN_SLOTS 16
/* OR-ed into an `act` / `relu` argument: round the stored result to TF32 (round-to-nearest-away, cvt.rna) so that the
 * tensor-core loaders can consume it without converting (the MMA would otherwise truncate the low 13 mantissa bits) */
#define SCSFM_ROUND_TF32 0x100

typedef struct ScsfmConv {
    /* forward operands */
    const float* in;      /* [B,Hi,Wi,Cin] */
    const float* w;       /* [Cout,kh,kw,Cin] */
    const float* bias;    /* [Cout] or NULL */
    float* out;           /* [B,Ho,Wo,Cout] */
    /* backward operands */
    const float* dout;    /* [B,Ho,Wo,Cout] gradient of the PRE-activation output */
    float* din;           /* dgrad result [B,Hi,Wi,Cin] (overwritten) */
    const float* addend;  /* optional tensor added to din (residual branch gradient); forward: added to out before the activation (residual) */
    float* dw;            /* [Cout,kh,kw,Cin], accumulated into (atomic +=) */
    float* dbias;         /* [Cout] or NULL, accumulated into */
    /* fused BatchNorm statistics of the forward output: sums[slot][g][c] = {sum, sum of squares}, fp64,
     * accumulated into (caller zeroes); SCSFM_BN_SLOTS replicas spread the L2 atomic traffic and are added
     * up by scsfm_bn_prepare.  Samples are split into bn_groups equal groups (one per network call when
     * several calls are batched into one launch). */
    double* bn_sums;
    int bn_groups;
    int B, Hi, Wi, Cin, Ho, Wo, Cout, kh, kw, stride, pad, pad_mode, act;
    /* Split-accumulate ("3xTF32") operands of the tensor-core entry points, each optional (NULL = plain TF32):
     * X_lo = tf32(X - trunc_tf32(X)) of the matching tensor (scsfm_split_tf32).  kind::tf32 reads only the upper 19 bits
     * of an fp32 operand, so the raw tensor IS the high part; with the low parts given the kernel accumulates
     * hi*hi + lo*hi + hi*lo into short fp32 accumulation chains (the dropped lo*lo term is 2^-22 relative), which restores
     * fp32-level accuracy of the products (cuDNN's/torch's "highest" matmul precision on the same hardware).
     *   fwd:   in_lo, w_lo      dgrad: dout_lo, w_lo (flipped like w)      wgrad: in_lo, dout_lo */
    const float* in_lo;
    const float* w_lo;
    const float* dout_lo;
    /* per-call experiment knobs (0 = the heuristics) and per-call profiling buffer: nothing in the library is
     * process-global mutable state */
    unsigned tune;
    unsigned long long* debug;   /* device array of 8 x (number of SMs) cycle counters written by the TMA conv kernel, or NULL */
    /* Eval-mode BatchNorm in the forward epilogue (NULL = off): z = act(fmaf(acc, bn_scale[c], bn_shift[c]) + addend), then
     * SCSFM_ROUND_TF32 if flagged -- the arithmetic of scsfm_bn_apply without batch sums, so the fused result is bitwise the
     * conv output followed by scsfm_bn_apply.  Per-output-channel [Cout] arrays from scsfm_bn_eval_prepare_batched.  Refused
     * together with `bias` or `bn_sums`. */
    const float* bn_scale;
    const float* bn_shift;
    /* forward only (NULL = off, 16-byte aligned, Cout % 4 == 0): also write tf32_lo(out) here, the split-accumulate low part a following tf32x3
     * convolution reads as in_lo (what scsfm_split_tf32 of the output would produce) */
    float* out_lo;
    /* 1: split-accumulate (tf32x3) arithmetic.  With it, in_lo / dout_lo may be NULL where scsfm_conv_reads_lo() says the
     * kernel chosen for the call computes them from the operands itself (w_lo is still required in the forward); a kernel
     * that reads a low part which was not passed makes the call fail with SCSFM_ERR_ARG.  0: split mode as implied by the
     * low parts passed. */
    int split;
} ScsfmConv;

/* ScsfmConv.tune */
#define SCSFM_TUNE_NO_TMA 0x1u                          /* fwd/dgrad: cp.async gather kernel only */
#define SCSFM_TUNE_MT(mt) (((unsigned)(mt) & 3u) << 4)       /* TMA kernel: 1|2 stacked 128-pixel sub-tiles (0 = auto) */
#define SCSFM_TUNE_TW(l2) (((unsigned)((l2) ? (l2) - 2 : 0) & 3u) << 6)   /* TMA kernel: tile width log2 3|4 (0 = auto) */
#define SCSFM_TUNE_BN(bn) (((bn) == 16 ? 1u : (bn) == 32 ? 2u : (bn) == 64 ? 3u : (bn) == 128 ? 4u : 0u) << 8)  /* weight rows in smem; TMA wgrad: Cout tile 32|64 */
#define SCSFM_TUNE_WGRAD(k) (((unsigned)(k) & 3u) << 12)     /* weight gradient: 0 auto, 1 gather kernel, 2 TMA kernel, 3 thin-layer fp32 kernel */

/* Exact-fp32 implicit-GEMM convolution on CUDA cores (every shape). */
int scsfm_conv2d_fwd_simt(const ScsfmConv* p, void* stream);
int scsfm_conv2d_dgrad_simt(const ScsfmConv* p, void* stream);
int scsfm_conv2d_wgrad_simt(const ScsfmConv* p, void* stream);

/* wgmma (tf32 operands, fp32 accumulation in registers) implicit-GEMM convolution; needs Cin % 4 == 0.
 * dgrad_tc: stride 1 or 2; p->w must hold the flipped/transposed weights [Cin,kh,kw,Cout] produced by
 * scsfm_weight_flip (the data gradient is the forward kernel run on dout). */
/* Stride-1 (sub-)convolutions with kh, kw <= 3 run the TMA halo-patch kernel (conv_tma.cu: one 4-D tiled TMA load
 * per (channel chunk, dx) brings the input patch of a 2-D output tile, the kh vertical taps reuse it); reflection-
 * padded layers run it zero-padded and recompute the border ring with the gather kernel; so do the zero-padded stride-2
 * forwards with kh, kw <= 3, and the 7x7 stems run conv_stem_fwd.cu (below).  Other shapes use the cp.async gather
 * kernel.  wgrad_tc: stride-1 and zero-padded stride-2 layers with
 * kh, kw <= 3 and the 7x7 stride-2 stems (4 or 8 channels) run the TMA weight-gradient kernel (conv_wgrad_tma.cu). */
int scsfm_conv2d_fwd_tc(const ScsfmConv* p, void* stream);
int scsfm_conv2d_dgrad_tc(const ScsfmConv* p, void* stream);
int scsfm_conv2d_wgrad_tc(const ScsfmConv* p, void* stream);
/* The 7x7 stride-2 pad-3 zero-padded stems with Cin = 4 or 8 (padded) and Cout = 64 run a forward
 * kernel of their own (conv_stem_fwd.cu): a TMA box of the tile's input rows, the im2col operand fed to wgmma from
 * registers, and lo(in) computed from that operand. */
/* Whether the kernel scsfm_conv2d_{fwd,dgrad,wgrad}_tc would pick for *p in split mode (tune knobs included) reads the
 * low parts of its activation operands: in_lo (SCSFM_PASS_FWD), dout_lo (SCSFM_PASS_DGRAD), in_lo and dout_lo
 * (SCSFM_PASS_WGRAD).  1 yes, 0 no (the kernel computes them itself), SCSFM_ERR_ARG for a bad descriptor or pass.  Only
 * the geometry, padding mode, epilogue pointers and tune of *p are looked at; nothing is launched. */
#define SCSFM_PASS_FWD 0
#define SCSFM_PASS_DGRAD 1
#define SCSFM_PASS_WGRAD 2
int scsfm_conv_reads_lo(const ScsfmConv* p, int pass);
/* Operand copies of a tensor for the tensor-core kernels: */
#define SCSFM_OPERAND_TF32 0     /* round-to-nearest TF32 (plain TF32 mode) */
#define SCSFM_OPERAND_RAW 1      /* bits unchanged (split mode: the MMA truncates, i.e. reads the high part) */
#define SCSFM_OPERAND_LO 2       /* tf32(x - trunc_tf32(x)) (split mode: the low part) */
/* flipped / transposed weights of the data gradient, `operand` = one of the above */
int scsfm_weight_flip(const float* w, int Cout, int kh, int kw, int Cin, float* wt, int operand, void* stream);
/* stride-2 data gradient: four parity-class weight sets back to back (Cin*kh*kw*Cout floats in total); p->w of
 * scsfm_conv2d_dgrad_tc must point to them when p->stride == 2 */
int scsfm_weight_flip_s2(const float* w, int Cout, int kh, int kw, int Cin, int pad, float* wt4, int operand, void* stream);

/* Every flip of a network in one launch (the weights change once per optimizer step).  table: device array of
 * (n_rows + 1) x 12 int64 {src pointer, dst pointer, Cout, kh, kw, Cin, jh, jw, dy_max, dx_max, tap step | operand << 8, first block};
 * one row per scsfm_weight_flip job / per stride-2 parity class with taps (jh x jw taps kept, starting at (dy_max, dx_max)
 * and walking backwards by `tap step`); a row owns ceil(Cout/32) * ceil(Cin/32) * jh * jw blocks (one 32 x 32 tile
 * of one tap each) starting at its first block; the last row is a sentinel whose first block is total_blocks. */
int scsfm_weight_flip_batched(const long long* table, int n_rows, int total_blocks, void* stream);

/* Disparity heads (DispResNet.py:79-82,98): 3x3 reflection-padded conv with one output channel, exact fp32.
 * in [B,H,W,C], w [9*C] (= [1,3,3,C]), out / dpre [B,H,W]; dw, dbias accumulated into. */
int scsfm_head_conv_fwd(const float* in, const float* w, const float* bias, float* out, int B, int H, int W, int C, int act, void* stream);
int scsfm_head_conv_wgrad(const float* in, const float* dpre, float* dw, float* dbias, int B, int H, int W, int C, void* stream);
/* gradient w.r.t. the reflection-PADDED head input, dpad [B,H+2,W+2,C] (overwritten; fold it with scsfm_fold_bwd) */
int scsfm_head_conv_dgrad(const float* dpre, const float* w, float* dpad, int B, int H, int W, int C, void* stream);

/* [B,C,H,W] (x1 or x2 sources, PoseResNet.py:65 torch.cat) -> NHWC [B,H,W,C*nsrc] */
int scsfm_nchw_to_nhwc(const float* a, const float* b, int B, int C, int H, int W, float* out, void* stream);
/* same with the channel count zero-padded to Cpad (7x7 stems on the tensor cores: 3 -> 4, 6 -> 8); operand = SCSFM_OPERAND_* */
int scsfm_nchw_to_nhwc_pad(const float* a, const float* b, int B, int C, int H, int W, int Cpad, float* out, int operand, void* stream);
/* rows of C floats -> rows of Cpad floats (zero padded, operand = SCSFM_OPERAND_*) and the inverse accumulation dst[r][c] += src[r][c] */
int scsfm_pad_channels(const float* src, long long rows, int C, int Cpad, float* dst, int operand, void* stream);
int scsfm_unpad_add(const float* src, long long rows, int C, int Cpad, float* dst, void* stream);
/* NHWC [B,H,W,C] -> NCHW */
int scsfm_nhwc_to_nchw(const float* in, int B, int C, int H, int W, float* out, void* stream);
/* Gradient of the network's input images through the 7x7 stride-2 pad-3 stem (resnet_encoder.py:93): the transposed convolution
 * of dy [N,Ho,Wo,64] (the stem's pre-BatchNorm gradient, 16-byte aligned; Ho = (H-1)/2+1, Wo = (W-1)/2+1) with the fp32 stem
 * weights w [64,7,7,Cin], Cin = 3 (DispResNet) or 6 (PoseResNet, the two images concatenated on channels), written (overwritten)
 * in NCHW: channels 0-2 to dimg1 [N,3,H,W], channels 3-5 to dimg2; a NULL image is skipped.  Exact fp32 FMAs, no atomics:
 * the result is deterministic. */
int scsfm_stem_dgrad(const float* dy, const float* w, int N, int H, int W, int Cin, float* dimg1, float* dimg2, void* stream);

/* BatchNorm2d (torchvision resnet.py blocks): prepare per-channel scale/shift from the fused batch sums
 * (sums[SCSFM_BN_SLOTS][groups][C][2], see ScsfmConv.bn_sums)
 * (training; updates running stats with `momentum`, unbiased variance) or from the running stats (eval).
 * saved[g][c] = {scale, shift, mean, invstd}. */
int scsfm_bn_prepare(const double* sums, int groups, int C, long long count_per_group, const float* gamma,
                     const float* beta, float* running_mean, float* running_var, float momentum, float eps,
                     int training, float* saved, void* stream);
/* z = relu?(bn(y) + residual) with the statistics prepared INSIDE the kernel: training (sums != NULL) from the fused batch
 * sums -- also writes `saved` and updates the running statistics like scsfm_bn_prepare; eval (sums == NULL) from the
 * running statistics.  flags: bit 0 = ReLU, SCSFM_ROUND_TF32 = round the result. */
int scsfm_bn_apply(const float* y, const double* sums, const float* gamma, const float* beta, float* running_mean,
                   float* running_var, float momentum, float eps, float* saved, const float* residual, float* z, float* z_lo,
                   long long rows, int C, int groups, int flags, void* stream);   /* z_lo (optional): low part of z (see ScsfmConv.in_lo) */
/* Eval-mode BatchNorm of every layer of a network in ONE launch: per layer, scale[c] = gamma[c] * invstd and
 * shift[c] = beta[c] - running_mean[c] * scale[c] with invstd = 1 / sqrtf(running_var[c] + eps) -- the expressions
 * scsfm_bn_apply uses in eval mode.  table: device array of n_layers x 8 int64 {gamma, beta, running_mean, running_var,
 * scale (out), shift (out), C, eps as the bits of a float}; one CTA per layer.  scale / shift 8-byte aligned (the convolution epilogues read them as float2). */
int scsfm_bn_eval_prepare_batched(const long long* table, int n_layers, void* stream);
/* backward: given dz (gradient of z), z, y -> dy (overwrites `dy`), dres (= dz masked by relu; may be NULL or
 * alias dz), dgamma/dbeta accumulated into. `work` holds groups*C*2 doubles.
 * relu: bit 0 = ReLU gate, SCSFM_ROUND_TF32 = round dy, SCSFM_BN_FROZEN = the statistics in `saved` are frozen (eval mode,
 * running statistics): dy = scale * dz' instead of the batch-statistics formula, one pass; dgamma / dbeta (both may be NULL,
 * then no sums are formed) get sum dz' * xhat and sum dz' with xhat from the running mean and invstd. */
#define SCSFM_BN_FROZEN 0x200
int scsfm_bn_backward(const float* dz, const float* z, const float* y, const float* saved, const float* gamma,
                      float* dy, float* dy_lo, float* dres, float* dgamma, float* dbeta, long long rows, int C, int groups,
                      int relu, double* work, void* stream);   /* dy_lo (optional): low part of dy (see ScsfmConv.dout_lo) */

/* MaxPool2d(3, 2, 1) (resnet_encoder.py:93): idx stores the argmax tap (0..8) per output element. */
int scsfm_maxpool_fwd(const float* x, int B, int H, int W, int C, float* y, unsigned char* idx, void* stream);
int scsfm_maxpool_bwd(const float* dy, const unsigned char* idx, int B, int H, int W, int C, float* dx, int accumulate,
                      void* stream);

/* nearest x2 upsample of `lo` concatenated with `skip` on channels (DispResNet.py:92-95). skip may be NULL. */
int scsfm_upcat_fwd(const float* lo, const float* skip, int B, int H, int W, int C1, int C2, float* out, void* stream);
/* Backward of ReflectionPad2d(1) (+ optional upsample/concat): dpad is the gradient w.r.t. the padded tensor
 * [B,H+2,W+2,C1+C2].  d_lo [B,H/2,W/2,C1] (overwritten; multiplied by act'(lo_act) if act != NONE),
 * d_skip [B,H,W,C2] overwritten, or NULL when its gradient is not wanted (not computed).  With C2 == 0 and upsample == 0: plain fold into d_lo [B,H,W,C1]
 * (accumulate flag honoured, act applied after accumulation). */
int scsfm_fold_bwd(const float* dpad, int B, int H, int W, int C1, int C2, int upsample, float* d_lo,
                   const float* lo_act, int act, int accumulate, float* d_skip, void* stream);

/* in place: d *= act'(out) where `out` is the activation OUTPUT (relu / elu / disp-sigmoid). */
int scsfm_act_bwd(float* d, const float* out, long long n, int act, void* stream);

/* pose head (PoseResNet.py:47-49): out[b,c] = scale * mean_hw x[b,hw,c]; backward broadcasts. */
int scsfm_spatial_mean_fwd(const float* x, int B, int HW, int C, float scale, float* out, void* stream);
int scsfm_spatial_mean_bwd(const float* dout, int B, int HW, int C, float scale, float* dx, void* stream);

/* Validation metrics (reference loss_functions.py:163-205, compute_errors): gt, pred [B,H,W]; per image the pixels inside the
 * crop rows [y1,y2) x columns [x1,x2) with 0.1 < gt < max_depth; prediction clamped to [1e-3, max_depth] and scaled by
 * median(gt) / median(pred) (lower medians, exact radix select).  out[b][8] = {abs_diff, abs_rel, sq_rel, a1, a2, a3,
 * median(gt), median(pred)} (NaN for an empty mask); work: (2 * B) floats + B ints of scratch. */
int scsfm_compute_errors(const float* gt, const float* pred, int B, int H, int W, int y1, int y2, int x1, int x2,
                         float max_depth, void* work, float* out, void* stream);

/* Offline depth evaluation of a chunk of images (reference eval_depth.py:32-56,159-227, DepthEvalEigen.evaluate_depth with
 * median scaling and compute_depth_errors), at the precision numpy uses.  Per image:
 *   - prediction pred[i] [h,w] float64 (test_disp.py's predictions.npy); its inverse 1 / (p + 1e-6) is resized to the ground
 *     truth's H x W as cv2.resize INTER_LINEAR does (half-pixel centres, edge clamp, fp64 weights; horizontal pass, then vertical,
 *     every operation rounded, no FMA) at the masked pixels only, then inverted again: 1 / (x + 1e-6);
 *   - mask: min_depth < gt < max_depth compared in the ground truth's dtype (float32 ground truth compares with float32(min_depth)),
 *     and the pixel inside the crop rows [y1,y2) x columns [x1,x2) (the whole image for NYU);
 *   - numpy medians (ranks (n-1)/2 and n/2 averaged; the ground truth's in its dtype, the prediction's in fp64), exact radix
 *     select; ratio = median(gt) / median(pred) in fp64; prediction * ratio clamped to [min_depth, max_depth];
 *   - out[i][SCSFM_EVAL_OUT] = {n, median(gt), median(pred), ratio, abs_rel, sq_rel, rmse, rmse_log, log10, a1, a2, a3}, fp64;
 *     log(gt) and log10(gt) are taken in the ground truth's dtype.  An empty mask (n = 0) gives NaN for everything but n, as
 *     np.median of an empty array does.
 * gt: packed ground truths, gt_elems elements of gt_dtype; images_host: HOST array of n_img descriptors.  Predictions are
 * depths (positive).  workspace: scsfm_eval_depth_workspace_bytes(images_host, n_img) bytes, 16-byte aligned (the descriptors
 * and 16 bytes per crop pixel).  The descriptors are copied from pageable host memory, which waits for the stream's earlier work.
 * Per-image results do not depend on the other images of the chunk. */
#define SCSFM_EVAL_GT_F32 0
#define SCSFM_EVAL_GT_F64 1
#define SCSFM_EVAL_OUT 12
typedef struct ScsfmEvalDepthImage {
    long long gt_offset;   /* element offset of the image's [H,W] ground truth in `gt` */
    int H, W;
    int y1, y2, x1, x2;    /* crop */
} ScsfmEvalDepthImage;
size_t scsfm_eval_depth_workspace_bytes(const ScsfmEvalDepthImage* images_host, int n_img);
int scsfm_eval_depth(const double* pred, int n_img, int h, int w, const void* gt, int gt_dtype, long long gt_elems,
                     const ScsfmEvalDepthImage* images_host, double min_depth, double max_depth, void* workspace,
                     size_t workspace_bytes, double* out, void* stream);

/* Training-time image transforms of one batch on the device (reference: custom_transforms.py:21-89 -- RandomHorizontalFlip,
 * RandomScaleCrop, ArrayToTensor, Normalize -- applied per sample by datasets/sequence_folders.py:59-62; the zoom is Pillow's
 * 8-bit BICUBIC Image.resize, restated bit for bit).  images [n_img][B][H][W][3] uint8 (decoded frames, image slot major);
 * params [B][5] int32 ON THE DEVICE = {flip, scaled_w, scaled_h, offset_x, offset_y} per sample (scaled_* >= W / H: the zoomed
 * size int(W * sx), int(H * sy); offsets inside [0, scaled - size]; {0, W, H, 0, 0} = the validation chain); mean3 / std3: HOST
 * pointers to three floats; out [n_img][B][3][H][W] float32; workspace: scsfm_augment_workspace_ints(B, H, W) int32, 16-byte
 * aligned.  No host synchronisation. */
long long scsfm_augment_workspace_ints(int B, int H, int W);
int scsfm_augment_batch(const unsigned char* images, const int* params, int n_img, int B, int H, int W, const float* mean3,
                        const float* std3, float* out, int* workspace, long long workspace_ints, void* stream);

/* Training-set preparation (reference data/prepare_train_data.py and its loaders; data/prepare_train_data.py here).
 *
 * Resize of B frames of one source size: PIL.Image.fromarray(img).resize((out_w, out_h), Image.BILINEAR) bit for bit (what
 * scipy.misc.imresize did, kitti_raw_loader.py:224): triangle filter of support max(in / out, 1), Pillow's 22-bit fixed-point
 * taps, horizontal pass into an 8-bit intermediate, then the vertical pass; a pass whose axis keeps its size is skipped.
 * in [B][H][W][3] uint8, out [B][out_h][out_w][3] uint8; workspace: scsfm_resize_bilinear_workspace_bytes(...) bytes,
 * 16-byte aligned.  Downscales of more than 31x per axis are refused. */
size_t scsfm_resize_bilinear_workspace_bytes(int B, int H, int W, int out_h, int out_w);
int scsfm_resize_bilinear_u8(const unsigned char* in, int B, int H, int W, int out_h, int out_w, unsigned char* out,
                             void* workspace, size_t workspace_bytes, void* stream);

/* Velodyne ground-truth depth of B frames (kitti_raw_loader.py:243-300, generate_depth_map, with its quirks).
 * points: float32 [N][4] (the .bin rows: forward, left, up, reflectance; the 4th column is ignored), frame b's points are rows
 * offsets[b] .. offsets[b+1]-1 (offsets: int64 [B+1] on the device, and the same values in HOST memory as offsets_host);
 * P: float64 [B][3][4] P_velo2im per frame; depth: float32 [B][Hd][Wd] (Hd = H / ratio, Wd = W / ratio; Wd >= 2).
 * For every point with x >= 0: u = P [x y z 1] in fp64 (left to right, no FMA), px = rint(u0/u2) - 1, py = rint(u1/u2) - 1
 * (half to even), kept if 0 <= px < Wd and 0 <= py < Hd.  Pixel value: float32(u2) of the last point on the pixel; for every
 * key py * (Wd-1) + px - 1 with >= 2 points (pixels (y, Wd-1) and (y+1, 0) share a key), the pixel of the key's first point
 * gets float32(min u2) of the key; negative values become 0, pixels without points 0.  Deterministic.  workspace:
 * scsfm_velo_depth_workspace_bytes(B, Hd, Wd) bytes (16 per pixel), 16-byte aligned. */
size_t scsfm_velo_depth_workspace_bytes(int B, int Hd, int Wd);
int scsfm_velo_depth(const float* points, const long long* offsets, const long long* offsets_host, const double* P, int B,
                     int Hd, int Wd, float* depth, void* workspace, size_t workspace_bytes, void* stream);

/* out[i] = round-to-nearest TF32 of in[i] (weights of the tensor-core convolutions, once per optimizer step) */
int scsfm_round_tf32(const float* in, float* out, long long n, void* stream);
/* lo[i] = tf32(in[i] - trunc_tf32(in[i])): the low part of the split-accumulate operands (ScsfmConv.in_lo / w_lo / dout_lo) */
int scsfm_split_tf32(const float* in, float* lo, long long n, void* stream);

/* Adam (torch.optim.Adam semantics, train.py:176-178) over a flat parameter arena.  The 1-based step count is
 * `step`, or *step_dev (device int) when step_dev != NULL so that a captured CUDA graph stays valid.
 * mirror (optional): receives the tensor-core operand copy of the updated parameters, mirror_operand = SCSFM_OPERAND_TF32
 * (rounded, plain TF32 mode) or SCSFM_OPERAND_LO (low part, split mode). */
int scsfm_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n, float lr,
                    float beta1, float beta2, float eps, float weight_decay, int step, const int* step_dev,
                    float* mirror, int mirror_operand, void* stream);
/* scsfm_adam_step for an arena with frozen parameters: chunk_mask (device, ceil(n / 64) bytes) says per 64-float chunk whether
 * it is trainable (nonzero).  Frozen chunks are not touched at all -- parameter, exp_avg, exp_avg_sq, weight decay, mirror --
 * as torch.optim.Adam skips parameters whose grad is None; every parameter of an arena starts on a 64-float boundary.
 * Trainable elements get exactly scsfm_adam_step's arithmetic (an all-ones mask gives the same bits). */
int scsfm_adam_step_masked(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n,
                           const unsigned char* chunk_mask, float lr, float beta1, float beta2, float eps, float weight_decay,
                           int step, const int* step_dev, float* mirror, int mirror_operand, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SCSFM_H_ */
