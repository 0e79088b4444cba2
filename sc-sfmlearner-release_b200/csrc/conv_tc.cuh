// Shared declarations of the tensor-core convolution kernels (conv_tc.cu: cp.async gather producers; conv_tma.cu:
// TMA halo-patch producers).
#pragma once
#include <cuda.h>

#include "nn_common.cuh"
#include "tc_common.cuh"

namespace scsfm {

// Chain-drain cycle counters of the TMA convolution kernels (ScsfmConv.debug slot 3, and slots 2, 4, 7 of the weight
// gradient): compiled in only with NVCC_EXTRA=-DSCSFM_DRAIN_COUNTERS.  Predicated off by a NULL debug pointer they still
// cost 1.2 % of the benchmarked step (H100, tf32x3; DESIGN.md §6), so the default build leaves them out.
#ifdef SCSFM_DRAIN_COUNTERS
constexpr bool DRAIN_COUNTERS = true;
#else
constexpr bool DRAIN_COUNTERS = false;
#endif

constexpr int TBM = 128;            // pixel tile of the TMA kernel (two consumer warpgroups of 64 rows)
constexpr int GBM = 64;             // tile rows of the cp.async gather kernels (one wgmma M = 64 warpgroup)
constexpr int TBK = 32;             // floats per k-block = one 128-byte swizzle row
constexpr int FW_PWARPS = 4;        // gather kernels: 4 producer warps + 1 consumer warpgroup (wgmma issue and accumulators)
constexpr int FW_THREADS = (FW_PWARPS + 4) * 32;
constexpr int A_STAGE_BYTES = GBM * 128;

// The tensor core adds into the accumulator with truncation: a long chain of MMAs into one accumulator carries a
// systematic relative error that grows with its length.  In split mode the consumer therefore accumulates CHAIN k-blocks
// (4 wgmma each) into a scratch accumulator started from zero and adds it to the running sum in fp32 registers
// (round-to-nearest); plain TF32 is bounded by its operand rounding and runs one chain.
constexpr int CHAIN_KB = 2;

template <int BN>
struct TcCfg {
    static constexpr int STAGES = 4;
    static constexpr int B_STAGE_BYTES = BN * 128;
    static constexpr size_t OPERANDS = (size_t)STAGES * (A_STAGE_BYTES + B_STAGE_BYTES);
    // epilogue: the accumulator tile [GBM][BN + 1] plus a 32 x 33 transpose scratch per warp, over the free operand ring
    static constexpr size_t EPI = (size_t)GBM * (BN + 1) * 4 + (size_t)(FW_PWARPS + 4) * 32 * 33 * 4;
    static constexpr size_t SMEM = 1024 + (OPERANDS > EPI ? OPERANDS : EPI) + 256;
};

// Operand precision: the tf32 MMA ignores the low 13 mantissa bits of whatever fp32 pattern sits in shared memory
// (a systematic bias per dot product if the operands were not rounded).  Converting with cvt.rna inside the loaders costs
// ~50% of the loader-bound kernel time, so the operands are rounded ONCE where they are produced instead: every
// kernel that writes a tensor later consumed by a convolution takes the SCSFM_ROUND_TF32 flag, and the weights are
// rounded per optimizer step (scsfm_round_tf32).  The loaders below therefore copy bits unchanged.

// Geometry of one (sub-)convolution as the kernel sees it.  A plain convolution uses the identity output map; a
// stride-2 data gradient is run as four parity-class stride-1 sub-convolutions (output pixels 2h+py, 2w+px) whose
// taps are the kernel rows/columns of matching parity -- no multiplications by inserted zeros.
struct TcView {
    int kh, kw;            // tap grid
    int oy0, ox0;          // input row = ho * in_stride + oy0 + dy
    int in_stride;
    int out_sy, out_oy, out_sx, out_ox, out_H, out_W;   // output pixel (ho, wo) -> (ho*out_sy + out_oy, wo*out_sx + out_ox)
    int border;            // 1: the GEMM rows are only the image-border pixels (2*(Ho+Wo)-4 per image), see border_pixel()
};

// Row j of the border-only view -> pixel: top row, bottom row, then the left/right pixels of the rows in between.
__host__ __device__ __forceinline__ void border_pixel(int j, int Ho, int Wo, int& ho, int& wo) {
    if (j < Wo) { ho = 0; wo = j; }
    else if (j < 2 * Wo) { ho = Ho - 1; wo = j - Wo; }
    else { const int k = j - 2 * Wo; ho = 1 + (k >> 1); wo = (k & 1) ? Wo - 1 : 0; }
}
__host__ __device__ __forceinline__ int border_count(int Ho, int Wo) { return 2 * (Ho + Wo) - 4; }


// cuTensorMapEncodeTiled resolved through the runtime (cudaGetDriverEntryPoint): libscsfm.so does not link libcuda, so it
// loads (and its host-side argument checks run) on machines without a driver.  Returns CUDA_ERROR_NOT_FOUND if absent.
CUresult encode_tiled(CUtensorMap* map, CUtensorMapDataType dtype, cuuint32_t rank, void* gaddr, const cuuint64_t* gdim,
                      const cuuint64_t* gstride, const cuuint32_t* box, const cuuint32_t* estr, CUtensorMapInterleave il,
                      CUtensorMapSwizzle sw, CUtensorMapL2promotion l2, CUtensorMapFloatOOBfill oob);
// fp32 NHWC activations seen as [B][rows][cols][C]: element (c, x, y, b) at base + c + x col_step + y row_step + b img_step
// (in elements: a parity view doubles a step), box = box_c x box_w x box_h x 1, zero fill out of bounds
int encode_nhwc(CUtensorMap* map, const float* base, int B, int rows, int cols, int C, long long col_step, long long row_step,
                long long img_step, int box_c, int box_w, int box_h, CUtensorMapSwizzle sw);
// weights [Cout][K] (K contiguous): box = 32 columns x box_rows rows, 128B swizzle (rows past Cout are zero-filled)
int encode_weights(CUtensorMap* map, const float* w, int Cout, int K, int box_rows);

// multiprocessors of the current device (132 if the query fails), looked up once
int sm_count();

// conv_tma.cu: zero-padded stride-1 (sub-)convolutions and stride-2 convolutions with kh, kw <= 3 through the TMA
// halo-patch kernel (stride 2: parity views of the input)
bool conv_tma_eligible(const ScsfmConv& p, const TcView& v);
bool conv_tma_forced(const ScsfmConv& p);      // a tile configuration is being forced through ScsfmConv.tune (tests / experiments)
int launch_conv_tma(const ScsfmConv& p, const TcView& v, cudaStream_t st);

// conv_stem_fwd.cu: forward of the 7x7 stride-2 pad-3 zero-padded stems with Cin 4 or 8 and Cout 64
// (TMA box of the tile's input rows, register A operand, lo(in) computed from it: in_lo is never read)
bool conv_stem_eligible(const ScsfmConv& p);
int launch_conv_stem_fwd(const ScsfmConv& p, cudaStream_t st);

// conv_wgrad_tma.cu: weight gradient of stride-1 and zero-padded stride-2 layers with kh, kw <= 3 and of the 7x7
// stride-2 stems with 4 or 8 channels (TMA halo patch, register A operand); with reflection padding it covers the
// interior pixels only (the ring goes through the gather kernel's border view)
bool conv_wgrad_tma_eligible(const ScsfmConv& p);
int launch_conv_wgrad_tma(const ScsfmConv& p, cudaStream_t st);

// conv_wgrad_thin.cu: 3x3 stride-1 pad-1 layers with Cout = 16 and Cin in {16, 32} on the fp32 FMA pipes (exact products: no low parts)
bool conv_wgrad_thin_eligible(const ScsfmConv& p);
int launch_conv_wgrad_thin(const ScsfmConv& p, cudaStream_t st);

// conv_simt.cu: exact-fp32 implicit GEMM on the CUDA cores (every shape); the weight gradient without the bias gradient
int launch_fwd_simt(const ScsfmConv& p, cudaStream_t st);
int launch_dgrad_simt(const ScsfmConv& p, cudaStream_t st);
int launch_wgrad_simt(const ScsfmConv& p, cudaStream_t st);
int launch_bias_grad(const float* dout, int rows, int C, float* dbias, cudaStream_t st);

}  // namespace scsfm
