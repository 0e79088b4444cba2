// Learned cameras for self-calibration under the training transforms.  A bank of n_cams cameras theta [n_cams, 4], each
// (fx, fy, cx, cy) in pixels at the training resolution, and one camera index per sample; one camera is the bank of one, with a
// null index meaning camera 0 for every sample.  Every sample of a batch sees its camera through its own flip / zoom / crop
// (custom_transforms.py:46-89), so its intrinsics are K_b = aug_b(theta[idx_b]):
//
//  * scsfm_camera_build_indexed evaluates aug_b with the operations, order and roundings of scsfm/augment.py:update_intrinsics
//    on a float32 matrix (the reference's expressions under numpy's casting rules): the flip and the crop offsets are float32
//    subtractions (a Python int against a float32 scalar), each zoom is a float64 product rounded back into the float32 matrix
//    (a float32 row times a float64 scalar).  With theta equal to the dataset's K the result is GpuAugment's K bit for bit;
//  * scsfm_camera_grad_indexed is the chain rule through that map (roundings taken as identity): each entry of K_b is an affine
//    function of one parameter, so d(loss)/dtheta[c] = sum over the samples b of camera c of four scaled entries of dK_b.  One CTA
//    per camera sums them in fp64 in a fixed order.
// (One calibration per KITTI raw recording day or one camera per uncalibrated video gives n_cams > 1.)
#include "common.cuh"

namespace scsfm {

constexpr int CAM_GRAD_THREADS = 256;

// sample b sees camera idx[b] (camera 0 for every sample when idx is null); an index outside [0, n_cams) gives a NaN K, and
// theta is never read out of bounds
__global__ void camera_build_kernel(const float* __restrict__ theta, int n_cams, const double* __restrict__ aug,
                                    const int* __restrict__ idx, int B, float* __restrict__ K) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    float* k = K + (size_t)b * 9;
    const int c = idx ? idx[b] : 0;
    if (c < 0 || c >= n_cams) {
#pragma unroll
        for (int i = 0; i < 9; ++i) k[i] = __int_as_float(0x7fc00000);
        return;
    }
    const float* th = theta + (size_t)c * 4;
    const double* a = aug + (size_t)b * SCSFM_CAMERA_AUG_DOUBLES;
    const double xs = a[0], ys = a[1];
    float cx = th[2];
    if (a[2] != 0.0) cx = __fsub_rn((float)a[5], cx);                        // K[0, 2] = in_w - K[0, 2]
    k[0] = __double2float_rn(__dmul_rn((double)th[0], xs));                 // K[0] *= x_scaling
    k[1] = 0.f;                                                              // zero skew (0 * x_scaling)
    k[2] = __fsub_rn(__double2float_rn(__dmul_rn((double)cx, xs)), (float)a[3]);          // ... then K[0, 2] -= offset_x
    k[3] = 0.f;
    k[4] = __double2float_rn(__dmul_rn((double)th[1], ys));                 // K[1] *= y_scaling
    k[5] = __fsub_rn(__double2float_rn(__dmul_rn((double)th[3], ys)), (float)a[4]);       // ... then K[1, 2] -= offset_y
    k[6] = 0.f;
    k[7] = 0.f;
    k[8] = 1.f;
}

// dtheta[c] += sum over the samples b with idx[b] == c of (x_scale dK00, y_scale dK11, +-x_scale dK02, y_scale dK12); one CTA
// per camera (gridDim.x = n_cams), a null idx puts every sample on camera 0 and an out-of-range index on none.  Thread t sums
// samples t, t + 256, ... in order, then a fixed shared-memory tree; no atomics, so two runs give the same bits
__global__ void __launch_bounds__(CAM_GRAD_THREADS)
camera_grad_kernel(const double* __restrict__ aug, const int* __restrict__ idx, const float* __restrict__ dK, int B,
                   float* __restrict__ dtheta) {
    __shared__ double red[4][CAM_GRAD_THREADS];
    const int t = threadIdx.x, c = blockIdx.x;
    double s[4] = {0.0, 0.0, 0.0, 0.0};
    for (int b = t; b < B; b += CAM_GRAD_THREADS) {
        if ((idx ? idx[b] : 0) != c) continue;
        const double* a = aug + (size_t)b * SCSFM_CAMERA_AUG_DOUBLES;
        const float* g = dK + (size_t)b * 9;
        const double xs = a[0], ys = a[1];
        s[0] += xs * (double)g[0];
        s[1] += ys * (double)g[4];
        s[2] += (a[2] != 0.0 ? -xs : xs) * (double)g[2];
        s[3] += ys * (double)g[5];
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) red[i][t] = s[i];
    __syncthreads();
    for (int h = CAM_GRAD_THREADS / 2; h > 0; h >>= 1) {
        if (t < h) {
#pragma unroll
            for (int i = 0; i < 4; ++i) red[i][t] += red[i][t + h];
        }
        __syncthreads();
    }
    float* d = dtheta + (size_t)c * 4;
    if (t < 4) d[t] = __fadd_rn(d[t], (float)red[t][0]);
}

}  // namespace scsfm

using namespace scsfm;

extern "C" int scsfm_camera_build_indexed(const float* theta, int n_cams, const double* aug, const int* idx, int B, float* K_out,
                                          void* stream) {
    SCSFM_CHECK_ARG(theta && aug && K_out, "camera_build_indexed: null pointer (theta, aug and K_out are required)");
    SCSFM_CHECK_ARG(n_cams > 0, "camera_build_indexed: number of cameras must be positive, got %d", n_cams);
    SCSFM_CHECK_ARG(idx || n_cams == 1, "camera_build_indexed: null idx with %d cameras (a null idx means camera 0 for every "
                    "sample, for n_cams = 1 only)", n_cams);
    SCSFM_CHECK_ARG(B > 0, "camera_build_indexed: batch size must be positive, got %d", B);
    camera_build_kernel<<<(B + 127) / 128, 128, 0, (cudaStream_t)stream>>>(theta, n_cams, aug, idx, B, K_out);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}

extern "C" int scsfm_camera_grad_indexed(const double* aug, const int* idx, const float* dK, int B, int n_cams, float* dtheta,
                                         void* stream) {
    SCSFM_CHECK_ARG(aug && dK && dtheta, "camera_grad_indexed: null pointer (aug, dK and dtheta are required)");
    SCSFM_CHECK_ARG(n_cams > 0, "camera_grad_indexed: number of cameras must be positive, got %d", n_cams);
    SCSFM_CHECK_ARG(idx || n_cams == 1, "camera_grad_indexed: null idx with %d cameras (a null idx means camera 0 for every "
                    "sample, for n_cams = 1 only)", n_cams);
    SCSFM_CHECK_ARG(B > 0, "camera_grad_indexed: batch size must be positive, got %d", B);
    camera_grad_kernel<<<n_cams, CAM_GRAD_THREADS, 0, (cudaStream_t)stream>>>(aug, idx, dK, B, dtheta);
    SCSFM_CHECK_LAUNCH();
    return SCSFM_OK;
}
