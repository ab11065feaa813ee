// camera.cu -- the depth-camera kernel (sm_90a), in its own translation unit so that the step-kernel instances are not touched by it; compiled once per
// precision (-DCAM_REAL=float / double, build.py).  Persistent CTAs of CAM_WPB warps, one environment per warp at a time (camera.inl).
#include <cuda_runtime.h>
#include "camera.inl"

namespace cassie {

constexpr int CAM_WPB = 4;   // 4 x CS_W reals of staging: 40 KB in double, within the static shared-memory limit

template <typename real>
__global__ void __launch_bounds__(32 * CAM_WPB) cassie_camera_kernel(CamArgs<real> A) {
  __shared__ __align__(16) real stage[CAM_WPB][CS_W];
  const int warp = threadIdx.x >> 5;
  for (int env = blockIdx.x * CAM_WPB + warp; env < A.n; env += gridDim.x * CAM_WPB) {
    camera_env(A, env, stage[warp]);
    __syncwarp();
  }
}

// one launch over every environment on `stream`; the grid is the resident CTAs of the device (or fewer, for small batches)
template <typename real> cudaError_t launch_camera(const CamArgs<real> &A, int device, cudaStream_t stream) {
  int sms = 0, per_sm = 0; cudaError_t e;
  if ((e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device)) != cudaSuccess) return e;
  if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, cassie_camera_kernel<real>, 32 * CAM_WPB, 0)) != cudaSuccess) return e;
  const int need = (A.n + CAM_WPB - 1) / CAM_WPB, cap = (sms > 0 ? sms : 1) * (per_sm > 0 ? per_sm : 1), grid = need < cap ? need : cap;
  cassie_camera_kernel<real><<<grid, 32 * CAM_WPB, 0, stream>>>(A);
  return cudaGetLastError();
}
template cudaError_t launch_camera<CAM_REAL>(const CamArgs<CAM_REAL> &, int, cudaStream_t);

}  // namespace cassie
