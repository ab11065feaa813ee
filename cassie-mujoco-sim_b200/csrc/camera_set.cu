// camera_set.cu -- the camera-set kernel (sm_90a), in its own translation unit beside the one-camera kernel (camera.cu); compiled once per precision
// (-DCAMSET_REAL=float / double, build.py).  Persistent CTAs of CAM_WPB warps, one environment per warp at a time, every camera of the set
// (camera_set.inl).
#include <cuda_runtime.h>
#include "camera_set.inl"

namespace cassie {

constexpr int CAMSET_WPB = 4;   // 4 x CSET_W reals of staging: 40.5 KB in double, within the static shared-memory limit
// resident CTAs per SM the register budget is held to: 6 in float (80 registers; the camera loop alone would take the allocation to 96 registers and
// the residency to 5 CTAs), 4 in double (its 128 registers allow no more)
template <typename real> constexpr int CAMSET_MIN_CTAS = sizeof(real) == 4 ? 6 : 4;

template <typename real>
__global__ void __launch_bounds__(32 * CAMSET_WPB, CAMSET_MIN_CTAS<real>) cassie_camset_kernel(CamSetArgs<real> A) {
  __shared__ __align__(16) real stage[CAMSET_WPB][CSET_W];
  const int warp = threadIdx.x >> 5;
  for (int env = blockIdx.x * CAMSET_WPB + warp; env < A.n; env += gridDim.x * CAMSET_WPB) {
    camera_set_env(A, env, stage[warp]);
    __syncwarp();
  }
}

// one launch over every environment on `stream`; the grid is the resident CTAs of the device (or fewer, for small batches)
template <typename real> cudaError_t launch_camera_set(const CamSetArgs<real> &A, int device, cudaStream_t stream) {
  int sms = 0, per_sm = 0; cudaError_t e;
  if ((e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device)) != cudaSuccess) return e;
  if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, cassie_camset_kernel<real>, 32 * CAMSET_WPB, 0)) != cudaSuccess) return e;
  const int need = (A.n + CAMSET_WPB - 1) / CAMSET_WPB, cap = (sms > 0 ? sms : 1) * (per_sm > 0 ? per_sm : 1), grid = need < cap ? need : cap;
  cassie_camset_kernel<real><<<grid, 32 * CAMSET_WPB, 0, stream>>>(A);
  return cudaGetLastError();
}
template cudaError_t launch_camera_set<CAMSET_REAL>(const CamSetArgs<CAMSET_REAL> &, int, cudaStream_t);

}  // namespace cassie
