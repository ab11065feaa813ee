// raycast.cu -- the ray-casting kernel (sm_90a), in its own translation unit so that the step-kernel instances are not touched by it; compiled once per
// precision (-DRAY_REAL=float / double, build.py).  Persistent CTAs of RAY_WPB warps, one environment per warp at a time (raycast.inl).
#include <cuda_runtime.h>
#include "raycast.inl"

namespace cassie {

constexpr int RAY_WPB = 8;

template <typename real>
__global__ void __launch_bounds__(32 * RAY_WPB) cassie_raycast_kernel(RayArgs<real> A) {
  __shared__ __align__(16) real stage[RAY_WPB][RS_W];
  const int warp = threadIdx.x >> 5;
  for (int env = blockIdx.x * RAY_WPB + warp; env < A.n; env += gridDim.x * RAY_WPB) {
    raycast_env(A, env, stage[warp]);
    __syncwarp();
  }
}

// one launch over every environment on `stream`; the grid is the resident CTAs of the device (or fewer, for small batches)
template <typename real> cudaError_t launch_raycast(const RayArgs<real> &A, int device, cudaStream_t stream) {
  int sms = 0, per_sm = 0; cudaError_t e;
  if ((e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device)) != cudaSuccess) return e;
  if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, cassie_raycast_kernel<real>, 32 * RAY_WPB, 0)) != cudaSuccess) return e;
  const int need = (A.n + RAY_WPB - 1) / RAY_WPB, cap = (sms > 0 ? sms : 1) * (per_sm > 0 ? per_sm : 1), grid = need < cap ? need : cap;
  cassie_raycast_kernel<real><<<grid, 32 * RAY_WPB, 0, stream>>>(A);
  return cudaGetLastError();
}
template cudaError_t launch_raycast<RAY_REAL>(const RayArgs<RAY_REAL> &, int, cudaStream_t);

}  // namespace cassie
