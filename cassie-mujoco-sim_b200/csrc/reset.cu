// reset.cu -- the restore kernel (sm_90a): environments take rows from a bank of start states under a device mask (reset.inl), in its own translation
// unit so that the step-kernel instances are not touched by it; compiled once per precision (-DRESET_REAL=float / double, build.py).  CTAs of RESET_WPB
// warps, one environment per warp at a time over a grid-stride range.
#include <cuda_runtime.h>
#include "reset.inl"

namespace cassie {

constexpr int RESET_WPB = 8;

template <typename real>
__global__ void __launch_bounds__(32 * RESET_WPB) cassie_reset_kernel(const __grid_constant__ ResetArgs A) {
  static_assert(reset_widths_ok<real>(), "every row of a restore must be a whole number of 16-byte words");
  const int warp = threadIdx.x >> 5;
  for (int env = blockIdx.x * RESET_WPB + warp; env < A.n; env += gridDim.x * RESET_WPB) reset_env(A, env);
}

// one launch over every environment on `stream`: no allocation, no synchronisation (it may be captured in a CUDA graph).  The grid covers the batch
// with at most 16 CTAs per SM; a restore moves a few kB per selected environment, so the launch is short
template <typename real> cudaError_t launch_reset(const ResetArgs &A, int device, cudaStream_t stream) {
  int sms = 0; cudaError_t e;
  if ((e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device)) != cudaSuccess) return e;
  const int need = (A.n + RESET_WPB - 1) / RESET_WPB, cap = (sms > 0 ? sms : 1) * 16, grid = need < cap ? need : cap;
  if (grid < 1) return cudaSuccess;
  cassie_reset_kernel<real><<<grid, 32 * RESET_WPB, 0, stream>>>(A);
  return cudaGetLastError();
}
template cudaError_t launch_reset<RESET_REAL>(const ResetArgs &, int, cudaStream_t);

}  // namespace cassie
