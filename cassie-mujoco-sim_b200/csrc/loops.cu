// loops.cu -- the loop-closure kernel (sm_90a): each selected environment's qpos and qvel projected onto the connect equalities (loops.inl), in its own
// translation unit so that the step-kernel instances are not touched by it; compiled once per precision (-DLOOPS_REAL=float / double, build.py).  CTAs
// of LOOPS_WPB warps, one environment per warp at a time over a grid-stride range, each warp with its workspace in shared memory.
#include <cuda_runtime.h>
#include "loops.inl"

namespace cassie {

constexpr int LOOPS_WPB = 4;

template <typename real>
__global__ void __launch_bounds__(32 * LOOPS_WPB) cassie_loops_kernel(const __grid_constant__ LoopArgs<real> A) {
  __shared__ __align__(16) unsigned char buf[LOOPS_WPB * LW_SIZE * sizeof(real)];
  const int warp = threadIdx.x >> 5;
  real *ws = reinterpret_cast<real *>(buf) + warp * LW_SIZE;
  for (int env = blockIdx.x * LOOPS_WPB + warp; env < A.n; env += gridDim.x * LOOPS_WPB) loops_env(A, env, ws);
}

// one launch over every environment on `stream`: no allocation, no synchronisation (it may be captured in a CUDA graph).  The grid covers the batch
// with at most 8 CTAs per SM
template <typename real> cudaError_t launch_loops(const LoopArgs<real> &A, int device, cudaStream_t stream) {
  int sms = 0; cudaError_t e;
  if ((e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device)) != cudaSuccess) return e;
  const int need = (A.n + LOOPS_WPB - 1) / LOOPS_WPB, cap = (sms > 0 ? sms : 1) * 8, grid = need < cap ? need : cap;
  if (grid < 1) return cudaSuccess;
  cassie_loops_kernel<real><<<grid, 32 * LOOPS_WPB, 0, stream>>>(A);
  return cudaGetLastError();
}
template cudaError_t launch_loops<LOOPS_REAL>(const LoopArgs<LOOPS_REAL> &, int, cudaStream_t);

}  // namespace cassie
