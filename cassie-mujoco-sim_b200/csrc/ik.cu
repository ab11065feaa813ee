// ik.cu -- the inverse-kinematics kernel (sm_90a): each selected environment's free coordinates posed to the target rows (ik.inl), in its own translation
// unit so that the step-kernel instances are not touched by it; compiled once per precision (-DIK_REAL=float / double, build.py).  One warp per CTA, one
// environment at a time over a grid-stride range, with its workspace (IW_SIZE reals: 29.7 KB in double) in shared memory.
#include <cuda_runtime.h>
#include "ik.inl"

namespace cassie {

template <typename real>
__global__ void __launch_bounds__(32) cassie_ik_kernel(const __grid_constant__ IkArgs<real> A) {
  __shared__ __align__(16) unsigned char buf[IW_SIZE * sizeof(real)];
  real *ws = reinterpret_cast<real *>(buf);
  for (int env = blockIdx.x; env < A.n; env += gridDim.x) ik_env(A, env, ws);
}

// one launch over every environment on `stream`: no allocation, no synchronisation (it may be captured in a CUDA graph).  The grid covers the batch
// with at most 16 CTAs per SM
template <typename real> cudaError_t launch_ik(const IkArgs<real> &A, int device, cudaStream_t stream) {
  int sms = 0; cudaError_t e;
  if ((e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device)) != cudaSuccess) return e;
  const int cap = (sms > 0 ? sms : 1) * 16, grid = A.n < cap ? A.n : cap;
  if (grid < 1) return cudaSuccess;
  cassie_ik_kernel<real><<<grid, 32, 0, stream>>>(A);
  return cudaGetLastError();
}
template cudaError_t launch_ik<IK_REAL>(const IkArgs<IK_REAL> &, int, cudaStream_t);

}  // namespace cassie
