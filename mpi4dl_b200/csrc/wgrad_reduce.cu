// wgrad_reduce.cu -- the fixed-order sum of the deterministic wgrad (common.cuh: WgradSlices, run_slices).
// Each slice copy holds one add per element (0 + v == v), so dw = (((dw + s0) + s1) + ...) has as many roundings per
// element as the default path's atomics, taken in slice order instead of completion order.
#include "common.cuh"

namespace spc {
namespace {

__global__ void __launch_bounds__(256) wgrad_reduce_kernel(float* __restrict__ dw, const float* __restrict__ buf, int n,
                                                            size_t wn) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < wn; i += (size_t)gridDim.x * blockDim.x) {
    float v = dw[i];
    for (int j = 0; j < n; ++j) v += buf[(size_t)j * wn + i];
    dw[i] = v;
  }
}

}  // namespace

int reduce_slices(float* dw, const float* buf, int n, size_t wn, cudaStream_t st) {
  if (wn == 0 || n <= 0) return SPC_OK;
  const size_t blocks = (wn + 255) / 256;
  wgrad_reduce_kernel<<<(unsigned)(blocks < 8 * 132 ? blocks : 8 * 132), 256, 0, st>>>(dw, buf, n, wn);
  count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

}  // namespace spc
