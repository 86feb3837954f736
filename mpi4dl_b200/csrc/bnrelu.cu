// bnrelu.cu -- fused training-mode BatchNorm2d (+ ReLU) around the spatial convolutions (SURVEY 8f-2).
//
// The spatial cells of the reference are chains of  ReLU -> conv -> BatchNorm2d  (amoebanet.py:365-398) or
// BatchNorm2d -> ReLU -> conv (resnet_spatial.py:165-180), run as separate eager kernels: per convolution the
// activations cross HBM ~7 more times (BN statistics 1 read, BN apply 1 read + 1 write, ReLU 1 read + 1 write,
// and the same again, doubled, in backward).  Statistics are PER TILE, not synchronised across ranks (N4).
// Here the normalisation and the following ReLU are one pass each way:
//   forward : spc_bn_stats (1 read: per-channel sum / sum of squares, fp32)   -> mean, rstd on the host side
//             spc_bn_apply (1 read + 1 write: z = relu((y - mean) * rstd * gamma + beta))
//   backward: spc_bn_bwd_reduce (2 reads: sum g, sum g*xhat with g = dz * [z > 0], z recomputed from y)
//             spc_bn_bwd_apply  (2 reads + 1 write: dy = gamma * rstd * (g - mean(g) - xhat * mean(g * xhat)))
// All kernels are pure HBM streams: 16-byte vector accesses over the contiguous H*W planes of NCHW, one
// (plane, chunk) per CTA iteration, fp32 math, block reduction + one atomic per channel per CTA.
#include "common.cuh"

namespace spc {
namespace {

constexpr int BN_THREADS = 256;
constexpr int BN_CHUNK = 8 * BN_THREADS * 8;   // elements per (plane, chunk) work item: 8 vectors of 8 per thread

template <typename T> struct Vec8;   // 8 consecutive elements
template <> struct Vec8<__nv_bfloat16> {
  uint4 v;
  __device__ __forceinline__ void load(const __nv_bfloat16* p) { v = *reinterpret_cast<const uint4*>(p); }
  __device__ __forceinline__ void store(__nv_bfloat16* p) const { *reinterpret_cast<uint4*>(p) = v; }
  __device__ __forceinline__ void get(float (&f)[8]) const {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      f[2 * i] = __uint_as_float(w[i] << 16);
      f[2 * i + 1] = __uint_as_float(w[i] & 0xFFFF0000u);
    }
  }
  __device__ __forceinline__ void set(const float (&f)[8]) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __nv_bfloat162 b = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t*>(&b);
    }
    v = make_uint4(w[0], w[1], w[2], w[3]);
  }
};
template <> struct Vec8<float> {
  float4 a, b;
  __device__ __forceinline__ void load(const float* p) {
    a = *reinterpret_cast<const float4*>(p);
    b = *reinterpret_cast<const float4*>(p + 4);
  }
  __device__ __forceinline__ void store(float* p) const {
    *reinterpret_cast<float4*>(p) = a;
    *reinterpret_cast<float4*>(p + 4) = b;
  }
  __device__ __forceinline__ void get(float (&f)[8]) const {
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
  }
  __device__ __forceinline__ void set(const float (&f)[8]) {
    a = make_float4(f[0], f[1], f[2], f[3]);
    b = make_float4(f[4], f[5], f[6], f[7]);
  }
};

__device__ __forceinline__ float block_sum(float v, float* red) {   // red: 8 floats of shared memory
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
  if (threadIdx.x < 32) {
    t = threadIdx.x < BN_THREADS / 32 ? red[threadIdx.x] : 0.f;
    for (int o = 4; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  }
  return t;   // valid in thread 0
}

struct BnGeom {
  int C;
  long long HW;
  long long planes;          // N * C
  int chunks;                // chunks per plane
  long long items;           // planes * chunks
};

// MODE 0: sum y, sum y^2.   MODE 1: sum g, sum g * xhat  (g = dz masked by relu(z) > 0)
template <typename T, int MODE>
__global__ void __launch_bounds__(BN_THREADS)
bn_reduce_kernel(const BnGeom g, const T* __restrict__ y, const T* __restrict__ dz, const float* __restrict__ mean,
                 const float* __restrict__ rstd, const float* __restrict__ gamma, const float* __restrict__ beta, int relu,
                 float* __restrict__ out0, float* __restrict__ out1) {
  __shared__ float red[8];
  for (long long it = blockIdx.x; it < g.items; it += gridDim.x) {
    const long long plane = it / g.chunks;
    const int chunk = (int)(it % g.chunks);
    const int c = (int)(plane % g.C);
    const long long e0 = (long long)chunk * BN_CHUNK;
    const long long e1 = min(g.HW, e0 + BN_CHUNK);
    const T* yp = y + plane * g.HW;
    const T* dp = MODE == 1 ? dz + plane * g.HW : nullptr;
    float m = 0.f, r = 0.f, ga = 0.f, be = 0.f;
    if (MODE == 1) { m = mean[c]; r = rstd[c]; ga = gamma[c]; be = beta[c]; }
    float s0 = 0.f, s1 = 0.f;
    for (long long e = e0 + (long long)threadIdx.x * 8; e < e1; e += BN_THREADS * 8) {
      Vec8<T> vy, vd;
      float fy[8], fd[8];
      vy.load(yp + e);
      vy.get(fy);
      if (MODE == 1) { vd.load(dp + e); vd.get(fd); }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (MODE == 0) {
          s0 += fy[i];
          s1 += fy[i] * fy[i];
        } else {
          const float xh = (fy[i] - m) * r;
          const float gg = (relu && xh * ga + be <= 0.f) ? 0.f : fd[i];
          s0 += gg;
          s1 += gg * xh;
        }
      }
    }
    const float t0 = block_sum(s0, red);
    const float t1 = block_sum(s1, red);
    if (threadIdx.x == 0) {
      atomicAdd(&out0[c], t0);
      atomicAdd(&out1[c], t1);
    }
  }
}

// MODE 0: z = relu?(xhat * gamma + beta).   MODE 1: dy = gamma * rstd * (g - a0 - xhat * a1), a0 = sum g / M, a1 = sum g xhat / M
template <typename T, int MODE>
__global__ void __launch_bounds__(BN_THREADS)
bn_apply_kernel(const BnGeom g, const T* __restrict__ y, const T* __restrict__ dz, const float* __restrict__ mean,
                const float* __restrict__ rstd, const float* __restrict__ gamma, const float* __restrict__ beta, int relu,
                const float* __restrict__ dsum, const float* __restrict__ dsumx, float inv_count, T* __restrict__ out) {
  for (long long it = blockIdx.x; it < g.items; it += gridDim.x) {
    const long long plane = it / g.chunks;
    const int chunk = (int)(it % g.chunks);
    const int c = (int)(plane % g.C);
    const long long e0 = (long long)chunk * BN_CHUNK;
    const long long e1 = min(g.HW, e0 + BN_CHUNK);
    const T* yp = y + plane * g.HW;
    const T* dp = MODE == 1 ? dz + plane * g.HW : nullptr;
    T* op = out + plane * g.HW;
    const float m = mean[c], r = rstd[c], ga = gamma[c], be = beta[c];
    float a0 = 0.f, a1 = 0.f;
    if (MODE == 1) { a0 = dsum[c] * inv_count; a1 = dsumx[c] * inv_count; }
    for (long long e = e0 + (long long)threadIdx.x * 8; e < e1; e += BN_THREADS * 8) {
      Vec8<T> vy, vd, vo;
      float fy[8], fd[8], fo[8];
      vy.load(yp + e);
      vy.get(fy);
      if (MODE == 1) { vd.load(dp + e); vd.get(fd); }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float xh = (fy[i] - m) * r;
        if (MODE == 0) {
          const float z = xh * ga + be;
          fo[i] = (relu && z <= 0.f) ? 0.f : z;
        } else {
          const float gg = (relu && xh * ga + be <= 0.f) ? 0.f : fd[i];
          fo[i] = ga * r * (gg - a0 - xh * a1);
        }
      }
      vo.set(fo);
      vo.store(op + e);
    }
  }
}

int bn_geom(int N, int C, long long HW, BnGeom* g, int* grid) {
  SPC_REQUIRE(N > 0 && C > 0 && HW > 0, "bn: bad shape N=%d C=%d HW=%lld", N, C, HW);
  SPC_REQUIRE(HW % 8 == 0, "bn: H*W = %lld must be a multiple of 8 (16-byte vector path)", HW);
  g->C = C; g->HW = HW; g->planes = (long long)N * C;
  g->chunks = (int)((HW + BN_CHUNK - 1) / BN_CHUNK);
  g->items = g->planes * g->chunks;
  long long b = g->items < 132 * 8 ? g->items : 132 * 8;
  *grid = (int)b;
  return SPC_OK;
}

}  // namespace
}  // namespace spc

using namespace spc;

extern "C" {

int spc_bn_stats(int N, int C, long long HW, int dtype, const void* y, float* sum, float* sumsq, void* stream) {
  SPC_REQUIRE(y && sum && sumsq, "bn_stats: null pointer");
  BnGeom g;
  int grid;
  int rc = bn_geom(N, C, HW, &g, &grid);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  SPC_CHECK_CUDA(cudaMemsetAsync(sum, 0, sizeof(float) * C, st));
  SPC_CHECK_CUDA(cudaMemsetAsync(sumsq, 0, sizeof(float) * C, st));
  if (dtype == SPC_BF16)
    bn_reduce_kernel<__nv_bfloat16, 0><<<grid, BN_THREADS, 0, st>>>(g, (const __nv_bfloat16*)y, nullptr, nullptr, nullptr,
                                                                    nullptr, nullptr, 0, sum, sumsq);
  else
    bn_reduce_kernel<float, 0><<<grid, BN_THREADS, 0, st>>>(g, (const float*)y, nullptr, nullptr, nullptr, nullptr, nullptr, 0,
                                                            sum, sumsq);
  count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

int spc_bn_apply(int N, int C, long long HW, int dtype, const void* y, const float* mean, const float* rstd,
                 const float* gamma, const float* beta, int relu, void* z, void* stream) {
  SPC_REQUIRE(y && mean && rstd && gamma && beta && z, "bn_apply: null pointer");
  BnGeom g;
  int grid;
  int rc = bn_geom(N, C, HW, &g, &grid);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == SPC_BF16)
    bn_apply_kernel<__nv_bfloat16, 0><<<grid, BN_THREADS, 0, st>>>(g, (const __nv_bfloat16*)y, nullptr, mean, rstd, gamma, beta,
                                                                   relu, nullptr, nullptr, 0.f, (__nv_bfloat16*)z);
  else
    bn_apply_kernel<float, 0><<<grid, BN_THREADS, 0, st>>>(g, (const float*)y, nullptr, mean, rstd, gamma, beta, relu, nullptr,
                                                           nullptr, 0.f, (float*)z);
  count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

int spc_bn_bwd_reduce(int N, int C, long long HW, int dtype, const void* dz, const void* y, const float* mean,
                      const float* rstd, const float* gamma, const float* beta, int relu, float* dsum, float* dsumx,
                      void* stream) {
  SPC_REQUIRE(dz && y && mean && rstd && gamma && beta && dsum && dsumx, "bn_bwd_reduce: null pointer");
  BnGeom g;
  int grid;
  int rc = bn_geom(N, C, HW, &g, &grid);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  SPC_CHECK_CUDA(cudaMemsetAsync(dsum, 0, sizeof(float) * C, st));
  SPC_CHECK_CUDA(cudaMemsetAsync(dsumx, 0, sizeof(float) * C, st));
  if (dtype == SPC_BF16)
    bn_reduce_kernel<__nv_bfloat16, 1><<<grid, BN_THREADS, 0, st>>>(g, (const __nv_bfloat16*)y, (const __nv_bfloat16*)dz, mean,
                                                                    rstd, gamma, beta, relu, dsum, dsumx);
  else
    bn_reduce_kernel<float, 1><<<grid, BN_THREADS, 0, st>>>(g, (const float*)y, (const float*)dz, mean, rstd, gamma, beta, relu,
                                                            dsum, dsumx);
  count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

int spc_bn_bwd_apply(int N, int C, long long HW, int dtype, const void* dz, const void* y, const float* mean,
                     const float* rstd, const float* gamma, const float* beta, int relu, const float* dsum,
                     const float* dsumx, void* dy, void* stream) {
  SPC_REQUIRE(dz && y && mean && rstd && gamma && beta && dsum && dsumx && dy, "bn_bwd_apply: null pointer");
  BnGeom g;
  int grid;
  int rc = bn_geom(N, C, HW, &g, &grid);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const float inv = 1.0f / (float)((double)N * (double)HW);
  if (dtype == SPC_BF16)
    bn_apply_kernel<__nv_bfloat16, 1><<<grid, BN_THREADS, 0, st>>>(g, (const __nv_bfloat16*)y, (const __nv_bfloat16*)dz, mean, rstd,
                                                                   gamma, beta, relu, dsum, dsumx, inv, (__nv_bfloat16*)dy);
  else
    bn_apply_kernel<float, 1><<<grid, BN_THREADS, 0, st>>>(g, (const float*)y, (const float*)dz, mean, rstd, gamma, beta, relu,
                                                           dsum, dsumx, inv, (float*)dy);
  count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

}  // extern "C"
