// bnrelu.cu -- fused training-mode BatchNorm2d (+ ReLU) around the spatial convolutions (SURVEY 8f-2).
//
// The spatial cells of the reference are chains of  ReLU -> conv -> BatchNorm2d  (amoebanet.py:365-398) or
// BatchNorm2d -> ReLU -> conv (resnet_spatial.py:165-180), run as separate eager kernels: per convolution the
// activations cross HBM ~7 more times (BN statistics 1 read, BN apply 1 read + 1 write, ReLU 1 read + 1 write,
// and the same again, doubled, in backward).  Statistics are PER TILE, not synchronised across ranks (N4).
// Here the normalisation and the following ReLU are one pass each way:
//   forward : spc_bn_stats (1 read: per-channel mean and biased variance)   -> rstd on the host side
//             spc_bn_apply (1 read + 1 write: z = relu((y - mean) * rstd * gamma + beta))
//   backward: spc_bn_bwd_reduce (2 reads: sum g, sum g*xhat with g = dz * [z > 0], z recomputed from y)
//             spc_bn_bwd_apply  (2 reads + 1 write: dy = gamma * rstd * (g - mean(g) - xhat * mean(g * xhat)))
// All streaming kernels are pure HBM streams: 16-byte vector accesses over the contiguous H*W planes of NCHW, one
// (plane, chunk) per CTA iteration, fp32 math.  The two reductions write one partial per (plane, chunk) to a
// workspace and a second, small kernel (one CTA per channel) merges a channel's partials in a fixed order in fp64:
// no floating-point atomics, so every output is bit-reproducible, and the variance is formed from sums of squared
// deviations (the parallel-variance combination of Chan et al.), never as E[y^2] - E[y]^2, which cancels when
// |mean| >> std.
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

template <typename T> __device__ __forceinline__ void zero(Vec8<T>& v);
template <> __device__ __forceinline__ void zero(Vec8<__nv_bfloat16>& v) { v.v = make_uint4(0, 0, 0, 0); }
template <> __device__ __forceinline__ void zero(Vec8<float>& v) { v.a = v.b = make_float4(0.f, 0.f, 0.f, 0.f); }

// Pairwise sum of 8 values: 3 rounding levels instead of 7.
template <typename F>
__device__ __forceinline__ F tree8(const F (&f)[8]) {
  return ((f[0] + f[1]) + (f[2] + f[3])) + ((f[4] + f[5]) + (f[6] + f[7]));
}

// Sum over the CTA, returned to EVERY thread: xor butterfly within each warp (every lane ends with the same bits), then
// the 8 warp sums in a fixed tree.  Fixed order, so the result does not depend on timing.  red: 8 slots of shared memory.
template <typename F>
__device__ __forceinline__ F block_sum(F v, F* red) {
  static_assert(BN_THREADS == 256, "the tree below sums 8 warps");
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();   // red may still be read by a previous call
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  F w[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) w[i] = red[i];
  return tree8(w);
}

struct BnGeom {
  int N, C;
  long long HW;
  long long planes;          // N * C
  int chunks;                // chunks per plane
  long long items;           // planes * chunks: one (plane, chunk) work item each, one workspace slot each
};

constexpr int BN_VECS = BN_CHUNK / (BN_THREADS * 8);   // vectors of 8 per thread per item

__device__ __forceinline__ int item_count(const BnGeom& g, int chunk) {
  return (int)min((long long)BN_CHUNK, g.HW - (long long)chunk * BN_CHUNK);
}

// Per (plane, chunk) item: its mean and M2 = sum (y - mean)^2, written to part[item] without atomics.  The item's 64
// values per thread stay in registers (one HBM read): pass 1 gives an fp32 mean m of the item, pass 2 sums d = y - m
// and d^2 (d has one rounding, relative to itself), and mean = m + sum d / n, M2 = sum d^2 - (sum d)^2 / n.  All sums
// are trees (per thread 6 levels, warp 5, CTA 3), so the relative error of a sum is at most 14 * 2^-24 of its sum of
// magnitudes; no raw sum of y^2 is ever formed, so nothing cancels.
template <typename T>
__global__ void __launch_bounds__(BN_THREADS)
bn_stats_kernel(const BnGeom g, const T* __restrict__ y, double2* __restrict__ part) {
  __shared__ float red[8];
  for (long long it = blockIdx.x; it < g.items; it += gridDim.x) {
    const long long plane = it / g.chunks;
    const int chunk = (int)(it % g.chunks);
    const int n = item_count(g, chunk);
    const T* yp = y + plane * g.HW + (long long)chunk * BN_CHUNK;
    Vec8<T> v[BN_VECS];
#pragma unroll
    for (int k = 0; k < BN_VECS; ++k) {
      const int e = (k * BN_THREADS + threadIdx.x) * 8;
      if (e < n) v[k].load(yp + e); else zero(v[k]);
    }
    float s[BN_VECS], q[BN_VECS];
#pragma unroll
    for (int k = 0; k < BN_VECS; ++k) {
      float f[8];
      v[k].get(f);
      s[k] = tree8(f);
    }
    const float m = block_sum(tree8(s), red) / (float)n;
#pragma unroll
    for (int k = 0; k < BN_VECS; ++k) {
      float d[8], d2[8];
      v[k].get(d);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        d[i] -= m;
        d2[i] = d[i] * d[i];
      }
      const bool ok = (k * BN_THREADS + threadIdx.x) * 8 < n;
      s[k] = ok ? tree8(d) : 0.f;
      q[k] = ok ? tree8(d2) : 0.f;
    }
    const float sd = block_sum(tree8(s), red);
    const float sq = block_sum(tree8(q), red);
    if (threadIdx.x == 0) part[it] = make_double2((double)m + (double)sd / n, (double)sq - (double)sd * sd / n);
  }
}

// Per item: sum g and sum g * xhat (g = dz masked by relu(z) > 0, z recomputed from y as bn_apply_kernel computes it),
// written to part[item] without atomics.
template <typename T>
__global__ void __launch_bounds__(BN_THREADS)
bn_bwd_reduce_kernel(const BnGeom g, const T* __restrict__ y, const T* __restrict__ dz, const float* __restrict__ mean,
                     const float* __restrict__ rstd, const float* __restrict__ gamma, const float* __restrict__ beta,
                     int relu, float2* __restrict__ part) {
  __shared__ float red[8];
  for (long long it = blockIdx.x; it < g.items; it += gridDim.x) {
    const long long plane = it / g.chunks;
    const int chunk = (int)(it % g.chunks);
    const int c = (int)(plane % g.C);
    const int n = item_count(g, chunk);
    const long long off = plane * g.HW + (long long)chunk * BN_CHUNK;
    const float m = mean[c], r = rstd[c], ga = gamma[c], be = beta[c];
    float s[BN_VECS], q[BN_VECS];
#pragma unroll
    for (int k = 0; k < BN_VECS; ++k) {
      const int e = (k * BN_THREADS + threadIdx.x) * 8;
      s[k] = q[k] = 0.f;
      if (e < n) {
        Vec8<T> vy, vd;
        float fy[8], gg[8], gx[8];
        vy.load(y + off + e);
        vd.load(dz + off + e);
        vy.get(fy);
        vd.get(gg);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float xh = (fy[i] - m) * r;
          if (relu && xh * ga + be <= 0.f) gg[i] = 0.f;
          gx[i] = gg[i] * xh;
        }
        s[k] = tree8(gg);
        q[k] = tree8(gx);
      }
    }
    const float t0 = block_sum(tree8(s), red);
    const float t1 = block_sum(tree8(q), red);
    if (threadIdx.x == 0) part[it] = make_float2(t0, t1);
  }
}

// The items of channel c: plane p = n * C + c, j-th item of the channel = (n, chunk) with j = n * chunks + chunk.
__device__ __forceinline__ long long channel_item(const BnGeom& g, int c, long long j) {
  return ((j / g.chunks) * g.C + c) * g.chunks + j % g.chunks;
}

// One CTA per channel merges its items in a fixed order in fp64: mean = sum n_i m_i / M, then
// M2 = sum (M2_i + n_i (m_i - mean)^2); mean and the biased variance M2 / M are rounded to fp32 once.
__global__ void __launch_bounds__(BN_THREADS)
bn_stats_merge_kernel(const BnGeom g, const double2* __restrict__ part, float* __restrict__ mean, float* __restrict__ var) {
  __shared__ double red[8];
  const int c = blockIdx.x;
  const long long per = (long long)g.N * g.chunks;
  const double M = (double)g.N * (double)g.HW;
  double s = 0.0;
  for (long long j = threadIdx.x; j < per; j += BN_THREADS)
    s += item_count(g, (int)(j % g.chunks)) * part[channel_item(g, c, j)].x;
  const double mu = block_sum(s, red) / M;
  double q = 0.0;
  for (long long j = threadIdx.x; j < per; j += BN_THREADS) {
    const double2 p = part[channel_item(g, c, j)];
    const double d = p.x - mu;
    q += p.y + item_count(g, (int)(j % g.chunks)) * d * d;
  }
  const double m2 = block_sum(q, red);
  if (threadIdx.x == 0) {
    mean[c] = (float)mu;
    var[c] = (float)fmax(m2 / M, 0.0);
  }
}

// One CTA per channel sums its items' (sum g, sum g * xhat) in a fixed order in fp64, rounded to fp32 once.
__global__ void __launch_bounds__(BN_THREADS)
bn_sum_merge_kernel(const BnGeom g, const float2* __restrict__ part, float* __restrict__ out0, float* __restrict__ out1) {
  __shared__ double red[8];
  const int c = blockIdx.x;
  const long long per = (long long)g.N * g.chunks;
  double s0 = 0.0, s1 = 0.0;
  for (long long j = threadIdx.x; j < per; j += BN_THREADS) {
    const float2 p = part[channel_item(g, c, j)];
    s0 += p.x;
    s1 += p.y;
  }
  const double t0 = block_sum(s0, red);
  const double t1 = block_sum(s1, red);
  if (threadIdx.x == 0) {
    out0[c] = (float)t0;
    out1[c] = (float)t1;
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
  g->N = N; g->C = C; g->HW = HW; g->planes = (long long)N * C;
  g->chunks = (int)((HW + BN_CHUNK - 1) / BN_CHUNK);
  g->items = g->planes * g->chunks;
  long long b = g->items < 132 * 8 ? g->items : 132 * 8;
  *grid = (int)b;
  return SPC_OK;
}

bool aligned(const void* p, uintptr_t a) { return ((uintptr_t)p & (a - 1)) == 0; }

// The NCHW tensors are read and written with 16-byte vectors, the per-channel fp32 vectors one float at a time.
#define BN_REQUIRE_ALIGNED(who, big, small)                                                                        \
  SPC_REQUIRE(big, who ": y, z, dz, dy and the workspace must be 16-byte aligned (a view with a storage offset?)"); \
  SPC_REQUIRE(small, who ": the per-channel vectors must be 4-byte aligned")

}  // namespace
}  // namespace spc

using namespace spc;

extern "C" {

size_t spc_bn_workspace_bytes(int N, int C, long long HW) {
  BnGeom g;
  int grid;
  if (N <= 0 || C <= 0 || HW <= 0 || HW % 8 || bn_geom(N, C, HW, &g, &grid)) return 0;
  return (size_t)g.items * sizeof(double2);
}

int spc_bn_stats(int N, int C, long long HW, int dtype, const void* y, float* mean, float* var, void* workspace,
                 size_t workspace_bytes, void* stream) {
  SPC_REQUIRE(y && mean && var && workspace, "bn_stats: null pointer");
  BnGeom g;
  int grid;
  int rc = bn_geom(N, C, HW, &g, &grid);
  if (rc) return rc;
  BN_REQUIRE_ALIGNED("bn_stats", aligned(y, 16) && aligned(workspace, 16), aligned(mean, 4) && aligned(var, 4));
  SPC_REQUIRE(workspace_bytes >= spc_bn_workspace_bytes(N, C, HW), "bn_stats: workspace of %zu bytes, %zu needed",
              workspace_bytes, spc_bn_workspace_bytes(N, C, HW));
  cudaStream_t st = (cudaStream_t)stream;
  double2* part = (double2*)workspace;
  if (dtype == SPC_BF16)
    bn_stats_kernel<__nv_bfloat16><<<grid, BN_THREADS, 0, st>>>(g, (const __nv_bfloat16*)y, part);
  else
    bn_stats_kernel<float><<<grid, BN_THREADS, 0, st>>>(g, (const float*)y, part);
  SPC_CHECK_CUDA(cudaGetLastError());
  bn_stats_merge_kernel<<<C, BN_THREADS, 0, st>>>(g, part, mean, var);
  count_launch(2);
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
  BN_REQUIRE_ALIGNED("bn_apply", aligned(y, 16) && aligned(z, 16),
                     aligned(mean, 4) && aligned(rstd, 4) && aligned(gamma, 4) && aligned(beta, 4));
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
                      void* workspace, size_t workspace_bytes, void* stream) {
  SPC_REQUIRE(dz && y && mean && rstd && gamma && beta && dsum && dsumx && workspace, "bn_bwd_reduce: null pointer");
  BnGeom g;
  int grid;
  int rc = bn_geom(N, C, HW, &g, &grid);
  if (rc) return rc;
  BN_REQUIRE_ALIGNED("bn_bwd_reduce", aligned(dz, 16) && aligned(y, 16) && aligned(workspace, 16),
                     aligned(mean, 4) && aligned(rstd, 4) && aligned(gamma, 4) && aligned(beta, 4) && aligned(dsum, 4) &&
                         aligned(dsumx, 4));
  SPC_REQUIRE(workspace_bytes >= spc_bn_workspace_bytes(N, C, HW), "bn_bwd_reduce: workspace of %zu bytes, %zu needed",
              workspace_bytes, spc_bn_workspace_bytes(N, C, HW));
  cudaStream_t st = (cudaStream_t)stream;
  float2* part = (float2*)workspace;
  if (dtype == SPC_BF16)
    bn_bwd_reduce_kernel<__nv_bfloat16><<<grid, BN_THREADS, 0, st>>>(g, (const __nv_bfloat16*)y, (const __nv_bfloat16*)dz, mean,
                                                                      rstd, gamma, beta, relu, part);
  else
    bn_bwd_reduce_kernel<float><<<grid, BN_THREADS, 0, st>>>(g, (const float*)y, (const float*)dz, mean, rstd, gamma, beta, relu,
                                                              part);
  SPC_CHECK_CUDA(cudaGetLastError());
  bn_sum_merge_kernel<<<C, BN_THREADS, 0, st>>>(g, part, dsum, dsumx);
  count_launch(2);
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
  BN_REQUIRE_ALIGNED("bn_bwd_apply", aligned(dz, 16) && aligned(y, 16) && aligned(dy, 16),
                     aligned(mean, 4) && aligned(rstd, 4) && aligned(gamma, 4) && aligned(beta, 4) && aligned(dsum, 4) &&
                         aligned(dsumx, 4));
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
