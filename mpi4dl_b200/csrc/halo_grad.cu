// halo_grad.cu -- the reverse halo exchange of the exact backward (SPCONV_EXACT_BACKWARD=1).
//
// The reference treats received halo strips as detached constants, so the gradient that a tile's outputs owe to
// its neighbours' edge pixels is dropped (SURVEY 8a N2).  The exact backward sends it back:
//   1. strip gradient: the part of the padded tile's input gradient that lies in pad strip d (the gradient w.r.t.
//      the received strip d), computed in fp32 -- conv (any R x S, stride 1/2), pool (avg / max) or, for
//      halo_exchange_layer, the pad ring of its output gradient;
//   2. the strips travel to neighbour d (the same transports as the forward exchange), which receives them as its
//      direction 8-d;
//   3. accumulate: dx[edge band e] += received strip e, the band spc_halo_pack reads, summed in fp32 in a fixed
//      order and rounded once to the storage dtype (no atomics: bit-reproducible).
// The work is a few strips of a tile, so these are CUDA-core kernels with fp32 accumulation.
#include "common.cuh"

namespace spc {
namespace {

// Strip d of a tile in the PADDED tile's coordinates: rows [r0, r0+sh), cols [c0, c0+sw) of the
// [H+2hh][W+2hw] tile (oracle _recv_region).  Its band inside the tile (what halo_pack sends towards d) has the same
// shape at unpadded rows [b_r0, ...), cols [b_c0, ...).
struct StripGeom {
  int sh[9], sw[9];
  long long off[10];   // prefix sums of per-plane-set element counts (N * C' * sh * sw)
};

__device__ __forceinline__ int strip_of(const long long (&off)[10], long long i) {
  int d = 0;
#pragma unroll
  for (int q = 1; q < 9; ++q) d += (i >= off[q]) ? 1 : 0;
  return d;
}

__device__ __forceinline__ int pad_row0(int d, int H, int hh) { return d / 3 == 0 ? 0 : (d / 3 == 1 ? hh : H + hh); }
__device__ __forceinline__ int pad_col0(int d, int W, int hw) { return d % 3 == 0 ? 0 : (d % 3 == 1 ? hw : W + hw); }

// ---- 1. conv: g_d[n][c][y][x] = sum_k sum_(r,s) dy[n][k][oy][ox] * w[k][c][r][s] over the windows covering the pixel.
// One thread per (strip pixel, block of CB channels): every dy value it loads serves CB channels, the filter loads
// are warp-uniform (the threads of a warp share the channel block).
constexpr int CB = 8;

struct ConvHaloParams {
  const void* dy;
  const void* w;
  float* g[9];
  int N, C, H, W, K, R, S, sh, sw, hh, hw, Ho, Wo, ncb;
  StripGeom s;   // off[] counts (n, channel block, y, x)
};

template <typename T>
__global__ void __launch_bounds__(256) conv_halo_dgrad_kernel(const ConvHaloParams p) {
  const long long total = p.s.off[9];
  const T* dy = reinterpret_cast<const T*>(p.dy);
  const T* w = reinterpret_cast<const T*>(p.w);
  const int RS = p.R * p.S;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int d = strip_of(p.s.off, i);
    const long long e = i - p.s.off[d];
    const int sw = p.s.sw[d], sh = p.s.sh[d];
    const int x = (int)(e % sw);
    const int y = (int)((e / sw) % sh);
    const long long q = e / ((long long)sw * sh);
    const int cb = (int)(q % p.ncb), n = (int)(q / p.ncb);
    const int hp = pad_row0(d, p.H, p.hh) + y, wp = pad_col0(d, p.W, p.hw) + x;   // padded-tile coordinates
    const int c0 = cb * CB;
    float acc[CB];
#pragma unroll
    for (int j = 0; j < CB; ++j) acc[j] = 0.f;
    // taps r with (hp - r) % sh == 0 and 0 <= (hp - r) / sh < Ho
    const int r_lo = max(0, hp - (p.Ho - 1) * p.sh), r_hi = min(p.R - 1, hp);
    const int s_lo = max(0, wp - (p.Wo - 1) * p.sw), s_hi = min(p.S - 1, wp);
    for (int r = r_lo; r <= r_hi; ++r) {
      if ((hp - r) % p.sh) continue;
      const int oy = (hp - r) / p.sh;
      for (int s = s_lo; s <= s_hi; ++s) {
        if ((wp - s) % p.sw) continue;
        const int ox = (wp - s) / p.sw;
        const T* dyp = dy + (((size_t)n * p.K) * p.Ho + oy) * p.Wo + ox;
        const T* wp_ = w + (size_t)c0 * RS + r * p.S + s;
        for (int k = 0; k < p.K; ++k) {
          const float g = to_f32<T>(dyp[(size_t)k * p.Ho * p.Wo]);
          const T* wk = wp_ + (size_t)k * p.C * RS;
#pragma unroll
          for (int j = 0; j < CB; ++j)
            if (c0 + j < p.C) acc[j] = fmaf(g, to_f32<T>(wk[(size_t)j * RS]), acc[j]);
        }
      }
    }
    float* out = p.g[d] + (((size_t)n * p.C + c0) * sh + y) * sw + x;
#pragma unroll
    for (int j = 0; j < CB; ++j)
      if (c0 + j < p.C) out[(size_t)j * sh * sw] = acc[j];
  }
}

// ---- 2. pool: the gradient pool_bwd_kernel would give the strip pixel (same window walk, same first-maximum rule).
struct PoolHaloParams {
  TileView in;   // x + received strips (max needs the window values)
  const void* dy;
  float* g[9];
  int k, stride, pad, mode, Ho, Wo;
  StripGeom s;   // off[] counts (n, c, y, x)
};

template <typename T>
__global__ void __launch_bounds__(256) pool_halo_bwd_kernel(const PoolHaloParams p) {
  const long long total = p.s.off[9];
  const float inv = 1.f / (float)(p.k * p.k);
  const T* dy = reinterpret_cast<const T*>(p.dy);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int d = strip_of(p.s.off, i);
    const long long e = i - p.s.off[d];
    const int sw = p.s.sw[d], sh = p.s.sh[d];
    const int x = (int)(e % sw);
    const int y = (int)((e / sw) % sh);
    const long long nc = e / ((long long)sw * sh);
    const int c = (int)(nc % p.in.C), n = (int)(nc / p.in.C);
    const int hp = pad_row0(d, p.in.H, p.pad) + y, wp = pad_col0(d, p.in.W, p.pad) + x;
    const int h = hp - p.pad, w = wp - p.pad;   // unpadded coordinates (outside the tile)
    int oy_lo = hp - p.k + 1 + p.stride - 1;
    oy_lo = oy_lo < 0 ? 0 : oy_lo / p.stride;
    int ox_lo = wp - p.k + 1 + p.stride - 1;
    ox_lo = ox_lo < 0 ? 0 : ox_lo / p.stride;
    const int oy_hi = min(p.Ho - 1, hp / p.stride), ox_hi = min(p.Wo - 1, wp / p.stride);
    const T* dyp = dy + ((size_t)n * p.in.C + c) * p.Ho * p.Wo;
    float g = 0.f;
    if (p.mode == SPC_POOL_AVG) {
      for (int oy = oy_lo; oy <= oy_hi; ++oy)
        for (int ox = ox_lo; ox <= ox_hi; ++ox) g += to_f32<T>(dyp[(size_t)oy * p.Wo + ox]);
      g *= inv;
    } else {
      for (int oy = oy_lo; oy <= oy_hi; ++oy)
        for (int ox = ox_lo; ox <= ox_hi; ++ox) {
          const int h0 = oy * p.stride - p.pad, w0 = ox * p.stride - p.pad;
          float best = -INFINITY;
          int bi = 0;
          for (int a = 0; a < p.k; ++a)
            for (int b = 0; b < p.k; ++b) {
              const float v = tile_load<T>(p.in, n, c, h0 + a, w0 + b);
              if (pool_max_takes(v, best)) { best = v; bi = a * p.k + b; }
            }
          if (bi == (h - h0) * p.k + (w - w0)) g += to_f32<T>(dyp[(size_t)oy * p.Wo + ox]);
        }
    }
    p.g[d][e] = g;
  }
}

// ---- 3. ring: g_d = the pad strip d of the padded output gradient (backward of halo_exchange_layer).
struct RingParams {
  const void* dy;   // [N][C][H+2hh][W+2hw]
  float* g[9];
  int C, H, W, hh, hw;
  StripGeom s;      // off[] counts (n, c, y, x)
};

template <typename T>
__global__ void halo_ring_kernel(const RingParams p) {
  const long long total = p.s.off[9];
  const int Hp = p.H + 2 * p.hh, Wp = p.W + 2 * p.hw;
  const T* dy = reinterpret_cast<const T*>(p.dy);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int d = strip_of(p.s.off, i);
    const long long e = i - p.s.off[d];
    const int sw = p.s.sw[d], sh = p.s.sh[d];
    const int x = (int)(e % sw);
    const int y = (int)((e / sw) % sh);
    const long long nc = e / ((long long)sw * sh);
    const int hp = pad_row0(d, p.H, p.hh) + y, wp = pad_col0(d, p.W, p.hw) + x;
    p.g[d][e] = to_f32<T>(dy[((size_t)nc * Hp + hp) * Wp + wp]);
  }
}

// ---- 4. accumulate: dx[n][c][h][w] += sum of the received strips whose band covers (h, w), e = 0..8 in order.
// The threads walk the edge bands only: per plane the t top and b bottom rows in full, then lc left and rc right
// columns of the m rows in between.
struct AccParams {
  void* dx;
  const float* g[9];
  int H, W, hh, hw;
  int t, b, m, lc, rc;
  long long per_plane, total;
};

template <typename T>
__global__ void halo_accumulate_kernel(const AccParams p) {
  T* dx = reinterpret_cast<T*>(p.dx);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.total; i += (long long)gridDim.x * blockDim.x) {
    const long long nc = i / p.per_plane;
    long long q = i - nc * p.per_plane;
    int h, w;
    const long long full = (long long)(p.t + p.b) * p.W;
    if (q < full) {
      const int r = (int)(q / p.W);
      h = r < p.t ? r : p.H - p.b + (r - p.t);
      w = (int)(q % p.W);
    } else {
      q -= full;
      const int per_row = p.lc + p.rc;
      h = p.t + (int)(q / per_row);
      const int j = (int)(q % per_row);
      w = j < p.lc ? j : p.W - p.rc + (j - p.lc);
    }
    T* px = dx + ((size_t)nc * p.H + h) * p.W + w;
    float v = to_f32<T>(*px);
#pragma unroll
    for (int e = 0; e < 9; ++e) {
      const float* g = p.g[e];
      if (g == nullptr) continue;
      const int dr = e / 3, dc = e % 3;
      const int sh = dr == 1 ? p.H : p.hh, sw = dc == 1 ? p.W : p.hw;
      const int y = dr == 2 ? h - (p.H - p.hh) : h;
      const int x = dc == 2 ? w - (p.W - p.hw) : w;
      if ((unsigned)y >= (unsigned)sh || (unsigned)x >= (unsigned)sw) continue;
      v += g[((size_t)nc * sh + y) * sw + x];
    }
    *px = from_f32<T>(v);
  }
}

inline int grid_for(long long total) {
  long long b = (total + 255) / 256;
  if (b > 132 * 16) b = 132 * 16;
  if (b < 1) b = 1;
  return (int)b;
}

// strip extents of a tile with halo (hh, hw); off[] counts `per_pixel_planes` x sh x sw per strip with g[d] != NULL
inline StripGeom geom(float* const g[9], long long planes, int H, int W, int hh, int hw) {
  StripGeom s{};
  long long off = 0;
  for (int d = 0; d < 9; ++d) {
    s.sh[d] = d / 3 == 1 ? H : hh;
    s.sw[d] = d % 3 == 1 ? W : hw;
    s.off[d] = off;
    if (d != 4 && g[d]) off += planes * s.sh[d] * s.sw[d];
  }
  s.off[9] = off;
  return s;
}

}  // namespace
}  // namespace spc

extern "C" {

int spc_conv2d_dgrad_halo(const spc_conv_desc* d, const void* dy, const void* w, float* const g[9], void* stream) {
  SPC_REQUIRE(d && dy && w && g, "conv2d_dgrad_halo: null pointer");
  SPC_REQUIRE(d->dtype == SPC_F32 || d->dtype == SPC_BF16, "conv2d_dgrad_halo: bad dtype %d", d->dtype);
  SPC_REQUIRE(d->pad_h == (d->R - 1) / 2 && d->pad_w == (d->S - 1) / 2 && d->stride_h >= 1 && d->stride_w >= 1,
              "conv2d_dgrad_halo: padding must be (k-1)/2 (Spatial not supported yet for this configuration)");
  spc::ConvHaloParams p{};
  p.dy = dy; p.w = w;
  p.N = d->N; p.C = d->C; p.H = d->H; p.W = d->W; p.K = d->K; p.R = d->R; p.S = d->S;
  p.sh = d->stride_h; p.sw = d->stride_w; p.hh = d->pad_h; p.hw = d->pad_w;
  p.Ho = (d->H + 2 * d->pad_h - d->R) / d->stride_h + 1;
  p.Wo = (d->W + 2 * d->pad_w - d->S) / d->stride_w + 1;
  p.ncb = (d->C + spc::CB - 1) / spc::CB;
  for (int i = 0; i < 9; ++i) p.g[i] = i == 4 ? nullptr : g[i];
  p.s = spc::geom(p.g, (long long)p.N * p.ncb, p.H, p.W, p.hh, p.hw);
  if (p.s.off[9] == 0) return SPC_OK;
  const int grid = spc::grid_for(p.s.off[9]);
  if (d->dtype == SPC_BF16) spc::conv_halo_dgrad_kernel<__nv_bfloat16><<<grid, 256, 0, (cudaStream_t)stream>>>(p);
  else spc::conv_halo_dgrad_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>(p);
  spc::count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

int spc_pool2d_bwd_halo(const spc_pool_desc* d, const void* x, const spc_halo* halo, const void* dy, float* const g[9],
                        void* stream) {
  SPC_REQUIRE(d && x && dy && g, "pool2d_bwd_halo: null pointer");
  SPC_REQUIRE(d->k >= 1 && d->stride >= 1 && d->pad == (d->k - 1) / 2,
              "pool2d_bwd_halo: pad must equal floor((k-1)/2), got k=%d pad=%d", d->k, d->pad);
  SPC_REQUIRE(d->mode == SPC_POOL_MAX || d->mode == SPC_POOL_AVG, "pool2d_bwd_halo: bad mode %d", d->mode);
  SPC_REQUIRE(d->dtype == SPC_F32 || d->dtype == SPC_BF16, "pool2d_bwd_halo: bad dtype %d", d->dtype);
  spc::PoolHaloParams p{};
  p.in = spc::make_view(x, halo, d->N, d->C, d->H, d->W, d->pad, d->pad);
  p.dy = dy;
  p.k = d->k; p.stride = d->stride; p.pad = d->pad; p.mode = d->mode;
  p.Ho = (d->H + 2 * d->pad - d->k) / d->stride + 1;
  p.Wo = (d->W + 2 * d->pad - d->k) / d->stride + 1;
  for (int i = 0; i < 9; ++i) p.g[i] = i == 4 ? nullptr : g[i];
  p.s = spc::geom(p.g, (long long)d->N * d->C, d->H, d->W, d->pad, d->pad);
  if (p.s.off[9] == 0) return SPC_OK;
  const int grid = spc::grid_for(p.s.off[9]);
  if (d->dtype == SPC_BF16) spc::pool_halo_bwd_kernel<__nv_bfloat16><<<grid, 256, 0, (cudaStream_t)stream>>>(p);
  else spc::pool_halo_bwd_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>(p);
  spc::count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

int spc_halo_ring(int N, int C, int H, int W, int halo_h, int halo_w, int dtype, const void* dy, float* const g[9],
                  void* stream) {
  SPC_REQUIRE(dy && g, "halo_ring: null pointer");
  SPC_REQUIRE(dtype == SPC_F32 || dtype == SPC_BF16, "halo_ring: bad dtype %d", dtype);
  spc::RingParams p{};
  p.dy = dy; p.C = C; p.H = H; p.W = W; p.hh = halo_h; p.hw = halo_w;
  for (int i = 0; i < 9; ++i) p.g[i] = i == 4 ? nullptr : g[i];
  p.s = spc::geom(p.g, (long long)N * C, H, W, halo_h, halo_w);
  if (p.s.off[9] == 0) return SPC_OK;
  const int grid = spc::grid_for(p.s.off[9]);
  if (dtype == SPC_BF16) spc::halo_ring_kernel<__nv_bfloat16><<<grid, 256, 0, (cudaStream_t)stream>>>(p);
  else spc::halo_ring_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>(p);
  spc::count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

int spc_halo_accumulate(int N, int C, int H, int W, int halo_h, int halo_w, int dtype, void* dx, const float* const g[9],
                        void* stream) {
  SPC_REQUIRE(dx && g, "halo_accumulate: null pointer");
  SPC_REQUIRE(dtype == SPC_F32 || dtype == SPC_BF16, "halo_accumulate: bad dtype %d", dtype);
  SPC_REQUIRE(halo_h >= 0 && halo_w >= 0 && halo_h <= H && halo_w <= W,
              "halo_accumulate: halo (%d,%d) larger than tile (%d,%d)", halo_h, halo_w, H, W);
  spc::AccParams p{};
  bool any = false;
  for (int i = 0; i < 9; ++i) {
    p.g[i] = i == 4 ? nullptr : g[i];
    any = any || p.g[i] != nullptr;
  }
  if (!any) return SPC_OK;
  p.dx = dx; p.H = H; p.W = W; p.hh = halo_h; p.hw = halo_w;
  p.t = halo_h < H ? halo_h : H;
  p.b = halo_h < H - p.t ? halo_h : H - p.t;
  p.m = H - p.t - p.b;
  p.lc = halo_w < W ? halo_w : W;
  p.rc = halo_w < W - p.lc ? halo_w : W - p.lc;
  p.per_plane = (long long)(p.t + p.b) * W + (long long)p.m * (p.lc + p.rc);
  p.total = (long long)N * C * p.per_plane;
  if (p.total == 0) return SPC_OK;
  const int grid = spc::grid_for(p.total);
  if (dtype == SPC_BF16) spc::halo_accumulate_kernel<__nv_bfloat16><<<grid, 256, 0, (cudaStream_t)stream>>>(p);
  else spc::halo_accumulate_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>(p);
  spc::count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

}  // extern "C"
