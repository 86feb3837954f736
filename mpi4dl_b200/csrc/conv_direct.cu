// conv_direct.cu -- CUDA-core (FFMA) direct convolution kernels for sm_90a.
//
// Role in the engine: the shape-complete path.  Every conv_spatial configuration the reference
// accepts (spatial.py:25-155: any odd RxS, stride 1/2, "same" padding) runs here; the wgmma
// GEMM path (gemm_tc.cu) takes over for the shapes that dominate the AmoebaNet-D / ResNet
// workloads.  It also computes the thin boundary strips whose receptive field touches
// neighbour halos, reading halo strips in place (TileView) instead of materialising the padded
// tensor the reference builds with ZeroPad2d + 8 slice copies (spatial.py:1020,405-413).
#include "common.cuh"

namespace spc {

namespace {

constexpr int DC_TH = 8;        // output rows per CTA (one warp per row)
constexpr int DC_LANES = 32;    // threads along W
constexpr int DC_PX = 4;        // output pixels per thread (col = lane + 32*j)
constexpr int DC_TW = DC_LANES * DC_PX;
// output channels per CTA: 16 (whole-tile launches) or 4 (thin boundary strips: 4x more CTAs)
constexpr int DC_THREADS = DC_TH * DC_LANES;

// VERT = false: CTA output tile 8 rows x 128 cols (lanes along W).  VERT = true: 128 rows x 8
// cols (lanes along H) for the thin left/right boundary strips.
template <typename T, bool VERT, int DC_KB>
__global__ void __launch_bounds__(DC_THREADS)
conv_direct_kernel(const DirectConvParams p, const int CB, const int tiles_x, const int kblocks) {
  extern __shared__ float smem[];
  constexpr int TILE_H = VERT ? DC_TW : DC_TH;
  constexpr int TILE_W = VERT ? DC_TH : DC_TW;
  const int PH = (TILE_H - 1) * p.sh + p.R;
  const int PW = (TILE_W - 1) * p.sw + p.S;
  const int PWp = PW | 1;  // odd pitch
  float* patch = smem;                          // [CB][PH][PWp]
  float* wsm = smem + (((size_t)CB * PH * PWp + 3) & ~(size_t)3);  // [CB][R][S][DC_KB], 16B aligned

  const int kb = blockIdx.x % kblocks;
  const int tile = blockIdx.x / kblocks;
  const int tx0 = (tile % tiles_x) * TILE_W;
  const int ty0 = (tile / tiles_x) * TILE_H;
  const int n = blockIdx.y;
  const int k0 = kb * DC_KB;
  const int lane = threadIdx.x % DC_LANES;
  const int ty = threadIdx.x / DC_LANES;
  const int C = p.in.C;

  float acc[DC_PX][DC_KB];
#pragma unroll
  for (int j = 0; j < DC_PX; ++j)
#pragma unroll
    for (int k = 0; k < DC_KB; ++k) acc[j][k] = 0.f;

  const int h_base = ty0 * p.sh - p.pt;
  const int w_base = tx0 * p.sw - p.pl;
  const int RS = p.R * p.S;

  for (int c0 = 0; c0 < C; c0 += CB) {
    __syncthreads();
    const int patch_elems = CB * PH * PW;
    // four independent global loads in flight per thread (addresses first, then loads, then smem stores)
    for (int i0 = threadIdx.x; i0 < patch_elems; i0 += 4 * DC_THREADS) {
      const T* ptr[4];
      int dst[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + u * DC_THREADS;
        ptr[u] = nullptr;
        dst[u] = -1;
        if (i < patch_elems) {
          const int pw = i % PW;
          const int t = i / PW;
          const int ph = t % PH;
          const int c = t / PH;
          dst[u] = (c * PH + ph) * PWp + pw;
          if (c0 + c < C) ptr[u] = tile_ptr<T>(p.in, n, c0 + c, h_base + ph, w_base + pw);
        }
      }
      float v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = ptr[u] ? to_f32<T>(__ldg(ptr[u])) : 0.f;
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (dst[u] >= 0) patch[dst[u]] = v[u];
    }
    const int w_elems = CB * RS * DC_KB;
    for (int i = threadIdx.x; i < w_elems; i += DC_THREADS) {
      const int k = i % DC_KB;
      const int t = i / DC_KB;
      const int rs = t % RS;
      const int c = t / RS;
      float v = 0.f;
      if (c0 + c < C && k0 + k < p.K) {
        const long long idx = p.w_off + (long long)(k0 + k) * p.wKs + (long long)(c0 + c) * p.wCs +
                              (long long)(rs / p.S) * p.wRs + (long long)(rs % p.S) * p.wSs;
        v = to_f32<T>(reinterpret_cast<const T*>(p.w)[idx]);
      }
      wsm[i] = v;
    }
    __syncthreads();

    const int cmax = min(CB, C - c0);
    for (int c = 0; c < cmax; ++c) {
      for (int r = 0; r < p.R; ++r) {
        const float* prow = patch + (c * PH + (VERT ? 0 : ty * p.sh) + r) * PWp;
        const float* wrow = wsm + (c * RS + r * p.S) * DC_KB;
        for (int s = 0; s < p.S; ++s) {
          float xv[DC_PX];
#pragma unroll
          for (int j = 0; j < DC_PX; ++j)
            xv[j] = VERT ? prow[((lane + DC_LANES * j) * p.sh) * PWp + ty * p.sw + s]
                         : prow[(lane + DC_LANES * j) * p.sw + s];
          const float4* wv = reinterpret_cast<const float4*>(wrow + s * DC_KB);
          float wk[DC_KB];
#pragma unroll
          for (int q = 0; q < DC_KB / 4; ++q) {
            const float4 t4 = wv[q];
            wk[4 * q] = t4.x; wk[4 * q + 1] = t4.y; wk[4 * q + 2] = t4.z; wk[4 * q + 3] = t4.w;
          }
#pragma unroll
          for (int j = 0; j < DC_PX; ++j)
#pragma unroll
            for (int k = 0; k < DC_KB; ++k) acc[j][k] = fmaf(xv[j], wk[k], acc[j][k]);
        }
      }
    }
  }

  T* y = reinterpret_cast<T*>(p.y);
#pragma unroll
  for (int k = 0; k < DC_KB; ++k) {
    if (k0 + k >= p.K) break;
    const float b = p.bias ? to_f32<T>(reinterpret_cast<const T*>(p.bias)[k0 + k]) : 0.f;
    const size_t plane = ((size_t)n * p.K + (k0 + k)) * p.YH;
#pragma unroll
    for (int j = 0; j < DC_PX; ++j) {
      const int oy = VERT ? ty0 + lane + DC_LANES * j : ty0 + ty;
      const int ox = VERT ? tx0 + ty : tx0 + lane + DC_LANES * j;
      if (oy < p.Ho && ox < p.Wo)
        y[(plane + (p.oy0 + oy * p.oys)) * p.YW + p.ox0 + ox * p.oxs] = from_f32<T>(acc[j][k] + b);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// wgrad: dw[k][c][r][s] += sum_{n,i,j} dy[n,k,i,j] * in(n,c,i*sh+r-ph, j*sw+s-pw)
constexpr int WG_KB = 16, WG_CB = 16, WG_TH = 4, WG_TW = 32, WG_THREADS = 256, WG_TAPS = 9;

template <typename T>
__global__ void __launch_bounds__(WG_THREADS)
wgrad_direct_kernel(const DirectWgradParams p, const int kblocks, const int cblocks, const int tiles_x,
                    const int tiles_y, const int tiles_per_cta, const int tap0, const int ntaps) {
  extern __shared__ float smem[];
  const int PH = (WG_TH - 1) * p.sh + p.R;
  const int PW = (WG_TW - 1) * p.sw + p.S;
  int plane = PH * PW;
  plane |= 1;
  constexpr int DYP = WG_TH * WG_TW + 1;
  float* dys = smem;                 // [WG_KB][DYP]
  float* xs = smem + WG_KB * DYP;    // [WG_CB][plane]

  const int kb = blockIdx.y % kblocks;
  const int cb = blockIdx.y / kblocks;
  const int k0 = kb * WG_KB, c0 = cb * WG_CB;
  const int kl = threadIdx.x / WG_CB, cl = threadIdx.x % WG_CB;
  const int C = p.in.C;
  const int total_tiles = p.in.N * tiles_x * tiles_y;
  const int t_begin = (blockIdx.x + p.split0) * tiles_per_cta;
  const int t_end = min(total_tiles, t_begin + tiles_per_cta);

  float acc[WG_TAPS];
#pragma unroll
  for (int t = 0; t < WG_TAPS; ++t) acc[t] = 0.f;

  const T* dy = reinterpret_cast<const T*>(p.dy);
  for (int tile = t_begin; tile < t_end; ++tile) {
    const int txi = tile % tiles_x;
    const int tyi = (tile / tiles_x) % tiles_y;
    const int n = tile / (tiles_x * tiles_y);
    const int oy0 = p.ry0 + tyi * WG_TH, ox0 = p.rx0 + txi * WG_TW;
    const int oy_end = p.ry0 + p.rH, ox_end = p.rx0 + p.rW;
    __syncthreads();
    for (int i = threadIdx.x; i < WG_KB * WG_TH * WG_TW; i += WG_THREADS) {
      const int px = i % WG_TW;
      const int py = (i / WG_TW) % WG_TH;
      const int k = i / (WG_TW * WG_TH);
      float v = 0.f;
      if (k0 + k < p.K && oy0 + py < oy_end && ox0 + px < ox_end)
        v = to_f32<T>(dy[(((size_t)n * p.K + k0 + k) * p.Ho + oy0 + py) * p.Wo + ox0 + px]);
      dys[k * DYP + py * WG_TW + px] = v;
    }
    for (int i = threadIdx.x; i < WG_CB * PH * PW; i += WG_THREADS) {
      const int pw = i % PW;
      const int ph = (i / PW) % PH;
      const int c = i / (PW * PH);
      float v = 0.f;
      if (c0 + c < C) v = tile_load<T>(p.in, n, c0 + c, oy0 * p.sh - p.ph + ph, ox0 * p.sw - p.pw + pw);
      xs[c * plane + ph * PW + pw] = v;
    }
    __syncthreads();
    const float* dyr = dys + kl * DYP;
    const float* xr = xs + cl * plane;
    for (int py = 0; py < WG_TH; ++py) {
      for (int px = 0; px < WG_TW; ++px) {
        const float g = dyr[py * WG_TW + px];
        const float* xb = xr + (py * p.sh) * PW + px * p.sw;
#pragma unroll
        for (int t = 0; t < WG_TAPS; ++t) {
          if (t < ntaps) {
            const int tap = tap0 + t;
            acc[t] = fmaf(g, xb[(tap / p.S) * PW + (tap % p.S)], acc[t]);
          }
        }
      }
    }
  }
  if (k0 + kl < p.K && c0 + cl < C) {
    float* dw = p.dw + blockIdx.x * p.slice_stride;
#pragma unroll
    for (int t = 0; t < WG_TAPS; ++t) {
      if (t < ntaps) atomicAdd(&dw[((size_t)(k0 + kl) * C + (c0 + cl)) * (p.R * p.S) + tap0 + t], acc[t]);
    }
  }
}

// slice = chunk: chunk split0 + blockIdx.y adds into db + blockIdx.y * slice_stride
template <typename T>
__global__ void bias_grad_kernel(const T* __restrict__ dy, float* __restrict__ db, int N, int K, int HW,
                                 int chunks, int split0, size_t slice_stride) {
  const int k = blockIdx.x;
  const int chunk = blockIdx.y + split0;
  float s = 0.f;
  for (int n = 0; n < N; ++n) {
    const T* base = dy + ((size_t)n * K + k) * HW;
    const int per = (HW + chunks - 1) / chunks;
    const int b = chunk * per, e = min(HW, b + per);
    for (int i = b + threadIdx.x; i < e; i += blockDim.x) s += to_f32<T>(base[i]);
  }
  __shared__ float red[32];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = (threadIdx.x < (blockDim.x >> 5)) ? red[threadIdx.x] : 0.f;
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) atomicAdd(&db[blockIdx.y * slice_stride + k], s);
  }
}

}  // namespace

int launch_conv_direct(const DirectConvParams& p, int dtype, cudaStream_t st) {
  if (p.Ho <= 0 || p.Wo <= 0 || p.in.N <= 0) return SPC_OK;
  const int TILE_H = p.vert ? DC_TW : DC_TH, TILE_W = p.vert ? DC_TH : DC_TW;
  const int PH = (TILE_H - 1) * p.sh + p.R;
  const int PW = ((TILE_W - 1) * p.sw + p.S) | 1;
  // thin strips (boundary fix-up) have few output pixels: use 4 output channels per CTA so that
  // the launch still fills the machine
  const int DC_KB = ((long long)p.Ho * p.Wo * p.in.N <= 64 * 1024) ? 4 : 16;
  int CB = p.in.C < 8 ? p.in.C : 8;
  auto bytes = [&](int cb) {
    return ((((size_t)cb * PH * PW + 3) & ~(size_t)3) + (size_t)cb * p.R * p.S * DC_KB) * sizeof(float);
  };
  while (CB > 1 && bytes(CB) > 96 * 1024) CB >>= 1;
  const size_t smem = bytes(CB);
  SPC_REQUIRE(smem <= 200 * 1024, "conv_direct: filter %dx%d stride %d needs %zu B smem", p.R, p.S, p.sh, smem);
  const int tiles_x = ceil_div(p.Wo, TILE_W), tiles_y = ceil_div(p.Ho, TILE_H);
  const int kblocks = ceil_div(p.K, DC_KB);
  dim3 grid((unsigned)((size_t)tiles_x * tiles_y * kblocks), p.in.N);
#define SPC_LAUNCH_DC2(TT, VV, KK)                                                                                  \
  do {                                                                                                               \
    const int rc = allow_dynamic_smem((const void*)conv_direct_kernel<TT, VV, KK>, 200 * 1024);                      \
    if (rc) return rc;                                                                                               \
    conv_direct_kernel<TT, VV, KK><<<grid, DC_THREADS, smem, st>>>(p, CB, tiles_x, kblocks);                         \
  } while (0)
#define SPC_LAUNCH_DC(TT, VV)                                          \
  do {                                                                 \
    if (DC_KB == 4) SPC_LAUNCH_DC2(TT, VV, 4); else SPC_LAUNCH_DC2(TT, VV, 16); \
  } while (0)
  if (dtype == SPC_BF16) {
    if (p.vert) SPC_LAUNCH_DC(__nv_bfloat16, true); else SPC_LAUNCH_DC(__nv_bfloat16, false);
  } else {
    if (p.vert) SPC_LAUNCH_DC(float, true); else SPC_LAUNCH_DC(float, false);
  }
#undef SPC_LAUNCH_DC
#undef SPC_LAUNCH_DC2
  spc::count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

// enough CTAs for ~4 waves of 132 SMs x 2 resident CTAs, but at least 8 tiles each
static int direct_tiles_per_cta(int N, int K, int C, int rH, int rW) {
  const int total_tiles = N * ceil_div(rW, WG_TW) * ceil_div(rH, WG_TH);
  int want = (132 * 8) / (ceil_div(K, WG_KB) * ceil_div(C, WG_CB));
  if (want < 1) want = 1;
  int tiles_per_cta = ceil_div(total_tiles, want);
  if (tiles_per_cta < 8) tiles_per_cta = 8;
  return tiles_per_cta;
}

// CTA columns (slices) of launch_wgrad_direct over an output rectangle of rH x rW; 0 if empty
static int wgrad_direct_slices(int N, int K, int C, int rH, int rW) {
  if (rH <= 0 || rW <= 0 || N <= 0) return 0;
  return ceil_div(N * ceil_div(rW, WG_TW) * ceil_div(rH, WG_TH), direct_tiles_per_cta(N, K, C, rH, rW));
}

double direct_wgrad_slice_floats(const spc_conv_desc* d, int rH, int rW) {
  const double wn = (double)d->K * d->C * d->R * d->S;
  return (double)wgrad_direct_slices(d->N, d->K, d->C, rH, rW) * wn;
}

int launch_wgrad_direct(const DirectWgradParams& p_in, int dtype, cudaStream_t st, const WgradSlices* sl) {
  DirectWgradParams p = p_in;
  if (p.rH == 0 && p.rW == 0) { p.ry0 = 0; p.rx0 = 0; p.rH = p.Ho; p.rW = p.Wo; }
  if (p.rH <= 0 || p.rW <= 0 || p.in.N <= 0) return SPC_OK;
  const int PH = (WG_TH - 1) * p.sh + p.R;
  const int PW = (WG_TW - 1) * p.sw + p.S;
  const size_t smem = ((size_t)WG_KB * (WG_TH * WG_TW + 1) + (size_t)WG_CB * ((PH * PW) | 1)) * sizeof(float);
  SPC_REQUIRE(smem <= 200 * 1024, "wgrad_direct: filter %dx%d needs %zu B smem", p.R, p.S, smem);
  const int tiles_x = ceil_div(p.rW, WG_TW), tiles_y = ceil_div(p.rH, WG_TH);
  const int kblocks = ceil_div(p.K, WG_KB), cblocks = ceil_div(p.in.C, WG_CB);
  const int tiles_per_cta = direct_tiles_per_cta(p.in.N, p.K, p.in.C, p.rH, p.rW);
  const int ctas_x = wgrad_direct_slices(p.in.N, p.K, p.in.C, p.rH, p.rW);
  const int taps = p.R * p.S;
  const size_t wn = (size_t)p.K * p.in.C * taps;
  const int rc = allow_dynamic_smem(dtype == SPC_BF16 ? (const void*)wgrad_direct_kernel<__nv_bfloat16>
                                                     : (const void*)wgrad_direct_kernel<float>, 200 * 1024);
  if (rc) return rc;
  // slice = CTA column: its tiles are summed in registers, its adds cover disjoint (k, c) blocks
  return run_slices(sl, ctas_x, wn, p.dw, st, [&](int s0, int ns, float* dst, size_t stride) {
    DirectWgradParams q = p;
    q.split0 = s0; q.dw = dst; q.slice_stride = stride;
    dim3 grid(ns, kblocks * cblocks);
    for (int tap0 = 0; tap0 < taps; tap0 += WG_TAPS) {
      const int nt = taps - tap0 < WG_TAPS ? taps - tap0 : WG_TAPS;
      if (dtype == SPC_BF16) {
        wgrad_direct_kernel<__nv_bfloat16><<<grid, WG_THREADS, smem, st>>>(q, kblocks, cblocks, tiles_x, tiles_y,
                                                                           tiles_per_cta, tap0, nt);
      } else {
        wgrad_direct_kernel<float><<<grid, WG_THREADS, smem, st>>>(q, kblocks, cblocks, tiles_x, tiles_y,
                                                                  tiles_per_cta, tap0, nt);
      }
      spc::count_launch();
      SPC_CHECK_CUDA(cudaGetLastError());
    }
    return SPC_OK;
  });
}

int launch_bias_grad(const void* dy, float* db, int N, int K, int HW, int dtype, int accumulate, cudaStream_t st,
                     const WgradSlices* sl) {
  if (!accumulate) SPC_CHECK_CUDA(cudaMemsetAsync(db, 0, sizeof(float) * K, st));
  int chunks = ceil_div(HW, 1 << 16);
  if (chunks > 64) chunks = 64;
  return run_slices(sl, chunks, (size_t)K, db, st, [&](int s0, int ns, float* dst, size_t stride) {
    dim3 grid(K, ns);
    if (dtype == SPC_BF16)
      bias_grad_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(dy), dst, N, K, HW,
                                                            chunks, s0, stride);
    else
      bias_grad_kernel<float><<<grid, 256, 0, st>>>(reinterpret_cast<const float*>(dy), dst, N, K, HW, chunks, s0,
                                                    stride);
    spc::count_launch();
    SPC_CHECK_CUDA(cudaGetLastError());
    return SPC_OK;
  });
}

}  // namespace spc
