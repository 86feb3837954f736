// pool.cu -- spatially-partitioned Max/Avg pooling forward and backward for sm_90a.
//
// Replaces Pool.forward (reference spatial.py:1503-1509): halo_exchange_layer (pad + 8-way
// exchange + 8 unpack copies) followed by nn.{Max,Avg}Pool2d(padding=0).  Here the window is
// read straight from the tile and its halo strips (TileView); the padded tensor never exists.
// These ops are pure HBM streaming (AI ~ 0): one read of x, one write of y.
#include "common.cuh"
#include "tc_common.cuh"

namespace spc {
namespace {

struct PoolParams {
  TileView in;
  const void* dy;
  void* out;   // y (fwd) or dx (bwd)
  int k, stride, pad, mode, Ho, Wo;
};

// ---- forward, generic: one thread per output element ---------------------------------------
template <typename T>
__global__ void pool_fwd_kernel(const PoolParams p) {
  const size_t total = (size_t)p.in.N * p.in.C * p.Ho * p.Wo;
  const float inv = 1.f / (float)(p.k * p.k);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int ox = (int)(i % p.Wo);
    const int oy = (int)((i / p.Wo) % p.Ho);
    const size_t nc = i / ((size_t)p.Wo * p.Ho);
    const int c = (int)(nc % p.in.C), n = (int)(nc / p.in.C);
    const int h0 = oy * p.stride - p.pad, w0 = ox * p.stride - p.pad;
    float r = (p.mode == SPC_POOL_MAX) ? -INFINITY : 0.f;
    for (int a = 0; a < p.k; ++a)
      for (int b = 0; b < p.k; ++b) {
        const float v = tile_load<T>(p.in, n, c, h0 + a, w0 + b);
        r = (p.mode == SPC_POOL_MAX) ? pool_max(r, v) : r + v;
      }
    if (p.mode == SPC_POOL_AVG) r *= inv;
    reinterpret_cast<T*>(p.out)[i] = from_f32<T>(r);
  }
}

template <typename T, int NEL>
__device__ __forceinline__ void load_vec(const T* __restrict__ src, float (&dst)[NEL]) {
  constexpr int NV = NEL * sizeof(T) / 16;
  uint4 raw[NV];
#pragma unroll
  for (int q = 0; q < NV; ++q) raw[q] = __ldg(reinterpret_cast<const uint4*>(src) + q);
  const T* e = reinterpret_cast<const T*>(raw);
#pragma unroll
  for (int j = 0; j < NEL; ++j) dst[j] = to_f32<T>(e[j]);
}
template <typename T, int NEL>
__device__ __forceinline__ void store_vec(T* __restrict__ dst, const float (&src)[NEL]) {
  constexpr int NV = NEL * sizeof(T) / 16;
  uint4 raw[NV];
  T* e = reinterpret_cast<T*>(raw);
#pragma unroll
  for (int j = 0; j < NEL; ++j) e[j] = from_f32<T>(src[j]);
#pragma unroll
  for (int q = 0; q < NV; ++q) reinterpret_cast<uint4*>(dst)[q] = raw[q];
}

// ---- forward, vectorised interior path -----------------------------------------------------
// Each thread produces VEC consecutive outputs of one row.  Input rows are fetched as 16-byte
// vectors (plus the window overhang as scalars through tile_load), so a warp reads full 128 B
// lines.  Used when W (and Wo) are multiples of the vector width; edges fall back per element.
template <typename T, int VEC, int K, int STRIDE>
__global__ void __launch_bounds__(256)
pool_fwd_vec_kernel(const PoolParams p) {
  constexpr int PAD = (K - 1) / 2;
  constexpr int SPAN = (VEC - 1) * STRIDE + K;           // input columns needed
  constexpr int IN_VEC = VEC * STRIDE;                    // aligned body columns
  const int wv = p.Wo / VEC;
  const size_t total = (size_t)p.in.N * p.in.C * p.Ho * wv;
  const float inv = 1.f / (float)(K * K);
  const T* x = reinterpret_cast<const T*>(p.in.x);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int vx = (int)(i % wv);
    const int oy = (int)((i / wv) % p.Ho);
    const size_t nc = i / ((size_t)wv * p.Ho);
    const int c = (int)(nc % p.in.C), n = (int)(nc / p.in.C);
    const int ox0 = vx * VEC;
    const int w0 = ox0 * STRIDE - PAD;   // first input column of the span
    const int h0 = oy * STRIDE - PAD;
    float acc[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) acc[j] = (p.mode == SPC_POOL_MAX) ? -INFINITY : 0.f;
#pragma unroll
    for (int a = 0; a < K; ++a) {
      const int h = h0 + a;
      float row[SPAN];
      const bool row_in = (unsigned)h < (unsigned)p.in.H;
      if (row_in) {
        // body: columns [w0+PAD, w0+PAD+IN_VEC) are aligned to IN_VEC elements
        const T* src = x + (((size_t)n * p.in.C + c) * p.in.H + h) * p.in.W + (w0 + PAD);
        if constexpr (sizeof(T) * IN_VEC % 16 == 0) {
          constexpr int NV = sizeof(T) * IN_VEC / 16;
          uint4 raw[NV];
#pragma unroll
          for (int q = 0; q < NV; ++q) raw[q] = __ldg(reinterpret_cast<const uint4*>(src) + q);
          const T* e = reinterpret_cast<const T*>(raw);
#pragma unroll
          for (int q = 0; q < IN_VEC; ++q)
            if (PAD + q < SPAN) row[PAD + q] = to_f32<T>(e[q]);
        } else {
#pragma unroll
          for (int q = 0; q < IN_VEC; ++q)
            if (PAD + q < SPAN) row[PAD + q] = to_f32<T>(src[q]);
        }
#pragma unroll
        for (int q = 0; q < PAD; ++q) row[q] = tile_load<T>(p.in, n, c, h, w0 + q);
#pragma unroll
        for (int q = PAD + IN_VEC; q < SPAN; ++q) row[q] = tile_load<T>(p.in, n, c, h, w0 + q);
      } else {
#pragma unroll
        for (int q = 0; q < SPAN; ++q) row[q] = tile_load<T>(p.in, n, c, h, w0 + q);
      }
#pragma unroll
      for (int j = 0; j < VEC; ++j)
#pragma unroll
        for (int b = 0; b < K; ++b) {
          const float v = row[j * STRIDE + b];
          acc[j] = (p.mode == SPC_POOL_MAX) ? pool_max(acc[j], v) : acc[j] + v;
        }
    }
    T outv[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) outv[j] = from_f32<T>((p.mode == SPC_POOL_AVG) ? acc[j] * inv : acc[j]);
    T* dst = reinterpret_cast<T*>(p.out) + (((size_t)n * p.in.C + c) * p.Ho + oy) * p.Wo + ox0;
    if constexpr (sizeof(T) * VEC == 16) {
      *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(outv);
    } else if constexpr (sizeof(T) * VEC == 8) {
      *reinterpret_cast<uint2*>(dst) = *reinterpret_cast<const uint2*>(outv);
    } else {
#pragma unroll
      for (int j = 0; j < VEC; ++j) dst[j] = outv[j];
    }
  }
}

// ---- forward, 3x3 window, warp-cooperative edges ---------------------------------------------
// Like pool_fwd_vec_kernel, but the window overhang (one column left, and one right for stride
// 1) comes from the neighbouring lanes' vectors through warp shuffles; only lanes at a warp or
// row boundary fall back to a scalar load.  Every lane of a warp walks the loop together.
template <typename T, int VEC, int STRIDE>
__global__ void __launch_bounds__(256)
pool3_fwd_kernel(const PoolParams p) {
  constexpr int IN_VEC = VEC * STRIDE;
  constexpr int SPAN = (VEC - 1) * STRIDE + 3;
  const int wv = p.Wo / VEC;
  const size_t total = (size_t)p.in.N * p.in.C * p.Ho * wv;
  const float inv = 1.f / 9.f;
  const T* x = reinterpret_cast<const T*>(p.in.x);
  const int lane = threadIdx.x & 31;
  const size_t warp0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) - lane;
  for (size_t base = warp0; base < total; base += (size_t)gridDim.x * blockDim.x) {
    const size_t i = base + lane;
    const bool valid = i < total;
    const size_t ii = valid ? i : total - 1;
    const int vx = (int)(ii % wv);
    const int oy = (int)((ii / wv) % p.Ho);
    const size_t nc = ii / ((size_t)wv * p.Ho);
    const int c = (int)(nc % p.in.C), n = (int)(nc / p.in.C);
    const int ox0 = vx * VEC;
    const int w0 = ox0 * STRIDE - 1;
    const int h0 = oy * STRIDE - 1;
    float acc[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) acc[j] = (p.mode == SPC_POOL_MAX) ? -INFINITY : 0.f;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const int h = h0 + a;
      float row[SPAN];
      const bool row_in = (unsigned)h < (unsigned)p.in.H;   // uniform across a row of outputs, not a warp
      float body[IN_VEC];
      if (row_in) {
        load_vec<T, IN_VEC>(x + (((size_t)n * p.in.C + c) * p.in.H + h) * p.in.W + (w0 + 1), body);
      } else {
#pragma unroll
        for (int q = 0; q < IN_VEC; ++q) body[q] = tile_load<T>(p.in, n, c, h, w0 + 1 + q);
      }
      // neighbours' edge elements (all 32 lanes participate)
      float left = __shfl_up_sync(0xffffffffu, body[IN_VEC - 1], 1);
      float right = __shfl_down_sync(0xffffffffu, body[0], 1);
      if (lane == 0 || vx == 0) left = tile_load<T>(p.in, n, c, h, w0);
      if (STRIDE == 1 && (lane == 31 || vx == wv - 1)) right = tile_load<T>(p.in, n, c, h, w0 + 1 + IN_VEC);
      row[0] = left;
#pragma unroll
      for (int q = 0; q < IN_VEC; ++q)
        if (1 + q < SPAN) row[1 + q] = body[q];
      if (STRIDE == 1) row[SPAN - 1] = right;
#pragma unroll
      for (int j = 0; j < VEC; ++j)
#pragma unroll
        for (int b = 0; b < 3; ++b) {
          const float v = row[j * STRIDE + b];
          acc[j] = (p.mode == SPC_POOL_MAX) ? pool_max(acc[j], v) : acc[j] + v;
        }
    }
    if (valid) {
      float outv[VEC];
#pragma unroll
      for (int j = 0; j < VEC; ++j) outv[j] = (p.mode == SPC_POOL_AVG) ? acc[j] * inv : acc[j];
      store_vec<T, VEC>(reinterpret_cast<T*>(p.out) + (((size_t)n * p.in.C + c) * p.Ho + oy) * p.Wo + ox0, outv);
    }
  }
}

// ---- forward, 3x3 stride 1, TMA-staged ----------------------------------------------------------
// A kernel whose warps load their own 16-byte vectors keeps only a few loads in flight per warp and
// is latency/occupancy bound.  Here one producer thread per CTA keeps P3_STAGES bulk-tensor loads of
// whole (64+2) x (16*VEC + 2*VEC) input boxes in flight; TMA's out-of-bounds zero fill IS the zero
// padding, so the 256 consumer threads run a branch-free stencil out of shared memory (one 16-byte
// vector per thread per row, neighbours by shuffle) and store 16 bytes per thread per output row.
// The box starts VEC columns left of the tile so its inner coordinate stays 16-byte aligned.
// Halos of a partitioned tile are not visible to TMA: callers re-do the 1-pixel output ring with
// pool3_s1_ring_kernel when the view has strips.
constexpr int P3_TH = 64;          // output rows per tile
constexpr int P3_STAGES = 4;
constexpr int P3_THREADS = 288;    // 8 consumer warps + 1 producer warp

template <typename T> struct P3Geom {
  static constexpr int VEC = 16 / sizeof(T);
  static constexpr int TW = 16 * VEC;                 // output columns per tile (256 bytes per row)
  static constexpr int BW = TW + 2 * VEC;             // box columns
  static constexpr int BH = P3_TH + 2;                // box rows
  static constexpr int BOX_BYTES = BW * BH * (int)sizeof(T);
  static constexpr int STAGE_BYTES = (BOX_BYTES + 1023) & ~1023;
  static constexpr int SMEM_BYTES = P3_STAGES * STAGE_BYTES + 1024 + 128;
};

template <typename T>
__global__ void __launch_bounds__(P3_THREADS, 2)
pool3_s1_tma_kernel(const __grid_constant__ CUtensorMap tmap, const PoolParams p, int tiles_w, int tiles_h,
                    int num_tiles) {
  using G = P3Geom<T>;
  constexpr int VEC = G::VEC;
  extern __shared__ uint8_t p3_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(p3_smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + P3_STAGES * G::STAGE_BYTES);
  uint64_t* empty = full + P3_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < P3_STAGES; ++i) { tc::mbar_init(&full[i], 1); tc::mbar_init(&empty[i], 8); }
    tc::fence_barrier_init();
  }
  __syncthreads();
  const int per_plane = tiles_w * tiles_h;
  if (warp == 8) {
    if (lane == 0) {
      tc::tma_prefetch_desc(&tmap);
      int s = 0, ph = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const int plane = t / per_plane, r = t - plane * per_plane;
        const int h0 = (r / tiles_w) * P3_TH, w0 = (r % tiles_w) * G::TW;
        tc::mbar_wait(&empty[s], ph ^ 1);
        tc::mbar_arrive_expect_tx(&full[s], G::BOX_BYTES);
        tc::tma_load_3d(smem + s * G::STAGE_BYTES, &tmap, &full[s], w0 - VEC, h0 - 1, plane);
        if (++s == P3_STAGES) { s = 0; ph ^= 1; }
      }
    }
    return;
  }
  const int cg = threadIdx.x & 15;          // 16-byte column group inside the tile
  const int rs = threadIdx.x >> 4;          // 4-row segment (0..15)
  const bool is_max = p.mode == SPC_POOL_MAX;
  const float inv = 1.f / 9.f;
  T* out = reinterpret_cast<T*>(p.out);
  int s = 0, ph = 0;
  for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
    const int plane = t / per_plane, r = t - plane * per_plane;
    const int h0 = (r / tiles_w) * P3_TH, w0 = (r % tiles_w) * G::TW;
    tc::mbar_wait(&full[s], ph);
    const T* sm = reinterpret_cast<const T*>(smem + s * G::STAGE_BYTES) + (rs * 4) * G::BW + VEC + cg * VEC;
    const int wq = w0 + cg * VEC;
    float h0v[VEC], h1v[VEC], h2v[VEC];
#pragma unroll
    for (int q = 0; q < VEC; ++q) { h0v[q] = 0.f; h1v[q] = 0.f; h2v[q] = 0.f; }
#pragma unroll
    for (int k = 0; k < 6; ++k) {           // box rows rs*4 + k = input rows h0 + rs*4 + k - 1
      const uint4 cur = *reinterpret_cast<const uint4*>(sm + k * G::BW);
      const T* e = reinterpret_cast<const T*>(&cur);
      float body[VEC];
#pragma unroll
      for (int q = 0; q < VEC; ++q) body[q] = to_f32<T>(e[q]);
      float left = __shfl_up_sync(0xffffffffu, body[VEC - 1], 1, 16);
      float right = __shfl_down_sync(0xffffffffu, body[0], 1, 16);
      if (cg == 0) left = to_f32<T>(sm[k * G::BW - 1]);
      if (cg == 15) right = to_f32<T>(sm[k * G::BW + VEC]);
#pragma unroll
      for (int q = 0; q < VEC; ++q) {
        h0v[q] = h1v[q];
        h1v[q] = h2v[q];
        const float a = q == 0 ? left : body[q - 1];
        const float b = q == VEC - 1 ? right : body[q + 1];
        h2v[q] = is_max ? pool_max(pool_max(a, body[q]), b) : (a + body[q] + b);
      }
      if (k >= 2) {
        const int h = h0 + rs * 4 + k - 2;
        if (h < p.in.H && wq < p.in.W) {
          float outv[VEC];
#pragma unroll
          for (int q = 0; q < VEC; ++q)
            outv[q] = is_max ? pool_max(pool_max(h0v[q], h1v[q]), h2v[q]) : (h0v[q] + h1v[q] + h2v[q]) * inv;
          store_vec<T, VEC>(out + ((size_t)plane * p.in.H + h) * p.in.W + wq, outv);
        }
      }
    }
    __syncwarp();
    if (lane == 0) tc::mbar_arrive(&empty[s]);
    if (++s == P3_STAGES) { s = 0; ph ^= 1; }
  }
}

// 1-pixel output ring of a 3x3 stride-1 pool, through the tile + halo view
template <typename T>
__global__ void pool3_s1_ring_kernel(const PoolParams p) {
  const int H = p.in.H, W = p.in.W;
  const int ring = (H >= 2 ? 2 * W : W) + (H > 2 ? 2 * (H - 2) : 0);
  const size_t total = (size_t)p.in.N * p.in.C * ring;
  const bool is_max = p.mode == SPC_POOL_MAX;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(i % ring);
    const size_t nc = i / ring;
    const int c = (int)(nc % p.in.C), n = (int)(nc / p.in.C);
    int h, w;
    if (r < W) { h = 0; w = r; }
    else if (H >= 2 && r < 2 * W) { h = H - 1; w = r - W; }
    else { const int q = r - 2 * W; h = 1 + (q >> 1); w = (q & 1) ? W - 1 : 0; }
    float acc = is_max ? -INFINITY : 0.f;
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
      for (int dx = -1; dx <= 1; ++dx) {
        const float v = tile_load<T>(p.in, n, c, h + dy, w + dx);
        acc = is_max ? pool_max(acc, v) : acc + v;
      }
    reinterpret_cast<T*>(p.out)[(nc * H + h) * (size_t)W + w] = from_f32<T>(is_max ? acc : acc * (1.f / 9.f));
  }
}

// x viewed as [planes][H][W]
template <typename T>
int launch_pool3_tma(const PoolParams& p, cudaStream_t st) {
  using G = P3Geom<T>;
  SPC_REQUIRE(p.in.x != nullptr && (uintptr_t)p.in.x % 16 == 0 && ((size_t)p.in.W * sizeof(T)) % 16 == 0,
              "pool: TMA needs a 16-byte aligned input and row pitch (W=%d)", p.in.W);
  const size_t planes = (size_t)p.in.N * p.in.C;
  CUtensorMap tm;
  const uint64_t dims[3] = {(uint64_t)p.in.W, (uint64_t)p.in.H, (uint64_t)planes};
  const uint64_t strides[3] = {0, (uint64_t)p.in.W * sizeof(T), (uint64_t)p.in.W * p.in.H * sizeof(T)};
  const uint32_t box[3] = {(uint32_t)G::BW, (uint32_t)G::BH, 1};
  int rc = make_tmap(&tm, p.in.x, sizeof(T) == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3,
                     dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE);
  if (rc) return rc;
  const int tiles_w = (p.in.W + G::TW - 1) / G::TW, tiles_h = (p.in.H + P3_TH - 1) / P3_TH;
  const size_t nt = planes * tiles_w * tiles_h;
  SPC_REQUIRE(nt < (1u << 31), "pool: too many tiles");
  auto kern = pool3_s1_tma_kernel<T>;
  rc = allow_dynamic_smem((const void*)kern, G::SMEM_BYTES);
  if (rc) return rc;
  const int sms = sm_count();
  const int grid = nt < (size_t)(2 * sms) ? (int)nt : 2 * sms;
  kern<<<grid, P3_THREADS, G::SMEM_BYTES, st>>>(tm, p, tiles_w, tiles_h, (int)nt);
  count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  bool halos = false;
  for (int i = 0; i < 9; ++i) halos = halos || p.in.strip[i] != nullptr;
  if (halos) {
    const int ring = 2 * p.in.W + 2 * p.in.H;
    const size_t total = planes * ring;
    const int blocks = (int)((total + 255) / 256 > 132 * 8 ? 132 * 8 : (total + 255) / 256);
    pool3_s1_ring_kernel<T><<<blocks, 256, 0, st>>>(p);
    count_launch();
    SPC_CHECK_CUDA(cudaGetLastError());
  }
  return SPC_OK;
}

// ---- backward: one thread per dx element (gather over the windows that cover it) -------------
template <typename T>
__global__ void pool_bwd_kernel(const PoolParams p) {
  const int H = p.in.H, W = p.in.W;
  const size_t total = (size_t)p.in.N * p.in.C * H * W;
  const float inv = 1.f / (float)(p.k * p.k);
  const T* dy = reinterpret_cast<const T*>(p.dy);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int w = (int)(i % W);
    const int h = (int)((i / W) % H);
    const size_t nc = i / ((size_t)W * H);
    const int c = (int)(nc % p.in.C), n = (int)(nc / p.in.C);
    // windows (oy,ox) with oy*stride - pad <= h <= oy*stride - pad + k - 1
    const int hp = h + p.pad, wp = w + p.pad;
    int oy_lo = (hp - p.k + 1 + p.stride - 1);
    oy_lo = oy_lo < 0 ? 0 : oy_lo / p.stride;
    int ox_lo = (wp - p.k + 1 + p.stride - 1);
    ox_lo = ox_lo < 0 ? 0 : ox_lo / p.stride;
    const int oy_hi = min(p.Ho - 1, hp / p.stride), ox_hi = min(p.Wo - 1, wp / p.stride);
    float g = 0.f;
    const T* dyp = dy + nc * (size_t)p.Ho * p.Wo;
    if (p.mode == SPC_POOL_AVG) {
      for (int oy = oy_lo; oy <= oy_hi; ++oy)
        for (int ox = ox_lo; ox <= ox_hi; ++ox) g += to_f32<T>(dyp[(size_t)oy * p.Wo + ox]);
      g *= inv;
    } else {
      for (int oy = oy_lo; oy <= oy_hi; ++oy)
        for (int ox = ox_lo; ox <= ox_hi; ++ox) {
          // argmax of window (first maximum in row-major order, ATen max_pool2d semantics)
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
    reinterpret_cast<T*>(p.out)[i] = from_f32<T>(g);
  }
}

// ---- backward, vectorised stride-2 paths (no halos, W % 16 == 0) -------------------------------
// One thread owns 8 consecutive outputs (oy, ox0..ox0+7) and writes the 2 x 16 input-gradient
// elements of rows 2*oy, 2*oy+1 as 16-byte vectors.
//  avg 3x3 s2 pad 1: dx[2m,2n]=g[m,n]; dx[2m,2n+1]=g[m,n]+g[m,n+1]; dx[2m+1,2n]=g[m,n]+g[m+1,n];
//                    dx[2m+1,2n+1]=g[m,n]+g[m,n+1]+g[m+1,n]+g[m+1,n+1]   (all / 9)
//  max 2x2 s2:       dx = g at the first maximal element of each window, else 0
template <typename T, int MODE>
__global__ void __launch_bounds__(256)
pool_bwd_s2_vec_kernel(const PoolParams p) {
  constexpr int V = 8;
  const int H = p.in.H, W = p.in.W, Ho = p.Ho, Wo = p.Wo;
  const int wv = Wo / V;
  const size_t total = (size_t)p.in.N * p.in.C * Ho * wv;
  const T* dy = reinterpret_cast<const T*>(p.dy);
  const T* x = reinterpret_cast<const T*>(p.in.x);
  T* dx = reinterpret_cast<T*>(p.out);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int vx = (int)(i % wv);
    const int oy = (int)((i / wv) % Ho);
    const size_t nc = i / ((size_t)wv * Ho);
    const int ox0 = vx * V;
    const T* g0 = dy + (nc * Ho + oy) * Wo + ox0;
    float g[V + 1], gn[V + 1];
    {
      float gv[V];
      load_vec<T, V>(g0, gv);
#pragma unroll
      for (int j = 0; j < V; ++j) g[j] = gv[j];
    }
    float o0[2 * V], o1[2 * V];
    if (MODE == SPC_POOL_AVG) {
      const bool has_r = ox0 + V < Wo, has_d = oy + 1 < Ho;
      g[V] = has_r ? to_f32<T>(g0[V]) : 0.f;
      if (has_d) {
        float gv[V];
        load_vec<T, V>(g0 + Wo, gv);
#pragma unroll
        for (int j = 0; j < V; ++j) gn[j] = gv[j];
        gn[V] = has_r ? to_f32<T>(g0[Wo + V]) : 0.f;
      } else {
#pragma unroll
        for (int j = 0; j <= V; ++j) gn[j] = 0.f;
      }
      const float inv = 1.f / 9.f;
#pragma unroll
      for (int j = 0; j < V; ++j) {
        o0[2 * j] = g[j] * inv;
        o0[2 * j + 1] = (g[j] + g[j + 1]) * inv;
        o1[2 * j] = (g[j] + gn[j]) * inv;
        o1[2 * j + 1] = (g[j] + g[j + 1] + gn[j] + gn[j + 1]) * inv;
      }
    } else {
      const T* x0 = x + (nc * H + 2 * oy) * W + 2 * ox0;
      float r0[2 * V], r1[2 * V];
      load_vec<T, 2 * V>(x0, r0);
      load_vec<T, 2 * V>(x0 + W, r1);
#pragma unroll
      for (int j = 0; j < V; ++j) {
        const float a = r0[2 * j], b = r0[2 * j + 1];
        const float c = r1[2 * j], d = r1[2 * j + 1];
        // pool_max_takes' rule, unrolled for 4 elements: the first maximum, or the last NaN of a window that has one.
        // Written as the plain comparisons plus a NaN override it runs faster than the helper's per-step test
        // (6.07 vs 7.03 ms for max 2x2 s2 backward, C=208 at 4096^2 bf16, H100 80GB HBM3 at 700 W).
        int best = 0;
        float m = a;
        if (b > m) { m = b; best = 1; }
        if (c > m) { m = c; best = 2; }
        if (d > m) { m = d; best = 3; }
        if (isnan(a) || isnan(b) || isnan(c) || isnan(d)) best = isnan(d) ? 3 : isnan(c) ? 2 : isnan(b) ? 1 : 0;
        o0[2 * j] = best == 0 ? g[j] : 0.f;
        o0[2 * j + 1] = best == 1 ? g[j] : 0.f;
        o1[2 * j] = best == 2 ? g[j] : 0.f;
        o1[2 * j + 1] = best == 3 ? g[j] : 0.f;
      }
    }
    T* d0 = dx + (nc * H + 2 * oy) * W + 2 * ox0;
    store_vec<T, 2 * V>(d0, o0);
    store_vec<T, 2 * V>(d0 + W, o1);
  }
}

template <typename T>
int run_fwd(const PoolParams& p, cudaStream_t st) {
  const size_t total = (size_t)p.in.N * p.in.C * p.Ho * p.Wo;
  if (total == 0) return SPC_OK;
  constexpr int VEC = 16 / sizeof(T);   // 8 bf16 or 4 fp32 outputs per thread
  const bool aligned = ((uintptr_t)p.in.x % 16 == 0) && ((uintptr_t)p.out % 16 == 0);
  const bool vec_ok = aligned && p.Wo % VEC == 0 && p.in.W % (VEC * p.stride) == 0 &&
                      p.in.W == p.Wo * p.stride;
  const size_t vtotal = total / VEC;
  const int blocks = (int)((vtotal + 255) / 256 > 132 * 32 ? 132 * 32 : (vtotal + 255) / 256);
  if (vec_ok && p.k == 3 && p.stride == 1) {
    return launch_pool3_tma<T>(p, st);
  } else if (vec_ok && p.k == 3 && p.stride == 2) {
    pool3_fwd_kernel<T, VEC, 2><<<blocks, 256, 0, st>>>(p);
  } else if (vec_ok && p.k == 2 && p.stride == 2) {
    pool_fwd_vec_kernel<T, VEC, 2, 2><<<blocks, 256, 0, st>>>(p);
  } else {
    const int b2 = (int)((total + 255) / 256 > 132 * 32 ? 132 * 32 : (total + 255) / 256);
    pool_fwd_kernel<T><<<b2, 256, 0, st>>>(p);
  }
  spc::count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

template <typename T>
int run_bwd(const PoolParams& p, cudaStream_t st) {
  const size_t total = (size_t)p.in.N * p.in.C * p.in.H * p.in.W;
  if (total == 0) return SPC_OK;
  const int blocks = (int)((total + 255) / 256 > 132 * 32 ? 132 * 32 : (total + 255) / 256);
  const bool aligned = ((uintptr_t)p.in.x % 16 == 0) && ((uintptr_t)p.out % 16 == 0) && ((uintptr_t)p.dy % 16 == 0);
  const bool even = aligned && p.in.W % 16 == 0 && p.in.H % 2 == 0 && p.in.W == 2 * p.Wo && p.in.H == 2 * p.Ho;
  if (p.mode == SPC_POOL_AVG && p.k == 3 && p.stride == 1 && aligned && p.in.W % (16 / sizeof(T)) == 0) {
    // avg 3x3 s1: dx = avgpool3x3(dy) with zero padding -- the forward kernel on dy, no halos
    PoolParams q = p;
    q.in = make_view(p.dy, nullptr, p.in.N, p.in.C, p.Ho, p.Wo, 1, 1);
    q.dy = nullptr;
    return launch_pool3_tma<T>(q, st);
  } else if (even && p.mode == SPC_POOL_AVG && p.k == 3 && p.stride == 2) {
    const size_t vt = total / 32;
    const int b2 = (int)((vt + 255) / 256 > 132 * 32 ? 132 * 32 : (vt + 255) / 256);
    pool_bwd_s2_vec_kernel<T, SPC_POOL_AVG><<<b2, 256, 0, st>>>(p);
  } else if (even && p.mode == SPC_POOL_MAX && p.k == 2 && p.stride == 2) {
    const size_t vt = total / 32;
    const int b2 = (int)((vt + 255) / 256 > 132 * 32 ? 132 * 32 : (vt + 255) / 256);
    pool_bwd_s2_vec_kernel<T, SPC_POOL_MAX><<<b2, 256, 0, st>>>(p);
  } else {
    pool_bwd_kernel<T><<<blocks, 256, 0, st>>>(p);
  }
  spc::count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

int fill(PoolParams& p, const spc_pool_desc* d, const void* x, const spc_halo* halo) {
  SPC_REQUIRE(d && x, "pool: null descriptor or input");
  SPC_REQUIRE(d->k >= 1 && d->stride >= 1 && d->pad == (d->k - 1) / 2,
              "pool: pad must equal floor((k-1)/2) (reference spatial.py:1457-1464), got k=%d pad=%d", d->k, d->pad);
  SPC_REQUIRE(d->mode == SPC_POOL_MAX || d->mode == SPC_POOL_AVG, "pool: bad mode %d", d->mode);
  SPC_REQUIRE(d->dtype == SPC_F32 || d->dtype == SPC_BF16, "pool: bad dtype %d", d->dtype);
  p.in = make_view(x, halo, d->N, d->C, d->H, d->W, d->pad, d->pad);
  p.k = d->k; p.stride = d->stride; p.pad = d->pad; p.mode = d->mode;
  p.Ho = (d->H + 2 * d->pad - d->k) / d->stride + 1;
  p.Wo = (d->W + 2 * d->pad - d->k) / d->stride + 1;
  return SPC_OK;
}

}  // namespace
}  // namespace spc

extern "C" int spc_pool2d_fwd(const spc_pool_desc* d, const void* x, const spc_halo* halo, void* y, void* stream) {
  spc::PoolParams p{};
  int rc = spc::fill(p, d, x, halo);
  if (rc) return rc;
  p.out = y; p.dy = nullptr;
  return d->dtype == SPC_BF16 ? spc::run_fwd<__nv_bfloat16>(p, (cudaStream_t)stream)
                              : spc::run_fwd<float>(p, (cudaStream_t)stream);
}

extern "C" int spc_pool2d_bwd(const spc_pool_desc* d, const void* x, const spc_halo* halo, const void* dy,
                              void* dx, void* stream) {
  spc::PoolParams p{};
  int rc = spc::fill(p, d, x, halo);
  if (rc) return rc;
  p.out = dx; p.dy = dy;
  return d->dtype == SPC_BF16 ? spc::run_bwd<__nv_bfloat16>(p, (cudaStream_t)stream)
                              : spc::run_bwd<float>(p, (cudaStream_t)stream);
}
