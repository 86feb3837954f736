// gemm_tc.cu -- Hopper wgmma GEMM path for the 1x1 ("pointwise") convolutions that carry most of the HBM
// traffic of the AmoebaNet-D / ResNet spatial stages (SURVEY 8d), and -- over column-shifted copies of the
// input -- for the multi-tap ones.
//
// NCHW makes a 1x1 convolution a plain GEMM per image with NO layout change:
//     fprop : Y[K x P] = W [K x C] * X [C x P]        P = H*W pixels, contiguous in memory
//     dgrad : dX[C x P] = W^T[C x K] * dY[K x P]
//     wgrad : dW[K x C] = dY[K x P] * X[C x P]^T       (reduction over pixels)
// fprop/dgrad: A = (padded) weights, K-major, TMA box {64 ch, 128 rows}, SWIZZLE_128B;
//              B = activations read IN PLACE by TMA as an MN-major operand: [ch][64 px] rows of 128 B,
//              SWIZZLE_128B; accumulator D[128 out-ch x 128 px] in the registers of two consumer warpgroups.
//              The epilogue goes registers -> swizzled staging block in smem -> TMA store.
// wgrad:       both operands K-major straight from NCHW (pixels = reduction dim, contiguous).
// Box shapes:  a [64 ch][64 px] box touches 64 channel planes = 64 different 2 MB pages, and with plane strides
//              of 8..32 MB they alias in the translation cache.  Layers with multi-page planes therefore move ONE
//              5-d box per stage, dims (64 px, 8 ch, P/64 px blocks, C/8 ch groups, image): the TMA unit walks
//              8 planes at a time and visits all pixel blocks of each before moving on; smem layout
//              [group][block][8 ch][128 B], which the GMMA descriptors express through LBO / SBO.
// Warp roles (384 threads): warp 0 = TMA producer, warpgroups 1 and 2 = wgmma consumers + epilogue.
// Persistent CTAs, one per SM.
#include "common.cuh"
#include "tc_common.cuh"

namespace spc {

using namespace tc;

namespace {

constexpr int TC_THREADS = 384;
constexpr int BK = 64;                 // channels per pipeline stage (one 128-byte swizzle row of A)
constexpr int A_BLK_BYTES = 128 * BK * 2;   // one 128-row M block of A per stage: 16 KB
constexpr int B_BLK_BYTES = BK * 64 * 2;    // one 64-pixel block of B per stage: 8 KB

// ---- weight repack: Wp[tap][m][c] (bf16, zero padded to [taps][Mpad][Cpad]) -----------------------
// element = w[m*sm + c*sc + (flip ? taps-1-tap : tap)]
//   fprop: m = out channel k, c = in channel:  sm = C*RS, sc = RS, flip = 0     (w is [K][C][R][S])
//   dgrad: m = c, c = k (transposed) and the filter is rotated by 180 degrees:  sm = RS, sc = C*RS, flip = 1
__global__ void repack_weights_kernel(const __nv_bfloat16* __restrict__ w, __nv_bfloat16* __restrict__ wp, int M,
                                      int Cc, int Mpad, int Cpad, int taps, long long sm, long long sc, int flip) {
  const int total = taps * Mpad * Cpad;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int c = i % Cpad;
    const int m = (i / Cpad) % Mpad;
    const int tap = i / (Cpad * Mpad);
    __nv_bfloat16 v = __float2bfloat16(0.f);
    if (m < M && c < Cc) v = w[(size_t)m * sm + (size_t)c * sc + (flip ? taps - 1 - tap : tap)];
    wp[i] = v;
  }
}

// ---- fprop / dgrad kernel -----------------------------------------------------------------------
constexpr int BN = 128;                       // pixels per tile (two 64-pixel swizzle blocks)
constexpr int OUT_BUF_BYTES = 128 * 128 * 2;  // epilogue staging: one 128-channel block of the tile's 128 pixels
constexpr int MAX_STAGES = 8;

struct PwParams {
  int M;                       // valid output channels
  int Cin;                     // reduction length (input channels)
  int P;                       // pixels per image
  int N;                       // images
  int tiles_per_image;
  int num_mg;                  // groups of MB*128 output channels (X tile re-read per group, from L2)
  int num_tiles;               // N * tiles_per_image * num_mg
  int stages;                  // pipeline depth (runtime, <= MAX_STAGES)
  int wres;                    // 1: all weight chunks stay resident in smem (loaded once per CTA)
  int out_bufs;                // 1 or 2 epilogue staging buffers
  int taps, S, ph, pw;         // filter taps (R*S), filter width, zero padding (tap mode)
  int W, Mpad;                 // image width (tap mode: tiles are 64-pixel row segments), padded M
  int shiftN;                  // N when the activations are S column-shifted copies, else 0
  int rowmul;                  // input row = rowmul * output row + tap row offset (2 for stride-2 convs)
  const __nv_bfloat16* bias;   // [M] or null
  int x5, y5;                  // 1: activations / outputs move as ONE 5-d box per tile whose traversal order is
                               // (8-channel group, 64-pixel block, channel, pixel): the TMA unit touches 8 channel
                               // planes (2 MB pages each) at a time and visits both pixel blocks of each before moving
                               // on, instead of walking 64 / 128 planes per pixel block (address-translation reach)
};

// Warp roles (384 threads = 3 warpgroups): warp 0 = TMA producer; warpgroups 1 and 2 = consumers.  Consumer g issues the
// wgmma (M = 64) for rows [64 g, 64 g + 64) of every 128-row block of output channels, keeps those accumulators in
// registers and writes them back through a swizzled staging block in smem and TMA stores.
template <int MB>
__global__ void __launch_bounds__(TC_THREADS, 1)
pw_gemm_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x,
               const __grid_constant__ CUtensorMap tmap_x4, const __grid_constant__ CUtensorMap tmap_y,
               const PwParams p) {
  constexpr int NB = BN / 64;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int kchunks = (p.Cin + BK - 1) / BK;
  const int iters = p.taps * kchunks;      // K loop: (filter tap, 64-channel chunk)
  const int wres_bytes = p.wres ? iters * MB * A_BLK_BYTES : 0;
  const int stage_bytes = (p.wres ? 0 : MB * A_BLK_BYTES) + NB * B_BLK_BYTES;
  uint8_t* wres = smem;
  uint8_t* stage0 = smem + wres_bytes;
  uint8_t* outbuf = stage0 + p.stages * stage_bytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(outbuf + p.out_bufs * OUT_BUF_BYTES);
  uint64_t* empty = full + MAX_STAGES;
  uint64_t* wfull = empty + MAX_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool x5 = p.x5, y5 = p.y5;

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.stages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 2); }   // empty: one per consumer
    mbar_init(wfull, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    // ================= TMA producer =================
    if (lane == 0) {
      tma_prefetch_desc(&tmap_w);
      tma_prefetch_desc(&tmap_x);
      if (p.wres) {
        // weights-stationary (one group of output channels): the CTA keeps the (padded) filter rows in smem for its
        // whole life
        mbar_arrive_expect_tx(wfull, wres_bytes);
        for (int it = 0; it < iters; ++it)
#pragma unroll
          for (int mb = 0; mb < MB; ++mb)
            tma_load_2d(wres + (it * MB + mb) * A_BLK_BYTES, &tmap_w, wfull, (it % kchunks) * BK,
                        (it / kchunks) * p.Mpad + mb * 128);
      }
      int s = 0, ph = 0;
      for (int tl = 0; tl * (int)gridDim.x < p.num_tiles; ++tl) {   // the consumers' tile order
        const int t = tl * gridDim.x + blockIdx.x;
        if (t >= p.num_tiles) continue;
        const int mg = t % p.num_mg;
        const int tt = t / p.num_mg;
        const int n = tt / p.tiles_per_image;
        const int p0 = (tt % p.tiles_per_image) * BN;
        for (int it = 0; it < iters; ++it) {
          const int kc = it % kchunks, tap = it / kchunks;
          mbar_wait(&empty[s], ph ^ 1);
          uint8_t* st = stage0 + s * stage_bytes;
          mbar_arrive_expect_tx(&full[s], stage_bytes);
          if (!p.wres) {
#pragma unroll
            for (int mb = 0; mb < MB; ++mb)
              tma_load_2d(st + mb * A_BLK_BYTES, &tmap_w, &full[s], kc * BK, tap * p.Mpad + mg * (MB * 128) + mb * 128);
            st += MB * A_BLK_BYTES;
          }
          if (p.taps == 1) {
            if (x5) {
              tma_load_5d(st, &tmap_x, &full[s], 0, 0, p0 >> 6, kc * (BK / 8), n);
            } else {
#pragma unroll
              for (int j = 0; j < NB; ++j) tma_load_3d(st + j * B_BLK_BYTES, &tmap_x, &full[s], p0 + j * 64, kc * BK, n);
            }
          } else {
            // shifted window of this tap; out-of-image rows / columns are zero-filled by TMA (= zero padding)
            const int dr = tap / p.S - p.ph;
            const int img = n + (tap % p.S) * p.shiftN;   // column shift = which pre-shifted copy
#pragma unroll
            for (int j = 0; j < NB; ++j) {
              const int q = p0 + j * 64, hq = q / p.W, wq = q - hq * p.W;
              tma_load_4d(st + j * B_BLK_BYTES, &tmap_x4, &full[s], wq, hq * p.rowmul + dr, kc * BK, img);
            }
          }
          if (++s == p.stages) { s = 0; ph ^= 1; }
        }
      }
    }
  } else if (threadIdx.x >= 128) {
    // ================= consumers: wgmma + epilogue =================
    const int wg = (threadIdx.x >> 7) - 1;     // rows [64 wg, 64 wg + 64) of every 128-row block
    const int w4 = (threadIdx.x >> 5) & 3;     // warp inside the warpgroup: fragment rows 16 w4 + lane / 4 (+ 8)
    const bool wg_lead = (threadIdx.x & 127) == 0;
    const bool leader = threadIdx.x == 128;    // issues the TMA stores
    float acc[MB][BN / 2];
    if (p.wres) mbar_wait(wfull, 0);
    int s = 0, ph = 0, ob = 0;
    // tiles blockIdx.x + k gridDim.x, counted in rounds: the loop `t += gridDim.x` costs pw_gemm_kernel<2> a register
    // spill in the epilogue
    for (int tl = 0; tl * (int)gridDim.x < p.num_tiles; ++tl) {
      const int t = tl * gridDim.x + blockIdx.x;
      if (t >= p.num_tiles) continue;
      const int mg = t % p.num_mg;
      const int tt = t / p.num_mg;
      const int n = tt / p.tiles_per_image;
      const int p0 = (tt % p.tiles_per_image) * BN;
      bool live[MB];                           // this warpgroup's 64 rows of block mb hold valid output channels
#pragma unroll
      for (int mb = 0; mb < MB; ++mb) live[mb] = mg * (MB * 128) + mb * 128 + 64 * wg < p.M;
      int prev = -1;
      for (int it = 0; it < iters; ++it) {
        mbar_wait(&full[s], ph);
        const uint32_t st = smem_u32(stage0 + s * stage_bytes);
        const uint32_t sa = p.wres ? smem_u32(wres + it * MB * A_BLK_BYTES) : st;
        const uint32_t sb = p.wres ? st : st + MB * A_BLK_BYTES;
        // always 4 k-steps and every block: wgmma under a data-dependent branch is serialised by ptxas (C7520); the
        // channels past Cin are zero in both operands (TMA zero fill, zero-padded weights), and so are the weight
        // rows past M
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          // B: MN-major SW128. 16 channels = two 8-row groups (SBO = 1024 B); 64-px blocks at LBO = 8 KB
          // (5-d box layout [8-ch group][px block][8 ch][128 B]: px blocks at LBO = 1 KB, channel groups at SBO = 2 KB)
          const uint64_t bdesc = x5 ? gmma_desc(sb + ks * (NB * 2048), 1024, NB * 1024)
                                    : gmma_desc(sb + ks * 2048, B_BLK_BYTES, 1024);
#pragma unroll
          for (int mb = 0; mb < MB; ++mb) {
            // A: K-major SW128. 8-row groups at SBO = 1024 B (this warpgroup's 64 rows start 8 KB in); +32 B per k-step
            const uint64_t adesc = gmma_desc(sa + mb * A_BLK_BYTES + wg * 8192 + ks * 32, 16, 1024);
            Wgmma<BN, 1>::mma(acc[mb], adesc, bdesc, (it | ks) ? 1u : 0u);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();                         // the previous stage's MMAs are done reading it
        if (prev >= 0 && wg_lead) mbar_arrive(&empty[prev]);
        prev = s;
        if (++s == p.stages) { s = 0; ph ^= 1; }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int mb = 0; mb < MB; ++mb) reg_fence(acc[mb]);
      if (prev >= 0 && wg_lead) mbar_arrive(&empty[prev]);
      // ===== epilogue: registers -> swizzled smem -> TMA store of [128 ch][64 px] boxes =====
#pragma unroll
      for (int mb = 0; mb < MB; ++mb) {
        const int k0 = mg * (MB * 128) + mb * 128;
        if (k0 >= p.M) break;                       // block-uniform: nothing valid in this block
        uint8_t* buf = outbuf + ob * OUT_BUF_BYTES;
        // the TMA store that last read this buffer must have finished reading it
        if (leader) { if (p.out_bufs == 2) tma_store_wait_read<1>(); else tma_store_wait_read<0>(); }
        named_bar_sync(1, 256);
        if (live[mb]) {
          const int r0 = 64 * wg + 16 * w4 + (lane >> 2);   // fragment rows r0 and r0 + 8 of the block
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = r0 + 8 * h;
            const int k = k0 + r;
            const float bias = (k < p.M && p.bias) ? __bfloat162float(p.bias[k]) : 0.f;
#pragma unroll
            for (int q = 0; q < BN / 8; ++q) {          // 8-pixel column group q: pixels 8q + 2 (lane % 4) + {0, 1}
              const int j = q >> 3;                     // 64-pixel block
              uint8_t* rowp = y5 ? buf + (r >> 3) * 2048 + j * 1024 + (r & 7) * 128 : buf + j * (128 * 128) + r * 128;
              const uint32_t v = pack_bf16x2(acc[mb][4 * q + 2 * h] + bias, acc[mb][4 * q + 2 * h + 1] + bias);
              // SWIZZLE_128B: 16-B chunk ^ (row % 8)
              *reinterpret_cast<uint32_t*>(rowp + (((q & 7) ^ (r & 7)) << 4) + (lane & 3) * 4) = v;
            }
          }
        }
        fence_proxy_async();        // make the smem writes visible to the TMA (async proxy)
        named_bar_sync(1, 256);
        if (leader) {
          if (y5) {
            tma_store_5d(&tmap_y, buf, 0, 0, p0 >> 6, k0 >> 3, n);
          } else {
#pragma unroll
            for (int j = 0; j < 2; ++j) tma_store_3d(&tmap_y, buf + j * (128 * 128), p0 + j * 64, k0, n);
          }
          tma_store_commit();
        }
        if (p.out_bufs == 2) ob ^= 1;
      }
    }
    if (leader) tma_store_wait_read<0>();
  }
}

constexpr int SMEM_LIMIT = 222 * 1024;   // of H100's 227 KB per block: room for a small co-resident kernel (halo post/collect)
constexpr int SMEM_AUX = 1024 /*align*/ + 512 /*barriers*/;

template <int MB>
int launch_pw(const CUtensorMap& tw, const CUtensorMap& tx, const CUtensorMap& tx4, const CUtensorMap& ty, PwParams p,
              cudaStream_t st) {
  const int kchunks = (p.Cin + BK - 1) / BK;
  const int budget = SMEM_LIMIT - SMEM_AUX;
  const int wres_bytes = p.taps * kchunks * MB * A_BLK_BYTES;
  const int sms = sm_count();
  const int grid = p.num_tiles < sms ? p.num_tiles : sms;
  // stationary weights: only with one group of output channels (every CTA then needs the same filter rows)
  p.wres = (wres_bytes <= 128 * 1024 && p.num_mg == 1) ? 1 : 0;
  const int stage_bytes = (p.wres ? 0 : MB * A_BLK_BYTES) + (BN / 64) * B_BLK_BYTES;
  const int rem = budget - (p.wres ? wres_bytes : 0);
  p.out_bufs = 2;
  p.stages = (rem - 2 * OUT_BUF_BYTES) / stage_bytes;
  if (p.stages < 3) { p.out_bufs = 1; p.stages = (rem - OUT_BUF_BYTES) / stage_bytes; }
  if (p.stages > MAX_STAGES) p.stages = MAX_STAGES;
  SPC_REQUIRE(p.stages >= 2, "wgmma conv: shared memory budget too small (MB=%d kchunks=%d)", MB, kchunks);
  const int smem = (p.wres ? wres_bytes : 0) + p.stages * stage_bytes + p.out_bufs * OUT_BUF_BYTES + SMEM_AUX;
  auto kern = pw_gemm_kernel<MB>;
  const int rc = allow_dynamic_smem((const void*)kern, SMEM_LIMIT);
  if (rc) return rc;
  kern<<<grid, TC_THREADS, smem, st>>>(tw, tx, tx4, ty, p);
  count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

int make_act_tmap(CUtensorMap* m, const void* base, int P, int Cc, int N, int box_rows) {
  const uint64_t dims[3] = {(uint64_t)P, (uint64_t)Cc, (uint64_t)N};
  const uint64_t strides[3] = {0, (uint64_t)P * 2, (uint64_t)P * Cc * 2};
  const uint32_t box[3] = {64, (uint32_t)box_rows, 1};
  return make_tmap(m, base, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

// [N][Cc][P] bf16 as (64 px, 8 channels, P/64 pixel blocks, Cc/8 channel groups, N): one box = `groups` channel
// groups x `blocks` pixel blocks, laid out in shared memory as [group][block][8 ch][128 B]
int make_act_tmap5(CUtensorMap* m, const void* base, int P, int Cc, int N, int groups, int blocks) {
  const uint64_t dims[5] = {64, 8, (uint64_t)P / 64, (uint64_t)Cc / 8, (uint64_t)N};
  const uint64_t strides[5] = {0, (uint64_t)P * 2, 128, (uint64_t)P * 16, (uint64_t)P * Cc * 2};
  const uint32_t box[5] = {64, 8, (uint32_t)blocks, (uint32_t)groups, 1};
  return make_tmap(m, base, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

int launch_shift_copies(const void* x, void* xs, size_t planes, int H, int W, int S, int pw, int cs, cudaStream_t st);

// Geometry of one wgmma convolution launch (fprop, or dgrad expressed as a convolution of dY).
struct TcConv {
  const __nv_bfloat16* w;      // original filter [K][C][R][S], repacked into wp; null: wp holds the packed weights
  __nv_bfloat16* wp;           // weights in [taps][Mpad][Cpad] layout (1024-aligned)
  long long sm, sc;            // strides of (output channel m, reduction channel c) in w
  int flip;                    // rotate taps by 180 degrees (dgrad)
  int M, Cin;                  // output channels, reduction channels
  int R, S, ph, pw;            // filter and zero padding
  int H, W, N;                 // input image
  int stride;                  // 1 or 2 (both axes)
};

// How one op of a bf16 convolution runs (tc_plan picks it)
enum class TcRoute {
  None,       // no tensor-core kernel for this op
  Pw,         // 1x1: pw_gemm_kernel, or pw_px_gemm_kernel (gemm_px.cu) where the plan gives a tile width; pw_wgrad_kernel
  PwS2,       // 1x1 stride 2: the same kernels on subsampled x (fprop, wgrad), or before a zero-upsample of dx (dgrad)
  Tap,        // multi-tap without shifted copies: conv_tap_kernel (fprop, dgrad), wgrad_tap_kernel (wgrad)
  TapGemm,    // multi-tap on pw_gemm_kernel / pw_wgrad_kernel in tap mode, over x or its shifted copies
  ParityS2,   // dgrad of a 3x3 stride-2 conv: the four parity classes of dx as one 2x2-tap GEMM over dy, then interleave
};

// Output channels per tile of pw_px_gemm_kernel for a layer with M output channels, or 0 where its tiles would not fit
// M clearly better than pw_gemm_kernel's, which computes 128-row blocks in groups of two (M <= 128: one block).  NT is
// the smallest instantiated tile width (56, 104, 208) that holds M, else 208 in several groups.  The tiles must waste
// fewer MMA rows than the 128-row blocks and hold at least 90 % valid channels: 52 -> 56, 104 -> 104, 208 k -> k groups
// of 208; 16, 64, 128 and 256 channels stay on pw_gemm_kernel.
int px_tile_channels(int M) {
  const int nt = M <= 56 ? 56 : (M <= 104 ? 104 : 208);
  const int pad = round_up(M, nt);
  const int blocks = (M + 127) / 128;
  const int old_rows = (blocks >= 2 ? round_up(blocks, 2) : 1) * 128;
  return (pad < old_rows && 10 * M >= 9 * pad) ? nt : 0;
}

// Y[N][M][Ho*Wo] = sum_taps Wp[tap][M x Cin] * shift_tap(X[N][Cin][H][W])  (+bias) on conv_tap_kernel (route Tap),
// pw_px_gemm_kernel (1x1, nt > 0) or pw_gemm_kernel; xs: where the column-shifted copies of X go, null for none
int run_conv_tc(const TcConv& c, TcRoute route, int nt, __nv_bfloat16* xs, const __nv_bfloat16* x,
                const __nv_bfloat16* bias, __nv_bfloat16* y, cudaStream_t st) {
  const int taps = c.R * c.S;
  const int cs = c.stride;
  const int Ho = c.H / cs, Wo = c.W / cs;
  const int Pin = c.H * c.W, P = Ho * Wo;            // P: output pixels per image
  const int rows = nt ? nt : 128;                    // output channels per weight box and output tile
  const int Mpad = round_up(c.M, rows), Cpad = round_up(c.Cin, BK);
  if (c.w) {
    const int total = taps * Mpad * Cpad;
    int blocks = (total + 255) / 256;
    if (blocks > 1184) blocks = 1184;
    repack_weights_kernel<<<blocks, 256, 0, st>>>(c.w, c.wp, c.M, c.Cin, Mpad, Cpad, taps, c.sm, c.sc, c.flip);
    count_launch();
    SPC_CHECK_CUDA(cudaGetLastError());
  }
  if (route == TcRoute::Tap)
    return run_conv_tap_v2(c.wp, Mpad, Cpad, x, bias, y, c.M, c.Cin, c.R, c.S, c.ph, c.H, c.W, c.N, st);
  if (xs) {
    int rc0 = launch_shift_copies(x, xs, (size_t)c.N * c.Cin, c.H, c.W, c.S, c.pw, cs, st);
    if (rc0) return rc0;
    x = xs;
  }
  CUtensorMap tw, tx, tx4, ty;
  // 5-d boxes (see PwParams::x5) for the layers whose channel planes span several 2 MB pages (from 4 MB planes)
  const bool box5 = (size_t)P * 2 >= ((size_t)4 << 20);
  const int x5 = (taps == 1 && cs == 1 && box5 && P % 64 == 0 && c.Cin % 8 == 0) ? 1 : 0;
  const int y5 = (taps == 1 && box5 && P % 64 == 0 && c.M % 8 == 0) ? 1 : 0;
  {
    const uint64_t dims[2] = {(uint64_t)Cpad, (uint64_t)taps * Mpad};
    const uint64_t strides[2] = {0, (uint64_t)Cpad * 2};
    const uint32_t box[2] = {BK, (uint32_t)rows};
    int rc = make_tmap(&tw, c.wp, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  int rc;
  if (taps > 1) {
    // (copies of) the input as [img][Cin][H][Wo]; img = n + s*N for the copy of filter column s
    const uint64_t dims[4] = {(uint64_t)Wo, (uint64_t)c.H, (uint64_t)c.Cin, (uint64_t)c.N * (xs ? c.S : 1)};
    const uint64_t strides[4] = {0, (uint64_t)Wo * 2, (uint64_t)c.H * Wo * 2, (uint64_t)c.H * Wo * c.Cin * 2};
    const uint32_t box[4] = {64, 1, BK, 1};
    rc = make_tmap(&tx4, x, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    tx = tx4;
  } else {
    rc = x5 ? make_act_tmap5(&tx, x, Pin, c.Cin, c.N, BK / 8, BN / 64) : make_act_tmap(&tx, x, Pin, c.Cin, c.N, BK);
    if (rc) return rc;
    tx4 = tx;
  }
  rc = y5 ? make_act_tmap5(&ty, y, P, c.M, c.N, rows / 8, 2) : make_act_tmap(&ty, y, P, c.M, c.N, rows);
  if (rc) return rc;
  if (nt) return run_pw_px(nt, tw, tx, ty, c.M, c.Cin, c.N, P, x5, y5, bias, sm_count(), st);
  PwParams p{};
  p.x5 = x5; p.y5 = y5;
  p.bias = bias; p.M = c.M; p.Cin = c.Cin; p.P = P; p.N = c.N;
  p.taps = taps; p.S = c.S; p.ph = c.ph; p.pw = c.pw; p.W = Wo; p.Mpad = Mpad;
  p.shiftN = xs ? c.N : 0;
  p.rowmul = cs;
  // groups of at most two 128-row blocks of output channels: a consumer thread holds 64 fp32 accumulators per block
  const int MBtot = Mpad / 128;
  const int mb = MBtot >= 2 ? 2 : 1;
  p.num_mg = (MBtot + mb - 1) / mb;
  p.tiles_per_image = (P + BN - 1) / BN;
  p.num_tiles = p.tiles_per_image * c.N * p.num_mg;
  return mb == 2 ? launch_pw<2>(tw, tx, tx4, ty, p, st) : launch_pw<1>(tw, tx, tx4, ty, p, st);
}

// ---- wgrad kernel: dW[K x C x taps] += dY[K x P] * shift_tap(X)[C x P]^T -------------------------
// Both operands are K-major straight from NCHW (pixels = reduction dim, contiguous).  One work
// item = (group of MG 128-row blocks of dY, one block of NBLK input channels, a pass of TG filter
// taps, a split of the pixel range); accumulators for all (tap, m-block) pairs of the item live in
// registers (NA = TG * MG <= WG_ACC / NBLK blocks of [64 rows x NBLK] per consumer thread set) and are flushed with fp32
// atomics.  NA is a template parameter and every k-step issues all NA MMAs: wgmma under a data-dependent branch is
// serialised by ptxas (C7520).  The last tap pass of a filter may use fewer than TG taps; the accumulators of its
// missing taps read stale tap slots of the stage and are never flushed.
constexpr int WG_ACC = 256;   // accumulator columns per consumer warpgroup: 128 fp32 registers per thread

struct WgParams {
  float* dw;        // [K][C][taps] fp32 (atomic accumulation)
  int K, C, P, N;
  int nblk;         // columns (input channels) per accumulator block: the kernel's NBLK
  int n_blocks;     // ceil(C / nblk)
  int MG;           // 128-row blocks of dY per item
  int mgroups;      // ceil(ceil(K/mrows) / MG)
  int splits;       // pixel-range splits per item
  int chunks_total; // N * ceil(P/64)
  int chunks_per_image;
  int stages;
  int taps, S, ph;  // filter taps (R*S), filter width, top padding
  int TG, passes;   // taps per pass, ceil(taps / TG)
  int W, shiftN;    // OUTPUT image width; N if x is the S column-shifted copies, else 0
  int rowmul;       // input row = rowmul * output row + tap row offset
  int mrows;        // dY rows per 128-row block (<= 128): K split EVENLY over its blocks, so every item streams the
                    // same number of valid rows and the CTAs that share an x chunk stay in lock-step (L2 hits)
  int pb;           // 64-pixel blocks per stage (1, or 2 = "wide" stages for 1x1 layers with multi-page channel planes)
  int dy5, x5;      // wide stages: operand moves as one 5-d box [8-ch group][px block][8 ch][128 B] (see PwParams::x5)
  int split0, nsplit;       // this launch runs splits [split0, split0 + nsplit)
  size_t slice_stride;      // split sp adds into dw + (sp - split0) * slice_stride (common.cuh: WgradSlices)
};

template <int NBLK, int NA>
__global__ void __launch_bounds__(TC_THREADS, 1)
pw_wgrad_kernel(const __grid_constant__ CUtensorMap tmap_dy, const __grid_constant__ CUtensorMap tmap_x,
                const __grid_constant__ CUtensorMap tmap_x4, const WgParams p) {
  static_assert(NA * NBLK <= WG_ACC, "accumulator registers");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int MG = p.MG;
  const int b_bytes = NBLK * 128;                          // one tap's [NBLK ch][64 px] box
  const int b_slot = (b_bytes + 1023) & ~1023;
  const int stage_bytes = p.pb * (MG * A_BLK_BYTES + p.TG * b_slot);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + p.stages * stage_bytes);
  uint64_t* empty = full + MAX_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.stages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 2); }   // empty: one per consumer
    fence_barrier_init();
  }
  __syncthreads();
  const int ngroups = p.mgroups * p.n_blocks * p.passes;
  const int it0 = p.split0 * ngroups, it1 = it0 + p.nsplit * ngroups;
  const int per_split = (p.chunks_total + p.splits - 1) / p.splits;

  // item -> (split, tap pass, channel block, m group), split-major: concurrently running CTAs cover all (m group,
  // channel block, pass) groups of the SAME pixel range, so the dY / x chunks every group re-reads come from L2, not HBM
#define WG_DECODE(it)                                                        \
  const int sp = (it) / ngroups;                                             \
  const int g_ = (it) % ngroups;                                             \
  const int pass = g_ % p.passes;                                            \
  const int nb = (g_ / p.passes) % p.n_blocks;                               \
  const int mgp = g_ / (p.passes * p.n_blocks);                              \
  const int tap0 = pass * p.TG;                                              \
  const int ntap = min(p.TG, p.taps - tap0);                                 \
  const int c_begin = sp * per_split, c_end = min(p.chunks_total, c_begin + per_split);

  if (warp == 0) {
    if (lane == 0) {
      tma_prefetch_desc(&tmap_dy);
      tma_prefetch_desc(&tmap_x);
      int s = 0, ph = 0;
      for (int it = it0 + blockIdx.x; it < it1; it += gridDim.x) {
        WG_DECODE(it)
        for (int ch = c_begin; ch < c_end; ++ch) {
          const int n = ch / p.chunks_per_image, p0 = (ch % p.chunks_per_image) * (64 * p.pb);
          mbar_wait(&empty[s], ph ^ 1);
          uint8_t* st = smem + s * stage_bytes;
          mbar_arrive_expect_tx(&full[s], p.pb * (MG * p.mrows * 128 + ntap * b_bytes));
          if (p.pb == 2) {   // wide stage (taps == 1): two 64-pixel blocks of every operand row
            for (int i = 0; i < MG; ++i) {
              uint8_t* da = st + i * (2 * A_BLK_BYTES);
              const int r0 = (mgp * MG + i) * p.mrows;
              if (p.dy5) {
                tma_load_5d(da, &tmap_dy, &full[s], 0, 0, p0 >> 6, r0 >> 3, n);
              } else {
                tma_load_3d(da, &tmap_dy, &full[s], p0, r0, n);
                tma_load_3d(da + A_BLK_BYTES, &tmap_dy, &full[s], p0 + 64, r0, n);
              }
            }
            uint8_t* xa = st + MG * (2 * A_BLK_BYTES);
            if (p.x5) {
              tma_load_5d(xa, &tmap_x, &full[s], 0, 0, p0 >> 6, (nb * NBLK) >> 3, n);
            } else {
              tma_load_3d(xa, &tmap_x, &full[s], p0, nb * NBLK, n);
              tma_load_3d(xa + b_slot, &tmap_x, &full[s], p0 + 64, nb * NBLK, n);
            }
            if (++s == p.stages) { s = 0; ph ^= 1; }
            continue;
          }
          for (int i = 0; i < MG; ++i)
            tma_load_3d(st + i * A_BLK_BYTES, &tmap_dy, &full[s], p0, (mgp * MG + i) * p.mrows, n);
          if (p.taps == 1) {
            tma_load_3d(st + MG * A_BLK_BYTES, &tmap_x, &full[s], p0, nb * NBLK, n);
          } else {
            const int hq = p0 / p.W, wq = p0 - hq * p.W;
            for (int t = 0; t < ntap; ++t) {
              const int tap = tap0 + t;
              tma_load_4d(st + MG * A_BLK_BYTES + t * b_slot, &tmap_x4, &full[s], wq, hq * p.rowmul + tap / p.S - p.ph,
                          nb * NBLK, n + (tap % p.S) * p.shiftN);
            }
          }
          if (++s == p.stages) { s = 0; ph ^= 1; }
        }
      }
    }
  } else if (threadIdx.x >= 128) {
    // ================= consumers: wgmma over rows [64 wg, 64 wg + 64) of every dY block, then the flush =================
    const int wg = (threadIdx.x >> 7) - 1;
    const int w4 = (threadIdx.x >> 5) & 3;
    const bool wg_lead = (threadIdx.x & 127) == 0;
    const bool live = 64 * wg < p.mrows;       // rows >= mrows of a block are not dY rows of this block
    float acc[NA][NBLK / 2];
    int s = 0, ph = 0;
    for (int it = it0 + blockIdx.x; it < it1; it += gridDim.x) {
      WG_DECODE(it)
      float* dw = p.dw + (size_t)(sp - p.split0) * p.slice_stride;   // the items of one split add disjoint blocks
      const int nacc = ntap * MG;              // accumulator a = (tap a / MG, dY block a % MG); a >= nacc: not flushed
      int prev = -1;
      for (int ch = c_begin; ch < c_end; ++ch) {
        mbar_wait(&full[s], ph);
        const uint32_t sa = smem_u32(smem + s * stage_bytes);
        wgmma_fence();
        {
          if (p.pb == 2) {
            // wide stage: pixel block j of a 5-d box sits 1 KB after block 0 inside every 2 KB channel group; of a pair
            // of 3-d boxes, one whole box later.  This warpgroup's 64 rows start 8 row groups (8 SBO) in.
            const uint32_t sb = sa + MG * (2 * A_BLK_BYTES);
            const uint32_t aj = p.dy5 ? 1024 : A_BLK_BYTES, asbo = p.dy5 ? 2048 : 1024;
            const uint32_t bj = p.x5 ? 1024 : b_slot, bsbo = p.x5 ? 2048 : 1024;
#pragma unroll
            for (int j = 0; j < 2; ++j) {
#pragma unroll
              for (int ks = 0; ks < 4; ++ks) {
                const uint64_t bdesc = gmma_desc(sb + j * bj + ks * 32, 16, bsbo);
#pragma unroll
                for (int a = 0; a < NA; ++a) {   // wide stages only with taps == 1: NA == MG
                  const uint64_t adesc = gmma_desc(sa + a * (2 * A_BLK_BYTES) + wg * 8 * asbo + j * aj + ks * 32, 16, asbo);
                  Wgmma<NBLK, 0>::mma(acc[a], adesc, bdesc, (ch > c_begin || ks > 0 || j > 0) ? 1u : 0u);
                }
              }
            }
          } else {
            const uint32_t sb = sa + MG * A_BLK_BYTES;
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
              for (int a = 0; a < NA; ++a) {
                const int t = a / MG, i = a - t * MG;
                const uint64_t bdesc = gmma_desc(sb + t * b_slot + ks * 32, 16, 1024);
                const uint64_t adesc = gmma_desc(sa + i * A_BLK_BYTES + wg * 8192 + ks * 32, 16, 1024);
                Wgmma<NBLK, 0>::mma(acc[a], adesc, bdesc, (ch > c_begin || ks > 0) ? 1u : 0u);
              }
            }
          }
        }
        wgmma_commit();
        wgmma_wait<1>();                         // the previous stage's MMAs are done reading it
        if (prev >= 0 && wg_lead) mbar_arrive(&empty[prev]);
        prev = s;
        if (++s == p.stages) { s = 0; ph ^= 1; }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int a = 0; a < NA; ++a) reg_fence(acc[a]);
      if (prev >= 0 && wg_lead) mbar_arrive(&empty[prev]);
      if (c_end > c_begin && live) {
#pragma unroll
        for (int a = 0; a < NA; ++a) {
          if (a < nacc) {
            const int t = a / MG, i = a - t * MG;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int rib = 64 * wg + 16 * w4 + (lane >> 2) + 8 * h;   // row inside the block
              const int k = rib < p.mrows ? (mgp * MG + i) * p.mrows + rib : p.K;
              if (k < p.K) {
#pragma unroll
                for (int q = 0; q < NBLK / 8; ++q) {
#pragma unroll
                  for (int e = 0; e < 2; ++e) {
                    const int c = nb * NBLK + 8 * q + 2 * (lane & 3) + e;
                    if (c < p.C) atomicAdd(&dw[((size_t)k * p.C + c) * p.taps + tap0 + t], acc[a][4 * q + 2 * h + e]);
                  }
                }
              }
            }
          }
        }
      }
    }
  }
#undef WG_DECODE
}

template <int NBLK, int NA>
int launch_wg(const CUtensorMap& tdy, const CUtensorMap& tx, const CUtensorMap& tx4, WgParams p, cudaStream_t st,
              const WgradSlices* sl) {
  const int b_slot = (NBLK * 128 + 1023) & ~1023;
  const int TG = NA / p.MG;                // taps per pass (chosen by launch_wg_na)
  p.TG = TG;
  p.passes = (p.taps + TG - 1) / TG;
  const int stage_bytes = p.pb * (p.MG * A_BLK_BYTES + TG * b_slot);
  p.stages = (SMEM_LIMIT - SMEM_AUX) / stage_bytes;
  if (p.stages > 6) p.stages = 6;
  SPC_REQUIRE(p.stages >= 2, "wgmma wgrad: smem budget");
  const int sms = sm_count();
  const int groups = p.mgroups * p.n_blocks * p.passes;
  // items = groups * splits on a persistent grid of `sms` CTAs.  Every item ends by adding its accumulators to dw with
  // fp32 atomics, and that flush is a chip-wide cost: with few pixels per item it dominates.  Pick the split count
  // that minimises   waves * chunks_per_item * t_chunk + items * elems_per_item / atomic_rate,
  // t_chunk = the slower of the item's MMA chain and its operand bytes at the per-SM share of L2 bandwidth
  // (estimates, not measurements: the choice only needs their ratio).
  int splits = 1;
  {
    const double clk = 1.7e9, atomic_rate = 60e9;
    const double bytes_chunk = (double)p.pb * (p.MG * p.mrows + p.TG * NBLK) * 128.0;
    const double mma_chunk = (double)p.pb * p.MG * p.TG * 4.0 * (NBLK > 64 ? NBLK : 64) / 256.0 * 256.0;
    const double t_chunk = (bytes_chunk / 32.0 > mma_chunk ? bytes_chunk / 32.0 : mma_chunk) / clk;
    const double elems = (double)p.MG * p.mrows * NBLK * p.TG;
    const int smax = (2 * sms) / groups > 1 ? (2 * sms) / groups : 1;
    double best = 1e30;
    for (int s = smax; s >= 1; --s) {        // descending: near-ties keep the finer split (better balance)
      if (s > p.chunks_total / 8 && s > 1) continue;
      const int items_s = groups * s, waves = (items_s + sms - 1) / sms;
      const double cpi = (double)((p.chunks_total + s - 1) / s);
      const double t = waves * cpi * t_chunk + (double)items_s * elems / atomic_rate;
      if (t < best * 0.98) { best = t; splits = s; }
    }
  }
  p.splits = splits;
  const int smem = p.stages * stage_bytes + SMEM_AUX;
  auto kern = pw_wgrad_kernel<NBLK, NA>;
  const int rc = allow_dynamic_smem((const void*)kern, SMEM_LIMIT);
  if (rc) return rc;
  return run_slices(sl, p.splits, (size_t)p.K * p.C * p.taps, p.dw, st, [&](int s0, int ns, float* dst, size_t stride) {
    WgParams q = p;
    q.split0 = s0; q.nsplit = ns; q.dw = dst; q.slice_stride = stride;
    const int items = groups * ns;
    kern<<<items < sms ? items : sms, TC_THREADS, smem, st>>>(tdy, tx, tx4, q);
    count_launch();
    SPC_CHECK_CUDA(cudaGetLastError());
    return SPC_OK;
  });
}

// accumulators per item: MG dY blocks x TG taps, a power of two <= WG_ACC / NBLK.  TG: all taps when they fit, else the
// most that fit the accumulator registers and leave room for >= 2 pipeline stages
template <int NBLK>
int launch_wg_na(const CUtensorMap& tdy, const CUtensorMap& tx, const CUtensorMap& tx4, const WgParams& p, cudaStream_t st,
                 const WgradSlices* sl) {
  constexpr int NACC = WG_ACC / NBLK;
  const int b_slot = (NBLK * 128 + 1023) & ~1023;
  int na = p.MG;
  while (na * 2 <= NACC && na / p.MG < p.taps &&
         p.MG * A_BLK_BYTES + (na * 2 / p.MG) * b_slot <= (SMEM_LIMIT - SMEM_AUX) / 2)
    na *= 2;
  if (na == 1) return launch_wg<NBLK, 1>(tdy, tx, tx4, p, st, sl);
  if (na == 2) return launch_wg<NBLK, 2>(tdy, tx, tx4, p, st, sl);
  if constexpr (NACC >= 4) { if (na == 4) return launch_wg<NBLK, 4>(tdy, tx, tx4, p, st, sl); }
  if constexpr (NACC >= 8) { if (na == 8) return launch_wg<NBLK, 8>(tdy, tx, tx4, p, st, sl); }
  if constexpr (NACC >= 16) { if (na == 16) return launch_wg<NBLK, 16>(tdy, tx, tx4, p, st, sl); }
  set_error("wgmma wgrad: no kernel for %d accumulators of %d channels", na, NBLK);
  return SPC_EUNSUPPORTED;
}

// x: activations [N][C][Hin][Wo] (taps == 1: Hin == Ho) or their S column-shifted (and, for
// stride 2, column-subsampled) copies [S][N][C][Hin][Wo].  Ho x Wo = extent of dy.
int run_wgrad(const __nv_bfloat16* x, const __nv_bfloat16* dy, float* dw, int K, int C, int N, int Ho, int Wo, int Hin,
              int R, int S, int ph, int stride, bool copies, cudaStream_t st, const WgradSlices* sl) {
  const int P = Ho * Wo;
  WgParams p{};
  p.dw = dw; p.K = K; p.C = C; p.P = P; p.N = N;
  p.taps = R * S; p.S = S; p.ph = ph; p.W = Wo; p.shiftN = copies ? N : 0; p.rowmul = stride;
  // accumulator width (input channels): C split evenly over blocks of <= 128, rounded up to an instantiated width
  p.n_blocks = (C + 127) / 128;
  {
    const int w = round_up((C + p.n_blocks - 1) / p.n_blocks, 16);
    p.nblk = w <= 16 ? 16 : (w <= 32 ? 32 : (w <= 64 ? 64 : 128));
  }
  int MBtot = (K + 127) / 128;
  p.mrows = round_up((K + MBtot - 1) / MBtot, 8);   // e.g. K = 416 -> 4 blocks of 104
  MBtot = (K + p.mrows - 1) / p.mrows;
  int MG = p.taps > 1 ? 1 : WG_ACC / p.nblk;
  if (MG > MBtot) MG = MBtot;
  MG = MG >= 4 ? 4 : (MG >= 2 ? 2 : 1);
  p.chunks_per_image = (P + 63) / 64;
  p.chunks_total = p.chunks_per_image * N;
  p.pb = 1;
  // wide stages (two 64-pixel blocks per operand row and stage, 5-d boxes): for 1x1 layers whose channel planes span
  // several 2 MB pages, same reason as PwParams::x5
  if (p.taps == 1 && P % 128 == 0 && (size_t)P * 2 >= ((size_t)2 << 20)) {
    const int b_slot = (p.nblk * 128 + 1023) & ~1023;
    while (MG > 1 && 2 * 2 * (MG * A_BLK_BYTES + b_slot) > SMEM_LIMIT - SMEM_AUX) MG >>= 1;
    p.pb = 2;
    p.chunks_per_image = P / 128;
    p.chunks_total = p.chunks_per_image * N;
    p.dy5 = K % 8 == 0 ? 1 : 0;   // mrows is a multiple of 8
    p.x5 = C % 8 == 0 ? 1 : 0;
  }
  p.MG = MG;
  p.mgroups = (MBtot + MG - 1) / MG;
  CUtensorMap tdy, tx, tx4;
  int rc = p.dy5 ? make_act_tmap5(&tdy, dy, P, K, N, p.mrows / 8, 2) : make_act_tmap(&tdy, dy, P, K, N, p.mrows);
  if (rc) return rc;
  if (p.taps > 1) {
    const uint64_t dims[4] = {(uint64_t)Wo, (uint64_t)Hin, (uint64_t)C, (uint64_t)N * (copies ? S : 1)};
    const uint64_t strides[4] = {0, (uint64_t)Wo * 2, (uint64_t)Hin * Wo * 2, (uint64_t)Hin * Wo * C * 2};
    const uint32_t box[4] = {64, 1, (uint32_t)p.nblk, 1};
    rc = make_tmap(&tx4, x, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    tx = tx4;
  } else {
    rc = p.x5 ? make_act_tmap5(&tx, x, P, C, N, p.nblk / 8, 2) : make_act_tmap(&tx, x, P, C, N, p.nblk);
    if (rc) return rc;
    tx4 = tx;
  }
  if (p.nblk == 16) return launch_wg_na<16>(tdy, tx, tx4, p, st, sl);
  if (p.nblk == 32) return launch_wg_na<32>(tdy, tx, tx4, p, st, sl);
  if (p.nblk == 64) return launch_wg_na<64>(tdy, tx, tx4, p, st, sl);
  return launch_wg_na<128>(tdy, tx, tx4, p, st, sl);
}

// ---- 3x3 stride-2 dgrad: the four output-parity classes of dX as channel groups of ONE 2x2-tap
// convolution over dY, then an interleave ("depth to space") pass.
//   dx[c, 2i+a, 2j+b] = sum_{u,v in {0,1}} sum_k Wq[(u,v)][(a,b)*C + c][k] * dy[k, i+u, j+v]
//   with Wq = w[k][c][r(a,u)][s(b,v)],  r(0,0)=1, r(1,0)=2, r(1,1)=0, r(0,1)=none (zero).
__global__ void repack_dgrad_s2_kernel(const __nv_bfloat16* __restrict__ w, __nv_bfloat16* __restrict__ wp, int K,
                                       int C, int Mpad, int Kpad) {
  const int total = 4 * Mpad * Kpad;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int k = i % Kpad;
    const int m = (i / Kpad) % Mpad;
    const int tap = i / (Kpad * Mpad);
    const int u = tap >> 1, v = tap & 1;
    __nv_bfloat16 val = __float2bfloat16(0.f);
    if (m < 4 * C && k < K) {
      const int cls = m / C, c = m % C;
      const int a = cls >> 1, b = cls & 1;
      const int r = a == 0 ? (u == 0 ? 1 : -1) : (u == 0 ? 2 : 0);
      const int sx = b == 0 ? (v == 0 ? 1 : -1) : (v == 0 ? 2 : 0);
      if (r >= 0 && sx >= 0) val = w[(((size_t)k * C + c) * 3 + r) * 3 + sx];
    }
    wp[i] = val;
  }
}
// dx[n][c][2i+a][2j+b] = t[n][(2a+b)*C + c][i][j]; 8 input pixels of both column classes per thread
__global__ void interleave_s2_kernel(const __nv_bfloat16* __restrict__ t, __nv_bfloat16* __restrict__ dx, int N, int C,
                                     int Ho, int Wo) {
  const int wv = Wo / 8;
  const size_t total = (size_t)N * C * 2 * Ho * wv;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int v = (int)(i % wv);
    const int oy = (int)((i / wv) % Ho);
    const int a = (int)((i / ((size_t)wv * Ho)) % 2);
    const size_t nc = i / ((size_t)wv * Ho * 2);
    const int c = (int)(nc % C);
    const size_t n = nc / C;
    const size_t plane = (size_t)Ho * Wo;
    const __nv_bfloat16* t0 = t + ((n * 4 + 2 * a) * C + c) * plane + (size_t)oy * Wo + v * 8;   // b = 0
    const uint4 e = __ldg(reinterpret_cast<const uint4*>(t0));
    const uint4 o = __ldg(reinterpret_cast<const uint4*>(t0 + (size_t)C * plane));               // b = 1
    uint4 lo, hi;
    lo.x = __byte_perm(e.x, o.x, 0x5410); lo.y = __byte_perm(e.x, o.x, 0x7632);
    lo.z = __byte_perm(e.y, o.y, 0x5410); lo.w = __byte_perm(e.y, o.y, 0x7632);
    hi.x = __byte_perm(e.z, o.z, 0x5410); hi.y = __byte_perm(e.z, o.z, 0x7632);
    hi.z = __byte_perm(e.w, o.w, 0x5410); hi.w = __byte_perm(e.w, o.w, 0x7632);
    uint4* d = reinterpret_cast<uint4*>(dx + ((nc * 2 * Ho) + 2 * oy + a) * (size_t)(2 * Wo) + v * 16);
    d[0] = lo; d[1] = hi;
  }
}

// ---- stride-2 pointwise convs: subsample / zero-upsample passes around the GEMM ------------------
// y[n,c,i,j] = x[n,c,2i,2j]; 8 outputs per thread (two 16-byte loads, one 16-byte store)
__global__ void subsample2_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, size_t planes,
                                  int H, int W) {
  const int Ho = H / 2, Wo = W / 2, wv = Wo / 8;
  const size_t total = planes * Ho * wv;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int v = (int)(i % wv);
    const int oy = (int)((i / wv) % Ho);
    const size_t pl = i / ((size_t)wv * Ho);
    const uint4* src = reinterpret_cast<const uint4*>(x + (pl * H + 2 * oy) * W + v * 16);
    const uint4 a = __ldg(src), b = __ldg(src + 1);
    uint4 o;
    o.x = __byte_perm(a.x, a.y, 0x5410);
    o.y = __byte_perm(a.z, a.w, 0x5410);
    o.z = __byte_perm(b.x, b.y, 0x5410);
    o.w = __byte_perm(b.z, b.w, 0x5410);
    *reinterpret_cast<uint4*>(y + (pl * Ho + oy) * Wo + v * 8) = o;
  }
}
// dx[n,c,2i,2j] = g[n,c,i,j], zero elsewhere
__global__ void upsample2_zero_kernel(const __nv_bfloat16* __restrict__ g, __nv_bfloat16* __restrict__ dx,
                                      size_t planes, int H, int W) {
  const int Ho = H / 2, Wo = W / 2, wv = Wo / 8;
  const size_t total = planes * Ho * wv;
  const uint4 z = make_uint4(0, 0, 0, 0);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int v = (int)(i % wv);
    const int oy = (int)((i / wv) % Ho);
    const size_t pl = i / ((size_t)wv * Ho);
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(g + (pl * Ho + oy) * Wo + v * 8));
    uint4 lo, hi;   // element e -> position 2e, zeros between
    lo.x = a.x & 0xFFFFu; lo.y = a.x >> 16; lo.z = a.y & 0xFFFFu; lo.w = a.y >> 16;
    hi.x = a.z & 0xFFFFu; hi.y = a.z >> 16; hi.z = a.w & 0xFFFFu; hi.w = a.w >> 16;
    uint4* d0 = reinterpret_cast<uint4*>(dx + (pl * H + 2 * oy) * W + v * 16);
    uint4* d1 = reinterpret_cast<uint4*>(dx + (pl * H + 2 * oy + 1) * W + v * 16);
    d0[0] = lo; d0[1] = hi; d1[0] = z; d1[1] = z;
  }
}
int launch_resample(bool up, const void* src, void* dst, size_t planes, int H, int W, cudaStream_t st) {
  const size_t total = planes * (H / 2) * (W / 16);
  size_t blocks = (total + 255) / 256;
  if (blocks > 132 * 32) blocks = 132 * 32;
  if (up)
    upsample2_zero_kernel<<<(int)blocks, 256, 0, st>>>((const __nv_bfloat16*)src, (__nv_bfloat16*)dst, planes, H, W);
  else
    subsample2_kernel<<<(int)blocks, 256, 0, st>>>((const __nv_bfloat16*)src, (__nv_bfloat16*)dst, planes, H, W);
  count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

// TMA tile loads need 16-byte aligned inner coordinates, so the
// horizontal taps of an R x S filter cannot be fetched as shifted boxes.  For S > 1 one pre-pass
// writes the S column-shifted, zero-filled copies  xs[s][plane][h][w] = x[plane][h][w + s - pw];
// every tap (r, s) is then an ALIGNED box of copy s at row offset r - ph.
// With column stride cs (stride-2 convs) the copies are also subsampled:
//     xs[s][plane][h][j] = x[plane][h][cs*j + s - pw],  j < W/cs.
__global__ void shift_copies_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ xs,
                                    size_t planes, int H, int W, int S, int pw, int cs) {
  const int Wv = W / cs;
  const int wv = Wv / 8;
  const size_t rows = planes * H;
  const size_t total = rows * wv * S;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int v = (int)(i % wv);
    const size_t row = (i / wv) % rows;
    const int sidx = (int)(i / ((size_t)wv * rows));
    const __nv_bfloat16* src = x + row * W;
    const int w0 = v * 8 * cs + sidx - pw;
    __nv_bfloat16 e[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int w = w0 + j * cs;
      e[j] = ((unsigned)w < (unsigned)W) ? src[w] : __float2bfloat16(0.f);
    }
    *reinterpret_cast<uint4*>(xs + ((size_t)sidx * rows + row) * Wv + v * 8) = *reinterpret_cast<const uint4*>(e);
  }
}
// Fast path, stride 1: one thread produces the 8-pixel vector of ALL S copies from three aligned
// 16-byte loads (previous / own / next vector); a copy shifted by `off` columns is a 16-bit
// funnel shift of that 24-element window.  |s - pw| <= 8.
template <int S, int PW>
__global__ void __launch_bounds__(256)
shift_copies_vec_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ xs, size_t planes, int H,
                        int W) {
  const int wv = W / 8;
  const size_t rows = planes * H;
  const size_t total = rows * wv;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int v = (int)(i % wv);
    const size_t row = i / wv;
    const uint4* src = reinterpret_cast<const uint4*>(x + row * W) + v;
    const uint4 z = make_uint4(0, 0, 0, 0);
    const uint4 a = v > 0 ? __ldg(src - 1) : z;
    const uint4 b = __ldg(src);
    const uint4 c = v < wv - 1 ? __ldg(src + 1) : z;
    const uint32_t win[13] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, c.x, c.y, c.z, c.w, 0u};
#pragma unroll
    for (int sidx = 0; sidx < S; ++sidx) {
      const int e0 = 8 + sidx - PW;            // first element of the window [a|b|c]: compile-time
      const int k = e0 >> 1;
      uint4 o;
      if (e0 & 1) {
        o.x = __funnelshift_r(win[k], win[k + 1], 16);
        o.y = __funnelshift_r(win[k + 1], win[k + 2], 16);
        o.z = __funnelshift_r(win[k + 2], win[k + 3], 16);
        o.w = __funnelshift_r(win[k + 3], win[k + 4], 16);
      } else {
        o.x = win[k]; o.y = win[k + 1]; o.z = win[k + 2]; o.w = win[k + 3];
      }
      *reinterpret_cast<uint4*>(xs + ((size_t)sidx * rows + row) * W + v * 8) = o;
    }
  }
}
// Fast path, stride 2, 3 filter columns, pw = 1: xs[s][j] = x[2j + s - 1]; 8 outputs per copy from the
// own 16 input pixels plus the last pixel of the previous vector.
__global__ void __launch_bounds__(256)
shift_copies_s2k3_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ xs, size_t planes, int H,
                         int W) {
  const int Wv = W / 2, wv = Wv / 8;
  const size_t rows = planes * H;
  const size_t total = rows * wv;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int v = (int)(i % wv);
    const size_t row = i / wv;
    const uint4* src = reinterpret_cast<const uint4*>(x + row * W) + 2 * v;
    const uint4 a = __ldg(src), b = __ldg(src + 1);
    const uint32_t prev = v > 0 ? (__ldg(reinterpret_cast<const uint32_t*>(src) - 1) >> 16) : 0u;   // x[16v - 1]
    uint4 ev, od, sh;
    ev.x = __byte_perm(a.x, a.y, 0x5410); ev.y = __byte_perm(a.z, a.w, 0x5410);     // x[16v + 0,2,4,...]
    ev.z = __byte_perm(b.x, b.y, 0x5410); ev.w = __byte_perm(b.z, b.w, 0x5410);
    od.x = __byte_perm(a.x, a.y, 0x7632); od.y = __byte_perm(a.z, a.w, 0x7632);     // x[16v + 1,3,5,...]
    od.z = __byte_perm(b.x, b.y, 0x7632); od.w = __byte_perm(b.z, b.w, 0x7632);
    sh.x = (od.x << 16) | prev;                                                      // x[16v - 1, 1, 3, ...]
    sh.y = __funnelshift_r(od.x, od.y, 16);
    sh.z = __funnelshift_r(od.y, od.z, 16);
    sh.w = __funnelshift_r(od.z, od.w, 16);
    __nv_bfloat16* dst = xs + row * Wv + v * 8;
    *reinterpret_cast<uint4*>(dst) = sh;                                  // s = 0: 2j - 1
    *reinterpret_cast<uint4*>(dst + rows * Wv) = ev;                      // s = 1: 2j
    *reinterpret_cast<uint4*>(dst + 2 * rows * Wv) = od;                  // s = 2: 2j + 1
  }
}
int launch_shift_copies(const void* x, void* xs, size_t planes, int H, int W, int S, int pw, int cs, cudaStream_t st) {
  const bool aligned = (reinterpret_cast<uintptr_t>(x) % 16 == 0) && (reinterpret_cast<uintptr_t>(xs) % 16 == 0);
  if (aligned && cs == 1 && W % 8 == 0 &&
      ((S == 7 && pw == 3) || (S == 3 && pw == 1) || (S == 5 && pw == 2) || (S == 2 && pw == 0))) {
    const size_t tot = planes * H * (W / 8);
    size_t blocks = (tot + 255) / 256;
    if (blocks > 132 * 32) blocks = 132 * 32;
    const __nv_bfloat16* xi = (const __nv_bfloat16*)x;
    __nv_bfloat16* xo = (__nv_bfloat16*)xs;
    if (S == 7) shift_copies_vec_kernel<7, 3><<<(int)blocks, 256, 0, st>>>(xi, xo, planes, H, W);
    else if (S == 3) shift_copies_vec_kernel<3, 1><<<(int)blocks, 256, 0, st>>>(xi, xo, planes, H, W);
    else if (S == 5) shift_copies_vec_kernel<5, 2><<<(int)blocks, 256, 0, st>>>(xi, xo, planes, H, W);
    else shift_copies_vec_kernel<2, 0><<<(int)blocks, 256, 0, st>>>(xi, xo, planes, H, W);
    count_launch();
    SPC_CHECK_CUDA(cudaGetLastError());
    return SPC_OK;
  }
  if (aligned && cs == 2 && S == 3 && pw == 1 && W % 16 == 0) {
    const size_t tot = planes * H * (W / 16);
    size_t blocks = (tot + 255) / 256;
    if (blocks > 132 * 32) blocks = 132 * 32;
    shift_copies_s2k3_kernel<<<(int)blocks, 256, 0, st>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)xs, planes, H, W);
    count_launch();
    SPC_CHECK_CUDA(cudaGetLastError());
    return SPC_OK;
  }
  const size_t total = planes * H * (W / cs / 8) * S;
  size_t blocks = (total + 255) / 256;
  if (blocks > 132 * 32) blocks = 132 * 32;
  shift_copies_kernel<<<(int)blocks, 256, 0, st>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)xs, planes, H, W, S, pw, cs);
  count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

bool tap_shape_ok(const spc_conv_desc* d) {   // odd RxS "same" convs, stride 1 or 2, on 64-pixel output row segments
  if (d->R * d->S == 1 || d->R * d->S > 49) return false;
  if ((d->R & 1) == 0 || (d->S & 1) == 0) return false;
  const bool s1 = d->stride_h == 1 && d->stride_w == 1, s2 = d->stride_h == 2 && d->stride_w == 2;
  if (!s1 && !s2) return false;
  if (s2 && (d->H % 2 || d->W % 2)) return false;
  const int Wo = d->W / d->stride_w;
  if (Wo % 64 != 0) return false;
  return (long long)d->H * d->W < (1ll << 31);
}

bool pw_shape_ok(const spc_conv_desc* d) {
  if (d->R != 1 || d->S != 1) return false;
  long long P = (long long)d->H * d->W;
  if (is_s2(d)) {
    if (d->H % 2 || d->W % 32) return false;   // 16-byte vectors on both sides of the resample
    P /= 4;
  } else if (d->stride_h != 1 || d->stride_w != 1) {
    return false;
  }
  if (P % 8 != 0 || P >= (1ll << 31)) return false;
  return true;
}

// Op 0 / 1 / 2 (fprop, dgrad, wgrad) of a bf16 convolution: its route, and where its buffers go in the workspace.
// tc_plan is the one place these are decided.
struct TcRegion {
  size_t off, bytes;   // from the workspace's first 1 KB boundary
};
struct TcPlan {
  TcRoute route;
  bool copies;         // the GEMM reads S column-shifted (stride 2: and subsampled) copies of its input, made in xs
  int nt;              // Pw / PwS2 fprop and dgrad: pw_px_gemm_kernel's tile width; 0: pw_gemm_kernel
  TcRegion wp;         // repacked weights (ParityS2: of the 2x2-tap GEMM)
  TcRegion xs;         // the shifted copies (ParityS2: of dy); PwS2: the subsampled x, or dgrad's W^T dy
  TcRegion tmp;        // ParityS2: the four parity-class planes of dx before the interleave
  size_t total;        // what spc_conv_workspace_bytes asks for: the regions plus slack for the alignment
};

TcPlan tc_plan(const spc_conv_desc* d, int op) {
  TcPlan pl{};
  const bool s2 = is_s2(d);
  const size_t taps = (size_t)d->R * d->S, N = d->N;
  const int cs = d->stride_w, Ho = d->H / cs, Wo = d->W / cs;
  // the GEMM: M output channels over Cin reduction channels (dgrad: the transposed filter over dy)
  const int M = op == 1 ? d->C : d->K, Cin = op == 1 ? d->K : d->C;
  if (d->dtype != SPC_BF16) return pl;
  if (pw_shape_ok(d)) {
    pl.route = s2 ? TcRoute::PwS2 : TcRoute::Pw;
    if (s2) pl.xs.bytes = N * d->C * Ho * Wo * 2;
    // pixel-major kernel: 1x1 layers whose output channels it tiles better, with at least two 128-pixel tiles per SM
    // (below that the persistent CTAs get one tile each and pw_gemm_kernel's 128-row blocks cost no more)
    const int nt = op == 2 ? 0 : px_tile_channels(M);
    if (nt && (long long)d->N * ((Ho * Wo + BN - 1) / BN) >= 2ll * sm_count()) pl.nt = nt;
  } else if (!tap_shape_ok(d)) {
    return pl;
  } else if (op == 1 && s2) {
    if (d->R != 3 || d->S != 3 || 4 * d->C > 2048) return pl;
    pl.route = TcRoute::ParityS2;
    pl.wp.bytes = 4ull * round_up(4 * d->C, 128) * round_up(d->K, BK) * 2;
    pl.xs.bytes = 2ull * N * d->K * Ho * Wo * 2;
    pl.tmp.bytes = 4ull * N * d->C * Ho * Wo * 2;
    pl.total = align1k(pl.wp.bytes) + align1k(pl.xs.bytes) + align1k(pl.tmp.bytes) + 8192;
  } else if (op == 2 ? wgrad_tap_supported(d->K, d->C, d->R, d->S, d->H, d->W, cs)
                     : tap_v2_supported(M, Cin, d->R, d->S, d->H, d->W, d->N, cs)) {
    pl.route = TcRoute::Tap;   // conv_tap.cu / wgrad_tap.cu form the horizontal taps in shared memory: no copies
  } else {
    pl.route = TcRoute::TapGemm;
    pl.copies = d->S > 1 || cs > 1;
    if (pl.copies) pl.xs.bytes = (size_t)d->S * N * Cin * d->H * Wo * 2;
  }
  if (pl.route != TcRoute::ParityS2) {
    // The total counts the weights at 128-row padding whatever nt is.  Where nt pads them further (M = 375..384,
    // 1124..1152, ...), the regions can outgrow it and tc_regions turns the call down.
    if (op != 2) pl.wp.bytes = taps * round_up(M, pl.nt ? pl.nt : 128) * round_up(Cin, BK) * 2;
    pl.total = (op == 2 ? 0 : taps * round_up(M, 128) * round_up(Cin, BK) * 2 + 1024) + 4096;
    if (pl.route == TcRoute::PwS2 || pl.copies) pl.total += align1k(pl.xs.bytes) + (pl.copies ? 2048 : 1024);
  }
  pl.xs.off = align1k(pl.wp.bytes);
  pl.tmp.off = align1k(pl.xs.off + pl.xs.bytes);
  return pl;
}

// The start of pl's regions in ws, once they are known to fit its ws_bytes
int tc_regions(const TcPlan& pl, void* ws, size_t ws_bytes, uint8_t** base) {
  const uintptr_t b = align1k(reinterpret_cast<uintptr_t>(ws));
  const size_t end = pl.tmp.off + pl.tmp.bytes, fit = b - reinterpret_cast<uintptr_t>(ws) + end;
  const size_t need = fit > pl.total ? fit : pl.total;
  SPC_REQUIRE(!end || (ws && ws_bytes >= need), "wgmma conv: workspace too small (%zu < %zu)", ws_bytes, need);
  *base = reinterpret_cast<uint8_t*>(b);
  return SPC_OK;
}

}  // namespace

bool tc_supported(const spc_conv_desc* d, int op) {
  const TcPlan pl = tc_plan(d, op);
  if (pl.route == TcRoute::Pw || pl.route == TcRoute::PwS2) return true;
  return pl.route != TcRoute::None && pl.total <= (24ull << 30);   // shifted copies would not fit comfortably
}

size_t tc_workspace_bytes(const spc_conv_desc* d, int op) { return tc_plan(d, op).total; }

int tc_conv_fwd(const spc_conv_desc* d, const void* x, const void* w, const void* bias, void* y, void* ws,
                size_t ws_bytes, cudaStream_t st) {
  const TcPlan pl = tc_plan(d, 0);
  uint8_t* base;
  int rc = tc_regions(pl, ws, ws_bytes, &base);
  if (rc) return rc;
  __nv_bfloat16* xs = reinterpret_cast<__nv_bfloat16*>(base + pl.xs.off);
  TcConv c{};
  c.w = reinterpret_cast<const __nv_bfloat16*>(w);
  c.wp = reinterpret_cast<__nv_bfloat16*>(base + pl.wp.off);
  c.sm = (long long)d->C * d->R * d->S; c.sc = (long long)d->R * d->S; c.flip = 0;
  c.M = d->K; c.Cin = d->C; c.R = d->R; c.S = d->S; c.ph = d->pad_h; c.pw = d->pad_w;
  c.H = d->H; c.W = d->W; c.N = d->N; c.stride = d->stride_h;
  if (pl.route == TcRoute::PwS2) {   // Y = W * subsample(X)
    rc = launch_resample(false, x, xs, (size_t)d->N * d->C, d->H, d->W, st);
    if (rc) return rc;
    x = xs; c.H /= 2; c.W /= 2; c.stride = 1;
  }
  return run_conv_tc(c, pl.route, pl.nt, pl.copies ? xs : nullptr, reinterpret_cast<const __nv_bfloat16*>(x),
                     reinterpret_cast<const __nv_bfloat16*>(bias), reinterpret_cast<__nv_bfloat16*>(y), st);
}

int tc_conv_dgrad(const spc_conv_desc* d, const void* dy, const void* w, void* dx, void* ws, size_t ws_bytes,
                  cudaStream_t st) {
  // dX[C x P] = W^T[C x K] * dY[K x P]
  const TcPlan pl = tc_plan(d, 1);
  uint8_t* base;
  int rc = tc_regions(pl, ws, ws_bytes, &base);
  if (rc) return rc;
  const __nv_bfloat16* dyb = reinterpret_cast<const __nv_bfloat16*>(dy);
  __nv_bfloat16* xs = reinterpret_cast<__nv_bfloat16*>(base + pl.xs.off);
  TcConv c{};
  c.wp = reinterpret_cast<__nv_bfloat16*>(base + pl.wp.off);
  if (pl.route == TcRoute::ParityS2) {   // four parity classes as channel groups, then interleave
    const int Ho = d->H / 2, Wo = d->W / 2;
    const int Mq = 4 * d->C, Mpad = round_up(Mq, 128), Kpad = round_up(d->K, BK);
    __nv_bfloat16* tmp = reinterpret_cast<__nv_bfloat16*>(base + pl.tmp.off);
    {
      const int total = 4 * Mpad * Kpad;
      int blocks = (total + 255) / 256;
      if (blocks > 1184) blocks = 1184;
      repack_dgrad_s2_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(w), c.wp, d->K, d->C, Mpad, Kpad);
      count_launch();
      SPC_CHECK_CUDA(cudaGetLastError());
    }
    c.M = Mq; c.Cin = d->K; c.R = 2; c.S = 2; c.ph = 0; c.pw = 0; c.H = Ho; c.W = Wo; c.N = d->N; c.stride = 1;
    rc = run_conv_tc(c, TcRoute::TapGemm, 0, xs, dyb, nullptr, tmp, st);
    if (rc) return rc;
    const size_t total = (size_t)d->N * d->C * 2 * Ho * (Wo / 8);
    size_t blocks = (total + 255) / 256;
    if (blocks > 132 * 32) blocks = 132 * 32;
    interleave_s2_kernel<<<(int)blocks, 256, 0, st>>>(tmp, reinterpret_cast<__nv_bfloat16*>(dx), d->N, d->C, Ho, Wo);
    count_launch();
    SPC_CHECK_CUDA(cudaGetLastError());
    return SPC_OK;
  }
  // correlation of dY with the transposed, 180-degree rotated filter
  c.w = reinterpret_cast<const __nv_bfloat16*>(w);
  c.sm = (long long)d->R * d->S; c.sc = (long long)d->C * d->R * d->S; c.flip = 1;
  c.M = d->C; c.Cin = d->K; c.R = d->R; c.S = d->S; c.ph = d->R - 1 - d->pad_h; c.pw = d->S - 1 - d->pad_w;
  c.H = d->H; c.W = d->W; c.N = d->N; c.stride = 1;
  if (pl.route == TcRoute::PwS2) {   // dX = zero_upsample(W^T * dY)
    c.H /= 2; c.W /= 2;
    rc = run_conv_tc(c, pl.route, pl.nt, nullptr, dyb, nullptr, xs, st);
    if (rc) return rc;
    return launch_resample(true, xs, dx, (size_t)d->N * d->C, d->H, d->W, st);
  }
  return run_conv_tc(c, pl.route, pl.nt, pl.copies ? xs : nullptr, dyb, nullptr, reinterpret_cast<__nv_bfloat16*>(dx),
                     st);
}

int tc_conv_wgrad(const spc_conv_desc* d, const void* x, const void* dy, float* dw, void* ws, size_t ws_bytes,
                  cudaStream_t st, const WgradSlices* sl) {
  // the kernels accumulate into dw with atomics; api.cu has zeroed it unless the caller accumulates
  const TcPlan pl = tc_plan(d, 2);
  uint8_t* base;
  int rc = tc_regions(pl, ws, ws_bytes, &base);
  if (rc) return rc;
  const __nv_bfloat16* xb = reinterpret_cast<const __nv_bfloat16*>(x);
  const __nv_bfloat16* dyb = reinterpret_cast<const __nv_bfloat16*>(dy);
  __nv_bfloat16* xs = reinterpret_cast<__nv_bfloat16*>(base + pl.xs.off);
  if (pl.route == TcRoute::Tap) return run_wgrad_tap(xb, dyb, dw, d->K, d->C, d->N, d->H, d->W, d->R, d->S, st, sl);
  int H = d->H, W = d->W, cs = d->stride_h;
  if (pl.route == TcRoute::PwS2) {   // dW = dY * subsample(X)^T
    rc = launch_resample(false, x, xs, (size_t)d->N * d->C, d->H, d->W, st);
    if (rc) return rc;
    xb = xs; H /= 2; W /= 2; cs = 1;
  } else if (pl.copies) {
    rc = launch_shift_copies(x, xs, (size_t)d->N * d->C, d->H, d->W, d->S, d->pad_w, cs, st);
    if (rc) return rc;
    xb = xs;
  }
  return run_wgrad(xb, dyb, dw, d->K, d->C, d->N, H / cs, W / cs, H, d->R, d->S, d->pad_h, cs, pl.copies, st, sl);
}

// Slice copies of tc_conv_wgrad: pw_wgrad_kernel (launch_wg) makes <= 2 * SMs / groups splits of a gradient of <= groups
// * 128 x 256 floats, so <= 2 * SMs * 32768 floats; wgrad_tap_kernel (run_wgrad_tap) fills <= 3 waves of items, or
// makes one slice per (image, strip) when those alone fill more
double tc_wgrad_slice_floats(const spc_conv_desc* d) {
  const double wn = (double)d->K * d->C * d->R * d->S, sms = sm_count();
  const double pw = 2.0 * sms * (wn < 32768.0 ? wn : 32768.0);
  const double tap = fmax(3.0 * sms, (double)d->N * (d->W / 64)) * wn;
  return d->R * d->S > 1 && d->stride_h == 1 && d->W % 64 == 0 ? fmax(tap, pw) : pw;
}

// Y[M][P] = W[M][Cin] * X[Cin][P] (bf16; w row-major with leading dimension ld) and dW[K][C] += dY[K][P] * X[C][P]^T on
// the pointwise wgmma kernels -- used by the halo fix-up (api.cu), where "channels" are (c, r, s) triples of the
// filter and "pixels" are the boundary outputs
size_t tc_pw_workspace_bytes(int M, int Cin) { return (size_t)round_up(M, 128) * round_up(Cin, BK) * 2 + 4096; }
int tc_pw_fwd(const void* w, int ld, int M, int Cin, const void* x, const void* bias, void* y, int P, void* ws, size_t ws_bytes,
              cudaStream_t st) {
  SPC_REQUIRE(ws && ws_bytes >= tc_pw_workspace_bytes(M, Cin), "wgmma conv: workspace too small");
  TcConv c{};
  c.w = reinterpret_cast<const __nv_bfloat16*>(w);
  c.wp = reinterpret_cast<__nv_bfloat16*>(align1k(reinterpret_cast<uintptr_t>(ws)));
  c.sm = ld; c.sc = 1; c.flip = 0;
  c.M = M; c.Cin = Cin; c.R = 1; c.S = 1; c.ph = 0; c.pw = 0; c.H = 1; c.W = P; c.N = 1; c.stride = 1;
  return run_conv_tc(c, TcRoute::Pw, 0, nullptr, reinterpret_cast<const __nv_bfloat16*>(x),
                     reinterpret_cast<const __nv_bfloat16*>(bias), reinterpret_cast<__nv_bfloat16*>(y), st);
}
int tc_pw_wgrad(const void* x, const void* dy, float* dw, int K, int C, int P, cudaStream_t st, const WgradSlices* sl) {
  return run_wgrad(reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<const __nv_bfloat16*>(dy), dw, K, C, 1, 1, P, 1, 1, 1,
                   0, 1, false, st, sl);
}

}  // namespace spc
