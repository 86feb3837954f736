// gemm_tf32.cu -- fp32 1x1 convolutions on the tensor cores in TF32 (opt-in: SPC_ALGO_TF32).
//
// Same GEMMs as gemm_tc.cu (NCHW: a 1x1 convolution is one GEMM per image), but wgmma with .tf32 operands has no
// transpose: both shared-memory operands must be K-major.  That decides the layout of each op:
//   wgrad : dW[K x C] += dY[K x P] * X[C x P]^T.  The reduction runs over pixels, contiguous in NCHW, so both operands
//           are K-major straight from TMA, as in pw_wgrad_kernel: a 128-byte SW128 row holds 32 fp32 pixels and a k8
//           step is 32 bytes, so descriptors and stage layout are those of the bf16 kernel.  The hardware uses the
//           top 19 bits of each fp32 word (truncation to tf32).
//   fprop : Y = W * X is reduced over channels, and X is pixel-contiguous (MN-major), which tf32 does not allow from
//   dgrad   shared memory.  So the kernel computes the transposed product  Y^T[P x M] = X^T[P x C] * W^T[C x M]:
//           A = X^T from registers (ld.shared from the TMA-staged [channel][32 px] rows, rounded with cvt.rna.tf32),
//           B = the weights, repacked K-major and rounded to tf32 ([M][C] for fprop, transposed for dgrad).
//           The epilogue transposes the fragments back to [channel][pixel] through a swizzled smem block, adds the
//           bias and stores with TMA.
// Stride 2: subsample / zero-upsample passes around the GEMM, as for bf16.
// Warp roles (384 threads): warp 0 = TMA producer, warpgroups 1 and 2 = wgmma consumers.  Persistent CTAs.
#include "common.cuh"
#include "tc_common.cuh"
#include "wgmma_tf32.cuh"

namespace spc {

namespace {

using namespace tc;

constexpr int T_THREADS = 384;
constexpr int T_BK = 32;                      // channels (fprop) / pixels (wgrad) per stage: one 128-byte fp32 row
constexpr int T_BN = 128;                     // pixels per fprop tile: four 32-pixel boxes
constexpr int T_XBOX = 32 * T_BK * 4;         // one [32 ch][32 px] box: 4 KB
constexpr int T_XSTAGE = 4 * T_XBOX;          // a tile's [32 ch][128 px]: 16 KB
constexpr int T_OUT_CH = 64;                  // output channels per epilogue staging block
constexpr int T_OUT_BYTES = T_OUT_CH * T_BN * 4;   // 32 KB: [4 px boxes][64 ch][128 B]
constexpr int T_MAX_STAGES = 8;
constexpr int T_SMEM_LIMIT = 222 * 1024;      // as gemm_tc.cu: room for a small co-resident kernel
constexpr int T_SMEM_AUX = 1024 /*align*/ + 512 /*barriers*/;
constexpr int T_A_BLK = 128 * 128;            // wgrad: one 128-row block of dY, 32 pixels: 16 KB

// [N][rows][P] fp32 activations, box = [box_rows][32 px]
int make_act_tmap_f32(CUtensorMap* m, const void* base, int P, int rows, int N, int box_rows) {
  const uint64_t dims[3] = {(uint64_t)P, (uint64_t)rows, (uint64_t)N};
  const uint64_t strides[3] = {0, (uint64_t)P * 4, (uint64_t)P * rows * 4};
  const uint32_t box[3] = {32, (uint32_t)box_rows, 1};
  return make_tmap(m, base, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

// ---- weight repack: Wp[m][c'] = tf32(w[m*sm + c*sc]), zero padded to [Mpad][Cpad] --------------------------------
// Inside every group of 8 channels the positions hold channels (0 2 4 6 1 3 5 7): the fprop kernel's A fragment then
// reads channel rows 2t and 2t + 1 (t = lane % 4), whose swizzled 16-byte chunks never collide (no bank conflicts).
//   fprop: m = out channel k, c = in channel:  sm = C, sc = 1      dgrad: m = c, c = k:  sm = 1, sc = C
__global__ void tf32_repack_weights_kernel(const float* __restrict__ w, float* __restrict__ wp, int M, int Cc, int Mpad,
                                           int Cpad, long long sm, long long sc) {
  const int total = Mpad * Cpad;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int pos = i % Cpad, m = i / Cpad;
    const int k = pos & 7;
    const int c = (pos & ~7) | (k < 4 ? 2 * k : 2 * k - 7);
    float v = 0.f;
    if (m < M && c < Cc) v = __uint_as_float(to_tf32(w[(size_t)m * sm + (size_t)c * sc]));
    wp[i] = v;
  }
}

// ---- fprop / dgrad kernel: Y^T[128 px x NT ch] per tile = X^T * Wp^T -------------------------------------------------
struct Tf32PwParams {
  int M;                 // valid output channels
  int Cin;               // reduction channels
  int N, tiles_per_image;
  int num_mg;            // groups of NT output channels (the X tile is re-read per group, from L2)
  int num_tiles;         // N * tiles_per_image * num_mg
  int stages;            // pipeline depth (<= T_MAX_STAGES)
  int wres;              // 1: all weight chunks stay resident in smem
  int out_bufs;          // 1 or 2 epilogue staging blocks
  const float* bias;     // [M] or null
};

// Consumer warpgroup g owns pixels [64 g, 64 g + 64) of the 128-pixel tile (the wgmma M dimension) and all NT output
// channels of its group (the N dimension): NT / 2 fp32 accumulators per thread.
template <int NT>
__global__ void __launch_bounds__(T_THREADS, 1)
tf32_pw_gemm_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x,
                    const __grid_constant__ CUtensorMap tmap_y, const Tf32PwParams p) {
  constexpr int W_BYTES = NT * 128;   // one 32-channel chunk of the group's NT weight rows
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int kchunks = (p.Cin + T_BK - 1) / T_BK;
  const int wres_bytes = p.wres ? kchunks * W_BYTES : 0;
  const int stage_bytes = (p.wres ? 0 : W_BYTES) + T_XSTAGE;
  uint8_t* wres = smem;
  uint8_t* stage0 = smem + wres_bytes;
  uint8_t* outbuf = stage0 + p.stages * stage_bytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(outbuf + p.out_bufs * T_OUT_BYTES);
  uint64_t* empty = full + T_MAX_STAGES;
  uint64_t* wfull = empty + T_MAX_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.stages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 2); }
    mbar_init(wfull, 1);
    fence_barrier_init();
  }
  __syncthreads();

  // 384 x 168 registers at launch: the producer warpgroup (one busy thread) hands its registers to the consumers,
  // whose NT / 2 accumulators and 16 A registers spill at 168 for NT = 256:  40 + 2 x 232 <= 3 x 168
  if (threadIdx.x < 128) {
    setmaxnreg_dec<40>();
    // ================= TMA producer =================
    if (warp == 0 && lane == 0) {
      tma_prefetch_desc(&tmap_w);
      tma_prefetch_desc(&tmap_x);
      if (p.wres) {
        mbar_arrive_expect_tx(wfull, wres_bytes);
        for (int kc = 0; kc < kchunks; ++kc) tma_load_2d(wres + kc * W_BYTES, &tmap_w, wfull, kc * T_BK, 0);
      }
      int s = 0, ph = 0;
      for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
        const int mg = t % p.num_mg, tt = t / p.num_mg;
        const int n = tt / p.tiles_per_image, p0 = (tt % p.tiles_per_image) * T_BN;
        for (int kc = 0; kc < kchunks; ++kc) {
          mbar_wait(&empty[s], ph ^ 1);
          uint8_t* st = stage0 + s * stage_bytes;
          mbar_arrive_expect_tx(&full[s], stage_bytes);
          if (!p.wres) {
            tma_load_2d(st, &tmap_w, &full[s], kc * T_BK, mg * NT);
            st += W_BYTES;
          }
#pragma unroll
          for (int j = 0; j < 4; ++j) tma_load_3d(st + j * T_XBOX, &tmap_x, &full[s], p0 + 32 * j, kc * T_BK, n);
          if (++s == p.stages) { s = 0; ph ^= 1; }
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    // ================= consumers: wgmma + epilogue =================
    const int wg = (threadIdx.x >> 7) - 1;
    const int w4 = (threadIdx.x >> 5) & 3;
    const int g = lane >> 2, t4 = lane & 3;
    const bool wg_lead = (threadIdx.x & 127) == 0;
    const bool leader = threadIdx.x == 128;   // issues the TMA stores
    // fragment rows: pixels pt and pt + 8 of the tile, both in 32-pixel box jb.  Element (channel row c, pixel q) of
    // a box sits at c * 128 + (((q / 4) ^ (c % 8)) * 16) + (q % 4) * 4 (SWIZZLE_128B).  A column t holds channel row
    // 2t of the k-step, column t + 4 channel row 2t + 1 (the repack's channel order).
    const int pt = 64 * wg + 16 * w4 + g;
    const int jb = pt >> 5, q4 = (pt & 31) >> 2;
    const int c0 = 2 * t4, c1 = 2 * t4 + 1;
    const uint32_t xoff0 = jb * T_XBOX + (pt & 3) * 4;
    const uint32_t off[4] = {xoff0 + c0 * 128 + ((q4 ^ c0) << 4), xoff0 + c0 * 128 + (((q4 + 2) ^ c0) << 4),
                             xoff0 + c1 * 128 + ((q4 ^ c1) << 4), xoff0 + c1 * 128 + (((q4 + 2) ^ c1) << 4)};
    float acc[NT / 2];
    if (p.wres) mbar_wait(wfull, 0);
    int s = 0, ph = 0, ob = 0;
    for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
      const int mg = t % p.num_mg, tt = t / p.num_mg;
      const int n = tt / p.tiles_per_image, p0 = (tt % p.tiles_per_image) * T_BN;
      for (int kc = 0; kc < kchunks; ++kc) {
        mbar_wait(&full[s], ph);
        const uint32_t st = smem_u32(stage0 + s * stage_bytes);
        const uint32_t sw = p.wres ? smem_u32(wres + kc * W_BYTES) : st;
        const uint32_t sx = p.wres ? st : st + W_BYTES;
        uint32_t a[4][4];
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            float v;
            asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(sx + off[r] + ks * 8 * 128));
            a[ks][r] = to_tf32(v);
          }
        // always all 4 k-steps: wgmma under a data-dependent branch is serialised by ptxas (C7520); channels past
        // Cin are zero in both operands (TMA zero fill, zero-padded weights)
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          // B: K-major SW128, 8-row groups at SBO = 1024 B, +32 B per k8 step
          const uint64_t bdesc = gmma_desc(sw + ks * 32, 16, 1024);
          WgmmaTf32<NT>::mma_rs(acc, a[ks], bdesc, (kc | ks) ? 1u : 0u);
        }
        wgmma_commit();
        // wait for this stage's MMAs before the A registers are reloaded (the wgmma reads them asynchronously)
        wgmma_wait<0>();
        reg_fence(acc);
        if (wg_lead) mbar_arrive(&empty[s]);
        if (++s == p.stages) { s = 0; ph ^= 1; }
      }
      // ===== epilogue: per 64-channel block, registers -> [4 px boxes][64 ch][128 B] swizzled smem -> TMA store =====
#pragma unroll
      for (int cb = 0; cb < NT / T_OUT_CH; ++cb) {
        const int k0 = mg * NT + cb * T_OUT_CH;
        if (k0 >= p.M) break;   // block-uniform
        uint8_t* buf = outbuf + ob * T_OUT_BYTES;
        if (leader) { if (p.out_bufs == 2) tma_store_wait_read<1>(); else tma_store_wait_read<0>(); }
        named_bar_sync(1, 256);
#pragma unroll
        for (int h = 0; h < 2; ++h) {   // fragment rows g and g + 8: pixels pt and pt + 8
          const int q = (pt & 31) + 8 * h;
          uint8_t* col = buf + jb * (T_OUT_CH * 128) + (q & 3) * 4;
#pragma unroll
          for (int j = 0; j < T_OUT_CH / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int cl = 8 * j + 2 * t4 + e;   // channel inside the block
              const int k = k0 + cl;
              const float bias = (p.bias && k < p.M) ? p.bias[k] : 0.f;
              *reinterpret_cast<float*>(col + cl * 128 + ((((q >> 2) ^ (cl & 7))) << 4)) =
                  acc[4 * (cb * (T_OUT_CH / 8) + j) + 2 * h + e] + bias;
            }
          }
        }
        fence_proxy_async();
        named_bar_sync(1, 256);
        if (leader) {
#pragma unroll
          for (int j = 0; j < 4; ++j) tma_store_3d(&tmap_y, buf + j * (T_OUT_CH * 128), p0 + 32 * j, k0, n);
          tma_store_commit();
        }
        if (p.out_bufs == 2) ob ^= 1;
      }
    }
    if (leader) tma_store_wait_read<0>();
  }
}

// output channels per group: one wgmma N of 64, 128 or 256
inline int fprop_nt(int M) { return M <= 64 ? 64 : (M <= 128 ? 128 : 256); }

template <int NT>
int launch_tf32_pw(const CUtensorMap& tw, const CUtensorMap& tx, const CUtensorMap& ty, Tf32PwParams p, cudaStream_t st) {
  const int kchunks = (p.Cin + T_BK - 1) / T_BK;
  const int budget = T_SMEM_LIMIT - T_SMEM_AUX;
  const int wres_bytes = kchunks * NT * 128;
  int smem = 0;
  // weights stay resident when they fit and every CTA needs the same rows (one group of output channels); else they
  // stream through the stages with the activations
  for (int wres = (wres_bytes <= 128 * 1024 && p.num_mg == 1) ? 1 : 0; wres >= 0; --wres) {
    const int stage_bytes = (wres ? 0 : NT * 128) + T_XSTAGE;
    const int rem = budget - (wres ? wres_bytes : 0);
    p.wres = wres;
    p.out_bufs = 2;
    p.stages = (rem - 2 * T_OUT_BYTES) / stage_bytes;
    if (p.stages < 3) { p.out_bufs = 1; p.stages = (rem - T_OUT_BYTES) / stage_bytes; }
    if (p.stages > T_MAX_STAGES) p.stages = T_MAX_STAGES;
    smem = (wres ? wres_bytes : 0) + p.stages * stage_bytes + p.out_bufs * T_OUT_BYTES + T_SMEM_AUX;
    if (p.stages >= 2) break;
  }
  SPC_REQUIRE(p.stages >= 2, "tf32 conv: shared memory budget too small (NT=%d kchunks=%d)", NT, kchunks);
  auto kern = tf32_pw_gemm_kernel<NT>;
  const int rc = allow_dynamic_smem((const void*)kern, T_SMEM_LIMIT);
  if (rc) return rc;
  const int sms = sm_count();
  kern<<<p.num_tiles < sms ? p.num_tiles : sms, T_THREADS, smem, st>>>(tw, tx, ty, p);
  count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

size_t wp_bytes(int M, int Cin) { return (size_t)round_up(M, fprop_nt(M)) * round_up(Cin, T_BK) * 4; }

// Y[N][M][P] = W'[M x Cin] * X[N][Cin][P] (+bias); W' = w (transpose = 0, w is [M][Cin]) or w^T (w is [Cin][M]).
// ws: at least wp_bytes(M, Cin) + 1024 bytes.
int run_tf32_pw(const float* w, int transpose, int M, int Cin, const float* x, const float* bias, float* y, int N, int P,
                void* ws, cudaStream_t st) {
  const int NT = fprop_nt(M);
  const int Mpad = round_up(M, NT), Cpad = round_up(Cin, T_BK);
  float* wp = reinterpret_cast<float*>(align1k(reinterpret_cast<uintptr_t>(ws)));
  {
    const int total = Mpad * Cpad;
    int blocks = (total + 255) / 256;
    if (blocks > 1184) blocks = 1184;
    tf32_repack_weights_kernel<<<blocks, 256, 0, st>>>(w, wp, M, Cin, Mpad, Cpad, transpose ? 1 : Cin,
                                                       transpose ? M : 1);
    count_launch();
    SPC_CHECK_CUDA(cudaGetLastError());
  }
  CUtensorMap tw, tx, ty;
  {
    const uint64_t dims[2] = {(uint64_t)Cpad, (uint64_t)Mpad};
    const uint64_t strides[2] = {0, (uint64_t)Cpad * 4};
    const uint32_t box[2] = {T_BK, (uint32_t)NT};
    int rc = make_tmap(&tw, wp, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  int rc = make_act_tmap_f32(&tx, x, P, Cin, N, T_BK);
  if (rc) return rc;
  rc = make_act_tmap_f32(&ty, y, P, M, N, T_OUT_CH);
  if (rc) return rc;
  Tf32PwParams p{};
  p.M = M; p.Cin = Cin; p.N = N; p.bias = bias;
  p.num_mg = Mpad / NT;
  p.tiles_per_image = (P + T_BN - 1) / T_BN;
  p.num_tiles = p.tiles_per_image * N * p.num_mg;
  if (NT == 64) return launch_tf32_pw<64>(tw, tx, ty, p, st);
  if (NT == 128) return launch_tf32_pw<128>(tw, tx, ty, p, st);
  return launch_tf32_pw<256>(tw, tx, ty, p, st);
}

// ---- wgrad kernel: dW[K x C] += dY[K x P] * X[C x P]^T ---------------------------------------------------------------
// pw_wgrad_kernel's 1x1 plan with 32-pixel chunks: one work item = (group of MG 128-row blocks of dY, one block of NBLK
// input channels, a split of the pixel range); its MG accumulator blocks [64 rows x NBLK] per consumer warpgroup live in
// registers and are flushed with fp32 atomics.  (A separate kernel rather than a template of pw_wgrad_kernel: an element
// type parameter would change the names of the bf16 instances.)
constexpr int T_WG_ACC = 256;   // accumulator columns per consumer warpgroup: 128 fp32 registers per thread

struct Tf32WgParams {
  float* dw;          // [K][C] fp32
  int K, C;
  int n_blocks;       // ceil(C / NBLK)
  int mgroups;        // ceil(ceil(K / mrows) / MG)
  int mrows;          // dY rows per 128-row block: K split evenly over its blocks
  int splits;         // pixel-range splits per item
  int chunks_total, chunks_per_image;   // 32-pixel chunks
  int stages;
  int split0, nsplit;       // this launch runs splits [split0, split0 + nsplit)
  size_t slice_stride;      // split sp adds into dw + (sp - split0) * slice_stride (common.cuh: WgradSlices)
};

template <int NBLK, int MG>
__global__ void __launch_bounds__(T_THREADS, 1)
tf32_pw_wgrad_kernel(const __grid_constant__ CUtensorMap tmap_dy, const __grid_constant__ CUtensorMap tmap_x,
                     const Tf32WgParams p) {
  static_assert(MG * NBLK <= T_WG_ACC, "accumulator registers");
  constexpr int B_BYTES = NBLK * 128;                     // [NBLK ch][32 px]
  constexpr int B_SLOT = (B_BYTES + 1023) & ~1023;
  constexpr int STAGE = MG * T_A_BLK + B_SLOT;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + p.stages * STAGE);
  uint64_t* empty = full + T_MAX_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.stages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 2); }
    fence_barrier_init();
  }
  __syncthreads();
  const int ngroups = p.mgroups * p.n_blocks;
  const int it0 = p.split0 * ngroups, it1 = it0 + p.nsplit * ngroups;
  const int per_split = (p.chunks_total + p.splits - 1) / p.splits;
  // item -> (split, channel block, m group); concurrently running CTAs cover all groups of the SAME pixel range, so
  // the chunks every group re-reads come from L2
#define TWG_DECODE(it)                                   \
  const int sp = (it) / ngroups, g_ = (it) % ngroups;    \
  const int nb = g_ % p.n_blocks, mgp = g_ / p.n_blocks; \
  const int c_begin = sp * per_split, c_end = min(p.chunks_total, c_begin + per_split);

  if (warp == 0) {
    if (lane == 0) {
      tma_prefetch_desc(&tmap_dy);
      tma_prefetch_desc(&tmap_x);
      int s = 0, ph = 0;
      for (int it = it0 + blockIdx.x; it < it1; it += gridDim.x) {
        TWG_DECODE(it)
        for (int ch = c_begin; ch < c_end; ++ch) {
          const int n = ch / p.chunks_per_image, p0 = (ch % p.chunks_per_image) * 32;
          mbar_wait(&empty[s], ph ^ 1);
          uint8_t* st = smem + s * STAGE;
          mbar_arrive_expect_tx(&full[s], MG * p.mrows * 128 + B_BYTES);
          for (int i = 0; i < MG; ++i) tma_load_3d(st + i * T_A_BLK, &tmap_dy, &full[s], p0, (mgp * MG + i) * p.mrows, n);
          tma_load_3d(st + MG * T_A_BLK, &tmap_x, &full[s], p0, nb * NBLK, n);
          if (++s == p.stages) { s = 0; ph ^= 1; }
        }
      }
    }
  } else if (threadIdx.x >= 128) {
    const int wg = (threadIdx.x >> 7) - 1;
    const int w4 = (threadIdx.x >> 5) & 3;
    const bool wg_lead = (threadIdx.x & 127) == 0;
    const bool live = 64 * wg < p.mrows;   // rows >= mrows of a block are not dY rows of this block
    float acc[MG][NBLK / 2];
    int s = 0, ph = 0;
    for (int it = it0 + blockIdx.x; it < it1; it += gridDim.x) {
      TWG_DECODE(it)
      float* dw = p.dw + (size_t)(sp - p.split0) * p.slice_stride;   // the items of one split add disjoint blocks
      int prev = -1;
      for (int ch = c_begin; ch < c_end; ++ch) {
        mbar_wait(&full[s], ph);
        const uint32_t sa = smem_u32(smem + s * STAGE);
        const uint32_t sb = sa + MG * T_A_BLK;
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          const uint64_t bdesc = gmma_desc(sb + ks * 32, 16, 1024);
#pragma unroll
          for (int i = 0; i < MG; ++i) {
            // A: K-major SW128, this warpgroup's 64 rows start 8 row groups (8 KB) in; +32 B per k8 step
            const uint64_t adesc = gmma_desc(sa + i * T_A_BLK + wg * 8192 + ks * 32, 16, 1024);
            WgmmaTf32<NBLK>::mma(acc[i], adesc, bdesc, (ch > c_begin || ks > 0) ? 1u : 0u);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();   // the previous stage's MMAs are done reading it
        if (prev >= 0 && wg_lead) mbar_arrive(&empty[prev]);
        prev = s;
        if (++s == p.stages) { s = 0; ph ^= 1; }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int i = 0; i < MG; ++i) reg_fence(acc[i]);
      if (prev >= 0 && wg_lead) mbar_arrive(&empty[prev]);
      if (c_end > c_begin && live) {
#pragma unroll
        for (int i = 0; i < MG; ++i) {
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
                  if (c < p.C) atomicAdd(&dw[(size_t)k * p.C + c], acc[i][4 * q + 2 * h + e]);
                }
              }
            }
          }
        }
      }
    }
  }
#undef TWG_DECODE
}

template <int NBLK, int MG>
int launch_tf32_wg(const CUtensorMap& tdy, const CUtensorMap& tx, Tf32WgParams p, cudaStream_t st, const WgradSlices* sl) {
  constexpr int STAGE = MG * T_A_BLK + ((NBLK * 128 + 1023) & ~1023);
  p.stages = (T_SMEM_LIMIT - T_SMEM_AUX) / STAGE;
  if (p.stages > 6) p.stages = 6;
  SPC_REQUIRE(p.stages >= 2, "tf32 wgrad: smem budget");
  const int sms = sm_count();
  const int groups = p.mgroups * p.n_blocks;
  // split count: as pw_wgrad_kernel's planner, minimise  waves * chunks_per_item * t_chunk + items * elems / atomic_rate
  // (estimates: only their ratio matters).  A tf32 k8 step moves the same bytes and takes the same MMA time as a bf16
  // k16 step, so the per-chunk costs are those of the bf16 kernel.
  int splits = 1;
  {
    const double clk = 1.7e9, atomic_rate = 60e9;
    const double bytes_chunk = (double)(MG * p.mrows + NBLK) * 128.0;
    const double mma_chunk = (double)MG * 4.0 * (NBLK > 64 ? NBLK : 64);
    const double t_chunk = (bytes_chunk / 32.0 > mma_chunk ? bytes_chunk / 32.0 : mma_chunk) / clk;
    const double elems = (double)MG * p.mrows * NBLK;
    const int smax = (2 * sms) / groups > 1 ? (2 * sms) / groups : 1;
    double best = 1e30;
    for (int s = smax; s >= 1; --s) {
      if (s > p.chunks_total / 8 && s > 1) continue;
      const int items_s = groups * s, waves = (items_s + sms - 1) / sms;
      const double cpi = (double)((p.chunks_total + s - 1) / s);
      const double t = waves * cpi * t_chunk + (double)items_s * elems / atomic_rate;
      if (t < best * 0.98) { best = t; splits = s; }
    }
  }
  p.splits = splits;
  const int smem = p.stages * STAGE + T_SMEM_AUX;
  auto kern = tf32_pw_wgrad_kernel<NBLK, MG>;
  const int rc = allow_dynamic_smem((const void*)kern, T_SMEM_LIMIT);
  if (rc) return rc;
  return run_slices(sl, p.splits, (size_t)p.K * p.C, p.dw, st, [&](int s0, int ns, float* dst, size_t stride) {
    Tf32WgParams q = p;
    q.split0 = s0; q.nsplit = ns; q.dw = dst; q.slice_stride = stride;
    const int items = groups * ns;
    kern<<<items < sms ? items : sms, T_THREADS, smem, st>>>(tdy, tx, q);
    count_launch();
    SPC_CHECK_CUDA(cudaGetLastError());
    return SPC_OK;
  });
}

template <int NBLK>
int launch_tf32_wg_mg(const CUtensorMap& tdy, const CUtensorMap& tx, const Tf32WgParams& p, int MG, cudaStream_t st,
                      const WgradSlices* sl) {
  if (MG == 1) return launch_tf32_wg<NBLK, 1>(tdy, tx, p, st, sl);
  if constexpr (NBLK <= 128) { if (MG == 2) return launch_tf32_wg<NBLK, 2>(tdy, tx, p, st, sl); }
  if constexpr (NBLK <= 64) { if (MG == 4) return launch_tf32_wg<NBLK, 4>(tdy, tx, p, st, sl); }
  set_error("tf32 wgrad: no kernel for %d blocks of %d channels", MG, NBLK);
  return SPC_EUNSUPPORTED;
}

// dw[K][C] += dy[N][K][P] * x[N][C][P]^T
int run_tf32_wgrad(const float* x, const float* dy, float* dw, int K, int C, int N, int P, cudaStream_t st,
                   const WgradSlices* sl) {
  Tf32WgParams p{};
  p.dw = dw; p.K = K; p.C = C;
  // accumulator width: C split evenly over blocks of <= 128 channels, rounded up to an instantiated width
  p.n_blocks = (C + 127) / 128;
  const int w = round_up((C + p.n_blocks - 1) / p.n_blocks, 8);
  const int nblk = w <= 32 ? 32 : (w <= 64 ? 64 : 128);
  int MBtot = (K + 127) / 128;
  p.mrows = round_up((K + MBtot - 1) / MBtot, 8);   // e.g. K = 416 -> 4 blocks of 104
  MBtot = (K + p.mrows - 1) / p.mrows;
  int MG = T_WG_ACC / nblk;
  if (MG > MBtot) MG = MBtot;
  MG = MG >= 4 ? 4 : (MG >= 2 ? 2 : 1);
  p.mgroups = (MBtot + MG - 1) / MG;
  p.chunks_per_image = (P + 31) / 32;
  p.chunks_total = p.chunks_per_image * N;
  CUtensorMap tdy, tx;
  int rc = make_act_tmap_f32(&tdy, dy, P, K, N, p.mrows);
  if (rc) return rc;
  rc = make_act_tmap_f32(&tx, x, P, C, N, nblk);
  if (rc) return rc;
  if (nblk == 32) return launch_tf32_wg_mg<32>(tdy, tx, p, MG, st, sl);
  if (nblk == 64) return launch_tf32_wg_mg<64>(tdy, tx, p, MG, st, sl);
  return launch_tf32_wg_mg<128>(tdy, tx, p, MG, st, sl);
}

// ---- stride-2 passes (fp32) -------------------------------------------------------------------------------------------
// y[n,c,i,j] = x[n,c,2i,2j]; 4 outputs per thread (two 16-byte loads, one 16-byte store)
__global__ void tf32_subsample2_kernel(const float* __restrict__ x, float* __restrict__ y, size_t planes, int H, int W) {
  const int Ho = H / 2, Wo = W / 2, wv = Wo / 4;
  const size_t total = planes * Ho * wv;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int v = (int)(i % wv);
    const int oy = (int)((i / wv) % Ho);
    const size_t pl = i / ((size_t)wv * Ho);
    const float4* src = reinterpret_cast<const float4*>(x + (pl * H + 2 * oy) * W + v * 8);
    const float4 a = __ldg(src), b = __ldg(src + 1);
    *reinterpret_cast<float4*>(y + (pl * Ho + oy) * Wo + v * 4) = make_float4(a.x, a.z, b.x, b.z);
  }
}
// dx[n,c,2i,2j] = g[n,c,i,j], zero elsewhere
__global__ void tf32_upsample2_zero_kernel(const float* __restrict__ g, float* __restrict__ dx, size_t planes, int H,
                                           int W) {
  const int Ho = H / 2, Wo = W / 2, wv = Wo / 4;
  const size_t total = planes * Ho * wv;
  const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int v = (int)(i % wv);
    const int oy = (int)((i / wv) % Ho);
    const size_t pl = i / ((size_t)wv * Ho);
    const float4 a = __ldg(reinterpret_cast<const float4*>(g + (pl * Ho + oy) * Wo + v * 4));
    float4* d0 = reinterpret_cast<float4*>(dx + (pl * H + 2 * oy) * W + v * 8);
    float4* d1 = reinterpret_cast<float4*>(dx + (pl * H + 2 * oy + 1) * W + v * 8);
    d0[0] = make_float4(a.x, 0.f, a.y, 0.f); d0[1] = make_float4(a.z, 0.f, a.w, 0.f);
    d1[0] = z; d1[1] = z;
  }
}
int launch_resample_f32(bool up, const float* src, float* dst, size_t planes, int H, int W, cudaStream_t st) {
  const size_t total = planes * (H / 2) * (W / 8);
  size_t blocks = (total + 255) / 256;
  if (blocks > 132 * 32) blocks = 132 * 32;
  if (up)
    tf32_upsample2_zero_kernel<<<(int)blocks, 256, 0, st>>>(src, dst, planes, H, W);
  else
    tf32_subsample2_kernel<<<(int)blocks, 256, 0, st>>>(src, dst, planes, H, W);
  count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

// repacked weights of op 0 / 1 (wgrad needs none)
size_t wbytes(const spc_conv_desc* d, int op) {
  if (op == 0) return align1k(wp_bytes(d->K, d->C) + 1024);
  if (op == 1) return align1k(wp_bytes(d->C, d->K) + 1024);
  return 0;
}

}  // namespace

// The shapes of gemm_tc.cu's pointwise path (1x1, stride 1 or 2, 16-byte aligned pixel rows), in fp32
bool tf32_supported(const spc_conv_desc* d) {
  if (d->dtype != SPC_F32 || d->R != 1 || d->S != 1) return false;
  long long P = (long long)d->H * d->W;
  if (is_s2(d)) {
    if (d->H % 2 || d->W % 32) return false;   // 16-byte vectors on both sides of the resample
    P /= 4;
  } else if (d->stride_h != 1 || d->stride_w != 1) {
    return false;
  }
  return P % 8 == 0 && P < (1ll << 31);
}

// [repacked weights | subsampled x (fprop, wgrad) or the GEMM output before the zero upsample (dgrad)]
size_t tf32_workspace_bytes(const spc_conv_desc* d, int op) {
  size_t b = wbytes(d, op) + 4096;
  if (is_s2(d)) b += align1k((size_t)d->N * d->C * (d->H / 2) * (d->W / 2) * 4) + 1024;
  return b;
}

int tf32_conv_fwd(const spc_conv_desc* d, const void* x, const void* w, const void* bias, void* y, void* ws,
                  size_t ws_bytes, cudaStream_t st) {
  SPC_REQUIRE(ws && ws_bytes >= tf32_workspace_bytes(d, 0), "tf32 conv: workspace too small");
  const float* xs = reinterpret_cast<const float*>(x);
  int P = d->H * d->W;
  if (is_s2(d)) {   // Y = W * subsample(X)
    float* sub = reinterpret_cast<float*>(align1k(reinterpret_cast<uintptr_t>(ws) + wbytes(d, 0)));
    int rc = launch_resample_f32(false, xs, sub, (size_t)d->N * d->C, d->H, d->W, st);
    if (rc) return rc;
    xs = sub;
    P = (d->H / 2) * (d->W / 2);
  }
  return run_tf32_pw(reinterpret_cast<const float*>(w), 0, d->K, d->C, xs, reinterpret_cast<const float*>(bias),
                     reinterpret_cast<float*>(y), d->N, P, ws, st);
}

int tf32_conv_dgrad(const spc_conv_desc* d, const void* dy, const void* w, void* dx, void* ws, size_t ws_bytes,
                    cudaStream_t st) {
  // dX[C x P] = W^T[C x K] * dY[K x P]
  SPC_REQUIRE(ws && ws_bytes >= tf32_workspace_bytes(d, 1), "tf32 conv: workspace too small");
  const float* wf = reinterpret_cast<const float*>(w);
  const float* dyf = reinterpret_cast<const float*>(dy);
  if (is_s2(d)) {   // dX = zero_upsample(W^T * dY)
    float* gs = reinterpret_cast<float*>(align1k(reinterpret_cast<uintptr_t>(ws) + wbytes(d, 1)));
    int rc = run_tf32_pw(wf, 1, d->C, d->K, dyf, nullptr, gs, d->N, (d->H / 2) * (d->W / 2), ws, st);
    if (rc) return rc;
    return launch_resample_f32(true, gs, reinterpret_cast<float*>(dx), (size_t)d->N * d->C, d->H, d->W, st);
  }
  return run_tf32_pw(wf, 1, d->C, d->K, dyf, nullptr, reinterpret_cast<float*>(dx), d->N, d->H * d->W, ws, st);
}

int tf32_conv_wgrad(const spc_conv_desc* d, const void* x, const void* dy, float* dw, void* ws, size_t ws_bytes,
                    cudaStream_t st, const WgradSlices* sl) {
  // accumulates with atomics: api.cu has already zeroed dw when !accumulate
  const float* xf = reinterpret_cast<const float*>(x);
  int P = d->H * d->W;
  if (is_s2(d)) {
    SPC_REQUIRE(ws && ws_bytes >= tf32_workspace_bytes(d, 2), "tf32 wgrad: workspace too small");
    float* sub = reinterpret_cast<float*>(align1k(reinterpret_cast<uintptr_t>(ws)));
    int rc = launch_resample_f32(false, xf, sub, (size_t)d->N * d->C, d->H, d->W, st);
    if (rc) return rc;
    xf = sub;
    P = (d->H / 2) * (d->W / 2);
  }
  return run_tf32_wgrad(xf, reinterpret_cast<const float*>(dy), dw, d->K, d->C, d->N, P, st, sl);
}

// Slice copies of tf32_conv_wgrad: as pw_wgrad_kernel's, launch_tf32_wg makes <= 2 * SMs / groups splits of a gradient of
// <= groups * 128 x 256 floats
double tf32_wgrad_slice_floats(const spc_conv_desc* d) {
  const double wn = (double)d->K * d->C * d->R * d->S, sms = sm_count();
  return 2.0 * sms * (wn < 32768.0 ? wn : 32768.0);
}

}  // namespace spc
