// gemm_px.cu -- pixel-major bf16 wgmma GEMM for the large 1x1 convolutions (fprop and dgrad; the stride-2 ones run on
// their subsampled / to-be-upsampled buffers).
//
// pw_gemm_kernel (gemm_tc.cu) computes Y[M x P] = W * X per image with the output channels as the wgmma M dimension,
// which is fixed at 64 per warpgroup, in 128-row blocks: an AmoebaNet-D layer with 52, 104, 208 or 416 output channels
// wastes 23 % (146 % for 52) of its MMAs on zero rows.  This kernel computes the transposed product
//     Y^T[P x M] = X^T[P x Cin] * Wp^T[Cin x M]
// with the pixels as the wgmma M dimension and the output channels as N, which only has to be a multiple of 8: a tile
// is 128 pixels x NT channels, NT in {56, 104, 208} (px_tile_channels in gemm_tc.cu picks it).
//   A = activations, read IN PLACE by TMA exactly as pw_gemm_kernel reads them: [64 ch][64 px] rows of 128 B, SW128,
//       or one 5-d box [8-ch group][px block][8 ch][128 B] (see PwParams::x5); MN-major operand (WgmmaTA).
//   B = weights repacked K-major [Mpad = multiple of NT rows][Cpad] (repack_weights_kernel), box {64 ch, NT rows},
//       SW128; resident in smem when one group of NT rows covers M and all chunks fit 128 KB, else streamed per stage.
//   D = [64 px x NT ch] per consumer warpgroup: NT / 2 fp32 registers per thread.
// Epilogue: stmatrix.trans writes the fragments (+ bias) as [ch][px] rows into a swizzled staging block, which TMA
// stores as [NT ch][64 px] boxes (or one 5-d box); TMA clips the rows past M and the pixels past P.
// Warp roles (384 threads): warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 = wgmma consumers + epilogue.
// Persistent CTAs, one per SM; consecutive tiles are the channel groups of one pixel tile, so the activations are read
// from HBM once and from L2 once per further group.
#include "common.cuh"
#include "tc_common.cuh"

namespace spc {

using namespace tc;

namespace {

constexpr int PX_THREADS = 384;
constexpr int PX_BK = 64;                          // channels per pipeline stage
constexpr int PX_BM = 128;                         // pixels per tile (two 64-pixel swizzle blocks)
constexpr int PX_X_BYTES = PX_BK * PX_BM * 2;      // activations per stage: 16 KB
constexpr int PX_MAX_STAGES = 8;
constexpr int PX_SMEM_LIMIT = 222 * 1024;          // as gemm_tc.cu: room for a small co-resident kernel
constexpr int PX_SMEM_AUX = 1024 /*align*/ + 512 /*barriers*/;

struct PxParams {
  int M;                       // valid output channels
  int Cin;                     // reduction length (input channels)
  int N, tiles_per_image;
  int num_mg;                  // groups of NT output channels
  int num_tiles;               // N * tiles_per_image * num_mg
  int stages;                  // pipeline depth (<= PX_MAX_STAGES)
  int wres;                    // 1: all weight chunks stay resident in smem
  int out_bufs;                // 1 or 2 epilogue staging blocks
  int x5, y5;                  // activations / outputs move as one 5-d box per tile (PwParams::x5 / y5)
  const __nv_bfloat16* bias;   // [M] or null
};

// 8x8 b16 matrices, stored transposed: register i of a lane holds (row lane / 4, columns 2 (lane % 4) + {0, 1}) of
// matrix i; lane 8 i + r gives the address of row r of the stored (transposed) matrix i, i.e. of fragment column r
__device__ __forceinline__ void stmatrix_x4_trans(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1),
               "r"(r2), "r"(r3)
               : "memory");
}
__device__ __forceinline__ void stmatrix_x2_trans(uint32_t addr, uint32_t r0, uint32_t r1) {
  asm volatile("stmatrix.sync.aligned.m8n8.x2.trans.shared.b16 [%0], {%1, %2};" ::"r"(addr), "r"(r0), "r"(r1) : "memory");
}

// Consumer warpgroup g owns pixels [64 g, 64 g + 64) of the 128-pixel tile (the wgmma M dimension) and all NT output
// channels of the tile's group (the N dimension).
template <int NT>
__global__ void __launch_bounds__(PX_THREADS, 1)
pw_px_gemm_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x,
                  const __grid_constant__ CUtensorMap tmap_y, const PxParams p) {
  constexpr int W_BYTES = NT * 128;          // one 64-channel chunk of the group's NT weight rows
  constexpr int OUT_BYTES = NT * PX_BM * 2;  // the tile's [NT ch][128 px] outputs
  constexpr int NQ = NT / 8;                 // 8-channel fragment column blocks
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int kchunks = (p.Cin + PX_BK - 1) / PX_BK;
  const int wres_bytes = p.wres ? kchunks * W_BYTES : 0;
  const int stage_bytes = (p.wres ? 0 : W_BYTES) + PX_X_BYTES;
  uint8_t* wres = smem;
  uint8_t* stage0 = smem + wres_bytes;
  uint8_t* outbuf = stage0 + p.stages * stage_bytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(outbuf + p.out_bufs * OUT_BYTES);
  uint64_t* empty = full + PX_MAX_STAGES;
  uint64_t* wfull = empty + PX_MAX_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool x5 = p.x5, y5 = p.y5;

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.stages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 2); }   // empty: one per consumer
    mbar_init(wfull, 1);
    fence_barrier_init();
  }
  __syncthreads();

  // 384 x 168 registers at launch: the producer warpgroup (one busy thread) hands its registers to the consumers,
  // 40 + 2 x 232 <= 3 x 168
  if (threadIdx.x < 128) {
    setmaxnreg_dec<40>();
    // ================= TMA producer =================
    if (warp == 0 && lane == 0) {
      tma_prefetch_desc(&tmap_w);
      tma_prefetch_desc(&tmap_x);
      if (p.wres) {
        mbar_arrive_expect_tx(wfull, wres_bytes);
        for (int kc = 0; kc < kchunks; ++kc) tma_load_2d(wres + kc * W_BYTES, &tmap_w, wfull, kc * PX_BK, 0);
      }
      int s = 0, ph = 0;
      for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
        const int mg = t % p.num_mg, tt = t / p.num_mg;
        const int n = tt / p.tiles_per_image, p0 = (tt % p.tiles_per_image) * PX_BM;
        for (int kc = 0; kc < kchunks; ++kc) {
          mbar_wait(&empty[s], ph ^ 1);
          uint8_t* st = stage0 + s * stage_bytes;
          mbar_arrive_expect_tx(&full[s], stage_bytes);
          if (!p.wres) {
            tma_load_2d(st, &tmap_w, &full[s], kc * PX_BK, mg * NT);
            st += W_BYTES;
          }
          if (x5) {
            tma_load_5d(st, &tmap_x, &full[s], 0, 0, p0 >> 6, kc * (PX_BK / 8), n);
          } else {
#pragma unroll
            for (int j = 0; j < 2; ++j) tma_load_3d(st + j * (PX_X_BYTES / 2), &tmap_x, &full[s], p0 + 64 * j, kc * PX_BK, n);
          }
          if (++s == p.stages) { s = 0; ph ^= 1; }
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    // ================= consumers: wgmma + epilogue =================
    const int wg = (threadIdx.x >> 7) - 1;
    const int w4 = (threadIdx.x >> 5) & 3;
    const bool wg_lead = (threadIdx.x & 127) == 0;
    const bool leader = threadIdx.x == 128;   // issues the TMA stores
    // stmatrix addresses: lane 8 i + r writes channel r of 8-channel block qb + i / 2, pixels 16 w4 + 8 (i % 2) .. + 7
    // of this warpgroup's 64-pixel block, as one swizzled 16-byte chunk (SWIZZLE_128B: chunk ^ (row % 8)).  Staging
    // layout: 3-d stores [px block][NT ch][128 B]; 5-d stores [8-ch group][px block][8 ch][128 B].
    const int mi = lane >> 3, cr = lane & 7;
    const uint32_t blk = y5 ? 2048 : 1024;    // distance of consecutive 8-channel blocks
    const uint32_t lane_off = (y5 ? wg * 1024 : wg * W_BYTES) + (mi >> 1) * blk + cr * 128 +
                              ((((16 * w4 + 8 * (mi & 1)) >> 3) ^ cr) << 4);
    float acc[NT / 2];
    if (p.wres) mbar_wait(wfull, 0);
    int s = 0, ph = 0, ob = 0;
    for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
      const int mg = t % p.num_mg, tt = t / p.num_mg;
      const int n = tt / p.tiles_per_image, p0 = (tt % p.tiles_per_image) * PX_BM;
      int prev = -1;
      for (int kc = 0; kc < kchunks; ++kc) {
        mbar_wait(&full[s], ph);
        const uint32_t st = smem_u32(stage0 + s * stage_bytes);
        const uint32_t sw = p.wres ? smem_u32(wres + kc * W_BYTES) : st;
        const uint32_t sx = p.wres ? st : st + W_BYTES;
        // always 4 k-steps: wgmma under a data-dependent branch is serialised by ptxas (C7520); the channels past Cin
        // are zero in both operands (TMA zero fill, zero-padded weights)
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          // A: MN-major SW128, this warpgroup's 64-pixel block; 16 channels = two 8-row groups at SBO
          // (3-d boxes: px blocks 8 KB apart, groups at 1 KB; 5-d box: px blocks 1 KB apart, groups at 2 KB)
          const uint64_t adesc = x5 ? gmma_desc(sx + wg * 1024 + ks * 4096, 1024, 2048)
                                    : gmma_desc(sx + wg * (PX_X_BYTES / 2) + ks * 2048, PX_X_BYTES / 2, 1024);
          // B: K-major SW128, 8-row groups at SBO = 1024 B, +32 B per k-step
          const uint64_t bdesc = gmma_desc(sw + ks * 32, 16, 1024);
          WgmmaTA<NT>::mma(acc, adesc, bdesc, (kc | ks) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();                         // the previous stage's MMAs are done reading it
        if (prev >= 0 && wg_lead) mbar_arrive(&empty[prev]);
        prev = s;
        if (++s == p.stages) { s = 0; ph ^= 1; }
      }
      wgmma_wait<0>();
      reg_fence(acc);
      if (prev >= 0 && wg_lead) mbar_arrive(&empty[prev]);
      // ===== epilogue: registers (+ bias) -> [ch][px] swizzled smem -> TMA store =====
      uint8_t* buf = outbuf + ob * OUT_BYTES;
      // the TMA store that last read this buffer must have finished reading it
      if (leader) { if (p.out_bufs == 2) tma_store_wait_read<1>(); else tma_store_wait_read<0>(); }
      named_bar_sync(1, 256);
      {
        const uint32_t base = smem_u32(buf) + lane_off;
        const int k0 = mg * NT + 2 * (lane & 3);   // fragment columns 2 (lane % 4) + {0, 1} of every 8-channel block
        float bv[NT / 4];
#pragma unroll
        for (int q = 0; q < NQ; ++q)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int k = k0 + 8 * q + e;
            bv[2 * q + e] = (p.bias && k < p.M) ? __bfloat162float(p.bias[k]) : 0.f;
          }
#pragma unroll
        for (int q = 0; q + 1 < NQ; q += 2) {
          // matrices: (pixels 0-7, block q), (pixels 8-15, block q), (0-7, q + 1), (8-15, q + 1)
          stmatrix_x4_trans(base + q * blk,
                            pack_bf16x2(acc[4 * q + 0] + bv[2 * q], acc[4 * q + 1] + bv[2 * q + 1]),
                            pack_bf16x2(acc[4 * q + 2] + bv[2 * q], acc[4 * q + 3] + bv[2 * q + 1]),
                            pack_bf16x2(acc[4 * q + 4] + bv[2 * q + 2], acc[4 * q + 5] + bv[2 * q + 3]),
                            pack_bf16x2(acc[4 * q + 6] + bv[2 * q + 2], acc[4 * q + 7] + bv[2 * q + 3]));
        }
        if constexpr (NQ & 1) {
          constexpr int q = NQ - 1;   // lanes 0..15 give the addresses of the two matrices of block q
          stmatrix_x2_trans(base + q * blk,
                            pack_bf16x2(acc[4 * q + 0] + bv[2 * q], acc[4 * q + 1] + bv[2 * q + 1]),
                            pack_bf16x2(acc[4 * q + 2] + bv[2 * q], acc[4 * q + 3] + bv[2 * q + 1]));
        }
      }
      fence_proxy_async();        // make the smem writes visible to the TMA (async proxy)
      named_bar_sync(1, 256);
      if (leader) {
        if (y5) {
          tma_store_5d(&tmap_y, buf, 0, 0, p0 >> 6, (mg * NT) >> 3, n);
        } else {
#pragma unroll
          for (int j = 0; j < 2; ++j) tma_store_3d(&tmap_y, buf + j * W_BYTES, p0 + 64 * j, mg * NT, n);
        }
        tma_store_commit();
      }
      if (p.out_bufs == 2) ob ^= 1;
    }
    if (leader) tma_store_wait_read<0>();
  }
}

template <int NT>
int launch_px(const CUtensorMap& tw, const CUtensorMap& tx, const CUtensorMap& ty, PxParams p, int sms,
              cudaStream_t st) {
  const int kchunks = (p.Cin + PX_BK - 1) / PX_BK;
  const int budget = PX_SMEM_LIMIT - PX_SMEM_AUX;
  const int wres_bytes = kchunks * NT * 128;
  const int out_bytes = NT * PX_BM * 2;
  int smem = 0;
  // weights stay resident when they fit and every CTA needs the same rows (one group of output channels); else they
  // stream through the stages with the activations
  for (int wres = (wres_bytes <= 128 * 1024 && p.num_mg == 1) ? 1 : 0; wres >= 0; --wres) {
    const int stage_bytes = (wres ? 0 : NT * 128) + PX_X_BYTES;
    const int rem = budget - (wres ? wres_bytes : 0);
    p.wres = wres;
    p.out_bufs = 2;
    p.stages = (rem - 2 * out_bytes) / stage_bytes;
    if (p.stages < 3) { p.out_bufs = 1; p.stages = (rem - out_bytes) / stage_bytes; }
    if (p.stages > PX_MAX_STAGES) p.stages = PX_MAX_STAGES;
    smem = (wres ? wres_bytes : 0) + p.stages * stage_bytes + p.out_bufs * out_bytes + PX_SMEM_AUX;
    if (p.stages >= 2) break;
  }
  SPC_REQUIRE(p.stages >= 2, "wgmma px conv: shared memory budget too small (NT=%d kchunks=%d)", NT, kchunks);
  auto kern = pw_px_gemm_kernel<NT>;
  const int rc = allow_dynamic_smem((const void*)kern, PX_SMEM_LIMIT);
  if (rc) return rc;
  kern<<<p.num_tiles < sms ? p.num_tiles : sms, PX_THREADS, smem, st>>>(tw, tx, ty, p);
  count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

}  // namespace

// Y[N][M][P] = Wp[M x Cin] * X[N][Cin][P] (+bias) on pw_px_gemm_kernel<NT>.  tw: the repacked weights [Mpad][Cpad],
// Mpad a multiple of NT, box {64 ch, NT rows}; tx: the activations as gemm_tc.cu maps them for pw_gemm_kernel
// (box {64 px, 64 ch, 1}, or the 5-d box of 8 channel groups x 2 pixel blocks when x5); ty: the outputs, box
// {64 px, NT ch, 1}, or the 5-d box of NT / 8 channel groups x 2 pixel blocks when y5.
int run_pw_px(int NT, const CUtensorMap& tw, const CUtensorMap& tx, const CUtensorMap& ty, int M, int Cin, int N, int P,
              int x5, int y5, const __nv_bfloat16* bias, int sms, cudaStream_t st) {
  PxParams p{};
  p.M = M; p.Cin = Cin; p.N = N; p.x5 = x5; p.y5 = y5; p.bias = bias;
  p.num_mg = (M + NT - 1) / NT;
  p.tiles_per_image = (P + PX_BM - 1) / PX_BM;
  p.num_tiles = p.tiles_per_image * N * p.num_mg;
  if (NT == 56) return launch_px<56>(tw, tx, ty, p, sms, st);
  if (NT == 104) return launch_px<104>(tw, tx, ty, p, sms, st);
  if (NT == 208) return launch_px<208>(tw, tx, ty, p, sms, st);
  set_error("wgmma px conv: no kernel for %d output channels per tile", NT);
  return SPC_EUNSUPPORTED;
}

}  // namespace spc
