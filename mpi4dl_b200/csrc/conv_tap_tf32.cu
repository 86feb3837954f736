// conv_tap_tf32.cu -- fp32 stride-1 multi-tap convolutions (3x3, 1x7, 7x1, any odd R x S up to 7 x 7) on the tensor
// cores in TF32: fprop, dgrad and wgrad (opt-in: SPC_ALGO_TF32_ALL).
//
// wgmma .tf32 has no transpose, so shared-memory operands must be K-major, and the activations are pixel-contiguous.
// As in gemm_tf32.cu, the kernel computes the transposed product, with the activations as the register operand:
//   fprop : Y^T[P x K] = sum_(r,s) X_(r,s)^T[P x C] * W_(r,s)^T[C x K],   X_(r,s)(y, x) = X(y + r - ph, x + s - pw)
//           A = X_(r,s)^T from registers (ld.shared + cvt.rna.tf32), B = the tap's weights repacked K-major in tf32.
//   dgrad : the same with dY for X and the rotated, transposed filter  W'_(r,s)[c][k] = w[k][c][R-1-r][S-1-s].
// The activations are 4-D tensor maps [N][C][H][W] read in 32-pixel row segments.  The box of a segment at (y, x0) for
// the taps of row r is [32 ch][40 px] from (y + r - ph, x0 - 4), unswizzled: a TMA box must start on a 16-byte
// boundary, so the 4 pixels of slack on each side hold the horizontal halo (pw <= 3), and tap (r, s) is the pixel
// offset s - pw + 4 in the ld.shared address.  The 40-word row pitch (8 mod 32) makes the m64k8 fragment loads (8
// pixels x 4 channels per warp) free of bank conflicts.  TMA fills coordinates outside the image with zeros: that is
// the zero padding of the interior pass; api.cu recomputes the outputs whose windows reach a received halo strip.
// Few reduction channels (Cin <= 8, the C = 3 stem): a 32-channel k-chunk would be mostly zeros, so each k8 step is
// instead one tap's 8 channels and a stage holds four taps ([4 taps][4 segments][8 ch][40 px], the same 20 KB).
//   wgrad : dW_(r,s)^T[C x K] = X_(r,s)[C x P] * dY[K x P]^T, again with the shifted activations as the register
//           operand (128 channels per CTA from a [128 ch][44 px] box, the tap an address offset) and dY as the K-major
//           B operand straight from TMA ([NT k][32 px], SWIZZLE_128B).  One work item = (tap, 128-channel block, group
//           of NT outputs, a range of row segments): all taps in one launch; flushed with fp32 atomics.
//
// Error: every fprop / dgrad output is a chain of R*S*ceil(Cin / 8) fp32 additions of k8 partial sums (<= 49 x 32 =
// 1568 for Cin <= 256); a wgrad item adds at most 4 x TW_MAX_CHAIN = 2048 k8 partial sums, and each dw element gets one
// atomic per row-segment split (<= ceil(segments / 512)).  A chain of L fp32 additions adds at most about L 2^-24 A, <= 2^-12 A for L <= 4096: with
// tf32-representable inputs (exact products) the result meets include/spconv.h's 2^-12 A, and with arbitrary inputs the
// rounding of both operands to tf32 (2^-11 relative each) adds the rest of (2^-9 + 2^-12) A.
// Warp roles (384 threads): warp 0 = TMA producer, warpgroups 1 and 2 = wgmma consumers.  Persistent CTAs.
#include "tap_tf32_common.cuh"

namespace spc {

namespace {

using namespace tc;

constexpr int TT_XW = 40;                     // pixels per box row: a segment and 4 pixels of slack on each side
constexpr int TT_SEG = TT_BK * TT_XW * 4;     // one [32 ch][40 px] box: 5 KB
constexpr int TT_XSTAGE = 4 * TT_SEG;         // a tile's four segments: 20 KB
constexpr int TT_SMALL_SEG = 8 * TT_XW * 4;   // small-Cin mode: one [8 ch][40 px] box: 1280 B
constexpr int TW_XW = 44;                     // wgrad: pixels per box row (4 slack left, 8 right; pitch 12 mod 32)
constexpr int TW_XBOX = 128 * TW_XW * 4;      // wgrad: one [128 ch][44 px] box: 22 KB

// ---- weight repack: Wp[rb][m][pos] = tf32(filter value), zero padded to [blocks][Mpad][Cpad] ------------------------
//   fprop: m = k, c = input channel, w[m][c][r][s]      dgrad: m = input channel, c = k, w[c][m][R-1-r][S-1-s]
//   row block rb = tap, pos = c;  small-Cin mode (Cpad = 32): rb = a group of four taps, pos = 8 * (tap % 4) + c
__global__ void tf32_tap_repack_kernel(const float* __restrict__ w, float* __restrict__ wp, int M, int Cc, int Mpad,
                                       int Cpad, int R, int S, int dgrad, int small) {
  const int blocks = small ? (R * S + 3) / 4 : R * S;
  const long long total = (long long)blocks * Mpad * Cpad;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int pos = (int)(i % Cpad), m = (int)((i / Cpad) % Mpad), rb = (int)(i / ((long long)Cpad * Mpad));
    const int tap = small ? 4 * rb + pos / 8 : rb, c = small ? pos % 8 : pos;
    const int r = tap / S, s = tap % S;
    float v = 0.f;
    if (m < M && c < Cc && tap < R * S) {
      const size_t src = dgrad ? (((size_t)c * M + m) * R + (R - 1 - r)) * S + (S - 1 - s)
                               : (((size_t)m * Cc + c) * R + r) * S + s;
      v = __uint_as_float(to_tf32(w[src]));
    }
    wp[i] = v;
  }
}

// ---- fprop / dgrad kernel: Y^T[128 px x NT ch] per tile, summed over taps and k-chunks --------------------------------
// A tile is four 32-pixel row segments (consecutive in the [N][H][ceil(W / 32)] segment order): 128 contiguous pixels of
// one row when W >= 128.  Segments past the last one lie at n >= N, which TMA loads as zeros and stores nowhere.
struct TapParams {
  int M;                 // valid output channels
  int Cin;               // reduction channels
  int H, R, S, ph, pw;
  int segs_row;          // ceil(W / 32)
  int kchunks;           // ceil(Cin / 32)
  int steps;             // R * S * kchunks, in the order (r, s, k-chunk); SMALL: ceil(R * S / 4), kchunks = 1
  int mpad;              // rows per tap of the repacked weights
  int num_mg;            // groups of NT output channels
  int num_tiles;         // tiles * num_mg
  int stages, wres, out_bufs;
  const float* bias;     // [M] or null
};

// SMALL: the small-Cin mode (a template parameter, so that the general path compiles as if it did not exist)
template <int NT, int SMALL>
__global__ void __launch_bounds__(TT_THREADS, 1)
tf32_tap_gemm_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x,
                     const __grid_constant__ CUtensorMap tmap_y, const TapParams p) {
  constexpr int W_BYTES = NT * 128;                  // one 32-channel chunk of the group's NT weight rows of one tap
  constexpr int OUT_CH = NT < 64 ? NT : 64;          // output channels per epilogue staging block
  constexpr int OUT_BYTES = OUT_CH * 128 * 4;        // [4 segments][OUT_CH ch][128 B]
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int wres_bytes = p.wres ? p.steps * W_BYTES : 0;
  const int stage_bytes = (p.wres ? 0 : W_BYTES) + TT_XSTAGE;
  uint8_t* wres = smem;
  uint8_t* stage0 = smem + wres_bytes;
  uint8_t* outbuf = stage0 + p.stages * stage_bytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(outbuf + p.out_bufs * OUT_BYTES);
  uint64_t* empty = full + TT_MAX_STAGES;
  uint64_t* wfull = empty + TT_MAX_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.stages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 2); }
    mbar_init(wfull, 1);
    fence_barrier_init();
  }
  __syncthreads();

  // register split as tf32_pw_gemm_kernel: 40 for the producer warpgroup, 232 for each consumer warpgroup
  if (threadIdx.x < 128) {
    setmaxnreg_dec<40>();
    // ================= TMA producer =================
    if (warp == 0 && lane == 0) {
      tma_prefetch_desc(&tmap_w);
      tma_prefetch_desc(&tmap_x);
      if (p.wres) {
        mbar_arrive_expect_tx(wfull, wres_bytes);
        for (int st = 0; st < p.steps; ++st)
          tma_load_2d(wres + st * W_BYTES, &tmap_w, wfull, (st % p.kchunks) * TT_BK, (st / p.kchunks) * p.mpad);
      }
      int s = 0, ph = 0;
      for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
        const int mg = t % p.num_mg, tt = t / p.num_mg;
        int n[4], y[4], x0[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) seg_coords(4 * tt + j, p.segs_row, p.H, n[j], y[j], x0[j]);
        for (int st = 0; st < p.steps; ++st) {
          const int kc = st % p.kchunks, tap = st / p.kchunks;
          const int dy = tap / p.S - p.ph;
          mbar_wait(&empty[s], ph ^ 1);
          uint8_t* sp = stage0 + s * stage_bytes;
          mbar_arrive_expect_tx(&full[s], stage_bytes);
          if (!p.wres) {
            tma_load_2d(sp, &tmap_w, &full[s], kc * TT_BK, tap * p.mpad + mg * NT);
            sp += W_BYTES;
          }
          if (SMALL) {
            // four taps of 8 channels; a tap past R*S loads a box wholly outside the image (zeros)
            for (int q = 0; q < 4; ++q) {
              const int tq = 4 * st + q;
              const int dq = tq < p.R * p.S ? tq / p.S - p.ph : -(1 << 20);
#pragma unroll
              for (int j = 0; j < 4; ++j)
                tma_load_4d(sp + (4 * q + j) * TT_SMALL_SEG, &tmap_x, &full[s], x0[j] - 4, y[j] + dq, 0, n[j]);
            }
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
              tma_load_4d(sp + j * TT_SEG, &tmap_x, &full[s], x0[j] - 4, y[j] + dy, kc * TT_BK, n[j]);
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
    const int g = lane >> 2, t4 = lane & 3;
    const bool wg_lead = (threadIdx.x & 127) == 0;
    const bool leader = threadIdx.x == 128;   // issues the TMA stores
    // fragment rows g, g + 8: pixels pt, pt + 8 of the tile, both in segment jb; columns t4, t4 + 4: channels.
    // Element (channel c, pixel q of the segment) of a box sits at (c * TT_XW + q + 4) * 4, plus the tap's offset.
    // A k8 step is 8 channel rows of the segment's box, or (small) the box of the next tap.
    const int pt = 64 * wg + 16 * w4 + g;
    const int jb = pt >> 5;
    const uint32_t xoff0 = jb * (SMALL ? TT_SMALL_SEG : TT_SEG) + (t4 * TT_XW + (pt & 31) + 4) * 4;
    const uint32_t off[4] = {xoff0, xoff0 + 8 * 4, xoff0 + 4 * TT_XW * 4, xoff0 + (4 * TT_XW + 8) * 4};
    float acc[NT / 2];
    if (p.wres) mbar_wait(wfull, 0);
    int s = 0, ph = 0, ob = 0;
    for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
      const int mg = t % p.num_mg, tt = t / p.num_mg;
      for (int st = 0; st < p.steps; ++st) {
        mbar_wait(&full[s], ph);
        const uint32_t sb = smem_u32(stage0 + s * stage_bytes);
        const uint32_t sw = p.wres ? smem_u32(wres + st * W_BYTES) : sb;
        // horizontal offset of each k-step's tap: one tap per stage, or (small) four consecutive taps
        const int tap0 = SMALL ? 4 * st : st / p.kchunks;
        const int s0 = tap0 % p.S;
        const uint32_t sx = (p.wres ? sb : sb + W_BYTES) + (s0 - p.pw) * 4;
        uint32_t koff[4];   // per k-step, computed before the loads so that all 16 issue back to back
        if (SMALL) {
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) koff[ks] = sx + ks * (4 * TT_SMALL_SEG) + (((tap0 + ks) % p.S) - s0) * 4;
        } else {
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) koff[ks] = sx + ks * (8 * TT_XW * 4);
        }
        uint32_t a[4][4];
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            float v;
            asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(koff[ks] + off[r]));
            a[ks][r] = to_tf32(v);
          }
        // always all 4 k-steps (no wgmma under a data-dependent branch); channels past Cin are zero in both operands
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          const uint64_t bdesc = gmma_desc(sw + ks * 32, 16, 1024);
          WgmmaTf32<NT>::mma_rs(acc, a[ks], bdesc, (st | ks) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();   // the A registers are reloaded next step
        reg_fence(acc);
        if (wg_lead) mbar_arrive(&empty[s]);
        if (++s == p.stages) { s = 0; ph ^= 1; }
      }
      // ===== epilogue: per OUT_CH-channel block, registers -> [4 segments][OUT_CH][128 B] swizzled smem -> TMA =====
      int n[4], y[4], x0[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) seg_coords(4 * tt + j, p.segs_row, p.H, n[j], y[j], x0[j]);
#pragma unroll
      for (int cb = 0; cb < NT / OUT_CH; ++cb) {
        const int k0 = mg * NT + cb * OUT_CH;
        if (k0 >= p.M) break;   // block-uniform
        uint8_t* buf = outbuf + ob * OUT_BYTES;
        if (leader) { if (p.out_bufs == 2) tma_store_wait_read<1>(); else tma_store_wait_read<0>(); }
        named_bar_sync(1, 256);
#pragma unroll
        for (int h = 0; h < 2; ++h) {   // fragment rows g and g + 8: pixels pt and pt + 8
          const int q = (pt & 31) + 8 * h;
          uint8_t* col = buf + jb * (OUT_CH * 128) + (q & 3) * 4;
#pragma unroll
          for (int j = 0; j < OUT_CH / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int cl = 8 * j + 2 * t4 + e;
              const int k = k0 + cl;
              const float bias = (p.bias && k < p.M) ? p.bias[k] : 0.f;
              *reinterpret_cast<float*>(col + cl * 128 + ((((q >> 2) ^ (cl & 7))) << 4)) =
                  acc[4 * (cb * (OUT_CH / 8) + j) + 2 * h + e] + bias;
            }
          }
        }
        fence_proxy_async();
        named_bar_sync(1, 256);
        if (leader) {
#pragma unroll
          for (int j = 0; j < 4; ++j) tma_store_4d(&tmap_y, buf + j * (OUT_CH * 128), x0[j], y[j], k0, n[j]);
          tma_store_commit();
        }
        if (p.out_bufs == 2) ob ^= 1;
      }
    }
    if (leader) tma_store_wait_read<0>();
  }
}

template <int NT, int SMALL>
int launch_tap_gemm(const CUtensorMap& tw, const CUtensorMap& tx, const CUtensorMap& ty, TapParams p, cudaStream_t st) {
  constexpr int OUT_BYTES = (NT < 64 ? NT : 64) * 128 * 4;
  const int budget = TT_SMEM_LIMIT - TT_SMEM_AUX;
  const int wres_bytes = p.steps * NT * 128;
  int smem = 0;
  // weights stay resident when they fit and every CTA needs the same rows (one group of output channels)
  for (int wres = (wres_bytes <= TT_WRES_MAX && p.num_mg == 1) ? 1 : 0; wres >= 0; --wres) {
    const int stage_bytes = (wres ? 0 : NT * 128) + TT_XSTAGE;
    const int rem = budget - (wres ? wres_bytes : 0);
    p.wres = wres;
    p.out_bufs = 2;
    p.stages = (rem - 2 * OUT_BYTES) / stage_bytes;
    if (p.stages < 3) { p.out_bufs = 1; p.stages = (rem - OUT_BYTES) / stage_bytes; }
    if (p.stages > TT_MAX_STAGES) p.stages = TT_MAX_STAGES;
    smem = (wres ? wres_bytes : 0) + p.stages * stage_bytes + p.out_bufs * OUT_BYTES + TT_SMEM_AUX;
    if (p.stages >= 2) break;
  }
  SPC_REQUIRE(p.stages >= 2, "tf32 tap conv: shared memory budget too small (NT=%d steps=%d)", NT, p.steps);
  auto kern = tf32_tap_gemm_kernel<NT, SMALL>;
  const int rc = allow_dynamic_smem((const void*)kern, TT_SMEM_LIMIT);
  if (rc) return rc;
  const int sms = sm_count();
  kern<<<p.num_tiles < sms ? p.num_tiles : sms, TT_THREADS, smem, st>>>(tw, tx, ty, p);
  count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

size_t tap_wp_bytes(int taps, int M, int Cin) {
  return (size_t)taps * round_up(M, tap_nt(M)) * round_up(Cin, TT_BK) * 4;
}

// fprop (dgrad = 0): y[N][K][H][W] = conv(x[N][C][H][W], w) + bias;  dgrad: y = dx[N][C][H][W] from x = dy[N][K][H][W]
int run_tap_gemm(const spc_conv_desc* d, int dgrad, const float* w, const float* x, const float* bias, float* y,
                 void* ws, cudaStream_t st) {
  const int M = dgrad ? d->C : d->K, Cin = dgrad ? d->K : d->C, taps = d->R * d->S;
  const int NT = tap_nt(M);
  const int small = Cin <= 8 ? 1 : 0;
  const int Mpad = round_up(M, NT), Cpad = round_up(Cin, TT_BK);
  const int rblocks = small ? (taps + 3) / 4 : taps;
  float* wp = reinterpret_cast<float*>(align1k(reinterpret_cast<uintptr_t>(ws)));
  {
    const long long total = (long long)rblocks * Mpad * Cpad;
    long long blocks = (total + 255) / 256;
    if (blocks > 1184) blocks = 1184;
    tf32_tap_repack_kernel<<<(int)blocks, 256, 0, st>>>(w, wp, M, Cin, Mpad, Cpad, d->R, d->S, dgrad, small);
    count_launch();
    SPC_CHECK_CUDA(cudaGetLastError());
  }
  CUtensorMap tw, tx, ty;
  {
    const uint64_t dims[2] = {(uint64_t)Cpad, (uint64_t)rblocks * Mpad};
    const uint64_t strides[2] = {0, (uint64_t)Cpad * 4};
    const uint32_t box[2] = {TT_BK, (uint32_t)NT};
    int rc = make_tmap(&tw, wp, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  int rc = make_act_tmap4(&tx, x, d->N, Cin, d->H, d->W, small ? 8 : TT_BK, TT_XW, false);
  if (rc) return rc;
  rc = make_act_tmap4(&ty, y, d->N, M, d->H, d->W, NT < 64 ? NT : 64, 32, true);
  if (rc) return rc;
  TapParams p{};
  p.M = M; p.Cin = Cin; p.bias = bias;
  p.H = d->H; p.R = d->R; p.S = d->S; p.ph = d->pad_h; p.pw = d->pad_w;
  p.segs_row = (d->W + 31) / 32;
  p.kchunks = Cpad / TT_BK;
  p.steps = rblocks * p.kchunks;
  p.mpad = Mpad;
  p.num_mg = Mpad / NT;
  const long long tiles = ((long long)d->N * d->H * p.segs_row + 3) / 4;
  SPC_REQUIRE(tiles * p.num_mg < (1ll << 31), "tf32 tap conv: too many tiles");
  p.num_tiles = (int)(tiles * p.num_mg);
  if (small) {
    switch (NT) {
      case 16: return launch_tap_gemm<16, 1>(tw, tx, ty, p, st);
      case 32: return launch_tap_gemm<32, 1>(tw, tx, ty, p, st);
      case 64: return launch_tap_gemm<64, 1>(tw, tx, ty, p, st);
      case 128: return launch_tap_gemm<128, 1>(tw, tx, ty, p, st);
      default: return launch_tap_gemm<256, 1>(tw, tx, ty, p, st);
    }
  }
  switch (NT) {
    case 16: return launch_tap_gemm<16, 0>(tw, tx, ty, p, st);
    case 32: return launch_tap_gemm<32, 0>(tw, tx, ty, p, st);
    case 64: return launch_tap_gemm<64, 0>(tw, tx, ty, p, st);
    case 128: return launch_tap_gemm<128, 0>(tw, tx, ty, p, st);
    default: return launch_tap_gemm<256, 0>(tw, tx, ty, p, st);
  }
}


// ---- wgrad kernel: dW_(r,s)^T[128 ch x NT k] += X_(r,s)[128 ch x P] * dY[NT k x P]^T per work item -------------------
struct TapWgParams {
  float* dw;             // [K][C][R][S] fp32
  int C, K, H, R, S, ph, pw;
  int segs_row;          // ceil(W / 32)
  int cblocks;           // ceil(C / 128)
  int num_kg;            // groups of NT outputs
  int splits;            // row-segment ranges per (tap, channel block, output group)
  int chunks_total;      // N * H * segs_row
  int stages;
  int split0, nsplit;    // this launch runs splits [split0, split0 + nsplit)
  size_t slice_stride;   // split sp adds into dw + (sp - split0) * slice_stride (common.cuh: WgradSlices)
};

template <int NT>
__global__ void __launch_bounds__(TT_THREADS, 1)
tf32_tap_wgrad_kernel(const __grid_constant__ CUtensorMap tmap_dy, const __grid_constant__ CUtensorMap tmap_x,
                      const TapWgParams p) {
  constexpr int B_BYTES = NT * 128;                  // [NT k][32 px], SWIZZLE_128B
  constexpr int STAGE = B_BYTES + TW_XBOX;           // a multiple of 1 KB
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + p.stages * STAGE);
  uint64_t* empty = full + TT_MAX_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < p.stages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 2); }
    fence_barrier_init();
  }
  __syncthreads();
  const int taps = p.R * p.S;
  const int groups = taps * p.cblocks * p.num_kg;
  const int it0 = p.split0 * groups, it1 = it0 + p.nsplit * groups;
  const int per_split = (p.chunks_total + p.splits - 1) / p.splits;
  // item -> (split, tap, channel block, output group): the items of one split run side by side and re-read its
  // segments from L2
#define TTW_DECODE(it)                                                                          \
  const int sp = (it) / groups, g_ = (it) % groups;                                            \
  const int tap = g_ % taps, cb = (g_ / taps) % p.cblocks, kg = g_ / taps / p.cblocks;          \
  const int c_begin = sp * per_split, c_end = min(p.chunks_total, c_begin + per_split);

  if (threadIdx.x < 128) {
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      tma_prefetch_desc(&tmap_dy);
      tma_prefetch_desc(&tmap_x);
      int s = 0, ph = 0;
      for (int it = it0 + blockIdx.x; it < it1; it += gridDim.x) {
        TTW_DECODE(it)
        const int dr = tap / p.S - p.ph;
        for (int ch = c_begin; ch < c_end; ++ch) {
          int n, y, x0;
          seg_coords(ch, p.segs_row, p.H, n, y, x0);
          mbar_wait(&empty[s], ph ^ 1);
          uint8_t* st = smem + s * STAGE;
          mbar_arrive_expect_tx(&full[s], STAGE);
          tma_load_4d(st, &tmap_dy, &full[s], x0, y, kg * NT, n);
          tma_load_4d(st + B_BYTES, &tmap_x, &full[s], x0 - 4, y + dr, cb * 128, n);
          if (++s == p.stages) { s = 0; ph ^= 1; }
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    const int wg = (threadIdx.x >> 7) - 1;
    const int w4 = (threadIdx.x >> 5) & 3;
    const int g = lane >> 2, t4 = lane & 3;
    const bool wg_lead = (threadIdx.x & 127) == 0;
    // A fragment: rows g, g + 8 = channels cr, cr + 8 of the block; columns t4, t4 + 4 = pixels of the k8 step.
    // Element (channel c, pixel q) sits at (c * TW_XW + q + 4) * 4: the 44-word pitch (12 mod 32) spreads a warp's
    // 8 channels x 4 pixels over 32 banks.
    const int cr = 64 * wg + 16 * w4 + g;
    const uint32_t xoff0 = (cr * TW_XW + t4 + 4) * 4;
    const uint32_t off[4] = {xoff0, xoff0 + 8 * TW_XW * 4, xoff0 + 4 * 4, xoff0 + (8 * TW_XW + 4) * 4};
    float acc[NT / 2];
    int s = 0, ph = 0;
    for (int it = it0 + blockIdx.x; it < it1; it += gridDim.x) {
      TTW_DECODE(it)
      float* dw = p.dw + (size_t)(sp - p.split0) * p.slice_stride;   // the items of one split add disjoint blocks
      const int dx = tap % p.S - p.pw;
      for (int ch = c_begin; ch < c_end; ++ch) {
        mbar_wait(&full[s], ph);
        const uint32_t sb = smem_u32(smem + s * STAGE);
        const uint32_t sx = sb + B_BYTES + dx * 4;
        uint32_t a[4][4];
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            float v;
            asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(sx + off[r] + ks * 8 * 4));
            a[ks][r] = to_tf32(v);
          }
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          const uint64_t bdesc = gmma_desc(sb + ks * 32, 16, 1024);
          WgmmaTf32<NT>::mma_rs(acc, a[ks], bdesc, (ch > c_begin || ks > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();   // the A registers are reloaded next step
        reg_fence(acc);
        if (wg_lead) mbar_arrive(&empty[s]);
        if (++s == p.stages) { s = 0; ph ^= 1; }
      }
      if (c_end > c_begin) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int c = cb * 128 + cr + 8 * h;
          if (c < p.C) {
#pragma unroll
            for (int j = 0; j < NT / 8; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int k = kg * NT + 8 * j + 2 * t4 + e;
                if (k < p.K) atomicAdd(&dw[((size_t)k * p.C + c) * taps + tap], acc[4 * j + 2 * h + e]);
              }
          }
        }
      }
    }
  }
#undef TTW_DECODE
}

template <int NT>
int launch_tap_wgrad(const CUtensorMap& tdy, const CUtensorMap& tx, TapWgParams p, cudaStream_t st, const WgradSlices* sl) {
  constexpr int STAGE = NT * 128 + TW_XBOX;
  p.stages = (TT_SMEM_LIMIT - TT_SMEM_AUX) / STAGE;
  if (p.stages > 6) p.stages = 6;
  SPC_REQUIRE(p.stages >= 2, "tf32 tap wgrad: smem budget");
  const int sms = sm_count();
  const long long groups = (long long)p.R * p.S * p.cblocks * p.num_kg;
  // at least two items per SM, at least 8 segments per item, at most TW_MAX_CHAIN segments per item
  long long splits = (2 * sms + groups - 1) / groups;
  if (splits > p.chunks_total / 8) splits = p.chunks_total / 8;
  const long long smin = (p.chunks_total + TW_MAX_CHAIN - 1) / TW_MAX_CHAIN;
  if (splits < smin) splits = smin;
  if (splits < 1) splits = 1;
  SPC_REQUIRE(groups * splits < (1ll << 31), "tf32 tap wgrad: too many work items");
  p.splits = (int)splits;
  auto kern = tf32_tap_wgrad_kernel<NT>;
  const int rc = allow_dynamic_smem((const void*)kern, TT_SMEM_LIMIT);
  if (rc) return rc;
  // smin makes up to chunks_total / TW_MAX_CHAIN splits: the deterministic path may need several passes for them
  return run_slices(sl, p.splits, (size_t)p.K * p.C * p.R * p.S, p.dw, st, [&](int s0, int ns, float* dst, size_t stride) {
    TapWgParams q = p;
    q.split0 = s0; q.nsplit = ns; q.dw = dst; q.slice_stride = stride;
    const long long items = groups * ns;
    kern<<<(int)(items < sms ? items : sms), TT_THREADS, p.stages * STAGE + TT_SMEM_AUX, st>>>(tdy, tx, q);
    count_launch();
    SPC_CHECK_CUDA(cudaGetLastError());
    return SPC_OK;
  });
}
}  // namespace

// fp32, stride 1, "same" padding, odd R x S up to 7 x 7 with more than one tap, 16-byte aligned rows (W % 4 == 0)
bool tf32_tap_supported(const spc_conv_desc* d) {
  if (d->dtype != SPC_F32 || d->stride_h != 1 || d->stride_w != 1) return false;
  if (d->R * d->S < 2 || d->R % 2 == 0 || d->S % 2 == 0 || d->R > 7 || d->S > 7) return false;
  if (d->pad_h != (d->R - 1) / 2 || d->pad_w != (d->S - 1) / 2) return false;
  return d->W % 4 == 0;
}

// the repacked weights of fprop (op 0) / dgrad (op 1); wgrad needs none
size_t tf32_tap_workspace_bytes(const spc_conv_desc* d, int op) {
  if (op == 2) return 0;
  return align1k(op == 0 ? tap_wp_bytes(d->R * d->S, d->K, d->C) : tap_wp_bytes(d->R * d->S, d->C, d->K)) + 1024;
}

int tf32_tap_fwd(const spc_conv_desc* d, const void* x, const void* w, const void* bias, void* y, void* ws,
                 size_t ws_bytes, cudaStream_t st) {
  SPC_REQUIRE(ws && ws_bytes >= tf32_tap_workspace_bytes(d, 0), "tf32 tap conv: workspace too small");
  return run_tap_gemm(d, 0, reinterpret_cast<const float*>(w), reinterpret_cast<const float*>(x),
                      reinterpret_cast<const float*>(bias), reinterpret_cast<float*>(y), ws, st);
}

int tf32_tap_dgrad(const spc_conv_desc* d, const void* dy, const void* w, void* dx, void* ws, size_t ws_bytes,
                   cudaStream_t st) {
  SPC_REQUIRE(ws && ws_bytes >= tf32_tap_workspace_bytes(d, 1), "tf32 tap conv: workspace too small");
  return run_tap_gemm(d, 1, reinterpret_cast<const float*>(w), reinterpret_cast<const float*>(dy), nullptr,
                      reinterpret_cast<float*>(dx), ws, st);
}

// dw[K][C][R][S] += the interior's share (zero padding), with atomics; api.cu adds the halo strips' share.  Needs no
// workspace.
int tf32_tap_wgrad(const spc_conv_desc* d, const void* x, const void* dy, float* dw, void*, size_t, cudaStream_t st,
                   const WgradSlices* sl) {
  TapWgParams p{};
  p.dw = dw; p.C = d->C; p.K = d->K; p.H = d->H; p.R = d->R; p.S = d->S; p.ph = d->pad_h; p.pw = d->pad_w;
  p.segs_row = (d->W + 31) / 32;
  const long long chunks = (long long)d->N * d->H * p.segs_row;
  SPC_REQUIRE(chunks < (1ll << 31), "tf32 tap wgrad: too many row segments");
  p.chunks_total = (int)chunks;
  const int NT = tap_nt(d->K);
  p.cblocks = (d->C + 127) / 128;
  p.num_kg = round_up(d->K, NT) / NT;
  CUtensorMap tdy, tx;
  int rc = make_act_tmap4(&tdy, dy, d->N, d->K, d->H, d->W, NT, 32, true);
  if (rc) return rc;
  rc = make_act_tmap4(&tx, x, d->N, d->C, d->H, d->W, 128, TW_XW, false);
  if (rc) return rc;
  switch (NT) {
    case 16: return launch_tap_wgrad<16>(tdy, tx, p, st, sl);
    case 32: return launch_tap_wgrad<32>(tdy, tx, p, st, sl);
    case 64: return launch_tap_wgrad<64>(tdy, tx, p, st, sl);
    case 128: return launch_tap_wgrad<128>(tdy, tx, p, st, sl);
    default: return launch_tap_wgrad<256>(tdy, tx, p, st, sl);
  }
}

// Slice copies of the tap wgrads: launch_tap_wgrad and conv_tap_s2_tf32.cu's launch_s2_wgrad make >= chunks /
// TW_MAX_CHAIN splits (the longest chain an item may sum), else <= 2 * SMs; the direct kernel's launches over the
// boundary rectangles (api.cu) make their CTA columns
double tf32_tap_wgrad_slice_floats(const spc_conv_desc* d) {
  int Ho, Wo;
  spc_conv_out_shape(d, &Ho, &Wo);
  const double wn = (double)d->K * d->C * d->R * d->S, chunks = (double)d->N * Ho * ((Wo + 31) / 32);
  const double interior = fmax(2.0 * sm_count(), ceil(chunks / TW_MAX_CHAIN)) * wn;
  return fmax(interior, fmax(direct_wgrad_slice_floats(d, Ho, d->pad_w), direct_wgrad_slice_floats(d, d->pad_h, Wo)));
}

}  // namespace spc
