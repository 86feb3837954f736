// conv_tap_s2_tf32.cu -- fp32 stride-2 multi-tap convolutions (R, S in {3, 5, 7}, "same" padding) on the tensor cores
// in TF32: fprop, dgrad and wgrad (opt-in: SPC_ALGO_TF32_STRIDED).
//
// The structure is conv_tap_tf32.cu's: the transposed product with the shifted activations as the register operand A
// (wgmma .tf32 has no transpose), the repacked weights / dY as the K-major SWIZZLE_128B operand B, 384 threads
// (warp 0 = TMA producer, warpgroups 1 and 2 = wgmma consumers), persistent CTAs.  x is read in place: no phase-split
// or subsampled copy in HBM.
//   fprop : Y^T[P_out x K] = sum_(r,s) X_(r,s)^T * W_(r,s)^T,   X_(r,s)(oy, ox) = X(2 oy + r - ph, 2 ox + s - pw).
//           A tile is four 32-output-pixel row segments.  The box of a segment at (oy, x0) for the taps of row r is
//           [32 ch][72 px] from (2 oy + r - ph, 2 x0 - 4), unswizzled, and the stride is in the ld.shared address:
//           output pixel q of the segment under tap (r, s) reads word 2 q + s - pw + 4 of its channel row.  A box pitch
//           is a multiple of 4 words, so the 32 addresses of a fragment load (8 pixels x 4 channels) fall on the 16
//           even banks: two-way conflicts, whatever the pitch.
//           Small-Cin mode (Cin <= 8, the C = 3 stem) as in conv_tap_tf32.cu: a k8 step is one tap's 8 channels, a stage
//           four taps.
//   dgrad : dx(2 i + a, 2 j + b) is, per parity class (a, b), a stride-1 correlation of dy with the taps r = a + ph,
//           s = b + pw (mod 2): dy(i + (a + ph - r) / 2, j + (b + pw - s) / 2) * w[k][c][r][s].  One launch runs the four
//           classes as four sets of tiles over the [N][H / 2][W / 2] pixels of a class, each with its own taps only
//           (3x3: 1, 2, 2 and 4), dy read at unit stride from conv_tap_tf32.cu's [32 ch][40 px] boxes.  The epilogue
//           stores the accumulators to dx directly, at a pixel stride of 2: dx is written once, in half-used sectors.
//           With R, S >= 3 every class has a tap, so all of dx is written.
//   wgrad : dW_(r,s)^T[C x K] = X_(r,s)[C x P_out] * dY[K x P_out]^T: 128 channels of x per CTA from a [128 ch][72 px]
//           box (pixel stride 2 in the fragment addresses, two-way conflicts as in fprop), dY [NT k][32 px] straight
//           from TMA.  One work item = (tap, 128-channel block, group of NT outputs, a range of row segments), all taps in
//           one launch, fp32 atomics: conv_tap_tf32.cu's split rule and chain limit.
// TMA fills coordinates outside the image with zeros: the zero padding of the interior pass; api.cu recomputes the
// outputs whose windows reach a received halo strip.
//
// Error: as conv_tap_tf32.cu.  An fprop output is a chain of R*S*ceil(Cin / 8) fp32 additions of k8 partial sums, a
// dgrad output of at most ceil(R / 2)*ceil(S / 2)*ceil(K / 8); a wgrad item adds at most 4 x TW_MAX_CHAIN of them and
// each dw element gets one atomic per row-segment split: all <= 4096, so include/spconv.h's bounds hold.
#include "tap_tf32_common.cuh"

namespace spc {

namespace {

using namespace tc;

constexpr int S2_XW = 72;                     // fprop / wgrad: pixels per box row (4 + 2 * 31 + 3 + 1 <= 70, 16-byte rows)
constexpr int S2_DXW = 40;                    // dgrad: a segment of dy and 4 pixels of slack on each side
constexpr int S2_WG_XBOX = 128 * S2_XW * 4;   // wgrad: one [128 ch][72 px] box: 36 KB
constexpr int S2_MAX_TAPS = 52;               // 7 x 7, rounded up to the small-Cin mode's groups of four

// The taps in the order the kernels walk them: fprop (r, s) row-major; dgrad class by class (cls_begin).  dy / dx are
// what a tap adds to the row / column the box is loaded from / read at.
struct TapTable {
  int dy[S2_MAX_TAPS];
  signed char dx[S2_MAX_TAPS];
  unsigned char r[S2_MAX_TAPS], s[S2_MAX_TAPS];
  int n;
  int cls_begin[5];
};
constexpr int S2_NO_ROW = -(1 << 20);         // dy of the small-Cin mode's taps past R * S: a row outside any image

enum { S2_FPROP = 0, S2_FPROP_SMALL = 1, S2_DGRAD = 2 };

// ---- weight repack: Wp[rb][m][pos] = tf32(filter value), zero padded to [blocks][Mpad][Cpad] ------------------------
//   fprop: m = k, c = input channel, w[m][c][r][s]      dgrad: m = input channel, c = k, w[c][m][r][s]
//   row block rb = tap of the table, pos = c;  small-Cin mode (Cpad = 32): rb = four taps, pos = 8 * (tap % 4) + c
__global__ void tf32_s2_repack_kernel(const float* __restrict__ w, float* __restrict__ wp, int M, int Cc, int Mpad,
                                      int Cpad, int R, int S, int dgrad, int small, const TapTable tt) {
  const int blocks = small ? (tt.n + 3) / 4 : tt.n;
  const long long total = (long long)blocks * Mpad * Cpad;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int pos = (int)(i % Cpad), m = (int)((i / Cpad) % Mpad), rb = (int)(i / ((long long)Cpad * Mpad));
    const int tap = small ? 4 * rb + pos / 8 : rb, c = small ? pos % 8 : pos;
    float v = 0.f;
    if (m < M && c < Cc && tap < tt.n) {
      const int r = tt.r[tap], s = tt.s[tap];
      const size_t src = dgrad ? (((size_t)c * M + m) * R + r) * S + s : (((size_t)m * Cc + c) * R + r) * S + s;
      v = __uint_as_float(to_tf32(w[src]));
    }
    wp[i] = v;
  }
}

// ---- fprop / dgrad kernel: Y^T[128 px x NT ch] per tile, summed over the tile's taps and k-chunks ---------------------
// A tile is four 32-pixel row segments, consecutive in the [N][rows][ceil(cols / 32)] segment order of the output
// (fprop) or of one parity class of dx (dgrad).  Segments past the last one lie at n >= N: TMA loads them as zeros.
struct S2Params {
  int M;                 // valid output channels
  int N;
  int rows, cols;        // the segment grid: Ho x Wo (fprop), H / 2 x W / 2 (dgrad)
  int segs_row;          // ceil(cols / 32)
  int kchunks;           // ceil(Cin / 32); small-Cin mode: 1
  int mpad;              // rows per tap of the repacked weights
  int num_mg;            // groups of NT output channels
  int num_tiles;         // tiles * classes * num_mg
  int stages, wres, out_bufs;
  const float* bias;     // [M] or null
  float* dx;             // dgrad: [N][M][2 rows][2 cols]
  TapTable tt;           // small-Cin mode: cls_begin counts groups of four taps
};

template <int NT, int MODE>
__global__ void __launch_bounds__(TT_THREADS, 1)
tf32_s2_gemm_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x,
                    const __grid_constant__ CUtensorMap tmap_y, const __grid_constant__ S2Params p) {
  constexpr bool SMALL = MODE == S2_FPROP_SMALL, DGRAD = MODE == S2_DGRAD;
  constexpr int PS = DGRAD ? 1 : 2;                  // pixel stride of the A operand, in words
  constexpr int XW = DGRAD ? S2_DXW : S2_XW;
  constexpr int SEG = (SMALL ? 8 : TT_BK) * XW * 4;  // one segment's box
  constexpr int XSTAGE = (SMALL ? 16 : 4) * SEG;     // a tile's four segments (small-Cin mode: of four taps)
  constexpr int NCLS = DGRAD ? 4 : 1;
  constexpr int W_BYTES = NT * 128;                  // one 32-channel chunk of the group's NT weight rows of one tap
  constexpr int OUT_CH = NT < 64 ? NT : 64;          // output channels per epilogue staging block
  constexpr int OUT_BYTES = OUT_CH * 128 * 4;        // [4 segments][OUT_CH ch][128 B]
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int wres_bytes = p.wres ? p.tt.cls_begin[NCLS] * p.kchunks * W_BYTES : 0;
  const int stage_bytes = (p.wres ? 0 : W_BYTES) + XSTAGE;
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

  // tile -> (group of output channels, parity class, four segments); the steps of a tile are those of its class
#define S2_DECODE(t)                                                                  \
  const int mg = (t) % p.num_mg, cls = ((t) / p.num_mg) % NCLS, tt = (t) / p.num_mg / NCLS; \
  const int st_begin = p.tt.cls_begin[cls] * p.kchunks, st_end = p.tt.cls_begin[cls + 1] * p.kchunks;

  if (threadIdx.x < 128) {
    setmaxnreg_dec<40>();
    // ================= TMA producer =================
    if (warp == 0 && lane == 0) {
      tma_prefetch_desc(&tmap_w);
      tma_prefetch_desc(&tmap_x);
      if (p.wres) {
        mbar_arrive_expect_tx(wfull, wres_bytes);
        const int steps = p.tt.cls_begin[NCLS] * p.kchunks;
        for (int st = 0; st < steps; ++st)
          tma_load_2d(wres + st * W_BYTES, &tmap_w, wfull, (st % p.kchunks) * TT_BK, (st / p.kchunks) * p.mpad);
      }
      int s = 0, ph = 0;
      for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
        S2_DECODE(t)
        int n[4], y[4], x0[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) seg_coords(4 * tt + j, p.segs_row, p.rows, n[j], y[j], x0[j]);
        for (int st = st_begin; st < st_end; ++st) {
          const int kc = st % p.kchunks, tap = st / p.kchunks;
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
              const int dq = p.tt.dy[4 * st + q];
#pragma unroll
              for (int j = 0; j < 4; ++j)
                tma_load_4d(sp + (4 * q + j) * SEG, &tmap_x, &full[s], PS * x0[j] - 4, PS * y[j] + dq, 0, n[j]);
            }
          } else {
            const int dy = p.tt.dy[tap];
#pragma unroll
            for (int j = 0; j < 4; ++j)
              tma_load_4d(sp + j * SEG, &tmap_x, &full[s], PS * x0[j] - 4, PS * y[j] + dy, kc * TT_BK, n[j]);
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
    // Element (channel c, pixel q of the segment) of a box sits at word c * XW + PS * q + 4, plus the tap's offset.
    // A k8 step is 8 channel rows of the segment's box, or (small) the box of the next tap.
    const int pt = 64 * wg + 16 * w4 + g;
    const int jb = pt >> 5;
    const uint32_t xoff0 = jb * SEG + (t4 * XW + PS * (pt & 31) + 4) * 4;
    const uint32_t off[4] = {xoff0, xoff0 + PS * 8 * 4, xoff0 + 4 * XW * 4, xoff0 + (4 * XW + PS * 8) * 4};
    float acc[NT / 2];
    if (p.wres) mbar_wait(wfull, 0);
    int s = 0, ph = 0, ob = 0;
    for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
      S2_DECODE(t)
      for (int st = st_begin; st < st_end; ++st) {
        mbar_wait(&full[s], ph);
        const uint32_t sb = smem_u32(stage0 + s * stage_bytes);
        const uint32_t sw = p.wres ? smem_u32(wres + st * W_BYTES) : sb;
        const uint32_t sx = p.wres ? sb : sb + W_BYTES;
        uint32_t koff[4];   // per k-step, computed before the loads so that all 16 issue back to back
        if (SMALL) {
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) koff[ks] = sx + ks * (4 * SEG) + p.tt.dx[4 * st + ks] * 4;
        } else {
          const uint32_t sxt = sx + p.tt.dx[st / p.kchunks] * 4;
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) koff[ks] = sxt + ks * (8 * XW * 4);
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
          WgmmaTf32<NT>::mma_rs(acc, a[ks], bdesc, (st > st_begin || ks > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();   // the A registers are reloaded next step
        reg_fence(acc);
        if (wg_lead) mbar_arrive(&empty[s]);
        if (++s == p.stages) { s = 0; ph ^= 1; }
      }
      if (DGRAD) {
        // ===== epilogue: registers -> dx(2 i + a, 2 j + b) of the tile's class, no staging =====
        int n, y, x0;
        seg_coords(4 * tt + jb, p.segs_row, p.rows, n, y, x0);
        if (n < p.N) {
          const size_t plane = (size_t)4 * p.rows * p.cols;
          float* row = p.dx + (size_t)n * p.M * plane + (size_t)(2 * y + (cls >> 1)) * (2 * p.cols) + (cls & 1);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int x = x0 + (pt & 31) + 8 * h;
            if (x < p.cols) {
#pragma unroll
              for (int j = 0; j < NT / 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const int c = mg * NT + 8 * j + 2 * t4 + e;
                  if (c < p.M) row[c * plane + 2 * x] = acc[4 * j + 2 * h + e];
                }
            }
          }
        }
      } else {
        // ===== epilogue: per OUT_CH-channel block, registers -> [4 segments][OUT_CH][128 B] swizzled smem -> TMA =====
        int n[4], y[4], x0[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) seg_coords(4 * tt + j, p.segs_row, p.rows, n[j], y[j], x0[j]);
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
    }
    if (!DGRAD && leader) tma_store_wait_read<0>();
  }
#undef S2_DECODE
}

template <int NT, int MODE>
int launch_s2_gemm(const CUtensorMap& tw, const CUtensorMap& tx, const CUtensorMap& ty, S2Params p, cudaStream_t st) {
  constexpr bool DGRAD = MODE == S2_DGRAD;
  constexpr int OUT_BYTES = DGRAD ? 0 : (NT < 64 ? NT : 64) * 128 * 4;   // dgrad stores from registers
  constexpr int XSTAGE = 4 * TT_BK * (DGRAD ? S2_DXW : S2_XW) * 4;
  const int budget = TT_SMEM_LIMIT - TT_SMEM_AUX;
  const int wres_bytes = p.tt.cls_begin[DGRAD ? 4 : 1] * p.kchunks * NT * 128;
  int smem = 0;
  // weights stay resident when they fit and every CTA needs the same rows (one group of output channels)
  for (int wres = (wres_bytes <= TT_WRES_MAX && p.num_mg == 1) ? 1 : 0; wres >= 0; --wres) {
    const int stage_bytes = (wres ? 0 : NT * 128) + XSTAGE;
    const int rem = budget - (wres ? wres_bytes : 0);
    p.wres = wres;
    p.out_bufs = DGRAD ? 0 : 2;
    p.stages = (rem - 2 * OUT_BYTES) / stage_bytes;
    if (!DGRAD && p.stages < 3) { p.out_bufs = 1; p.stages = (rem - OUT_BYTES) / stage_bytes; }
    if (p.stages > TT_MAX_STAGES) p.stages = TT_MAX_STAGES;
    smem = (wres ? wres_bytes : 0) + p.stages * stage_bytes + p.out_bufs * OUT_BYTES + TT_SMEM_AUX;
    if (p.stages >= 2) break;
  }
  SPC_REQUIRE(p.stages >= 2, "tf32 stride-2 tap conv: shared memory budget too small (NT=%d)", NT);
  auto kern = tf32_s2_gemm_kernel<NT, MODE>;
  const int rc = allow_dynamic_smem((const void*)kern, TT_SMEM_LIMIT);
  if (rc) return rc;
  const int sms = sm_count();
  kern<<<p.num_tiles < sms ? p.num_tiles : sms, TT_THREADS, smem, st>>>(tw, tx, ty, p);
  count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

template <int MODE>
int launch_s2_gemm_nt(int NT, const CUtensorMap& tw, const CUtensorMap& tx, const CUtensorMap& ty, const S2Params& p,
                      cudaStream_t st) {
  switch (NT) {
    case 16: return launch_s2_gemm<16, MODE>(tw, tx, ty, p, st);
    case 32: return launch_s2_gemm<32, MODE>(tw, tx, ty, p, st);
    case 64: return launch_s2_gemm<64, MODE>(tw, tx, ty, p, st);
    case 128: return launch_s2_gemm<128, MODE>(tw, tx, ty, p, st);
    default: return launch_s2_gemm<256, MODE>(tw, tx, ty, p, st);
  }
}

// fprop: (r, s) row-major, one class.  dgrad: the taps of class (a, b) = cls / 2, cls % 2, class after class.
TapTable make_taps(const spc_conv_desc* d, int dgrad) {
  TapTable t{};
  for (int i = 0; i < S2_MAX_TAPS; ++i) t.dy[i] = S2_NO_ROW;
  for (int cls = 0; cls < (dgrad ? 4 : 1); ++cls) {
    t.cls_begin[cls] = t.n;
    for (int r = 0; r < d->R; ++r)
      for (int s = 0; s < d->S; ++s) {
        const int a = cls >> 1, b = cls & 1;
        if (dgrad && ((a + d->pad_h - r) % 2 || (b + d->pad_w - s) % 2)) continue;
        t.r[t.n] = (unsigned char)r; t.s[t.n] = (unsigned char)s;
        // floor division: a + pad - r is even here
        t.dy[t.n] = (dgrad ? (a + d->pad_h - r) / 2 : r - d->pad_h);
        t.dx[t.n] = (signed char)(dgrad ? (b + d->pad_w - s) / 2 : s - d->pad_w);
        ++t.n;
      }
  }
  for (int cls = dgrad ? 4 : 1; cls < 5; ++cls) t.cls_begin[cls] = t.n;
  return t;
}

size_t s2_wp_bytes(int taps, int M, int Cin) {
  return (size_t)taps * round_up(M, tap_nt(M)) * round_up(Cin, TT_BK) * 4;
}

// fprop (dgrad = 0): y[N][K][H/2][W/2] = conv(x[N][C][H][W], w) + bias;  dgrad: y = dx[N][C][H][W] from x = dy
int run_s2_gemm(const spc_conv_desc* d, int dgrad, const float* w, const float* x, const float* bias, float* y,
                void* ws, cudaStream_t st) {
  const int M = dgrad ? d->C : d->K, Cin = dgrad ? d->K : d->C;
  const int Ho = d->H / 2, Wo = d->W / 2;
  const int NT = tap_nt(M);
  const int small = (!dgrad && Cin <= 8) ? 1 : 0;
  const int Mpad = round_up(M, NT), Cpad = round_up(Cin, TT_BK);
  S2Params p{};
  p.tt = make_taps(d, dgrad);
  const int rblocks = small ? (p.tt.n + 3) / 4 : p.tt.n;
  float* wp = reinterpret_cast<float*>(align1k(reinterpret_cast<uintptr_t>(ws)));
  {
    const long long total = (long long)rblocks * Mpad * Cpad;
    long long blocks = (total + 255) / 256;
    if (blocks > 1184) blocks = 1184;
    tf32_s2_repack_kernel<<<(int)blocks, 256, 0, st>>>(w, wp, M, Cin, Mpad, Cpad, d->R, d->S, dgrad, small, p.tt);
    count_launch();
    SPC_CHECK_CUDA(cudaGetLastError());
  }
  if (small) { p.tt.cls_begin[1] = rblocks; }
  CUtensorMap tw, tx, ty;
  {
    const uint64_t dims[2] = {(uint64_t)Cpad, (uint64_t)rblocks * Mpad};
    const uint64_t strides[2] = {0, (uint64_t)Cpad * 4};
    const uint32_t box[2] = {TT_BK, (uint32_t)NT};
    int rc = make_tmap(&tw, wp, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  int rc = dgrad ? make_act_tmap4(&tx, x, d->N, Cin, Ho, Wo, TT_BK, S2_DXW, false)
                 : make_act_tmap4(&tx, x, d->N, Cin, d->H, d->W, small ? 8 : TT_BK, S2_XW, false);
  if (rc) return rc;
  // dgrad stores from registers: its kernel takes the map of dy in the place of the output's
  rc = dgrad ? make_act_tmap4(&ty, x, d->N, Cin, Ho, Wo, TT_BK, S2_DXW, false)
             : make_act_tmap4(&ty, y, d->N, M, Ho, Wo, NT < 64 ? NT : 64, 32, true);
  if (rc) return rc;
  p.M = M; p.N = d->N; p.bias = bias; p.dx = y;
  p.rows = Ho; p.cols = Wo;
  p.segs_row = (Wo + 31) / 32;
  p.kchunks = Cpad / TT_BK;
  p.mpad = Mpad;
  p.num_mg = Mpad / NT;
  const long long tiles = ((long long)d->N * Ho * p.segs_row + 3) / 4;
  SPC_REQUIRE(tiles * p.num_mg * 4 < (1ll << 31), "tf32 stride-2 tap conv: too many tiles");
  p.num_tiles = (int)(tiles * p.num_mg * (dgrad ? 4 : 1));
  if (dgrad) return launch_s2_gemm_nt<S2_DGRAD>(NT, tw, tx, ty, p, st);
  if (small) return launch_s2_gemm_nt<S2_FPROP_SMALL>(NT, tw, tx, ty, p, st);
  return launch_s2_gemm_nt<S2_FPROP>(NT, tw, tx, ty, p, st);
}

// ---- wgrad kernel: dW_(r,s)^T[128 ch x NT k] += X_(r,s)[128 ch x P_out] * dY[NT k x P_out]^T per work item -----------
struct S2WgParams {
  float* dw;             // [K][C][R][S] fp32
  int C, K, Ho, R, S, ph, pw;
  int segs_row;          // ceil(Wo / 32)
  int cblocks;           // ceil(C / 128)
  int num_kg;            // groups of NT outputs
  int splits;            // row-segment ranges per (tap, channel block, output group)
  int chunks_total;      // N * Ho * segs_row
  int stages;
  int split0, nsplit;    // this launch runs splits [split0, split0 + nsplit)
  size_t slice_stride;   // split sp adds into dw + (sp - split0) * slice_stride (common.cuh: WgradSlices)
};

template <int NT>
__global__ void __launch_bounds__(TT_THREADS, 1)
tf32_s2_wgrad_kernel(const __grid_constant__ CUtensorMap tmap_dy, const __grid_constant__ CUtensorMap tmap_x,
                     const S2WgParams p) {
  constexpr int B_BYTES = NT * 128;                  // [NT k][32 px], SWIZZLE_128B
  constexpr int STAGE = B_BYTES + S2_WG_XBOX;        // a multiple of 1 KB
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
#define S2W_DECODE(it)                                                                          \
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
        S2W_DECODE(it)
        const int dr = tap / p.S - p.ph;
        for (int ch = c_begin; ch < c_end; ++ch) {
          int n, y, x0;
          seg_coords(ch, p.segs_row, p.Ho, n, y, x0);
          mbar_wait(&empty[s], ph ^ 1);
          uint8_t* st = smem + s * STAGE;
          mbar_arrive_expect_tx(&full[s], STAGE);
          tma_load_4d(st, &tmap_dy, &full[s], x0, y, kg * NT, n);
          tma_load_4d(st + B_BYTES, &tmap_x, &full[s], 2 * x0 - 4, 2 * y + dr, cb * 128, n);
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
    // A fragment: rows g, g + 8 = channels cr, cr + 8 of the block; columns t4, t4 + 4 = output pixels of the k8 step.
    // Element (channel c, output pixel q) sits at word c * S2_XW + 2 q + 4, plus the tap's s - pw.
    const int cr = 64 * wg + 16 * w4 + g;
    const uint32_t xoff0 = (cr * S2_XW + 2 * t4 + 4) * 4;
    const uint32_t off[4] = {xoff0, xoff0 + 8 * S2_XW * 4, xoff0 + 8 * 4, xoff0 + (8 * S2_XW + 8) * 4};
    float acc[NT / 2];
    int s = 0, ph = 0;
    for (int it = it0 + blockIdx.x; it < it1; it += gridDim.x) {
      S2W_DECODE(it)
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
            asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(sx + off[r] + ks * 16 * 4));
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
#undef S2W_DECODE
}

template <int NT>
int launch_s2_wgrad(const CUtensorMap& tdy, const CUtensorMap& tx, S2WgParams p, cudaStream_t st, const WgradSlices* sl) {
  constexpr int STAGE = NT * 128 + S2_WG_XBOX;
  p.stages = (TT_SMEM_LIMIT - TT_SMEM_AUX) / STAGE;
  if (p.stages > 6) p.stages = 6;
  SPC_REQUIRE(p.stages >= 2, "tf32 stride-2 tap wgrad: smem budget");
  const int sms = sm_count();
  const long long groups = (long long)p.R * p.S * p.cblocks * p.num_kg;
  // at least two items per SM, at least 8 segments per item, at most TW_MAX_CHAIN segments per item
  long long splits = (2 * sms + groups - 1) / groups;
  if (splits > p.chunks_total / 8) splits = p.chunks_total / 8;
  const long long smin = (p.chunks_total + TW_MAX_CHAIN - 1) / TW_MAX_CHAIN;
  if (splits < smin) splits = smin;
  if (splits < 1) splits = 1;
  SPC_REQUIRE(groups * splits < (1ll << 31), "tf32 stride-2 tap wgrad: too many work items");
  p.splits = (int)splits;
  auto kern = tf32_s2_wgrad_kernel<NT>;
  const int rc = allow_dynamic_smem((const void*)kern, TT_SMEM_LIMIT);
  if (rc) return rc;
  // smin makes up to chunks_total / TW_MAX_CHAIN splits: the deterministic path may need several passes for them
  return run_slices(sl, p.splits, (size_t)p.K * p.C * p.R * p.S, p.dw, st, [&](int s0, int ns, float* dst, size_t stride) {
    S2WgParams q = p;
    q.split0 = s0; q.nsplit = ns; q.dw = dst; q.slice_stride = stride;
    const long long items = groups * ns;
    kern<<<(int)(items < sms ? items : sms), TT_THREADS, p.stages * STAGE + TT_SMEM_AUX, st>>>(tdy, tx, q);
    count_launch();
    SPC_CHECK_CUDA(cudaGetLastError());
    return SPC_OK;
  });
}
}  // namespace

// fp32, stride 2 x 2, "same" padding, R and S in {3, 5, 7}, even H, W % 8 == 0 (16-byte aligned rows of x and of y)
bool tf32_tap_s2_supported(const spc_conv_desc* d) {
  if (d->dtype != SPC_F32 || d->stride_h != 2 || d->stride_w != 2) return false;
  if (d->R < 3 || d->S < 3 || d->R % 2 == 0 || d->S % 2 == 0 || d->R > 7 || d->S > 7) return false;
  if (d->pad_h != (d->R - 1) / 2 || d->pad_w != (d->S - 1) / 2) return false;
  return d->H % 2 == 0 && d->W % 8 == 0;
}

// the repacked weights of fprop (op 0) / dgrad (op 1); wgrad needs none
size_t tf32_tap_s2_workspace_bytes(const spc_conv_desc* d, int op) {
  if (op == 2) return 0;
  return align1k(op == 0 ? s2_wp_bytes(d->R * d->S, d->K, d->C) : s2_wp_bytes(d->R * d->S, d->C, d->K)) + 1024;
}

int tf32_tap_s2_fwd(const spc_conv_desc* d, const void* x, const void* w, const void* bias, void* y, void* ws,
                    size_t ws_bytes, cudaStream_t st) {
  SPC_REQUIRE(ws && ws_bytes >= tf32_tap_s2_workspace_bytes(d, 0), "tf32 stride-2 tap conv: workspace too small");
  return run_s2_gemm(d, 0, reinterpret_cast<const float*>(w), reinterpret_cast<const float*>(x),
                     reinterpret_cast<const float*>(bias), reinterpret_cast<float*>(y), ws, st);
}

int tf32_tap_s2_dgrad(const spc_conv_desc* d, const void* dy, const void* w, void* dx, void* ws, size_t ws_bytes,
                      cudaStream_t st) {
  SPC_REQUIRE(ws && ws_bytes >= tf32_tap_s2_workspace_bytes(d, 1), "tf32 stride-2 tap conv: workspace too small");
  return run_s2_gemm(d, 1, reinterpret_cast<const float*>(w), reinterpret_cast<const float*>(dy), nullptr,
                     reinterpret_cast<float*>(dx), ws, st);
}

// dw[K][C][R][S] += the interior's share (zero padding), with atomics; api.cu adds the halo strips' share.  Needs no
// workspace.
int tf32_tap_s2_wgrad(const spc_conv_desc* d, const void* x, const void* dy, float* dw, void*, size_t, cudaStream_t st,
                      const WgradSlices* sl) {
  S2WgParams p{};
  const int Ho = d->H / 2, Wo = d->W / 2;
  p.dw = dw; p.C = d->C; p.K = d->K; p.Ho = Ho; p.R = d->R; p.S = d->S; p.ph = d->pad_h; p.pw = d->pad_w;
  p.segs_row = (Wo + 31) / 32;
  const long long chunks = (long long)d->N * Ho * p.segs_row;
  SPC_REQUIRE(chunks < (1ll << 31), "tf32 stride-2 tap wgrad: too many row segments");
  p.chunks_total = (int)chunks;
  const int NT = tap_nt(d->K);
  p.cblocks = (d->C + 127) / 128;
  p.num_kg = round_up(d->K, NT) / NT;
  CUtensorMap tdy, tx;
  int rc = make_act_tmap4(&tdy, dy, d->N, d->K, Ho, Wo, NT, 32, true);
  if (rc) return rc;
  rc = make_act_tmap4(&tx, x, d->N, d->C, d->H, d->W, 128, S2_XW, false);
  if (rc) return rc;
  switch (NT) {
    case 16: return launch_s2_wgrad<16>(tdy, tx, p, st, sl);
    case 32: return launch_s2_wgrad<32>(tdy, tx, p, st, sl);
    case 64: return launch_s2_wgrad<64>(tdy, tx, p, st, sl);
    case 128: return launch_s2_wgrad<128>(tdy, tx, p, st, sl);
    default: return launch_s2_wgrad<256>(tdy, tx, p, st, sl);
  }
}

}  // namespace spc
