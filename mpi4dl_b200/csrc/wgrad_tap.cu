// wgrad_tap.cu -- weight gradient of the multi-tap stride-1 convolutions (1x7 / 3x3 / 5x5) on wgmma, with the
// horizontally shifted operand formed in shared memory -- the wgrad counterpart of conv_tap.cu; replaces round 1's
// pw_wgrad_kernel over S column-shifted HBM copies of the input for these shapes.
//
//     dW[k][c][r][s] = sum_{n,h,w} dY[n][k][h][w] * X[n][c][h + r - ph][w + s - pw]          (pixels = reduction dim)
//
// Both operands are K-major straight from NCHW (64 contiguous pixels of a row = one 128-byte swizzle row per channel).
// P operand (M side, accumulator rows) = the tensor with MORE channels, unshifted, loaded by TMA as it is;
// Q operand (N side, accumulator columns) = the other tensor: every row is loaded ONCE with 8 pixels of slack (aligned
// box), and the shifter warps write its S column-shifted tiles [Qch][64 px] next to each other in shared memory; one
// wgmma (N = QC = Qch rounded up to 16) per tap.  mode A: P = dY, Q = X;  mode B: P = X, Q = dY, which is mode A
// with both tap indices mirrored (dW[k][c][R-1-r][S-1-s]).
// Line buffer: a CTA walks down a 64-pixel-wide column strip; step j = P row ha + j meets Q rows j .. j + R' - 1 of a
// ring of shifted row tile-sets, so every Q row is loaded and shifted once and used by R' steps.  Accumulators of the
// NT = 256 / QC taps of a pass live in the registers of two consumer warpgroups (<= 128 fp32 per thread; more taps ->
// more passes over the strip); fp32 atomics at the end.  A pass with fewer than NT taps skips the wgmma of its spare
// accumulators (a warp-uniform branch; ptxas does not serialise the wgmma for it) and does not flush them.
// All passes of a filter run in one launch: the pass is the fastest-varying part of the work item, so the passes of
// one (image, strip, row range) run on neighbouring CTAs at the same time and read the same P and Q rows, which come
// from HBM once and from L2 for the other passes.
//
// Warp roles (640 threads): 0 = TMA producer, 4..11 = two consumer warpgroups (wgmma + flush), 12..19 = shifter;
// setmaxnreg moves the registers of the producer warpgroup and the shifters to the consumers.
#include <stdlib.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace spc {

using namespace tc;

namespace {

constexpr int WT_THREADS = 640;
constexpr int SHIFT_THREADS = 256;
constexpr int RAW_ROW = 160;       // raw Q row: [Qch][80 px], dense rows of 160 bytes
constexpr int MAXP = 8;            // P row stages (ring depths are chosen by the launcher: bytes in flight)
constexpr int MAXRAW = 8;          // raw Q row slots
constexpr int MAXQ = 16;           // Q row ring slots
constexpr int MAXPASS = 8;         // tap rectangles of one filter (<= 7: R or S <= 7 and >= 2 taps per pass)

struct WtParams {
  float* dw;
  int K, C, R, S;              // dW is [K][C][R][S]
  int H, W, N;
  int modeB;                   // 0: P = dY (lanes = k), Q = X;  1: P = X (lanes = c), Q = dY, taps mirrored
  int Pch, Qch, Qc16;          // channels of the P / Q operand, Q padded to 16
  int p_bytes;                 // P tile bytes: round_up(Pch, 8) * 128
  int p_blk;                   // P stage stride (1024-aligned)
  int qt_bytes;                // one shifted Q tile: Qc16 * 128
  int ph, pw;
  // tap rectangles ("passes"): filter rows [r0, r0 + nr), columns [s0, s0 + ns) = rect[pass][0..3]
  int npass;
  int rect[MAXPASS][4];
  int nr_max, ns_max;          // the largest pass rectangle: the shared-memory rings are sized for it
  int rq;                      // Q row ring slots (>= nr_max + 1)
  int psn, rawn;               // P row stages, raw Q row slots
  int nbw;                     // 64-pixel blocks per strip row (strip width = 64 * nbw): rows of few channels are
                               // small, and the TMA loads are latency-bound -> wider strips keep more bytes in flight
  int raw_bytes;               // raw Q row bytes: Qc16 * 160
  int strips, row_splits, rows_per_split;
  // this launch runs slices (image, strip, row range) [split0, split0 + nsplit), all passes of each; slice s adds into
  // dw + (s - split0) * slice_stride (common.cuh: WgradSlices)
  int split0, nsplit;
  size_t slice_stride;
};

struct Ring {
  int i = 0;
  __device__ __forceinline__ int slot(int n) const { return i % n; }
  __device__ __forceinline__ int phase(int n) const { return (i / n) & 1; }
};

template <int D>
__device__ __forceinline__ uint4 shift_window(const uint32_t (&w)[8]) {
  static_assert(D >= -4 && D <= 4, "shift range");
  constexpr int e0 = 4 + D;
  constexpr int k = e0 >> 1;
  uint4 o;
  if (e0 & 1) {
    o.x = __funnelshift_r(w[k], w[k + 1], 16);
    o.y = __funnelshift_r(w[k + 1], w[k + 2], 16);
    o.z = __funnelshift_r(w[k + 2], w[k + 3], 16);
    o.w = __funnelshift_r(w[k + 3], w[k + 4], 16);
  } else {
    o.x = w[k]; o.y = w[k + 1]; o.z = w[k + 2]; o.w = w[k + 3];
  }
  return o;
}

// write the shifted tiles of filter columns [s0, s0 + ns) of one raw Q row for channels cb and cb + 32; the tile of
// column s sits at (s - s0) * qt_bytes
template <int S, int SI>
struct ShiftCols {
  static __device__ __forceinline__ void run(const uint32_t (&win)[2][8], int cb, int qc16, int q, uint8_t* dst, int qt_bytes,
                                             int s0, int ns) {
    if constexpr (SI < S) {
      if (SI >= s0 && SI < s0 + ns) {
        uint8_t* t = dst + (SI - s0) * qt_bytes;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int c = cb + 32 * i;
          if (c < qc16) *reinterpret_cast<uint4*>(t + c * 128 + ((q ^ (c & 7)) << 4)) = shift_window<SI - S / 2>(win[i]);
        }
      }
      ShiftCols<S, SI + 1>::run(win, cb, qc16, q, dst, qt_bytes, s0, ns);
    }
  }
};

template <int S, int QC>
__global__ void __launch_bounds__(WT_THREADS, 1)
wgrad_tap_kernel(const __grid_constant__ CUtensorMap tmap_p, const __grid_constant__ CUtensorMap tmap_q,
                 const __grid_constant__ WtParams p) {
  constexpr bool SHIFT = S > 1;
  constexpr int NT = 256 / QC;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int qblk_bytes = p.ns_max * p.qt_bytes;             // the shifted tiles of one 64-pixel block of a Q row
  const int qrow_bytes = p.nbw * qblk_bytes;                // ... of a whole strip row
  const int prow_bytes = p.nbw * p.p_blk;
  const int rawrow_bytes = p.nbw * p.raw_bytes;
  uint8_t* p_base = smem;
  uint8_t* qt_base = p_base + p.psn * prow_bytes;
  uint8_t* raw_base = qt_base + p.rq * qrow_bytes;
  uint8_t* bar_base = raw_base + (SHIFT ? p.rawn * rawrow_bytes : 0);
  uint64_t* p_full = reinterpret_cast<uint64_t*>(bar_base);
  uint64_t* p_empty = p_full + MAXP;
  uint64_t* qt_full = p_empty + MAXP;
  uint64_t* qt_empty = qt_full + MAXQ;
  uint64_t* raw_full = qt_empty + MAXQ;
  uint64_t* raw_empty = raw_full + MAXRAW;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    // p_empty / qt_empty: one arrive per consumer warpgroup
    for (int i = 0; i < MAXP; ++i) { mbar_init(&p_full[i], 1); mbar_init(&p_empty[i], 2); }
    for (int i = 0; i < MAXQ; ++i) { mbar_init(&qt_full[i], SHIFT ? SHIFT_THREADS : 1); mbar_init(&qt_empty[i], 2); }
    for (int i = 0; i < MAXRAW; ++i) { mbar_init(&raw_full[i], 1); mbar_init(&raw_empty[i], SHIFT_THREADS); }
    fence_barrier_init();
  }
  __syncthreads();
  const int it0 = p.split0 * p.npass, it1 = it0 + p.nsplit * p.npass;

  // item -> (image n, column strip, row range [ha, hb), tap rectangle = pass)
#define WT_ITEM(it)                                                               \
  const int pass_ = (it) % p.npass, rest_ = (it) / p.npass;                       \
  const int sp_ = rest_ % p.row_splits;                                           \
  const int strip_ = (rest_ / p.row_splits) % p.strips;                           \
  const int n_ = rest_ / (p.row_splits * p.strips);                               \
  const int r0 = p.rect[pass_][0], nr = p.rect[pass_][1];                         \
  const int s0 = p.rect[pass_][2], ns = p.rect[pass_][3];                         \
  const int w0 = strip_ * 64 * p.nbw;                                             \
  const int ha = sp_ * p.rows_per_split, hb = min(p.H, ha + p.rows_per_split);    \
  const int rows = hb - ha;                                                       \
  const int q_first = ha + r0 - p.ph;   /* image row of Q ring row 0 */           \
  const int q_rows = rows + nr - 1;

  // 640 x 96 registers at launch; the consumers' <= 128 accumulators need more: 24 + 2 x 56 + 2 x 168 <= 480.  Each
  // role sets its count at the top of its own branch, so that ptxas allocates that branch at that count.
  if (warp < 4) {
    setmaxnreg_dec<24>();
    // ================= producer =================
    if (warp == 0 && lane == 0) {
      tma_prefetch_desc(&tmap_p);
      tma_prefetch_desc(&tmap_q);
      Ring qr, pr, rr;     // Q ring rows / P rows / raw rows issued so far (global counters across items)
      for (int it = it0 + blockIdx.x; it < it1; it += gridDim.x) {
        WT_ITEM(it)
        (void)s0; (void)ns;
        if (rows <= 0) continue;
        for (int i = 0; i < q_rows; ++i) {
          if (SHIFT) {
            const int s = rr.slot(p.rawn);
            mbar_wait(&raw_empty[s], rr.phase(p.rawn) ^ 1);
            mbar_arrive_expect_tx(&raw_full[s], rawrow_bytes);
            for (int b = 0; b < p.nbw; ++b)
              tma_load_4d(raw_base + s * rawrow_bytes + b * p.raw_bytes, &tmap_q, &raw_full[s], w0 + 64 * b - 8, q_first + i, 0, n_);
            ++rr.i;
          } else {
            const int s = qr.slot(p.rq);
            mbar_wait(&qt_empty[s], qr.phase(p.rq) ^ 1);
            mbar_arrive_expect_tx(&qt_full[s], p.nbw * p.qt_bytes);
            for (int b = 0; b < p.nbw; ++b)
              tma_load_4d(qt_base + s * qrow_bytes + b * qblk_bytes, &tmap_q, &qt_full[s], w0 + 64 * b, q_first + i, 0, n_);
            ++qr.i;
          }
          if (i >= nr - 1) {     // P row of step j = i - (nr - 1)
            const int j = i - (nr - 1);
            const int s = pr.slot(p.psn);
            mbar_wait(&p_empty[s], pr.phase(p.psn) ^ 1);
            mbar_arrive_expect_tx(&p_full[s], p.nbw * p.p_bytes);
            for (int b = 0; b < p.nbw; ++b)
              tma_load_4d(p_base + s * prow_bytes + b * p.p_blk, &tmap_p, &p_full[s], w0 + 64 * b, ha + j, 0, n_);
            ++pr.i;
          }
        }
      }
    }
  } else if (warp >= 12) {
    setmaxnreg_dec<56>();
    // ================= shifter: raw Q row -> S' shifted K-major tiles =================
    if (SHIFT) {
      const int tid = threadIdx.x - 12 * 32;
      const int q = tid & 7, c0 = tid >> 3;
      Ring qr, rr;
      for (int it = it0 + blockIdx.x; it < it1; it += gridDim.x) {
        WT_ITEM(it)
        (void)w0; (void)n_; (void)q_first;
        if (rows <= 0) continue;
        for (int i = 0; i < q_rows; ++i) {
          const int rs = rr.slot(p.rawn);
          mbar_wait(&raw_full[rs], rr.phase(p.rawn));
          const int qs = qr.slot(p.rq);
          for (int b = 0; b < p.nbw; ++b) {
            const uint8_t* raw = raw_base + rs * rawrow_bytes + b * p.raw_bytes;
            // channels c0 + 32 k, k < 4, in two halves: 16 registers of windows at a time (the shifter has 56)
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
              const int cb = c0 + 64 * hf;
              uint32_t win[2][8];
#pragma unroll
              for (int k = 0; k < 2; ++k) {
                const int c = cb + 32 * k;
                if (c < p.Qc16) {   // warp-uniform (4 consecutive channels per warp, Qc16 multiple of 16)
                  const uint8_t* row = raw + c * RAW_ROW;
                  const uint4 own = *reinterpret_cast<const uint4*>(row + 16 * (q + 1));
                  uint32_t lz = __shfl_up_sync(0xffffffffu, own.z, 1), lw = __shfl_up_sync(0xffffffffu, own.w, 1);
                  uint32_t rx = __shfl_down_sync(0xffffffffu, own.x, 1), ry = __shfl_down_sync(0xffffffffu, own.y, 1);
                  if (q == 0) { const uint2 h = *reinterpret_cast<const uint2*>(row + 8); lz = h.x; lw = h.y; }
                  if (q == 7) { const uint2 h = *reinterpret_cast<const uint2*>(row + 16 * 9); rx = h.x; ry = h.y; }
                  win[k][0] = lz; win[k][1] = lw; win[k][2] = own.x; win[k][3] = own.y;
                  win[k][4] = own.z; win[k][5] = own.w; win[k][6] = rx; win[k][7] = ry;
                }
              }
              if (b == p.nbw - 1 && hf == 1) mbar_arrive(&raw_empty[rs]);       // the whole raw row has been read
              if (b == 0 && hf == 0) mbar_wait(&qt_empty[qs], qr.phase(p.rq) ^ 1);
              ShiftCols<S, 0>::run(win, cb, p.Qc16, q, qt_base + qs * qrow_bytes + b * qblk_bytes, p.qt_bytes, s0, ns);
            }
          }
          ++rr.i;
          fence_proxy_async();
          mbar_arrive(&qt_full[qs]);
          ++qr.i;
        }
      }
    }
  } else {
    setmaxnreg_inc<168>();
    // ================= consumers: wgmma over (row step, 64-pixel block, tap), then fp32 atomics on dW =================
    const int wg = (threadIdx.x >> 7) - 1;
    const int w4 = (threadIdx.x >> 5) & 3;
    const bool wg_lead = (threadIdx.x & 127) == 0;
    float acc[NT][QC / 2];
    Ring qr, pr;          // qr.i = ring index of Q row 0 of the current item
    for (int it = it0 + blockIdx.x; it < it1; it += gridDim.x) {
      WT_ITEM(it)
      (void)w0; (void)n_; (void)q_first;
      if (rows <= 0) continue;
      const int ntaps = nr * ns;
      int rel_p = -1, rel_q = -1;             // slots read by the last committed wgmma group
      for (int j = 0; j < rows; ++j) {
        // Q rows j .. j + nr - 1 must have landed: all of them at the first step, then one new row per step
        for (int i = (j == 0 ? 0 : nr - 1); i < nr; ++i) {
          const int g = qr.i + j + i;
          mbar_wait(&qt_full[g % p.rq], (g / p.rq) & 1);
        }
        const int ps = pr.slot(p.psn);
        mbar_wait(&p_full[ps], pr.phase(p.psn));
        wgmma_fence();
        for (int b = 0; b < p.nbw; ++b) {
          const uint32_t sa = smem_u32(p_base + ps * prow_bytes + b * p.p_blk) + wg * 8192;
#pragma unroll
          for (int a = 0; a < NT; ++a) {
            if (a >= ntaps) break;              // warp-uniform: a pass with fewer taps skips its spare accumulators
            const int r = a / ns, si = a - r * ns;
            const int g = qr.i + j + r;
            const uint32_t sq = smem_u32(qt_base + (g % p.rq) * qrow_bytes + b * qblk_bytes + si * p.qt_bytes);
#pragma unroll
            for (int ks = 0; ks < 4; ++ks)   // 64 pixels = 4 k-steps of 16; +32 bytes inside the 128-byte swizzle row
              Wgmma<QC, 0>::mma(acc[a], gmma_desc(sa + ks * 32, 16, 1024), gmma_desc(sq + ks * 32, 16, 1024),
                                (j | b | ks) ? 1u : 0u);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (wg_lead) {
          if (rel_p >= 0) mbar_arrive(&p_empty[rel_p]);
          if (rel_q >= 0) mbar_arrive(&qt_empty[rel_q]);
        }
        rel_p = ps;
        rel_q = (qr.i + j) % p.rq;            // Q row j: step j was its last use (r = 0)
        ++pr.i;
      }
      wgmma_wait<0>();
#pragma unroll
      for (int a = 0; a < NT; ++a) reg_fence(acc[a]);
      if (wg_lead) {
        mbar_arrive(&p_empty[rel_p]);
        mbar_arrive(&qt_empty[rel_q]);
        // rows j = rows .. rows + nr - 2 of the ring were loaded for the last steps and are dead now: release them
        for (int i = rows; i < q_rows; ++i) mbar_arrive(&qt_empty[(qr.i + i) % p.rq]);
      }
      qr.i += q_rows;
      float* dw = p.dw + (size_t)(rest_ - p.split0) * p.slice_stride;   // the passes of one slice add disjoint taps
#pragma unroll
      for (int a = 0; a < NT; ++a) {
        if (a < ntaps) {
          int r = r0 + a / ns, s = s0 + a % ns;
          if (p.modeB) { r = p.R - 1 - r; s = p.S - 1 - s; }
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int pl = 64 * wg + 16 * w4 + (lane >> 2) + 8 * h;   // P channel = accumulator row
            if (pl < p.Pch) {
#pragma unroll
              for (int q = 0; q < QC / 8; ++q) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const int qc = 8 * q + 2 * (lane & 3) + e;
                  if (qc < p.Qch) {
                    const int k = p.modeB ? qc : pl, c = p.modeB ? pl : qc;
                    atomicAdd(&dw[(((size_t)k * p.C + c) * p.R + r) * p.S + s], acc[a][4 * q + 2 * h + e]);
                  }
                }
              }
            }
          }
        }
      }
    }
  }
#undef WT_ITEM
}

constexpr int WT_SMEM_LIMIT = 222 * 1024;   // of H100's 227 KB per block
constexpr int WT_SMEM_AUX = 1024 + 1024;

template <int S, int QC>
int launch_wt(const CUtensorMap& tp, const CUtensorMap& tq, const WtParams& p, int smem, cudaStream_t st,
              const WgradSlices* sl) {
  auto kern = wgrad_tap_kernel<S, QC>;
  const int rc = allow_dynamic_smem((const void*)kern, WT_SMEM_LIMIT);
  if (rc) return rc;
  const int sms = sm_count();
  const int slices = p.N * p.strips * p.row_splits;
  return run_slices(sl, slices, (size_t)p.K * p.C * p.R * p.S, p.dw, st, [&](int s0, int ns, float* dst, size_t stride) {
    WtParams q = p;
    q.split0 = s0; q.nsplit = ns; q.dw = dst; q.slice_stride = stride;
    const int items = ns * p.npass;
    kern<<<items < sms ? items : sms, WT_THREADS, smem, st>>>(tp, tq, q);
    count_launch();
    SPC_CHECK_CUDA(cudaGetLastError());
    return SPC_OK;
  });
}

// tap rectangles ("passes") of an R x S filter at most maxt taps each; returns the count (0: no plan)
int plan_passes(int R, int S, int maxt, int (*rect)[4]) {
  if (maxt < 1) return 0;
  int n = 0;
  if (R * S <= maxt) { rect[n][0] = 0; rect[n][1] = R; rect[n][2] = 0; rect[n][3] = S; return 1; }
  if (S <= maxt) {                      // whole filter rows per pass
    const int nr = maxt / S;
    for (int r0 = 0; r0 < R; r0 += nr, ++n) { rect[n][0] = r0; rect[n][1] = min(nr, R - r0); rect[n][2] = 0; rect[n][3] = S; }
    return n;
  }
  if (R == 1) {                         // split the columns of a 1 x S filter evenly
    const int np = (S + maxt - 1) / maxt, per = (S + np - 1) / np;
    for (int s0 = 0; s0 < S; s0 += per, ++n) { rect[n][0] = 0; rect[n][1] = 1; rect[n][2] = s0; rect[n][3] = min(per, S - s0); }
    return n;
  }
  return 0;
}

}  // namespace

bool wgrad_tap_supported(int K, int C, int R, int S, int H, int W, int stride) {
  if (stride != 1 || R * S == 1 || (W % 64) != 0 || H < 1) return false;
  // S == 1 (7x1): no horizontal shift is needed and round 1's pw_wgrad_kernel (row-shifted TMA boxes, no copies) is
  // 1.4x faster than the line buffer there (profiles/r2_tap_probe_v2d.txt) -- it keeps those shapes
  if (!(S == 3 || S == 5 || S == 7) || (R & 1) == 0 || R > 7) return false;
  if (K > 128 || C > 128) return false;
  // the shapes this kernel serves are those with a plan of 128 / QC taps per pass, the set it was measured on
  // against the shifted-copy path; it runs them in passes of up to 256 / QC taps
  const int Qc16 = round_up(K >= C ? C : K, 16);
  int rect[MAXPASS][4];
  return plan_passes(R, S, 128 / Qc16, rect) > 0;
}

// dw += wgrad(x [N][C][H][W], dy [N][K][H][W]) over the zero-padded tile (pad = (R-1)/2, (S-1)/2), bf16 inputs
int run_wgrad_tap(const __nv_bfloat16* x, const __nv_bfloat16* dy, float* dw, int K, int C, int N, int H, int W, int R, int S,
                  cudaStream_t st, const WgradSlices* sl) {
  WtParams p{};
  p.dw = dw; p.K = K; p.C = C; p.R = R; p.S = S; p.H = H; p.W = W; p.N = N;
  p.ph = (R - 1) / 2; p.pw = (S - 1) / 2;
  p.modeB = K >= C ? 0 : 1;
  p.Pch = p.modeB ? C : K; p.Qch = p.modeB ? K : C;
  p.Qc16 = round_up(p.Qch, 16);
  p.p_bytes = round_up(p.Pch, 8) * 128;
  p.p_blk = round_up(p.p_bytes, 1024);
  p.qt_bytes = p.Qc16 * 128;
  p.raw_bytes = p.Qc16 * RAW_ROW;
  const __nv_bfloat16* P = p.modeB ? x : dy;
  const __nv_bfloat16* Q = p.modeB ? dy : x;
  const int npass = plan_passes(R, S, 256 / p.Qc16, p.rect);   // NT = 256 / QC taps per pass
  SPC_REQUIRE(npass > 0 && npass <= MAXPASS, "wgrad_tap: %dx%d filter with %d Q channels does not fit the accumulators",
              R, S, p.Qch);
  p.npass = npass;
  for (int pi = 0; pi < npass; ++pi) {
    p.nr_max = max(p.nr_max, p.rect[pi][1]);
    p.ns_max = max(p.ns_max, p.rect[pi][3]);
  }
  CUtensorMap tp, tq;
  {
    const uint64_t dims[4] = {(uint64_t)W, (uint64_t)H, (uint64_t)p.Pch, (uint64_t)N};
    const uint64_t strides[4] = {0, (uint64_t)W * 2, (uint64_t)H * W * 2, (uint64_t)H * W * p.Pch * 2};
    const uint32_t box[4] = {64, 1, (uint32_t)round_up(p.Pch, 8), 1};
    int rc = make_tmap(&tp, P, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  {
    const uint64_t dims[4] = {(uint64_t)W, (uint64_t)H, (uint64_t)p.Qch, (uint64_t)N};
    const uint64_t strides[4] = {0, (uint64_t)W * 2, (uint64_t)H * W * 2, (uint64_t)H * W * p.Qch * 2};
    const uint32_t box[4] = {(uint32_t)(S > 1 ? 80 : 64), 1, (uint32_t)p.Qc16, 1};
    int rc = make_tmap(&tq, Q, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, dims, strides, box,
                       S > 1 ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  const int sms = sm_count();
  // few channels -> small rows -> wider strips (more bytes per ring slot)
  p.nbw = 1;
  {
    const int rowb = round_up(p.Pch, 8) * 128 + p.Qc16 * 128;
    while (p.nbw < 4 && rowb * p.nbw < 12 * 1024 && W % (128 * p.nbw) == 0) p.nbw *= 2;
  }
  p.strips = W / (64 * p.nbw);
  // mode B mirrors the tap indices: the rectangles are planned in the kernel's (mirrored) index space either way
  const int qrow_bytes = p.nbw * p.ns_max * p.qt_bytes, prow = p.nbw * p.p_blk, rawrow = S > 1 ? p.nbw * p.raw_bytes : 0;
  // ring depths.  Rows of many channels (>= ~12 KB per strip row) keep enough bytes in flight with 3 P stages,
  // 2 raw rows and nr + 3 shifted rows (measured: deeper rings cost 10 % there); small rows are latency-bound
  // on the ~2 us L2 round trip of their TMA loads, so they take whatever depth fits.
  const bool small_rows = prow + p.nbw * p.qt_bytes < 12 * 1024;
  p.psn = 3; p.rawn = S > 1 ? 2 : 0; p.rq = p.nr_max + 1;
  int rem = WT_SMEM_LIMIT - WT_SMEM_AUX - p.psn * prow - p.rawn * rawrow - p.rq * qrow_bytes;
  SPC_REQUIRE(rem >= 0, "wgrad_tap: shared memory too small (rows %d, %d bytes per row)", p.nr_max, qrow_bytes);
  if (small_rows) {
    for (bool grew = true; grew;) {
      grew = false;
      if (S > 1 && p.rawn < MAXRAW && rem >= rawrow) { ++p.rawn; rem -= rawrow; grew = true; }
      if (p.psn < MAXP && rem >= prow) { ++p.psn; rem -= prow; grew = true; }
      if (p.rq < MAXQ && p.rq < p.nr_max + 8 && rem >= qrow_bytes) { ++p.rq; rem -= qrow_bytes; grew = true; }
    }
  } else {
    while (p.rq < p.nr_max + 3 && p.rq < MAXQ && rem >= qrow_bytes) { ++p.rq; rem -= qrow_bytes; }
  }
  // row splits: fill the persistent grid with whole waves of (image, strip, row range, pass) items
  const int base_items = N * p.strips * npass;
  int best = 1;
  double best_eff = 0.0;
  for (int sp = 1; sp <= 64 && H / sp >= 8 * p.nr_max; ++sp) {
    const int items = base_items * sp, waves = (items + sms - 1) / sms;
    if (waves > 3) break;
    const double eff = (double)items / ((double)waves * sms) *
                       (1.0 - (double)(p.nr_max - 1) * sp / (H + (p.nr_max - 1) * sp));
    if (eff > best_eff + 1e-9) { best_eff = eff; best = sp; }
  }
  p.row_splits = best;
  p.rows_per_split = (H + best - 1) / best;
  const int smem = p.psn * prow + p.rq * qrow_bytes + p.rawn * rawrow + WT_SMEM_AUX;
#define WT_CASE(s, qc) if (S == s && p.Qc16 == qc) return launch_wt<s, qc>(tp, tq, p, smem, st, sl);
#define WT_CASES(s) WT_CASE(s, 16) WT_CASE(s, 32) WT_CASE(s, 48) WT_CASE(s, 64) WT_CASE(s, 80) WT_CASE(s, 96) \
                    WT_CASE(s, 112) WT_CASE(s, 128)
  WT_CASES(3) WT_CASES(5) WT_CASES(7)
#undef WT_CASES
#undef WT_CASE
  set_error("wgrad_tap: unsupported filter width %d / %d Q channels", S, p.Qc16);
  return SPC_EUNSUPPORTED;
}

}  // namespace spc
