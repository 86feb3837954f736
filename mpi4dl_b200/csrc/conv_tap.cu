// conv_tap.cu -- wgmma implicit-GEMM kernel for the multi-tap ("same", stride 1) convolutions of the
// spatial stages: 1x7 / 7x1 (AmoebaNet-D cells), 3x3 (ResNet), fprop and -- with the rotated,
// transposed filter -- dgrad.  Replaces round 1's approach (S column-shifted COPIES of the input in HBM
// because TMA tile loads need 16-byte aligned inner coordinates, then one TMA load per tap: 8x the
// algorithmic HBM bytes for 1x7 and 8.5x L2->SM amplification for 7x1).  Here:
//
//   * one output tile = NB rows x 64 pixels of all (<= 128) output channels; per 64-channel chunk the
//     producer loads the NB + R - 1 input ROW BLOCKS the tile needs ONCE (16-byte aligned boxes, 8
//     pixels of slack on both sides, out-of-image = zero fill = the zero padding);
//   * vertical taps (r) are just different row blocks of that buffer (UMMA descriptor start address);
//   * horizontal taps (s) are formed IN SHARED MEMORY by four "shifter" warps: each 16-byte chunk of the
//     operand tile of tap (r, s) is a funnel shift of the aligned 24-pixel window around it, written in
//     the swizzled MN-major layout wgmma reads.  Nothing shifted ever exists in HBM or L2;
//   * weights stay resident in shared memory when they fit, else stream through a small ring;
//   * accumulators (128 pixels x 128 channels) live in the registers of two consumer warpgroups, which issue the
//     wgmma and write each tile row through a swizzled staging block and a TMA store.
//
// Warp roles (640 threads): 0 = TMA producer (activation row blocks and weight blocks, interleaved), 4..11 = two
// consumer warpgroups, 12..19 = shifter; setmaxnreg moves the registers of the producer warpgroup and the shifters to
// the consumers.  All hand-offs are mbarriers; persistent CTAs, one per SM.
#include "common.cuh"
#include "tc_common.cuh"

namespace spc {

using namespace tc;

namespace {

constexpr int TAP_THREADS = 640;
constexpr int BLK = 8192;          // one operand block: [64 ch][64 px] bf16, 128-byte rows, SWIZZLE_128B
constexpr int RAW_SHIFT_ROW = 160;  // raw row block of the shift path: [cbox ch][80 px], dense rows of 160 B
constexpr int MAXRING = 8;
constexpr int STAGE_BYTES = 128 * 128;   // epilogue staging buffer: one [128 ch][64 px] block

struct TapParams {
  int M, Cin, H, W, N;
  int R, ph;                 // filter rows, top padding (S / pw are template parameters)
  int Mpad;                  // rows per tap in the repacked weights (multiple of 128)
  int mrows;                 // rows per A block in smem (round_up(M, 8))
  int a_blk;                 // bytes per A block (mrows * 128 rounded up to 1024)
  int kchunks;
  int cbox;                  // channels per raw box: 64, or round_up(Cin, 16) when Cin < 64
  int raw_blk;               // bytes of one raw row block: cbox * (160 shift path | 128 direct path)
  int tiles_w, tiles_h, num_tiles;
  int a_resident, ast, ops;  // weights resident?; weight ring depth; operand ring depth
  int rawb;                  // raw (activation row block) buffers in the ring: 2..MAXRING, sized by bytes in flight
  int opblk;                 // bytes of one 64-pixel block of an operand tile: cbox * 128
  int group;                 // 1: an operand-ring slot holds the S tiles of one filter ROW (one hand-shake per row), 0: one tap
  int rows_raw;              // NB + R - 1
  const __nv_bfloat16* bias;
  __nv_bfloat16* y;
};

struct RingState {
  int s = 0, ph = 0;
  __device__ __forceinline__ void next(int n) { if (++s == n) { s = 0; ph ^= 1; } }
};

// 8 output pixels = the 16-pixel window w[0..7] (pixels -4 .. +11 around the chunk) shifted by D pixels, |D| <= 4
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

constexpr int SHIFT_THREADS = 256;   // 8 shifter warps; thread -> (16-byte chunk q = tid & 7, channel c0 = tid >> 3 (+32))

// The shifter's work for ONE filter row r of one (tile, chunk): every thread first loads the pixel windows of its
// <= 2*NB items (block j, channel c, chunk q) into registers -- one aligned 16-byte load each, the 4 pixels on
// either side come from the neighbour lanes by shuffle (the first / last chunk of a row read the 8-pixel slack
// of the raw block instead) -- and then, for every filter column SI (compile-time shift SI - S/2), waits for a free
// operand-ring slot, writes its items in the swizzled MN-major layout and publishes the tile.  Shared-memory reads:
// once per filter ROW instead of three times per TAP.
template <int NB, int S, int SI>
struct ShiftRow {
  static __device__ __forceinline__ void stores(const uint32_t (&win)[2 * NB][8], int cv, int tid, uint8_t* op_base, int opblk,
                                                int group, uint64_t* op_full, uint64_t* op_empty, RingState& ro, int ops) {
    if constexpr (SI < S) {
      const int q = tid & 7, c0 = tid >> 3;
      const int tile_bytes = NB * opblk;
      if (!group || SI == 0) mbar_wait(&op_empty[ro.s], ro.ph ^ 1);
      uint8_t* opb = op_base + ro.s * (group ? S : 1) * tile_bytes + (group ? SI * tile_bytes : 0);
#pragma unroll
      for (int i = 0; i < 2 * NB; ++i) {
        const int j = i >> 1, c = c0 + 32 * (i & 1);
        if (c < cv)
          *reinterpret_cast<uint4*>(opb + j * opblk + c * 128 + ((q ^ (c & 7)) << 4)) = shift_window<SI - S / 2>(win[i]);
      }
      if (!group || SI == S - 1) {
        fence_proxy_async();            // generic-proxy writes -> visible to the tensor core (async proxy)
        mbar_arrive(&op_full[ro.s]);
        ro.next(ops);
      }
      ShiftRow<NB, S, SI + 1>::stores(win, cv, tid, op_base, opblk, group, op_full, op_empty, ro, ops);
    }
  }
  static __device__ __forceinline__ void run(const uint8_t* rawr, int raw_blk, int cv, int tid, uint8_t* op_base, int opblk,
                                             int group, uint64_t* op_full, uint64_t* op_empty, RingState& ro, int ops) {
    static_assert(S / 2 <= 4, "filter width <= 9");
    const int q = tid & 7, c0 = tid >> 3;
    uint32_t win[2 * NB][8];
#pragma unroll
    for (int i = 0; i < 2 * NB; ++i) {
      const int j = i >> 1, c = c0 + 32 * (i & 1);
      if (c < cv) {   // warp-uniform: a warp holds 4 consecutive channels and cv is a multiple of 16
        const uint8_t* row = rawr + j * raw_blk + c * RAW_SHIFT_ROW;        // pixels w0-8 .. w0+71, 160 bytes
        const uint4 own = *reinterpret_cast<const uint4*>(row + 16 * (q + 1));
        uint32_t lz = __shfl_up_sync(0xffffffffu, own.z, 1), lw = __shfl_up_sync(0xffffffffu, own.w, 1);
        uint32_t rx = __shfl_down_sync(0xffffffffu, own.x, 1), ry = __shfl_down_sync(0xffffffffu, own.y, 1);
        if (q == 0) { const uint2 h = *reinterpret_cast<const uint2*>(row + 8); lz = h.x; lw = h.y; }
        if (q == 7) { const uint2 h = *reinterpret_cast<const uint2*>(row + 16 * 9); rx = h.x; ry = h.y; }
        win[i][0] = lz; win[i][1] = lw; win[i][2] = own.x; win[i][3] = own.y;
        win[i][4] = own.z; win[i][5] = own.w; win[i][6] = rx; win[i][7] = ry;
      }
    }
    stores(win, cv, tid, op_base, opblk, group, op_full, op_empty, ro, ops);
  }
};

// Warp roles (640 threads): warp 0 = TMA producer (warps 1-3 idle), warpgroups 1-2 = wgmma consumers + epilogue (rows
// [64 g, 64 g + 64) of the output channels each), warps 12-19 = shifter.  KS = 16-channel k-steps per chunk (cbox / 16):
// a compile-time count, so that no wgmma sits under a data-dependent branch (ptxas would serialise all of them).
template <int NB, int S, int KS>
__global__ void __launch_bounds__(TAP_THREADS, 1)
conv_tap_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x,
                const __grid_constant__ CUtensorMap tmap_y, const TapParams p) {
  constexpr bool SHIFT = S > 1;
  constexpr int NPIX = NB * 64;
  const int RAW_BLK = p.raw_blk;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int taps = p.R * S;
  const int a_blocks = p.a_resident ? taps * p.kchunks : p.ast;
  uint8_t* a_base = smem;
  uint8_t* raw_base = a_base + a_blocks * p.a_blk;
  uint8_t* op_base = raw_base + p.rawb * p.rows_raw * RAW_BLK;
  const int slot_bytes = (p.group ? S : 1) * NB * p.opblk;            // one operand-ring slot
  uint8_t* stage_base = op_base + (SHIFT ? p.ops * slot_bytes : 0);   // epilogue staging: [128 ch][64 px] swizzled
  uint8_t* bar_base = stage_base + STAGE_BYTES;
  uint64_t* raw_full = reinterpret_cast<uint64_t*>(bar_base);
  uint64_t* raw_empty = raw_full + MAXRING;
  uint64_t* a_full = raw_empty + MAXRING;
  uint64_t* a_empty = a_full + MAXRING;
  uint64_t* op_full = a_empty + MAXRING;
  uint64_t* op_empty = op_full + MAXRING;
  uint64_t* a_res_full = op_empty + MAXRING;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int i = 0; i < MAXRING; ++i) {
      mbar_init(&raw_full[i], 1);
      mbar_init(&raw_empty[i], SHIFT ? SHIFT_THREADS : 2);   // shift path: the shifter threads, else the two consumers
      mbar_init(&a_full[i], 1); mbar_init(&a_empty[i], 2);
      mbar_init(&op_full[i], SHIFT_THREADS); mbar_init(&op_empty[i], 2);
    }
    mbar_init(a_res_full, 1);
    fence_barrier_init();
  }
  __syncthreads();

#define TAP_TILE_DECODE(t)                                        \
  const int tw_ = (t) % p.tiles_w;                                \
  const int th_ = ((t) / p.tiles_w) % p.tiles_h;                  \
  const int n_ = (t) / (p.tiles_w * p.tiles_h);                   \
  const int w0 = tw_ * 64, h0 = th_ * NB;

  // 640 x 96 registers at launch.  The producer warpgroup (one busy thread) and the shifters (S = 1: idle) hand theirs
  // to the consumers, whose accumulators would spill at 96: 24 + 2 x 80 + 2 x 144 (S = 1: 24 + 2 x 24 + 2 x 200) <= 480.
  // Each role sets its count at the top of its own branch, so that ptxas allocates that branch at that count.
  if (warp < 4) {
    setmaxnreg_dec<24>();
    // ================= TMA producer: activation row blocks + (streamed) weight blocks =================
    // One thread issues both, INTERLEAVED: the TMA unit serves a CTA's requests in order, so a burst of all row
    // blocks of the next chunk (80 KB) in front of the small per-tap weight loads starved the MMA of weights for
    // ~2 us per chunk (r2 ncu: tensor pipe 24 %, L2->SM 4.4 TB/s).  Row blocks of chunk g+1 are therefore
    // spread over the taps of chunk g, behind each tap's weight block.
    if (warp == 0 && lane == 0) {
      tma_prefetch_desc(&tmap_x);
      tma_prefetch_desc(&tmap_w);
      if (p.a_resident) {
        mbar_arrive_expect_tx(a_res_full, taps * p.kchunks * p.mrows * 128);
        for (int tap = 0; tap < taps; ++tap)
          for (int kc = 0; kc < p.kchunks; ++kc)
            tma_load_2d(a_base + (tap * p.kchunks + kc) * p.a_blk, &tmap_w, a_res_full, kc * 64, tap * p.Mpad);
      }
      RingState rb, ra;
      const int xoff = SHIFT ? 8 : 0;
      int ct = blockIdx.x, ckc = 0;                       // current chunk (tile, channel chunk)
      if (ct < p.num_tiles) {                             // its row blocks: all at once (nothing to overlap with yet)
        TAP_TILE_DECODE(ct)
        mbar_wait(&raw_empty[rb.s], rb.ph ^ 1);
        mbar_arrive_expect_tx(&raw_full[rb.s], p.rows_raw * RAW_BLK);
        for (int i = 0; i < p.rows_raw; ++i)
          tma_load_4d(raw_base + (rb.s * p.rows_raw + i) * RAW_BLK, &tmap_x, &raw_full[rb.s], w0 - xoff, h0 - p.ph + i, 0, n_);
        rb.next(p.rawb);
      }
      while (ct < p.num_tiles) {
        int nt = ct, nkc = ckc + 1;                       // next chunk
        if (nkc == p.kchunks) { nkc = 0; nt = ct + gridDim.x; }
        const bool has_next = nt < p.num_tiles;
        TAP_TILE_DECODE(has_next ? nt : ct)
        uint8_t* dst = raw_base + rb.s * p.rows_raw * RAW_BLK;
        bool armed = false;
        int row = 0;
        for (int tap = 0; tap < taps; ++tap) {
          if (!p.a_resident) {
            mbar_wait(&a_empty[ra.s], ra.ph ^ 1);
            mbar_arrive_expect_tx(&a_full[ra.s], p.mrows * 128);
            tma_load_2d(a_base + ra.s * p.a_blk, &tmap_w, &a_full[ra.s], ckc * 64, tap * p.Mpad);
            ra.next(p.ast);
          }
          if (has_next) {
            if (!armed && mbar_test_wait(&raw_empty[rb.s], rb.ph ^ 1)) {
              mbar_arrive_expect_tx(&raw_full[rb.s], p.rows_raw * RAW_BLK);
              armed = true;
            }
            if (armed) {
              const int quota = ((tap + 1) * p.rows_raw + taps - 1) / taps;
              for (; row < quota; ++row)
                tma_load_4d(dst + row * RAW_BLK, &tmap_x, &raw_full[rb.s], w0 - xoff, h0 - p.ph + row, nkc * 64, n_);
            }
          }
        }
        if (has_next) {
          if (!armed) {
            mbar_wait(&raw_empty[rb.s], rb.ph ^ 1);
            mbar_arrive_expect_tx(&raw_full[rb.s], p.rows_raw * RAW_BLK);
          }
          for (; row < p.rows_raw; ++row)
            tma_load_4d(dst + row * RAW_BLK, &tmap_x, &raw_full[rb.s], w0 - xoff, h0 - p.ph + row, nkc * 64, n_);
          rb.next(p.rawb);
        }
        ct = nt; ckc = nkc;
      }
    }
  } else if (warp >= 12) {
    setmaxnreg_dec<SHIFT ? 80 : 24>();
    // ================= shifter: raw row blocks -> swizzled operand tile of tap (r, s) =================
    if (SHIFT) {
      const int tid = threadIdx.x - 12 * 32;   // 0..255
      RingState rb, ro;
      for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
        for (int kc = 0; kc < p.kchunks; ++kc) {
          mbar_wait(&raw_full[rb.s], rb.ph);
          // every channel row the MMA reads (KS * 16 = cbox): rows past Cin are zero, TMA zero-fills them in the raw box
          const int cv = p.cbox;
          const uint8_t* rawb = raw_base + rb.s * p.rows_raw * RAW_BLK;
          for (int r = 0; r < p.R; ++r)
            ShiftRow<NB, S, 0>::run(rawb + r * RAW_BLK, RAW_BLK, cv, tid, op_base, p.opblk, p.group, op_full, op_empty, ro, p.ops);
          mbar_arrive(&raw_empty[rb.s]);      // all shifter threads are done reading this raw buffer
          rb.next(p.rawb);
        }
      }
    }
  } else {
    setmaxnreg_inc<SHIFT ? 144 : 200>();
    // ================= consumers: wgmma over (chunk, tap), then registers -> NCHW rows =================
    const int wg = (threadIdx.x >> 7) - 1;
    const int w4 = (threadIdx.x >> 5) & 3;
    const bool wg_lead = (threadIdx.x & 127) == 0;
    const bool leader = threadIdx.x == 128;    // issues the TMA stores
    float acc[NPIX / 2];
    if (p.a_resident) mbar_wait(a_res_full, 0);
    RingState rb, ra, ro;
    for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
      TAP_TILE_DECODE(t)
      // ring slots read by the last committed wgmma group; released once the next group is committed and the
      // previous one has completed (wgmma_wait<1>)
      int rel_op = -1, rel_a = -1, rel_raw = -1;
      for (int kc = 0; kc < p.kchunks; ++kc) {
        if (!SHIFT) mbar_wait(&raw_full[rb.s], rb.ph);
        for (int tap = 0; tap < taps; ++tap) {
          uint32_t sb;
          const int si = tap % S;                                   // filter column (compile-time S)
          if (SHIFT) {
            if (!p.group || si == 0) mbar_wait(&op_full[ro.s], ro.ph);
            sb = smem_u32(op_base + ro.s * slot_bytes + (p.group ? si * NB * p.opblk : 0));
          } else {
            sb = smem_u32(raw_base + (rb.s * p.rows_raw + tap) * RAW_BLK);   // S == 1: tap == filter row
          }
          uint32_t sa;
          if (p.a_resident) {
            sa = smem_u32(a_base + (tap * p.kchunks + kc) * p.a_blk);
          } else {
            mbar_wait(&a_full[ra.s], ra.ph);
            sa = smem_u32(a_base + ra.s * p.a_blk);
          }
          wgmma_fence();
#pragma unroll
          for (int ks = 0; ks < KS; ++ks) {
            // B: MN-major SW128, 16 channels = two 8-row groups (SBO 1024 B); 64-pixel blocks (= tile rows) at LBO
            const uint64_t bdesc = gmma_desc(sb + ks * 2048, SHIFT ? p.opblk : RAW_BLK, 1024);
            // A: K-major SW128, 8-row groups at SBO 1024 B, this warpgroup's 64 rows 8 KB in; +32 B per k-step
            const uint64_t adesc = gmma_desc(sa + wg * 8192 + ks * 32, 16, 1024);
            Wgmma<NPIX, 1>::mma(acc, adesc, bdesc, (kc | tap | ks) ? 1u : 0u);
          }
          wgmma_commit();
          wgmma_wait<1>();
          if (wg_lead) {
            if (rel_op >= 0) mbar_arrive(&op_empty[rel_op]);
            if (rel_a >= 0) mbar_arrive(&a_empty[rel_a]);
            if (rel_raw >= 0) mbar_arrive(&raw_empty[rel_raw]);
          }
          rel_op = rel_a = rel_raw = -1;
          if (SHIFT && (!p.group || si == S - 1)) { rel_op = ro.s; ro.next(p.ops); }
          if (!p.a_resident) { rel_a = ra.s; ra.next(p.ast); }
          if (!SHIFT && tap == taps - 1) { rel_raw = rb.s; rb.next(p.rawb); }
        }
      }
      wgmma_wait<0>();
      reg_fence(acc);
      if (wg_lead) {
        if (rel_op >= 0) mbar_arrive(&op_empty[rel_op]);
        if (rel_a >= 0) mbar_arrive(&a_empty[rel_a]);
        if (rel_raw >= 0) mbar_arrive(&raw_empty[rel_raw]);
      }
      const int r0 = 64 * wg + 16 * w4 + (lane >> 2);   // fragment rows (output channels) r0 and r0 + 8
      const float b0 = (r0 < p.M && p.bias) ? __bfloat162float(p.bias[r0]) : 0.f;
      const float b1 = (r0 + 8 < p.M && p.bias) ? __bfloat162float(p.bias[r0 + 8]) : 0.f;
#pragma unroll
      for (int j = 0; j < NB; ++j) {
        // the TMA store that last read the staging buffer must be done reading it
        if (leader) tma_store_wait_read<0>();
        named_bar_sync(1, 256);
#pragma unroll
        for (int q = 0; q < 8; ++q) {                   // 8-pixel column group of tile row j
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = r0 + 8 * h;
            const float bias = h ? b1 : b0;
            const int i = 4 * (8 * j + q) + 2 * h;
            const uint32_t v = pack_bf16x2(acc[i] + bias, acc[i + 1] + bias);
            // SWIZZLE_128B: 16-byte chunk ^ (row % 8)
            *reinterpret_cast<uint32_t*>(stage_base + r * 128 + ((q ^ (r & 7)) << 4) + (lane & 3) * 4) = v;
          }
        }
        fence_proxy_async();                              // smem writes -> visible to the TMA (async proxy)
        named_bar_sync(1, 256);
        // rows past the image and channels past M are clipped by the tensor map
        if (leader && h0 + j < p.H) {
          tma_store_4d(&tmap_y, stage_base, w0, h0 + j, 0, n_);
          tma_store_commit();
        }
      }
    }
    if (leader) tma_store_wait_read<0>();
  }
#undef TAP_TILE_DECODE
}

constexpr int TAP_SMEM_LIMIT = 222 * 1024;   // of H100's 227 KB per block
constexpr int TAP_SMEM_AUX = 1024 /*align*/ + 1024 /*barriers*/;

struct TapPlan {
  int NB;
  TapParams p;
  int smem;
};

// shared-memory plan for an R x S conv with M <= 128 output channels; returns false if nothing fits
bool plan_tap(int M, int Cin, int R, int S, int H, int W, int N, TapPlan* out) {
  TapParams p{};
  p.M = M; p.Cin = Cin; p.H = H; p.W = W; p.N = N; p.R = R;
  p.mrows = round_up(M, 8);
  p.a_blk = round_up(p.mrows * 128, 1024);
  p.kchunks = (Cin + 63) / 64;
  const int taps = R * S;
  const bool shift = S > 1;
  p.cbox = Cin >= 64 ? 64 : round_up(Cin, 16);
  p.raw_blk = p.cbox * (shift ? RAW_SHIFT_ROW : 128);
  const int raw_blk = p.raw_blk;
  const int budget = TAP_SMEM_LIMIT - TAP_SMEM_AUX;
  // an M = 128 MMA reads 128 rows of A whatever mrows is: the bytes after the last A block must exist -> the raw
  // buffers follow the A region (always >= 16 KB)
  p.opblk = p.cbox * 128;
  const int budget_ops = budget - STAGE_BYTES;
  // one tile = 2 rows of 64 pixels: 128 accumulator columns, 64 fp32 registers per consumer thread
  for (int NB = 2; NB >= 2; NB -= 2) {
    p.rows_raw = NB + R - 1;
    const int raw_buf = p.rows_raw * raw_blk;                   // one raw buffer (all row blocks of a chunk)
    const int a_res = taps * p.kchunks * p.a_blk;
    for (int resident = 1; resident >= 0; --resident) {
      for (int group = shift ? 1 : 0; group >= 0; --group) {
        // operand-ring slot: the S tiles of one filter row (one shifter <-> MMA hand-shake per row: the ~500-cycle
        // round trip per hand-shake dominated the small-channel layers), else one tile
        const int slot = (group ? S : 1) * NB * p.opblk;
        // minimum configuration: 2 raw buffers, (shift) 2 operand slots, weights resident or a ring of 3 blocks
        int ast = resident ? 0 : 3;
        int a_bytes = resident ? a_res : ast * p.a_blk;
        int rawb = 2, ops = shift ? 2 : 0;
        int rem = budget_ops - a_bytes - rawb * raw_buf - ops * slot;
        if (rem < 0) continue;
        if (shift && !group && rem >= slot) { ++ops; rem -= slot; }
        while (!resident && ast < MAXRING && rem >= p.a_blk) { ++ast; rem -= p.a_blk; }
        while (rawb < 4 && rem >= raw_buf) { ++rawb; rem -= raw_buf; }
        while (shift && ops < 4 && rem >= slot) { ++ops; rem -= slot; }
        a_bytes = resident ? a_res : ast * p.a_blk;
        p.a_resident = resident; p.ast = ast; p.ops = ops; p.rawb = rawb; p.group = group;
        out->NB = NB; out->p = p;
        out->smem = a_bytes + rawb * raw_buf + ops * slot + STAGE_BYTES + TAP_SMEM_AUX;
        return true;
      }
    }
  }
  return false;
}

template <int NB, int S, int KS>
int launch_tap(const CUtensorMap& tw, const CUtensorMap& tx, const CUtensorMap& ty, const TapParams& p, int smem,
               cudaStream_t st) {
  auto kern = conv_tap_kernel<NB, S, KS>;
  const int rc = allow_dynamic_smem((const void*)kern, TAP_SMEM_LIMIT);
  if (rc) return rc;
  const int sms = sm_count();
  const int grid = p.num_tiles < sms ? p.num_tiles : sms;
  kern<<<grid, TAP_THREADS, smem, st>>>(tw, tx, ty, p);
  count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

}  // namespace

bool tap_v2_supported(int M, int Cin, int R, int S, int H, int W, int N, int stride) {
  if (stride != 1 || M > 128 || R * S == 1 || (W % 64) != 0 || H < 2) return false;
  if (!(S == 1 || S == 3 || S == 5 || S == 7) || (R & 1) == 0 || R > 7) return false;
  TapPlan pl;
  return plan_tap(M, Cin, R, S, H, W, N, &pl);
}

// wp: repacked weights [taps][Mpad][Cpad] bf16 (taps in (r, s) order), x: [N][Cin][H][W], y: [N][M][H][W]
int run_conv_tap_v2(const __nv_bfloat16* wp, int Mpad, int Cpad, const __nv_bfloat16* x, const __nv_bfloat16* bias,
                    __nv_bfloat16* y, int M, int Cin, int R, int S, int ph, int H, int W, int N, cudaStream_t st) {
  TapPlan pl;
  SPC_REQUIRE(plan_tap(M, Cin, R, S, H, W, N, &pl), "tap conv: no shared-memory plan for M=%d Cin=%d %dx%d", M, Cin, R, S);
  TapParams& p = pl.p;
  p.ph = ph; p.Mpad = Mpad; p.bias = bias; p.y = y;
  p.tiles_w = W / 64;
  p.tiles_h = (H + pl.NB - 1) / pl.NB;
  p.num_tiles = p.tiles_w * p.tiles_h * N;
  CUtensorMap tw, tx, ty;
  {
    const uint64_t dims[2] = {(uint64_t)Cpad, (uint64_t)R * S * Mpad};
    const uint64_t strides[2] = {0, (uint64_t)Cpad * 2};
    const uint32_t box[2] = {64, (uint32_t)p.mrows};
    int rc = make_tmap(&tw, wp, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  {
    const uint64_t dims[4] = {(uint64_t)W, (uint64_t)H, (uint64_t)Cin, (uint64_t)N};
    const uint64_t strides[4] = {0, (uint64_t)W * 2, (uint64_t)H * W * 2, (uint64_t)H * W * Cin * 2};
    const uint32_t box[4] = {(uint32_t)(S > 1 ? 80 : 64), 1, (uint32_t)p.cbox, 1};
    int rc = make_tmap(&tx, x, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, dims, strides, box,
                       S > 1 ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  {
    const uint64_t dims[4] = {(uint64_t)W, (uint64_t)H, (uint64_t)M, (uint64_t)N};
    const uint64_t strides[4] = {0, (uint64_t)W * 2, (uint64_t)H * W * 2, (uint64_t)H * W * M * 2};
    const uint32_t box[4] = {64, 1, 128, 1};
    int rc = make_tmap(&ty, y, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
#define TAP_CASE(s, ks) if (S == s && p.cbox == 16 * ks) return launch_tap<2, s, ks>(tw, tx, ty, p, pl.smem, st);
#define TAP_CASES(s) TAP_CASE(s, 1) TAP_CASE(s, 2) TAP_CASE(s, 3) TAP_CASE(s, 4)
  TAP_CASES(1) TAP_CASES(3) TAP_CASES(5) TAP_CASES(7)
#undef TAP_CASES
#undef TAP_CASE
  set_error("tap conv: unsupported filter width %d", S);
  return SPC_EUNSUPPORTED;
}

}  // namespace spc
