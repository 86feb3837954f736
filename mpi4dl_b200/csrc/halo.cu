// halo.cu -- halo strip pack / pad / crop kernels and the peer-memory mailbox transport.
//
// Replaces the reference's per-direction `.clone()` + torch.cuda.synchronize() + dist.isend /
// torch.zeros + synchronize + dist.irecv / req.wait() / 8 slice-assign copies
// (spatial.py:336-413): one pack kernel writes every outgoing strip -- straight into the
// neighbours' receive buffers when they are CUDA-IPC peer mappings (NVLink P2P stores) -- and
// a device-side flag (release/acquire at system scope) orders producer and consumer streams.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace spc {

static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static long long g_launches = 0;
void count_launch(int n) { g_launches += n; }
long long launches(int reset) { long long v = g_launches; if (reset) g_launches = 0; return v; }

// grow-only device scratch for the halo fix-up (single host thread per process)
static void* g_scratch = nullptr;
static size_t g_scratch_bytes = 0;
void* boundary_scratch(size_t bytes) {
  if (bytes > g_scratch_bytes) {
    if (g_scratch) { cudaDeviceSynchronize(); cudaFree(g_scratch); }
    g_scratch = nullptr; g_scratch_bytes = 0;
    const size_t want = (bytes + (16u << 20)) & ~(size_t)((1u << 20) - 1);
    if (cudaMalloc(&g_scratch, want) != cudaSuccess) return nullptr;
    g_scratch_bytes = want;
  }
  return g_scratch;
}

namespace {

struct PackParams {
  const void* x;
  void* send[9];
  int N, C, H, W, hh, hw;
  long long off[10];  // prefix sums of strip element counts
};

// The strip a tile sends towards direction d is the band of REAL rows/cols adjacent to that
// edge (reference spatial.py:239-309 locations_send, expressed in unpadded coordinates).
template <typename T>
__global__ void halo_pack_kernel(const PackParams p) {
  const long long total = p.off[9];
  const T* x = reinterpret_cast<const T*>(p.x);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    int d = 0;
#pragma unroll
    for (int q = 1; q < 9; ++q) d += (i >= p.off[q]) ? 1 : 0;
    const long long e = i - p.off[d];
    const int dr = d / 3, dc = d % 3;
    const int sh = (dr == 1) ? p.H : p.hh;
    const int sw = (dc == 1) ? p.W : p.hw;
    const int xw = (int)(e % sw);
    const int yh = (int)((e / sw) % sh);
    const long long nc = e / ((long long)sw * sh);
    const int h = (dr == 0) ? yh : (dr == 2 ? p.H - p.hh + yh : yh);
    const int w = (dc == 0) ? xw : (dc == 2 ? p.W - p.hw + xw : xw);
    reinterpret_cast<T*>(p.send[d])[e] = x[(nc * p.H + h) * p.W + w];
  }
}

template <typename T>
__global__ void halo_pad_kernel(const TileView v, T* __restrict__ y) {
  const int Hp = v.H + 2 * v.hh, Wp = v.W + 2 * v.hw;
  const size_t total = (size_t)v.N * v.C * Hp * Wp;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int w = (int)(i % Wp);
    const int h = (int)((i / Wp) % Hp);
    const size_t nc = i / ((size_t)Wp * Hp);
    y[i] = from_f32<T>(tile_load<T>(v, (int)(nc / v.C), (int)(nc % v.C), h - v.hh, w - v.hw));
  }
}

template <typename T>
__global__ void halo_crop_kernel(const T* __restrict__ dy, T* __restrict__ dx, int NC, int H, int W, int hh, int hw) {
  const int Hp = H + 2 * hh, Wp = W + 2 * hw;
  const size_t total = (size_t)NC * H * W;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int w = (int)(i % W);
    const int h = (int)((i / W) % H);
    const size_t nc = i / ((size_t)W * H);
    dx[i] = dy[(nc * Hp + h + hh) * Wp + w + hw];
  }
}

// ---- fused protocol kernels -----------------------------------------------------------------
// post:    wait until every neighbour has drained the slot we are about to overwrite (ack flags,
//          local memory) -> pack all strips straight into the neighbours' slots (peer stores) ->
//          the LAST block publishes the sequence number on the neighbours' arrival flags.
// collect: wait for the neighbours' arrival flags -> copy the received strips out of the mailbox
//          into private buffers (they are needed again by wgrad) -> the last block acks.
// Graph-capturable: no host-side state in the launch arguments.  The sequence number of the exchange is *seq_word + 1;
// its parity selects the half of the double-buffered slot (payload pointers advance by par_bytes) and the flag bank
// (flag pointers advance by 9 words).  wait_lag: 0 = wait for the current sequence (arrivals), 2 = wait for
// sequence-2 (acks of the slot half about to be overwritten).
struct FlagSet {
  uint32_t* wait[9];     // flags to wait on (>= sequence - wait_lag), NULL = skip
  uint32_t* signal[9];   // flags to publish the sequence number on when the whole grid is done, NULL = skip
  unsigned int* counter; // grid completion counter (device memory, self-resetting)
  uint32_t* seq_word;
  int advance_seq;       // the last block stores the new sequence number (collect = end of the exchange)
  int wait_lag;
  long long par_bytes;
  unsigned long long timeout_ns;   // 0 = spin forever
};

__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// returns the sequence number of this exchange; threads 0..8 wait for their direction's flag
__device__ __forceinline__ uint32_t wait_flags(const FlagSet& f) {
  const uint32_t seq = *reinterpret_cast<const volatile uint32_t*>(f.seq_word) + 1u;
  const int par = (int)(seq & 1u);
  const uint32_t wseq = f.wait_lag ? (seq > (uint32_t)f.wait_lag ? seq - (uint32_t)f.wait_lag : 0u) : seq;
  if (threadIdx.x < 9) {
    const uint32_t* w = f.wait[threadIdx.x];
    if (w != nullptr && wseq != 0u) {
      w += par * 9;
      uint32_t v;
      const unsigned long long t0 = f.timeout_ns ? global_ns() : 0ull;
      do {
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(w) : "memory");
        if ((int32_t)(v - wseq) >= 0) break;
        __nanosleep(32);
        if (f.timeout_ns && global_ns() - t0 > f.timeout_ns) {
          // a peer died or never posted: surface an error instead of spinning the GPU forever
          printf("libspconv: halo flag wait timed out (direction %d, have %u, want %u) -- trapping\n", (int)threadIdx.x, v,
                 wseq);
          __trap();
        }
      } while (true);
    }
  }
  __syncthreads();
  return seq;
}

__device__ __forceinline__ void signal_when_grid_done(const FlagSet& f, uint32_t seq) {
  __threadfence_system();          // this thread's (peer) stores are visible system-wide
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int done = atomicAdd(f.counter, 1u);
    if (done == gridDim.x - 1) {   // every block has fenced its stores
      __threadfence_system();
      const int par = (int)(seq & 1u);
      for (int i = 0; i < 9; ++i)
        if (f.signal[i])
          asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(f.signal[i] + par * 9), "r"(seq) : "memory");
      *f.counter = 0u;
      if (f.advance_seq) *reinterpret_cast<volatile uint32_t*>(f.seq_word) = seq;
    }
  }
}

template <typename T>
__global__ void halo_post_kernel(const PackParams p, const FlagSet f) {
  const uint32_t seq = wait_flags(f);
  const long long pofs = (long long)(seq & 1u) * f.par_bytes;   // slot half of this sequence number
  const long long total = p.off[9];
  const T* x = reinterpret_cast<const T*>(p.x);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    int d = 0;
#pragma unroll
    for (int q = 1; q < 9; ++q) d += (i >= p.off[q]) ? 1 : 0;
    const long long e = i - p.off[d];
    const int dr = d / 3, dc = d % 3;
    const int sh = (dr == 1) ? p.H : p.hh;
    const int sw = (dc == 1) ? p.W : p.hw;
    const int xw = (int)(e % sw);
    const int yh = (int)((e / sw) % sh);
    const long long nc = e / ((long long)sw * sh);
    const int h = (dr == 0) ? yh : (dr == 2 ? p.H - p.hh + yh : yh);
    const int w = (dc == 0) ? xw : (dc == 2 ? p.W - p.hw + xw : xw);
    reinterpret_cast<T*>(reinterpret_cast<char*>(p.send[d]) + pofs)[e] = x[(nc * p.H + h) * p.W + w];
  }
  signal_when_grid_done(f, seq);
}

struct CollectParams {
  const uint8_t* src[9];
  uint8_t* dst[9];
  long long off[10];   // prefix sums of byte counts (multiples of 2)
};

// Reverse direction of the exact backward: the same protocol as halo_post_kernel, but the payload is a set of
// caller-given (fp32) strip buffers src[d] copied into the neighbours' slots dst[d], instead of a pack of the tile.
__global__ void halo_post_strips_kernel(const CollectParams p, const FlagSet f) {
  const uint32_t seq = wait_flags(f);
  const long long pofs = (long long)(seq & 1u) * f.par_bytes;
  const long long total = p.off[9] / 4;   // 4-byte units
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long b = i * 4;
    int d = 0;
#pragma unroll
    for (int q = 1; q < 9; ++q) d += (b >= p.off[q]) ? 1 : 0;
    const long long e = b - p.off[d];
    *reinterpret_cast<uint32_t*>(p.dst[d] + pofs + e) = *reinterpret_cast<const uint32_t*>(p.src[d] + e);
  }
  signal_when_grid_done(f, seq);
}

__global__ void halo_collect_kernel(const CollectParams p, const FlagSet f) {
  const uint32_t seq = wait_flags(f);
  const long long pofs = (long long)(seq & 1u) * f.par_bytes;
  const long long total = p.off[9] / 2;   // 2-byte units (strips of bf16 columns may be 2-byte sized)
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long b = i * 2;
    int d = 0;
#pragma unroll
    for (int q = 1; q < 9; ++q) d += (b >= p.off[q]) ? 1 : 0;
    const long long e = b - p.off[d];
    *reinterpret_cast<uint16_t*>(p.dst[d] + e) = *reinterpret_cast<const volatile uint16_t*>(p.src[d] + pofs + e);
  }
  signal_when_grid_done(f, seq);
}


// ---- halo fix-up over the boundary outputs only ------------------------------------------------------------------
__device__ __forceinline__ void boundary_decode(const BoundaryRects& b, int p, int& n, int& i, int& j) {
  n = p / b.per_image;
  const int q = p - n * b.per_image;
  int r = 0;
#pragma unroll
  for (int t = 1; t < 4; ++t) r += (t < b.n && q >= b.start[t]) ? 1 : 0;
  const int e = q - b.start[r];
  const int rw = b.x1[r] - b.x0[r];
  i = b.y0[r] + e / rw;
  j = b.x0[r] + e % rw;
}

__global__ void halo_im2col_kernel(const TileView v, const BoundaryRects b, int R, int S, int sh, int sw, int ph, int pw,
                                   __nv_bfloat16* __restrict__ V) {
  const size_t total = (size_t)v.C * R * S * b.padded;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int p = (int)(idx % b.padded);
    const int ct = (int)(idx / b.padded);
    float val = 0.f;
    if (p < b.total) {
      int n, i, j;
      boundary_decode(b, p, n, i, j);
      const int s = ct % S, r = (ct / S) % R, c = ct / (R * S);
      val = tile_load<__nv_bfloat16>(v, n, c, i * sh + r - ph, j * sw + s - pw);   // halo-only view: 0 inside the tile
    }
    V[idx] = __float2bfloat16(val);
  }
}

__global__ void boundary_gather_kernel(const __nv_bfloat16* __restrict__ dy, const BoundaryRects b, int K, int Ho, int Wo,
                                       __nv_bfloat16* __restrict__ G) {
  const size_t total = (size_t)K * b.padded;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int p = (int)(idx % b.padded);
    const int k = (int)(idx / b.padded);
    __nv_bfloat16 val = __float2bfloat16(0.f);
    if (p < b.total) {
      int n, i, j;
      boundary_decode(b, p, n, i, j);
      val = dy[(((size_t)n * K + k) * Ho + i) * Wo + j];
    }
    G[idx] = val;
  }
}

__global__ void boundary_scatter_kernel(const __nv_bfloat16* __restrict__ O, const BoundaryRects b, int K, int Ho, int Wo,
                                            __nv_bfloat16* __restrict__ y) {
  const size_t total = (size_t)K * b.total;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int p = (int)(idx % b.total);
    const int k = (int)(idx / b.total);
    int n, i, j;
    boundary_decode(b, p, n, i, j);
    y[(((size_t)n * K + k) * Ho + i) * Wo + j] = O[(size_t)k * b.padded + p];
  }
}

inline int grid_for(size_t total) {
  size_t b = (total + 255) / 256;
  if (b > 132 * 16) b = 132 * 16;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace
}  // namespace spc

namespace spc {
int launch_halo_im2col(const TileView& halo_only, const BoundaryRects& b, int R, int S, int sh, int sw, int ph, int pw, void* V,
                       cudaStream_t st) {
  const size_t total = (size_t)halo_only.C * R * S * b.padded;
  if (!total) return SPC_OK;
  halo_im2col_kernel<<<grid_for(total), 256, 0, st>>>(halo_only, b, R, S, sh, sw, ph, pw, (__nv_bfloat16*)V);
  count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}
int launch_boundary_gather(const void* dy, const BoundaryRects& b, int K, int Ho, int Wo, void* G, cudaStream_t st) {
  const size_t total = (size_t)K * b.padded;
  if (!total) return SPC_OK;
  boundary_gather_kernel<<<grid_for(total), 256, 0, st>>>((const __nv_bfloat16*)dy, b, K, Ho, Wo, (__nv_bfloat16*)G);
  count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}
int launch_boundary_scatter(const void* O, const BoundaryRects& b, int K, int Ho, int Wo, void* y, cudaStream_t st) {
  const size_t total = (size_t)K * b.total;
  if (!total) return SPC_OK;
  boundary_scatter_kernel<<<grid_for(total), 256, 0, st>>>((const __nv_bfloat16*)O, b, K, Ho, Wo, (__nv_bfloat16*)y);
  count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}
}  // namespace spc

struct spc_mailbox {
  void* base;        // data area followed by flags
  size_t bytes;      // data bytes (rounded up to 256)
  int nflags;
  int owner;         // 1: cudaMalloc'ed here, 0: IPC mapping of a peer allocation
};

extern "C" {

const char* spc_last_error(void) { return spc::g_err; }
int spc_version(void) { return SPC_VERSION; }
long long spc_launch_count(int reset) { return spc::launches(reset); }

int spc_device_info(int device, int* sm_count, int* cc) {
  cudaDeviceProp prop;
  SPC_CHECK_CUDA(cudaGetDeviceProperties(&prop, device));
  if (sm_count) *sm_count = prop.multiProcessorCount;
  if (cc) *cc = prop.major * 10 + prop.minor;
  SPC_REQUIRE(prop.major == 9 && prop.minor == 0, "libspconv is built for sm_90a only; device %d is sm_%d%d", device,
              prop.major, prop.minor);
  return SPC_OK;
}

int spc_halo_pack(int N, int C, int H, int W, int halo_h, int halo_w, int dtype, const void* x, void* const send[9],
                  void* stream) {
  SPC_REQUIRE(x && send, "halo_pack: null pointer");
  SPC_REQUIRE(halo_h <= H && halo_w <= W, "halo_pack: halo (%d,%d) larger than tile (%d,%d)", halo_h, halo_w, H, W);
  spc::PackParams p{};
  p.x = x; p.N = N; p.C = C; p.H = H; p.W = W; p.hh = halo_h; p.hw = halo_w;
  long long off = 0;
  for (int d = 0; d < 9; ++d) {
    p.off[d] = off;
    p.send[d] = (d == 4) ? nullptr : send[d];
    if (p.send[d]) {
      const long long sh = (d / 3 == 1) ? H : halo_h, sw = (d % 3 == 1) ? W : halo_w;
      off += (long long)N * C * sh * sw;
    }
  }
  p.off[9] = off;
  if (off == 0) return SPC_OK;
  if (dtype == SPC_BF16)
    spc::halo_pack_kernel<__nv_bfloat16><<<spc::grid_for(off), 256, 0, (cudaStream_t)stream>>>(p);
  else
    spc::halo_pack_kernel<float><<<spc::grid_for(off), 256, 0, (cudaStream_t)stream>>>(p);
  spc::count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

int spc_halo_pad(int N, int C, int H, int W, int halo_h, int halo_w, int dtype, const void* x, const spc_halo* halo,
                 void* y, void* stream) {
  SPC_REQUIRE(x && y, "halo_pad: null pointer");
  spc::TileView v = spc::make_view(x, halo, N, C, H, W, halo_h, halo_w);
  const size_t total = (size_t)N * C * (H + 2 * halo_h) * (W + 2 * halo_w);
  if (total == 0) return SPC_OK;
  if (dtype == SPC_BF16)
    spc::halo_pad_kernel<__nv_bfloat16><<<spc::grid_for(total), 256, 0, (cudaStream_t)stream>>>(v, (__nv_bfloat16*)y);
  else
    spc::halo_pad_kernel<float><<<spc::grid_for(total), 256, 0, (cudaStream_t)stream>>>(v, (float*)y);
  spc::count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

int spc_halo_crop(int N, int C, int H, int W, int halo_h, int halo_w, int dtype, const void* dy, void* dx,
                  void* stream) {
  SPC_REQUIRE(dy && dx, "halo_crop: null pointer");
  const size_t total = (size_t)N * C * H * W;
  if (total == 0) return SPC_OK;
  if (dtype == SPC_BF16)
    spc::halo_crop_kernel<__nv_bfloat16><<<spc::grid_for(total), 256, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)dy, (__nv_bfloat16*)dx, N * C, H, W, halo_h, halo_w);
  else
    spc::halo_crop_kernel<float><<<spc::grid_for(total), 256, 0, (cudaStream_t)stream>>>(
        (const float*)dy, (float*)dx, N * C, H, W, halo_h, halo_w);
  spc::count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

// flag word idx of a mailbox: the flags follow the data area
static uint32_t* mb_flag(spc_mailbox* mb, int idx) {
  return reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(mb->base) + mb->bytes) + idx;
}

// spin bound of the flag waits: SPCONV_SPIN_TIMEOUT_S seconds (default 120; 0 = spin forever)
static unsigned long long spin_timeout_ns() {
  static long long v = -1;
  if (v < 0) {
    const char* e = getenv("SPCONV_SPIN_TIMEOUT_S");
    const double sec = e ? atof(e) : 120.0;
    v = sec > 0 ? (long long)(sec * 1e9) : 0;
  }
  return (unsigned long long)v;
}

int spc_halo_post_auto(int N, int C, int H, int W, int halo_h, int halo_w, int dtype, const void* x,
                       void* const send0[9], size_t slot_bytes, spc_mailbox* self, spc_mailbox* const peers[9],
                       const int ack_idx0[9], const int arrival_idx0[9], int seq_idx, int counter_idx, void* stream) {
  SPC_REQUIRE(self && seq_idx >= 0 && seq_idx < self->nflags && counter_idx >= 0 && counter_idx < self->nflags,
              "halo_post_auto: bad sequence / counter flag index");
  SPC_REQUIRE(x && send0 && peers && ack_idx0 && arrival_idx0, "halo_post: null pointer");
  spc::PackParams p{};
  p.x = x; p.N = N; p.C = C; p.H = H; p.W = W; p.hh = halo_h; p.hw = halo_w;
  spc::FlagSet f{};
  long long off = 0;
  for (int d = 0; d < 9; ++d) {
    p.off[d] = off;
    p.send[d] = (d == 4) ? nullptr : send0[d];
    if (p.send[d]) {
      SPC_REQUIRE(peers[d] != nullptr, "halo_post: no peer mailbox for direction %d", d);
      const long long sh = (d / 3 == 1) ? H : halo_h, sw = (d % 3 == 1) ? W : halo_w;
      off += (long long)N * C * sh * sw;
      f.wait[d] = mb_flag(self, ack_idx0[d]);
      f.signal[d] = mb_flag(peers[d], arrival_idx0[d]);
    }
  }
  p.off[9] = off;
  if (off == 0) return SPC_OK;
  f.seq_word = mb_flag(self, seq_idx);
  f.advance_seq = 0; f.wait_lag = 2; f.par_bytes = (long long)slot_bytes;
  f.timeout_ns = spin_timeout_ns();
  // per-slot completion counter (two streams may run exchanges of different layers concurrently)
  f.counter = reinterpret_cast<unsigned int*>(mb_flag(self, counter_idx));
  const int grid = spc::grid_for(off) > 64 ? 64 : spc::grid_for(off);
  if (dtype == SPC_BF16) spc::halo_post_kernel<__nv_bfloat16><<<grid, 256, 0, (cudaStream_t)stream>>>(p, f);
  else spc::halo_post_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>(p, f);
  spc::count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

int spc_halo_collect_auto(void* const dst[9], const void* const src0[9], const size_t bytes[9], size_t slot_bytes,
                          spc_mailbox* self, spc_mailbox* const peers[9], const int arrival_idx0[9],
                          const int ack_idx0[9], int seq_idx, int counter_idx, void* stream) {
  SPC_REQUIRE(self && seq_idx >= 0 && seq_idx < self->nflags && counter_idx >= 0 && counter_idx < self->nflags,
              "halo_collect_auto: bad sequence / counter flag index");
  SPC_REQUIRE(dst && src0 && bytes && peers, "halo_collect: null pointer");
  spc::CollectParams p{};
  spc::FlagSet f{};
  long long off = 0;
  for (int d = 0; d < 9; ++d) {
    p.off[d] = off;
    if (d != 4 && dst[d] && bytes[d]) {
      SPC_REQUIRE(peers[d] != nullptr && src0[d] != nullptr, "halo_collect: missing source for direction %d", d);
      p.dst[d] = reinterpret_cast<uint8_t*>(dst[d]);
      p.src[d] = reinterpret_cast<const uint8_t*>(src0[d]);
      off += (long long)bytes[d];
      f.wait[d] = mb_flag(self, arrival_idx0[d]);
      f.signal[d] = mb_flag(peers[d], ack_idx0[d]);
    }
  }
  p.off[9] = off;
  if (off == 0) return SPC_OK;
  f.seq_word = mb_flag(self, seq_idx);
  f.advance_seq = 1; f.wait_lag = 0; f.par_bytes = (long long)slot_bytes;
  f.timeout_ns = spin_timeout_ns();
  f.counter = reinterpret_cast<unsigned int*>(mb_flag(self, counter_idx));
  const int grid = spc::grid_for((size_t)off / 2) > 64 ? 64 : spc::grid_for((size_t)off / 2);
  spc::halo_collect_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(p, f);
  spc::count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

int spc_halo_post_strips_auto(const void* const src[9], const size_t bytes[9], void* const send0[9], size_t slot_bytes,
                              spc_mailbox* self, spc_mailbox* const peers[9], const int ack_idx0[9],
                              const int arrival_idx0[9], int seq_idx, int counter_idx, void* stream) {
  SPC_REQUIRE(src && bytes && send0 && self && peers && ack_idx0 && arrival_idx0, "halo_post_strips: null pointer");
  SPC_REQUIRE(seq_idx >= 0 && seq_idx < self->nflags && counter_idx >= 0 && counter_idx < self->nflags,
              "halo_post_strips_auto: bad sequence / counter flag index");
  spc::CollectParams p{};
  spc::FlagSet f{};
  long long off = 0;
  for (int d = 0; d < 9; ++d) {
    p.off[d] = off;
    if (d != 4 && send0[d] && bytes[d]) {
      SPC_REQUIRE(peers[d] != nullptr && src[d] != nullptr, "halo_post_strips: missing source for direction %d", d);
      SPC_REQUIRE(bytes[d] % 4 == 0, "halo_post_strips: strip %d is %zu bytes, not a multiple of 4", d, bytes[d]);
      p.dst[d] = reinterpret_cast<uint8_t*>(send0[d]);
      p.src[d] = reinterpret_cast<const uint8_t*>(src[d]);
      off += (long long)bytes[d];
      f.wait[d] = mb_flag(self, ack_idx0[d]);
      f.signal[d] = mb_flag(peers[d], arrival_idx0[d]);
    }
  }
  p.off[9] = off;
  if (off == 0) return SPC_OK;
  f.seq_word = mb_flag(self, seq_idx);
  f.advance_seq = 0; f.wait_lag = 2; f.par_bytes = (long long)slot_bytes;
  f.timeout_ns = spin_timeout_ns();
  f.counter = reinterpret_cast<unsigned int*>(mb_flag(self, counter_idx));
  const int grid = spc::grid_for((size_t)off / 4) > 64 ? 64 : spc::grid_for((size_t)off / 4);
  spc::halo_post_strips_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(p, f);
  spc::count_launch();
  SPC_CHECK_CUDA(cudaGetLastError());
  return SPC_OK;
}

// ---- mailbox ---------------------------------------------------------------------------------
static size_t mb_round(size_t b) { return (b + 255) & ~(size_t)255; }

int spc_mailbox_create(spc_mailbox** out, size_t bytes, int nflags) {
  SPC_REQUIRE(out && nflags >= 0, "mailbox_create: bad arguments");
  spc_mailbox* mb = new spc_mailbox();
  mb->bytes = mb_round(bytes); mb->nflags = nflags; mb->owner = 1; mb->base = nullptr;
  const size_t total = mb->bytes + mb_round(sizeof(uint32_t) * (size_t)nflags);
  cudaError_t e = cudaMalloc(&mb->base, total);  // plain cudaMalloc: IPC-exportable
  if (e != cudaSuccess) {
    spc::set_error("mailbox_create: cudaMalloc(%zu) failed: %s", total, cudaGetErrorString(e));
    delete mb;
    return SPC_ENOMEM;
  }
  e = cudaMemset(mb->base, 0, total);
  if (e != cudaSuccess) { spc::set_error("mailbox_create: memset: %s", cudaGetErrorString(e)); return SPC_ECUDA; }
  *out = mb;
  return SPC_OK;
}

void spc_mailbox_destroy(spc_mailbox* mb) {
  if (!mb) return;
  if (mb->owner) cudaFree(mb->base); else cudaIpcCloseMemHandle(mb->base);
  delete mb;
}

void* spc_mailbox_data(spc_mailbox* mb) { return mb ? mb->base : nullptr; }

int spc_mailbox_export(spc_mailbox* mb, unsigned char handle[SPC_IPC_HANDLE_BYTES]) {
  SPC_REQUIRE(mb && mb->owner && handle, "mailbox_export: need a locally created mailbox");
  static_assert(sizeof(cudaIpcMemHandle_t) == SPC_IPC_HANDLE_BYTES, "IPC handle size");
  cudaIpcMemHandle_t h;
  SPC_CHECK_CUDA(cudaIpcGetMemHandle(&h, mb->base));
  memcpy(handle, &h, sizeof(h));
  return SPC_OK;
}

int spc_mailbox_open(spc_mailbox** out, const unsigned char handle[SPC_IPC_HANDLE_BYTES], size_t bytes, int nflags) {
  SPC_REQUIRE(out && handle, "mailbox_open: null pointer");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof(h));
  void* p = nullptr;
  SPC_CHECK_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  spc_mailbox* mb = new spc_mailbox();
  mb->base = p; mb->bytes = mb_round(bytes); mb->nflags = nflags; mb->owner = 0;
  *out = mb;
  return SPC_OK;
}

}  // extern "C"
