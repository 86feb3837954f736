// common.cuh -- shared device helpers for libspconv (sm_90a).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/spconv.h"

namespace spc {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);   // bookkeeping for spc_launch_count()

#define SPC_CHECK_CUDA(expr)                                                              \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      spc::set_error("%s:%d CUDA error %s: %s", __FILE__, __LINE__, #expr,                \
                     cudaGetErrorString(_e));                                             \
      return SPC_ECUDA;                                                                   \
    }                                                                                     \
  } while (0)

#define SPC_REQUIRE(cond, ...)                                                            \
  do {                                                                                    \
    if (!(cond)) {                                                                        \
      spc::set_error(__VA_ARGS__);                                                        \
      return SPC_EINVAL;                                                                  \
    }                                                                                     \
  } while (0)

template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// Max pooling follows ATen's max_pool2d rule, `val > maxval || isnan(val)`: v replaces the running maximum m when it
// is larger or NaN.  So a window holding a NaN pools to NaN, its gradient goes to the (last) NaN, and among tied
// maxima the first one in row-major window order takes the gradient.  fmaxf would drop the NaN instead.
// pool_max_takes is the argmax step of the backward kernels (the bitwise | keeps it one predicate, no branch);
// pool_bwd_s2_vec_kernel applies the same rule unrolled for its 2x2 windows.
__device__ __forceinline__ bool pool_max_takes(float v, float m) { return (v > m) | (v != v); }
// The forward value: max.NaN is NaN when either operand is, so a fold over the window in any order gives ATen's value
// in one instruction, as fmaxf did (only the NaN's payload may differ).
__device__ __forceinline__ float pool_max(float m, float v) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(m), "f"(v));
  return r;
}

// A tile plus its received halo strips, addressed in UNPADDED tile coordinates: h in
// [-hh, H+hh), w in [-hw, W+hw).  Anything not covered by the tile or a non-NULL strip reads
// as 0 -- this is ZeroPad2d + copy_halo_exchange_values (reference spatial.py:1020,405-413)
// without ever materialising the padded tensor.
struct TileView {
  const void* x;
  const void* strip[9];
  int N, C, H, W;
  int hh, hw;  // halo strip extents
};

template <typename T>
__device__ __forceinline__ float tile_load(const TileView& v, int n, int c, int h, int w) {
  const bool hin = (unsigned)h < (unsigned)v.H;
  const bool win = (unsigned)w < (unsigned)v.W;
  if (hin && win) {
    if (v.x == nullptr) return 0.f;  // halo-only view (used for linear boundary corrections)
    return to_f32<T>(reinterpret_cast<const T*>(v.x)[(((size_t)n * v.C + c) * v.H + h) * v.W + w]);
  }
  const int dr = h < 0 ? 0 : (hin ? 1 : 2);
  const int dc = w < 0 ? 0 : (win ? 1 : 2);
  const T* s = reinterpret_cast<const T*>(v.strip[dr * 3 + dc]);
  if (s == nullptr) return 0.f;
  const int sh = (dr == 1) ? v.H : v.hh;
  const int sw = (dc == 1) ? v.W : v.hw;
  const int y = (dr == 0) ? h + v.hh : (dr == 2 ? h - v.H : h);
  const int xx = (dc == 0) ? w + v.hw : (dc == 2 ? w - v.W : w);
  if ((unsigned)y >= (unsigned)sh || (unsigned)xx >= (unsigned)sw) return 0.f;
  return to_f32<T>(s[(((size_t)n * v.C + c) * sh + y) * sw + xx]);
}

// Address of element (n,c,h,w) of the tile-or-halo view, or nullptr where the view reads as zero.
// Splitting the address computation from the load lets callers batch several independent loads.
template <typename T>
__device__ __forceinline__ const T* tile_ptr(const TileView& v, int n, int c, int h, int w) {
  const bool hin = (unsigned)h < (unsigned)v.H;
  const bool win = (unsigned)w < (unsigned)v.W;
  if (hin && win) {
    if (v.x == nullptr) return nullptr;
    return reinterpret_cast<const T*>(v.x) + (((size_t)n * v.C + c) * v.H + h) * v.W + w;
  }
  const int dr = h < 0 ? 0 : (hin ? 1 : 2);
  const int dc = w < 0 ? 0 : (win ? 1 : 2);
  const T* s = reinterpret_cast<const T*>(v.strip[dr * 3 + dc]);
  if (s == nullptr) return nullptr;
  const int sh = (dr == 1) ? v.H : v.hh;
  const int sw = (dc == 1) ? v.W : v.hw;
  const int y = (dr == 0) ? h + v.hh : (dr == 2 ? h - v.H : h);
  const int xx = (dc == 0) ? w + v.hw : (dc == 2 ? w - v.W : w);
  if ((unsigned)y >= (unsigned)sh || (unsigned)xx >= (unsigned)sw) return nullptr;
  return s + (((size_t)n * v.C + c) * sh + y) * sw + xx;
}

inline TileView make_view(const void* x, const spc_halo* halo, int N, int C, int H, int W, int hh, int hw) {
  TileView v;
  v.x = x;
  for (int i = 0; i < 9; ++i) v.strip[i] = halo ? halo->strip[i] : nullptr;
  v.strip[4] = nullptr;
  v.N = N; v.C = C; v.H = H; v.W = W; v.hh = hh; v.hw = hw;
  return v;
}

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
inline int round_up(int a, int b) { return (a + b - 1) / b * b; }
inline size_t align1k(size_t b) { return (b + 1023) & ~(size_t)1023; }
inline size_t al256(size_t b) { return (b + 255) & ~(size_t)255; }
inline size_t dtype_size(int dt) { return dt == SPC_BF16 ? 2 : 4; }
inline bool is_s2(const spc_conv_desc* d) { return d->stride_h == 2 && d->stride_w == 2; }

// ---- host.cu ------------------------------------------------------------------------------------------------------
int sm_count();   // SMs of the current device, cached; 132 (the H100 SXM's) when no device answers
// Opt kernel in to `bytes` of dynamic shared memory.  Remembered per kernel address: every instantiation of a kernel
// template is a kernel of its own and needs its own opt-in.
int allow_dynamic_smem(const void* kernel, int bytes);

// ---- deterministic wgrad (spc_conv2d_wgrad_deterministic): wgrad_reduce.cu ------------------------------------------
// Every wgrad kernel flushes its partial sums with fp32 atomics.  Its work is cut into slices (a pixel-range split, an
// (image, strip, row range), a CTA column, a bias chunk) within which no two adds land on the same element of dw.  A
// launch covers slices [split0, split0 + nsplit) and adds slice s into dw + (s - split0) * slice_stride.  The default
// path launches all slices with stride 0: everything lands in dw, in the order the CTAs finish.  The deterministic path
// gives each slice its own zeroed copy (0 + v == v exactly) and sums the copies into dw in slice order.
struct WgradSlices {
  float* buf;      // slice copies, 256-byte aligned
  size_t elems;    // capacity in floats
};
// dw[i] = (((dw[i] + buf[0][i]) + buf[1][i]) + ... + buf[n-1][i]), buf[j] = buf + j * wn
int reduce_slices(float* dw, const float* buf, int n, size_t wn, cudaStream_t st);
// Run launch(split0, nsplit, dst, slice_stride) over slices [0, slices) of a gradient of wn floats at dw.  sl == nullptr:
// one launch of every slice straight into dw.  Otherwise passes of as many slices as sl->buf holds, each summed into dw
// before the next; a pass of one slice adds straight into dw.  The sum is one left-to-right chain, so the bits do not
// depend on the pass size.
template <class Launch>
int run_slices(const WgradSlices* sl, int slices, size_t wn, float* dw, cudaStream_t st, Launch&& launch) {
  if (!sl) return launch(0, slices, dw, (size_t)0);
  const size_t fit = wn ? sl->elems / wn : 0;
  const int per = fit >= (size_t)slices ? slices : (int)(fit > 0 ? fit : 1);
  for (int s0 = 0; s0 < slices; s0 += per) {
    const int n = slices - s0 < per ? slices - s0 : per;
    if (n == 1) {
      const int rc = launch(s0, 1, dw, (size_t)0);
      if (rc) return rc;
      continue;
    }
    SPC_CHECK_CUDA(cudaMemsetAsync(sl->buf, 0, (size_t)n * wn * sizeof(float), st));
    int rc = launch(s0, n, sl->buf, wn);
    if (rc) return rc;
    rc = reduce_slices(dw, sl->buf, n, wn, st);
    if (rc) return rc;
  }
  return SPC_OK;
}

// ---- direct (CUDA-core) kernels: conv_direct.cu ----------------------------------------
// Generalised correlation: y[n,k, oy0+i*oys, ox0+j*oxs] = bias[k] + sum_{c,r,s}
//   w[w_off + k*wKs + c*wCs + r*wRs + s*wSs] * in(n, c, i*sh + r - pt, j*sw + s - pl)
// The affine weight view lets fprop, dgrad (transposed + flipped filter) and the stride-2
// dgrad parity classes share one kernel without repacking weights.
struct DirectConvParams {
  TileView in;
  const void* w;
  const void* bias;
  void* y;
  int K, R, S, sh, sw, pt, pl;
  int Ho, Wo;                       // logical output extent of this launch
  int YH, YW, oy0, ox0, oys, oxs;   // physical output tensor and mapping
  long long w_off, wKs, wCs, wRs, wSs;
  int vert;                         // 1: CTA tile is 128 rows x 8 cols (thin column strips) instead of 8 x 128
};
int launch_conv_direct(const DirectConvParams& p, int dtype, cudaStream_t st);

struct DirectWgradParams {
  TileView in;        // x + halos
  const void* dy;     // [N][K][Ho][Wo]
  float* dw;          // [K][C][R][S] fp32, accumulated with atomics (zeroed by caller)
  int K, R, S, sh, sw, ph, pw, Ho, Wo;
  int ry0, rx0, rH, rW;   // output sub-rectangle to reduce over (rH == 0: the whole output)
  int split0;             // slice (CTA column) of blockIdx.x == 0; slice s adds into dw + (s - split0) * slice_stride
  size_t slice_stride;
};
int launch_wgrad_direct(const DirectWgradParams& p, int dtype, cudaStream_t st, const WgradSlices* sl = nullptr);
int launch_bias_grad(const void* dy, float* db, int N, int K, int HW, int dtype, int accumulate, cudaStream_t st,
                     const WgradSlices* sl = nullptr);
// The most slice-copy floats one launch_wgrad_direct of d over an output rectangle of rH x rW can need: its CTA columns
// times the gradient's size
double direct_wgrad_slice_floats(const spc_conv_desc* d, int rH, int rW);

// ---- halo fix-up as a small GEMM over the boundary outputs only (halo.cu kernels, api.cu orchestration) ----------
void* boundary_scratch(size_t bytes);   // grow-only device scratch of the fix-up's operands
// The boundary outputs of a tile (those whose window reaches a received strip) are listed as <= 4 disjoint output
// rectangles; P_b = their pixel count (x N), padded to a multiple of 64.
struct BoundaryRects {
  int n;                       // rectangles in use
  int y0[4], y1[4], x0[4], x1[4];
  int start[5];                // prefix sums of the pixel counts PER IMAGE
  int N, per_image, total;     // images, pixels per image, N * per_image
  int padded;                  // total rounded up to 64
};
// V[(c,r,s)][p] = the pixel the tap (r,s) of boundary output p reads in channel c, through `view`: tile + strips for
// fprop (full windows), the halo-only view for wgrad (0 where the tap stays inside the tile); bf16
int launch_halo_im2col(const TileView& halo_only, const BoundaryRects& b, int R, int S, int sh, int sw, int ph, int pw, void* V,
                       cudaStream_t st);
// G[k][p] = dy[n][k][i][j] at the boundary outputs;  y[n][k][i][j] = O[k][p]
int launch_boundary_gather(const void* dy, const BoundaryRects& b, int K, int Ho, int Wo, void* G, cudaStream_t st);
int launch_boundary_scatter(const void* O, const BoundaryRects& b, int K, int Ho, int Wo, void* y, cudaStream_t st);
size_t tc_pw_workspace_bytes(int M, int Cin);
int tc_pw_fwd(const void* w, int ld, int M, int Cin, const void* x, const void* bias, void* y, int P, void* ws, size_t ws_bytes,
              cudaStream_t st);
int tc_pw_wgrad(const void* x, const void* dy, float* dw, int K, int C, int P, cudaStream_t st,
                const WgradSlices* sl = nullptr);

// ---- wgmma pointwise GEMM path: gemm_tc.cu -----------------------------------------------
bool tc_supported(const spc_conv_desc* d, int op);
size_t tc_workspace_bytes(const spc_conv_desc* d, int op);
int tc_conv_fwd(const spc_conv_desc* d, const void* x, const void* w, const void* bias, void* y,
                void* ws, size_t ws_bytes, cudaStream_t st);
int tc_conv_dgrad(const spc_conv_desc* d, const void* dy, const void* w, void* dx, void* ws,
                  size_t ws_bytes, cudaStream_t st);
int tc_conv_wgrad(const spc_conv_desc* d, const void* x, const void* dy, float* dw, void* ws,
                  size_t ws_bytes, cudaStream_t st, const WgradSlices* sl = nullptr);
// the most slice-copy floats one launch of tc_conv_wgrad can need (an upper bound its planners keep to)
double tc_wgrad_slice_floats(const spc_conv_desc* d);

// ---- bf16 tap convolutions without shifted copies (stride 1, <= 128 channels): conv_tap.cu, wgrad_tap.cu ----------
bool tap_v2_supported(int M, int Cin, int R, int S, int H, int W, int N, int stride);
int run_conv_tap_v2(const __nv_bfloat16* wp, int Mpad, int Cpad, const __nv_bfloat16* x, const __nv_bfloat16* bias,
                    __nv_bfloat16* y, int M, int Cin, int R, int S, int ph, int H, int W, int N, cudaStream_t st);
bool wgrad_tap_supported(int K, int C, int R, int S, int H, int W, int stride);
int run_wgrad_tap(const __nv_bfloat16* x, const __nv_bfloat16* dy, float* dw, int K, int C, int N, int H, int W, int R, int S,
                  cudaStream_t st, const WgradSlices* sl);

// ---- fp32 1x1 convolutions on TF32 wgmma (SPC_ALGO_TF32): gemm_tf32.cu ---------------------------------------------
bool tf32_supported(const spc_conv_desc* d);
size_t tf32_workspace_bytes(const spc_conv_desc* d, int op);
int tf32_conv_fwd(const spc_conv_desc* d, const void* x, const void* w, const void* bias, void* y, void* ws,
                  size_t ws_bytes, cudaStream_t st);
int tf32_conv_dgrad(const spc_conv_desc* d, const void* dy, const void* w, void* dx, void* ws, size_t ws_bytes,
                    cudaStream_t st);
int tf32_conv_wgrad(const spc_conv_desc* d, const void* x, const void* dy, float* dw, void* ws, size_t ws_bytes,
                    cudaStream_t st, const WgradSlices* sl = nullptr);
// the most slice-copy floats one launch of tf32_conv_wgrad can need
double tf32_wgrad_slice_floats(const spc_conv_desc* d);

// ---- fp32 stride-1 multi-tap convolutions on TF32 wgmma (SPC_ALGO_TF32_ALL): conv_tap_tf32.cu ----------------------
bool tf32_tap_supported(const spc_conv_desc* d);
size_t tf32_tap_workspace_bytes(const spc_conv_desc* d, int op);
int tf32_tap_fwd(const spc_conv_desc* d, const void* x, const void* w, const void* bias, void* y, void* ws,
                 size_t ws_bytes, cudaStream_t st);
int tf32_tap_dgrad(const spc_conv_desc* d, const void* dy, const void* w, void* dx, void* ws, size_t ws_bytes,
                   cudaStream_t st);
// the interior's share of dw (zero padding), added with atomics; api.cu adds the halo strips' share
int tf32_tap_wgrad(const spc_conv_desc* d, const void* x, const void* dy, float* dw, void* ws, size_t ws_bytes,
                   cudaStream_t st, const WgradSlices* sl = nullptr);
// the most slice-copy floats one launch of tf32_tap_wgrad or tf32_tap_s2_wgrad can need, and one of the direct kernel
// over a boundary rectangle that adds the strips' share
double tf32_tap_wgrad_slice_floats(const spc_conv_desc* d);

// ---- fp32 stride-2 multi-tap convolutions on TF32 wgmma (SPC_ALGO_TF32_STRIDED): conv_tap_s2_tf32.cu ---------------
bool tf32_tap_s2_supported(const spc_conv_desc* d);
size_t tf32_tap_s2_workspace_bytes(const spc_conv_desc* d, int op);
int tf32_tap_s2_fwd(const spc_conv_desc* d, const void* x, const void* w, const void* bias, void* y, void* ws,
                    size_t ws_bytes, cudaStream_t st);
int tf32_tap_s2_dgrad(const spc_conv_desc* d, const void* dy, const void* w, void* dx, void* ws, size_t ws_bytes,
                      cudaStream_t st);
// the interior's share of dw (zero padding), added with atomics; api.cu adds the halo strips' share
int tf32_tap_s2_wgrad(const spc_conv_desc* d, const void* x, const void* dy, float* dw, void* ws, size_t ws_bytes,
                      cudaStream_t st, const WgradSlices* sl = nullptr);

}  // namespace spc
