// api.cu -- C-ABI entry points for convolution (include/spconv.h) and algorithm dispatch.
//
// Dispatch: shapes the wgmma implicit-GEMM path supports (gemm_tc.cu) run there over the
// whole tile with zero padding; if the tile has neighbours, the thin output strips whose
// receptive field reaches into a halo are then recomputed by a small GEMM over just those
// outputs, which reads the received strips in place.  Interior compute therefore never waits on
// the halo exchange -- the overlap the reference left as dead code (spatial.py:415-866).
// fp32 runs there only when the caller opts in: SPC_ALGO_TF32 for its 1x1 layers (gemm_tf32.cu, which have no halo),
// SPC_ALGO_TF32_ALL for those and the stride-1 multi-tap layers (conv_tap_tf32.cu: the interior with zero padding; the
// forward's boundary strips are recomputed on the direct kernel, and wgrad adds the strips' share on it),
// SPC_ALGO_TF32_STRIDED for all of those and the stride-2 multi-tap layers (conv_tap_s2_tf32.cu, the same plan).
// Everything else runs entirely on the direct kernel; when its interior and boundary passes are
// split (spc_conv2d_fwd_interior / _boundary, fp32 or SPC_ALGO_DIRECT), it recomputes the strips.
#include "common.cuh"

namespace spc {
namespace {

int validate(const spc_conv_desc* d) {
  SPC_REQUIRE(d != nullptr, "conv: null descriptor");
  SPC_REQUIRE(d->N >= 0 && d->C > 0 && d->K > 0 && d->H > 0 && d->W > 0, "conv: bad shape N=%d C=%d K=%d H=%d W=%d",
              d->N, d->C, d->K, d->H, d->W);
  SPC_REQUIRE(d->R >= 1 && d->S >= 1 && d->stride_h >= 1 && d->stride_w >= 1, "conv: bad filter/stride");
  // reference spatial.py:115-121: halo_len = (k-1)/2 must equal the conv padding ("same")
  SPC_REQUIRE(d->pad_h == (d->R - 1) / 2 && d->pad_w == (d->S - 1) / 2,
              "conv: Spatial not supported yet for this configuration (pad (%d,%d) != ((R-1)/2,(S-1)/2) for %dx%d)",
              d->pad_h, d->pad_w, d->R, d->S);
  SPC_REQUIRE(d->dtype == SPC_F32 || d->dtype == SPC_BF16, "conv: bad dtype %d", d->dtype);
  SPC_REQUIRE(d->pad_h <= d->H && d->pad_w <= d->W, "conv: halo larger than the tile");
  return SPC_OK;
}

bool has_halo(const spc_halo* h) {
  if (!h) return false;
  for (int i = 0; i < 9; ++i)
    if (i != 4 && h->strip[i]) return true;
  return false;
}

DirectConvParams fwd_params(const spc_conv_desc* d, const void* x, const spc_halo* halo, const void* w,
                            const void* bias, void* y) {
  DirectConvParams p{};
  p.in = make_view(x, halo, d->N, d->C, d->H, d->W, d->pad_h, d->pad_w);
  p.w = w; p.bias = bias; p.y = y;
  p.K = d->K; p.R = d->R; p.S = d->S; p.sh = d->stride_h; p.sw = d->stride_w;
  p.pt = d->pad_h; p.pl = d->pad_w;
  spc_conv_out_shape(d, &p.Ho, &p.Wo);
  p.YH = p.Ho; p.YW = p.Wo; p.oy0 = 0; p.ox0 = 0; p.oys = 1; p.oxs = 1;
  p.w_off = 0; p.wKs = (long long)d->C * d->R * d->S; p.wCs = (long long)d->R * d->S; p.wRs = d->S; p.wSs = 1;
  return p;
}

// The kernel family that runs op (0 fprop, 1 dgrad, 2 wgrad) of d; every entry point below switches on it.
enum class ConvPath { Direct, Bf16, Tf32Pw, Tf32Tap, Tf32TapS2 };

ConvPath conv_path(const spc_conv_desc* d, int op) {
  if (d->algo == SPC_ALGO_DIRECT) return ConvPath::Direct;
  // fp32 storage reaches the tensor cores only when the caller opts in to TF32 (gemm_tf32.cu, conv_tap_tf32.cu,
  // conv_tap_s2_tf32.cu)
  if (d->dtype == SPC_F32) {
    if (d->algo != SPC_ALGO_TF32 && d->algo != SPC_ALGO_TF32_ALL && d->algo != SPC_ALGO_TF32_STRIDED)
      return ConvPath::Direct;
    if (tf32_supported(d)) return ConvPath::Tf32Pw;
    if (d->algo != SPC_ALGO_TF32 && tf32_tap_supported(d)) return ConvPath::Tf32Tap;
    if (d->algo == SPC_ALGO_TF32_STRIDED && tf32_tap_s2_supported(d)) return ConvPath::Tf32TapS2;
    return ConvPath::Direct;
  }
  return tc_supported(d, op) ? ConvPath::Bf16 : ConvPath::Direct;
}

// conv_path, or SPC_EUNSUPPORTED when the caller asked for the tensor cores (SPC_ALGO_TCGEN05) and op has none
int checked_path(const spc_conv_desc* d, int op, ConvPath* path) {
  *path = conv_path(d, op);
  if (d->algo == SPC_ALGO_TCGEN05 && *path == ConvPath::Direct) {
    static const char* const name[3] = {"conv_fwd", "conv_dgrad", "conv_wgrad"};
    set_error("%s: SPC_ALGO_TCGEN05 requested but the shape is not supported by the tensor-core path", name[op]);
    return SPC_EUNSUPPORTED;
  }
  return SPC_OK;
}

// ---- halo fix-up of the tensor-core paths: a small GEMM over the boundary outputs only ------------------------------
// After the interior pass ran the whole tile with zero padding, only the outputs whose window reaches a received
// strip are wrong (P_b of them: a few rows / columns).  fprop: V[(c,r,s)][p] = im2col of tile + strips over those
// P_b outputs, then ONE pointwise GEMM  O[K][P_b] = w[K][C*R*S] * V (+bias)  on the wgmma kernel -- the filter tensor
// IS that matrix -- and a scatter that overwrites them.  wgrad: the halo pixels' share is linear, so with V taken
// from the HALO-ONLY view  dW[K][C*R*S] += dY_b[K][P_b] * V^T  (pw_wgrad_kernel accumulating straight into dw).
static bool boundary_rects(const spc_conv_desc* d, const spc_halo* halo, int Ho, int Wo, BoundaryRects* b) {
  const int top = min(Ho, ceil_div(d->pad_h, d->stride_h));
  int bot0 = ceil_div(d->H + d->pad_h - d->R + 1, d->stride_h);      // first output row touching the bottom halo
  bot0 = max(top, min(Ho, bot0));
  const int left = min(Wo, ceil_div(d->pad_w, d->stride_w));
  int right0 = ceil_div(d->W + d->pad_w - d->S + 1, d->stride_w);
  right0 = max(left, min(Wo, right0));
  const bool any_top = halo->strip[0] || halo->strip[1] || halo->strip[2];
  const bool any_bot = halo->strip[6] || halo->strip[7] || halo->strip[8];
  const bool any_left = halo->strip[0] || halo->strip[3] || halo->strip[6];
  const bool any_right = halo->strip[2] || halo->strip[5] || halo->strip[8];
  const int sy0 = any_top ? top : 0, sy1 = any_bot ? bot0 : Ho;       // rows not already covered by the bands
  int n = 0, acc = 0;
  auto add = [&](int y0, int y1, int x0, int x1) {
    if (y1 <= y0 || x1 <= x0) return;
    b->y0[n] = y0; b->y1[n] = y1; b->x0[n] = x0; b->x1[n] = x1;
    b->start[n] = acc;
    acc += (y1 - y0) * (x1 - x0);
    ++n;
  };
  if (any_top) add(0, top, 0, Wo);
  if (any_bot) add(bot0, Ho, 0, Wo);
  if (any_left) add(sy0, sy1, 0, left);
  if (any_right) add(sy0, sy1, right0, Wo);
  for (int i = n; i < 5; ++i) b->start[i] = acc;
  for (int i = n; i < 4; ++i) { b->y0[i] = b->y1[i] = b->x0[i] = 0; b->x1[i] = 1; }
  b->n = n; b->N = d->N; b->per_image = acc; b->total = acc * d->N;
  b->padded = (b->total + 63) & ~63;
  return b->total > 0;
}

static int boundary_fwd_tc(const spc_conv_desc* d, const void* x, const spc_halo* halo, const void* w, const void* bias,
                           void* y, cudaStream_t st) {
  int Ho, Wo;
  spc_conv_out_shape(d, &Ho, &Wo);
  BoundaryRects b;
  if (!boundary_rects(d, halo, Ho, Wo, &b)) return SPC_OK;
  const int CT = d->C * d->R * d->S;
  const size_t vbytes = al256((size_t)CT * b.padded * 2), obytes = al256((size_t)d->K * b.padded * 2);
  const size_t wsb = tc_pw_workspace_bytes(d->K, CT);
  char* base = (char*)boundary_scratch(vbytes + obytes + wsb + 2048);
  SPC_REQUIRE(base != nullptr, "boundary scratch allocation failed");
  void* V = base; void* O = base + vbytes; void* ws = base + vbytes + obytes;
  // fprop gathers the FULL windows (tile + strips) of the boundary outputs and overwrites them: the result is rounded
  // to bf16 once, like every other output (adding a halo-only correction to the already rounded interior value
  // rounds twice -- 335 of 4.4e8 stem outputs left the parity tolerance that way)
  TileView v = make_view(x, halo, d->N, d->C, d->H, d->W, d->pad_h, d->pad_w);
  int rc = launch_halo_im2col(v, b, d->R, d->S, d->stride_h, d->stride_w, d->pad_h, d->pad_w, V, st);
  if (rc) return rc;
  rc = tc_pw_fwd(w, CT, d->K, CT, V, bias, O, b.padded, ws, wsb, st);
  if (rc) return rc;
  return launch_boundary_scatter(O, b, d->K, Ho, Wo, y, st);
}

static int boundary_wgrad_tc(const spc_conv_desc* d, const spc_halo* halo, const void* dy, float* dw, cudaStream_t st,
                             const WgradSlices* sl) {
  int Ho, Wo;
  spc_conv_out_shape(d, &Ho, &Wo);
  BoundaryRects b;
  if (!boundary_rects(d, halo, Ho, Wo, &b)) return SPC_OK;
  const int CT = d->C * d->R * d->S;
  const size_t vbytes = al256((size_t)CT * b.padded * 2), gbytes = al256((size_t)d->K * b.padded * 2);
  char* base = (char*)boundary_scratch(vbytes + gbytes + 2048);
  SPC_REQUIRE(base != nullptr, "boundary scratch allocation failed");
  void* V = base; void* G = base + vbytes;
  TileView v = make_view(nullptr, halo, d->N, d->C, d->H, d->W, d->pad_h, d->pad_w);
  int rc = launch_halo_im2col(v, b, d->R, d->S, d->stride_h, d->stride_w, d->pad_h, d->pad_w, V, st);
  if (rc) return rc;
  rc = launch_boundary_gather(dy, b, d->K, Ho, Wo, G, st);
  if (rc) return rc;
  return tc_pw_wgrad(V, G, dw, d->K, CT, b.padded, st, sl);   // dw[k][(c,r,s)] += sum_p G[k][p] * V[(c,r,s)][p]
}

// Launch the direct kernel on the output sub-rectangle [y0,y1) x [x0,x1).
int fwd_rect(DirectConvParams p, int dtype, int y0, int y1, int x0, int x1, cudaStream_t st) {
  if (y1 <= y0 || x1 <= x0) return SPC_OK;
  p.oy0 = y0; p.ox0 = x0;
  p.pt -= y0 * p.sh; p.pl -= x0 * p.sw;
  p.Ho = y1 - y0; p.Wo = x1 - x0;
  p.vert = (p.Wo <= 16 && p.Ho > p.Wo) ? 1 : 0;   // thin column strip: 128-row x 8-col CTA tiles
  return launch_conv_direct(p, dtype, st);
}

}  // namespace
}  // namespace spc

using namespace spc;

extern "C" {

void spc_conv_out_shape(const spc_conv_desc* d, int* Ho, int* Wo) {
  if (Ho) *Ho = (d->H + 2 * d->pad_h - d->R) / d->stride_h + 1;
  if (Wo) *Wo = (d->W + 2 * d->pad_w - d->S) / d->stride_w + 1;
}

int spc_conv_uses_tcgen05(const spc_conv_desc* d, int op) { return d && conv_path(d, op) != ConvPath::Direct; }

// Slice copies of the deterministic wgrad: the most slices one launch of this shape's wgrad can have, times the
// gradient's size (each kernel family bounds its own), capped at SPC_WGRAD_SLICE_BYTES_MAX (larger launches run in
// passes, with the same bits); bias: <= 64 chunks of K.
static size_t wgrad_slice_bytes(const spc_conv_desc* d) {
  double need = 64.0 * d->K;
  switch (conv_path(d, 2)) {
    case ConvPath::Direct: {
      int Ho, Wo;
      spc_conv_out_shape(d, &Ho, &Wo);
      need = fmax(need, direct_wgrad_slice_floats(d, Ho, Wo));
      break;
    }
    case ConvPath::Bf16: need = fmax(need, tc_wgrad_slice_floats(d)); break;
    case ConvPath::Tf32Pw: need = fmax(need, tf32_wgrad_slice_floats(d)); break;
    case ConvPath::Tf32Tap:
    case ConvPath::Tf32TapS2: need = fmax(need, tf32_tap_wgrad_slice_floats(d)); break;
  }
  return (size_t)fmin(need * sizeof(float), (double)SPC_WGRAD_SLICE_BYTES_MAX);
}

size_t spc_conv_workspace_bytes(const spc_conv_desc* d, int op) {
  if (!d) return 0;
  if (op == 3) return validate(d) ? 0 : al256(spc_conv_workspace_bytes(d, 2)) + al256(wgrad_slice_bytes(d));
  switch (conv_path(d, op)) {
    case ConvPath::Direct: return 0;
    case ConvPath::Bf16: return tc_workspace_bytes(d, op);
    case ConvPath::Tf32Pw: return tf32_workspace_bytes(d, op);
    case ConvPath::Tf32Tap: return tf32_tap_workspace_bytes(d, op);
    case ConvPath::Tf32TapS2: return tf32_tap_s2_workspace_bytes(d, op);
  }
  return 0;
}

// Boundary strips: output rows / columns whose window reaches outside the tile, recomputed from
// tile + received halo strips.  Valid after ANY interior pass that used zero padding.
static int fwd_boundary(const spc_conv_desc* d, DirectConvParams p, const spc_halo* halo, cudaStream_t st) {
  if (!has_halo(halo)) return SPC_OK;
  if (d->dtype == SPC_BF16 && d->algo != SPC_ALGO_DIRECT) return boundary_fwd_tc(d, p.in.x, halo, p.w, p.bias, p.y, st);
  // fp32 and SPC_ALGO_DIRECT: the direct kernel on each boundary rectangle
  BoundaryRects b;
  if (!boundary_rects(d, halo, p.Ho, p.Wo, &b)) return SPC_OK;
  for (int i = 0; i < b.n; ++i) {
    const int rc = fwd_rect(p, d->dtype, b.y0[i], b.y1[i], b.x0[i], b.x1[i], st);
    if (rc) return rc;
  }
  return SPC_OK;
}

static int fwd_interior(const spc_conv_desc* d, ConvPath path, const void* x, const void* w, const void* bias, void* y,
                        void* ws, size_t ws_bytes, cudaStream_t st) {
  switch (path) {
    case ConvPath::Direct: break;
    case ConvPath::Bf16: return tc_conv_fwd(d, x, w, bias, y, ws, ws_bytes, st);
    case ConvPath::Tf32Pw: return tf32_conv_fwd(d, x, w, bias, y, ws, ws_bytes, st);
    case ConvPath::Tf32Tap: return tf32_tap_fwd(d, x, w, bias, y, ws, ws_bytes, st);
    case ConvPath::Tf32TapS2: return tf32_tap_s2_fwd(d, x, w, bias, y, ws, ws_bytes, st);
  }
  return launch_conv_direct(fwd_params(d, x, nullptr, w, bias, y), d->dtype, st);
}

int spc_conv2d_fwd(const spc_conv_desc* d, const void* x, const spc_halo* halo, const void* w, const void* bias,
                   void* y, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = validate(d);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (d->N == 0) return SPC_OK;
  SPC_REQUIRE(x && w && y, "conv_fwd: null tensor pointer");
  ConvPath path;
  rc = checked_path(d, 0, &path);
  if (rc) return rc;
  if (path == ConvPath::Direct)   // direct kernel reads tile + strips in one pass
    return launch_conv_direct(fwd_params(d, x, halo, w, bias, y), d->dtype, st);
  rc = fwd_interior(d, path, x, w, bias, y, workspace, workspace_bytes, st);
  if (rc) return rc;
  return fwd_boundary(d, fwd_params(d, x, halo, w, bias, y), halo, st);
}

int spc_conv2d_fwd_interior(const spc_conv_desc* d, const void* x, const void* w, const void* bias, void* y,
                            void* workspace, size_t workspace_bytes, void* stream) {
  int rc = validate(d);
  if (rc) return rc;
  if (d->N == 0) return SPC_OK;
  SPC_REQUIRE(x && w && y, "conv_fwd_interior: null tensor pointer");
  ConvPath path;
  rc = checked_path(d, 0, &path);
  if (rc) return rc;
  return fwd_interior(d, path, x, w, bias, y, workspace, workspace_bytes, (cudaStream_t)stream);
}

int spc_conv2d_fwd_boundary(const spc_conv_desc* d, const void* x, const spc_halo* halo, const void* w,
                            const void* bias, void* y, void* stream) {
  int rc = validate(d);
  if (rc) return rc;
  if (d->N == 0) return SPC_OK;
  SPC_REQUIRE(x && w && y, "conv_fwd_boundary: null tensor pointer");
  return fwd_boundary(d, fwd_params(d, x, halo, w, bias, y), halo, (cudaStream_t)stream);
}

int spc_conv2d_dgrad(const spc_conv_desc* d, const void* dy, const void* w, void* dx, void* workspace,
                     size_t workspace_bytes, void* stream) {
  int rc = validate(d);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (d->N == 0) return SPC_OK;
  SPC_REQUIRE(dy && w && dx, "conv_dgrad: null tensor pointer");
  ConvPath path;
  rc = checked_path(d, 1, &path);
  if (rc) return rc;
  switch (path) {
    case ConvPath::Direct: break;
    case ConvPath::Bf16: return tc_conv_dgrad(d, dy, w, dx, workspace, workspace_bytes, st);
    case ConvPath::Tf32Pw: return tf32_conv_dgrad(d, dy, w, dx, workspace, workspace_bytes, st);
    case ConvPath::Tf32Tap: return tf32_tap_dgrad(d, dy, w, dx, workspace, workspace_bytes, st);
    case ConvPath::Tf32TapS2: return tf32_tap_s2_dgrad(d, dy, w, dx, workspace, workspace_bytes, st);
  }

  int Ho, Wo;
  spc_conv_out_shape(d, &Ho, &Wo);
  const int sh = d->stride_h, sw = d->stride_w, R = d->R, S = d->S;
  // Decompose by output parity class (a,b): each class is a stride-1 correlation of dy with a
  // flipped sub-filter (taps r = r_a + sh*t), written with output stride (sh,sw).
  bool need_zero = false;
  for (int a = 0; a < sh; ++a) if ((a + d->pad_h) % sh >= R) need_zero = true;
  for (int b = 0; b < sw; ++b) if ((b + d->pad_w) % sw >= S) need_zero = true;
  // rows/cols of dx beyond the reach of any output window are also zero; simplest: clear first
  if (need_zero || (Ho - 1) * sh + R - d->pad_h < d->H || (Wo - 1) * sw + S - d->pad_w < d->W)
    SPC_CHECK_CUDA(cudaMemsetAsync(dx, 0, (size_t)d->N * d->C * d->H * d->W * dtype_size(d->dtype), st));
  for (int a = 0; a < sh; ++a) {
    const int ra = (a + d->pad_h) % sh;
    if (ra >= R) continue;
    const int Ta = (R - ra + sh - 1) / sh;
    const int qa = (a + d->pad_h - ra) / sh;
    for (int b = 0; b < sw; ++b) {
      const int sb = (b + d->pad_w) % sw;
      if (sb >= S) continue;
      const int Tb = (S - sb + sw - 1) / sw;
      const int qb = (b + d->pad_w - sb) / sw;
      DirectConvParams p{};
      p.in = make_view(dy, nullptr, d->N, d->K, Ho, Wo, 0, 0);
      p.w = w; p.bias = nullptr; p.y = dx;
      p.K = d->C; p.R = Ta; p.S = Tb; p.sh = 1; p.sw = 1;
      p.pt = (Ta - 1) - qa; p.pl = (Tb - 1) - qb;
      p.Ho = (d->H - a + sh - 1) / sh; p.Wo = (d->W - b + sw - 1) / sw;
      p.YH = d->H; p.YW = d->W; p.oy0 = a; p.ox0 = b; p.oys = sh; p.oxs = sw;
      p.w_off = (long long)(ra + sh * (Ta - 1)) * S + (sb + sw * (Tb - 1));
      p.wKs = (long long)R * S;               // output channel of this launch = c
      p.wCs = (long long)d->C * R * S;        // input channel of this launch = k
      p.wRs = -(long long)sh * S; p.wSs = -(long long)sw;
      rc = launch_conv_direct(p, d->dtype, st);
      if (rc) return rc;
    }
  }
  return SPC_OK;
}

// The halo pixels' share of dw (exact by linearity) after an interior pass with zero padding: the direct kernel over the
// outputs whose windows reach a strip, reading the strips through the halo-only view (zero inside the tile)
static int wgrad_boundary_direct(const spc_conv_desc* d, const spc_halo* halo, const void* dy, float* dw, int Ho, int Wo,
                                 cudaStream_t st, const WgradSlices* sl) {
  BoundaryRects b;
  if (!has_halo(halo) || !boundary_rects(d, halo, Ho, Wo, &b)) return SPC_OK;
  for (int i = 0; i < b.n; ++i) {
    DirectWgradParams q{};
    q.in = make_view(nullptr, halo, d->N, d->C, d->H, d->W, d->pad_h, d->pad_w);
    q.dy = dy; q.dw = dw;
    q.K = d->K; q.R = d->R; q.S = d->S; q.sh = d->stride_h; q.sw = d->stride_w; q.ph = d->pad_h; q.pw = d->pad_w;
    q.Ho = Ho; q.Wo = Wo;
    q.ry0 = b.y0[i]; q.rx0 = b.x0[i]; q.rH = b.y1[i] - b.y0[i]; q.rW = b.x1[i] - b.x0[i];
    const int rc = launch_wgrad_direct(q, SPC_F32, st, sl);
    if (rc) return rc;
  }
  return SPC_OK;
}

// sl == nullptr: every kernel adds straight into dw / db; else through slice copies summed in order (common.cuh)
static int wgrad(const spc_conv_desc* d, const void* x, const spc_halo* halo, const void* dy, float* dw, float* db,
                 int accumulate, void* workspace, size_t workspace_bytes, cudaStream_t st, const WgradSlices* sl) {
  int rc = SPC_OK;
  int Ho, Wo;
  spc_conv_out_shape(d, &Ho, &Wo);
  const size_t wn = (size_t)d->K * d->C * d->R * d->S;
  if (!accumulate) SPC_CHECK_CUDA(cudaMemsetAsync(dw, 0, wn * sizeof(float), st));
  if (d->N == 0) {
    if (db && !accumulate) SPC_CHECK_CUDA(cudaMemsetAsync(db, 0, sizeof(float) * d->K, st));
    return SPC_OK;
  }
  ConvPath path;
  rc = checked_path(d, 2, &path);
  if (rc) return rc;
  switch (path) {
    case ConvPath::Direct: {
      DirectWgradParams p{};
      p.in = make_view(x, halo, d->N, d->C, d->H, d->W, d->pad_h, d->pad_w);
      p.dy = dy; p.dw = dw;
      p.K = d->K; p.R = d->R; p.S = d->S; p.sh = d->stride_h; p.sw = d->stride_w; p.ph = d->pad_h; p.pw = d->pad_w;
      p.Ho = Ho; p.Wo = Wo;
      rc = launch_wgrad_direct(p, d->dtype, st, sl);
      break;
    }
    case ConvPath::Bf16:
      rc = tc_conv_wgrad(d, x, dy, dw, workspace, workspace_bytes, st, sl);
      // add the halo pixels' contribution (exact by linearity): boundary GEMM over the outputs whose windows reach a
      // strip
      if (!rc && has_halo(halo)) rc = boundary_wgrad_tc(d, halo, dy, dw, st, sl);
      break;
    case ConvPath::Tf32Pw:   // 1x1: no output window reaches a halo strip, so there is nothing to add for the strips
      rc = tf32_conv_wgrad(d, x, dy, dw, workspace, workspace_bytes, st, sl);
      break;
    case ConvPath::Tf32Tap:
    case ConvPath::Tf32TapS2:
      rc = path == ConvPath::Tf32Tap ? tf32_tap_wgrad(d, x, dy, dw, workspace, workspace_bytes, st, sl)
                                     : tf32_tap_s2_wgrad(d, x, dy, dw, workspace, workspace_bytes, st, sl);
      if (!rc) rc = wgrad_boundary_direct(d, halo, dy, dw, Ho, Wo, st, sl);
      break;
  }
  if (rc) return rc;
  if (db) return launch_bias_grad(dy, db, d->N, d->K, Ho * Wo, d->dtype, accumulate, st, sl);
  return SPC_OK;
}

int spc_conv2d_wgrad(const spc_conv_desc* d, const void* x, const spc_halo* halo, const void* dy, float* dw,
                     float* db, int accumulate, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = validate(d);
  if (rc) return rc;
  SPC_REQUIRE(dw && (d->N == 0 || (x && dy)), "conv_wgrad: null tensor pointer");
  return wgrad(d, x, halo, dy, dw, db, accumulate, workspace, workspace_bytes, (cudaStream_t)stream, nullptr);
}

int spc_conv2d_wgrad_deterministic(const spc_conv_desc* d, const void* x, const spc_halo* halo, const void* dy, float* dw,
                                   float* db, int accumulate, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = validate(d);
  if (rc) return rc;
  SPC_REQUIRE(dw && (d->N == 0 || (x && dy)), "conv_wgrad_deterministic: null tensor pointer");
  // [0, op 2's workspace): the kernels' own operands; the rest holds slice copies.  Less than op 3's size still works,
  // in more passes with the same bits; none at all adds one slice per launch straight into dw.
  const size_t own = al256(spc_conv_workspace_bytes(d, 2));
  SPC_REQUIRE(workspace_bytes >= own && (own == 0 || workspace),
              "conv_wgrad_deterministic: workspace of %zu bytes, need at least %zu", workspace_bytes, own);
  WgradSlices sl{nullptr, 0};
  if (workspace && workspace_bytes > own) {
    sl.buf = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + own);
    sl.elems = (workspace_bytes - own) / sizeof(float);
  }
  return wgrad(d, x, halo, dy, dw, db, accumulate, workspace, workspace_bytes, (cudaStream_t)stream, &sl);
}

}  // extern "C"
