/*
 * spconv.h -- C ABI of libspconv.so: the H100 (sm_90a) spatial-parallel convolution engine
 * that sits under the torchgems Python API (mpi4dl_b200/torchgems/spatial.py).
 *
 * The reference (OSU-Nowlab/MPI4DL) has NO FFI: its hot path is Python calling
 * torch.nn.Conv2d / nn.AvgPool2d / nn.MaxPool2d / nn.ZeroPad2d and torch.distributed
 * (src/torchgems/spatial.py).  Each entry point below names the reference call site it
 * replaces.  Conventions (SURVEY.md section 8b):
 *   - plain pointers + sizes only; no torch / C++ types cross the boundary;
 *   - every pointer is a DEVICE pointer unless said otherwise; the caller owns all tensors;
 *   - all work is enqueued asynchronously on the given cudaStream_t (passed as void*);
 *   - return 0 on success, a negative SPC_E* code otherwise; spc_last_error() gives text;
 *   - not thread-safe per context (the reference is one host thread per process/GPU).
 *
 * Tensors are NCHW contiguous.  "Tile" = the part of the image owned by this rank
 * (train_spatial.py:241-290).  A tile's halo is delivered as up to 8 packed strips, indexed by
 * the reference's 3x3 neighbour stencil (spatial.py:961-964):   0 1 2 / 3 [4] 5 / 6 7 8
 *   strips 1,7 (top,bottom): [N][C][halo_h][W]     strips 3,5 (left,right): [N][C][H][halo_w]
 *   strips 0,2,6,8 (corners): [N][C][halo_h][halo_w]
 * exactly the message shapes of the reference (spatial.py:311-334 get_shapes_recv).  A NULL
 * strip means "no neighbour there": zeros are used (ZeroPad2d, spatial.py:142-144,1020).
 */
#ifndef SPCONV_H_
#define SPCONV_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SPC_VERSION 102

enum { SPC_OK = 0, SPC_EINVAL = -1, SPC_ECUDA = -2, SPC_EUNSUPPORTED = -3, SPC_ENOMEM = -4 };
enum { SPC_F32 = 0, SPC_BF16 = 1 };             /* storage dtype of x / w / y; accumulation is fp32 */
enum { SPC_POOL_MAX = 0, SPC_POOL_AVG = 1 };
/* SPC_ALGO_TF32: like AUTO, but fp32 storage may use the TF32 tensor cores (fp32 accumulation) where the shape
 * qualifies: 1x1 filters, stride 1 or 2, on the shapes the bf16 1x1 path takes (H*W / stride^2 a multiple of 8;
 * stride 2 also needs even H and W % 32 == 0).  Every other fp32 shape (multi-tap filters, misaligned pixel counts)
 * runs on the direct kernels as with AUTO, and bf16 behaves exactly as with AUTO.  Rounding: fprop and dgrad round
 * both operands (x or dy, and w) to tf32 (10 fraction bits) to nearest; wgrad feeds dy and x to the tensor cores
 * unconverted, which use the top 19 bits of each word, i.e. truncate them.  Products are exact and summed in fp32.
 * Error bound per element, with A = the same operation on |x|, |w|, |dy| (and |b|) in exact arithmetic:
 *   inputs already tf32-representable:  |got - exact| <= 2^-12 A
 *   arbitrary fp32 inputs:              |got - exact| <= (2^-9 + 2^-12) A
 * SPC_ALGO_TF32_ALL: SPC_ALGO_TF32, plus fprop, dgrad and wgrad of the fp32 stride-1 multi-tap filters: odd R x S up to
 * 7 x 7 (3x3, 1x7, 7x1, ...), "same" padding, any N, C, K, H, and W % 4 == 0.  Their 1x1 layers run exactly as with
 * SPC_ALGO_TF32 (same kernels, bit-identical results); every other fp32 shape runs on the direct kernels, and bf16 as
 * with AUTO.  Rounding (fprop / dgrad: both operands to nearest tf32; wgrad: x to nearest, dy truncated) and error
 * bound are those of SPC_ALGO_TF32 above, with A summed over all taps.  With halo strips the interior runs on the
 * tensor cores with zero padding; the forward's outputs whose windows reach a strip are recomputed, and wgrad's share
 * of the strips is added, in fp32 on the direct kernel.
 * SPC_ALGO_TF32_STRIDED: SPC_ALGO_TF32_ALL (same kernels, bit-identical results on the shapes it takes), plus fprop,
 * dgrad and wgrad of the fp32 multi-tap filters with stride_h == stride_w == 2: R and S each 3, 5 or 7, "same" padding,
 * even H, W % 8 == 0, any N, C, K.  dgrad writes all of dx.  1x7 / 7x1 at stride 2, mixed strides and every other fp32
 * shape run on the direct kernels.  Rounding, error bound and the treatment of halo strips are those of
 * SPC_ALGO_TF32_ALL above (dgrad has no halo).
 * SPC_ALGO_TCGEN05 still rejects fp32 (SPC_EUNSUPPORTED). */
enum {
  SPC_ALGO_AUTO = 0, SPC_ALGO_DIRECT = 1, SPC_ALGO_TCGEN05 = 2, SPC_ALGO_TF32 = 3, SPC_ALGO_TF32_ALL = 4,
  SPC_ALGO_TF32_STRIDED = 5
};

/* Geometry of one spatially-partitioned convolution on one tile.
 * Mirrors conv_spatial.__init__ (spatial.py:26-155): padding is "same"
 * (pad_h = (R-1)/2, pad_w = (S-1)/2, :115-121), dilation = 1, groups = 1 (:130-140). */
typedef struct {
  int32_t N, C, H, W;          /* input tile, unpadded */
  int32_t K, R, S;             /* filter [K][C][R][S] */
  int32_t stride_h, stride_w;
  int32_t pad_h, pad_w;        /* == halo_len_height / halo_len_width */
  int32_t dtype;               /* SPC_F32 | SPC_BF16 */
  int32_t algo;                /* SPC_ALGO_*; AUTO picks the tensor-core (wgmma) path when the shape qualifies */
} spc_conv_desc;

typedef struct {
  int32_t N, C, H, W;
  int32_t k, stride, pad;      /* square window; pad == floor((k-1)/2) (spatial.py:1457-1464) */
  int32_t mode;                /* SPC_POOL_MAX | SPC_POOL_AVG */
  int32_t dtype;
} spc_pool_desc;

/* Received halo strips of a tile (device pointers, NULL = zero padding there). */
typedef struct {
  const void* strip[9];
} spc_halo;

/* ---- library / device ------------------------------------------------------------------- */
int         spc_version(void);
const char* spc_last_error(void);
/* sm count, compute capability major*10+minor; fails loudly when the device is not sm_90 */
int         spc_device_info(int device, int* sm_count, int* cc);
/* number of kernels this library has launched since the last reset (bench.py's gpu_launches) */
long long   spc_launch_count(int reset);

/* ---- convolution ------------------------------------------------------------------------ */
/* y = conv(pad+halo(x), w) + bias.   Replaces spatial.py:1019-1029 (ZeroPad2d :1020,
 * copy_halo_exchange_values :405-413, nn.Conv2d.forward :1027).  y: [N][K][Ho][Wo].
 * bias may be NULL.  workspace: spc_conv_workspace_bytes() bytes (may be NULL if 0). */
int spc_conv2d_fwd(const spc_conv_desc* d, const void* x, const spc_halo* halo, const void* w,
                   const void* bias, void* y, void* workspace, size_t workspace_bytes,
                   void* stream);

/* The same convolution in two stream-ordered halves, so that the halo exchange (on a second
 * stream) overlaps the bulk of the compute -- the design the reference left as dead code
 * (spatial.py:415-866 make_tensor_halo_compute / compute_halo_exchange / merge_final_image):
 *   interior: the whole tile with ZERO padding (no halo needed; tensor cores where the shape qualifies);
 *   boundary: recompute the output rows/cols whose window reaches a received strip. */
int spc_conv2d_fwd_interior(const spc_conv_desc* d, const void* x, const void* w, const void* bias,
                            void* y, void* workspace, size_t workspace_bytes, void* stream);
int spc_conv2d_fwd_boundary(const spc_conv_desc* d, const void* x, const spc_halo* halo,
                            const void* w, const void* bias, void* y, void* stream);

/* dx = crop(dgrad(dy, w)) -- autograd of spatial.py:1027 followed by ZeroPad2d backward.
 * Reference semantics (SURVEY 8a N2): received halos are constants, so no gradient is sent
 * back to neighbours; dx gets only this tile's own dy contributions.  dx: [N][C][H][W].
 * The opt-in exact backward adds the neighbours' part with spc_conv2d_dgrad_halo / spc_halo_accumulate below. */
int spc_conv2d_dgrad(const spc_conv_desc* d, const void* dy, const void* w, void* dx,
                     void* workspace, size_t workspace_bytes, void* stream);

/* dw[K][C][R][S] (fp32) and db[K] (fp32, may be NULL) over the padded tile INCLUDING the
 * received halos (autograd of spatial.py:1027 w.r.t. weight/bias).  accumulate != 0 adds
 * into dw/db instead of overwriting. */
int spc_conv2d_wgrad(const spc_conv_desc* d, const void* x, const spc_halo* halo, const void* dy,
                     float* dw, float* db, int accumulate, void* workspace,
                     size_t workspace_bytes, void* stream);

/* spc_conv2d_wgrad with bit-reproducible results: the same arguments, and dw / db are bit-identical whenever x, the
 * strips, dy and (accumulate != 0) the initial dw / db are, on GPUs with the same SM count.  The default wgrad adds its
 * partial sums into dw with fp32 atomics in whatever order the CTAs finish; this one gives each slice of the work (a
 * pixel-range split, an image strip, a CTA column, a bias chunk: units whose adds never meet on one element) a zeroed
 * copy in the workspace and sums the copies into dw in slice order, the halo strips' share after the tile's.  Each
 * element gets as many fp32 roundings as with spc_conv2d_wgrad, so the per-element error bounds stated above for each
 * path (bf16, TF32 1x1 / tap / stride-2, direct) hold unchanged; the bits may differ from spc_conv2d_wgrad's.
 * workspace: spc_conv_workspace_bytes(d, 3) bytes, non-zero on every path.  It exceeds op 2's by at most
 * SPC_WGRAD_SLICE_BYTES_MAX; launches with more slices than fit run in passes, with the same bits.  A smaller workspace,
 * down to op 2's size, is accepted and gives the same bits in more passes.
 * torchgems calls this instead of spc_conv2d_wgrad when torch.are_deterministic_algorithms_enabled(). */
#define SPC_WGRAD_SLICE_BYTES_MAX ((size_t)256 << 20)
int spc_conv2d_wgrad_deterministic(const spc_conv_desc* d, const void* x, const spc_halo* halo, const void* dy,
                                   float* dw, float* db, int accumulate, void* workspace,
                                   size_t workspace_bytes, void* stream);

size_t spc_conv_workspace_bytes(const spc_conv_desc* d,
                                int op /*0 fwd, 1 dgrad, 2 wgrad, 3 spc_conv2d_wgrad_deterministic*/);
/* 1 if the tensor-core (wgmma) kernel will be used for this op, else 0 (direct kernel); the name is historical */
int    spc_conv_uses_tcgen05(const spc_conv_desc* d, int op);
/* output extent of a tile: Ho = (H + 2*pad_h - R)/stride_h + 1 */
void   spc_conv_out_shape(const spc_conv_desc* d, int* Ho, int* Wo);

/* ---- pooling ---------------------------------------------------------------------------- */
/* Replaces Pool.forward (spatial.py:1503-1509): halo_exchange_layer + nn.{Max,Avg}Pool2d with
 * padding=0 on the explicitly zero-padded tile (so avg always divides by k*k and max sees 0 at
 * true image borders). */
int spc_pool2d_fwd(const spc_pool_desc* d, const void* x, const spc_halo* halo, void* y, void* stream);
/* dx = crop(pool backward); max routes to the first maximal element (ATen semantics).
 * NaN follows ATen's max_pool2d too (`v > max || isnan(v)`): a window that holds a NaN pools to NaN in the
 * forward, and its gradient goes to the NaN (the last one in row-major window order if there are several). */
int spc_pool2d_bwd(const spc_pool_desc* d, const void* x, const spc_halo* halo, const void* dy,
                   void* dx, void* stream);

/* ---- fused BatchNorm2d (training mode, per-tile statistics) + ReLU ------------------------ *
 * The cells of the spatial stages chain ReLU -> conv -> nn.BatchNorm2d (models/amoebanet.py:365-398 of the
 * reference) / BatchNorm2d -> ReLU -> conv (resnet_spatial.py:165-180) as separate eager kernels; statistics
 * are over the LOCAL tile only (SURVEY 8a N4).  These four entry points do normalisation + the following ReLU
 * in one HBM pass each way.  y, z, dz, dy: [N][C][H*W] (NCHW, H*W % 8 == 0), dtype SPC_F32 | SPC_BF16, 16-byte aligned;
 * all per-channel vectors are fp32 device arrays of C elements, 4-byte aligned.  A misaligned pointer is SPC_EINVAL.
 *   spc_bn_stats     : mean[c] = sum y / M, var[c] = sum (y - mean)^2 / M (biased), M = N*H*W (replaces the statistics pass)
 *   spc_bn_apply     : z = relu?((y - mean[c]) * rstd[c] * gamma[c] + beta[c])     (BN apply + nn.ReLU)
 *   spc_bn_bwd_reduce: dsum[c] = sum g, dsumx[c] = sum g * xhat, g = dz * [z > 0]  (= dbeta, dgamma)
 *   spc_bn_bwd_apply : dy = gamma * rstd * (g - dsum/M - xhat * dsumx/M)
 * spc_bn_stats and spc_bn_bwd_reduce write one partial per (plane, 16384-element chunk) to `workspace`
 * (spc_bn_workspace_bytes(N, C, HW) bytes, 16-byte aligned) and merge each channel's partials in a fixed order in fp64:
 * no floating-point atomics, every output of the four entry points is bit-reproducible.  Error bounds per channel,
 * against exact arithmetic on the stored y (and the same mean, rstd, gamma, beta for the backward sums):
 *   |mean - exact| <= 2^-23 |exact mean| + 2^-19 mean|y - exact mean|
 *   |var - exact|  <= 2^-16 exact var + 2^-30 mean(y^2)
 *   |dsum - exact| <= 2^-19 sum|g|,   |dsumx - exact| <= 2^-19 sum|g * xhat|
 * (tests/test_bnrelu_bounds.py derives these and the per-element bounds of z and dy). */
size_t spc_bn_workspace_bytes(int N, int C, long long HW);   /* 0 for an invalid shape */
int spc_bn_stats(int N, int C, long long HW, int dtype, const void* y, float* mean, float* var, void* workspace,
                 size_t workspace_bytes, void* stream);
int spc_bn_apply(int N, int C, long long HW, int dtype, const void* y, const float* mean, const float* rstd,
                 const float* gamma, const float* beta, int relu, void* z, void* stream);
int spc_bn_bwd_reduce(int N, int C, long long HW, int dtype, const void* dz, const void* y, const float* mean,
                      const float* rstd, const float* gamma, const float* beta, int relu, float* dsum,
                      float* dsumx, void* workspace, size_t workspace_bytes, void* stream);
int spc_bn_bwd_apply(int N, int C, long long HW, int dtype, const void* dz, const void* y, const float* mean,
                     const float* rstd, const float* gamma, const float* beta, int relu, const float* dsum,
                     const float* dsumx, void* dy, void* stream);

/* ---- halo strips ------------------------------------------------------------------------ */
/* Pack the strips a tile SENDS (spatial.py:336-357: the first/last halo rows/cols inside the
 * tile, .clone()d per direction) into send[d] for every d with send[d] != NULL.  send[d] may be
 * a peer-GPU pointer (CUDA IPC mapping): one kernel writes all strips straight into the
 * neighbours' receive buffers over NVLink. Strip d goes to the neighbour in direction d, who
 * receives it as ITS strip 8-d (tags, spatial.py:170-172). */
int spc_halo_pack(int N, int C, int H, int W, int halo_h, int halo_w, int dtype, const void* x,
                  void* const send[9], void* stream);
/* Materialise the padded tile (halo_exchange_layer.forward output, spatial.py:1404-1413):
 * y[N][C][H+2hh][W+2hw] = x in the middle, strips / zeros around. */
int spc_halo_pad(int N, int C, int H, int W, int halo_h, int halo_w, int dtype, const void* x,
                 const spc_halo* halo, void* y, void* stream);
/* Backward of spc_halo_pad: crop the middle. */
int spc_halo_crop(int N, int C, int H, int W, int halo_h, int halo_w, int dtype, const void* dy,
                  void* dx, void* stream);

/* ---- peer-memory halo transport (one process per GPU, NVLink / NVSwitch) ------------------
 * Replaces dist.isend/irecv + torch.cuda.synchronize() fences (spatial.py:351-393,401-403).
 * A "mailbox" is a device allocation owned by this rank holding `slots` receive areas of
 * `bytes` each plus per-slot arrival flags.  Peers map it with CUDA IPC and their pack kernel
 * (spc_halo_pack with peer pointers) writes into it; ordering uses device-side flags
 * (release/acquire at system scope), never a host synchronisation. */
typedef struct spc_mailbox spc_mailbox;
#define SPC_IPC_HANDLE_BYTES 64
int   spc_mailbox_create(spc_mailbox** out, size_t bytes, int nflags);
void  spc_mailbox_destroy(spc_mailbox* mb);
void* spc_mailbox_data(spc_mailbox* mb);                       /* local device pointer */
int   spc_mailbox_export(spc_mailbox* mb, unsigned char handle[SPC_IPC_HANDLE_BYTES]);
/* Map a peer's mailbox (handle obtained from the peer through torch.distributed). */
int   spc_mailbox_open(spc_mailbox** out, const unsigned char handle[SPC_IPC_HANDLE_BYTES],
                       size_t bytes, int nflags);
/* Fused protocol steps (one kernel each), graph-capturable: no host-side state in the launch arguments.
 *   post:    wait until the local ack flags ack_idx0[d] show that every neighbour has drained the slot half about
 *            to be overwritten -> pack every strip d with send0[d] != NULL into send0[d] (peer slot) -> when the
 *            whole grid is done, publish the sequence number on peers[d]'s arrival flag arrival_idx0[d].
 *   collect: wait for the local arrival flags arrival_idx0[d] -> copy bytes[d] from src0[d] (local mailbox slot)
 *            to dst[d] -> when the whole grid is done, publish the sequence number on peers[d]'s ack flag
 *            ack_idx0[d] and store it to flag seq_idx.
 * The sequence number s of the exchange is (local flag seq_idx) + 1, read on the device; its parity selects the
 * half of the double-buffered slot (send0[d] / src0[d] + (s&1)*slot_bytes) and the flag bank (index + (s&1)*9).
 * post waits for the acks of sequence s-2 (s <= 2: none); collect waits for the arrivals of s.  post and collect
 * of one exchange must be enqueued in that order on one stream.  counter_idx: a flag word private to the layer's
 * slot, used as the grid-completion counter (exchanges of different layers may run on different streams).
 * The flag waits are bounded: after SPCONV_SPIN_TIMEOUT_S seconds (default 120, 0 = unbounded) the kernel
 * prints the direction it is stuck on and traps, so a dead peer surfaces as a CUDA error, not a hang.
 * Replaces the reference's start_halo_exchange / end_halo_exchange (spatial.py:336-403). */
int spc_halo_post_auto(int N, int C, int H, int W, int halo_h, int halo_w, int dtype, const void* x,
                       void* const send0[9], size_t slot_bytes, spc_mailbox* self,
                       spc_mailbox* const peers[9], const int ack_idx0[9], const int arrival_idx0[9],
                       int seq_idx, int counter_idx, void* stream);
int spc_halo_collect_auto(void* const dst[9], const void* const src0[9], const size_t bytes[9],
                          size_t slot_bytes, spc_mailbox* self, spc_mailbox* const peers[9],
                          const int arrival_idx0[9], const int ack_idx0[9], int seq_idx, int counter_idx,
                          void* stream);
/* ---- exact backward: the reverse halo exchange (opt-in, SPCONV_EXACT_BACKWARD=1) -------------
 * The reference's backward treats received strips as constants (SURVEY 8a N2), so the gradient a tile's outputs
 * owe to its neighbours' edge pixels is dropped.  The exact backward sends it back.  Strip gradient d = the part
 * of the padded tile's input gradient that lies in pad strip d (same shapes as the received strips, but always
 * fp32).  It travels to the neighbour in direction d, which receives it as ITS strip 8-d -- the pairing of the
 * forward exchange -- and adds strip e into the band of real rows / columns it sent towards e (the band
 * spc_halo_pack reads).  g[d] == NULL: no strip gradient for that direction (no neighbour there).
 *   spc_conv2d_dgrad_halo: g[d][n][c][..] = sum_k sum_(r,s) dy[n][k][oy][ox] * w[k][c][r][s] over the output
 *                          windows that cover the strip pixel (fp32 accumulation; any R x S, stride, dtype);
 *   spc_pool2d_bwd_halo:   the same for pooling; x and the received strips give the max windows, which route to
 *                          their first maximal element exactly as spc_pool2d_bwd does;
 *   spc_halo_ring:         the pad ring of halo_exchange_layer's output gradient dy[N][C][H+2hh][W+2hw];
 *   spc_halo_accumulate:   dx[edge band e] += g[e] for every e with g[e] != NULL: each pixel sums every strip that
 *                          covers it (corners: row, column and corner strip) in the order e = 0..8 in fp32 and is
 *                          rounded once to `dtype`.  No atomics: the result is bit-reproducible. */
int spc_conv2d_dgrad_halo(const spc_conv_desc* d, const void* dy, const void* w, float* const g[9], void* stream);
int spc_pool2d_bwd_halo(const spc_pool_desc* d, const void* x, const spc_halo* halo, const void* dy,
                        float* const g[9], void* stream);
int spc_halo_ring(int N, int C, int H, int W, int halo_h, int halo_w, int dtype, const void* dy, float* const g[9],
                  void* stream);
int spc_halo_accumulate(int N, int C, int H, int W, int halo_h, int halo_w, int dtype, void* dx,
                        const float* const g[9], void* stream);
/* Reverse post for the mailbox transport: spc_halo_post_auto's protocol (wait the acks of sequence s-2 of this
 * slot, write into slot half s&1, publish s when the whole grid is done), but the payload is bytes[d] (a multiple
 * of 4) copied from the caller's buffer src[d] to send0[d] instead of a pack of a tile.  Pair it with
 * spc_halo_collect_auto on the same slot (its own flag block and sequence word, separate from the forward
 * slot's), then spc_halo_accumulate.  Graph-capturable like the forward pair. */
int spc_halo_post_strips_auto(const void* const src[9], const size_t bytes[9], void* const send0[9],
                              size_t slot_bytes, spc_mailbox* self, spc_mailbox* const peers[9],
                              const int ack_idx0[9], const int arrival_idx0[9], int seq_idx, int counter_idx,
                              void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SPCONV_H_ */
