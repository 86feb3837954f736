// tap_tf32_common.cuh -- what the TF32 tap kernels of conv_tap_tf32.cu (stride 1) and conv_tap_s2_tf32.cu (stride 2)
// share: the smem budget, the activation tensor maps and the row-segment order of the tiles.
#pragma once
#include "common.cuh"
#include "tc_common.cuh"
#include "wgmma_tf32.cuh"

namespace spc {

namespace {

constexpr int TT_THREADS = 384;
constexpr int TT_BK = 32;                     // channels per k-chunk / pixels per row segment
constexpr int TT_MAX_STAGES = 8;
constexpr int TT_SMEM_LIMIT = 222 * 1024;     // as gemm_tf32.cu
constexpr int TT_SMEM_AUX = 1024 /*align*/ + 512 /*barriers*/;
constexpr int TT_WRES_MAX = 128 * 1024;       // resident weights at most
constexpr int TW_MAX_CHAIN = 512;             // wgrad: row segments per item at most (the error bound of the kernels)

// [N][rows][H][W] fp32, box = [1][box_rows][1][box_w px]
inline int make_act_tmap4(CUtensorMap* m, const void* base, int N, int rows, int H, int W, int box_rows, int box_w,
                          bool swizzle) {
  const uint64_t dims[4] = {(uint64_t)W, (uint64_t)H, (uint64_t)rows, (uint64_t)N};
  const uint64_t strides[4] = {0, (uint64_t)W * 4, (uint64_t)H * W * 4, (uint64_t)rows * H * W * 4};
  const uint32_t box[4] = {(uint32_t)box_w, 1, (uint32_t)box_rows, 1};
  return make_tmap(m, base, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, dims, strides, box,
                   swizzle ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE);
}

// row segment seg of the [N][H][ceil(W / 32)] order -> image, row, first pixel
__device__ __forceinline__ void seg_coords(int seg, int segs_row, int H, int& n, int& y, int& x0) {
  x0 = (seg % segs_row) * 32;
  const int row = seg / segs_row;
  y = row % H;
  n = row / H;
}

// output channels per group: one wgmma N of 16, 32, 64, 128 or 256
inline int tap_nt(int M) { return M <= 16 ? 16 : (M <= 32 ? 32 : (M <= 64 ? 64 : (M <= 128 ? 128 : 256))); }

}  // namespace
}  // namespace spc
