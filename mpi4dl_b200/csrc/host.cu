// host.cu -- host helpers every kernel family shares: the SM count, the dynamic shared-memory opt-in and the TMA
// descriptor encoder.
#include <mutex>
#include <unordered_set>

#include "common.cuh"
#include "tc_common.cuh"

namespace spc {

int sm_count() {
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  }
  return sms;
}

int allow_dynamic_smem(const void* kernel, int bytes) {
  static std::mutex mu;
  static std::unordered_set<const void*> done;
  std::lock_guard<std::mutex> lock(mu);
  if (done.count(kernel)) return SPC_OK;
  SPC_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  done.insert(kernel);
  return SPC_OK;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int make_tmap(CUtensorMap* m, const void* base, CUtensorMapDataType type, int rank, const uint64_t* dims,
              const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swizzle) {
  // the driver entry point, fetched through the runtime
  static EncodeTiledFn enc = nullptr;
  if (!enc) {
    void* fp = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      enc = reinterpret_cast<EncodeTiledFn>(fp);
  }
  if (!enc) {
    set_error("cuTensorMapEncodeTiled entry point not available");
    return SPC_ECUDA;
  }
  // the driver-API encode needs a current context on THIS thread; a backward pass can be the first CUDA work of an
  // autograd worker thread, which the runtime binds only at its first runtime call.  Once per thread: cudaFree is not
  // allowed while a stream is being captured into a CUDA graph, and it is not free either.
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) {
    if (cudaFree(nullptr) != cudaSuccess) {
      set_error("TMA descriptor: no CUDA context on this thread");
      return SPC_ECUDA;
    }
    ctx_bound = true;
  }
  cuuint64_t gd[5], gs[5];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) {
    gd[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i > 0) gs[i - 1] = strides_bytes[i];
  }
  const CUresult r = enc(m, type, (cuuint32_t)rank, const_cast<void*>(base), gd, gs, bx, es,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d) type=%d rank=%d dims=[%llu,%llu,%llu] strides=[%llu,%llu]", (int)r,
              (int)type, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
              (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 1 ? strides_bytes[1] : 0),
              (unsigned long long)(rank > 2 ? strides_bytes[2] : 0));
    return SPC_ECUDA;
  }
  return SPC_OK;
}

}  // namespace spc
