// Host-side helpers of the tensor-core kernels (declared in tc_host.cuh).
#include "tc_host.cuh"

namespace muse {

namespace {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* ptr = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || ptr == nullptr) {
    set_last_error("cudaGetDriverEntryPoint(cuTensorMapEncodeTiled) failed: %s", cudaGetErrorString(e));
    return nullptr;
  }
  fn = reinterpret_cast<EncodeTiledFn>(ptr);
  return fn;
}

}  // namespace

int make_tmap(CUtensorMap* map, const char* who, CUtensorMapDataType dtype, const void* base,
              std::initializer_list<long long> dims, std::initializer_list<long long> byte_strides,
              std::initializer_list<long long> box) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return MUSE_ERR_CUDA;
  const int rank = static_cast<int>(dims.size());
  cuuint64_t d[5], st[4];
  cuuint32_t bx[5], estr[5];
  bool aligned = (reinterpret_cast<uintptr_t>(base) & 15) == 0;
  for (int i = 0; i < rank; ++i) {
    d[i] = static_cast<cuuint64_t>(dims.begin()[i]);
    bx[i] = static_cast<cuuint32_t>(box.begin()[i]);
    estr[i] = 1;
  }
  for (int i = 0; i + 1 < rank; ++i) {
    st[i] = static_cast<cuuint64_t>(byte_strides.begin()[i]);
    aligned = aligned && st[i] % 16 == 0;
  }
  if (!aligned) {
    set_last_error("%s: operand base must be 16B aligned and its row strides multiples of 16 bytes", who);
    return MUSE_ERR_INVALID;
  }
  CUresult r = fn(map, dtype, rank, const_cast<void*>(base), d, st, bx, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("%s: cuTensorMapEncodeTiled failed with CUresult %d (rank %d, inner extent %lld, outer extent %lld)",
                   who, (int)r, rank, dims.begin()[0], dims.begin()[rank - 1]);
    return MUSE_ERR_CUDA;
  }
  return MUSE_OK;
}

int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

}  // namespace muse
