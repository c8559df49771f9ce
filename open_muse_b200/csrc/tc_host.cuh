// Host-side helpers of the tensor-core kernels (GEMM, convolution, attention); defined in tc_host.cu.
#pragma once
#include <cuda.h>

#include <initializer_list>

#include "common.cuh"

namespace muse {

// TMA tensor map of bf16 or fp32 elements (dtype) with the 128-byte swizzle, zero-filled out of bounds, rank =
// dims.size() <= 5.  dims[0] is the contiguous dimension, byte_strides[i] the stride of dims[i + 1], box[i] the box extent
// along dims[i] (box[0] at most 128 bytes).  The base must be 16-byte aligned and every stride a multiple of 16 bytes
// (MUSE_ERR_INVALID otherwise); `who` prefixes the error message.
int make_tmap(CUtensorMap* map, const char* who, CUtensorMapDataType dtype, const void* base,
              std::initializer_list<long long> dims, std::initializer_list<long long> byte_strides,
              std::initializer_list<long long> box);

// multiprocessor count of the current device, queried once
int sm_count();

// Raises the dynamic shared-memory limit of kernel K to `bytes`, once: later calls return MUSE_OK straight away.
template <auto K>
int set_max_dynamic_smem(int bytes) {
  static bool done = false;
  if (done) return MUSE_OK;
  const cudaError_t e = cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) {
    set_last_error("cudaFuncSetAttribute(max dynamic shared memory = %d B): %s", bytes, cudaGetErrorString(e));
    return MUSE_ERR_CUDA;
  }
  done = true;
  return MUSE_OK;
}

}  // namespace muse
