// Library plumbing of libmuse_b200.so (include/muse_b200.h): ABI version, error message, PDL switch, device selection.
// Every op's entry point is defined in the file that implements it.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>

#include "common.cuh"

namespace muse {

static thread_local char g_err[512] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// Programmatic dependent launch switch (common.cuh).  Process-wide; the initial value comes from MUSE_B200_PDL.
static int g_pdl = -1;
bool pdl_enabled() {
  if (g_pdl < 0) {
    const char* e = getenv("MUSE_B200_PDL");
    g_pdl = (e != nullptr) ? (atoi(e) != 0) : MUSE_B200_PDL_DEFAULT;
  }
  return g_pdl != 0;
}

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("%s: CUDA launch failed: %s", what, cudaGetErrorString(e));
    return MUSE_ERR_CUDA;
  }
  return MUSE_OK;
}

}  // namespace muse

using namespace muse;

extern "C" {

int muse_abi_version(void) { return MUSE_B200_ABI_VERSION; }
const char* muse_last_error(void) { return g_err; }

int muse_set_device(int device) {
  cudaError_t e = cudaSetDevice(device);
  if (e != cudaSuccess) { set_last_error("cudaSetDevice(%d): %s", device, cudaGetErrorString(e)); return MUSE_ERR_CUDA; }
  return MUSE_OK;
}

int muse_device_info(int* sm_major, int* sm_minor, int* num_sms) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) { set_last_error("cudaGetDevice: %s", cudaGetErrorString(e)); return MUSE_ERR_CUDA; }
  cudaDeviceGetAttribute(sm_major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(sm_minor, cudaDevAttrComputeCapabilityMinor, dev);
  cudaDeviceGetAttribute(num_sms, cudaDevAttrMultiProcessorCount, dev);
  return MUSE_OK;
}

int muse_set_pdl(int enabled) {
  g_pdl = enabled ? 1 : 0;
  return MUSE_OK;
}
int muse_get_pdl(void) { return pdl_enabled() ? 1 : 0; }

}  // extern "C"
