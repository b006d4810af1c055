// Library-level entry points of libspann3r_b200.so (include/spann3r_b200.h): version, ABI struct sizes, last error and
// device check.  Each operation's entry point is defined beside its kernels.
#include "../../include/spann3r_b200.h"

#include "gemm.cuh"

extern "C" {

int s3r_version(void) { return S3R_VERSION; }
int s3r_abi_sizeof(int which) {
  switch (which) {
    case 0: return (int)sizeof(s3r_gemm_desc);
    case 1: return (int)sizeof(s3r_model_w);
    case 2: return (int)sizeof(s3r_bank);
    case 3: return (int)sizeof(s3r_loss_desc);
    case 4: return (int)sizeof(s3r_attn_train_desc);
  }
  return -1;
}
const char* s3r_last_error(void) { return s3r::last_error(); }

int s3r_device_ok(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) {
    cudaGetLastError();
    return 0;
  }
  int dev = 0, major = 0, minor = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  return (major == 9 && minor == 0) ? 1 : 0;
}

}  // extern "C"
