// Error reporting + version entry points of the C-ABI (include/qlora_b200.h), and the per-device and environment helpers
// of qb200_internal.h.
// Upstream bitsandbytes' CUDA_CHECK_RETURN prints and exit(1)s the process
// (SURVEY.md 8b); here every entry point returns a status code instead.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "qb200_internal.h"

namespace qb200 {
static thread_local char t_last_error[512] = "";

int set_error(int code, const char* msg) {
  snprintf(t_last_error, sizeof(t_last_error), "%s", msg ? msg : "");
  return code;
}

int check_launch(const char* what) {
  const cudaError_t err = cudaPeekAtLastError();
  if (err == cudaSuccess) return 0;
  (void)cudaGetLastError();  // clear the (non-sticky) launch error
  snprintf(t_last_error, sizeof(t_last_error), "%s: %s (%s)", what, cudaGetErrorName(err), cudaGetErrorString(err));
  return int(err);
}

int env_int(const char* name, int dflt) {
  const char* e = getenv(name);
  return e ? atoi(e) : dflt;
}

int current_device() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) dev = 0;
  return dev;
}

int device_sm_count() {
  static int sms[kMaxDevices] = {0};
  const int dev = current_device();
  if (sms[dev] == 0) {
    int n = 0;
    sms[dev] = (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0) ? n : 132;
  }
  return sms[dev];
}

bool use_pdl() {
  static const bool v = env_int("QB200_PDL", 1) != 0;
  return v;
}
}  // namespace qb200

extern "C" int qb200_version(void) { return 100; /* 0.1.0 */ }
extern "C" const char* qb200_last_error(void) { return qb200::t_last_error; }
