// vitron_b200 — library bookkeeping: version, error text, device query.
#include "common.cuh"
#include "vitron_b200.h"
#include <stdio.h>
#include <string.h>

static char g_last_error[256] = "";

void vb_set_last_error(cudaError_t e) {
  snprintf(g_last_error, sizeof(g_last_error), "%s: %s", cudaGetErrorName(e), cudaGetErrorString(e));
}

int vb_num_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0)
      sms = 132;   // H100 SXM
  }
  return sms;
}

static bool g_pdl = false;
bool vb_pdl_enabled() { return g_pdl; }
extern "C" int vb200_set_pdl(int enable) {
  const int prev = g_pdl ? 1 : 0;
  g_pdl = enable != 0;
  return prev;
}

extern "C" const char* vb200_version(void) { return "vitron_b200 0.1 (sm_90a)"; }
extern "C" const char* vb200_last_error(void) { return g_last_error; }
extern "C" int vb200_device_ok(void) {
  int dev = 0, major = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return 0;
  int minor = 0;
  if (cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev) != cudaSuccess) return 0;
  return major == 9 && minor == 0 ? 1 : 0;   // the library holds sm_90a code only
}
