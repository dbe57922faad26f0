#include "common.cuh"
#include <stdarg.h>

namespace rih {
static thread_local char g_err[1024] = "";
int g_pdl = 0;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// Optional cap on the SMs that work launched on a given stream may occupy (rih_set_stream_cta_limit): a convolution pipeline that runs
// concurrently with the latency-bound token decoder leaves the remaining SMs / thread slots to it.  Persistent GEMM grids are capped to `ctas`
// CTAs; element-wise kernels on such a stream launch a quarter of their usual CTAs per SM (ew_ctas), so that a 448-thread GEMM CTA of the
// decoder always finds thread slots next to them instead of waiting for a wave of 8 x 256-thread CTAs per SM to drain.
constexpr int CAP_SLOTS = 16;
static cudaStream_t g_cap_stream[CAP_SLOTS] = {};
static int g_cap_ctas[CAP_SLOTS] = {};
int set_stream_cta_limit(cudaStream_t s, int ctas) {
  for (int i = 0; i < CAP_SLOTS; ++i) if (g_cap_stream[i] == s || g_cap_ctas[i] == 0) { g_cap_stream[i] = s; g_cap_ctas[i] = ctas > 0 ? ctas : 0; return 0; }
  return 1;
}
int stream_cta_limit(cudaStream_t s, int num_sms) {
  for (int i = 0; i < CAP_SLOTS; ++i) if (g_cap_ctas[i] > 0 && g_cap_stream[i] == s) return g_cap_ctas[i] < num_sms ? g_cap_ctas[i] : num_sms;
  return num_sms;
}
long long ew_ctas(cudaStream_t s) {
  for (int i = 0; i < CAP_SLOTS; ++i) if (g_cap_ctas[i] > 0 && g_cap_stream[i] == s && 3 * g_cap_ctas[i] < 2 * sm_count()) return sm_count() * 4;
  return sm_count() * 16;
}

// SMs of the current device (132 on an H100 SXM), queried once per device
int sm_count() {
  static int n[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
  if (!n[dev]) {
    int v = 0;
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    n[dev] = v > 0 ? v : 132;
  }
  return n[dev];
}

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("kernel launch %s failed: %s", what, cudaGetErrorString(e));
    return 3;
  }
  return 0;
}
}  // namespace rih

RIH_API const char* rih_last_error(void) { return rih::g_err; }
RIH_API int rih_version(void) { return 200; }

// Programmatic dependent launch for every kernel of the library (see common.cuh): 1 = on, 0 = plain stream-ordered launches.  Scheduling only:
// results are unchanged (no reference counterpart).
RIH_API int rih_set_pdl(int on) { rih::g_pdl = on ? 1 : 0; return 0; }

// Device properties probe (used by the host side to fail loudly on a device other than sm_90).
RIH_API int rih_device_info(int device, int* cc_major, int* cc_minor, int* sm_count, size_t* smem_optin) {
  cudaDeviceProp p;
  RIH_CUDA(cudaGetDeviceProperties(&p, device));
  if (cc_major) *cc_major = p.major;
  if (cc_minor) *cc_minor = p.minor;
  if (sm_count) *sm_count = p.multiProcessorCount;
  if (smem_optin) *smem_optin = p.sharedMemPerBlockOptin;
  return 0;
}
