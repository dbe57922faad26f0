#include "common.cuh"
#include <stdarg.h>

namespace rih {
static thread_local char g_err[1024] = "";
int g_pdl = 0;
int g_reverse = 0;
int g_l2_hints = 0;
int g_kb_rotate = 0;

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
int g_ew_cap = 1;
long long ew_ctas(cudaStream_t s) {
  if (g_ew_cap) for (int i = 0; i < CAP_SLOTS; ++i) if (g_cap_ctas[i] > 0 && g_cap_stream[i] == s && 3 * g_cap_ctas[i] < 2 * sm_count()) return sm_count() * 4;
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

// Traversal direction of the NEXT launches: 1 = the tensor-core GEMM / convolution kernels walk their output tiles, and the BatchNorm passes
// their rows, from the last to the first.  A consumer that starts where its producer finished finds the most recently written part of an
// activation (whatever of it fits in the 50 MB L2) still cached; alternating the direction kernel by kernel ("serpentine") keeps that true
// along a whole chain of layers.  Scheduling only: results are unchanged up to summation order in atomically accumulated statistics.
RIH_API int rih_set_traversal(int reverse) { rih::g_reverse = reverse ? 1 : 0; return 0; }

// 1 = activations that a GEMM / 1x1 convolution / BatchNorm pass streams through once are loaded with the L2 evict-first priority, so that they do
// not displace the previous kernel's output (which the next kernel is about to read) from the L2.  Scheduling only.
// 1 (default) = element-wise kernels launched on a CTA-capped stream (rih_set_stream_cta_limit) use a quarter of their usual grid.  Scheduling only.
// 1 = every output tile of the tensor-core GEMM / convolution kernels starts its k loop at a tile-dependent k-block and wraps around, so
// that concurrently running CTAs do not all fetch the same 128-byte slice of their rows at the same time.  Results agree up to fp32
// summation order inside the tensor core accumulation.
RIH_API int rih_set_k_rotation(int on) { rih::g_kb_rotate = on ? 1 : 0; return 0; }
RIH_API int rih_set_ew_cap(int on) { rih::g_ew_cap = on ? 1 : 0; return 0; }

RIH_API int rih_set_l2_hints(int on) { rih::g_l2_hints = on ? 1 : 0; return 0; }

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
