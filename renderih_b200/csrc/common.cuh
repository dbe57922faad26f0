// Common helpers for the renderih_b200 C-ABI CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#define RIH_API extern "C" __attribute__((visibility("default")))

namespace rih {

// ---- error convention (SURVEY 8b): 0 = ok, non-zero + rih_last_error() ----
void set_error(const char* fmt, ...);
int check_launch(const char* what);
int set_stream_cta_limit(cudaStream_t s, int ctas);
int stream_cta_limit(cudaStream_t s, int num_sms);
long long ew_ctas(cudaStream_t s);      // grid cap of element-wise kernels on stream s (16 per SM, or 4 per SM on a CTA-capped stream)
int sm_count();                         // SMs of the current device

#define RIH_REQUIRE(cond, ...)                        \
  do {                                                \
    if (!(cond)) {                                    \
      rih::set_error(__VA_ARGS__);                    \
      return 1;                                       \
    }                                                 \
  } while (0)

#define RIH_CUDA(call)                                                        \
  do {                                                                        \
    cudaError_t e__ = (call);                                                 \
    if (e__ != cudaSuccess) {                                                 \
      rih::set_error("%s failed: %s", #call, cudaGetErrorString(e__));        \
      return 2;                                                               \
    }                                                                         \
  } while (0)

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// ---- programmatic dependent launch (PDL) ----
// Every kernel of this library is launched through launch_k() and starts with pdl_sync() (or its two halves).  With g_pdl != 0 the launch
// carries cudaLaunchAttributeProgrammaticStreamSerialization: the kernel may be scheduled as soon as every CTA of its stream predecessor has
// executed griddepcontrol.launch_dependents (first instruction of all our kernels) -- its CTAs become resident on free SMs, run their
// prologue (barrier init, tensor-map prefetch) and then block in griddepcontrol.wait until the predecessor has COMPLETED and
// its memory operations are visible.  That takes the launch latency and the prologue off the dependent chains of the decoder (hundreds of
// 5-15 us kernels).  Nothing before pdl_wait() may touch global memory a predecessor writes.  Under CUDA-graph capture the edges become
// programmatic dependencies of the graph.  g_pdl == 0: plain launches; griddepcontrol.* are no-ops then.
extern int g_pdl;
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_sync() { pdl_launch_dependents(); pdl_wait(); }

template <class... KArgs, class... Args>
static inline void launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = g_pdl ? 1 : 0;
  cfg.attrs = attr; cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);     // errors surface through check_launch() (cudaGetLastError)
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// Sum of v over a block of NW warps, returned to every thread: each warp's shuffle sum, then the warps' partials in warp order.
// s_red holds NW floats; the leading barrier lets consecutive calls reuse it.
template <int NW>
__device__ __forceinline__ float block_sum(float v, float* s_red, int tid) {
  v = warp_sum(v);
  __syncthreads();
  if ((tid & 31) == 0) s_red[tid >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int i = 0; i < NW; ++i) t += s_red[i];
  return t;
}

// i = q * d + r with a 32-bit fast path (64-bit integer division costs ~100 instructions and dominated the elementwise kernels)
__device__ __forceinline__ void divmod(long long i, int d, bool small, long long& q, int& r) {
  if (small) {
    const unsigned u = (unsigned)i, qq = u / (unsigned)d;
    q = qq; r = (int)(u - qq * (unsigned)d);
  } else {
    q = i / d; r = (int)(i - q * d);
  }
}

// Counter-based RNG for dropout masks (stateless: regenerated in backward from the same key): murmur3's 32-bit finaliser over the
// element index xor a per-launch key (8 integer instructions per element; the 64-bit splitmix used before cost ~3x that and showed
// up in the attention kernels, where a mask is drawn per score).
__device__ __forceinline__ uint32_t hash_u32(uint64_t seed, uint64_t idx) {
  const uint32_t key = (uint32_t)seed ^ ((uint32_t)(seed >> 32) * 0x9E3779B1u);
  uint32_t x = ((uint32_t)idx ^ key) + (uint32_t)(idx >> 32) * 0x85EBCA6Bu;
  x ^= x >> 16; x *= 0x85EBCA6Bu;
  x ^= x >> 13; x *= 0xC2B2AE35u;
  x ^= x >> 16;
  return x;
}
// keep-scale for dropout: returns 0 (dropped) or 1/(1-p)
__device__ __forceinline__ float dropout_scale(uint64_t seed, uint64_t idx, uint32_t thresh, float inv_keep) {
  return hash_u32(seed, idx) >= thresh ? inv_keep : 0.f;
}
static inline uint32_t dropout_thresh(float p) {
  double t = (double)p * 4294967296.0;
  if (t < 0) t = 0;
  if (t > 4294967295.0) t = 4294967295.0;
  return (uint32_t)t;
}

}  // namespace rih
