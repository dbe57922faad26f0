// NHWC image-side elementwise / reduction kernels: BatchNorm (train+eval), max-pool, bilinear x2,
// global average pool, layout conversion. All tensors are fp32 [rows, C] with an explicit row stride.
#include "common.cuh"
using namespace rih;

// ============================================================== layout conversion
// NCHW [N,C,H,W] -> NHWC [N,H,W,Cp] (channels >= C zero-filled). reference input layout: models/model.py:25
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ x, float* __restrict__ y, int N, int C, int HW, int Cp, int ldy) {
  pdl_sync();
  __shared__ float tile[32][33];
  int n = blockIdx.z;
  int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int c = c0 + i, p = p0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && p < HW) ? x[((size_t)n * C + c) * HW + p] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int p = p0 + i, c = c0 + threadIdx.x;
    if (p < HW && c < Cp) y[((size_t)n * HW + p) * ldy + c] = tile[threadIdx.x][i];
  }
}
__global__ void nhwc_to_nchw_kernel(const float* __restrict__ x, float* __restrict__ y, int N, int C, int HW, int ldx, int c_off) {
  pdl_sync();
  __shared__ float tile[32][33];
  int n = blockIdx.z;
  int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int p = p0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && p < HW) ? x[((size_t)n * HW + p) * ldx + c_off + c] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int c = c0 + i, p = p0 + threadIdx.x;
    if (c < C && p < HW) y[((size_t)n * C + c) * HW + p] = tile[threadIdx.x][i];
  }
}
// few-channel images (the RGB input): one thread per pixel, plane reads coalesced across the warp, pixel writes contiguous
__global__ void nchw_to_nhwc_small_kernel(const float* __restrict__ x, float* __restrict__ y, int C, int HW, int Cp, int ldy, long long total) {
  pdl_sync();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / HW; const int p = (int)(i - n * HW);
    float* q = y + i * ldy;
    for (int c = 0; c < Cp; ++c) q[c] = c < C ? x[(n * C + c) * HW + p] : 0.f;
  }
}
RIH_API int rih_nchw_to_nhwc(const float* x, float* y, int N, int C, int HW, int Cp, int ldy, cudaStream_t s) {
  RIH_REQUIRE(Cp >= C && ldy >= Cp, "nchw_to_nhwc: bad channel padding");
  if (Cp <= 8) {
    const long long total = (long long)N * HW;
    if (total == 0) return 0;
    launch_k(nchw_to_nhwc_small_kernel, (int)min(ew_ctas(s), (total + 255) / 256), 256, 0, s, x, y, C, HW, Cp, ldy, total);
    return check_launch("nchw_to_nhwc");
  }
  dim3 grid(cdiv(HW, 32), cdiv(Cp, 32), N), block(32, 8);
  launch_k(nchw_to_nhwc_kernel, grid, block, 0, s, x, y, N, C, HW, Cp, ldy);
  return check_launch("nchw_to_nhwc");
}
// y NCHW [N,C,HW] <- channels [c_off, c_off+C) of x NHWC
RIH_API int rih_nhwc_to_nchw(const float* x, float* y, int N, int C, int HW, int ldx, int c_off, cudaStream_t s) {
  dim3 grid(cdiv(HW, 32), cdiv(C, 32), N), block(32, 8);
  launch_k(nhwc_to_nchw_kernel, grid, block, 0, s, x, y, N, C, HW, ldx, c_off);
  return check_launch("nhwc_to_nchw");
}

// NCHW RGB image -> zero-bordered NHWC4 [N][H+6][W+8][4] (3 rows / columns of zeros in front, RGB + one zero channel): the layout the
// implicit-GEMM stem reads (rih_stem_conv_fwd).  One thread per padded pixel, coalesced plane reads, one float4 store.
__global__ void nchw_to_nhwc4_pad_kernel(const float* __restrict__ x, float4* __restrict__ y, int N, int H, int W) {
  pdl_sync();
  const int Hp = H + 6, Wp = W + 8;
  const long long total = (long long)N * Hp * Wp;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int wp = (int)(i % Wp); long long t = i / Wp; const int hp = (int)(t % Hp); const int n = (int)(t / Hp);
    const int h = hp - 3, w = wp - 3;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if ((unsigned)h < (unsigned)H && (unsigned)w < (unsigned)W) {
      const float* p = x + ((size_t)n * 3 * H + h) * W + w;
      v.x = p[0]; v.y = p[(size_t)H * W]; v.z = p[2 * (size_t)H * W];
    }
    y[i] = v;
  }
}
RIH_API int rih_nchw_to_nhwc4_pad(const float* x, float* y, int N, int H, int W, cudaStream_t s) {
  RIH_REQUIRE(N > 0 && H > 0 && W > 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0, "nchw_to_nhwc4_pad: bad arguments");
  const long long total = (long long)N * (H + 6) * (W + 8);
  launch_k(nchw_to_nhwc4_pad_kernel, (int)min(ew_ctas(s), (total + 255) / 256), 256, 0, s, x, reinterpret_cast<float4*>(y), N, H, W);
  return check_launch("nchw_to_nhwc4_pad");
}

// generic strided 2-D copy / add:  y[r, 0:C] (+)= x[r, 0:C]
__global__ void copy2d_kernel(const float* __restrict__ x, int ldx, float* __restrict__ y, int ldy, long long rows, int C, int acc) {
  pdl_sync();
  long long total = rows * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long r; int c; divmod(i, C, total < (1ll << 32), r, c);
    float v = x[r * ldx + c];
    float* q = y + r * ldy + c;
    *q = acc ? (*q + v) : v;
  }
}
RIH_API int rih_copy2d(const float* x, int ldx, float* y, int ldy, long long rows, int C, int accumulate, cudaStream_t s) {
  if (rows * C == 0) return 0;
  int grid = (int)min(ew_ctas(s), (rows * C + 255) / 256);
  launch_k(copy2d_kernel, grid, 256, 0, s, x, ldx, y, ldy, rows, C, accumulate);
  return check_launch("copy2d");
}

// ============================================================== BatchNorm
// column statistics over M rows: partial sums in double, atomically merged.  ws = double[2*C] (zeroed here)
__global__ void bn_stats_kernel(const float* __restrict__ x, int ld, int M, int C, int rows_per_cta, double* __restrict__ ws) {
  pdl_sync();
  int c = blockIdx.x * 32 + threadIdx.x;
  int r0 = blockIdx.y * rows_per_cta, r1 = min(M, r0 + rows_per_cta);
  double s = 0.0, ss = 0.0;
  if (c < C) {
    for (int r = r0 + threadIdx.y; r < r1; r += blockDim.y) {
      float v = x[(size_t)r * ld + c];
      s += v; ss += (double)v * v;
    }
  }
  __shared__ double sh[2][8][33];
  sh[0][threadIdx.y][threadIdx.x] = s; sh[1][threadIdx.y][threadIdx.x] = ss;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    for (int i = 1; i < 8; ++i) { s += sh[0][i][threadIdx.x]; ss += sh[1][i][threadIdx.x]; }
    atomicAdd(ws + c, s); atomicAdd(ws + C + c, ss);
  }
}
// Thread -> (channel quad, first row) mapping shared by the element-wise BatchNorm passes: the launch has a multiple of C/4 threads, so
// a thread keeps ONE channel quad for its whole grid-stride loop and the per-channel terms are computed once per thread.
struct BnMap { int q; long long r0, rstride; };
// Streamed inputs of the element-wise BatchNorm passes are loaded with the evict-first priority, so that they do not displace the previous
// kernel's output (which the next kernel is about to read) from the L2.
__device__ __forceinline__ float4 ld4_stream(const float* p) { return __ldcs(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ BnMap bn_map(int C4) {
  const long long gid = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long T = (long long)gridDim.x * blockDim.x;
  BnMap m; m.q = (int)(gid % C4); m.r0 = gid / C4; m.rstride = T / C4;
  return m;
}
static inline int bn_grid(long long M, int C4, int threads, long long cap = -1) {
  int g = 1, a = C4, b = threads;                 // grid must be a multiple of C4 / gcd(C4, threads)
  while (b) { int t = a % b; a = b; b = t; }
  g = C4 / a;
  long long want = (M * C4 + threads - 1) / threads;
  if (cap < 0) cap = (long long)sm_count() * 16;
  if (want > cap) want = cap;
  if (want < 1) want = 1;
  return (int)((want + g - 1) / g * g);
}

// column sums / sums of squares of x into ws[0:C], ws[C:2C] (fp64; ws is zeroed here)
RIH_API int rih_bn_colstats(const float* x, int ld, int M, int C, double* ws, cudaStream_t s) {
  RIH_REQUIRE(M > 0 && C > 0, "bn_colstats: empty");
  RIH_CUDA(cudaMemsetAsync(ws, 0, sizeof(double) * 2 * C, s));
  int gx = cdiv(C, 32);
  int target = cdiv(sm_count() * 8, gx);
  int rows_per_cta = max(64, cdiv(M, target));
  dim3 grid(gx, cdiv(M, rows_per_cta)), block(32, 8);
  launch_k(bn_stats_kernel, grid, block, 0, s, x, ld, M, C, rows_per_cta, ws);
  return check_launch("bn_stats");
}

// BatchNorm forward in ONE pass over the activation: the per-channel mean / rstd are derived by every thread for its own channel quad
//   training (stats != NULL): from the fp64 column sums (a convolution's fused epilogue or rih_bn_colstats), torch.nn.BatchNorm2d
//                             semantics: biased variance for the normalisation, momentum update of the running statistics with the
//                             unbiased variance, num_batches_tracked += 1 -- written once, by the threads that own row 0
//   eval     (stats == NULL): from the running statistics
// then y = (x - mean) * rstd * gamma + beta (+res) (relu).  mean / rstd are also stored for the backward pass.  C % 4 == 0, ld % 4 == 0.
__global__ void __launch_bounds__(256)
bn_forward_kernel(const float* __restrict__ x, int ldx, const double* __restrict__ stats, long long M, int C4, float eps, float momentum,
                  const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ res, int ldr,
                  float* __restrict__ y, int ldy, int relu, unsigned char* __restrict__ relu_mask, float* __restrict__ mean_out, float* __restrict__ rstd_out,
                  float* __restrict__ running_mean, float* __restrict__ running_var, long long* __restrict__ tracked) {
  pdl_sync();
  const BnMap mp = bn_map(C4);
  const int c = mp.q * 4, C = C4 * 4;
  float mu[4], rs[4];
  if (stats) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const double m = stats[c + j] / (double)M;
      double var = stats[C + c + j] / (double)M - m * m;
      if (var < 0) var = 0;
      mu[j] = (float)m;
      rs[j] = (float)(1.0 / sqrt(var + (double)eps));
      if (mp.r0 == 0 && running_mean) {
        const double unbiased = M > 1 ? var * (double)M / (double)(M - 1) : var;
        running_mean[c + j] = (1.f - momentum) * running_mean[c + j] + momentum * (float)m;
        running_var[c + j] = (1.f - momentum) * running_var[c + j] + momentum * (float)unbiased;
      }
    }
    if (mp.r0 == 0 && mp.q == 0 && tracked) *tracked += 1;
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) { mu[j] = running_mean[c + j]; rs[j] = 1.f / sqrtf(running_var[c + j] + eps); }
  }
  if (mp.r0 == 0) {
    *reinterpret_cast<float4*>(mean_out + c) = make_float4(mu[0], mu[1], mu[2], mu[3]);
    *reinterpret_cast<float4*>(rstd_out + c) = make_float4(rs[0], rs[1], rs[2], rs[3]);
  }
  const float4 g = *reinterpret_cast<const float4*>(gamma + c), b = *reinterpret_cast<const float4*>(beta + c);
  for (long long r = mp.r0; r < M; r += mp.rstride) {
    const float4 v = ld4_stream(x + r * ldx + c);
    float4 o;
    o.x = (v.x - mu[0]) * rs[0] * g.x + b.x; o.y = (v.y - mu[1]) * rs[1] * g.y + b.y;
    o.z = (v.z - mu[2]) * rs[2] * g.z + b.z; o.w = (v.w - mu[3]) * rs[3] * g.w + b.w;
    if (res) {
      const float4 q = ld4_stream(res + r * ldr + c);
      o.x += q.x; o.y += q.y; o.z += q.z; o.w += q.w;
    }
    if (relu) {
      // one byte per channel quad records which of the four outputs passed the ReLU: the backward passes of a residual block read it
      // (1/16 of the bytes) instead of the whole forward output
      if (relu_mask) relu_mask[r * C4 + mp.q] = (unsigned char)((o.x > 0.f ? 1 : 0) | (o.y > 0.f ? 2 : 0) | (o.z > 0.f ? 4 : 0) | (o.w > 0.f ? 8 : 0));
      o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f);
    }
    *reinterpret_cast<float4*>(y + r * ldy + c) = o;
  }
}
// reference: torch.nn.BatchNorm2d forward (torchvision ResNet blocks; models/encoder.py:54; models/model_zoo/__init__.py:57,66)
RIH_API int rih_bn_forward(const float* x, int ldx, const double* stats, long long M, int C, float eps, float momentum,
                           const float* gamma, const float* beta, const float* res, int ldr, float* y, int ldy, int relu, unsigned char* relu_mask,
                           float* mean_out, float* rstd_out, float* running_mean, float* running_var, long long* tracked, cudaStream_t s) {
  RIH_REQUIRE(C % 4 == 0 && ldx % 4 == 0 && ldy % 4 == 0 && (!res || ldr % 4 == 0), "bn_forward: needs C,ld %% 4 == 0");
  RIH_REQUIRE(M > 0 && (stats || (running_mean && running_var)), "bn_forward: eval mode needs the running statistics");
  launch_k(bn_forward_kernel, bn_grid(M, C / 4, 256, ew_ctas(s)), 256, 0, s, x, ldx, stats, M, C / 4, eps, momentum, gamma, beta, res, ldr, y, ldy, relu,
           relu_mask, mean_out, rstd_out, running_mean, running_var, tracked);
  return check_launch("bn_forward");
}

// backward pass 1: g = dy * (y > 0 if relu);  ws[0:C] = sum g, ws[C:2C] = sum g*xhat
// block = 8 channel quads (32 channels, float4 loads) x 32 row lanes; fp64 accumulation, one fp64 atomic pair per channel per CTA
__global__ void __launch_bounds__(256)
bn_bwd_reduce_kernel(const float* __restrict__ dy, int lddy, const float* __restrict__ y, int ldy, const unsigned char* __restrict__ relu_mask,
                     const float* __restrict__ x, int ldx, const float* __restrict__ mean, const float* __restrict__ rstd,
                     const float* __restrict__ gamma, const float* __restrict__ beta,
                     int M, int C, int rows_per_cta, int relu, double* __restrict__ ws) {
  pdl_sync();
  const int tx = threadIdx.x & 7, ty = threadIdx.x >> 3;
  const int c = blockIdx.x * 32 + tx * 4;
  const int r0 = blockIdx.y * rows_per_cta, r1 = min(M, r0 + rows_per_cta);
  double s[4] = {0, 0, 0, 0}, sx[4] = {0, 0, 0, 0};
  if (c < C) {
    const float4 mu = *reinterpret_cast<const float4*>(mean + c), rs = *reinterpret_cast<const float4*>(rstd + c);
    float4 ga = make_float4(0.f, 0.f, 0.f, 0.f), be = ga;
    if (relu && !y) { ga = *reinterpret_cast<const float4*>(gamma + c); be = *reinterpret_cast<const float4*>(beta + c); }
    for (int r = r0 + ty; r < r1; r += 32) {
      float4 g = *reinterpret_cast<const float4*>(dy + (size_t)r * lddy + c);
      const float4 xv = *reinterpret_cast<const float4*>(x + (size_t)r * ldx + c);
      if (relu && relu_mask) {
        const unsigned m4 = relu_mask[(size_t)r * (C >> 2) + (c >> 2)];
        if (!(m4 & 1)) g.x = 0.f; if (!(m4 & 2)) g.y = 0.f; if (!(m4 & 4)) g.z = 0.f; if (!(m4 & 8)) g.w = 0.f;
      } else if (relu) {
        // ReLU mask: from the saved output, or (no residual) recomputed from x with the forward's exact expression (bn_forward_kernel)
        float4 yy;
        if (y) yy = *reinterpret_cast<const float4*>(y + (size_t)r * ldy + c);
        else { yy.x = (xv.x - mu.x) * rs.x * ga.x + be.x; yy.y = (xv.y - mu.y) * rs.y * ga.y + be.y;
               yy.z = (xv.z - mu.z) * rs.z * ga.z + be.z; yy.w = (xv.w - mu.w) * rs.w * ga.w + be.w; }
        if (!(yy.x > 0.f)) g.x = 0.f; if (!(yy.y > 0.f)) g.y = 0.f; if (!(yy.z > 0.f)) g.z = 0.f; if (!(yy.w > 0.f)) g.w = 0.f;
      }
      s[0] += g.x; s[1] += g.y; s[2] += g.z; s[3] += g.w;
      sx[0] += (double)g.x * ((xv.x - mu.x) * rs.x); sx[1] += (double)g.y * ((xv.y - mu.y) * rs.y);
      sx[2] += (double)g.z * ((xv.z - mu.z) * rs.z); sx[3] += (double)g.w * ((xv.w - mu.w) * rs.w);
    }
  }
  __shared__ double sh[2][32][33];
#pragma unroll
  for (int i = 0; i < 4; ++i) { sh[0][ty][tx * 4 + i] = s[i]; sh[1][ty][tx * 4 + i] = sx[i]; }
  __syncthreads();
  if (threadIdx.x < 64) {
    const int which = threadIdx.x >> 5, col = threadIdx.x & 31;
    double acc = 0.0;
    for (int i = 0; i < 32; ++i) acc += sh[which][i][col];
    const int cc = blockIdx.x * 32 + col;
    if (cc < C) atomicAdd(ws + which * C + cc, acc);
  }
}
// backward pass 2 (the per-channel finalisation folded in): dx = gamma*rstd*(g - sum_g/M - xhat*sum_gx/M) [train] ; dres (+)= g ;
// optional mask by (x>0) for Conv->ReLU->BN; the threads that own row 0 write dgamma / dbeta.  Same thread mapping as bn_forward_kernel.
__global__ void __launch_bounds__(256)
bn_bwd_apply_kernel(const float* __restrict__ dy, int lddy, const float* __restrict__ y, int ldy, const unsigned char* __restrict__ relu_mask,
                    const float* __restrict__ x, int ldx, const float* __restrict__ mean, const float* __restrict__ rstd,
                    const float* __restrict__ gamma, const float* __restrict__ beta, const double* __restrict__ ws,
                    float* __restrict__ dx, int lddx, float* __restrict__ dres, int lddr, int dres_acc,
                    float* __restrict__ dgamma, float* __restrict__ dbeta, int param_acc,
                    long long M, int C4, int relu, int training, int mask_input) {
  pdl_sync();
  const BnMap mp = bn_map(C4);
  const int c = mp.q * 4, C = C4 * 4;
  const float invM = 1.f / (float)M;
  const float4 mu4 = *reinterpret_cast<const float4*>(mean + c), rs4 = *reinterpret_cast<const float4*>(rstd + c);
  const float4 ga4 = *reinterpret_cast<const float4*>(gamma + c);
  float4 be4 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (relu && !y) be4 = *reinterpret_cast<const float4*>(beta + c);
  const float muv[4] = {mu4.x, mu4.y, mu4.z, mu4.w}, rsv[4] = {rs4.x, rs4.y, rs4.z, rs4.w}, gav[4] = {ga4.x, ga4.y, ga4.z, ga4.w};
  const float bev[4] = {be4.x, be4.y, be4.z, be4.w};
  float sgv[4], sxv[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) { sgv[j] = (float)ws[c + j]; sxv[j] = (float)ws[C + c + j]; }
  if (mp.r0 == 0) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (dgamma) dgamma[c + j] = param_acc ? dgamma[c + j] + sxv[j] : sxv[j];
      if (dbeta) dbeta[c + j] = param_acc ? dbeta[c + j] + sgv[j] : sgv[j];
    }
  }
  for (long long r = mp.r0; r < M; r += mp.rstride) {
    const float4 g4 = ld4_stream(dy + r * lddy + c);
    float g[4] = {g4.x, g4.y, g4.z, g4.w};
    const float4 x4 = ld4_stream(x + r * ldx + c);
    const float xv[4] = {x4.x, x4.y, x4.z, x4.w};
    if (relu && relu_mask) {
      const unsigned m4 = relu_mask[r * C4 + mp.q];
#pragma unroll
      for (int j = 0; j < 4; ++j) if (!(m4 & (1u << j))) g[j] = 0.f;
    } else if (relu) {
      float yv[4];
      if (y) { const float4 y4 = *reinterpret_cast<const float4*>(y + r * ldy + c); yv[0] = y4.x; yv[1] = y4.y; yv[2] = y4.z; yv[3] = y4.w; }
      else {   // no residual: the forward output is a function of x alone -- same expression as bn_forward_kernel, so the mask is bit-identical
#pragma unroll
        for (int j = 0; j < 4; ++j) yv[j] = (xv[j] - muv[j]) * rsv[j] * gav[j] + bev[j];
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) if (!(yv[j] > 0.f)) g[j] = 0.f;
    }
    if (dres) {
      float* q = dres + r * lddr + c;
      if (dres_acc) { float4 o = *reinterpret_cast<float4*>(q); o.x += g[0]; o.y += g[1]; o.z += g[2]; o.w += g[3]; *reinterpret_cast<float4*>(q) = o; }
      else *reinterpret_cast<float4*>(q) = make_float4(g[0], g[1], g[2], g[3]);
    }
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float t;
      if (training) {
        const float xh = (xv[j] - muv[j]) * rsv[j];
        t = gav[j] * rsv[j] * (g[j] - sgv[j] * invM - xh * sxv[j] * invM);
      } else {
        t = gav[j] * rsv[j] * g[j];
      }
      if (mask_input && !(xv[j] > 0.f)) t = 0.f;
      o[j] = t;
    }
    *reinterpret_cast<float4*>(dx + r * lddx + c) = make_float4(o[0], o[1], o[2], o[3]);
  }
}
// ws: double[2C] (sum g, sum g*xhat; zeroed here)
// ReLU mask of a residual block: relu_mask (one byte per channel quad, written by rih_bn_forward) or, without it, y (the forward output);
// pass both NULL for non-residual blocks and the mask is recomputed from x (needs beta) -- one tensor read less in each of the two passes
RIH_API int rih_bn_bwd(const float* dy, int lddy, const float* y, int ldy, const unsigned char* relu_mask, const float* x, int ldx,
                       const float* mean, const float* rstd, const float* gamma, const float* beta,
                       float* dx, int lddx, float* dres, int lddr, int dres_acc,
                       float* dgamma, float* dbeta, int param_acc,
                       long long M, int C, int relu, int training, int mask_input,
                       double* ws, cudaStream_t s) {
  RIH_REQUIRE(C % 4 == 0 && lddy % 4 == 0 && ldx % 4 == 0 && lddx % 4 == 0, "bn_bwd: needs C,ld %% 4 == 0");
  RIH_REQUIRE(M < (1ll << 31), "bn_bwd: too many rows");
  RIH_REQUIRE(!relu || y || relu_mask || beta, "bn_bwd: the ReLU mask needs the mask bytes, the forward output or beta");
  RIH_CUDA(cudaMemsetAsync(ws, 0, sizeof(double) * 2 * C, s));
  int gx = cdiv(C, 32);
  int target = cdiv(sm_count() * 8, gx);
  int rows_per_cta = max(64, cdiv(M, target));
  dim3 grid(gx, cdiv(M, rows_per_cta));
  launch_k(bn_bwd_reduce_kernel, grid, 256, 0, s, dy, lddy, y, ldy, relu_mask, x, ldx, mean, rstd, gamma, beta, (int)M, C, rows_per_cta, relu, ws);
  if (int e = check_launch("bn_bwd_reduce")) return e;
  launch_k(bn_bwd_apply_kernel, bn_grid(M, C / 4, 256, ew_ctas(s)), 256, 0, s, dy, lddy, y, ldy, relu_mask, x, ldx, mean, rstd, gamma, beta, ws, dx, lddx,
           dres, lddr, dres_acc, dgamma, dbeta, param_acc, M, C / 4, relu, training, mask_input);
  return check_launch("bn_bwd_apply");
}

// relu backward in place/out of place for Conv->ReLU fused epilogues: dx = dy * (y > 0)
__global__ void relu_bwd_kernel(const float* __restrict__ dy, int lddy, const float* __restrict__ y, int ldy, float* __restrict__ dx, int lddx,
                                long long rows, int C) {
  pdl_sync();
  long long total = rows * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long r; int c; divmod(i, C, total < (1ll << 32), r, c);
    dx[r * lddx + c] = y[r * ldy + c] > 0.f ? dy[r * lddy + c] : 0.f;
  }
}
RIH_API int rih_relu_bwd(const float* dy, int lddy, const float* y, int ldy, float* dx, int lddx, long long rows, int C, cudaStream_t s) {
  if (rows * C == 0) return 0;
  int grid = (int)min(ew_ctas(s), (rows * C + 255) / 256);
  launch_k(relu_bwd_kernel, grid, 256, 0, s, dy, lddy, y, ldy, dx, lddx, rows, C);
  return check_launch("relu_bwd");
}

// ============================================================== max-pool 3x3 / stride 2 / pad 1 (torchvision stem)
// first-max-wins in (r,s) scan order, matching ATen max_pool2d; idx stores r*3+s (uint8)
__global__ void maxpool_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, unsigned char* __restrict__ idx,
                                   int N, int H, int W, int C, int Ho, int Wo) {
  pdl_sync();
  long long total = (long long)N * Ho * Wo * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % C); long long t = i / C; int ow = (int)(t % Wo); t /= Wo; int oh = (int)(t % Ho); int n = (int)(t / Ho);
    float best = -INFINITY; int bi = -1;
    for (int r = 0; r < 3; ++r) {
      int ih = oh * 2 - 1 + r; if ((unsigned)ih >= (unsigned)H) continue;
      for (int s = 0; s < 3; ++s) {
        int iw = ow * 2 - 1 + s; if ((unsigned)iw >= (unsigned)W) continue;
        float v = x[((size_t)(n * H + ih) * W + iw) * C + c];
        if (bi < 0 || v > best || isnan(v)) { best = v; bi = r * 3 + s; }
      }
    }
    y[i] = best; idx[i] = (unsigned char)bi;
  }
}
__global__ void maxpool_bwd_kernel(const float* __restrict__ dy, const unsigned char* __restrict__ idx, float* __restrict__ dx,
                                   int N, int H, int W, int C, int Ho, int Wo) {
  pdl_sync();
  long long total = (long long)N * H * W * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % C); long long t = i / C; int iw = (int)(t % W); t /= W; int ih = (int)(t % H); int n = (int)(t / H);
    float acc = 0.f;
    for (int r = 0; r < 3; ++r) {
      int a = ih + 1 - r; if (a < 0 || (a & 1)) continue; int oh = a >> 1; if (oh >= Ho) continue;
      for (int s = 0; s < 3; ++s) {
        int b = iw + 1 - s; if (b < 0 || (b & 1)) continue; int ow = b >> 1; if (ow >= Wo) continue;
        size_t o = ((size_t)(n * Ho + oh) * Wo + ow) * C + c;
        if (idx[o] == r * 3 + s) acc += dy[o];
      }
    }
    dx[i] = acc;
  }
}
// float4 (4 channels per thread) variants: the 268 MB stem activation is streamed once at full width
__global__ void maxpool4_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, unsigned char* __restrict__ idx,
                                    int N, int H, int W, int C4, int Ho, int Wo) {
  pdl_sync();
  const long long total = (long long)N * Ho * Wo * C4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % C4); long long t = i / C4; int ow = (int)(t % Wo); t /= Wo; int oh = (int)(t % Ho); int n = (int)(t / Ho);
    float best[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
    int bi[4] = {-1, -1, -1, -1};
    for (int r = 0; r < 3; ++r) {
      const int ih = oh * 2 - 1 + r; if ((unsigned)ih >= (unsigned)H) continue;
      for (int s = 0; s < 3; ++s) {
        const int iw = ow * 2 - 1 + s; if ((unsigned)iw >= (unsigned)W) continue;
        const float4 v4 = *reinterpret_cast<const float4*>(x + (((size_t)(n * H + ih) * W + iw) * C4 + c) * 4);
        const float v[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (bi[k] < 0 || v[k] > best[k] || isnan(v[k])) { best[k] = v[k]; bi[k] = r * 3 + s; }
      }
    }
    *reinterpret_cast<float4*>(y + i * 4) = make_float4(best[0], best[1], best[2], best[3]);
    *reinterpret_cast<uchar4*>(idx + i * 4) = make_uchar4((unsigned char)bi[0], (unsigned char)bi[1], (unsigned char)bi[2], (unsigned char)bi[3]);
  }
}
__global__ void maxpool4_bwd_kernel(const float* __restrict__ dy, const unsigned char* __restrict__ idx, float* __restrict__ dx,
                                    int N, int H, int W, int C4, int Ho, int Wo) {
  pdl_sync();
  const long long total = (long long)N * H * W * C4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % C4); long long t = i / C4; int iw = (int)(t % W); t /= W; int ih = (int)(t % H); int n = (int)(t / H);
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int r = 0; r < 3; ++r) {
      const int a = ih + 1 - r; if (a < 0 || (a & 1)) continue; const int oh = a >> 1; if (oh >= Ho) continue;
      for (int s = 0; s < 3; ++s) {
        const int b = iw + 1 - s; if (b < 0 || (b & 1)) continue; const int ow = b >> 1; if (ow >= Wo) continue;
        const size_t o = (((size_t)(n * Ho + oh) * Wo + ow) * C4 + c) * 4;
        const uchar4 id = *reinterpret_cast<const uchar4*>(idx + o);
        const float4 g = *reinterpret_cast<const float4*>(dy + o);
        const unsigned char tag = (unsigned char)(r * 3 + s);
        if (id.x == tag) acc[0] += g.x; if (id.y == tag) acc[1] += g.y; if (id.z == tag) acc[2] += g.z; if (id.w == tag) acc[3] += g.w;
      }
    }
    *reinterpret_cast<float4*>(dx + i * 4) = make_float4(acc[0], acc[1], acc[2], acc[3]);
  }
}
RIH_API int rih_maxpool3x3s2_fwd(const float* x, float* y, unsigned char* idx, int N, int H, int W, int C, cudaStream_t s) {
  int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
  const bool vec = (C % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0 && (reinterpret_cast<uintptr_t>(idx) & 3) == 0;
  long long total = (long long)N * Ho * Wo * (vec ? C / 4 : C);
  int grid = (int)min(ew_ctas(s), (total + 255) / 256);
  if (vec) launch_k(maxpool4_fwd_kernel, grid, 256, 0, s, x, y, idx, N, H, W, C / 4, Ho, Wo);
  else launch_k(maxpool_fwd_kernel, grid, 256, 0, s, x, y, idx, N, H, W, C, Ho, Wo);
  return check_launch("maxpool_fwd");
}
RIH_API int rih_maxpool3x3s2_bwd(const float* dy, const unsigned char* idx, float* dx, int N, int H, int W, int C, cudaStream_t s) {
  int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
  const bool vec = (C % 4 == 0) && ((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(dx)) & 15) == 0 && (reinterpret_cast<uintptr_t>(idx) & 3) == 0;
  long long total = (long long)N * H * W * (vec ? C / 4 : C);
  int grid = (int)min(ew_ctas(s), (total + 255) / 256);
  if (vec) launch_k(maxpool4_bwd_kernel, grid, 256, 0, s, dy, idx, dx, N, H, W, C / 4, Ho, Wo);
  else launch_k(maxpool_bwd_kernel, grid, 256, 0, s, dy, idx, dx, N, H, W, C, Ho, Wo);
  return check_launch("maxpool_bwd");
}

// ============================================================== bilinear x2, align_corners=True (models/encoder.py:51)
__device__ __forceinline__ void bil_coord(int o, float scale, int in, int& i0, int& i1, float& l1) {
  float src = scale * (float)o;
  i0 = (int)src;
  if (i0 > in - 1) i0 = in - 1;
  i1 = i0 + ((i0 < in - 1) ? 1 : 0);
  l1 = src - (float)i0;
}
__global__ void bilinear2x_fwd_kernel(const float* __restrict__ x, int ldx, float* __restrict__ y, int ldy, int N, int H, int W, int C) {
  pdl_sync();
  int Ho = 2 * H, Wo = 2 * W;
  float sh = (Ho > 1) ? (float)(H - 1) / (float)(Ho - 1) : 0.f, sw = (Wo > 1) ? (float)(W - 1) / (float)(Wo - 1) : 0.f;
  long long total = (long long)N * Ho * Wo * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % C); long long t = i / C; int ow = (int)(t % Wo); t /= Wo; int oh = (int)(t % Ho); int n = (int)(t / Ho);
    int h0, h1, w0, w1; float lh, lw;
    bil_coord(oh, sh, H, h0, h1, lh); bil_coord(ow, sw, W, w0, w1, lw);
    float hh = 1.f - lh, ww = 1.f - lw;
    const float* b = x + (size_t)n * H * W * ldx + c;
    float v = hh * (ww * b[((size_t)h0 * W + w0) * ldx] + lw * b[((size_t)h0 * W + w1) * ldx]) +
              lh * (ww * b[((size_t)h1 * W + w0) * ldx] + lw * b[((size_t)h1 * W + w1) * ldx]);
    y[((size_t)(n * Ho + oh) * Wo + ow) * ldy + c] = v;
  }
}
__global__ void bilinear2x_bwd_kernel(const float* __restrict__ dy, int lddy, float* __restrict__ dx, int lddx, int N, int H, int W, int C) {
  pdl_sync();
  int Ho = 2 * H, Wo = 2 * W;
  float sh = (Ho > 1) ? (float)(H - 1) / (float)(Ho - 1) : 0.f, sw = (Wo > 1) ? (float)(W - 1) / (float)(Wo - 1) : 0.f;
  long long total = (long long)N * Ho * Wo * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % C); long long t = i / C; int ow = (int)(t % Wo); t /= Wo; int oh = (int)(t % Ho); int n = (int)(t / Ho);
    int h0, h1, w0, w1; float lh, lw;
    bil_coord(oh, sh, H, h0, h1, lh); bil_coord(ow, sw, W, w0, w1, lw);
    float hh = 1.f - lh, ww = 1.f - lw;
    float g = dy[((size_t)(n * Ho + oh) * Wo + ow) * lddy + c];
    float* b = dx + (size_t)n * H * W * lddx + c;
    atomicAdd(b + ((size_t)h0 * W + w0) * lddx, hh * ww * g);
    atomicAdd(b + ((size_t)h0 * W + w1) * lddx, hh * lw * g);
    atomicAdd(b + ((size_t)h1 * W + w0) * lddx, lh * ww * g);
    atomicAdd(b + ((size_t)h1 * W + w1) * lddx, lh * lw * g);
  }
}
RIH_API int rih_bilinear_up_fwd(const float* x, int ldx, float* y, int ldy, int N, int H, int W, int C, int f, cudaStream_t s);
RIH_API int rih_bilinear_up_bwd(const float* dy, int lddy, float* dx, int lddx, int N, int H, int W, int C, int f, cudaStream_t s);
static inline bool bil_vec_ok(const void* a, int lda, const void* b, int ldb, int C) {
  return C % 4 == 0 && lda % 4 == 0 && ldb % 4 == 0 && ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b)) & 15) == 0;
}
RIH_API int rih_bilinear2x_fwd(const float* x, int ldx, float* y, int ldy, int N, int H, int W, int C, cudaStream_t s) {
  if (bil_vec_ok(x, ldx, y, ldy, C)) return rih_bilinear_up_fwd(x, ldx, y, ldy, N, H, W, C, 2, s);      // float4 kernel
  long long total = (long long)N * 4 * H * W * C;
  int grid = (int)min(ew_ctas(s), (total + 255) / 256);
  launch_k(bilinear2x_fwd_kernel, grid, 256, 0, s, x, ldx, y, ldy, N, H, W, C);
  return check_launch("bilinear2x_fwd");
}
// dx must be zero-initialised by the caller (scatter-add)
RIH_API int rih_bilinear2x_bwd(const float* dy, int lddy, float* dx, int lddx, int N, int H, int W, int C, cudaStream_t s) {
  if (bil_vec_ok(dy, lddy, dx, lddx, C)) return rih_bilinear_up_bwd(dy, lddy, dx, lddx, N, H, W, C, 2, s);   // gather form: overwrites dx, no atomics
  long long total = (long long)N * 4 * H * W * C;
  int grid = (int)min(ew_ctas(s), (total + 255) / 256);
  launch_k(bilinear2x_bwd_kernel, grid, 256, 0, s, dy, lddy, dx, lddx, N, H, W, C);
  return check_launch("bilinear2x_bwd");
}

// ============================================================== bilinear x f, align_corners=True, float4 channels
// F.interpolate(size=(f*H, f*W), mode='bilinear', align_corners=True) of HRnet_encoder.forward (models/encoder.py:227-230): the
// three coarse HRNet branches are up-sampled x2 / x4 / x8 and written straight into their channel slice of the 720-wide concat
// buffer (y points at the slice, ldy is the full row stride), so torch.cat (encoder.py:231) costs no extra pass.
__global__ void bilinear_up4_fwd_kernel(const float* __restrict__ x, int ldx, float* __restrict__ y, int ldy, int N, int H, int W, int C4, int f) {
  pdl_sync();
  const int Ho = f * H, Wo = f * W;
  const float sh = (Ho > 1) ? (float)(H - 1) / (float)(Ho - 1) : 0.f, sw = (Wo > 1) ? (float)(W - 1) / (float)(Wo - 1) : 0.f;
  const long long total = (long long)N * Ho * Wo * C4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % C4); long long t = i / C4; int ow = (int)(t % Wo); t /= Wo; int oh = (int)(t % Ho); int n = (int)(t / Ho);
    int h0, h1, w0, w1; float lh, lw;
    bil_coord(oh, sh, H, h0, h1, lh); bil_coord(ow, sw, W, w0, w1, lw);
    const float hh = 1.f - lh, ww = 1.f - lw;
    const float* b = x + (size_t)n * H * W * ldx + c * 4;
    const float4 a00 = *reinterpret_cast<const float4*>(b + ((size_t)h0 * W + w0) * ldx), a01 = *reinterpret_cast<const float4*>(b + ((size_t)h0 * W + w1) * ldx);
    const float4 a10 = *reinterpret_cast<const float4*>(b + ((size_t)h1 * W + w0) * ldx), a11 = *reinterpret_cast<const float4*>(b + ((size_t)h1 * W + w1) * ldx);
    float4 v;
    v.x = hh * (ww * a00.x + lw * a01.x) + lh * (ww * a10.x + lw * a11.x);
    v.y = hh * (ww * a00.y + lw * a01.y) + lh * (ww * a10.y + lw * a11.y);
    v.z = hh * (ww * a00.z + lw * a01.z) + lh * (ww * a10.z + lw * a11.z);
    v.w = hh * (ww * a00.w + lw * a01.w) + lh * (ww * a10.w + lw * a11.w);
    *reinterpret_cast<float4*>(y + ((size_t)(n * Ho + oh) * Wo + ow) * ldy + c * 4) = v;
  }
}
// backward as a gather: every input pixel (h, w) sums the contributions of the output pixels whose interpolation window
// touches it (rows oh with src(oh) in (h-1, h+1)), no atomics, deterministic.
__global__ void bilinear_up4_bwd_kernel(const float* __restrict__ dy, int lddy, float* __restrict__ dx, int lddx, int N, int H, int W, int C4, int f) {
  pdl_sync();
  const int Ho = f * H, Wo = f * W;
  const float sh = (Ho > 1) ? (float)(H - 1) / (float)(Ho - 1) : 0.f, sw = (Wo > 1) ? (float)(W - 1) / (float)(Wo - 1) : 0.f;
  const long long total = (long long)N * H * W * C4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % C4); long long t = i / C4; int w = (int)(t % W); t /= W; int h = (int)(t % H); int n = (int)(t / H);
    // candidate output rows: src = sh * oh in (h - 1, h + 1)  ->  oh in ((h-1)/sh, (h+1)/sh); scan a safe superset and test exactly
    const int oh_lo = max(0, (h - 1) * f - f), oh_hi = min(Ho - 1, (h + 1) * f + f);
    const int ow_lo = max(0, (w - 1) * f - f), ow_hi = min(Wo - 1, (w + 1) * f + f);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int oh = oh_lo; oh <= oh_hi; ++oh) {
      int h0, h1; float lh;
      bil_coord(oh, sh, H, h0, h1, lh);
      float wh = 0.f;
      if (h0 == h) wh += 1.f - lh;
      if (h1 == h) wh += lh;
      if (wh == 0.f) continue;
      for (int ow = ow_lo; ow <= ow_hi; ++ow) {
        int w0, w1; float lw;
        bil_coord(ow, sw, W, w0, w1, lw);
        float wwt = 0.f;
        if (w0 == w) wwt += 1.f - lw;
        if (w1 == w) wwt += lw;
        if (wwt == 0.f) continue;
        const float4 g = *reinterpret_cast<const float4*>(dy + ((size_t)(n * Ho + oh) * Wo + ow) * lddy + c * 4);
        const float k = wh * wwt;
        acc.x = fmaf(k, g.x, acc.x); acc.y = fmaf(k, g.y, acc.y); acc.z = fmaf(k, g.z, acc.z); acc.w = fmaf(k, g.w, acc.w);
      }
    }
    *reinterpret_cast<float4*>(dx + ((size_t)(n * H + h) * W + w) * lddx + c * 4) = acc;
  }
}
RIH_API int rih_bilinear_up_fwd(const float* x, int ldx, float* y, int ldy, int N, int H, int W, int C, int f, cudaStream_t s) {
  RIH_REQUIRE(f >= 1 && C % 4 == 0 && ldx % 4 == 0 && ldy % 4 == 0 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0,
              "bilinear_up_fwd: needs C, strides multiples of 4 floats and 16-byte aligned pointers (C=%d ldx=%d ldy=%d)", C, ldx, ldy);
  long long total = (long long)N * f * H * f * W * (C / 4);
  if (total == 0) return 0;
  int grid = (int)min(ew_ctas(s), (total + 255) / 256);
  launch_k(bilinear_up4_fwd_kernel, grid, 256, 0, s, x, ldx, y, ldy, N, H, W, C / 4, f);
  return check_launch("bilinear_up_fwd");
}
// dx[N*H*W, C] = adjoint of rih_bilinear_up_fwd applied to dy[N*fH*fW, C] (row stride lddy); overwrites dx
RIH_API int rih_bilinear_up_bwd(const float* dy, int lddy, float* dx, int lddx, int N, int H, int W, int C, int f, cudaStream_t s) {
  RIH_REQUIRE(f >= 1 && C % 4 == 0 && lddx % 4 == 0 && lddy % 4 == 0 && ((reinterpret_cast<uintptr_t>(dx) | reinterpret_cast<uintptr_t>(dy)) & 15) == 0,
              "bilinear_up_bwd: needs C, strides multiples of 4 floats and 16-byte aligned pointers");
  long long total = (long long)N * H * W * (C / 4);
  if (total == 0) return 0;
  int grid = (int)min(ew_ctas(s), (total + 127) / 128);
  launch_k(bilinear_up4_bwd_kernel, grid, 128, 0, s, dy, lddy, dx, lddx, N, H, W, C / 4, f);
  return check_launch("bilinear_up_bwd");
}

// ============================================================== HRNet fuse: y = act(sum_j nearest_up(t_j, f_j))
// HighResolutionModule.forward (models/model_zoo/hrnet.py:222-230): y = x[0]; y = y + fuse(x[j]) ...; relu(y).  Terms coming from a
// coarser branch carry nn.Upsample(scale_factor=2^(j-i), mode='nearest') (hrnet.py:185); it is folded into the read index here.
// Terms are added in list order (the reference's left-to-right association).
struct FuseTerms { const float* p[4]; int ld[4]; int f[4]; int n; };
__global__ void fuse_sum_kernel(FuseTerms a, float* __restrict__ y, int ldy, int N, int H, int W, int C4, int relu) {
  pdl_sync();
  const long long total = (long long)N * H * W * C4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % C4); long long t = i / C4; int w = (int)(t % W); t /= W; int h = (int)(t % H); int n = (int)(t / H);
    float4 acc;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (j < a.n) {
        const int f = a.f[j], Hj = H / f, Wj = W / f;
        const float4 v = *reinterpret_cast<const float4*>(a.p[j] + ((size_t)(n * Hj + h / f) * Wj + w / f) * a.ld[j] + c * 4);
        if (j == 0) acc = v;
        else { acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w; }
      }
    }
    if (relu) { acc.x = fmaxf(acc.x, 0.f); acc.y = fmaxf(acc.y, 0.f); acc.z = fmaxf(acc.z, 0.f); acc.w = fmaxf(acc.w, 0.f); }
    *reinterpret_cast<float4*>(y + ((size_t)(n * H + h) * W + w) * ldy + c * 4) = acc;
  }
}
RIH_API int rih_fuse_sum(const float* const* terms, const int* lds, const int* factors, int nterms, float* y, int ldy,
                         int N, int H, int W, int C, int relu, cudaStream_t s) {
  RIH_REQUIRE(nterms >= 1 && nterms <= 4 && C % 4 == 0 && ldy % 4 == 0, "fuse_sum: 1..4 terms, channels multiple of 4");
  FuseTerms a;
  a.n = nterms;
  for (int j = 0; j < 4; ++j) {
    a.p[j] = j < nterms ? terms[j] : nullptr; a.ld[j] = j < nterms ? lds[j] : 0; a.f[j] = j < nterms ? factors[j] : 1;
    if (j < nterms) RIH_REQUIRE(a.f[j] >= 1 && H % a.f[j] == 0 && W % a.f[j] == 0 && a.ld[j] % 4 == 0 && (reinterpret_cast<uintptr_t>(a.p[j]) & 15) == 0,
                                "fuse_sum: term %d has a bad factor / stride / alignment", j);
  }
  long long total = (long long)N * H * W * (C / 4);
  if (total == 0) return 0;
  int grid = (int)min(ew_ctas(s), (total + 255) / 256);
  launch_k(fuse_sum_kernel, grid, 256, 0, s, a, y, ldy, N, H, W, C / 4, relu);
  return check_launch("fuse_sum");
}
// adjoint of a nearest x f up-sample: dx[n,h,w,:] = sum_{a,b<f} (y > 0 ? dy : 0)[n, f*h+a, f*w+b, :]   (y == nullptr: no mask)
__global__ void pool_sum_kernel(const float* __restrict__ dy, int lddy, const float* __restrict__ y, int ldy, float* __restrict__ dx, int lddx,
                                int N, int H, int W, int C4, int f) {
  pdl_sync();
  const long long total = (long long)N * H * W * C4;
  const int Hf = H * f, Wf = W * f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % C4); long long t = i / C4; int w = (int)(t % W); t /= W; int h = (int)(t % H); int n = (int)(t / H);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int a = 0; a < f; ++a)
      for (int b = 0; b < f; ++b) {
        const size_t row = (size_t)(n * Hf + h * f + a) * Wf + w * f + b;
        float4 g = *reinterpret_cast<const float4*>(dy + row * lddy + c * 4);
        if (y) {
          const float4 m = *reinterpret_cast<const float4*>(y + row * ldy + c * 4);
          g.x = m.x > 0.f ? g.x : 0.f; g.y = m.y > 0.f ? g.y : 0.f; g.z = m.z > 0.f ? g.z : 0.f; g.w = m.w > 0.f ? g.w : 0.f;
        }
        acc.x += g.x; acc.y += g.y; acc.z += g.z; acc.w += g.w;
      }
    *reinterpret_cast<float4*>(dx + ((size_t)(n * H + h) * W + w) * lddx + c * 4) = acc;
  }
}
// H, W are the COARSE (output) sizes; dy / y are [N, f*H, f*W, C]
RIH_API int rih_pool_sum(const float* dy, int lddy, const float* y, int ldy, float* dx, int lddx, int N, int H, int W, int C, int f, cudaStream_t s) {
  RIH_REQUIRE(f >= 1 && C % 4 == 0 && lddy % 4 == 0 && lddx % 4 == 0 && (!y || ldy % 4 == 0), "pool_sum: channels / strides must be multiples of 4");
  long long total = (long long)N * H * W * (C / 4);
  if (total == 0) return 0;
  int grid = (int)min(ew_ctas(s), (total + 127) / 128);
  launch_k(pool_sum_kernel, grid, 128, 0, s, dy, lddy, y, ldy, dx, lddx, N, H, W, C / 4, f);
  return check_launch("pool_sum");
}

// ============================================================== global average pool [N, HW, C] -> [N, C]
__global__ void gap_fwd_kernel(const float* __restrict__ x, int ldx, float* __restrict__ y, int N, int HW, int C) {
  pdl_sync();
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * C) return;
  int n = i / C, c = i - n * C;
  float s = 0.f;
  for (int p = 0; p < HW; ++p) s += x[((size_t)n * HW + p) * ldx + c];
  y[i] = s / (float)HW;
}
__global__ void gap_bwd_kernel(const float* __restrict__ dy, float* __restrict__ dx, int lddx, int N, int HW, int C, int acc) {
  pdl_sync();
  long long total = (long long)N * HW * C;
  float inv = 1.f / (float)HW;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % C); long long t = i / C; int n = (int)(t / HW);
    float v = dy[(size_t)n * C + c] * inv;
    float* q = dx + t * lddx + c;
    *q = acc ? *q + v : v;
  }
}
RIH_API int rih_gap_fwd(const float* x, int ldx, float* y, int N, int HW, int C, cudaStream_t s) {
  launch_k(gap_fwd_kernel, cdiv((long long)N * C, 256), 256, 0, s, x, ldx, y, N, HW, C);
  return check_launch("gap_fwd");
}
RIH_API int rih_gap_bwd(const float* dy, float* dx, int lddx, int N, int HW, int C, int accumulate, cudaStream_t s) {
  long long total = (long long)N * HW * C;
  int grid = (int)min(ew_ctas(s), (total + 255) / 256);
  launch_k(gap_bwd_kernel, grid, 256, 0, s, dy, dx, lddx, N, HW, C, accumulate);
  return check_launch("gap_bwd");
}

// ============================================================== stride-2 helpers for the tensor-core convolution path
// parity stack: xp[(ph*2+pw)*N + n, i, j, :] = x[n, 2i+ph, 2j+pw, :]   (space-to-depth by pixel parity, H and W even)
__global__ void parity_stack_kernel(const float* __restrict__ x, int ldx, float* __restrict__ xp, int N, int H, int W, int C4) {
  pdl_sync();
  const int H2 = H / 2, W2 = W / 2;
  long long total = (long long)N * H * W * C4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % C4); long long t = i / C4; int w = (int)(t % W); t /= W; int h = (int)(t % H); int n = (int)(t / H);
    float4 v = *reinterpret_cast<const float4*>(x + ((size_t)(n * H + h) * W + w) * ldx + c * 4);
    int p = (h & 1) * 2 + (w & 1);
    *reinterpret_cast<float4*>(xp + ((((size_t)p * N + n) * H2 + (h >> 1)) * W2 + (w >> 1)) * (size_t)(C4 * 4) + c * 4) = v;
  }
}
RIH_API int rih_parity_stack(const float* x, int ldx, float* xp, int N, int H, int W, int C, cudaStream_t s) {
  RIH_REQUIRE(H % 2 == 0 && W % 2 == 0 && C % 4 == 0 && ldx % 4 == 0, "parity_stack: H, W must be even and C, ld multiples of 4");
  long long total = (long long)N * H * W * (C / 4);
  int grid = (int)min(ew_ctas(s), (total + 255) / 256);
  launch_k(parity_stack_kernel, grid, 256, 0, s, x, ldx, xp, N, H, W, C / 4);
  return check_launch("parity_stack");
}
// zero insertion: yd[n, 2i, 2j, :] = y[n, i, j, :], 0 elsewhere (yd is [N, 2Ho, 2Wo, C] contiguous)
__global__ void dilate2x_kernel(const float* __restrict__ y, int ldy, float* __restrict__ yd, int N, int Ho, int Wo, int C4) {
  pdl_sync();
  const int H = 2 * Ho, W = 2 * Wo;
  long long total = (long long)N * H * W * C4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % C4); long long t = i / C4; int w = (int)(t % W); t /= W; int h = (int)(t % H); int n = (int)(t / H);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!((h | w) & 1)) v = *reinterpret_cast<const float4*>(y + ((size_t)(n * Ho + (h >> 1)) * Wo + (w >> 1)) * ldy + c * 4);
    reinterpret_cast<float4*>(yd)[i] = v;
  }
}
RIH_API int rih_dilate2x(const float* y, int ldy, float* yd, int N, int Ho, int Wo, int C, cudaStream_t s) {
  RIH_REQUIRE(C % 4 == 0 && ldy % 4 == 0, "dilate2x: C, ld must be multiples of 4");
  long long total = (long long)N * 4 * Ho * Wo * (C / 4);
  int grid = (int)min(ew_ctas(s), (total + 255) / 256);
  launch_k(dilate2x_kernel, grid, 256, 0, s, y, ldy, yd, N, Ho, Wo, C / 4);
  return check_launch("dilate2x");
}

// ============================================================== non-overlapping patches (kernel == stride): im2col without blow-up
// P[(n,gh,gw), (r,s,c)] = x[n, p*gh+r, p*gw+s, c]   -- img_feat_to_grid.proj, models/model_attn/img_attn.py:48,60
__global__ void patchify_kernel(const float* __restrict__ x, int ldx, float* __restrict__ P, int N, int H, int W, int C4, int p, int scatter) {
  pdl_sync();
  const int gh_n = H / p, gw_n = W / p;
  long long total = (long long)N * H * W * C4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % C4); long long t = i / C4; int s_ = (int)(t % p); t /= p; int r = (int)(t % p); t /= p;
    int gw = (int)(t % gw_n); t /= gw_n; int gh = (int)(t % gh_n); int n = (int)(t / gh_n);
    float* px = const_cast<float*>(x) + ((size_t)(n * H + gh * p + r) * W + gw * p + s_) * ldx + c * 4;
    float* pp = P + (size_t)i * 4;
    if (!scatter) *reinterpret_cast<float4*>(pp) = *reinterpret_cast<const float4*>(px);
    else *reinterpret_cast<float4*>(px) = *reinterpret_cast<const float4*>(pp);
  }
}
// scatter = 0: P <- patches of x ; scatter = 1: x <- P (the exact inverse; used for the gradient)
RIH_API int rih_patchify(float* x, int ldx, float* P, int N, int H, int W, int C, int p, int scatter, cudaStream_t s) {
  RIH_REQUIRE(p >= 1 && H % p == 0 && W % p == 0 && C % 4 == 0 && ldx % 4 == 0, "patchify: bad geometry");
  long long total = (long long)N * H * W * (C / 4);
  int grid = (int)min(ew_ctas(s), (total + 255) / 256);
  launch_k(patchify_kernel, grid, 256, 0, s, x, ldx, P, N, H, W, C / 4, p, scatter);
  return check_launch("patchify");
}

// ============================================================== explicit im2col for few-channel convolutions (the 7x7/2 RGB stem)
// A[(n,oh,ow), (r,s,c)] = x[n, oh*stride+r-pad, ow*stride+s-pad, c] (0 outside), columns >= R*S*C zero-padded up to Kpad.
// With Cin = 3 the implicit-GEMM gathers cannot be vectorised or fed by TMA; materialising the 147(+13)-wide rows once lets the
// stem run as a dense tensor-core GEMM (forward) and a dense split-K GEMM (weight gradient).
// TR/TS/TC > 0: compile-time filter shape (constant divisions); 0 = runtime shape
template <int TR, int TS, int TC>
__global__ void im2col_kernel(const float* __restrict__ x, int ldx, float* __restrict__ A, int N, int H, int W, int C_, int Ho, int Wo,
                              int R_, int S_, int stride, int pad, int Kpad) {
  pdl_sync();
  const int R = TR > 0 ? TR : R_, S = TS > 0 ? TS : S_, C = TC > 0 ? TC : C_;
  const long long total = (long long)N * Ho * Wo * Kpad;
  const bool small = total < (1ll << 32);
  const int K = R * S * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long m; int k;
    divmod(i, Kpad, small, m, k);
    float v = 0.f;
    if (k < K) {
      const int c = k % C, rs = k / C, s_ = rs % S, r = rs / S;
      const int ow = (int)(m % Wo); const long long t = m / Wo; const int oh = (int)(t % Ho), n = (int)(t / Ho);
      const int ih = oh * stride - pad + r, iw = ow * stride - pad + s_;
      if ((unsigned)ih < (unsigned)H && (unsigned)iw < (unsigned)W) v = x[((size_t)(n * H + ih) * W + iw) * ldx + c];
    }
    A[i] = v;
  }
}
// float4 stores: one thread per 4 consecutive columns of a row of A.  Within a filter row r the S*C columns map to S*C CONTIGUOUS
// floats of the NHWC input (pixels iw0 .. iw0+S-1, all channels), so neighbouring threads read neighbouring addresses.
template <int TR, int TS, int TC>
__global__ void im2col4_kernel(const float* __restrict__ x, int ldx, float* __restrict__ A, int N, int H, int W, int Ho, int Wo,
                               int stride, int pad, int Kpad4) {
  pdl_sync();
  constexpr int K = TR * TS * TC, SC = TS * TC;
  const long long total = (long long)N * Ho * Wo * Kpad4;
  const bool small = total < (1ll << 32);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long m; int k4;
    divmod(i, Kpad4, small, m, k4);
    const int ow = (int)(m % Wo); const long long t = m / Wo; const int oh = (int)(t % Ho), n = (int)(t / Ho);
    const int ih0 = oh * stride - pad, iw0 = ow * stride - pad;
    float v[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int k = k4 * 4 + e;
      v[e] = 0.f;
      if (k < K) {
        const int r = k / SC, off = k - r * SC, s_ = off / TC, c = off - s_ * TC;
        const int ih = ih0 + r, iw = iw0 + s_;
        if ((unsigned)ih < (unsigned)H && (unsigned)iw < (unsigned)W) v[e] = __ldg(x + ((size_t)(n * H + ih) * W + iw) * ldx + c);
      }
    }
    reinterpret_cast<float4*>(A)[i] = make_float4(v[0], v[1], v[2], v[3]);
  }
}
RIH_API int rih_im2col(const float* x, int ldx, float* A, int N, int H, int W, int C, int R, int S, int stride, int pad, int Kpad, cudaStream_t s) {
  RIH_REQUIRE(Kpad >= R * S * C && Kpad % 4 == 0, "im2col: Kpad must be a multiple of 4 and >= R*S*C");
  const int Ho = (H + 2 * pad - R) / stride + 1, Wo = (W + 2 * pad - S) / stride + 1;
  const long long total = (long long)N * Ho * Wo * Kpad;
  if ((reinterpret_cast<uintptr_t>(A) & 15) == 0 && C == 3 && R == S && (R == 7 || R == 3)) {
    const int g4 = (int)min((long long)sm_count() * 32, (total / 4 + 255) / 256);
    if (R == 7) launch_k(im2col4_kernel<7, 7, 3>, g4, 256, 0, s, x, ldx, A, N, H, W, Ho, Wo, stride, pad, Kpad / 4);
    else launch_k(im2col4_kernel<3, 3, 3>, g4, 256, 0, s, x, ldx, A, N, H, W, Ho, Wo, stride, pad, Kpad / 4);
    return check_launch("im2col");
  }
  int grid = (int)min((long long)sm_count() * 32, (total + 255) / 256);
  if (R == 7 && S == 7 && C == 3) launch_k(im2col_kernel<7, 7, 3>, grid, 256, 0, s, x, ldx, A, N, H, W, C, Ho, Wo, R, S, stride, pad, Kpad);
  else if (R == 3 && S == 3 && C == 3) launch_k(im2col_kernel<3, 3, 3>, grid, 256, 0, s, x, ldx, A, N, H, W, C, Ho, Wo, R, S, stride, pad, Kpad);   // HRNet stem
  else launch_k(im2col_kernel<0, 0, 0>, grid, 256, 0, s, x, ldx, A, N, H, W, C, Ho, Wo, R, S, stride, pad, Kpad);
  return check_launch("im2col");
}

// ============================================================== input pipeline on the GPU (SURVEY 8 f4)
// uint8 HWC BGR frames (what cv.imread / the reference's datasets hold) -> normalised float32 NCHW RGB network input, with the optional
// horizontal flip of the augmentation: the per-sample host work of core/loader.py:151-152 (cv.flip), :178-181 (cv.cvtColor BGR2RGB,
// / 255, permute(2,0,1), transforms.Normalize(mean, std)).  Same operation order (divide by 255, subtract mean, divide by std) so the
// result is bit-identical to the torch / torchvision ops; the host -> device copy shrinks 4x (uint8 instead of float32).
__global__ void preprocess_u8_kernel(const unsigned char* __restrict__ src, const unsigned char* __restrict__ flip, float* __restrict__ dst,
                                     int B, int H, int W, float m0, float m1, float m2, float s0, float s1, float s2) {
  pdl_sync();
  const long long total = (long long)B * H * W;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(i % W); const long long t = i / W; const int y = (int)(t % H); const int b = (int)(t / H);
    const int sx = (flip && flip[b]) ? (W - 1 - x) : x;
    const unsigned char* p = src + (((size_t)b * H + y) * W + sx) * 3;
    const float bl = (float)p[0] / 255.f, gr = (float)p[1] / 255.f, rd = (float)p[2] / 255.f;
    float* o = dst + (size_t)b * 3 * H * W + (size_t)y * W + x;
    o[0] = (rd - m0) / s0;
    o[(size_t)H * W] = (gr - m1) / s1;
    o[2 * (size_t)H * W] = (bl - m2) / s2;
  }
}
// src: [B,H,W,3] uint8 BGR; flip: [B] uint8 flags or NULL; dst: [B,3,H,W] float32 RGB, (x/255 - mean[c]) / std[c]
RIH_API int rih_preprocess_u8(const unsigned char* src, const unsigned char* flip, float* dst, int B, int H, int W,
                              const float* mean3_host, const float* std3_host, cudaStream_t s) {
  RIH_REQUIRE(B >= 0 && H > 0 && W > 0, "preprocess_u8: bad shape");
  const long long total = (long long)B * H * W;
  if (total == 0) return 0;
  int grid = (int)min(ew_ctas(s), (total + 255) / 256);
  launch_k(preprocess_u8_kernel, grid, 256, 0, s, src, flip, dst, B, H, W, mean3_host[0], mean3_host[1], mean3_host[2], std3_host[0], std3_host[1], std3_host[2]);
  return check_launch("preprocess_u8");
}

// ---------------------------------------------------------------- eval-mode BatchNorm folding
// One launch folds EVERY BatchNorm of a network into per-channel (scale, shift) vectors for rih_conv2d_bn_eval_fwd:
//   table[4 b .. 4 b + 3] = device addresses of (gamma, beta, running_mean, running_var) of BatchNorm b,  chan_bn[i] = the BatchNorm that owns
//   flat channel i,  bn_off[b] = its first flat channel.  Reads the live parameter / buffer storage, so a CUDA graph that replays this launch
//   always sees the current running statistics.
__global__ void bn_fold_kernel(const unsigned long long* __restrict__ table, const int* __restrict__ chan_bn, const int* __restrict__ bn_off,
                               const float* __restrict__ eps, float* __restrict__ scale, float* __restrict__ shift, int total) {
  pdl_sync();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int b = chan_bn[i], c = i - bn_off[b];
  const float* gamma = reinterpret_cast<const float*>(table[4 * b]);
  const float* beta = reinterpret_cast<const float*>(table[4 * b + 1]);
  const float* mean = reinterpret_cast<const float*>(table[4 * b + 2]);
  const float* var = reinterpret_cast<const float*>(table[4 * b + 3]);
  const float sc = gamma[c] * (1.0f / sqrtf(var[c] + eps[b]));
  scale[i] = sc;
  shift[i] = beta[c] - mean[c] * sc;
}

RIH_API int rih_bn_fold(const unsigned long long* table, const int* chan_bn, const int* bn_off, const float* eps, float* scale, float* shift,
                        int total, cudaStream_t s) {
  RIH_REQUIRE(table && chan_bn && bn_off && eps && scale && shift && total > 0, "bn_fold: null argument / empty table");
  launch_k(bn_fold_kernel, dim3((total + 255) / 256), dim3(256), 0, s, table, chan_bn, bn_off, eps, scale, shift, total);
  return check_launch("bn_fold");
}
