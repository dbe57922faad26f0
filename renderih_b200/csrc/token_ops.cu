// Token-side kernels of the DualGraph decoder: LayerNorm, Chebyshev SpMM (+[x, Lx] interleave),
// position-embedding add (+ nearest x2 vertex upsample), column sums, dropout, global-feature broadcast.
#include "common.cuh"
#include "adam.cuh"
using namespace rih;

// ============================================================== LayerNorm
// reference call sites (eps 1e-6): models/model_attn/gcn.py:91-97,103-110 ; self_attn.py:20,60 ; decoder.py:91-93
// y = LN(a (+ b)) * gamma + beta, optional ReLU.  One warp per row.
__global__ void layernorm_fwd_kernel(const float* __restrict__ a, int lda, const float* __restrict__ b, int ldb,
                                     const float* __restrict__ gamma, const float* __restrict__ beta,
                                     float* __restrict__ y, int ldy, float* __restrict__ mean, float* __restrict__ rstd,
                                     int M, int F, float eps, int relu) {
  pdl_sync();
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int r = warp; r < M; r += nwarps) {
    const float* pa = a + (size_t)r * lda;
    const float* pb = b ? b + (size_t)r * ldb : nullptr;
    float s = 0.f;
    for (int c = lane; c < F; c += 32) s += pa[c] + (pb ? pb[c] : 0.f);
    float mu = warp_sum(s) / (float)F;
    float ss = 0.f;
    for (int c = lane; c < F; c += 32) { float d = pa[c] + (pb ? pb[c] : 0.f) - mu; ss += d * d; }
    float rs = 1.f / sqrtf(warp_sum(ss) / (float)F + eps);
    if (lane == 0) { mean[r] = mu; rstd[r] = rs; }
    float* py = y + (size_t)r * ldy;
    for (int c = lane; c < F; c += 32) {
      float v = (pa[c] + (pb ? pb[c] : 0.f) - mu) * rs * gamma[c] + beta[c];
      py[c] = relu ? fmaxf(v, 0.f) : v;
    }
  }
}
RIH_API int rih_layernorm_fwd(const float* a, int lda, const float* b, int ldb, const float* gamma, const float* beta,
                              float* y, int ldy, float* mean, float* rstd, int M, int F, float eps, int relu, cudaStream_t s) {
  if (M == 0) return 0;
  int grid = min(sm_count() * 8, cdiv(M, 8));
  launch_k(layernorm_fwd_kernel, grid, 256, 0, s, a, lda, b, ldb, gamma, beta, y, ldy, mean, rstd, M, F, eps, relu);
  return check_launch("layernorm_fwd");
}

// dx = rstd * (g*gamma - mean_c(g*gamma) - xhat * mean_c(g*gamma*xhat)), g = dy * (y>0 if relu)
// dgamma += sum_r g*xhat ; dbeta += sum_r g        (F <= 32*LN_MAXC)
// MAXC = columns per lane (F <= 32 * MAXC), THREADS per CTA: narrow rows use 32 warps per CTA so that a warp walks only a few rows
// (the per-row dependent chain load -> 2 warp reductions -> store is latency bound) while the per-CTA parameter-gradient atomics stay few.
template <int MAXC, int THREADS>
__global__ void __launch_bounds__(THREADS)
layernorm_bwd_kernel(const float* __restrict__ dy, int lddy, const float* __restrict__ a, int lda,
                     const float* __restrict__ b, int ldb, const float* __restrict__ gamma, const float* __restrict__ beta,
                     const float* __restrict__ mean, const float* __restrict__ rstd,
                     float* __restrict__ dx, int lddx, int dx_acc, float* __restrict__ dgamma, float* __restrict__ dbeta,
                     int M, int F, int relu) {
  pdl_sync();
  constexpr int WARPS = THREADS / 32;
  int warp_in_cta = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int warp = blockIdx.x * WARPS + warp_in_cta;
  int nwarps = gridDim.x * WARPS;
  float ag[MAXC], ab[MAXC], gam[MAXC], bet[MAXC];
#pragma unroll
  for (int j = 0; j < MAXC; ++j) {
    const int c = lane + 32 * j;
    ag[j] = 0.f; ab[j] = 0.f;
    gam[j] = c < F ? gamma[c] : 0.f; bet[j] = (c < F && relu) ? beta[c] : 0.f;
  }
  for (int r = warp; r < M; r += nwarps) {
    const float* pa = a + (size_t)r * lda;
    const float* pb = b ? b + (size_t)r * ldb : nullptr;
    const float* pg = dy + (size_t)r * lddy;
    float mu = mean[r], rs = rstd[r];
    float s1 = 0.f, s2 = 0.f;
    float gg[MAXC], xh[MAXC];
#pragma unroll
    for (int j = 0; j < MAXC; ++j) {
      int c = lane + 32 * j;
      gg[j] = 0.f; xh[j] = 0.f;
      if (c < F) {
        float x = pa[c] + (pb ? pb[c] : 0.f);
        float h = (x - mu) * rs;
        float g = pg[c];
        if (relu && !(h * gam[j] + bet[j] > 0.f)) g = 0.f;
        ag[j] += g * h; ab[j] += g;
        float gw = g * gam[j];
        gg[j] = gw; xh[j] = h;
        s1 += gw; s2 += gw * h;
      }
    }
    s1 = warp_sum(s1) / (float)F; s2 = warp_sum(s2) / (float)F;
    float* pd = dx + (size_t)r * lddx;
#pragma unroll
    for (int j = 0; j < MAXC; ++j) {
      int c = lane + 32 * j;
      if (c < F) {
        float v = rs * (gg[j] - s1 - xh[j] * s2);
        pd[c] = dx_acc ? pd[c] + v : v;
      }
    }
  }
  // CTA reduction of the parameter gradients, then one atomicAdd per column per CTA
  __shared__ float sg[WARPS][32 * MAXC + 1];
  __shared__ float sb[WARPS][32 * MAXC + 1];
#pragma unroll
  for (int j = 0; j < MAXC; ++j) { sg[warp_in_cta][lane + 32 * j] = ag[j]; sb[warp_in_cta][lane + 32 * j] = ab[j]; }
  __syncthreads();
  for (int c = threadIdx.x; c < F; c += THREADS) {
    float g = 0.f, bb = 0.f;
    for (int w = 0; w < WARPS; ++w) { g += sg[w][c]; bb += sb[w][c]; }
    if (dgamma) atomicAdd(dgamma + c, g);
    if (dbeta) atomicAdd(dbeta + c, bb);
  }
}
// dgamma / dbeta are ACCUMULATED into (caller zeroes them at step start)
RIH_API int rih_layernorm_bwd(const float* dy, int lddy, const float* a, int lda, const float* b, int ldb,
                              const float* gamma, const float* beta, const float* mean, const float* rstd,
                              float* dx, int lddx, int dx_acc, float* dgamma, float* dbeta, int M, int F, int relu, cudaStream_t s) {
  RIH_REQUIRE(F <= 512, "layernorm_bwd: F=%d exceeds 512", F);
  if (M == 0) return 0;
#define RIH_LN_BWD(MC, TH)                                                                                                        \
  launch_k(layernorm_bwd_kernel<MC, TH>, min(sm_count() * (1024 / TH), cdiv(M, TH / 32)), TH, 0, s, dy, lddy, a, lda, b, ldb, gamma, beta, mean, rstd, dx, lddx, dx_acc, \
                                                                                      dgamma, dbeta, M, F, relu)
  if (F <= 64) RIH_LN_BWD(2, 1024);
  else if (F <= 128) RIH_LN_BWD(4, 1024);
  else if (F <= 256) RIH_LN_BWD(8, 512);
  else RIH_LN_BWD(16, 256);
#undef RIH_LN_BWD
  return check_launch("layernorm_bwd");
}

// ============================================================== Chebyshev K=2 basis: out[b,v,f,0] = x[b,v,f]; out[b,v,f,1] = (L x)[b,v,f]
// reference: graph_conv_cheby, models/model_attn/gcn.py:34-69 (dense torch.mm(L, x0) at :54 and the Fin x K interleave at :61-63)
__global__ void cheb_fwd_kernel(const float* __restrict__ x, int ldx, const int* __restrict__ rowptr, const int* __restrict__ col,
                                const float* __restrict__ val, float* __restrict__ out, int B, int V, int F) {
  pdl_sync();
  long long total = (long long)B * V * F;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int f = (int)(i % F); long long t = i / F; int v = (int)(t % V); int b = (int)(t / V);
    const float* xb = x + (size_t)b * V * ldx + f;
    float acc = 0.f;
    for (int e = rowptr[v]; e < rowptr[v + 1]; ++e) acc = fmaf(val[e], xb[(size_t)col[e] * ldx], acc);
    reinterpret_cast<float2*>(out)[i] = make_float2(xb[(size_t)v * ldx], acc);
  }
}
// dx[b,v,f] (+)= d[b,v,f,0] + sum_u L[u,v] d[b,u,f,1]   (CSR of L^T passed in)
__global__ void cheb_bwd_kernel(const float* __restrict__ d, const int* __restrict__ rowptr, const int* __restrict__ col,
                                const float* __restrict__ val, float* __restrict__ dx, int lddx, int acc_flag, int B, int V, int F) {
  pdl_sync();
  long long total = (long long)B * V * F;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int f = (int)(i % F); long long t = i / F; int v = (int)(t % V); int b = (int)(t / V);
    const float* db = d + (size_t)b * V * F * 2 + 2 * f;
    float acc = db[(size_t)v * F * 2];
    for (int e = rowptr[v]; e < rowptr[v + 1]; ++e) acc = fmaf(val[e], db[(size_t)col[e] * F * 2 + 1], acc);
    float* q = dx + ((size_t)b * V + v) * lddx + f;
    *q = acc_flag ? *q + acc : acc;
  }
}
// float4 variants (F % 4 == 0): 4 features per thread, 16-byte gathers of the <= 11 neighbours of a vertex
__global__ void cheb4_fwd_kernel(const float* __restrict__ x, int ldx, const int* __restrict__ rowptr, const int* __restrict__ col,
                                 const float* __restrict__ val, float* __restrict__ out, int B, int V, int F4) {
  pdl_sync();
  const long long total = (long long)B * V * F4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int f = (int)(i % F4); long long t = i / F4; int v = (int)(t % V); int b = (int)(t / V);
    const float* xb = x + (size_t)b * V * ldx + f * 4;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int e = rowptr[v]; e < rowptr[v + 1]; ++e) {
      const float w = val[e];
      const float4 n = *reinterpret_cast<const float4*>(xb + (size_t)col[e] * ldx);
      acc.x = fmaf(w, n.x, acc.x); acc.y = fmaf(w, n.y, acc.y); acc.z = fmaf(w, n.z, acc.z); acc.w = fmaf(w, n.w, acc.w);
    }
    const float4 s = *reinterpret_cast<const float4*>(xb + (size_t)v * ldx);
    float4* o = reinterpret_cast<float4*>(out) + i * 2;       // out row [B*V, 2F]: (x_f, (Lx)_f) interleaved
    o[0] = make_float4(s.x, acc.x, s.y, acc.y);
    o[1] = make_float4(s.z, acc.z, s.w, acc.w);
  }
}
__global__ void cheb4_bwd_kernel(const float* __restrict__ d, const int* __restrict__ rowptr, const int* __restrict__ col,
                                 const float* __restrict__ val, float* __restrict__ dx, int lddx, int acc_flag, int B, int V, int F4) {
  pdl_sync();
  const long long total = (long long)B * V * F4;
  const int F = F4 * 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int f = (int)(i % F4); long long t = i / F4; int v = (int)(t % V); int b = (int)(t / V);
    const float* db = d + (size_t)b * V * F * 2 + 8 * f;        // 4 features = 8 interleaved floats
    const float4 s0 = *reinterpret_cast<const float4*>(db + (size_t)v * F * 2), s1 = *reinterpret_cast<const float4*>(db + (size_t)v * F * 2 + 4);
    float4 acc = make_float4(s0.x, s0.z, s1.x, s1.z);
    for (int e = rowptr[v]; e < rowptr[v + 1]; ++e) {
      const float w = val[e];
      const float* nb = db + (size_t)col[e] * F * 2;
      const float4 n0 = *reinterpret_cast<const float4*>(nb), n1 = *reinterpret_cast<const float4*>(nb + 4);
      acc.x = fmaf(w, n0.y, acc.x); acc.y = fmaf(w, n0.w, acc.y); acc.z = fmaf(w, n1.y, acc.z); acc.w = fmaf(w, n1.w, acc.w);
    }
    float4* q = reinterpret_cast<float4*>(dx + ((size_t)b * V + v) * lddx + f * 4);
    if (acc_flag) { float4 o = *q; o.x += acc.x; o.y += acc.y; o.z += acc.z; o.w += acc.w; *q = o; }
    else *q = acc;
  }
}
RIH_API int rih_cheb_fwd(const float* x, int ldx, const int* rowptr, const int* col, const float* val, float* out,
                         int B, int V, int F, cudaStream_t s) {
  long long total = (long long)B * V * F;
  if (total == 0) return 0;
  if (F % 4 == 0 && ldx % 4 == 0 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) & 15) == 0) {
    int grid = (int)min(ew_ctas(s), (total / 4 + 255) / 256);
    launch_k(cheb4_fwd_kernel, grid, 256, 0, s, x, ldx, rowptr, col, val, out, B, V, F / 4);
    return check_launch("cheb_fwd");
  }
  int grid = (int)min(ew_ctas(s), (total + 255) / 256);
  launch_k(cheb_fwd_kernel, grid, 256, 0, s, x, ldx, rowptr, col, val, out, B, V, F);
  return check_launch("cheb_fwd");
}
RIH_API int rih_cheb_bwd(const float* d, const int* rowptrT, const int* colT, const float* valT, float* dx, int lddx, int accumulate,
                         int B, int V, int F, cudaStream_t s) {
  long long total = (long long)B * V * F;
  if (total == 0) return 0;
  if (F % 4 == 0 && lddx % 4 == 0 && ((reinterpret_cast<uintptr_t>(d) | reinterpret_cast<uintptr_t>(dx)) & 15) == 0) {
    int grid = (int)min(ew_ctas(s), (total / 4 + 255) / 256);
    launch_k(cheb4_bwd_kernel, grid, 256, 0, s, d, rowptrT, colT, valT, dx, lddx, accumulate, B, V, F / 4);
    return check_launch("cheb_bwd");
  }
  int grid = (int)min(ew_ctas(s), (total + 255) / 256);
  launch_k(cheb_bwd_kernel, grid, 256, 0, s, d, rowptrT, colT, valT, dx, lddx, accumulate, B, V, F);
  return check_launch("cheb_bwd");
}

// ============================================================== y[b,u,:] = x[b,u/p,:] + emb[u,:]
// reference: position_embeddings add, models/model_attn/DualGraph.py:76-80 ; graph_upsample(x,2) DualGraph.py:11-18,135-137 ;
//            grid position embeddings, img_attn.py:57-63
__global__ void posemb_fwd_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ emb, float* __restrict__ y, int ldy,
                                  int B, int U, int F, int p) {
  pdl_sync();
  long long total = (long long)B * U * F;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int f = (int)(i % F); long long t = i / F; int u = (int)(t % U); int b = (int)(t / U);
    y[((size_t)b * U + u) * ldy + f] = x[((size_t)b * (U / p) + u / p) * ldx + f] + emb[(size_t)u * F + f];
  }
}
// dx[b,v,:] = sum_{i<p} dy[b,p*v+i,:]
__global__ void posemb_bwd_x_kernel(const float* __restrict__ dy, int lddy, float* __restrict__ dx, int lddx, int B, int U, int F, int p) {
  pdl_sync();
  int V = U / p;
  long long total = (long long)B * V * F;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int f = (int)(i % F); long long t = i / F; int v = (int)(t % V); int b = (int)(t / V);
    float acc = 0.f;
    for (int j = 0; j < p; ++j) acc += dy[((size_t)b * U + p * v + j) * lddy + f];
    dx[((size_t)b * V + v) * lddx + f] = acc;
  }
}
// demb[u,:] += sum_b dy[b,u,:]
__global__ void posemb_bwd_emb_kernel(const float* __restrict__ dy, int lddy, float* __restrict__ demb, int B, int U, int F) {
  pdl_sync();
  long long total = (long long)U * F;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int f = (int)(i % F); int u = (int)(i / F);
    float acc = 0.f;
    for (int b = 0; b < B; ++b) acc += dy[((size_t)b * U + u) * lddy + f];
    demb[i] += acc;
  }
}
RIH_API int rih_posemb_fwd(const float* x, int ldx, const float* emb, float* y, int ldy, int B, int U, int F, int p, cudaStream_t s) {
  RIH_REQUIRE(p >= 1 && U % p == 0, "posemb_fwd: U %% p != 0");
  long long total = (long long)B * U * F;
  if (total == 0) return 0;
  int grid = (int)min(ew_ctas(s), (total + 255) / 256);
  launch_k(posemb_fwd_kernel, grid, 256, 0, s, x, ldx, emb, y, ldy, B, U, F, p);
  return check_launch("posemb_fwd");
}
RIH_API int rih_posemb_bwd(const float* dy, int lddy, float* dx, int lddx, float* demb, int B, int U, int F, int p, cudaStream_t s) {
  RIH_REQUIRE(p >= 1 && U % p == 0, "posemb_bwd: U %% p != 0");
  if (dx) {
    long long total = (long long)B * (U / p) * F;
    int grid = (int)min(ew_ctas(s), (total + 255) / 256);
    launch_k(posemb_bwd_x_kernel, grid, 256, 0, s, dy, lddy, dx, lddx, B, U, F, p);
    if (int e = check_launch("posemb_bwd_x")) return e;
  }
  if (demb) {
    long long total = (long long)U * F;
    int grid = (int)min(ew_ctas(s), (total + 255) / 256);
    launch_k(posemb_bwd_emb_kernel, grid, 256, 0, s, dy, lddy, demb, B, U, F);
    if (int e = check_launch("posemb_bwd_emb")) return e;
  }
  return 0;
}

// ============================================================== column sum: out[n] (+)= sum_m x[m,n]   (bias gradients)
__global__ void colsum_kernel(const float* __restrict__ x, int ld, int M, int N, int rows_per_cta, float* __restrict__ out) {
  pdl_sync();
  int c = blockIdx.x * 32 + threadIdx.x;
  int r0 = blockIdx.y * rows_per_cta, r1 = min(M, r0 + rows_per_cta);
  float s = 0.f;
  if (c < N) for (int r = r0 + threadIdx.y; r < r1; r += blockDim.y) s += x[(size_t)r * ld + c];
  __shared__ float sh[8][33];
  sh[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && c < N) {
    for (int i = 1; i < 8; ++i) s += sh[i][threadIdx.x];
    atomicAdd(out + c, s);
  }
}
RIH_API int rih_colsum(const float* x, int ld, int M, int N, float* out, int accumulate, cudaStream_t s) {
  if (!accumulate) RIH_CUDA(cudaMemsetAsync(out, 0, sizeof(float) * N, s));
  if (M == 0) return 0;
  int gx = cdiv(N, 32);
  int target = cdiv(sm_count() * 4, gx);
  int rows_per_cta = max(32, cdiv(M, target));
  dim3 grid(gx, cdiv(M, rows_per_cta)), block(32, 8);
  launch_k(colsum_kernel, grid, block, 0, s, x, ld, M, N, rows_per_cta, out);
  return check_launch("colsum");
}

// ============================================================== dropout (stateless counter RNG, device-resident seed)
// mask index = row*C + col over the logical [rows, C] tensor; seed = *seed_ptr + site*const  (same map as the GEMM epilogue)
__global__ void dropout_kernel(const float* __restrict__ x, int ldx, float* __restrict__ y, int ldy, long long rows, int C,
                               const unsigned long long* __restrict__ seed_ptr, unsigned long long site, uint32_t thresh, float inv_keep) {
  pdl_sync();
  long long total = rows * C;
  unsigned long long seed = *seed_ptr + site * 0xD1B54A32D192ED03ull;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long r; int c; divmod(i, C, total < (1ll << 32), r, c);
    y[r * ldy + c] = x[r * ldx + c] * dropout_scale(seed, (uint64_t)i, thresh, inv_keep);
  }
}
// forward and backward are the same map (dx = dy * keep_scale)
RIH_API int rih_dropout(const float* x, int ldx, float* y, int ldy, long long rows, int C, float p,
                        const unsigned long long* seed_ptr, unsigned long long site, cudaStream_t s) {
  if (rows * C == 0) return 0;
  RIH_REQUIRE(p > 0.f && p < 1.f && seed_ptr, "dropout: p out of range or missing seed");
  int grid = (int)min(ew_ctas(s), (rows * C + 255) / 256);
  launch_k(dropout_kernel, grid, 256, 0, s, x, ldx, y, ldy, rows, C, seed_ptr, site, dropout_thresh(p), 1.f / (1.f - p));
  return check_launch("dropout");
}
// backward pre-pass of a fused GEMM epilogue  y = dropout(relu(z)) (+res):  g = dy * keep_scale * (y_pre_res > 0 if relu)
// (y given is the stored output; only valid with relu when no residual was added)
__global__ void epilogue_bwd_kernel(const float* __restrict__ dy, int lddy, const float* __restrict__ y, int ldy, float* __restrict__ g, int ldg,
                                    long long rows, int C, int relu, const unsigned long long* __restrict__ seed_ptr, unsigned long long site,
                                    uint32_t thresh, float inv_keep) {
  pdl_sync();
  long long total = rows * C;
  unsigned long long seed = thresh ? (*seed_ptr + site * 0xD1B54A32D192ED03ull) : 0ull;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long r; int c; divmod(i, C, total < (1ll << 32), r, c);
    float v = dy[r * lddy + c];
    if (thresh) v *= dropout_scale(seed, (uint64_t)i, thresh, inv_keep);
    if (relu && !(y[r * ldy + c] > 0.f)) v = 0.f;
    g[r * ldg + c] = v;
  }
}
RIH_API int rih_epilogue_bwd(const float* dy, int lddy, const float* y, int ldy, float* g, int ldg, long long rows, int C, int relu,
                             float dropout_p, const unsigned long long* seed_ptr, unsigned long long site, cudaStream_t s) {
  if (rows * C == 0) return 0;
  RIH_REQUIRE(dropout_p == 0.f || (seed_ptr && dropout_p < 1.f), "epilogue_bwd: dropout needs a device seed");
  int grid = (int)min(ew_ctas(s), (rows * C + 255) / 256);
  launch_k(epilogue_bwd_kernel, grid, 256, 0, s, dy, lddy, y, ldy, g, ldg, rows, C, relu, seed_ptr, site,
                                           dropout_p > 0.f ? dropout_thresh(dropout_p) : 0u, dropout_p > 0.f ? 1.f / (1.f - dropout_p) : 1.f);
  return check_launch("epilogue_bwd");
}
__global__ void seed_advance_kernel(unsigned long long* seed) {
  pdl_sync(); *seed = *seed * 6364136223846793005ull + 1442695040888963407ull; }
RIH_API int rih_seed_advance(unsigned long long* seed_ptr, cudaStream_t s) {
  launch_k(seed_advance_kernel, 1, 1, 0, s, seed_ptr);
  return check_launch("seed_advance");
}

// ============================================================== decoder entry: Lf[b,v,0:G] = g[b,:], Lf[b,v,G:G+3] = pe[v,:], + emb[v,:]
// reference: models/decoder.py:132-135 (repeat + cat) fused with the level-0 position-embedding add (DualGraph.py:76-80)
__global__ void gf_broadcast_fwd_kernel(const float* __restrict__ g, const float* __restrict__ pe, const float* __restrict__ emb,
                                        float* __restrict__ y, int B, int V, int G) {
  pdl_sync();
  int F = G + 3;
  long long total = (long long)B * V * F;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int f = (int)(i % F); long long t = i / F; int v = (int)(t % V); int b = (int)(t / V);
    float base = f < G ? g[(size_t)b * G + f] : pe[v * 3 + (f - G)];
    y[i] = base + emb[(size_t)v * F + f];
  }
}
// dg[b,f] = sum_v dy[b,v,f] (f<G) ; demb[v,f] += sum_b dy[b,v,f]
__global__ void gf_broadcast_bwd_kernel(const float* __restrict__ dy, float* __restrict__ dg, int B, int V, int G) {
  pdl_sync();
  int F = G + 3;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * G) return;
  int b = i / G, f = i - b * G;
  float acc = 0.f;
  for (int v = 0; v < V; ++v) acc += dy[((size_t)b * V + v) * F + f];
  dg[i] = acc;
}
RIH_API int rih_gf_broadcast_fwd(const float* g, const float* pe, const float* emb, float* y, int B, int V, int G, cudaStream_t s) {
  long long total = (long long)B * V * (G + 3);
  int grid = (int)min(ew_ctas(s), (total + 255) / 256);
  launch_k(gf_broadcast_fwd_kernel, grid, 256, 0, s, g, pe, emb, y, B, V, G);
  return check_launch("gf_broadcast_fwd");
}
RIH_API int rih_gf_broadcast_bwd(const float* dy, float* dg, float* demb, int B, int V, int G, cudaStream_t s) {
  launch_k(gf_broadcast_bwd_kernel, cdiv((long long)B * G, 256), 256, 0, s, dy, dg, B, V, G);
  if (int e = check_launch("gf_broadcast_bwd")) return e;
  if (demb) {
    long long total = (long long)V * (G + 3);
    int grid = (int)min(ew_ctas(s), (total + 255) / 256);
    launch_k(posemb_bwd_emb_kernel, grid, 256, 0, s, dy, G + 3, demb, B, V, G + 3);
    if (int e = check_launch("gf_broadcast_bwd_emb")) return e;
  }
  return 0;
}

// ============================================================== fused AdamW over a flat fp32 buffer (SURVEY 8f-3; torch.optim.AdamW semantics)
__global__ void adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                             long long n, float decay, float b1, float omb1, float b2, float omb2, float eps, float step_size, float bc2_sqrt, float gscale) {
  pdl_sync();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float pi = p[i], mi = m[i], vi = v[i];
    adam_update(pi, mi, vi, g[i] * gscale, decay, b1, omb1, b2, omb2, eps, step_size, bc2_sqrt);
    p[i] = pi; m[i] = mi; v[i] = vi;
  }
}
// torch.optim.AdamW.step (single-tensor path of torch/optim/adamw.py): every scalar (1 - beta, the bias corrections, lr / bc1, 1 - lr * wd) is
// formed in DOUBLE on the host exactly like torch forms them as Python floats, then rounded to float once -- the kernel then matches
// torch.optim.AdamW on identical gradients to fp32 round-off (tests/test_train_gpu.py).  grad_scale folds the data-parallel mean (1 / world).
RIH_API int rih_adamw_step(float* p, const float* g, float* m, float* v, long long n, double lr, double beta1, double beta2,
                           double eps, double weight_decay, int step, double grad_scale, cudaStream_t s) {
  RIH_REQUIRE(n >= 0 && step >= 1, "adamw_step: n must be >= 0 and step >= 1 (got n=%lld step=%d)", n, step);
  if (n == 0) return 0;
  const double bc1 = 1.0 - pow(beta1, (double)step);
  const double bc2 = 1.0 - pow(beta2, (double)step);
  int grid = (int)min(ew_ctas(s), (n + 255) / 256);
  launch_k(adamw_kernel, grid, 256, 0, s, p, g, m, v, n, (float)(1.0 - lr * weight_decay), (float)beta1, (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2),
           (float)eps, (float)(lr / bc1), (float)sqrt(bc2), (float)grad_scale);
  return check_launch("adamw");
}
