// Fused multi-head attention core (SIMT fp32, exact softmax): O = dropout(softmax(Q K^T * scale)) V
// One CTA per (batch, head[, query split]): the whole K/V of a head (<= 512 keys, d <= 128, d % 4 == 0) lives in shared
// memory; each warp processes a block of query rows at once with register blocking and 128-bit shared-memory reads.
// reference: SelfAttn.self_attn  models/model_attn/self_attn.py:63-76 ; inter_attn.inter_attn  inter_attn.py:73-123
// Tensor addressing: element (b, row, h, dd) of T is  T + b*T_bs + row*ldT + h*d + dd.
#include "common.cuh"
#include <type_traits>
using namespace rih;

constexpr int ATT_WARPS = 8;
// query rows per warp block: forward 4 or 8, backward (both phases) 2 or 4 -- more rows amortise the K/V shared-memory reads over
// more FMAs but cost registers (MAXJ * R score accumulators per lane); chosen per launch from the key count (see att_rows)
static int g_att_force_rf = 0, g_att_force_rb = 0;   // testing / tuning override (rih_attn_set_row_blocks)
static inline int att_rows_fwd(int Skr) { return g_att_force_rf ? g_att_force_rf : 4; }      // measured best at all 9 decoder shapes
static inline int att_rows_bwd(int Smax) { return g_att_force_rb ? g_att_force_rb : 4; }

__device__ __forceinline__ float dot4(float4 a, float4 b, float acc) {
  acc = fmaf(a.x, b.x, acc); acc = fmaf(a.y, b.y, acc); acc = fmaf(a.z, b.z, acc); return fmaf(a.w, b.w, acc);
}
__device__ __forceinline__ void axpy4(float4& acc, float p, float4 v) {
  acc.x = fmaf(p, v.x, acc.x); acc.y = fmaf(p, v.y, acc.y); acc.z = fmaf(p, v.z, acc.z); acc.w = fmaf(p, v.w, acc.w);
}

// Shared-memory geometry shared by forward and backward:
//   key-like tiles [rows][d + 4] (row stride 16-byte aligned, conflict-free LDS.128 across consecutive rows)
//   G = d/4 feature groups per lane set, JS = 32/G interleaved row splits for the P.V-type accumulations
//   probabilities are stored permuted as p[(j % JS) * T + j / JS] so that a lane's rows are contiguous
struct AttGeo {
  int d, dp, G, JS, Skr, T;   // Skr = keys rounded up to 32, T = Skr / JS
  int js_shift;               // JS is a power of two (32 / G, G = d / 4 in {1,2,4,8,16,32}) whenever G divides 32
};
__host__ __device__ __forceinline__ AttGeo make_geo(int d, int Sk) {
  AttGeo g;
  g.d = d; g.dp = d + 4; g.G = d / 4; if (g.G > 32) g.G = 32;
  g.JS = 32 / g.G;
  const int q = (4 * g.JS > 32) ? 4 * g.JS : 32;      // rows padded so that T = Skr / JS is a multiple of 4 (float4 reads of p)
  g.Skr = ((Sk + q - 1) / q) * q; g.T = g.Skr / g.JS;
  g.js_shift = 0; while ((1 << g.js_shift) < g.JS) ++g.js_shift;
  return g;
}

// acc[r] (+)= sum_j p[r][perm(j)] * M[j][g*4 .. g*4+3] for the lane's row split; then butterfly-reduce over splits.
template <int R>
__device__ __forceinline__ void pv_accumulate(const float* __restrict__ M, int ldm, const float* __restrict__ p, int pstride,
                                              const AttGeo& g, int lane, float4 (&acc)[R]) {
  const int gi = lane % g.G, js = lane / g.G;
#pragma unroll
  for (int r = 0; r < R; ++r) acc[r] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int t = 0; t < g.T; t += 4) {
    float4 p4[R];
#pragma unroll
    for (int r = 0; r < R; ++r) p4[r] = *reinterpret_cast<const float4*>(p + r * pstride + js * g.T + t);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int j = js + g.JS * (t + u);
      const float4 v = *reinterpret_cast<const float4*>(M + (size_t)j * ldm + gi * 4);
#pragma unroll
      for (int r = 0; r < R; ++r) axpy4(acc[r], (u == 0 ? p4[r].x : u == 1 ? p4[r].y : u == 2 ? p4[r].z : p4[r].w), v);
    }
  }
  for (int off = g.G; off < 32; off <<= 1) {
#pragma unroll
    for (int r = 0; r < R; ++r) {
      acc[r].x += __shfl_xor_sync(0xffffffffu, acc[r].x, off); acc[r].y += __shfl_xor_sync(0xffffffffu, acc[r].y, off);
      acc[r].z += __shfl_xor_sync(0xffffffffu, acc[r].z, off); acc[r].w += __shfl_xor_sync(0xffffffffu, acc[r].w, off);
    }
  }
}

template <int MAXJ, int R>
__global__ void __launch_bounds__(ATT_WARPS * 32)
attn_fwd_kernel(const float* __restrict__ q, long long q_bs, int ldq, const float* __restrict__ k, long long k_bs, int ldk,
                const float* __restrict__ v, long long v_bs, int ldv, float* __restrict__ o, long long o_bs, int ldo,
                float* __restrict__ lse, int H, int Sq, int Sk, int d, float scale, int rows_per_cta,
                const unsigned long long* __restrict__ seed_ptr, unsigned long long site, uint32_t thresh, float inv_keep) {
  pdl_sync();
  const unsigned long long seed = thresh ? (*seed_ptr + site * 0xD1B54A32D192ED03ull) : 0ull;
  extern __shared__ __align__(16) float smem[];
  const AttGeo g = make_geo(d, Sk);
  float* Ks = smem;                               // [Skr][dp]  (rows >= Sk zero)
  float* Vs = Ks + (size_t)g.Skr * g.dp;          // [Skr][dp]
  float* qs = Vs + (size_t)g.Skr * g.dp;          // [W][R][d]
  float* ps = qs + ATT_WARPS * R * d;             // [W][R][Skr]
  const int bh = blockIdx.x, b = bh / H, h = bh % H;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const float* kb = k + (size_t)b * k_bs + h * d;
  const float* vb = v + (size_t)b * v_bs + h * d;
  const int d4 = d / 4;
  for (int i = tid; i < g.Skr * d4; i += blockDim.x) {
    int j = i / d4, c = (i - j * d4) * 4;
    float4 kk = make_float4(0.f, 0.f, 0.f, 0.f), vv = kk;
    if (j < Sk) {
      kk = *reinterpret_cast<const float4*>(kb + (size_t)j * ldk + c);
      vv = *reinterpret_cast<const float4*>(vb + (size_t)j * ldv + c);
    }
    *reinterpret_cast<float4*>(Ks + j * g.dp + c) = kk;
    *reinterpret_cast<float4*>(Vs + j * g.dp + c) = vv;
  }
  __syncthreads();
  const int r0 = blockIdx.y * rows_per_cta, r1 = min(Sq, r0 + rows_per_cta);
  float* myq = qs + warp * R * d;
  float* myp = ps + (size_t)warp * R * g.Skr;
  for (int i0 = r0 + warp * R; i0 < r1; i0 += ATT_WARPS * R) {
    for (int e = lane; e < R * d4; e += 32) {
      int r = e / d4, c = (e - r * d4) * 4;
      int i = min(i0 + r, r1 - 1);
      *reinterpret_cast<float4*>(myq + r * d + c) = *reinterpret_cast<const float4*>(q + (size_t)b * q_bs + (size_t)i * ldq + h * d + c);
    }
    __syncwarp();
    float s[R][MAXJ];
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int jj = 0; jj < MAXJ; ++jj) s[r][jj] = 0.f;
    for (int c = 0; c < d; c += 4) {
      float4 q4[R];
#pragma unroll
      for (int r = 0; r < R; ++r) q4[r] = *reinterpret_cast<const float4*>(myq + r * d + c);
#pragma unroll
      for (int jj = 0; jj < MAXJ; ++jj) {
        const int j = lane + 32 * jj;
        if (j < g.Skr) {
          const float4 k4 = *reinterpret_cast<const float4*>(Ks + j * g.dp + c);
#pragma unroll
          for (int r = 0; r < R; ++r) s[r][jj] = dot4(q4[r], k4, s[r][jj]);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < MAXJ; ++jj) {
        const int j = lane + 32 * jj;
        s[r][jj] = (j < Sk) ? s[r][jj] * scale : -INFINITY;
        mx = fmaxf(mx, s[r][jj]);
      }
      mx = warp_max(mx);
      float sum = 0.f;
#pragma unroll
      for (int jj = 0; jj < MAXJ; ++jj) {
        const int j = lane + 32 * jj;
        s[r][jj] = (j < Sk) ? expf(s[r][jj] - mx) : 0.f;
        sum += s[r][jj];
      }
      sum = warp_sum(sum);
      const float inv = 1.f / sum;
      const int i = i0 + r;
      const size_t drop_base = ((size_t)bh * Sq + i) * Sk;
#pragma unroll
      for (int jj = 0; jj < MAXJ; ++jj) {
        const int j = lane + 32 * jj;
        if (j < g.Skr) {
          float p = s[r][jj] * inv;
          if (thresh && j < Sk) p *= dropout_scale(seed, drop_base + j, thresh, inv_keep);
          myp[r * g.Skr + (j & (g.JS - 1)) * g.T + (j >> g.js_shift)] = p;
        }
      }
      if (lane == 0 && lse && i < r1) lse[(size_t)bh * Sq + i] = mx + logf(sum);
    }
    __syncwarp();
    float4 acc[R];
    pv_accumulate<R>(Vs, g.dp, myp, g.Skr, g, lane, acc);
    if (lane < g.G) {
#pragma unroll
      for (int r = 0; r < R; ++r)
        if (i0 + r < r1) *reinterpret_cast<float4*>(o + (size_t)b * o_bs + (size_t)(i0 + r) * ldo + h * d + lane * 4) = acc[r];
    }
    __syncwarp();
  }
}

static bool att_aligned(const void* p, long long bs, int ld) { return ((reinterpret_cast<uintptr_t>(p) & 15) == 0) && (bs % 4 == 0) && (ld % 4 == 0); }

RIH_API int rih_attn_fwd(const float* q, long long q_bs, int ldq, const float* k, long long k_bs, int ldk,
                         const float* v, long long v_bs, int ldv, float* o, long long o_bs, int ldo, float* lse,
                         int B, int H, int Sq, int Sk, int d, float scale, float dropout_p, const unsigned long long* seed_ptr, unsigned long long site, cudaStream_t s) {
  RIH_REQUIRE(Sk > 0 && Sk <= 512, "attn_fwd: Sk=%d unsupported (max 512)", Sk);
  RIH_REQUIRE(d >= 4 && d <= 128 && (d & (d - 1)) == 0, "attn_fwd: head dim %d unsupported (power of two in 4..128)", d);
  RIH_REQUIRE(att_aligned(q, q_bs, ldq) && att_aligned(k, k_bs, ldk) && att_aligned(v, v_bs, ldv) && att_aligned(o, o_bs, ldo),
              "attn_fwd: operands must be 16-byte aligned with strides that are multiples of 4 floats");
  if (B * H == 0 || Sq == 0) return 0;
  const int Skr = make_geo(d, Sk).Skr;
  const int RF = att_rows_fwd(Skr);
  size_t smem = sizeof(float) * (2 * (size_t)Skr * (d + 4) + ATT_WARPS * RF * d + (size_t)ATT_WARPS * RF * Skr);
  RIH_REQUIRE(smem <= 227 * 1024, "attn_fwd: shared memory %zu too large", smem);
  int ysplit = 1;
  while (B * H * ysplit < sm_count() * 2 && Sq / (ysplit * 2) >= 32) ysplit *= 2;
  int rows_per_cta = cdiv(Sq, ysplit);
  rows_per_cta = (rows_per_cta + RF - 1) / RF * RF;
  dim3 grid(B * H, cdiv(Sq, rows_per_cta));
  uint32_t thresh = dropout_p > 0.f ? dropout_thresh(dropout_p) : 0u;
  float ik = dropout_p > 0.f ? 1.f / (1.f - dropout_p) : 1.f;
#define RIH_ATT_FWD(MJ, RR)                                                                                                            \
  {                                                                                                                                    \
    static bool attr = false;                                                                                                          \
    if (!attr) { RIH_CUDA(cudaFuncSetAttribute(attn_fwd_kernel<MJ, RR>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024)); attr = true; } \
    launch_k(attn_fwd_kernel<MJ, RR>, grid, ATT_WARPS * 32, smem, s, q, q_bs, ldq, k, k_bs, ldk, v, v_bs, ldv, o, o_bs, ldo, lse, H, Sq, Sk, d, scale, \
                                                                rows_per_cta, seed_ptr, site, thresh, ik);                             \
  }
  if (Skr <= 128) { if (RF == 8) RIH_ATT_FWD(4, 8) else RIH_ATT_FWD(4, 4) }
  else if (Skr <= 320) { if (RF == 8) RIH_ATT_FWD(10, 8) else RIH_ATT_FWD(10, 4) }
  else { if (RF == 8) RIH_ATT_FWD(16, 8) else RIH_ATT_FWD(16, 4) }
#undef RIH_ATT_FWD
  return check_launch("attn_fwd");
}

// ------------------------------------------------------------------ backward
// Phase A (warp per block of R query rows): dS -> dQ = scale * dS K.
// Phase B (warp per block of R key rows)  : P~^T, dS^T -> dV = P~^T dO, dK = scale * dS^T Q.  No atomics, deterministic.
template <int MAXJ, int R>
__global__ void __launch_bounds__(ATT_WARPS * 32)
attn_bwd_kernel(const float* __restrict__ q, long long q_bs, int ldq, const float* __restrict__ k, long long k_bs, int ldk,
                const float* __restrict__ v, long long v_bs, int ldv, const float* __restrict__ o, long long o_bs, int ldo,
                const float* __restrict__ dout, long long do_bs, int lddo, const float* __restrict__ lse,
                float* __restrict__ dq, long long dq_bs, int lddq, float* __restrict__ dk, long long dk_bs, int lddk,
                float* __restrict__ dv, long long dv_bs, int lddv,
                int H, int Sq, int Sk, int d, float scale, const unsigned long long* __restrict__ seed_ptr, unsigned long long site, uint32_t thresh, float inv_keep) {
  pdl_sync();
  const unsigned long long seed = thresh ? (*seed_ptr + site * 0xD1B54A32D192ED03ull) : 0ull;
  extern __shared__ __align__(16) float smem[];
  const AttGeo gk = make_geo(d, Sk);   // splits over keys (phase A accumulations)
  const AttGeo gq = make_geo(d, Sq);   // splits over queries (phase B accumulations)
  const int Smax = max(gk.Skr, gq.Skr);
  const int dp = d + 4, d4 = d / 4;
  float* Qs = smem;                              // [Sqr][dp]
  float* dOs = Qs + (size_t)gq.Skr * dp;         // [Sqr][dp]
  float* Ks = dOs + (size_t)gq.Skr * dp;         // [Skr][dp]
  float* Vs = Ks + (size_t)gk.Skr * dp;          // [Skr][dp]
  float* Dl = Vs + (size_t)gk.Skr * dp;          // [Sqr]
  float* Ls = Dl + gq.Skr;                       // [Sqr]
  float* w1 = Ls + gq.Skr;                       // [W][R][Smax]
  float* w2 = w1 + (size_t)ATT_WARPS * R * Smax; // [W][R][Smax]
  float* rw = w2 + (size_t)ATT_WARPS * R * Smax; // [W][2][R][d]  row operands of the current block
  const int bh = blockIdx.x, b = bh / H, h = bh % H;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const float* qb = q + (size_t)b * q_bs + h * d;
  const float* dob = dout + (size_t)b * do_bs + h * d;
  const float* kb = k + (size_t)b * k_bs + h * d;
  const float* vb = v + (size_t)b * v_bs + h * d;
  for (int i = tid; i < gq.Skr * d4; i += blockDim.x) {
    int r = i / d4, c = (i - r * d4) * 4;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), bb = a;
    if (r < Sq) { a = *reinterpret_cast<const float4*>(qb + (size_t)r * ldq + c); bb = *reinterpret_cast<const float4*>(dob + (size_t)r * lddo + c); }
    *reinterpret_cast<float4*>(Qs + r * dp + c) = a;
    *reinterpret_cast<float4*>(dOs + r * dp + c) = bb;
  }
  for (int i = tid; i < gk.Skr * d4; i += blockDim.x) {
    int r = i / d4, c = (i - r * d4) * 4;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), bb = a;
    if (r < Sk) { a = *reinterpret_cast<const float4*>(kb + (size_t)r * ldk + c); bb = *reinterpret_cast<const float4*>(vb + (size_t)r * ldv + c); }
    *reinterpret_cast<float4*>(Ks + r * dp + c) = a;
    *reinterpret_cast<float4*>(Vs + r * dp + c) = bb;
  }
  for (int i = warp; i < gq.Skr; i += ATT_WARPS) {
    float acc = 0.f;
    if (i < Sq) {
      const float* orow = o + (size_t)b * o_bs + (size_t)i * ldo + h * d;
      const float* drow = dob + (size_t)i * lddo;
      for (int dd = lane; dd < d; dd += 32) acc += orow[dd] * drow[dd];
    }
    acc = warp_sum(acc);
    if (lane == 0) { Dl[i] = acc; Ls[i] = (i < Sq) ? lse[(size_t)bh * Sq + i] : 0.f; }
  }
  __syncthreads();
  float* my1 = w1 + (size_t)warp * R * Smax;
  float* my2 = w2 + (size_t)warp * R * Smax;
  float* ra = rw + warp * 2 * R * d;      // [R][d] first row operand
  float* rb = ra + R * d;                 // [R][d] second row operand
  // ---------------- phase A: query-row blocks
  for (int i0 = warp * R; i0 < Sq; i0 += ATT_WARPS * R) {
    for (int e = lane; e < R * d4; e += 32) {
      int r = e / d4, c = (e - r * d4) * 4;
      int i = min(i0 + r, Sq - 1);
      *reinterpret_cast<float4*>(ra + r * d + c) = *reinterpret_cast<const float4*>(Qs + i * dp + c);
      *reinterpret_cast<float4*>(rb + r * d + c) = *reinterpret_cast<const float4*>(dOs + i * dp + c);
    }
    __syncwarp();
    float sc[R][MAXJ], dpt[R][MAXJ];
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int jj = 0; jj < MAXJ; ++jj) { sc[r][jj] = 0.f; dpt[r][jj] = 0.f; }
    for (int c = 0; c < d; c += 4) {
      float4 q4[R], g4[R];
#pragma unroll
      for (int r = 0; r < R; ++r) { q4[r] = *reinterpret_cast<const float4*>(ra + r * d + c); g4[r] = *reinterpret_cast<const float4*>(rb + r * d + c); }
#pragma unroll
      for (int jj = 0; jj < MAXJ; ++jj) {
        const int j = lane + 32 * jj;
        if (j < gk.Skr) {
          const float4 k4 = *reinterpret_cast<const float4*>(Ks + j * dp + c);
          const float4 v4 = *reinterpret_cast<const float4*>(Vs + j * dp + c);
#pragma unroll
          for (int r = 0; r < R; ++r) { sc[r][jj] = dot4(q4[r], k4, sc[r][jj]); dpt[r][jj] = dot4(g4[r], v4, dpt[r][jj]); }
        }
      }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int i = min(i0 + r, Sq - 1);
      const float Li = Ls[i], Di = Dl[i];
      const size_t drop_base = ((size_t)bh * Sq + i) * Sk;
#pragma unroll
      for (int jj = 0; jj < MAXJ; ++jj) {
        const int j = lane + 32 * jj;
        if (j < gk.Skr) {
          float dsv = 0.f;
          if (j < Sk) {
            const float p = expf(sc[r][jj] * scale - Li);
            const float m = thresh ? dropout_scale(seed, drop_base + j, thresh, inv_keep) : 1.f;
            dsv = p * (m * dpt[r][jj] - Di);
          }
          my1[r * Smax + (j & (gk.JS - 1)) * gk.T + (j >> gk.js_shift)] = dsv;
        }
      }
    }
    __syncwarp();
    float4 acc[R];
    pv_accumulate<R>(Ks, dp, my1, Smax, gk, lane, acc);
    if (lane < gk.G) {
#pragma unroll
      for (int r = 0; r < R; ++r)
        if (i0 + r < Sq) {
          float4 t = acc[r]; t.x *= scale; t.y *= scale; t.z *= scale; t.w *= scale;
          *reinterpret_cast<float4*>(dq + (size_t)b * dq_bs + (size_t)(i0 + r) * lddq + h * d + lane * 4) = t;
        }
    }
    __syncwarp();
  }
  // ---------------- phase B: key-row blocks
  const size_t drop_bh = (size_t)bh * Sq * Sk;
  for (int j0 = warp * R; j0 < Sk; j0 += ATT_WARPS * R) {
    for (int e = lane; e < R * d4; e += 32) {
      int r = e / d4, c = (e - r * d4) * 4;
      int j = min(j0 + r, Sk - 1);
      *reinterpret_cast<float4*>(ra + r * d + c) = *reinterpret_cast<const float4*>(Ks + j * dp + c);
      *reinterpret_cast<float4*>(rb + r * d + c) = *reinterpret_cast<const float4*>(Vs + j * dp + c);
    }
    __syncwarp();
    float sc[R][MAXJ], dpt[R][MAXJ];
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int ii = 0; ii < MAXJ; ++ii) { sc[r][ii] = 0.f; dpt[r][ii] = 0.f; }
    for (int c = 0; c < d; c += 4) {
      float4 k4[R], v4[R];
#pragma unroll
      for (int r = 0; r < R; ++r) { k4[r] = *reinterpret_cast<const float4*>(ra + r * d + c); v4[r] = *reinterpret_cast<const float4*>(rb + r * d + c); }
#pragma unroll
      for (int ii = 0; ii < MAXJ; ++ii) {
        const int i = lane + 32 * ii;
        if (i < gq.Skr) {
          const float4 q4 = *reinterpret_cast<const float4*>(Qs + i * dp + c);
          const float4 g4 = *reinterpret_cast<const float4*>(dOs + i * dp + c);
#pragma unroll
          for (int r = 0; r < R; ++r) { sc[r][ii] = dot4(q4, k4[r], sc[r][ii]); dpt[r][ii] = dot4(g4, v4[r], dpt[r][ii]); }
        }
      }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int j = min(j0 + r, Sk - 1);
#pragma unroll
      for (int ii = 0; ii < MAXJ; ++ii) {
        const int i = lane + 32 * ii;
        if (i < gq.Skr) {
          float pt = 0.f, dsv = 0.f;
          if (i < Sq) {
            const float p = expf(sc[r][ii] * scale - Ls[i]);
            const float m = thresh ? dropout_scale(seed, drop_bh + (uint32_t)(i * Sk + j), thresh, inv_keep) : 1.f;
            pt = p * m;
            dsv = p * (m * dpt[r][ii] - Dl[i]);
          }
          const int pi = (i & (gq.JS - 1)) * gq.T + (i >> gq.js_shift);
          my1[r * Smax + pi] = pt;
          my2[r * Smax + pi] = dsv;
        }
      }
    }
    __syncwarp();
    float4 av[R], ak[R];
    pv_accumulate<R>(dOs, dp, my1, Smax, gq, lane, av);
    pv_accumulate<R>(Qs, dp, my2, Smax, gq, lane, ak);
    if (lane < gq.G) {
#pragma unroll
      for (int r = 0; r < R; ++r)
        if (j0 + r < Sk) {
          float4 t = ak[r]; t.x *= scale; t.y *= scale; t.z *= scale; t.w *= scale;
          *reinterpret_cast<float4*>(dk + (size_t)b * dk_bs + (size_t)(j0 + r) * lddk + h * d + lane * 4) = t;
          *reinterpret_cast<float4*>(dv + (size_t)b * dv_bs + (size_t)(j0 + r) * lddv + h * d + lane * 4) = av[r];
        }
    }
    __syncwarp();
  }
}

RIH_API int rih_attn_bwd(const float* q, long long q_bs, int ldq, const float* k, long long k_bs, int ldk,
                         const float* v, long long v_bs, int ldv, const float* o, long long o_bs, int ldo,
                         const float* dout, long long do_bs, int lddo, const float* lse,
                         float* dq, long long dq_bs, int lddq, float* dk, long long dk_bs, int lddk, float* dv, long long dv_bs, int lddv,
                         int B, int H, int Sq, int Sk, int d, float scale, float dropout_p, const unsigned long long* seed_ptr, unsigned long long site, cudaStream_t s) {
  RIH_REQUIRE(d >= 4 && d <= 128 && (d & (d - 1)) == 0, "attn_bwd: head dim %d unsupported (power of two in 4..128)", d);
  RIH_REQUIRE(Sk <= 512 && Sq <= 512, "attn_bwd: sequence length above 512 unsupported (Sq=%d Sk=%d)", Sq, Sk);
  RIH_REQUIRE(att_aligned(q, q_bs, ldq) && att_aligned(k, k_bs, ldk) && att_aligned(v, v_bs, ldv) && att_aligned(o, o_bs, ldo) &&
              att_aligned(dout, do_bs, lddo) && att_aligned(dq, dq_bs, lddq) && att_aligned(dk, dk_bs, lddk) && att_aligned(dv, dv_bs, lddv),
              "attn_bwd: operands must be 16-byte aligned with strides that are multiples of 4 floats");
  if (B * H == 0 || Sq == 0 || Sk == 0) return 0;
  const int Sqr = make_geo(d, Sq).Skr, Skr = make_geo(d, Sk).Skr, Smax = Sqr > Skr ? Sqr : Skr;
  const int RB = att_rows_bwd(Smax);
  size_t smem = sizeof(float) * ((size_t)(2 * Sqr + 2 * Skr) * (d + 4) + 2 * (size_t)Sqr + 2 * (size_t)ATT_WARPS * RB * Smax + (size_t)ATT_WARPS * 2 * RB * d);
  RIH_REQUIRE(smem <= 227 * 1024, "attn_bwd: shared memory %zu too large (Sq=%d Sk=%d d=%d)", smem, Sq, Sk, d);
  uint32_t thresh = dropout_p > 0.f ? dropout_thresh(dropout_p) : 0u;
  float ik = dropout_p > 0.f ? 1.f / (1.f - dropout_p) : 1.f;
#define RIH_ATT_BWD(MJ, RR)                                                                                                            \
  {                                                                                                                                    \
    static bool attr = false;                                                                                                          \
    if (!attr) { RIH_CUDA(cudaFuncSetAttribute(attn_bwd_kernel<MJ, RR>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024)); attr = true; } \
    launch_k(attn_bwd_kernel<MJ, RR>, B * H, ATT_WARPS * 32, smem, s, q, q_bs, ldq, k, k_bs, ldk, v, v_bs, ldv, o, o_bs, ldo, dout, do_bs, lddo, lse, \
                                                                 dq, dq_bs, lddq, dk, dk_bs, lddk, dv, dv_bs, lddv, H, Sq, Sk, d, scale, seed_ptr, site, thresh, ik); \
  }
  if (Smax <= 128) { if (RB == 4) RIH_ATT_BWD(4, 4) else RIH_ATT_BWD(4, 2) }
  else if (Smax <= 320) { if (RB == 4) RIH_ATT_BWD(10, 4) else RIH_ATT_BWD(10, 2) }
  else { if (RB == 4) RIH_ATT_BWD(16, 4) else RIH_ATT_BWD(16, 2) }
#undef RIH_ATT_BWD
  return check_launch("attn_bwd");
}

// Tuning / testing hook: force the per-warp row blocks (forward 4 | 8, backward 2 | 4; 0 = automatic choice from the key count).
RIH_API int rih_attn_set_row_blocks(int rows_fwd, int rows_bwd) {
  RIH_REQUIRE((rows_fwd == 0 || rows_fwd == 4 || rows_fwd == 8) && (rows_bwd == 0 || rows_bwd == 2 || rows_bwd == 4), "attn_set_row_blocks: fwd in {0,4,8}, bwd in {0,2,4}");
  g_att_force_rf = rows_fwd; g_att_force_rb = rows_bwd;
  return 0;
}

// ================================================================================================ tensor-core attention core
// The same operator with its contractions on the tensor cores (warp-level mma.sync.m16n8k8, 3xTF32 or single-pass TF32), fused flash-style
// so that no score matrix leaves the SM:
//   forward  attn_fused_fwd_kernel: one CTA per (64 query rows, batch * head); K / V stream through shared memory in blocks of 64 keys
//            (cp.async, double-buffered); S = scale Q K^T, online softmax over the key blocks, P~ = P o M (dropout mask), O = P~ V.  Per query
//            row it writes the statistics (m, 1 / l): the row max of S and the reciprocal of l = sum_j exp(S_ij - m), so P_ij = exp(S_ij - m) / l.
//   backward (the FlashAttention-2 split: no atomics, deterministic): D_i = dO_i . O_i, dP~ = dO V^T, dS = P o (M o dP~ - D)
//            attn_fused_bwd_dq_kernel  : one CTA per (64 query rows, batch * head), loops over the key blocks:   dQ = scale dS K
//            attn_fused_bwd_dkdv_kernel: one CTA per (64 keys, batch * head), loops over the query blocks: dK = scale dS^T Q, dV = P~^T dO
//            Both recompute S with the forward's fragments, products and k order, so P is the forward's P.  Recomputing S and dP~ in two
//            kernels costs one more pass of tensor work than one CTA per head owning all keys would, but gives a grid ~5x wider and
//            keeps dK / dV of any head within registers.
// Fragments: a warp owns 16 rows.  The C fragment of S (rows g, g + 8; columns 2t, 2t + 1 of an 8-column tile) is used as the A fragment of
// the next product (P~ V, dS K, ...) by permuting k within each 8-step: slot t <-> column 2t, slot t + 4 <-> column 2t + 1; the B operand is
// read with the same permutation.  Shared-memory tiles are [rows][D + 4] floats, on which every fragment pattern used is conflict-free.
// 3xTF32: x = hi + lo with hi = x rounded to TF32 (split_tf32 in gemm_tc.cuh), c += lo*hi + hi*lo + hi*hi; TF32: one product on the raw
// fp32 bits (the tensor core reads their TF32 part).  Head dims are padded with zeros to D in {8, 16, 32, 64, 128}.
// The dropout mask is dropout_scale(seed + site * 0xD1B54A32D192ED03, ((b H + h) Sq + i) Sk + j) in every kernel.
namespace {
constexpr int FA_WARPS = 4, FA_THREADS = 32 * FA_WARPS, FA_ROWS = 16 * FA_WARPS;   // rows (queries or keys) owned by a CTA
constexpr int FA_BLK = 64;                                                            // keys (forward, dQ) per streamed block
template <int D> __host__ __device__ constexpr int fa_qblk() { return D > 64 ? 32 : 64; }              // queries (dK / dV) per streamed block

__device__ __forceinline__ void cp_async16(float* dst, const float* src, bool ok) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(src), "r"(ok ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// rows [r0, r0 + R) x columns [0, D) of one head of a token matrix (base: the head's column 0 of the sequence's row 0; nrows / d valid rows /
// columns) -> tile [R][D + 4], zero outside
template <int R, int D>
__device__ __forceinline__ void load_tile(float* tile, const float* base, int ld, int r0, int nrows, int d) {
  constexpr int C = D / 4;
  for (int e = threadIdx.x; e < R * C; e += FA_THREADS) {
    const int r = e / C, c = (e - r * C) * 4;
    const bool ok = r0 + r < nrows && c < d;
    cp_async16(tile + r * (D + 4) + c, ok ? base + (size_t)(r0 + r) * ld + c : base, ok);
  }
}

template <int NS> struct FragA { uint32_t h[4], l[4]; };
template <int NS> struct FragB { uint32_t h[2], l[2]; };
template <int NS> __device__ __forceinline__ void tf32_split(float x, uint32_t& h, uint32_t& l) {
  if constexpr (NS == 1) {
    h = __float_as_uint(x); l = 0u;
  } else {
    h = (__float_as_uint(x) + 0x1000u) & 0xFFFFE000u;
    l = __float_as_uint(x - __uint_as_float(h));
  }
}
template <int NS> __device__ __forceinline__ FragA<NS> frag_a(float a0, float a1, float a2, float a3) {
  FragA<NS> f;
  tf32_split<NS>(a0, f.h[0], f.l[0]); tf32_split<NS>(a1, f.h[1], f.l[1]); tf32_split<NS>(a2, f.h[2], f.l[2]); tf32_split<NS>(a3, f.h[3], f.l[3]);
  return f;
}
template <int NS> __device__ __forceinline__ FragB<NS> frag_b(float b0, float b1) {
  FragB<NS> f;
  tf32_split<NS>(b0, f.h[0], f.l[0]); tf32_split<NS>(b1, f.h[1], f.l[1]);
  return f;
}
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
// c += a b.  TR: the transpose of a forward product (a holds the forward's B operand, b its A); the cross terms then swap places so that
// every element sees the forward's sequence of products.
template <int NS, bool TR>
__device__ __forceinline__ void mma_x(float (&c)[4], const FragA<NS>& a, const FragB<NS>& b) {
  if constexpr (NS == 3) {
    if constexpr (TR) { mma_tf32(c, a.h, b.l); mma_tf32(c, a.l, b.h); }
    else { mma_tf32(c, a.l, b.h); mma_tf32(c, a.h, b.l); }
  }
  mma_tf32(c, a.h, b.h);
}

// s[16 x 8 NT] = A[16 rows] . Bt[8 NT rows]^T over D (both tiles [rows][D + 4])
template <int D, int NT, int NS, bool TR>
__device__ __forceinline__ void qk_block(float (&s)[NT][4], const float* A, const float* Bt, int lane) {
  constexpr int LD = D + 4;
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
  for (int k0 = 0; k0 < D; k0 += 8) {
    const float* a = A + g * LD + k0 + t;
    const FragA<NS> fa = frag_a<NS>(a[0], a[8 * LD], a[4], a[8 * LD + 4]);
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const float* b = Bt + (nt * 8 + g) * LD + k0 + t;
      mma_x<NS, TR>(s[nt], fa, frag_b<NS>(b[0], b[4]));
    }
  }
}
// acc[16 x D] += p[16 x 8 NT] (C fragments) . V[8 NT rows][D]
template <int D, int NT, int NS>
__device__ __forceinline__ void pv_block(float (&acc)[D / 8][4], const float (&p)[NT][4], const float* V, int lane) {
  constexpr int LD = D + 4;
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int kt = 0; kt < NT; ++kt) {
    const FragA<NS> fa = frag_a<NS>(p[kt][0], p[kt][2], p[kt][1], p[kt][3]);
    const float* v = V + (kt * 8 + 2 * t) * LD + g;
#pragma unroll
    for (int nt = 0; nt < D / 8; ++nt) mma_x<NS, false>(acc[nt], fa, frag_b<NS>(v[nt * 8], v[LD + nt * 8]));
  }
}
// D_i = dO_i . O_i, in one fixed order for both backward kernels
__device__ __forceinline__ float row_term(const float* __restrict__ o, const float* __restrict__ g, int d) {
  float acc = 0.f;
  for (int c = 0; c < d; c += 4) {
    const float4 a = *reinterpret_cast<const float4*>(o + c), b = *reinterpret_cast<const float4*>(g + c);
    acc = fmaf(a.x, b.x, acc); acc = fmaf(a.y, b.y, acc); acc = fmaf(a.z, b.z, acc); acc = fmaf(a.w, b.w, acc);
  }
  return acc;
}
}  // namespace

template <int D, int NS>
__global__ void __launch_bounds__(FA_THREADS)
attn_fused_fwd_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ k, int ldk, const float* __restrict__ v, int ldv,
                      float* __restrict__ o, int ldo, float2* __restrict__ stats, int H, int Sq, int Sk, int d, int nqb, float scale,
                      const unsigned long long* __restrict__ seed_ptr, unsigned long long site, uint32_t thresh, float inv_keep) {
  constexpr int LD = D + 4, DT = D / 8, NT = FA_BLK / 8;
  extern __shared__ __align__(16) float smem[];
  float* Qs = smem;                       // [64][LD]
  float* Ks = Qs + FA_ROWS * LD;          // [2][64][LD]
  float* Vs = Ks + 2 * FA_BLK * LD;       // [2][64][LD]
  const int bh = blockIdx.x / nqb, b = bh / H, h = bh - b * H, i0 = (blockIdx.x - bh * nqb) * FA_ROWS;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const float* qb = q + (size_t)b * Sq * ldq + h * d;
  const float* kb = k + (size_t)b * Sk * ldk + h * d;
  const float* vb = v + (size_t)b * Sk * ldv + h * d;
  pdl_sync();
  const unsigned long long seed = thresh ? (*seed_ptr + site * 0xD1B54A32D192ED03ull) : 0ull;
  load_tile<FA_ROWS, D>(Qs, qb, ldq, i0, Sq, d);
  load_tile<FA_BLK, D>(Ks, kb, ldk, 0, Sk, d);
  load_tile<FA_BLK, D>(Vs, vb, ldv, 0, Sk, d);
  cp_async_commit();
  const int nkb = (Sk + FA_BLK - 1) / FA_BLK;
  const int row[2] = {i0 + warp * 16 + g, i0 + warp * 16 + g + 8};
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float acc[DT][4];
#pragma unroll
  for (int i = 0; i < DT; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
  for (int kbk = 0; kbk < nkb; ++kbk) {
    const int buf = kbk & 1;
    if (kbk + 1 < nkb) {
      load_tile<FA_BLK, D>(Ks + (buf ^ 1) * FA_BLK * LD, kb, ldk, (kbk + 1) * FA_BLK, Sk, d);
      load_tile<FA_BLK, D>(Vs + (buf ^ 1) * FA_BLK * LD, vb, ldv, (kbk + 1) * FA_BLK, Sk, d);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    float s[NT][4];
    qk_block<D, NT, NS, false>(s, Qs + warp * 16 * LD, Ks + buf * FA_BLK * LD, lane);
    const int j0 = kbk * FA_BLK + 2 * t;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float mx = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float x = (j0 + nt * 8 + e < Sk) ? s[nt][2 * r + e] * scale : -INFINITY;
          s[nt][2 * r + e] = x;
          mx = fmaxf(mx, x);
        }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float mn = fmaxf(m[r], mx), corr = expf(m[r] - mn);   // every key block holds a valid key: mn is finite
      m[r] = mn;
      const size_t drop = ((size_t)bh * Sq + row[r]) * Sk + j0;
      float sum = 0.f;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float p = expf(s[nt][2 * r + e] - mn);
          sum += p;
          if (thresh) p *= dropout_scale(seed, drop + nt * 8 + e, thresh, inv_keep);
          s[nt][2 * r + e] = p;
        }
      l[r] = l[r] * corr + sum;
#pragma unroll
      for (int i = 0; i < DT; ++i) { acc[i][2 * r] *= corr; acc[i][2 * r + 1] *= corr; }
    }
    pv_block<D, NT, NS>(acc, s, Vs + buf * FA_BLK * LD, lane);
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
    const float inv = 1.f / l[r];
    if (row[r] < Sq) {
      float* orow = o + (size_t)(b * Sq + row[r]) * ldo + h * d;
#pragma unroll
      for (int i = 0; i < DT; ++i) {
        const int c = i * 8 + 2 * t;
        if (c < d) *reinterpret_cast<float2*>(orow + c) = make_float2(acc[i][2 * r] * inv, acc[i][2 * r + 1] * inv);
      }
      if (t == 0) stats[(size_t)bh * Sq + row[r]] = make_float2(m[r], inv);
    }
  }
}

template <int D, int NS>
__global__ void __launch_bounds__(FA_THREADS)
attn_fused_bwd_dq_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ k, int ldk, const float* __restrict__ v, int ldv,
                         const float* __restrict__ o, int ldo, const float* __restrict__ dout, int lddo, const float2* __restrict__ stats,
                         float* __restrict__ dq, int lddq, int H, int Sq, int Sk, int d, int nqb, float scale,
                         const unsigned long long* __restrict__ seed_ptr, unsigned long long site, uint32_t thresh, float inv_keep) {
  constexpr int LD = D + 4, DT = D / 8, NT = FA_BLK / 8;
  extern __shared__ __align__(16) float smem[];
  float* Qs = smem;                       // [64][LD]
  float* Gs = Qs + FA_ROWS * LD;          // [64][LD]  dO
  float* Ks = Gs + FA_ROWS * LD;          // [2][64][LD]
  float* Vs = Ks + 2 * FA_BLK * LD;       // [2][64][LD]
  const int bh = blockIdx.x / nqb, b = bh / H, h = bh - b * H, i0 = (blockIdx.x - bh * nqb) * FA_ROWS;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const float* qb = q + (size_t)b * Sq * ldq + h * d;
  const float* gb = dout + (size_t)b * Sq * lddo + h * d;
  const float* ob = o + (size_t)b * Sq * ldo + h * d;
  const float* kb = k + (size_t)b * Sk * ldk + h * d;
  const float* vb = v + (size_t)b * Sk * ldv + h * d;
  pdl_sync();
  const unsigned long long seed = thresh ? (*seed_ptr + site * 0xD1B54A32D192ED03ull) : 0ull;
  load_tile<FA_ROWS, D>(Qs, qb, ldq, i0, Sq, d);
  load_tile<FA_ROWS, D>(Gs, gb, lddo, i0, Sq, d);
  load_tile<FA_BLK, D>(Ks, kb, ldk, 0, Sk, d);
  load_tile<FA_BLK, D>(Vs, vb, ldv, 0, Sk, d);
  cp_async_commit();
  const int row[2] = {i0 + warp * 16 + g, i0 + warp * 16 + g + 8};
  float2 st[2];
  float Dr[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const bool ok = row[r] < Sq;
    st[r] = ok ? stats[(size_t)bh * Sq + row[r]] : make_float2(0.f, 0.f);
    Dr[r] = ok ? row_term(ob + (size_t)row[r] * ldo, gb + (size_t)row[r] * lddo, d) : 0.f;
  }
  const int nkb = (Sk + FA_BLK - 1) / FA_BLK;
  float acc[DT][4];
#pragma unroll
  for (int i = 0; i < DT; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
  for (int kbk = 0; kbk < nkb; ++kbk) {
    const int buf = kbk & 1;
    if (kbk + 1 < nkb) {
      load_tile<FA_BLK, D>(Ks + (buf ^ 1) * FA_BLK * LD, kb, ldk, (kbk + 1) * FA_BLK, Sk, d);
      load_tile<FA_BLK, D>(Vs + (buf ^ 1) * FA_BLK * LD, vb, ldv, (kbk + 1) * FA_BLK, Sk, d);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const float* Kb = Ks + buf * FA_BLK * LD;
    float s[NT][4], dp[NT][4];
    qk_block<D, NT, NS, false>(s, Qs + warp * 16 * LD, Kb, lane);
    qk_block<D, NT, NS, false>(dp, Gs + warp * 16 * LD, Vs + buf * FA_BLK * LD, lane);
    const int j0 = kbk * FA_BLK + 2 * t;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const size_t drop = ((size_t)bh * Sq + row[r]) * Sk + j0;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float ds = 0.f;
          if (j0 + nt * 8 + e < Sk) {
            const float p = expf(s[nt][2 * r + e] * scale - st[r].x) * st[r].y;
            const float mk = thresh ? dropout_scale(seed, drop + nt * 8 + e, thresh, inv_keep) : 1.f;
            ds = p * (mk * dp[nt][2 * r + e] - Dr[r]);
          }
          s[nt][2 * r + e] = ds;
        }
    }
    pv_block<D, NT, NS>(acc, s, Kb, lane);
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (row[r] >= Sq) continue;
    float* drow = dq + (size_t)(b * Sq + row[r]) * lddq + h * d;
#pragma unroll
    for (int i = 0; i < DT; ++i) {
      const int c = i * 8 + 2 * t;
      if (c < d) *reinterpret_cast<float2*>(drow + c) = make_float2(acc[i][2 * r] * scale, acc[i][2 * r + 1] * scale);
    }
  }
}

template <int D, int NS>
__global__ void __launch_bounds__(FA_THREADS)
attn_fused_bwd_dkdv_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ k, int ldk, const float* __restrict__ v, int ldv,
                           const float* __restrict__ o, int ldo, const float* __restrict__ dout, int lddo, const float2* __restrict__ stats,
                           float* __restrict__ dk, int lddk, float* __restrict__ dv, int lddv, int H, int Sq, int Sk, int d, int nkb, float scale,
                           const unsigned long long* __restrict__ seed_ptr, unsigned long long site, uint32_t thresh, float inv_keep) {
  constexpr int LD = D + 4, DT = D / 8, QB = fa_qblk<D>(), NT = QB / 8;
  extern __shared__ __align__(16) float smem[];
  float* Ks = smem;                       // [64][LD]
  float* Vs = Ks + FA_ROWS * LD;          // [64][LD]
  float* Qs = Vs + FA_ROWS * LD;          // [2][QB][LD]
  float* Gs = Qs + 2 * QB * LD;           // [2][QB][LD]  dO
  float* Rs = Gs + 2 * QB * LD;           // [2][3][QB]   row max, 1 / row sum, D
  const int bh = blockIdx.x / nkb, b = bh / H, h = bh - b * H, j0 = (blockIdx.x - bh * nkb) * FA_ROWS;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const float* qb = q + (size_t)b * Sq * ldq + h * d;
  const float* gb = dout + (size_t)b * Sq * lddo + h * d;
  const float* ob = o + (size_t)b * Sq * ldo + h * d;
  const float* kb = k + (size_t)b * Sk * ldk + h * d;
  const float* vb = v + (size_t)b * Sk * ldv + h * d;
  pdl_sync();
  const unsigned long long seed = thresh ? (*seed_ptr + site * 0xD1B54A32D192ED03ull) : 0ull;
  auto row_terms = [&](int qblk, float* R) {      // statistics and D of query block qblk (rows past Sq: P = 0)
    const int i = qblk * QB + threadIdx.x;
    if (threadIdx.x < QB) {
      const bool ok = i < Sq;
      const float2 st = ok ? stats[(size_t)bh * Sq + i] : make_float2(0.f, 0.f);
      R[threadIdx.x] = st.x; R[QB + threadIdx.x] = st.y;
      R[2 * QB + threadIdx.x] = ok ? row_term(ob + (size_t)i * ldo, gb + (size_t)i * lddo, d) : 0.f;
    }
  };
  load_tile<FA_ROWS, D>(Ks, kb, ldk, j0, Sk, d);
  load_tile<FA_ROWS, D>(Vs, vb, ldv, j0, Sk, d);
  load_tile<QB, D>(Qs, qb, ldq, 0, Sq, d);
  load_tile<QB, D>(Gs, gb, lddo, 0, Sq, d);
  cp_async_commit();
  row_terms(0, Rs);
  const int nqb = (Sq + QB - 1) / QB;
  const int key[2] = {j0 + warp * 16 + g, j0 + warp * 16 + g + 8};
  float ak[DT][4], av[DT][4];
#pragma unroll
  for (int i = 0; i < DT; ++i) {
    ak[i][0] = ak[i][1] = ak[i][2] = ak[i][3] = 0.f;
    av[i][0] = av[i][1] = av[i][2] = av[i][3] = 0.f;
  }
  for (int qbk = 0; qbk < nqb; ++qbk) {
    const int buf = qbk & 1;
    if (qbk + 1 < nqb) {
      load_tile<QB, D>(Qs + (buf ^ 1) * QB * LD, qb, ldq, (qbk + 1) * QB, Sq, d);
      load_tile<QB, D>(Gs + (buf ^ 1) * QB * LD, gb, lddo, (qbk + 1) * QB, Sq, d);
      cp_async_commit();
      row_terms(qbk + 1, Rs + (buf ^ 1) * 3 * QB);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const float* Qb = Qs + buf * QB * LD;
    const float* Gb = Gs + buf * QB * LD;
    const float* R = Rs + buf * 3 * QB;
    float s[NT][4], dp[NT][4];
    qk_block<D, NT, NS, true>(s, Ks + warp * 16 * LD, Qb, lane);    // S^T: rows = keys, columns = queries
    qk_block<D, NT, NS, true>(dp, Vs + warp * 16 * LD, Gb, lane);   // dP~^T
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int il = nt * 8 + 2 * t + e;
        const float mi = R[il], inv = R[QB + il], Di = R[2 * QB + il];
        const size_t drop = ((size_t)bh * Sq + qbk * QB + il) * Sk;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const float p = expf(s[nt][2 * r + e] * scale - mi) * inv;
          const float mk = thresh ? dropout_scale(seed, drop + key[r], thresh, inv_keep) : 1.f;
          s[nt][2 * r + e] = p * (mk * dp[nt][2 * r + e] - Di);    // dS^T
          dp[nt][2 * r + e] = p * mk;                              // P~^T
        }
      }
    pv_block<D, NT, NS>(av, dp, Gb, lane);   // dV += P~^T dO
    pv_block<D, NT, NS>(ak, s, Qb, lane);    // dK += dS^T Q
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (key[r] >= Sk) continue;
    float* krow = dk + (size_t)(b * Sk + key[r]) * lddk + h * d;
    float* vrow = dv + (size_t)(b * Sk + key[r]) * lddv + h * d;
#pragma unroll
    for (int i = 0; i < DT; ++i) {
      const int c = i * 8 + 2 * t;
      if (c < d) {
        *reinterpret_cast<float2*>(krow + c) = make_float2(ak[i][2 * r] * scale, ak[i][2 * r + 1] * scale);
        *reinterpret_cast<float2*>(vrow + c) = make_float2(av[i][2 * r], av[i][2 * r + 1]);
      }
    }
  }
}

namespace {
// f(integral_constant<D>, integral_constant<NS>) for the padded head dim of d and the split count
template <class F> int fa_dispatch(int d, int nsplit, F&& f) {
  auto go = [&](auto dd) { return nsplit == 3 ? f(dd, std::integral_constant<int, 3>()) : f(dd, std::integral_constant<int, 1>()); };
  if (d <= 8) return go(std::integral_constant<int, 8>());
  if (d <= 16) return go(std::integral_constant<int, 16>());
  if (d <= 32) return go(std::integral_constant<int, 32>());
  if (d <= 64) return go(std::integral_constant<int, 64>());
  return go(std::integral_constant<int, 128>());
}
template <class K> int fa_smem_attr(K kernel, size_t smem) {
  RIH_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  return 0;
}
int attn_tc_check(const char* who, int Sq, int Sk, int d, int nsplit) {
  RIH_REQUIRE(Sk > 0 && Sk <= 512, "%s: Sk=%d unsupported (max 512)", who, Sk);
  RIH_REQUIRE(d >= 4 && d <= 128 && d % 4 == 0, "%s: head dim %d unsupported (a multiple of 4 in 4..128)", who, d);
  RIH_REQUIRE(nsplit == 1 || nsplit == 3, "%s: nsplit must be 1 (TF32) or 3 (3xTF32)", who);
  RIH_REQUIRE(Sq >= 0, "%s: Sq=%d", who, Sq);
  return 0;
}
bool tok_aligned(const void* p, int ld) { return ((reinterpret_cast<uintptr_t>(p) & 15) == 0) && ld % 4 == 0; }
}  // namespace

// Forward on the tensor cores.  q/k/v/o: token matrices [B*S, ld] (head h = columns [h*d, (h+1)*d)), rows 16-byte aligned.
//   slot 8  stats: [B*H*Sq, 2] receives per query row (m, 1/l): row max of the scaled scores and the reciprocal of sum_j exp(S_ij - m),
//                  kept for the backward pass (which recomputes P from them)
//   slot 9, 10: reserved, must be NULL / 0
// nsplit: 1 = TF32, 3 = 3xTF32 (fp32-faithful).  Sk <= 512, d % 4 == 0, d <= 128.
// reference: SelfAttn.self_attn models/model_attn/self_attn.py:63-76, inter_attn.py:90-105
RIH_API int rih_attn_tc_fwd(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, float* o, int ldo, float* stats,
                            const float* reserved, int reserved_ld, int B, int H, int Sq, int Sk, int d, float scale, float dropout_p,
                            const unsigned long long* seed_ptr, unsigned long long site, int nsplit, cudaStream_t s) {
  if (int e = attn_tc_check("attn_tc_fwd", Sq, Sk, d, nsplit)) return e;
  RIH_REQUIRE(reserved == nullptr && reserved_ld == 0, "attn_tc_fwd: arguments 9 and 10 are reserved and must be NULL / 0");
  RIH_REQUIRE(tok_aligned(q, ldq) && tok_aligned(k, ldk) && tok_aligned(v, ldv) && tok_aligned(o, ldo),
              "attn_tc_fwd: operands must be 16-byte aligned with row strides that are multiples of 4 floats");
  if (B * H == 0 || Sq == 0) return 0;
  RIH_REQUIRE(stats, "attn_tc_fwd: the row-statistics output is required");
  const uint32_t thresh = dropout_p > 0.f ? dropout_thresh(dropout_p) : 0u;
  const float ik = dropout_p > 0.f ? 1.f / (1.f - dropout_p) : 1.f;
  RIH_REQUIRE(!thresh || seed_ptr, "attn_tc_fwd: dropout needs a device seed");
  const int nqb = cdiv(Sq, FA_ROWS);
  if (int e = fa_dispatch(d, nsplit, [&](auto dd, auto ns) {
        constexpr int D = decltype(dd)::value, NS = decltype(ns)::value;
        const size_t smem = sizeof(float) * (FA_ROWS + 4 * FA_BLK) * (D + 4);
        static bool attr = false;
        if (!attr) { if (int e2 = fa_smem_attr(attn_fused_fwd_kernel<D, NS>, smem)) return e2; attr = true; }
        launch_k(attn_fused_fwd_kernel<D, NS>, (long long)B * H * nqb, FA_THREADS, smem, s, q, ldq, k, ldk, v, ldv, o, ldo,
                 reinterpret_cast<float2*>(stats), H, Sq, Sk, d, nqb, scale, seed_ptr, site, thresh, ik);
        return 0;
      }))
    return e;
  return check_launch("attn_tc_fwd");
}

// Backward on the tensor cores.  slot 8: the forward's row statistics; slot 9: O, the forward's output (row stride ldo, slot 11);
// slot 10: reserved, must be NULL.  dq / dk / dv are written (not accumulated).
RIH_API int rih_attn_tc_bwd(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, const float* dout, int lddo,
                            const float* stats, const float* o, const float* reserved, int ldo, float* dq, int lddq, float* dk, int lddk,
                            float* dv, int lddv, int B, int H, int Sq, int Sk, int d, float scale, float dropout_p,
                            const unsigned long long* seed_ptr, unsigned long long site, int nsplit, cudaStream_t s) {
  if (int e = attn_tc_check("attn_tc_bwd", Sq, Sk, d, nsplit)) return e;
  RIH_REQUIRE(reserved == nullptr, "attn_tc_bwd: argument 10 is reserved and must be NULL");
  RIH_REQUIRE(tok_aligned(q, ldq) && tok_aligned(k, ldk) && tok_aligned(v, ldv) && tok_aligned(dout, lddo) && tok_aligned(o, ldo) &&
              tok_aligned(dq, lddq) && tok_aligned(dk, lddk) && tok_aligned(dv, lddv),
              "attn_tc_bwd: operands must be 16-byte aligned with row strides that are multiples of 4 floats");
  if (B * H == 0 || Sq == 0) return 0;
  RIH_REQUIRE(stats && o, "attn_tc_bwd: the row statistics and O are required");
  const uint32_t thresh = dropout_p > 0.f ? dropout_thresh(dropout_p) : 0u;
  const float ik = dropout_p > 0.f ? 1.f / (1.f - dropout_p) : 1.f;
  RIH_REQUIRE(!thresh || seed_ptr, "attn_tc_bwd: dropout needs a device seed");
  const float2* st = reinterpret_cast<const float2*>(stats);
  const int nqb = cdiv(Sq, FA_ROWS), nkb = cdiv(Sk, FA_ROWS);
  if (int e = fa_dispatch(d, nsplit, [&](auto dd, auto ns) {
        constexpr int D = decltype(dd)::value, NS = decltype(ns)::value, QB = fa_qblk<D>();
        const size_t smem_q = sizeof(float) * (2 * FA_ROWS + 4 * FA_BLK) * (D + 4);
        const size_t smem_k = sizeof(float) * ((2 * FA_ROWS + 4 * QB) * (D + 4) + 6 * QB);
        static bool attr = false;
        if (!attr) {
          if (int e2 = fa_smem_attr(attn_fused_bwd_dq_kernel<D, NS>, smem_q)) return e2;
          if (int e2 = fa_smem_attr(attn_fused_bwd_dkdv_kernel<D, NS>, smem_k)) return e2;
          attr = true;
        }
        launch_k(attn_fused_bwd_dq_kernel<D, NS>, (long long)B * H * nqb, FA_THREADS, smem_q, s, q, ldq, k, ldk, v, ldv, o, ldo, dout, lddo,
                 st, dq, lddq, H, Sq, Sk, d, nqb, scale, seed_ptr, site, thresh, ik);
        launch_k(attn_fused_bwd_dkdv_kernel<D, NS>, (long long)B * H * nkb, FA_THREADS, smem_k, s, q, ldq, k, ldk, v, ldv, o, ldo, dout,
                 lddo, st, dk, lddk, dv, lddv, H, Sq, Sk, d, nkb, scale, seed_ptr, site, thresh, ik);
        return 0;
      }))
    return e;
  return check_launch("attn_tc_bwd");
}
