// Fused multi-head attention core (SIMT fp32, exact softmax): O = dropout(softmax(Q K^T * scale)) V
// One CTA per (batch, head[, query split]): the whole K/V of a head (<= 512 keys, d <= 128, d % 4 == 0) lives in shared
// memory; each warp processes a block of query rows at once with register blocking and 128-bit shared-memory reads.
// reference: SelfAttn.self_attn  models/model_attn/self_attn.py:63-76 ; inter_attn.inter_attn  inter_attn.py:73-123
// Tensor addressing: element (b, row, h, dd) of T is  T + b*T_bs + row*ldT + h*d + dd.
#include "common.cuh"
#include "bgemm.cuh"
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
// The same operator with its four contractions on the wgmma tensor cores (TMA -> shared memory -> wgmma, 3xTF32 or TF32), as
// batched per-head GEMMs over 4-D tensor maps (gemm_tc.cu: bgemm_tf32) around two warp-per-row softmax kernels:
//   forward : S = scale * Q K^T  ->  P = softmax(S), P~ = dropout(P)  ->  O = P~ V
//   backward: dP~ = dO V^T  ->  dS = P o (dP~ o M - rowsum(dP~ o M o P)), P~ = P o M  ->  dQ = scale dS K, dK = scale dS^T Q, dV = P~^T dO
// The score matrices [B*H, Sq, Skp] (Skp = Sk rounded up to 4 floats so that rows are 16-byte aligned for TMA) live in HBM / L2
// between the launches, like the reference's attn tensor (self_attn.py:69-72); P is kept for the backward pass.
constexpr int SM_MAXT = 16;   // keys per lane (Sk <= 512)

__global__ void __launch_bounds__(256)
attn_softmax_fwd_kernel(float* __restrict__ P, float* __restrict__ Pd, long long rows, int Sq, int Sk, int Skp,
                        const unsigned long long* __restrict__ seed_ptr, unsigned long long site, uint32_t thresh, float inv_keep) {
  pdl_sync();
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const unsigned long long seed = thresh ? (*seed_ptr + site * 0xD1B54A32D192ED03ull) : 0ull;
  float* p = P + row * Skp;
  float x[SM_MAXT];
  float mx = -INFINITY;
#pragma unroll
  for (int t = 0; t < SM_MAXT; ++t) {
    const int j = lane + 32 * t;
    x[t] = (j < Sk) ? p[j] : -INFINITY;
    mx = fmaxf(mx, x[t]);
  }
  mx = warp_max(mx);
  float sum = 0.f;
#pragma unroll
  for (int t = 0; t < SM_MAXT; ++t) {
    const int j = lane + 32 * t;
    x[t] = (j < Sk) ? expf(x[t] - mx) : 0.f;
    sum += x[t];
  }
  sum = warp_sum(sum);
  const float inv = 1.f / sum;
  const size_t drop_base = (size_t)row * Sk;
#pragma unroll
  for (int t = 0; t < SM_MAXT; ++t) {
    const int j = lane + 32 * t;
    if (j < Sk) {
      const float pr = x[t] * inv;
      p[j] = pr;
      if (thresh) Pd[row * Skp + j] = pr * dropout_scale(seed, drop_base + j, thresh, inv_keep);
    }
  }
}

// dS (in place over dP) and, with dropout, P~ = P o M (the operand of dV = P~^T dO)
__global__ void __launch_bounds__(256)
attn_softmax_bwd_kernel(const float* __restrict__ P, float* __restrict__ dP, float* __restrict__ Pd, long long rows, int Sq, int Sk, int Skp,
                        const unsigned long long* __restrict__ seed_ptr, unsigned long long site, uint32_t thresh, float inv_keep) {
  pdl_sync();
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const unsigned long long seed = thresh ? (*seed_ptr + site * 0xD1B54A32D192ED03ull) : 0ull;
  const float* p = P + row * Skp;
  float* g = dP + row * Skp;
  const size_t drop_base = (size_t)row * Sk;
  float pr[SM_MAXT], gm[SM_MAXT];
  float dl = 0.f;
#pragma unroll
  for (int t = 0; t < SM_MAXT; ++t) {
    const int j = lane + 32 * t;
    pr[t] = 0.f; gm[t] = 0.f;
    if (j < Sk) {
      pr[t] = p[j];
      const float m = thresh ? dropout_scale(seed, drop_base + j, thresh, inv_keep) : 1.f;
      gm[t] = g[j] * m;
      if (thresh) Pd[row * Skp + j] = pr[t] * m;
      dl = fmaf(gm[t], pr[t], dl);
    }
  }
  dl = warp_sum(dl);
#pragma unroll
  for (int t = 0; t < SM_MAXT; ++t) {
    const int j = lane + 32 * t;
    if (j < Sk) g[j] = pr[t] * (gm[t] - dl);
  }
}

static inline tc::BOperand tok(const float* p, int S, int d, int ld) { return tc::BOperand{p, 1, S, d, ld}; }
static inline tc::BOperand scr(const float* p, int R, int C, int Cp) { return tc::BOperand{p, 0, R, C, Cp}; }
static int attn_tc_check(const char* who, int Sq, int Sk, int d, int ldp) {
  RIH_REQUIRE(Sk > 0 && Sk <= 32 * SM_MAXT, "%s: Sk=%d unsupported (max %d)", who, Sk, 32 * SM_MAXT);
  RIH_REQUIRE(d >= 4 && d % 4 == 0, "%s: head dim %d must be a multiple of 4", who, d);
  RIH_REQUIRE(ldp >= Sk && ldp % 4 == 0, "%s: score row stride %d must be >= Sk and a multiple of 4 floats", who, ldp);
  return 0;
}

// Forward on the tensor cores.  q/k/v/o: token matrices [B*S, ld] (head h = columns [h*d, (h+1)*d)); P: [B*H, Sq, ldp] receives the
// softmax probabilities (kept for backward); Pd: same shape, dropped / rescaled probabilities (only touched when dropout_p > 0).
// nsplit: 1 = TF32, 3 = 3xTF32 (fp32-faithful).  reference: SelfAttn.self_attn models/model_attn/self_attn.py:63-76, inter_attn.py:90-105
RIH_API int rih_attn_tc_fwd(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, float* o, int ldo, float* P, float* Pd, int ldp,
                            int B, int H, int Sq, int Sk, int d, float scale, float dropout_p, const unsigned long long* seed_ptr, unsigned long long site,
                            int nsplit, cudaStream_t s) {
  if (int e = attn_tc_check("attn_tc_fwd", Sq, Sk, d, ldp)) return e;
  RIH_REQUIRE(nsplit == 1 || nsplit == 3, "attn_tc_fwd: nsplit must be 1 (TF32) or 3 (3xTF32)");
  if (B * H == 0 || Sq == 0) return 0;
  tc::set_nsplit(nsplit); tc::set_acc_scale(1.f);
  if (int e = tc::bgemm_tf32(tok(q, Sq, d, ldq), 0, tok(k, Sk, d, ldk), 0, scr(P, Sq, Sk, ldp), B, H, Sq, Sk, d, scale, s)) return e;
  const uint32_t thresh = dropout_p > 0.f ? dropout_thresh(dropout_p) : 0u;
  const float ik = dropout_p > 0.f ? 1.f / (1.f - dropout_p) : 1.f;
  RIH_REQUIRE(!thresh || (Pd && seed_ptr), "attn_tc_fwd: dropout needs the Pd buffer and a device seed");
  const long long rows = (long long)B * H * Sq;
  launch_k(attn_softmax_fwd_kernel, cdiv(rows, 8), 256, 0, s, P, Pd, rows, Sq, Sk, ldp, seed_ptr, site, thresh, ik);
  if (int e = check_launch("attn_softmax_fwd")) return e;
  return tc::bgemm_tf32(scr(thresh ? Pd : P, Sq, Sk, ldp), 0, tok(v, Sk, d, ldv), 1, tok(o, Sq, d, ldo), B, H, Sq, d, Sk, 1.f, s);
}

// Backward on the tensor cores.  ws: [B*H, Sq, ldp] scratch (dP~ then dS); Pd: scratch for P~ (dropout only).
RIH_API int rih_attn_tc_bwd(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, const float* dout, int lddo, const float* P,
                            float* ws, float* Pd, int ldp, float* dq, int lddq, float* dk, int lddk, float* dv, int lddv,
                            int B, int H, int Sq, int Sk, int d, float scale, float dropout_p, const unsigned long long* seed_ptr, unsigned long long site,
                            int nsplit, cudaStream_t s) {
  if (int e = attn_tc_check("attn_tc_bwd", Sq, Sk, d, ldp)) return e;
  RIH_REQUIRE(nsplit == 1 || nsplit == 3, "attn_tc_bwd: nsplit must be 1 (TF32) or 3 (3xTF32)");
  if (B * H == 0 || Sq == 0) return 0;
  tc::set_nsplit(nsplit); tc::set_acc_scale(1.f);
  if (int e = tc::bgemm_tf32(tok(dout, Sq, d, lddo), 0, tok(v, Sk, d, ldv), 0, scr(ws, Sq, Sk, ldp), B, H, Sq, Sk, d, 1.f, s)) return e;
  const uint32_t thresh = dropout_p > 0.f ? dropout_thresh(dropout_p) : 0u;
  const float ik = dropout_p > 0.f ? 1.f / (1.f - dropout_p) : 1.f;
  RIH_REQUIRE(!thresh || (Pd && seed_ptr), "attn_tc_bwd: dropout needs the Pd buffer and a device seed");
  const long long rows = (long long)B * H * Sq;
  launch_k(attn_softmax_bwd_kernel, cdiv(rows, 8), 256, 0, s, P, ws, Pd, rows, Sq, Sk, ldp, seed_ptr, site, thresh, ik);
  if (int e = check_launch("attn_softmax_bwd")) return e;
  const float* Pt = thresh ? Pd : P;
  if (int e = tc::bgemm_tf32(scr(ws, Sq, Sk, ldp), 0, tok(k, Sk, d, ldk), 1, tok(dq, Sq, d, lddq), B, H, Sq, d, Sk, scale, s)) return e;     // dQ = scale dS K
  if (int e = tc::bgemm_tf32(scr(ws, Sq, Sk, ldp), 1, tok(q, Sq, d, ldq), 1, tok(dk, Sk, d, lddk), B, H, Sk, d, Sq, scale, s)) return e;     // dK = scale dS^T Q
  return tc::bgemm_tf32(scr(Pt, Sq, Sk, ldp), 1, tok(dout, Sq, d, lddo), 1, tok(dv, Sk, d, lddv), B, H, Sk, d, Sq, 1.f, s);                 // dV = P~^T dO
}
