// The pose optimiser's hand-prior and contact terms (GeOptimizer.loss_fn, pose_data_optimize/hocontact/postprocess/
// geo_optimizer_both_batch.py:567-616, 705-757, summed at :805-825) for both hands, forward and backward:
//   * the anchor layer (manopth/manopth/anchorutils.py:51-65): anchor a = v0 + w1 (v1 - v0) + w2 (v2 - v0) of its face (v0, v1, v2);
//   * quat-norm  mean((|q|^2 - 1)^2) over B x 16 on the unnormalised quaternions (geo_loss.py:197-202);
//   * edge       mean((|v_i - v_j| - L0)^2) over B x E (geo_loss.py:180-183, 241-244);
//   * contact    sum e |A_main[anchor_id] - A_sub|^2 / sum mask, 0 when sum mask <= 0 (geo_loss.py:20-27, optimiser :603-612);
//   * ergonomics hand_pose_ergonomics_loss (geo_loss.py:360-444) on M = zero_ja^T ja, ja = invM_U_n_0^T R(normalize(q)) invU_M_n_1^T
//     (scripts/HandPoseConverter.py:214-231); the host folds zero_ja^T invM_U_n_0^T into one matrix P per joint, so M = P R C.
// Each term is summed over both hands, as the reference's `+=` does.  One CTA per sample handles both hands; a one-CTA reduction sums the
// per-sample partials in a fixed order and decides the empty-mask case on the device.  The backward gathers vertex gradients through
// vertex -> edge and vertex -> anchor CSRs built at construction.  No float atomics: results are bitwise reproducible.
#include <algorithm>

#include "common.cuh"
#include "hand_pose.cuh"
using namespace rih;

namespace {

constexpr int V = 778, V3 = 2334, THREADS = 256, NWARPS = THREADS / 32, A_MAX = 128, NJ = 15, NPART = 8;
constexpr float PI_F = 3.14159265358979323846f;

struct GeoConsts {
  const int* fvi;         // [A,3] anchor faces
  const float* aw;        // [A,2] anchor weights
  const int* anc_ptr;     // [V+1] vertex -> (anchor, corner) CSR
  const int* anc_ent;     // [nnz] anchor index
  const float* anc_coef;  // [nnz] corner coefficient: 1 - w1 - w2, w1 or w2
  const int* edges;       // [E,2]
  const float* rest;      // [2,E] rest edge lengths of the right / left hand
  const int* e_ptr;       // [V+1] vertex -> edge CSR
  const int* e_other;     // [2E] the edge's other vertex
  const int* e_id;        // [2E] the edge's index
  const float* conv;      // [2,15,18] per hand and joint 1..15: P (row-major 3x3) then C
};

// anchorutils.py:57-64, with the reference's operation order (no contraction into FMAs)
__device__ __forceinline__ void anchor_pos(const float* vb, const int* f, const float* w, float* out) {
  for (int c = 0; c < 3; ++c) {
    const float o = vb[f[0] * 3 + c];
    const float b1 = __fsub_rn(vb[f[1] * 3 + c], o), b2 = __fsub_rn(vb[f[2] * 3 + c], o);
    out[c] = __fadd_rn(__fadd_rn(__fmul_rn(w[0], b1), __fmul_rn(w[1], b2)), o);
  }
}

// F.normalize(q, eps=1e-12) (quatutils.py:7-30), the left hand's (w, x, -y, -z) (HandPoseConverter.py:220-222), R, then M = P R C.
__device__ void joint_matrix(const float* q, int side, const float* conv, float* p, float* M) {
  const float nrm = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  const float d = fmaxf(nrm, 1e-12f);
  const float s = side ? -1.f : 1.f;
  p[0] = q[0] / d; p[1] = q[1] / d; p[2] = s * (q[2] / d); p[3] = s * (q[3] / d);
  float R[9], T[9];
  quat_to_R(p[0], p[1], p[2], p[3], R);
  mat3_mul(conv, R, T);
  mat3_mul(T, conv + 9, M);
}

// atan2's backward as torch takes it: k = dL/d(angle in radians) (= dL/d(degrees) * 180 / pi)  ->  dL/dy, dL/dx
__device__ __forceinline__ void atan2_grad(float y, float x, float k, float& dy, float& dx) {
  const float r2 = x * x + y * y;
  dy = k * x / r2;
  dx = -k * y / r2;
}

// One sample's hand_pose_ergonomics_loss term (geo_loss.py:360-444) for one hand: the mean over B is taken by the caller, so the step-1
// terms carry their 1/10 and the step-2 term its 1/4.  With dM != NULL also d(term)/dM [15][9].  Kinks (relu, max, clamp) sit where
// the squared term and its derivative are 0, so torch's tie rules give the same gradient as the one-sided ones used here; the only
// jump is the in-place zeroing of negative bend angles before step 4 (:429), whose gradient is 0 where the angle is negative.
__device__ float ergo_sample(const float (*M)[9], float (*dM)[9]) {
  float f1 = 0.f, f2 = 0.f, f3 = 0.f;
  float bend[NJ];
  for (int t = 0; t < NJ; ++t) {
    const float* m = M[t];
    float g[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (t % 3 != 0) {        // step 1, forbid_ts_idx: x.z^2 + y.z^2 + (z.z - 1)^2
      f1 += (m[6] * m[6] + m[7] * m[7] + (m[8] - 1.f) * (m[8] - 1.f)) / 10.f;
      g[6] += 2.f * m[6] / 10.f; g[7] += 2.f * m[7] / 10.f; g[8] += 2.f * (m[8] - 1.f) / 10.f;
    } else {
      const float r = (m[7] - m[5]) / 2.f;      // rot_vec . x = (M21 - M12) / 2
      if (t != 12) {         // step 2: no twist
        f2 += r * r / 4.f;
        g[7] += r / 4.f; g[5] -= r / 4.f;
      } else {               // thumb base: twist above 0.5
        const float u = fmaxf(r - 0.5f, 0.f);
        f2 += u * u;
        g[7] += u; g[5] -= u;
      }
      // splank limit, atan2(-x.z, x.x) in degrees
      const float sa = atan2f(-m[6], m[0]) * 180.f / PI_F;
      const float up = fmaxf(sa - c_spl_hi[t], 0.f), lo = fmaxf(c_spl_lo[t] - sa, 0.f);
      const float l = fmaxf(up, lo) / 180.f * PI_F;
      f3 += l * l;
      const float k = 2.f * l * (up > 0.f ? 1.f : (lo > 0.f ? -1.f : 0.f));
      float dy, dx;
      atan2_grad(-m[6], m[0], k, dy, dx);
      g[6] -= dy; g[0] += dx;
    }
    // bend limit, atan2(x.y, x.x) in degrees
    bend[t] = atan2f(m[3], m[0]) * 180.f / PI_F;
    const float up = fmaxf(bend[t] - c_bend_hi[t], 0.f), lo = fmaxf(c_bend_lo[t] - bend[t], 0.f);
    const float l = fmaxf(up, lo) / 180.f * PI_F;
    f3 += l * l;
    if (dM) {
      const float k = 2.f * l * (up > 0.f ? 1.f : (lo > 0.f ? -1.f : 0.f));
      float dy, dx;
      atan2_grad(m[3], m[0], k, dy, dx);
      g[3] += dy; g[0] += dx;
      for (int e = 0; e < 9; ++e) dM[t][e] = g[e];
    }
  }
  // step 4: negative bend angles zeroed in place, then min(b10 - b7 * 3 / 4, 0)^2 in radians
  const float b7 = bend[7] < 0.f ? 0.f : bend[7], b10 = bend[10] < 0.f ? 0.f : bend[10];
  const float r7 = b7 / 180.f * PI_F, r10 = b10 / 180.f * PI_F;
  const float c = fminf(r10 - r7 * 3.f / 4.f, 0.f);
  if (dM) {
    // dL/d(rad) -> dL/d(degrees) * 180 / pi = dL/d(rad): the two scale factors cancel
    const int ts[2] = {10, 7};
    const float kd[2] = {bend[10] < 0.f ? 0.f : 2.f * c, bend[7] < 0.f ? 0.f : -2.f * c * 3.f / 4.f};
    for (int i = 0; i < 2; ++i) {
      float dy, dx;
      atan2_grad(M[ts[i]][3], M[ts[i]][0], kd[i], dy, dx);
      dM[ts[i]][3] += dy; dM[ts[i]][0] += dx;
    }
  }
  return f1 + f2 + f3 + c * c;
}

struct Stage {
  float v[2][V3];
  float anc[2][A_MAX][3];
  float M[2][NJ][9];
  float red[NWARPS];
};

__device__ void stage_sample(Stage& s, const GeoConsts& gc, int A, const float* __restrict__ v_r, const float* __restrict__ v_l, int b, int tid) {
  const float* src[2] = {v_r + (size_t)b * V3, v_l + (size_t)b * V3};
  for (int o = tid; o < 2 * V3; o += THREADS) { const int h = o >= V3; s.v[h][o - h * V3] = src[h][o - h * V3]; }
  __syncthreads();
  for (int o = tid; o < 2 * A; o += THREADS) { const int h = o >= A, a = o - h * A; anchor_pos(s.v[h], gc.fvi + a * 3, gc.aw + a * 2, s.anc[h][a]); }
}

__global__ void __launch_bounds__(THREADS)
geo_prior_fwd_kernel(GeoConsts gc, int A, int E, int D, const float* __restrict__ q_r, const float* __restrict__ q_l,
                     const float* __restrict__ v_r, const float* __restrict__ v_l, const int* __restrict__ anchor_id,
                     const float* __restrict__ elastic, const int* __restrict__ mask, float* __restrict__ part, long long* __restrict__ count) {
  pdl_sync();
  __shared__ Stage s;
  __shared__ float s_ergo[2];
  const int b = blockIdx.x, tid = threadIdx.x;
  stage_sample(s, gc, A, v_r, v_l, b, tid);
  if (tid < 2 * NJ) {
    const int h = tid / NJ, t = tid % NJ;
    const float* q = (h ? q_l : q_r) + (size_t)b * 64 + (t + 1) * 4;
    float p[4];
    joint_matrix(q, h, gc.conv + (h * NJ + t) * 18, p, s.M[h][t]);
  }
  __syncthreads();
  if (tid == 0 || tid == 32) { const int h = tid >> 5; s_ergo[h] = ergo_sample(s.M[h], nullptr); }
  float qn[2] = {0.f, 0.f}, ed[2] = {0.f, 0.f}, cn = 0.f;
  long long mk = 0;
  if (tid < 32) {
    const int h = tid >> 4, j = tid & 15;
    const float* q = (h ? q_l : q_r) + (size_t)b * 64 + j * 4;
    const float d = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3] - 1.f;
    qn[h] = d * d;
  }
  for (int e = tid; e < E; e += THREADS) {
    const int i = gc.edges[2 * e], j = gc.edges[2 * e + 1];
    for (int h = 0; h < 2; ++h) {
      const float dx = s.v[h][i * 3] - s.v[h][j * 3], dy = s.v[h][i * 3 + 1] - s.v[h][j * 3 + 1], dz = s.v[h][i * 3 + 2] - s.v[h][j * 3 + 2];
      const float d = sqrtf(dx * dx + dy * dy + dz * dz) - gc.rest[h * E + e];
      ed[h] += d * d;
    }
  }
  const size_t base = (size_t)b * A * D;
  for (int o = tid; o < A * D; o += THREADS) {
    const int i = o / D, id = anchor_id[base + o];
    float d2 = 0.f;
    for (int c = 0; c < 3; ++c) { const float d = s.anc[1][i][c] - s.anc[0][id][c]; d2 += d * d; }
    cn += elastic[base + o] * d2;
    mk += mask[base + o];
  }
  float out[5];
  out[0] = block_sum<NWARPS>(qn[0], s.red, tid); out[1] = block_sum<NWARPS>(qn[1], s.red, tid);
  out[2] = block_sum<NWARPS>(ed[0], s.red, tid); out[3] = block_sum<NWARPS>(ed[1], s.red, tid);
  out[4] = block_sum<NWARPS>(cn, s.red, tid);
  // integer mask count: a warp-shuffle sum of 64-bit partials, then the warps in order
  __shared__ long long s_mk[NWARPS];
  for (int o = 16; o > 0; o >>= 1) mk += __shfl_xor_sync(0xffffffffu, mk, o);
  if ((tid & 31) == 0) s_mk[tid >> 5] = mk;
  __syncthreads();
  if (tid == 0) {
    long long m = 0;
    for (int w = 0; w < NWARPS; ++w) m += s_mk[w];
    float* p = part + (size_t)b * NPART;
    p[0] = out[0]; p[1] = out[1]; p[2] = out[2]; p[3] = out[3]; p[4] = out[4]; p[5] = s_ergo[0]; p[6] = s_ergo[1]; p[7] = 0.f;
    count[b] = m;
  }
}

// Sums the per-sample partials over the batch in a fixed order and applies the reference's normalisations.
// out = [quat_norm, edge, contact, ergonomics]; den_out = the mask total as a float, 0 when the total is <= 0.
__global__ void __launch_bounds__(THREADS)
geo_prior_reduce_kernel(const float* __restrict__ part, const long long* __restrict__ count, int B, int E, float* __restrict__ out,
                        float* __restrict__ den_out) {
  pdl_sync();
  __shared__ float s_red[NWARPS];
  __shared__ long long s_mk[NWARPS];
  const int tid = threadIdx.x;
  float acc[7] = {0, 0, 0, 0, 0, 0, 0};
  long long mk = 0;
  for (int b = tid; b < B; b += THREADS) {
    for (int k = 0; k < 7; ++k) acc[k] += part[(size_t)b * NPART + k];
    mk += count[b];
  }
  float S[7];
  for (int k = 0; k < 7; ++k) S[k] = block_sum<NWARPS>(acc[k], s_red, tid);
  for (int o = 16; o > 0; o >>= 1) mk += __shfl_xor_sync(0xffffffffu, mk, o);
  if ((tid & 31) == 0) s_mk[tid >> 5] = mk;
  __syncthreads();
  if (tid == 0) {
    long long m = 0;
    for (int w = 0; w < NWARPS; ++w) m += s_mk[w];
    const float nq = (float)B * 16.f, ne = (float)B * (float)E;
    out[0] = S[0] / nq + S[1] / nq;
    out[1] = S[2] / ne + S[3] / ne;
    const float den = m > 0 ? (float)m : 0.f;      // geo_loss.py:23-24, decided here instead of on the host
    out[2] = m > 0 ? S[4] / den : 0.f;
    out[3] = S[5] / (float)B + S[6] / (float)B;
    *den_out = den;
  }
}

__global__ void __launch_bounds__(THREADS)
geo_prior_bwd_kernel(GeoConsts gc, int A, int E, int D, int B, const float* __restrict__ q_r, const float* __restrict__ q_l,
                     const float* __restrict__ v_r, const float* __restrict__ v_l, const int* __restrict__ anchor_id,
                     const float* __restrict__ elastic, const float* __restrict__ g_terms, const float* __restrict__ den_in,
                     float* __restrict__ dq_r, float* __restrict__ dq_l, float* __restrict__ dv_r, float* __restrict__ dv_l) {
  pdl_sync();
  __shared__ Stage s;
  __shared__ float s_dM[2][NJ][9];
  __shared__ float s_dA[2][A_MAX][3];
  const int b = blockIdx.x, tid = threadIdx.x;
  const float g_qn = g_terms[0] / ((float)B * 16.f);
  const float g_ed = g_terms[1] * 2.f / ((float)B * (float)E);
  const float den = *den_in;
  const float g_ct = den > 0.f ? g_terms[2] / den : 0.f;
  const float g_er = g_terms[3] / (float)B;
  const bool want_q = dq_r || dq_l, want_v = dv_r || dv_l;
  if (want_v) stage_sample(s, gc, A, v_r, v_l, b, tid);
  if (want_q && tid < 2 * NJ) {
    const int h = tid / NJ, t = tid % NJ;
    float p[4];
    joint_matrix((h ? q_l : q_r) + (size_t)b * 64 + (t + 1) * 4, h, gc.conv + (h * NJ + t) * 18, p, s.M[h][t]);
  }
  __syncthreads();
  if (want_q && (tid == 0 || tid == 32)) { const int h = tid >> 5; ergo_sample(s.M[h], s_dM[h]); }
  if (want_v) {
    // contact: d/dA_main[a] = sum over (i, k) with anchor_id == a of 2 e (A_main[a] - A_sub[i]); d/dA_sub[i] = -sum_k of the same
    const size_t base = (size_t)b * A * D;
    for (int o = tid; o < 2 * A; o += THREADS) {
      const int h = o >= A, a = o - h * A;
      float g[3] = {0.f, 0.f, 0.f};
      if (h == 0) {
        for (int i = 0; i < A; ++i)
          for (int k = 0; k < D; ++k)
            if (anchor_id[base + i * D + k] == a) {
              const float e2 = 2.f * elastic[base + i * D + k];
              for (int c = 0; c < 3; ++c) g[c] += e2 * (s.anc[0][a][c] - s.anc[1][i][c]);
            }
      } else {
        for (int k = 0; k < D; ++k) {
          const int id = anchor_id[base + a * D + k];
          const float e2 = 2.f * elastic[base + a * D + k];
          for (int c = 0; c < 3; ++c) g[c] -= e2 * (s.anc[0][id][c] - s.anc[1][a][c]);
        }
      }
      for (int c = 0; c < 3; ++c) s_dA[h][a][c] = g_ct * g[c];
    }
  }
  __syncthreads();
  if (want_q && tid < 32) {
    const int h = tid >> 4, j = tid & 15;
    float* dq = h ? dq_l : dq_r;
    if (dq) {
      const float* q = (h ? q_l : q_r) + (size_t)b * 64 + j * 4;
      const float n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
      float d[4];
      for (int c = 0; c < 4; ++c) d[c] = g_qn * 2.f * (n2 - 1.f) * 2.f * q[c];
      if (j > 0) {
        const int t = j - 1;
        const float* P = gc.conv + (h * NJ + t) * 18;
        const float* C = P + 9;
        float G[9], T[9], dR[9];
        for (int e = 0; e < 9; ++e) G[e] = g_er * s_dM[h][t][e];
        // M = P R C  ->  dR = P^T G C^T
        for (int r = 0; r < 3; ++r)
          for (int c = 0; c < 3; ++c) T[r * 3 + c] = P[r] * G[c] + P[3 + r] * G[3 + c] + P[6 + r] * G[6 + c];
        for (int r = 0; r < 3; ++r)
          for (int c = 0; c < 3; ++c) dR[r * 3 + c] = T[r * 3] * C[c * 3] + T[r * 3 + 1] * C[c * 3 + 1] + T[r * 3 + 2] * C[c * 3 + 2];
        const float nrm = sqrtf(n2), den_q = fmaxf(nrm, 1e-12f);
        const float sg = h ? -1.f : 1.f;
        const float p[4] = {q[0] / den_q, q[1] / den_q, sg * (q[2] / den_q), sg * (q[3] / den_q)};
        float R[9], dp[4];
        quat_to_R(p[0], p[1], p[2], p[3], R);
        quat_R_backward(p, R, dR, dp);
        dp[2] *= sg; dp[3] *= sg;
        // q / max(|q|, eps): dq = dp / c - q (q . dp) / (|q| c^2) where |q| >= eps
        const float qdp = q[0] * dp[0] + q[1] * dp[1] + q[2] * dp[2] + q[3] * dp[3];
        const float k = (nrm >= 1e-12f && nrm > 0.f) ? qdp / (nrm * den_q * den_q) : 0.f;
        for (int c = 0; c < 4; ++c) d[c] += dp[c] / den_q - q[c] * k;
      }
      float* o = dq + (size_t)b * 64 + j * 4;
      for (int c = 0; c < 4; ++c) o[c] = d[c];
    }
  }
  if (want_v) {
    for (int o = tid; o < 2 * V; o += THREADS) {
      const int h = o >= V, vtx = o - h * V;
      float* dv = h ? dv_l : dv_r;
      if (!dv) continue;
      const float* vv = s.v[h];
      float g[3] = {0.f, 0.f, 0.f};
      for (int p = gc.e_ptr[vtx]; p < gc.e_ptr[vtx + 1]; ++p) {
        const int j = gc.e_other[p], e = gc.e_id[p];
        const float dx = vv[vtx * 3] - vv[j * 3], dy = vv[vtx * 3 + 1] - vv[j * 3 + 1], dz = vv[vtx * 3 + 2] - vv[j * 3 + 2];
        const float len = sqrtf(dx * dx + dy * dy + dz * dz);
        const float k = len > 0.f ? g_ed * (len - gc.rest[h * E + e]) / len : 0.f;    // torch.norm's gradient is 0 at 0
        g[0] += k * dx; g[1] += k * dy; g[2] += k * dz;
      }
      for (int p = gc.anc_ptr[vtx]; p < gc.anc_ptr[vtx + 1]; ++p) {
        const int a = gc.anc_ent[p];
        const float w = gc.anc_coef[p];
        for (int c = 0; c < 3; ++c) g[c] += w * s_dA[h][a][c];
      }
      float* out = dv + (size_t)b * V3 + vtx * 3;
      out[0] = g[0]; out[1] = g[1]; out[2] = g[2];
    }
  }
}

__global__ void geo_anchor_fwd_kernel(const int* __restrict__ fvi, const float* __restrict__ aw, int A, const float* __restrict__ verts, int nv,
                                      long long n, float* __restrict__ out) {
  pdl_sync();
  for (long long o = blockIdx.x * (long long)blockDim.x + threadIdx.x; o < n; o += (long long)gridDim.x * blockDim.x) {
    const long long b = o / A;
    const int a = (int)(o - b * A);
    anchor_pos(verts + b * nv * 3, fvi + a * 3, aw + a * 2, out + o * 3);
  }
}

__global__ void geo_anchor_bwd_kernel(const int* __restrict__ ptr, const int* __restrict__ ent, const float* __restrict__ coef, int A,
                                      const float* __restrict__ g_anc, int nv, long long n, float* __restrict__ dv) {
  pdl_sync();
  for (long long o = blockIdx.x * (long long)blockDim.x + threadIdx.x; o < n; o += (long long)gridDim.x * blockDim.x) {
    const long long b = o / nv;
    const int vtx = (int)(o - b * nv);
    float g[3] = {0.f, 0.f, 0.f};
    for (int p = ptr[vtx]; p < ptr[vtx + 1]; ++p) {
      const float* ga = g_anc + (b * A + ent[p]) * 3;
      for (int c = 0; c < 3; ++c) g[c] += coef[p] * ga[c];
    }
    for (int c = 0; c < 3; ++c) dv[o * 3 + c] = g[c];
  }
}

GeoConsts consts(const void* const* t) {
  return GeoConsts{(const int*)t[0], (const float*)t[1], (const int*)t[2], (const int*)t[3], (const float*)t[4], (const int*)t[5],
                   (const float*)t[6], (const int*)t[7], (const int*)t[8], (const int*)t[9], (const float*)t[10]};
}

int check_prior(const void* const* tables, int A, int E, int D, int B, const char* who) {
  RIH_REQUIRE(tables, "%s: NULL table array", who);
  for (int i = 0; i < 11; ++i) RIH_REQUIRE(tables[i] != nullptr, "%s: table %d is NULL", who, i);
  RIH_REQUIRE(A >= 1 && A <= A_MAX, "%s: %d anchors (1..%d)", who, A, A_MAX);
  RIH_REQUIRE(E >= 1 && D >= 1 && B >= 1, "%s: bad sizes E=%d D=%d B=%d", who, E, D, B);
  return 0;
}

}  // namespace

// The anchor layer (manopth/manopth/anchorlayer.py:21-27, anchorutils.py:51-65): verts [B,nv,3] -> anchors [B,A,3] with
// anchor a = v0 + w1 (v1 - v0) + w2 (v2 - v0) of face fvi[a] = (v0, v1, v2) and weights aw[a] = (w1, w2).  Indices are not checked here.
RIH_API int rih_geo_anchor_fwd(const int* fvi, const float* aw, int A, const float* verts, int nv, int B, float* anchors, cudaStream_t s) {
  RIH_REQUIRE(fvi && aw && A >= 1 && nv >= 1 && B >= 0, "geo_anchor_fwd: bad arguments (A=%d nv=%d B=%d)", A, nv, B);
  const long long n = (long long)B * A;
  if (n == 0) return 0;
  launch_k(geo_anchor_fwd_kernel, (unsigned)std::min<long long>(cdiv(n, 256), ew_ctas(s)), 256, 0, s, fvi, aw, A, verts, nv, n, anchors);
  return check_launch("geo_anchor_fwd");
}

// Backward of rih_geo_anchor_fwd: d_verts [B,nv,3] gathered through the vertex -> anchor CSR (ptr [nv+1], ent = anchor, coef = the
// vertex's coefficient 1 - w1 - w2, w1 or w2), so every vertex sums its anchors in a fixed order.
RIH_API int rih_geo_anchor_bwd(const int* ptr, const int* ent, const float* coef, int A, const float* g_anchors, int nv, int B, float* d_verts,
                               cudaStream_t s) {
  RIH_REQUIRE(ptr && A >= 1 && nv >= 1 && B >= 0, "geo_anchor_bwd: bad arguments (A=%d nv=%d B=%d)", A, nv, B);
  const long long n = (long long)B * nv;
  if (n == 0) return 0;
  launch_k(geo_anchor_bwd_kernel, (unsigned)std::min<long long>(cdiv(n, 256), ew_ctas(s)), 256, 0, s, ptr, ent, coef, A, g_anchors, nv, n, d_verts);
  return check_launch("geo_anchor_bwd");
}

// Forward of the four terms of both hands (geo_optimizer_both_batch.py:567-616, 705-757): one CTA per sample writes partial sums to
// part [B,8] and its mask count to count [B] (int64), then one CTA reduces them in a fixed order.
// tables: 11 device pointers (see GeoConsts); quat_r / quat_l [B,16,4] unnormalised; verts_r / verts_l [B,778,3]; anchor_id [B,A,D]
// int32 in [0,A); elastic [B,A,D]; mask [B,A,D] int32.  -> out [4] = quat-norm, edge, contact, ergonomics; den [1] = the mask total as
// a float, 0 when it is <= 0 (the contact term is 0 then).
RIH_API int rih_geo_prior_fwd(const void* const* tables, int A, int E, const float* quat_r, const float* quat_l, const float* verts_r,
                              const float* verts_l, const int* anchor_id, const float* elastic, const int* mask, int D, int B, float* part,
                              long long* count, float* out, float* den, cudaStream_t s) {
  if (int e = check_prior(tables, A, E, D, B, "geo_prior_fwd")) return e;
  RIH_REQUIRE(quat_r && quat_l && verts_r && verts_l && anchor_id && elastic && mask && part && count && out && den, "geo_prior_fwd: NULL argument");
  launch_k(geo_prior_fwd_kernel, B, THREADS, 0, s, consts(tables), A, E, D, quat_r, quat_l, verts_r, verts_l, anchor_id, elastic, mask, part, count);
  if (int e = check_launch("geo_prior_fwd")) return e;
  launch_k(geo_prior_reduce_kernel, 1, THREADS, 0, s, (const float*)part, (const long long*)count, B, E, out, den);
  return check_launch("geo_prior_reduce");
}

// Backward of rih_geo_prior_fwd.  g_terms [4]: the upstream gradients of the four terms, read on the device; den: the forward's mask
// total.  -> d_quat_r / d_quat_l [B,16,4], d_verts_r / d_verts_l [B,778,3]; each may be NULL when not needed.
RIH_API int rih_geo_prior_bwd(const void* const* tables, int A, int E, const float* quat_r, const float* quat_l, const float* verts_r,
                              const float* verts_l, const int* anchor_id, const float* elastic, int D, int B, const float* g_terms,
                              const float* den, float* d_quat_r, float* d_quat_l, float* d_verts_r, float* d_verts_l, cudaStream_t s) {
  if (int e = check_prior(tables, A, E, D, B, "geo_prior_bwd")) return e;
  RIH_REQUIRE(quat_r && quat_l && verts_r && verts_l && anchor_id && elastic && g_terms && den, "geo_prior_bwd: NULL argument");
  if (!(d_quat_r || d_quat_l || d_verts_r || d_verts_l)) return 0;
  launch_k(geo_prior_bwd_kernel, B, THREADS, 0, s, consts(tables), A, E, D, B, quat_r, quat_l, verts_r, verts_l, anchor_id, elastic, g_terms,
           den, d_quat_r, d_quat_l, d_verts_r, d_verts_l);
  return check_launch("geo_prior_bwd");
}
