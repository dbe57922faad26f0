// The pose optimiser's discriminator nature loss (GeOptimizer.NatureLoss, pose_data_optimize/hocontact/postprocess/
// geo_optimizer_both_batch.py:110-132, called at :802 on the normalised poses' joints 1..15) and its discriminator
// (Pos2dDiscriminator(num_joints=15, hid_dim=512), Ver2Code/Discriminator/discrim.py:66-105), forward and input gradient:
//   * features: quaternion_to_matrix (utlize.py:41-69, two_s = 2 / |q|^2) then matrix_to_euler_angles(R, 'XYZ') (utlize.py:208-289),
//     which reduces to (atan2(-R12, R22), asin(R02), atan2(-R01, R00)); feature 3 j + c for joint j + 1;
//   * MLP: d1 = lrelu(L1 x), d2 = lrelu(L2 d1), d3 = lrelu(L3 d2 + d1), d4 = L4 d3, d5 = lrelu(L_last d4), p = softmax(L_pred d5),
//     LeakyReLU slope 0.01 whose backward takes the slope at an input of exactly 0;
//   * loss: per hand mask = p1 < 1.5 p0, binary_cross_entropy(p[mask], (0, 1)) averaged over 2 n elements with torch's clamps, 0 for
//     an empty mask; the two hands summed.
// Exact fp32 on CUDA cores: one CTA owns a tile of 16 rows, keeps its activations in shared memory and streams the weights from L2
// through a register-prefetched shared-memory chunk.  The forward stores each hidden unit's sign as a bit (d > 0 iff the
// pre-activation is > 0), which is all the input-gradient chain needs.  Reductions run in a fixed order and there are no float
// atomics, so results are bitwise reproducible.  Nothing here depends on the GEMM precision mode of the rest of the library.
#include "common.cuh"
using namespace rih;

namespace {

constexpr int NJ = 15, NF = 45, H = 512, TR = 16, THREADS = 256, KC = 16, MS_LD = H + 4, NWARPS = THREADS / 32;
constexpr int SIGN_WORDS = 4 * H / 32;          // per row: the sign bits of d1, d2, d3 and d5
constexpr float SLOPE = 0.01f;

struct Params {
  const float* w[6];     // pose_layer_1..4, layer_last, layer_pred weights ([out, in] row-major, as torch stores them)
  const float* b[6];
};

struct Smem {
  float a[H][TR];        // activations / gradients, unit-major: a[unit][row]
  float b[H][TR];
  float ms[KC][MS_LD];   // one chunk of the weight matrix, reduction index-major
  float x[NF][TR];       // features, and in the backward their gradient
  float gl[TR][2];       // backward: d(logits)
  int live[TR];
};

__device__ __forceinline__ float lrelu(float z) { return z > 0.f ? z : SLOPE * z; }

// quaternion_to_matrix (utlize.py:54-69): the five entries the XYZ angles read
struct Rot5 { float r00, r01, r02, r12, r22; };
__device__ __forceinline__ Rot5 quat_rot(float r, float i, float j, float k, float& two_s) {
  two_s = 2.f / (r * r + i * i + j * j + k * k);
  return Rot5{1.f - two_s * (j * j + k * k), two_s * (i * j - k * r), two_s * (i * k + j * r), two_s * (j * k - i * r),
              1.f - two_s * (i * i + j * j)};
}

// Row `row` of the tile -> the pose of hand h = row >= B, sample row - h B.  NULL when past the end.
__device__ __forceinline__ const float* row_pose(const float* pa, long long lda, const float* pb, long long ldb, int B, int row) {
  return row < B ? pa + (long long)row * lda : pb + (long long)(row - B) * ldb;
}

// acc[r][c] += sum_i M[i][j] in[i][row] over i < I for rows rg*4 + r and units j = cg*4 + (c & 3) + 256 (c >> 2), with
//   TRANS:  M[i][j] = W[j * I + i]   (forward: W is [512, I])
//   !TRANS: M[i][j] = W[i * 512 + j] (backward, dx = dy W: W is [I, 512])
// The chunk of KC rows of M is staged in s.ms; the next chunk is loaded into registers while the current one is used.
template <bool TRANS, int I>
__device__ void matmul(Smem& s, const float* __restrict__ W, const float (*in)[TR], float (&acc)[4][8], int tid) {
  constexpr int PER = KC * H / THREADS;     // 32 values per thread per chunk
  const int rg = tid >> 6, cg = tid & 63;
  float pre[PER];
  auto load = [&](int i0) {
    if constexpr (TRANS) {
      if constexpr ((I & 3) == 0) {
#pragma unroll
        for (int m = 0; m < PER / 4; ++m) {
          const int f = tid + m * THREADS, j = f >> 2, c4 = f & 3;
          const float4 v = *reinterpret_cast<const float4*>(W + (size_t)j * I + i0 + 4 * c4);
          pre[4 * m] = v.x; pre[4 * m + 1] = v.y; pre[4 * m + 2] = v.z; pre[4 * m + 3] = v.w;
        }
      }                           // a row length that is not a multiple of 4 (layer 1) is staged straight from global memory
    } else {
#pragma unroll
      for (int m = 0; m < PER / 4; ++m) {
        const int f = tid + m * THREADS, kk = f >> 7, c = (f & 127) * 4;
        const float4 v = i0 + kk < I ? *reinterpret_cast<const float4*>(W + (size_t)(i0 + kk) * H + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        pre[4 * m] = v.x; pre[4 * m + 1] = v.y; pre[4 * m + 2] = v.z; pre[4 * m + 3] = v.w;
      }
    }
  };
  auto store = [&](int i0) {
    if constexpr (TRANS) {
      if constexpr ((I & 3) == 0) {
#pragma unroll
        for (int m = 0; m < PER / 4; ++m) {
          const int f = tid + m * THREADS, j = f >> 2, c4 = f & 3;
#pragma unroll
          for (int e = 0; e < 4; ++e) s.ms[4 * c4 + e][j] = pre[4 * m + e];
        }
      } else {
        for (int f = tid; f < KC * H; f += THREADS) {
          const int j = f / KC, kk = f % KC;
          s.ms[kk][j] = i0 + kk < I ? W[(size_t)j * I + i0 + kk] : 0.f;
        }
      }
    } else {
#pragma unroll
      for (int m = 0; m < PER / 4; ++m) {
        const int f = tid + m * THREADS, kk = f >> 7, c = (f & 127) * 4;
        *reinterpret_cast<float4*>(&s.ms[kk][c]) = make_float4(pre[4 * m], pre[4 * m + 1], pre[4 * m + 2], pre[4 * m + 3]);
      }
    }
  };
  load(0);
  for (int i0 = 0; i0 < I; i0 += KC) {
    __syncthreads();              // the previous chunk has been read (and, on entry, `in` has been written)
    store(i0);
    __syncthreads();
    if (i0 + KC < I) load(i0 + KC);
    const int n = min(KC, I - i0);
    for (int kk = 0; kk < n; ++kk) {
      const float4 av = *reinterpret_cast<const float4*>(&in[i0 + kk][rg * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&s.ms[kk][cg * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&s.ms[kk][256 + cg * 4]);
      const float a[4] = {av.x, av.y, av.z, av.w};
      const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[r][c] = fmaf(a[r], bb[c], acc[r][c]);
    }
  }
  __syncthreads();                // every thread is done reading `in` and s.ms
}

__device__ __forceinline__ int unit_of(int cg, int c) { return cg * 4 + (c & 3) + 256 * (c >> 2); }

// Sign bit of unit j = unit_of(cg, c) in row (rg*4 + r): word ((c >> 2) * 2 + warp half) * 4 + (c & 3) of the layer, bit = lane.
__device__ __forceinline__ int sign_word(int layer, int c, int cg) { return layer * (H / 32) + ((c >> 2) * 2 + (cg >> 5)) * 4 + (c & 3); }

__device__ void store_signs(unsigned* __restrict__ signs, int layer, const float (&v)[4][8], int row0, int n, int tid) {
  const int rg = tid >> 6, cg = tid & 63, lane = tid & 31;
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const unsigned bits = __ballot_sync(0xffffffffu, v[r][c] > 0.f);
      const int row = row0 + rg * 4 + r;
      if (lane == ((r * 8 + c) & 31) && row < n) signs[(size_t)row * SIGN_WORDS + sign_word(layer, c, cg)] = bits;
    }
}

__device__ __forceinline__ float slope_of(const unsigned* __restrict__ srow, int layer, int c, int cg, int lane) {
  return (srow[sign_word(layer, c, cg)] >> lane) & 1u ? 1.f : SLOPE;
}

__device__ void init_bias(float (&acc)[4][8], const float* __restrict__ bias, int cg) {
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const float bv = bias ? bias[unit_of(cg, c)] : 0.f;
#pragma unroll
    for (int r = 0; r < 4; ++r) acc[r][c] = bv;
  }
}

__device__ void write_tile(float (*out)[TR], const float (&v)[4][8], int tid) {
  const int rg = tid >> 6, cg = tid & 63;
#pragma unroll
  for (int c = 0; c < 8; ++c)
    *reinterpret_cast<float4*>(&out[unit_of(cg, c)][rg * 4]) = make_float4(v[0][c], v[1][c], v[2][c], v[3][c]);
}

__global__ void __launch_bounds__(THREADS, 2)
nature_disc_fwd_kernel(Params P, const float* __restrict__ pa, long long lda, const float* __restrict__ pb, long long ldb, int B, int n,
                       float* __restrict__ probs, unsigned* __restrict__ signs) {
  pdl_sync();
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem& s = *reinterpret_cast<Smem*>(smem_raw);
  const int tid = threadIdx.x, row0 = blockIdx.x * TR, rg = tid >> 6, cg = tid & 63;
  if (tid < TR * NJ) {
    const int r = tid / NJ, jt = tid % NJ, row = row0 + r;
    float e[3] = {0.f, 0.f, 0.f};
    if (row < n) {
      const float* q = row_pose(pa, lda, pb, ldb, B, row) + jt * 4;
      float two_s;
      const Rot5 R = quat_rot(q[0], q[1], q[2], q[3], two_s);
      e[0] = atan2f(-R.r12, R.r22); e[1] = asinf(R.r02); e[2] = atan2f(-R.r01, R.r00);
    }
    for (int c = 0; c < 3; ++c) s.x[jt * 3 + c][r] = e[c];
  }
  float acc[4][8];
  // d1 = lrelu(L1 x) -> a
  init_bias(acc, P.b[0], cg);
  matmul<true, NF>(s, P.w[0], s.x, acc, tid);
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[r][c] = lrelu(acc[r][c]);
  if (signs) store_signs(signs, 0, acc, row0, n, tid);
  write_tile(s.a, acc, tid);
  // d2 = lrelu(L2 d1) -> b
  init_bias(acc, P.b[1], cg);
  matmul<true, H>(s, P.w[1], s.a, acc, tid);
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[r][c] = lrelu(acc[r][c]);
  if (signs) store_signs(signs, 1, acc, row0, n, tid);
  write_tile(s.b, acc, tid);
  // d3 = lrelu(L3 d2 + d1) -> a, in place: each thread reads and writes only its own d1 entries
  init_bias(acc, P.b[2], cg);
  matmul<true, H>(s, P.w[2], s.b, acc, tid);
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[r][c] = lrelu(acc[r][c] + s.a[unit_of(cg, c)][rg * 4 + r]);
  if (signs) store_signs(signs, 2, acc, row0, n, tid);
  write_tile(s.a, acc, tid);
  // d4 = L4 d3 -> b
  init_bias(acc, P.b[3], cg);
  matmul<true, H>(s, P.w[3], s.a, acc, tid);
  write_tile(s.b, acc, tid);
  // d5 = lrelu(L_last d4) -> a
  init_bias(acc, P.b[4], cg);
  matmul<true, H>(s, P.w[4], s.b, acc, tid);
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[r][c] = lrelu(acc[r][c]);
  if (signs) store_signs(signs, 3, acc, row0, n, tid);
  write_tile(s.a, acc, tid);
  __syncthreads();
  // logits = L_pred d5: one warp per (row, class), lanes over units, a fixed butterfly; then softmax over the two classes
  const int warp = tid >> 5, lane = tid & 31;
  for (int o = warp; o < TR * 2; o += NWARPS) {
    const int r = o >> 1, cls = o & 1;
    float v = 0.f;
    for (int u = lane; u < H; u += 32) v = fmaf(P.w[5][cls * H + u], s.a[u][r], v);
    v = warp_sum(v);
    if (lane == 0) s.gl[r][cls] = v + P.b[5][cls];
  }
  __syncthreads();
  if (tid < TR && row0 + tid < n) {
    const float l0 = s.gl[tid][0], l1 = s.gl[tid][1], m = fmaxf(l0, l1);
    const float e0 = expf(l0 - m), e1 = expf(l1 - m), den = e0 + e1;
    probs[(size_t)(row0 + tid) * 2] = e0 / den;
    probs[(size_t)(row0 + tid) * 2 + 1] = e1 / den;
  }
}

// The input-gradient chain of the discriminator for one tile of rows, from d(probs) to d(pose).
__global__ void __launch_bounds__(THREADS, 2)
nature_disc_bwd_kernel(Params P, const float* __restrict__ pa, long long lda, const float* __restrict__ pb, long long ldb, int B, int n,
                       const float* __restrict__ probs, const unsigned* __restrict__ signs, const float* __restrict__ g_probs,
                       float* __restrict__ da, float* __restrict__ db) {
  pdl_sync();
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem& s = *reinterpret_cast<Smem*>(smem_raw);
  const int tid = threadIdx.x, row0 = blockIdx.x * TR, rg = tid >> 6, cg = tid & 63, lane = tid & 31;
  // softmax backward (torch: p * (g - sum g p)); a row with zero d(probs) takes no part and gets a zero gradient
  int live = 0;
  if (tid < TR) {
    const int row = row0 + tid;
    float g0 = 0.f, g1 = 0.f;
    if (row < n) {
      const float p0 = probs[(size_t)row * 2], p1 = probs[(size_t)row * 2 + 1];
      const float u0 = g_probs[(size_t)row * 2], u1 = g_probs[(size_t)row * 2 + 1];
      if (u0 != 0.f || u1 != 0.f) {
        const float dot = u0 * p0 + u1 * p1;
        g0 = p0 * (u0 - dot); g1 = p1 * (u1 - dot);
        live = 1;
      }
    }
    s.gl[tid][0] = g0; s.gl[tid][1] = g1; s.live[tid] = live;
  }
  if (!__syncthreads_or(live)) {
    // no row of the tile carries a gradient
    for (int o = tid; o < TR * NJ * 4; o += THREADS) {
      const int row = row0 + o / (NJ * 4);
      if (row < n) (row < B ? da + (size_t)row * NJ * 4 : db + (size_t)(row - B) * NJ * 4)[o % (NJ * 4)] = 0.f;
    }
    return;
  }
  const unsigned* srow[4];
  for (int r = 0; r < 4; ++r) srow[r] = signs + (size_t)min(row0 + rg * 4 + r, n - 1) * SIGN_WORDS;
  // g_z5 = (W_pred^T g_logits) * lrelu'(z5) -> a
  float acc[4][8];
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int u = unit_of(cg, c);
    const float w0 = P.w[5][u], w1 = P.w[5][H + u];
#pragma unroll
    for (int r = 0; r < 4; ++r)
      acc[r][c] = (s.gl[rg * 4 + r][0] * w0 + s.gl[rg * 4 + r][1] * w1) * slope_of(srow[r], 3, c, cg, lane);
  }
  write_tile(s.a, acc, tid);
  // g_z4 = g_d4 = L_last^T g_z5 -> b
  init_bias(acc, nullptr, cg);
  matmul<false, H>(s, P.w[4], s.a, acc, tid);
  write_tile(s.b, acc, tid);
  // g_z3 = (L4^T g_z4) * lrelu'(z3) -> a
  init_bias(acc, nullptr, cg);
  matmul<false, H>(s, P.w[3], s.b, acc, tid);
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[r][c] *= slope_of(srow[r], 2, c, cg, lane);
  write_tile(s.a, acc, tid);
  // g_z2 = (L3^T g_z3) * lrelu'(z2) -> b
  init_bias(acc, nullptr, cg);
  matmul<false, H>(s, P.w[2], s.a, acc, tid);
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[r][c] *= slope_of(srow[r], 1, c, cg, lane);
  write_tile(s.b, acc, tid);
  // g_z1 = (L2^T g_z2 + g_z3) * lrelu'(z1) -> a, in place (the residual d3 = lrelu(L3 d2 + d1))
  init_bias(acc, nullptr, cg);
  matmul<false, H>(s, P.w[1], s.b, acc, tid);
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[r][c] = (acc[r][c] + s.a[unit_of(cg, c)][rg * 4 + r]) * slope_of(srow[r], 0, c, cg, lane);
  write_tile(s.a, acc, tid);
  __syncthreads();
  // g_x = L1^T g_z1: [TR, 45], a fixed-order dot over the 512 units
  for (int o = tid; o < TR * NF; o += THREADS) {
    const int r = o / NF, f = o % NF;
    float v = 0.f;
    for (int u = 0; u < H; ++u) v = fmaf(s.a[u][r], P.w[0][u * NF + f], v);
    s.x[f][r] = v;
  }
  __syncthreads();
  // the XYZ angles and quaternion_to_matrix backward (torch's atan2 / asin derivatives) -> d(pose)
  if (tid < TR * NJ) {
    const int r = tid / NJ, jt = tid % NJ, row = row0 + r;
    if (row < n) {
      float* out = (row < B ? da + (size_t)row * NJ * 4 : db + (size_t)(row - B) * NJ * 4) + jt * 4;
      if (!s.live[r]) {
        out[0] = out[1] = out[2] = out[3] = 0.f;
      } else {
        const float* q = row_pose(pa, lda, pb, ldb, B, row) + jt * 4;
        const float qr = q[0], qi = q[1], qj = q[2], qk = q[3];
        float ts;
        const Rot5 R = quat_rot(qr, qi, qj, qk, ts);
        const float g0 = s.x[jt * 3][r], g1 = s.x[jt * 3 + 1][r], g2 = s.x[jt * 3 + 2][r];
        // e0 = atan2(y, x), y = -R12, x = R22: de/dy = x / (x^2 + y^2), de/dx = -y / (x^2 + y^2)
        float r2 = R.r22 * R.r22 + R.r12 * R.r12;
        const float g12 = -(g0 * R.r22 / r2), g22 = g0 * R.r12 / r2;
        const float g02 = g1 / sqrtf(1.f - R.r02 * R.r02);       // asin' = (1 - x^2)^-1/2
        r2 = R.r00 * R.r00 + R.r01 * R.r01;
        const float g01 = -(g2 * R.r00 / r2), g00 = g2 * R.r01 / r2;
        // R00 = 1 - s (j^2 + k^2), R01 = s (i j - k r), R02 = s (i k + j r), R12 = s (j k - i r), R22 = 1 - s (i^2 + j^2)
        const float gs = -g00 * (qj * qj + qk * qk) + g01 * (qi * qj - qk * qr) + g02 * (qi * qk + qj * qr) + g12 * (qj * qk - qi * qr) -
                         g22 * (qi * qi + qj * qj);
        float d[4];
        d[0] = ts * (-g01 * qk + g02 * qj - g12 * qi);
        d[1] = ts * (g01 * qj + g02 * qk - g12 * qr - 2.f * g22 * qi);
        d[2] = ts * (-2.f * g00 * qj + g01 * qi + g02 * qr + g12 * qk - 2.f * g22 * qj);
        d[3] = ts * (-2.f * g00 * qk - g01 * qr + g02 * qi + g12 * qj);
        // s = 2 / |q|^2: ds/dq = -s q / (|q|^2 / 2) = -s^2 q
        const float gn = -gs * ts * ts;
        out[0] = d[0] + gn * qr; out[1] = d[1] + gn * qi; out[2] = d[2] + gn * qj; out[3] = d[3] + gn * qk;
      }
    }
  }
}

// Per hand h (rows h B .. h B + B - 1 of probs): mask = p1 < 1.5 p0, the BCE sum over masked rows of
// -max(log1p(-p0), -100) - max(log(p1), -100) and the mask count; then loss = sum_h (n_h > 0 ? S_h / (2 n_h) : 0).
__global__ void __launch_bounds__(THREADS)
nature_loss_fwd_kernel(const float* __restrict__ probs, int B, float* __restrict__ loss, int* __restrict__ count) {
  pdl_sync();
  __shared__ float s_red[NWARPS];
  __shared__ int s_cnt[NWARPS];
  const int tid = threadIdx.x;
  float total = 0.f;
  for (int h = 0; h < 2; ++h) {
    float acc = 0.f;
    int cnt = 0;
    for (int b = tid; b < B; b += THREADS) {
      const float p0 = probs[((size_t)h * B + b) * 2], p1 = probs[((size_t)h * B + b) * 2 + 1];
      if (p1 < 1.5f * p0) {
        acc += -fmaxf(log1pf(-p0), -100.f) - fmaxf(logf(p1), -100.f);
        ++cnt;
      }
    }
    acc = warp_sum(acc);
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    __syncthreads();
    if ((tid & 31) == 0) { s_red[tid >> 5] = acc; s_cnt[tid >> 5] = cnt; }
    __syncthreads();
    float S = 0.f;
    int N = 0;
    for (int w = 0; w < NWARPS; ++w) { S += s_red[w]; N += s_cnt[w]; }
    if (N > 0) total += S / (float)(2 * N);      // the reference skips an empty hand on the host (:123, :127); decided here
    if (tid == 0) count[h] = N;
  }
  if (tid == 0) *loss = total;
}

// torch's binary_cross_entropy backward (g (p - y) / max(p (1 - p), 1e-12) / (2 n)) for the masked rows, zero elsewhere.
__global__ void nature_loss_bwd_kernel(const float* __restrict__ probs, const int* __restrict__ count, int B, const float* __restrict__ g_loss,
                                       float* __restrict__ g_probs) {
  pdl_sync();
  const float g = *g_loss;
  for (int row = blockIdx.x * blockDim.x + threadIdx.x; row < 2 * B; row += gridDim.x * blockDim.x) {
    const int N = count[row >= B];
    const float p0 = probs[(size_t)row * 2], p1 = probs[(size_t)row * 2 + 1];
    float g0 = 0.f, g1 = 0.f;
    if (N > 0 && p1 < 1.5f * p0) {
      const float numel = (float)(2 * N);
      g0 = g * p0 / fmaxf(p0 * (1.f - p0), 1e-12f) / numel;
      g1 = g * (p1 - 1.f) / fmaxf(p1 * (1.f - p1), 1e-12f) / numel;
    }
    g_probs[(size_t)row * 2] = g0;
    g_probs[(size_t)row * 2 + 1] = g1;
  }
}

int params_of(const void* const* p, Params& P, const char* who) {
  RIH_REQUIRE(p, "%s: NULL parameter array", who);
  for (int i = 0; i < 6; ++i) {
    P.w[i] = (const float*)p[2 * i];
    P.b[i] = (const float*)p[2 * i + 1];
    RIH_REQUIRE(P.w[i] && P.b[i], "%s: parameter %d is NULL", who, 2 * i);
    RIH_REQUIRE(((uintptr_t)P.w[i] & 15) == 0, "%s: weight %d is not 16-byte aligned", who, i);
  }
  return 0;
}

int check_rows(const float* pa, long long lda, const float* pb, long long ldb, int B, const char* who) {
  RIH_REQUIRE((pa || B == 0) && B >= 0 && lda >= NJ * 4, "%s: bad pose argument (B=%d lda=%lld)", who, B, lda);
  RIH_REQUIRE(!pb || ldb >= NJ * 4, "%s: bad second pose stride %lld", who, ldb);
  return 0;
}

template <class K>
int set_smem(K kernel) {
  RIH_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem)));
  return 0;
}

}  // namespace

// Pos2dDiscriminator.forward (Ver2Code/Discriminator/discrim.py:89-105, utlize.py:41-69,208-289) for 15 joints and 512 hidden units on
// n = B rows of pose_a, then B rows of pose_b when it is not NULL (both hands in one launch).  pose_*: [B,15,4] quaternions (real part
// first) with joint stride 4, component stride 1 and a row stride of ld_* floats, so a [:, 1:] view of [B,16,4] is read in place.
// params: 12 device pointers, weight then bias of pose_layer_1..4, layer_last, layer_pred.  -> probs [n,2]; signs [n,64] (may be
// NULL): the sign bits of the four activated hidden layers, read by rih_nature_disc_bwd.
RIH_API int rih_nature_disc_fwd(const void* const* params, const float* pose_a, long long ld_a, const float* pose_b, long long ld_b, int B,
                                float* probs, unsigned* signs, cudaStream_t s) {
  Params P;
  if (int e = params_of(params, P, "nature_disc_fwd")) return e;
  if (int e = check_rows(pose_a, ld_a, pose_b, ld_b, B, "nature_disc_fwd")) return e;
  const int n = pose_b ? 2 * B : B;
  if (n == 0) return 0;
  RIH_REQUIRE(probs, "nature_disc_fwd: NULL probs");
  if (int e = set_smem(nature_disc_fwd_kernel)) return e;
  launch_k(nature_disc_fwd_kernel, cdiv(n, TR), THREADS, sizeof(Smem), s, P, pose_a, ld_a, pose_b, ld_b, B, n, probs, signs);
  return check_launch("nature_disc_fwd");
}

// Backward of rih_nature_disc_fwd with respect to the poses: g_probs [n,2] -> d_pose_a, d_pose_b [B,15,4] contiguous (d_pose_b
// with pose_b).  probs and signs are the forward's.  Rows whose d(probs) is zero are skipped and get a zero gradient.
RIH_API int rih_nature_disc_bwd(const void* const* params, const float* pose_a, long long ld_a, const float* pose_b, long long ld_b, int B,
                                const float* probs, const unsigned* signs, const float* g_probs, float* d_pose_a, float* d_pose_b,
                                cudaStream_t s) {
  Params P;
  if (int e = params_of(params, P, "nature_disc_bwd")) return e;
  if (int e = check_rows(pose_a, ld_a, pose_b, ld_b, B, "nature_disc_bwd")) return e;
  const int n = pose_b ? 2 * B : B;
  if (n == 0) return 0;
  RIH_REQUIRE(probs && signs && g_probs && d_pose_a && (!pose_b || d_pose_b), "nature_disc_bwd: NULL argument");
  if (int e = set_smem(nature_disc_bwd_kernel)) return e;
  launch_k(nature_disc_bwd_kernel, cdiv(n, TR), THREADS, sizeof(Smem), s, P, pose_a, ld_a, pose_b, ld_b, B, n, probs, signs, g_probs,
           d_pose_a, d_pose_b);
  return check_launch("nature_disc_bwd");
}

// GeOptimizer.NatureLoss (geo_optimizer_both_batch.py:110-132) on the discriminator's output for both hands, probs [2B,2] (right
// rows first): one CTA, fixed order.  -> loss [1] (0-dim), count [2] int32: each hand's mask count.  The empty-mask rule is decided on
// the device.
RIH_API int rih_nature_loss_fwd(const float* probs, int B, float* loss, int* count, cudaStream_t s) {
  RIH_REQUIRE(probs && loss && count && B >= 1, "nature_loss_fwd: bad arguments (B=%d)", B);
  launch_k(nature_loss_fwd_kernel, 1, THREADS, 0, s, probs, B, loss, count);
  return check_launch("nature_loss_fwd");
}

// Backward of rih_nature_loss_fwd: g_loss [1] read on the device, count the forward's -> g_probs [2B,2].
RIH_API int rih_nature_loss_bwd(const float* probs, const int* count, int B, const float* g_loss, float* g_probs, cudaStream_t s) {
  RIH_REQUIRE(probs && count && g_loss && g_probs && B >= 1, "nature_loss_bwd: bad arguments (B=%d)", B);
  launch_k(nature_loss_bwd_kernel, cdiv(2LL * B, 256), 256, 0, s, probs, count, B, g_loss, g_probs);
  return check_launch("nature_loss_bwd");
}
