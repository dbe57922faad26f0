// Fitting MANO to 3-D hand joints on the device (utils/mano_from_3djoint/convert2mano.py:133-245): the adaptive IK that initialises the
// fit (AIK.py:16-104, including the template scaling of convert2mano.py:166-168), the rotation-matrix -> axis-angle conversion the loop
// feeds the PCA pose with (utils.py:90-216) and its gradient, the L1 joint loss (:189-192) with its gradient, and the linear learning-rate
// decay (:199-200).  Batched over frames; nothing here synchronises with the host or allocates, so one optimiser iteration (with
// rih_mano_fwd / _bwd and rih_ge_adam_step) replays from one CUDA graph.  No atomics: every frame is computed on its own in a fixed order,
// so a frame's result does not depend on the batch it is fitted in.
#include <math.h>

#include "common.cuh"
using namespace rih;

namespace {

// ------------------------------------------------------------------------------------------------------------------ adaptive IK
struct M3 { double a[9]; };

__device__ __forceinline__ M3 mul(const M3& x, const M3& y) {
  M3 r;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) r.a[i * 3 + j] = x.a[i * 3] * y.a[j] + x.a[i * 3 + 1] * y.a[3 + j] + x.a[i * 3 + 2] * y.a[6 + j];
  return r;
}

__device__ __forceinline__ double det3(const M3& m) {
  const double* a = m.a;
  return a[0] * (a[4] * a[8] - a[5] * a[7]) - a[1] * (a[3] * a[8] - a[5] * a[6]) + a[2] * (a[3] * a[7] - a[4] * a[6]);
}

// np.linalg.inv: the adjugate over the determinant (a singular or NaN matrix gives inf / NaN, as numpy's result feeds NaN onward).
__device__ __forceinline__ M3 inv3(const M3& m) {
  const double* a = m.a;
  const double id = 1.0 / det3(m);
  M3 r;
  r.a[0] = (a[4] * a[8] - a[5] * a[7]) * id; r.a[1] = (a[2] * a[7] - a[1] * a[8]) * id; r.a[2] = (a[1] * a[5] - a[2] * a[4]) * id;
  r.a[3] = (a[5] * a[6] - a[3] * a[8]) * id; r.a[4] = (a[0] * a[8] - a[2] * a[6]) * id; r.a[5] = (a[2] * a[3] - a[0] * a[5]) * id;
  r.a[6] = (a[3] * a[7] - a[4] * a[6]) * id; r.a[7] = (a[1] * a[6] - a[0] * a[7]) * id; r.a[8] = (a[0] * a[4] - a[1] * a[3]) * id;
  return r;
}

// H = U diag(S) V^T with S descending, by one-sided (Hestenes) Jacobi: plane rotations applied to the columns of B = H V and of V until
// B's columns are orthogonal, so S[i] = |b_i| and u_i = b_i / S[i] keep their accuracy relative to S[0] however small S[1] or S[2] are
// (an eigen-decomposition of H^T H would square the condition number).  u3 = +-(u1 x u2): when the palm is flat, b3 is rounding error,
// so only its sign (the pairing H v3 = S[2] u3) is taken from it; with S[2] below the flip threshold either sign ends in the same
// proper rotation.  U is orthonormal in every case.  V U^T, all AIK uses, is unique when the singular values are distinct.
__device__ __forceinline__ void svd3(const M3& H, M3& U, double S[3], M3& V) {
  double Bm[9], W[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
#pragma unroll
  for (int i = 0; i < 9; ++i) Bm[i] = H.a[i];
  for (int sweep = 0; sweep < 12; ++sweep) {
#pragma unroll
    for (int pq = 0; pq < 3; ++pq) {
      const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
      const double a = Bm[p] * Bm[p] + Bm[3 + p] * Bm[3 + p] + Bm[6 + p] * Bm[6 + p];
      const double b = Bm[q] * Bm[q] + Bm[3 + q] * Bm[3 + q] + Bm[6 + q] * Bm[6 + q];
      const double g = Bm[p] * Bm[q] + Bm[3 + p] * Bm[3 + q] + Bm[6 + p] * Bm[6 + q];
      if (g == 0.0) continue;
      const double z = (b - a) / (2.0 * g);
      const double t = (z >= 0 ? 1.0 : -1.0) / (fabs(z) + hypot(z, 1.0));
      const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double bp = Bm[k * 3 + p], bq = Bm[k * 3 + q];
        Bm[k * 3 + p] = c * bp - s * bq;
        Bm[k * 3 + q] = s * bp + c * bq;
        const double wp = W[k * 3 + p], wq = W[k * 3 + q];
        W[k * 3 + p] = c * wp - s * wq;
        W[k * 3 + q] = s * wp + c * wq;
      }
    }
  }
  double n[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) n[c] = sqrt(Bm[c] * Bm[c] + Bm[3 + c] * Bm[3 + c] + Bm[6 + c] * Bm[6 + c]);
  int o0 = 0, o1 = 1, o2 = 2;                  // column order, descending norm (ties keep the lower index, as a stable sort)
  if (n[o0] < n[o1]) { int u = o0; o0 = o1; o1 = u; }
  if (n[o1] < n[o2]) { int u = o1; o1 = o2; o2 = u; }
  if (n[o0] < n[o1]) { int u = o0; o0 = o1; o1 = u; }
  const int ord[3] = {o0, o1, o2};
  double b3[3] = {0, 0, 0};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int k = ord[c];                      // selects, not an index: Bm and W stay in registers
    const double nk = k == 0 ? n[0] : k == 1 ? n[1] : n[2];
    S[c] = nk;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const double bv = k == 0 ? Bm[r * 3] : k == 1 ? Bm[r * 3 + 1] : Bm[r * 3 + 2];
      V.a[r * 3 + c] = k == 0 ? W[r * 3] : k == 1 ? W[r * 3 + 1] : W[r * 3 + 2];
      if (c < 2) U.a[r * 3 + c] = bv / nk;
      else b3[r] = bv;
    }
  }
  const double x0 = U.a[3] * U.a[7] - U.a[6] * U.a[4];
  const double x1 = U.a[6] * U.a[1] - U.a[0] * U.a[7];
  const double x2 = U.a[0] * U.a[4] - U.a[3] * U.a[1];
  const double sg = (b3[0] * x0 + b3[1] * x1 + b3[2] * x2) < 0.0 ? -1.0 : 1.0;
  U.a[2] = sg * x0; U.a[5] = sg * x1; U.a[8] = sg * x2;
}

// transforms3d.axangles.axangle2mat(axis, angle, is_normalized=False): a zero axis divides 0 / 0 (NaN), as in numpy.
__device__ __forceinline__ M3 axangle2mat(double x, double y, double z, double angle) {
  const double n = sqrt(x * x + y * y + z * z);
  x = x / n; y = y / n; z = z / n;
  const double c = cos(angle), s = sin(angle), C = 1.0 - c;
  const double xs = x * s, ys = y * s, zs = z * s, xC = x * C, yC = y * C, zC = z * C;
  const double xyC = x * yC, yzC = y * zC, zxC = z * xC;
  M3 r = {{x * xC + c, xyC - zs, zxC + ys, xyC + zs, y * yC + c, yzC - xs, zxC - ys, yzC + xs, z * zC + c}};
  return r;
}

// One thread per frame; see rih_mfit_aik.
__global__ void mfit_aik_kernel(const double* __restrict__ template_, int template_per_frame, double t_norm, int prescale,
                                const double* __restrict__ joints, int B, double* __restrict__ pose_R) {
  pdl_sync();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const double* J = joints + (long long)b * 63;
  const double* Tb = template_ + (template_per_frame ? (long long)b * 63 : 0);
  auto T = [&](int k, int c) { return Tb[k * 3 + c]; };
  // convert2mano.py:166-168: ratio, P = joints * ratio, P = P - P[0] + template[0]
  const double d0 = J[27] - J[0], d1 = J[28] - J[1], d2 = J[29] - J[2];
  const double ratio = t_norm / sqrt(d0 * d0 + d1 * d1 + d2 * d2);
  const double p00 = J[0] * ratio, p01 = J[1] * ratio, p02 = J[2] * ratio;
  auto P = [&](int k, int c) {
    return prescale ? (J[k * 3 + c] * ratio - (c == 0 ? p00 : c == 1 ? p01 : p02)) + T(0, c) : J[k * 3 + c];
  };

  // Kabsch root on the palm bones 1, 5, 9, 13, 17 (AIK.py:46-70): H = T0 P0^T, R0 = V U^T, the third column of V flipped only for a
  // reflection with a (near) zero singular value.
  M3 H = {{0, 0, 0, 0, 0, 0, 0, 0, 0}};
#pragma unroll
  for (int f = 0; f < 5; ++f) {
    const int k = 1 + 4 * f;
    double tv[3], pv[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) { tv[c] = T(k, c) - T(0, c); pv[c] = P(k, c) - P(0, c); }
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) H.a[i * 3 + j] += tv[i] * pv[j];
  }
  M3 U, V;
  double S[3];
  svd3(H, U, S, V);
  M3 Ut;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) Ut.a[i * 3 + j] = U.a[j * 3 + i];
  M3 R0 = mul(V, Ut);
  if (fabs(det3(R0) + 1.0) < 1e-6 && (fabs(S[0]) < 1e-4 || fabs(S[1]) < 1e-4 || fabs(S[2]) < 1e-4)) {
    V.a[2] = -V.a[2]; V.a[5] = -V.a[5]; V.a[8] = -V.a[8];
    R0 = mul(V, Ut);
  }
  double* out = pose_R + (long long)b * 144;
#pragma unroll
  for (int i = 0; i < 9; ++i) out[i] = R0.a[i];

  // swing rotations along each finger (AIK.py:81-97, config.kinematic_tree / SNAP_PARENT), scattered by ID2ROT (AIK.py:99-102)
  for (int f = 0; f < 5; ++f) {
    const int a = 1 + 4 * f;
    M3 Rpa = R0;                               // R[a] = R[0]
    double q[3];                               // q[a] = R[a] (T[a] - T[0]) + q[0], q[0] = T[0]
    {
      const double t0 = T(a, 0) - T(0, 0), t1 = T(a, 1) - T(0, 1), t2 = T(a, 2) - T(0, 2);
#pragma unroll
      for (int i = 0; i < 3; ++i) q[i] = (Rpa.a[i * 3] * t0 + Rpa.a[i * 3 + 1] * t1 + Rpa.a[i * 3 + 2] * t2) + T(0, i);
    }
    for (int s = 0; s < 3; ++s) {
      const int pa = a + s, k = pa + 1;
      if (s > 0) {                             // q[pa] = R[pa] (T[pa] - T[pa_pa]) + q[pa_pa]
        const double t0 = T(pa, 0) - T(pa - 1, 0), t1 = T(pa, 1) - T(pa - 1, 1), t2 = T(pa, 2) - T(pa - 1, 2);
        double nq[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) nq[i] = (Rpa.a[i * 3] * t0 + Rpa.a[i * 3 + 1] * t1 + Rpa.a[i * 3 + 2] * t2) + q[i];
        q[0] = nq[0]; q[1] = nq[1]; q[2] = nq[2];
      }
      const M3 Ri = inv3(Rpa);
      const double e0 = P(k, 0) - q[0], e1 = P(k, 1) - q[1], e2 = P(k, 2) - q[2];
      double dp[3], dt[3];
#pragma unroll
      for (int i = 0; i < 3; ++i) { dp[i] = Ri.a[i * 3] * e0 + Ri.a[i * 3 + 1] * e1 + Ri.a[i * 3 + 2] * e2; dt[i] = T(k, i) - T(pa, i); }
      const double cx = dt[1] * dp[2] - dt[2] * dp[1], cy = dt[2] * dp[0] - dt[0] * dp[2], cz = dt[0] * dp[1] - dt[1] * dp[0];
      const double cn = sqrt(cx * cx + cy * cy + cz * cz) + 1e-8;
      const double temp = (sqrt(dt[0] * dt[0] + dt[1] * dt[1] + dt[2] * dt[2]) + 1e-8) * (sqrt(dp[0] * dp[0] + dp[1] * dp[1] + dp[2] * dp[2]) + 1e-8);
      const double alpha = acos((dt[0] * dp[0] + dt[1] * dp[1] + dt[2] * dp[2]) / temp);
      M3 Rk = axangle2mat(cx / cn, cy / cn, cz / cn, alpha);
      // the zero twist: axangle2mat(delta_t, 0) is exactly I unless delta_t is zero (then NaN)
      if (!(dt[0] * dt[0] + dt[1] * dt[1] + dt[2] * dt[2] > 0.0))
#pragma unroll
        for (int i = 0; i < 9; ++i) Rk.a[i] = nan("");
      const int slot = f == 0 ? 13 : f == 1 ? 1 : f == 2 ? 4 : f == 3 ? 10 : 7;     // ID2ROT of joint a + 1
      double* o = out + (slot + s) * 9;
#pragma unroll
      for (int i = 0; i < 9; ++i) o[i] = Rk.a[i];
      Rpa = mul(Rpa, Rk);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------ mat2aa
// utils.py:123-216 on m = R^T in fp32 with torch's operation order; the sums are explicitly rounded so no contraction changes them.
struct AaFwd {
  float m[9];     // R^T
  int br;         // selected branch 0..3
  float t, r;     // t of the branch, r = sqrt(t)
  float qr[4];    // the branch's raw quaternion
  float q[4];     // normalised: (qr / r) * 0.5
  float sin2, sinh, two;
  float aa[3];    // before the NaN -> 0 rule
};

__device__ __forceinline__ void aa_forward(const float* R, AaFwd& f) {
  float* m = f.m;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) m[i * 3 + j] = R[j * 3 + i];
  const bool d2 = m[8] < 1e-6f, d0d1 = m[0] > m[4], d0nd1 = m[0] < -m[4];
  f.br = d2 ? (d0d1 ? 0 : 1) : (d0nd1 ? 2 : 3);
  const float s01 = __fadd_rn(m[1], m[3]), s02 = __fadd_rn(m[6], m[2]), s12 = __fadd_rn(m[5], m[7]);
  const float a12 = __fsub_rn(m[5], m[7]), a20 = __fsub_rn(m[6], m[2]), a01 = __fsub_rn(m[1], m[3]);
  switch (f.br) {
    case 0: f.t = __fsub_rn(__fsub_rn(__fadd_rn(1.f, m[0]), m[4]), m[8]); f.qr[0] = a12; f.qr[1] = f.t; f.qr[2] = s01; f.qr[3] = s02; break;
    case 1: f.t = __fsub_rn(__fadd_rn(__fsub_rn(1.f, m[0]), m[4]), m[8]); f.qr[0] = a20; f.qr[1] = s01; f.qr[2] = f.t; f.qr[3] = s12; break;
    case 2: f.t = __fadd_rn(__fsub_rn(__fsub_rn(1.f, m[0]), m[4]), m[8]); f.qr[0] = a01; f.qr[1] = s02; f.qr[2] = s12; f.qr[3] = f.t; break;
    default: f.t = __fadd_rn(__fadd_rn(__fadd_rn(1.f, m[0]), m[4]), m[8]); f.qr[0] = f.t; f.qr[1] = a12; f.qr[2] = a20; f.qr[3] = a01; break;
  }
  f.r = sqrtf(f.t);
#pragma unroll
  for (int i = 0; i < 4; ++i) f.q[i] = __fmul_rn(__fdiv_rn(f.qr[i], f.r), 0.5f);
  f.sin2 = __fadd_rn(__fadd_rn(__fmul_rn(f.q[1], f.q[1]), __fmul_rn(f.q[2], f.q[2])), __fmul_rn(f.q[3], f.q[3]));
  f.sinh = sqrtf(f.sin2);
  const float c = f.q[0];
  f.two = __fmul_rn(2.f, c < 0.f ? atan2f(-f.sinh, -c) : atan2f(f.sinh, c));
  const float k = f.sin2 > 0.f ? __fdiv_rn(f.two, f.sinh) : 2.f;
#pragma unroll
  for (int i = 0; i < 3; ++i) f.aa[i] = __fmul_rn(f.q[i + 1], k);
}

__global__ void mfit_aa_fwd_kernel(const float* __restrict__ R, long long N, float* __restrict__ aa) {
  pdl_sync();
  for (long long n = blockIdx.x * (long long)blockDim.x + threadIdx.x; n < N; n += (long long)gridDim.x * blockDim.x) {
    AaFwd f;
    aa_forward(R + n * 9, f);
#pragma unroll
    for (int i = 0; i < 3; ++i) aa[n * 3 + i] = isnan(f.aa[i]) ? 0.f : f.aa[i];
  }
}

// The autograd backward of that formulation through the selected branch: each step is torch's derivative formula for the operation
// (div: g / y and -g x / y^2, sqrt: g / (2 sqrt), atan2: g x / (x^2 + y^2), -g y / (x^2 + y^2)), so 0 / 0 at an exactly zero rotation
// gives the reference's NaN.  The NaN -> 0 assignment zeroes the gradient of the entries it replaced.
__global__ void mfit_aa_bwd_kernel(const float* __restrict__ R, const float* __restrict__ g_aa, long long N, float* __restrict__ dR) {
  pdl_sync();
  for (long long n = blockIdx.x * (long long)blockDim.x + threadIdx.x; n < N; n += (long long)gridDim.x * blockDim.x) {
    AaFwd f;
    aa_forward(R + n * 9, f);
    float g[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) g[i] = isnan(f.aa[i]) ? 0.f : g_aa[n * 3 + i];
    // aa_i = q_{i+1} * k
    const float k = f.sin2 > 0.f ? __fdiv_rn(f.two, f.sinh) : 2.f;
    float dq[4] = {0.f, 0.f, 0.f, 0.f};
    float dk = 0.f;
#pragma unroll
    for (int i = 0; i < 3; ++i) { dq[i + 1] = __fmul_rn(g[i], k); dk = __fadd_rn(dk, __fmul_rn(g[i], f.q[i + 1])); }
    // k = where(sin2 > 0, two / sinh, 2)
    const float dkp = f.sin2 > 0.f ? dk : 0.f;
    const float d_two = __fdiv_rn(dkp, f.sinh);
    float d_sinh = -__fdiv_rn(__fmul_rn(dkp, f.two), __fmul_rn(f.sinh, f.sinh));
    // two = 2 * atan2(+-sinh, +-c)
    const float dw = __fmul_rn(d_two, 2.f);
    const float c = f.q[0];
    const float den = __fadd_rn(__fmul_rn(f.sinh, f.sinh), __fmul_rn(c, c));
    float d_c;
    if (c < 0.f) {                             // atan2(-sinh, -c)
      d_sinh = __fadd_rn(d_sinh, -__fdiv_rn(__fmul_rn(dw, -c), den));
      d_c = -__fdiv_rn(__fmul_rn(dw, f.sinh), den);
    } else {
      d_sinh = __fadd_rn(d_sinh, __fdiv_rn(__fmul_rn(dw, c), den));
      d_c = __fdiv_rn(__fmul_rn(dw, -f.sinh), den);
    }
    dq[0] = __fadd_rn(dq[0], d_c);
    // sinh = sqrt(sin2), sin2 = sum q_i^2
    const float d_sin2 = __fdiv_rn(d_sinh, __fmul_rn(2.f, f.sinh));
#pragma unroll
    for (int i = 1; i < 4; ++i) dq[i] = __fadd_rn(dq[i], __fmul_rn(__fmul_rn(d_sin2, 2.f), f.q[i]));
    // q = (qr / r) * 0.5, r = sqrt(t): one divisor per component, summed into d t
    float dqr[4], dr = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float gd = __fmul_rn(dq[i], 0.5f);
      dqr[i] = __fdiv_rn(gd, f.r);
      dr = __fadd_rn(dr, -__fmul_rn(gd, __fdiv_rn(__fdiv_rn(f.qr[i], f.r), f.r)));
    }
    float dt = __fdiv_rn(dr, __fmul_rn(2.f, f.r));
    float dm[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    // the branch's quaternion components and t (m index: 0 = 00, 1 = 01, 2 = 02, 3 = 10, 4 = 11, 5 = 12, 6 = 20, 7 = 21, 8 = 22)
    float ga12 = 0.f, ga20 = 0.f, ga01 = 0.f, gs01 = 0.f, gs02 = 0.f, gs12 = 0.f;
    switch (f.br) {
      case 0: ga12 = dqr[0]; dt = __fadd_rn(dt, dqr[1]); gs01 = dqr[2]; gs02 = dqr[3];
              dm[0] += dt; dm[4] -= dt; dm[8] -= dt; break;
      case 1: ga20 = dqr[0]; gs01 = dqr[1]; dt = __fadd_rn(dt, dqr[2]); gs12 = dqr[3];
              dm[0] -= dt; dm[4] += dt; dm[8] -= dt; break;
      case 2: ga01 = dqr[0]; gs02 = dqr[1]; gs12 = dqr[2]; dt = __fadd_rn(dt, dqr[3]);
              dm[0] -= dt; dm[4] -= dt; dm[8] += dt; break;
      default: dt = __fadd_rn(dt, dqr[0]); ga12 = dqr[1]; ga20 = dqr[2]; ga01 = dqr[3];
              dm[0] += dt; dm[4] += dt; dm[8] += dt; break;
    }
    dm[5] += ga12 + gs12; dm[7] += gs12 - ga12;
    dm[6] += ga20 + gs02; dm[2] += gs02 - ga20;
    dm[1] += ga01 + gs01; dm[3] += gs01 - ga01;
    float* o = dR + n * 9;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) o[i * 3 + j] = dm[j * 3 + i];
  }
}

// ------------------------------------------------------------------------------------------------------------------ loss
// One warp per frame, lane i < 21 holds joint i.  d_i = (j_i - j_0) - target_i; loss = sum |d| / 63, summed in a fixed order;
// g_i = sign(d_i) / 63 and joint 0 also receives - sum_i g_i (the - j[:, 0:1] term).
__global__ void mfit_joint_l1_kernel(const float* __restrict__ j, const float* __restrict__ target, int B, float* __restrict__ loss,
                                     float* __restrict__ g_j, float* __restrict__ hist, const int* __restrict__ step, int n_hist) {
  pdl_sync();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B) return;
  const float* jb = j + (long long)warp * 63;
  const float inv = __fdiv_rn(1.f, 63.f);
  float a = 0.f, g[3] = {0.f, 0.f, 0.f};
  if (lane < 21) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float d = __fsub_rn(__fsub_rn(jb[lane * 3 + c], jb[c]), target[(long long)warp * 63 + lane * 3 + c]);
      a = __fadd_rn(a, fabsf(d));
      g[c] = d > 0.f ? inv : (d < 0.f ? -inv : (d == 0.f ? 0.f : d));    // torch.sign: NaN stays NaN
    }
  }
  float s0 = g[0], s1 = g[1], s2 = g[2];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    s0 += __shfl_xor_sync(0xffffffffu, s0, o);
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
  }
  if (lane < 21) {
    float* gb = g_j + (long long)warp * 63 + lane * 3;
    if (lane == 0) { gb[0] = g[0] - s0; gb[1] = g[1] - s1; gb[2] = g[2] - s2; }
    else { gb[0] = g[0]; gb[1] = g[1]; gb[2] = g[2]; }
  }
  if (lane == 0) {
    const float l = __fdiv_rn(a, 63.f);
    if (loss) loss[warp] = l;
    if (hist && step) {
      const int k = *step;
      if (k < n_hist) hist[(long long)k * B + warp] = l;
    }
  }
}

// lr = lr0 * (n - i) / n for the step i just taken (*step counts the steps taken, so i = *step - 1), in Python's double order.
__global__ void mfit_lr_kernel(double* lr, const int* step, double lr0, int n) {
  pdl_sync();
  const int i = *step - 1;
  lr[0] = __ddiv_rn(__dmul_rn(lr0, (double)(n - i)), (double)n);
}

}  // namespace

// adaptive_IK (utils/mano_from_3djoint/AIK.py:16-104) for B frames in float64, optionally after convert2mano.py's template scaling
// (:164-168).  template_ (device, float64): [21,3] shared by every frame, or [B,21,3] with template_per_frame != 0 (convert2mano.py
// passes the layer's float32 joints at pose_R = I); joints [B,21,3] (device, float64).  prescale == 0: joints are AIK's P as given.
// prescale != 0: joints are the targets in the CSV's units, and P = joints * ratio shifted so that P[0] = template[0], with
// ratio = t_norm / |joints[9] - joints[0]| and t_norm = np.linalg.norm(template[9] - template[0]) as the reference forms it from the
// float32 template (a float32 norm).  Writes pose_R [B,16,3,3] (float64): the Kabsch root
// (V[:, 2] negated only when |det + 1| < 1e-6 and some singular value < 1e-4, :59-66) and the 15 swing rotations along the fingers in
// MANO order (config.py:84-126).  A bone exactly parallel to its template bone gives NaN, as axangle2mat's 0 / 0 does in the reference.
RIH_API int rih_mfit_aik(const double* template_, int template_per_frame, double t_norm, int prescale, const double* joints, int B,
                         double* pose_R, cudaStream_t s) {
  RIH_REQUIRE(B >= 0, "mfit_aik: negative batch");
  if (B == 0) return 0;
  launch_k(mfit_aik_kernel, cdiv(B, 64), 64, 0, s, template_, template_per_frame, t_norm, prescale, joints, B, pose_R);
  return check_launch("mfit_aik");
}

// mat2aa (utils/mano_from_3djoint/utils.py:198-216 -> mat2quat :123-184 -> quat2aa :90-121) on R [N,3,3] fp32: the branch chosen by
// R^T[2,2] < 1e-6, R^T[0,0] > R^T[1,1] and R^T[0,0] < -R^T[1,1], atan2 on the half angle, k = 2 when sin^2 = 0, NaN -> 0.  aa [N,3].
RIH_API int rih_mfit_rotmat_to_aa_fwd(const float* R, long long N, float* aa, cudaStream_t s) {
  RIH_REQUIRE(N >= 0, "mfit_rotmat_to_aa_fwd: negative count");
  if (N == 0) return 0;
  launch_k(mfit_aa_fwd_kernel, (int)min(ew_ctas(s), (N + 127) / 128), 128, 0, s, R, N, aa);
  return check_launch("mfit_rotmat_to_aa_fwd");
}

// The autograd gradient of rih_mfit_rotmat_to_aa_fwd (utils.py:90-216 differentiated as torch does, convert2mano.py:194): dR [N,3,3] from
// g_aa [N,3], through the selected branch.  NaN at an exactly zero rotation (the 0 / 0 of two_theta / sin_theta and of sqrt's backward),
// as in the reference; entries the forward set from NaN to 0 pass no gradient.
RIH_API int rih_mfit_rotmat_to_aa_bwd(const float* R, const float* g_aa, long long N, float* dR, cudaStream_t s) {
  RIH_REQUIRE(N >= 0, "mfit_rotmat_to_aa_bwd: negative count");
  if (N == 0) return 0;
  launch_k(mfit_aa_bwd_kernel, (int)min(ew_ctas(s), (N + 127) / 128), 128, 0, s, R, g_aa, N, dR);
  return check_launch("mfit_rotmat_to_aa_bwd");
}

// The joint loss of convert2mano.py:187-192 per frame and its gradient: loss[b] = mean |(j - j[:, 0:1]) - target| over 63 values, target =
// (joints - joints[0:1]) / 100 as float32; g_j [B,21,3] the gradient of sum_b loss[b] (joint 0 gets minus the sum of the others' terms).
// loss may be NULL; when hist and step are not NULL and *step < n_hist, loss[b] is also stored in hist[*step][b].
RIH_API int rih_mfit_joint_l1(const float* j, const float* target, int B, float* loss, float* g_j, float* hist, const int* step, int n_hist,
                              cudaStream_t s) {
  RIH_REQUIRE(B >= 0 && n_hist >= 0, "mfit_joint_l1: negative batch or history length");
  if (B == 0) return 0;
  launch_k(mfit_joint_l1_kernel, cdiv(B, 4), 128, 0, s, j, target, B, loss, g_j, hist, step, n_hist);
  return check_launch("mfit_joint_l1");
}

// The learning-rate decay of convert2mano.py:199-200 after the step counted in *step (device, incremented by rih_ge_adam_step):
// lr[0] = lr0 * (n - i) / n with i = *step - 1, formed as Python forms it (double multiply, then divide).
RIH_API int rih_mfit_lr_step(double* lr, const int* step, double lr0, int n, cudaStream_t s) {
  RIH_REQUIRE(n >= 1, "mfit_lr_step: n must be >= 1 (got %d)", n);
  launch_k(mfit_lr_kernel, 1, 1, 0, s, lr, step, lr0, n);
  return check_launch("mfit_lr_step");
}
