// Quaternion -> joint-matrix pieces and joint-angle limits shared by the ergonomics prior (geo_loss.cu), the joint-limit validity judge
// (valid_judge.cu) and the quaternion hand model (manopth.cu): HandPoseConverter.mano_quat_2_mat_tensor's rotation (quatutils.py:168-221),
// its backward, and the 3x3 products around it.
#pragma once

namespace rih {

// Joint-angle limits in degrees per joint index t = 0..14 (MANO joint t + 1), identical in hand_pose_ergonomics_loss (geo_loss.py:399-414)
// and ValidationJudge (ValidJudger.py:80-108).  Splank limits apply where t % 3 == 0 (the finger and thumb bases).
static __constant__ float c_bend_lo[15] = {-25, -4, -8, -25, -7, -8, -22, -8, -8, -25, -10, -8, -20, -35, -10};
static __constant__ float c_bend_hi[15] = {70, 110, 90, 80, 100, 90, 70, 90, 90, 70, 100, 90, 40, 50, 100};
static __constant__ float c_spl_lo[15] = {-25, 0, 0, -15, 0, 0, -20, 0, 0, -25, 0, 0, -30, 0, 0};
static __constant__ float c_spl_hi[15] = {15, 0, 0, 15, 0, 0, 30, 0, 0, 15, 0, 0, 30, 0, 0};

// quatutils.py:191-216: entries of the rotation matrix over |q|^2
__device__ __forceinline__ void quat_to_R(float w, float x, float y, float z, float* R) {
  const float ww = w * w, wx = w * x, wy = w * y, wz = w * z, xx = x * x, xy = x * y, xz = x * z, yy = y * y, yz = y * z, zz = z * z;
  const float n = ww + xx + yy + zz;
  R[0] = (ww + xx - yy - zz) / n; R[1] = 2.f * (xy - wz) / n;       R[2] = 2.f * (wy + xz) / n;
  R[3] = 2.f * (wz + xy) / n;     R[4] = (ww - xx + yy - zz) / n;   R[5] = 2.f * (yz - wx) / n;
  R[6] = 2.f * (xz - wy) / n;     R[7] = 2.f * (wx + yz) / n;       R[8] = (ww - xx - yy + zz) / n;
}

// R = M(p) / n = quat_to_R(p) with n = |p|^2, gradient g on R  ->  dL/dp:  sum_ab g_ab (dM_ab/dp) / n - 2 p (sum_ab g_ab R_ab) / n
__device__ inline void quat_R_backward(const float* p, const float* R, const float* g, float* d) {
  const float w = p[0], x = p[1], y = p[2], z = p[3];
  const float n = w * w + x * x + y * y + z * z;
  float gRR = 0.f;
  for (int e = 0; e < 9; ++e) gRR += g[e] * R[e];
  const float dw = 2.f * (w * (g[0] + g[4] + g[8]) + z * (g[3] - g[1]) + y * (g[2] - g[6]) + x * (g[7] - g[5]));
  const float dx = 2.f * (x * (g[0] - g[4] - g[8]) + y * (g[1] + g[3]) + z * (g[2] + g[6]) + w * (g[7] - g[5]));
  const float dy = 2.f * (y * (-g[0] + g[4] - g[8]) + x * (g[1] + g[3]) + z * (g[5] + g[7]) + w * (g[2] - g[6]));
  const float dz = 2.f * (z * (-g[0] - g[4] + g[8]) + x * (g[2] + g[6]) + y * (g[5] + g[7]) + w * (g[3] - g[1]));
  d[0] = (dw - 2.f * w * gRR) / n; d[1] = (dx - 2.f * x * gRR) / n; d[2] = (dy - 2.f * y * gRR) / n; d[3] = (dz - 2.f * z * gRR) / n;
}

__device__ __forceinline__ void mat3_mul(const float* A, const float* B, float* C) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) C[r * 3 + c] = A[r * 3] * B[c] + A[r * 3 + 1] * B[3 + c] + A[r * 3 + 2] * B[6 + c];
}

}  // namespace rih
