// Quaternion -> joint-matrix pieces and joint-angle limits shared by the ergonomics prior (geo_loss.cu) and the joint-limit validity judge (valid_judge.cu):
// HandPoseConverter.mano_quat_2_mat_tensor's rotation (quatutils.py:168-221) and the 3x3 products around it.
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

__device__ __forceinline__ void mat3_mul(const float* A, const float* B, float* C) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) C[r * 3 + c] = A[r * 3] * B[c] + A[r * 3 + 1] * B[3 + c] + A[r * 3 + 2] * B[6 + c];
}

}  // namespace rih
