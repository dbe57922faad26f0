// The pose data pipeline's conversion and augmentation stages (pose_data_optimize/scripts/HandPoseConverter.py, HandPoseArguer.py,
// Ver2Code/NatureJudge/PoseArgue.py): euler <-> MANO quaternion <-> axis-angle per pose and joint, and the bend / splank augmentation of
// every (frame, copy) in one launch.
//
// The rotation arithmetic is a float64 statement of the scipy.spatial.transform.Rotation operations those scripts call (scipy 1.18,
// _rotation_xp.py, and the Cython backend numpy inputs take, whose results it equals):
//   from_euler('xyz', degrees=True)  extrinsic: q = qz (qy qx), elementary quaternions (sin(a/2) e_axis, cos(a/2)), a = deg * (pi/180);
//   as_matrix                         the x2 - y2 - z2 + w2 / 2(xy - zw) ... formula of the stored (unnormalised) quaternion;
//   from_matrix                       det <= 0 is an error in scipy and gives NaN here; a matrix whose Gramian fails
//                                     isclose(M M^T, I, rtol=1e-5, atol=1e-12) is replaced by its polar factor (scipy: U V^T of the SVD;
//                                     here Newton's X <- (X + X^-T) / 2, which reaches the same factor to float64 rounding); then the
//                                     quaternion branch chosen by the first maximum of (M00, M11, M22, trace), normalised;
//   as_euler('xyz', degrees=True)     _get_angles: the second angle 2 atan2(hypot(c,d), hypot(a,b)) decides the gimbal cases (within
//                                     1e-7 of 0 or pi: third angle 0), then pi/2 is subtracted and each angle wrapped into (-pi, pi];
//   from_rotvec / as_rotvec           their small-angle series below 1e-3 rad; as_rotvec canonicalises to w >= 0 first;
//   from_quat                         normalisation.
// No gimbal-lock warning is raised.
#include "common.cuh"
using namespace rih;

namespace {

constexpr int PD_THREADS = 128;
constexpr double PI = 3.141592653589793;

struct Quat { double x, y, z, w; };        // scipy's scalar-last order

__device__ __forceinline__ Quat compose(const Quat& p, const Quat& q) {
  const double cx = p.y * q.z - p.z * q.y, cy = p.z * q.x - p.x * q.z, cz = p.x * q.y - p.y * q.x;
  return {p.w * q.x + q.w * p.x + cx, p.w * q.y + q.w * p.y + cy, p.w * q.z + q.w * p.z + cz,
          p.w * q.w - p.x * q.x - p.y * q.y - p.z * q.z};
}

__device__ Quat from_euler_xyz(double ex, double ey, double ez) {
  const double k = PI / 180.0;
  double s, c;
  sincos(ex * k / 2.0, &s, &c);
  Quat q = {s, 0.0, 0.0, c};
  sincos(ey * k / 2.0, &s, &c);
  q = compose({0.0, s, 0.0, c}, q);
  sincos(ez * k / 2.0, &s, &c);
  return compose({0.0, 0.0, s, c}, q);
}

__device__ void as_matrix(const Quat& q, double* M) {
  const double x2 = q.x * q.x, y2 = q.y * q.y, z2 = q.z * q.z, w2 = q.w * q.w;
  const double xy = q.x * q.y, zw = q.z * q.w, xz = q.x * q.z, yw = q.y * q.w, yz = q.y * q.z, xw = q.x * q.w;
  M[0] = x2 - y2 - z2 + w2;  M[1] = 2 * (xy - zw);       M[2] = 2 * (xz + yw);
  M[3] = 2 * (xy + zw);      M[4] = -x2 + y2 - z2 + w2;  M[5] = 2 * (yz - xw);
  M[6] = 2 * (xz - yw);      M[7] = 2 * (yz + xw);       M[8] = -x2 - y2 + z2 + w2;
}

__device__ __forceinline__ void mat3_mul(const double* A, const double* B, double* C) {
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) C[r * 3 + c] = A[r * 3] * B[c] + A[r * 3 + 1] * B[3 + c] + A[r * 3 + 2] * B[6 + c];
}

// transpose of the inverse: the cofactor matrix over the determinant
__device__ __forceinline__ double cofactors(const double* M, double* K) {
  K[0] = M[4] * M[8] - M[5] * M[7]; K[1] = M[5] * M[6] - M[3] * M[8]; K[2] = M[3] * M[7] - M[4] * M[6];
  K[3] = M[2] * M[7] - M[1] * M[8]; K[4] = M[0] * M[8] - M[2] * M[6]; K[5] = M[1] * M[6] - M[0] * M[7];
  K[6] = M[1] * M[5] - M[2] * M[4]; K[7] = M[2] * M[3] - M[0] * M[5]; K[8] = M[0] * M[4] - M[1] * M[3];
  return M[0] * K[0] + M[1] * K[1] + M[2] * K[2];
}

__device__ Quat from_matrix(double* M) {
  double K[9];
  const double det = cofactors(M, K);
  if (!(det > 0.0)) {
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    return {nan, nan, nan, nan};
  }
  bool orthogonal = true;
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double g = M[r * 3] * M[c * 3] + M[r * 3 + 1] * M[c * 3 + 1] + M[r * 3 + 2] * M[c * 3 + 2];
      orthogonal &= fabs(g - (r == c ? 1.0 : 0.0)) <= 1e-12 + (r == c ? 1e-5 : 0.0);
    }
  if (!orthogonal) {
    // polar factor: quadratic convergence from the float32-level non-orthogonality of the converter products in two or three steps
    double d = det;
    for (int it = 0; it < 12; ++it) {
      double step = 0.0;
#pragma unroll
      for (int e = 0; e < 9; ++e) {
        const double x = 0.5 * (M[e] + K[e] / d);
        step = fmax(step, fabs(x - M[e]));
        M[e] = x;
      }
      if (step <= 1e-16) break;
      d = cofactors(M, K);
    }
  }
  const double tr = M[0] + M[4] + M[8];
  int choice = 0;
  double best = M[0];
  if (M[4] > best) { choice = 1; best = M[4]; }
  if (M[8] > best) { choice = 2; best = M[8]; }
  if (tr > best) choice = 3;
  double q[4];
  if (choice == 3) {
    q[0] = M[7] - M[5]; q[1] = M[2] - M[6]; q[2] = M[3] - M[1]; q[3] = 1 + tr;
  } else {
    const int i = choice, j = (i + 1) % 3, k = (j + 1) % 3;
    q[i] = 1 - tr + 2 * M[i * 4];
    q[j] = M[j * 3 + i] + M[i * 3 + j];
    q[k] = M[k * 3 + i] + M[i * 3 + k];
    q[3] = M[k * 3 + j] - M[j * 3 + k];
  }
  const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  return {q[0] / n, q[1] / n, q[2] / n, q[3] / n};
}

__device__ __forceinline__ double wrap_pi(double a) {
  if (a < -PI) return a + 2 * PI;
  if (a > PI) return a - 2 * PI;
  return a;
}

// as_euler('xyz', degrees=True): extrinsic, i, j, k = 0, 1, 2, sign +1, lambda = pi/2
__device__ void as_euler_xyz(const Quat& q, double* e) {
  const double a = q.w - q.y, b = q.x + q.z, c = q.y + q.w, d = q.z - q.x;
  double th1 = 2 * atan2(hypot(c, d), hypot(a, b));
  const bool case1 = fabs(th1) <= 1e-7, case2 = fabs(th1 - PI) <= 1e-7;
  const double half_sum = atan2(b, a), half_diff = atan2(d, c);
  double th0, th2;
  if (!case1 && !case2) {
    th0 = half_sum - half_diff;
    th2 = half_sum + half_diff;
  } else {
    th2 = 0.0;
    th0 = case1 ? 2 * half_sum : -2 * half_diff;
  }
  th1 -= PI / 2;
  const double k = 180.0 / PI;
  e[0] = wrap_pi(th0) * k;
  e[1] = wrap_pi(th1) * k;
  e[2] = wrap_pi(th2) * k;
}

__device__ Quat from_rotvec(double x, double y, double z) {
  const double angle = sqrt(x * x + y * y + z * z);
  const double a2 = angle * angle;
  const double scale = angle <= 1e-3 ? 0.5 - a2 / 48 + a2 * a2 / 3840 : sin(angle / 2) / angle;
  return {x * scale, y * scale, z * scale, cos(angle / 2)};
}

__device__ void as_rotvec(Quat q, double* v) {
  const bool flip = q.w < 0 || (q.w == 0 && (q.x < 0 || (q.x == 0 && (q.y < 0 || (q.y == 0 && q.z < 0)))));
  if (flip) q = {-q.x, -q.y, -q.z, -q.w};
  const double angle = 2 * atan2(sqrt(q.x * q.x + q.y * q.y + q.z * q.z), q.w);
  const double a2 = angle * angle;
  const double scale = angle <= 1e-3 ? 2 + a2 / 12 + 7 * a2 * a2 / 2880 : angle / sin(angle / 2);
  v[0] = scale * q.x; v[1] = scale * q.y; v[2] = scale * q.z;
}

__device__ __forceinline__ Quat from_quat(double x, double y, double z, double w) {
  const double n = sqrt(x * x + y * y + z * z + w * w);
  return {x / n, y / n, z / n, w / n};
}

// the converter's 3x3 pair of joint j: conv[j*18 .. +9) = invM_U_n_0, conv[j*18+9 .. +9) = invU_M_n_1, float32 row-major
__device__ __forceinline__ void load_conv(const float* __restrict__ conv, int j, bool transpose, double* A, double* C) {
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int s = transpose ? c * 3 + r : r * 3 + c;
      A[r * 3 + c] = (double)conv[j * 18 + s];
      C[r * 3 + c] = (double)conv[j * 18 + 9 + s];
    }
}

// MANO quaternion (w, x, y, z) float32, the left hand's y and z negated
__device__ __forceinline__ void store_mano_quat(float* __restrict__ out, const Quat& q, bool left) {
  const float s = left ? -1.f : 1.f;
  reinterpret_cast<float4*>(out)[0] = make_float4((float)q.w, (float)q.x, s * (float)q.y, s * (float)q.z);
}

enum Op { EULER_TO_QUAT = 0, QUAT_TO_EULER = 1, AA_TO_QUAT = 2, QUAT_TO_FLAT = 3 };

// one thread per (pose, joint); n = N * 16
template <int OP>
__global__ void __launch_bounds__(PD_THREADS) pose_convert_kernel(const void* __restrict__ in, long long n, int left, int flag,
                                                                  const float* __restrict__ conv, const float* __restrict__ hands_mean,
                                                                  void* __restrict__ out) {
  pdl_sync();
  const long long t = (long long)blockIdx.x * PD_THREADS + threadIdx.x;
  if (t >= n) return;
  const int j = (int)(t % 16);
  if (OP == EULER_TO_QUAT) {                       // HandPoseConverter.euler_2_mano_quat (:159-188)
    const double* e = static_cast<const double*>(in) + t * 3;
    double R[9], A[9], C[9], T[9], M[9];
    as_matrix(from_euler_xyz(e[0], e[1], e[2]), R);
    load_conv(conv, j, false, A, C);
    mat3_mul(A, R, T);
    mat3_mul(T, C, M);
    if (left && j == 0)
      for (int e2 = 3; e2 < 9; ++e2) M[e2] = -M[e2];
    store_mano_quat(static_cast<float*>(out) + t * 4, from_matrix(M), left);
  } else if (OP == QUAT_TO_EULER) {                // HandPoseConverter.mano_quat_2_euler (:190-212)
    const double* q = static_cast<const double*>(in) + t * 4;
    const double s = left ? -1.0 : 1.0;
    double R[9], A[9], C[9], T[9], M[9];
    as_matrix(from_quat(q[1], s * q[2], s * q[3], q[0]), R);
    if (left && j == 0)
      for (int e2 = 3; e2 < 9; ++e2) R[e2] = -R[e2];
    load_conv(conv, j, true, A, C);
    mat3_mul(A, R, T);
    mat3_mul(T, C, M);
    as_euler_xyz(from_matrix(M), static_cast<double*>(out) + t * 3);
  } else if (OP == AA_TO_QUAT) {                   // HandPoseConverter.axis_angle_2_mano_quat (:272-301); flag = flat_hand
    const float* a = static_cast<const float*>(in) + t * 3;
    float v[3] = {a[0], a[1], a[2]};
    if (!flag && j > 0)
      for (int c = 0; c < 3; ++c) v[c] = __fadd_rn(v[c], hands_mean[(j - 1) * 3 + c]);
    store_mano_quat(static_cast<float*>(out) + t * 4, from_rotvec(v[0], v[1], v[2]), left);
  } else {                                         // HandPoseConverter.mano_quat_flat_2_normal (:303-332); flag = return quaternions
    const float4 p = reinterpret_cast<const float4*>(in)[t];
    const double s = left ? -1.0 : 1.0;
    double v[3];
    as_rotvec(from_quat(p.y, s * p.z, s * p.w, p.x), v);
    if (j > 0)
      for (int c = 0; c < 3; ++c) v[c] -= (double)hands_mean[(j - 1) * 3 + c];
    if (flag)
      store_mano_quat(static_cast<float*>(out) + t * 4, from_rotvec((float)v[0], (float)v[1], (float)v[2]), left);
    else
      for (int c = 0; c < 3; ++c) static_cast<double*>(out)[t * 3 + c] = v[c];
  }
}

// ------------------------------------------------------------------------------------------------------------------------ augmentation
// The 20 draws of a frame copy, in the reference's order: bend_argue's 15 joints (soft, strict, thumb-normal, normal, root lists), then
// splank_argue's 5.  Per joint: its bend slot (every joint but the root) and its splank slot (the finger and thumb bases).
__constant__ signed char c_bend_slot[16] = {-1, 11, 0, 6, 12, 1, 7, 14, 3, 9, 13, 2, 8, 4, 5, 10};
__constant__ signed char c_splank_slot[16] = {-1, 15, -1, -1, 16, -1, -1, 18, -1, -1, 17, -1, -1, 19, -1, -1};

// Philox-4x32-10 (Salmon et al., SC'11) of counter (draw index, offset) and key seed -> a double in [0, 1) from 53 bits, as numpy forms
// its doubles from two 32-bit words
__device__ __forceinline__ double philox_uniform(unsigned long long draw, unsigned long long seed, unsigned long long offset) {
  unsigned int c0 = (unsigned int)draw, c1 = (unsigned int)(draw >> 32), c2 = (unsigned int)offset, c3 = (unsigned int)(offset >> 32);
  unsigned int k0 = (unsigned int)seed, k1 = (unsigned int)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const unsigned int hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const unsigned int hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return ((double)(c0 >> 5) * 67108864.0 + (double)(c1 >> 6)) * (1.0 / 9007199254740992.0);
}

// angle_random_adjust (HandPoseArguer.py:166-173): pos = max(min(M, hi - a), 0), neg = min(max(-M, lo - a), 0), (pos - neg) u + neg with
// the product and the sum rounded separately, as numpy evaluates them
__device__ __forceinline__ double adjustment(double angle, const double* __restrict__ ranges, int slot, double max_adj, long long draw,
                                             const double* __restrict__ u, unsigned long long seed, unsigned long long offset,
                                             double* __restrict__ adj) {
  const double pos = fmax(fmin(max_adj, ranges[slot * 2 + 1] - angle), 0.0);
  const double neg = fmin(fmax(-max_adj, ranges[slot * 2] - angle), 0.0);
  const double r = u ? u[draw] : philox_uniform((unsigned long long)draw, seed, offset);
  const double v = __dadd_rn(__dmul_rn(pos - neg, r), neg);
  if (adj) adj[draw] = v;
  return v;
}

// apply_adjustment (HandPoseArguer.py:82-96) for one joint: euler(R(e) R(d)) with d an elementary euler triple
__device__ void adjust(double* e, double dx, double dy, double dz) {
  double R[9], D[9], M[9];
  as_matrix(from_euler_xyz(e[0], e[1], e[2]), R);
  as_matrix(from_euler_xyz(dx, dy, dz), D);
  mat3_mul(R, D, M);
  as_euler_xyz(from_matrix(M), e);
}

// one thread per (frame i, copy a, joint j); output row i * A + a
__global__ void __launch_bounds__(PD_THREADS) pose_argue_kernel(const double* __restrict__ euler, long long n, int A,
                                                                const double* __restrict__ ranges, double max_bend, double max_splank,
                                                                const double* __restrict__ u, unsigned long long seed,
                                                                unsigned long long offset, double* __restrict__ out,
                                                                double* __restrict__ adj) {
  pdl_sync();
  const long long t = (long long)blockIdx.x * PD_THREADS + threadIdx.x;
  if (t >= n) return;
  const int j = (int)(t % 16);
  const long long row = t / 16, i = row / A, a = row % A;
  const double* src = euler + (i * 16 + j) * 3;
  double e[3] = {src[0], src[1], src[2]};
  const int kb = c_bend_slot[j], ks = c_splank_slot[j];
  const double bend = kb < 0 ? 0.0 : adjustment(e[2], ranges, kb, max_bend, (i * 20 + kb) * A + a, u, seed, offset, adj);
  const double splank = ks < 0 ? 0.0 : adjustment(e[1], ranges, ks, max_splank, (i * 20 + ks) * A + a, u, seed, offset, adj);
  // every joint takes both round trips, as in the reference, whether or not it was adjusted
  adjust(e, 0.0, 0.0, bend);
  adjust(e, 0.0, splank, 0.0);
  double* dst = out + t * 3;
  dst[0] = e[0]; dst[1] = e[1]; dst[2] = e[2];
}

template <int OP>
int launch_convert(const char* what, const void* in, long long N, int side, int flag, const float* conv, const float* hands_mean, void* out,
                   cudaStream_t s) {
  RIH_REQUIRE(in && out && conv, "%s: NULL argument", what);
  RIH_REQUIRE(!(OP == AA_TO_QUAT || OP == QUAT_TO_FLAT) || hands_mean, "%s: NULL hands_mean", what);
  RIH_REQUIRE(N >= 1, "%s: N >= 1 (got %lld)", what, N);
  RIH_REQUIRE(side == 0 || side == 1, "%s: side must be 0 (right) or 1 (left), got %d", what, side);
  const long long n = N * 16;
  launch_k(pose_convert_kernel<OP>, cdiv(n, PD_THREADS), PD_THREADS, 0, s, in, n, side, flag, conv, hands_mean, out);
  return check_launch(what);
}

}  // namespace

// HandPoseConverter.euler_2_mano_quat (pose_data_optimize/scripts/HandPoseConverter.py:159-188).  euler [N,16,3] float64 degrees ('xyz');
// conv [16,18] float32: invM_U_n_0 then invU_M_n_1 per joint, row-major; side 0 = right, 1 = left (root flip, y and z negated).
// Writes quat [N,16,4] float32 (w, x, y, z).
RIH_API int rih_pose_euler_to_mano_quat(const double* euler, long long N, int side, const float* conv, float* quat, cudaStream_t s) {
  return launch_convert<EULER_TO_QUAT>("pose_euler_to_mano_quat", euler, N, side, 0, conv, nullptr, quat, s);
}

// HandPoseConverter.mano_quat_2_euler (HandPoseConverter.py:190-212).  quat [N,16,4] float64 (w, x, y, z); conv as above.  Writes
// euler [N,16,3] float64 degrees.  The input is not modified.
RIH_API int rih_pose_mano_quat_to_euler(const double* quat, long long N, int side, const float* conv, double* euler, cudaStream_t s) {
  return launch_convert<QUAT_TO_EULER>("pose_mano_quat_to_euler", quat, N, side, 0, conv, nullptr, euler, s);
}

// HandPoseConverter.axis_angle_2_mano_quat (HandPoseConverter.py:272-301).  aa [N,16,3] float32 axis-angle; hands_mean [15,3] float32 is
// added to joints 1..15 unless flat_hand.  Writes quat [N,16,4] float32 (w, x, y, z).
RIH_API int rih_pose_axis_angle_to_mano_quat(const float* aa, long long N, int side, int flat_hand, const float* conv, const float* hands_mean,
                                             float* quat, cudaStream_t s) {
  return launch_convert<AA_TO_QUAT>("pose_axis_angle_to_mano_quat", aa, N, side, flat_hand ? 1 : 0, conv, hands_mean, quat, s);
}

// HandPoseConverter.mano_quat_flat_2_normal (HandPoseConverter.py:303-332).  quat [N,16,4] float32 (w, x, y, z); hands_mean [15,3] float32
// is subtracted from joints 1..15 of the axis-angle.  return_quat = 0: writes out [N,16,3] float64 axis-angle; 1: writes out [N,16,4]
// float32, that axis-angle through axis_angle_2_mano_quat(flat_hand=True).
RIH_API int rih_pose_mano_quat_flat_to_normal(const float* quat, long long N, int side, int return_quat, const float* conv,
                                              const float* hands_mean, void* out, cudaStream_t s) {
  return launch_convert<QUAT_TO_FLAT>("pose_mano_quat_flat_to_normal", quat, N, side, return_quat ? 1 : 0, conv, hands_mean, out, s);
}

// HandPoseArguer.argue_pose / PoseArguer.argue_pose (HandPoseArguer.py:33-173, Ver2Code/NatureJudge/PoseArgue.py:34-174) for all B * A
// augmented poses.  euler [B,16,3] float64 degrees; ranges [20,2] float64 (lo, hi) of the 20 draws of a copy in the reference's order
// (bend joints 2,5,11,8, 13, 14, 3,6,12,9,15, 1,4,10,7, then splank joints 1,4,10,7,13); max_bend / max_splank the adjustment maxima.
// Uniforms: u [B,20,A] float64 when u is not NULL, else Philox-4x32-10 keyed by seed at counter (draw index, offset), the draw index
// being the same [B,20,A] position.  Writes out [B*A,16,3] float64 (row i * A + a) and, when adj is not NULL, the applied adjustments
// in degrees [B,20,A].
RIH_API int rih_pose_argue(const double* euler, long long B, int A, const double* ranges, double max_bend, double max_splank, const double* u,
                           unsigned long long seed, unsigned long long offset, double* out, double* adj, cudaStream_t s) {
  RIH_REQUIRE(euler && ranges && out, "pose_argue: NULL argument");
  RIH_REQUIRE(B >= 1 && A >= 1, "pose_argue: B >= 1 and A >= 1 (got %lld, %d)", B, A);
  const long long n = B * A * 16;
  launch_k(pose_argue_kernel, cdiv(n, PD_THREADS), PD_THREADS, 0, s, euler, n, A, ranges, max_bend, max_splank, u, seed, offset, out, adj);
  return check_launch("pose_argue");
}
