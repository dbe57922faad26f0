// The joint-limit validity judge of the pose data pipeline (pose_data_optimize/Ver2Code/ValidJudge/ValidJudger.py:41-123) for both hands
// of every frame in one launch, one thread per frame.
//
// Per hand and joint t = 0..14 (MANO joint t + 1): R is quaternion_to_rotation_matrix of the quaternion as given -- no normalisation
// first, the left hand's y and z negated (HandPoseConverter.mano_quat_2_mat_tensor, :214-231) -- and M = zero_ja^T ja = P R C with the
// host-folded converter matrices (geo_loss.py _conv_table).  The splank angle atan2(-M20, M00) and the bend angle atan2(M10, M00), in
// degrees, are checked against the reference's ranges; the score is max(max splank excess, max bend excess) in radians.  Steps 1 and 2
// of ValidationJudge are computed and discarded by the reference and are not computed here.
#include "common.cuh"
#include "hand_pose.cuh"
using namespace rih;

namespace {

constexpr int VJ_THREADS = 128;
constexpr float PI_F = 3.14159265358979323846f;
// ComputeValidation's threshold 0.1 / 180 * pi, a Python float rounded to float32 where it meets the float32 scores
constexpr float VJ_THRESH = (float)(0.1 / 180 * 3.141592653589793);

__device__ __forceinline__ float nan_max(float a, float b) { return (a != a || a > b) ? a : b; }      // torch.max: NaN propagates
__device__ __forceinline__ float relu(float a) { return a != a ? a : (a > 0.f ? a : 0.f); }

// relu(a - hi), relu(lo - a), their max, / 180 * pi
__device__ __forceinline__ float excess(float a, float lo, float hi) {
  return __fmul_rn(__fdiv_rn(nan_max(relu(__fsub_rn(a, hi)), relu(__fsub_rn(lo, a))), 180.f), PI_F);
}

// ValidationJudge for one hand: q [16,4] (joint 0 unused), conv [15,18] = P then C per joint.
__device__ float judge(const float* __restrict__ q, const float* __restrict__ conv, bool left) {
  float s_spl = 0.f, s_bend = 0.f;
  for (int t = 0; t < 15; ++t) {
    const float4 p = reinterpret_cast<const float4*>(q)[t + 1];
    const float sg = left ? -1.f : 1.f;
    float R[9], T[9], M[9];
    quat_to_R(p.x, p.y, sg * p.z, sg * p.w, R);
    mat3_mul(conv + t * 18, R, T);
    mat3_mul(T, conv + t * 18 + 9, M);
    if (t % 3 == 0) {
      const float sa = __fdiv_rn(__fmul_rn(atan2f(-M[6], M[0]), 180.f), PI_F);
      s_spl = nan_max(s_spl, excess(sa, c_spl_lo[t], c_spl_hi[t]));
    }
    const float ba = __fdiv_rn(__fmul_rn(atan2f(M[3], M[0]), 180.f), PI_F);
    s_bend = nan_max(excess(ba, c_bend_lo[t], c_bend_hi[t]), s_bend);
  }
  return nan_max(s_spl, s_bend);
}

__global__ void __launch_bounds__(VJ_THREADS) valid_judge_kernel(const float* __restrict__ q_left, const float* __restrict__ q_right,
                                                                 const float* __restrict__ conv, int B, float* __restrict__ score,
                                                                 long long* __restrict__ invalid) {
  pdl_sync();
  const int b = blockIdx.x * VJ_THREADS + threadIdx.x;
  int bad = 0;
  if (b < B) {
    const float l = judge(q_left + (size_t)b * 64, conv, true);
    const float r = judge(q_right + (size_t)b * 64, conv + 15 * 18, false);
    score[b] = l;
    score[B + b] = r;
    bad = __fadd_rn((float)(r > VJ_THRESH), l) > VJ_THRESH;           // ((right_res > th) + left_res > th) > 0
  }
  bad = __syncthreads_count(bad);
  if (threadIdx.x == 0 && bad) atomicAdd(reinterpret_cast<unsigned long long*>(invalid), (unsigned long long)bad);
}

}  // namespace

// ValidJudger.ComputeValidation (ValidJudger.py:113-123) for B frames.  q_left / q_right [B,16,4] float32 MANO quaternions; conv [2,15,18]
// float32 per hand (left, then right) and joint 1..15: P = zero_ja^T invM_U_n_0^T (row-major 3x3), then C = invU_M_n_1^T.  Writes
// score [2,B] (left row, then right row; radians) and invalid [1] = the number of frames where either hand is over the limit.
RIH_API int rih_valid_judge(const float* q_left, const float* q_right, const float* conv, int B, float* score, long long* invalid,
                            cudaStream_t s) {
  RIH_REQUIRE(q_left && q_right && conv && score && invalid, "valid_judge: NULL argument");
  RIH_REQUIRE(B >= 1, "valid_judge: B >= 1 (got %d)", B);
  RIH_CUDA(cudaMemsetAsync(invalid, 0, sizeof(long long), s));
  launch_k(valid_judge_kernel, cdiv(B, VJ_THREADS), VJ_THREADS, 0, s, q_left, q_right, conv, B, score, invalid);
  return check_launch("valid_judge");
}
