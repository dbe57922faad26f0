// The two-hand pose optimiser's step on the device (GeOptimizer.set_opt_val / loss_fn / optimize,
// pose_data_optimize/hocontact/postprocess/geo_optimizer_both_batch.py:133-930): the pose assembly of loss_fn (:480-485, :501-513) forward
// and backward, torch.optim.Adam over the optimised variables with every group's lr and the step count read from device memory, and
// ReduceLROnPlateau's step on the device-resident total loss.  Nothing here synchronises with the host or allocates, so a whole optimiser
// iteration replays from one CUDA graph while the scheduler changes the learning rates.  No float atomics: results are bitwise reproducible.
//
// The optimised variables live in ONE flat fp32 buffer in the reference's param-group order (:414-423):
//   [ hand_tsl B*3 | obj_tsl B*3 | right-hand variable joints B*n_r*4 | left-hand variable joints B*n_l*4 ].
#include "common.cuh"
#include "adam.cuh"
using namespace rih;

namespace {

// joint_src [2][16]: for hand h and joint j, k >= 0 -> row k of that hand's variable joints, k < 0 -> row -k-1 of its gt joints.
__global__ void ge_assemble_fwd_kernel(const float* __restrict__ flat, const float* __restrict__ gt_r, const float* __restrict__ gt_l,
                                       const int* __restrict__ joint_src, int B, int n_r, int n_l, float* __restrict__ pose_r,
                                       float* __restrict__ pose_l, float* __restrict__ tsl_r, float* __restrict__ tsl_l) {
  pdl_sync();
  const long long nt = 3LL * B, np = 64LL * B;
  const long long total = 2 * np + 2 * nt;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    if (i < 2 * np) {
      const int h = i >= np;
      const long long e = i - h * np;
      const int b = (int)(e >> 6), j = (int)(e >> 2) & 15, c = (int)e & 3;
      const int n_var = h ? n_l : n_r;
      const int k = joint_src[h * 16 + j];
      float val;
      if (k >= 0) {
        const long long off = 2 * nt + (h ? 4LL * B * n_r : 0);
        val = flat[off + ((long long)b * n_var + k) * 4 + c];
      } else {
        const float* gt = h ? gt_l : gt_r;
        val = gt[((long long)b * (16 - n_var) + (-k - 1)) * 4 + c];
      }
      (h ? pose_l : pose_r)[e] = val;
    } else {
      const long long e = i - 2 * np;                 // [0, 2 nt): hand_tsl then obj_tsl, as in the flat buffer
      if (e < nt) tsl_r[e] = flat[e];
      else tsl_l[e - nt] = flat[e];
    }
  }
}

// var_joint [2][16]: the joint index of each hand's variable row k (k < n_var).  Every element of d_flat is written exactly once.
__global__ void ge_assemble_bwd_kernel(const float* __restrict__ d_pose_r, const float* __restrict__ d_pose_l, const float* __restrict__ d_tsl_r,
                                       const float* __restrict__ d_tsl_l, const int* __restrict__ var_joint, int B, int n_r, int n_l,
                                       float* __restrict__ d_flat) {
  pdl_sync();
  const long long nt = 3LL * B, nr = 4LL * B * n_r, nl = 4LL * B * n_l;
  const long long total = 2 * nt + nr + nl;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    float val;
    if (i < nt) {
      val = d_tsl_r ? d_tsl_r[i] : 0.f;
    } else if (i < 2 * nt) {
      val = d_tsl_l ? d_tsl_l[i - nt] : 0.f;
    } else {
      const int h = i >= 2 * nt + nr;
      const long long e = i - 2 * nt - (h ? nr : 0);
      const int n_var = h ? n_l : n_r;
      const long long row = e >> 2;
      const int c = (int)e & 3, b = (int)(row / n_var), k = (int)(row - (long long)b * n_var);
      const float* d = h ? d_pose_l : d_pose_r;
      val = d ? d[((long long)b * 16 + var_joint[h * 16 + k]) * 4 + c] : 0.f;
    }
    d_flat[i] = val;
  }
}

constexpr int GE_MAX_GROUPS = 4;
struct SegEnds { long long e[GE_MAX_GROUPS]; };

// torch.optim.Adam (betas, eps, no weight decay, no amsgrad) at step t = *step + 1 with group g's lr = lr[g] over [seg.e[g-1], seg.e[g]),
// n = seg.e[ngroups-1].
// torch forms bias_correction1 = 1 - beta1 ** t, step_size = lr / bias_correction1 and sqrt(1 - beta2 ** t) as Python doubles; the powers
// come from a host-built table (CUDA's double pow is not correctly rounded), the subtraction, division and square root are IEEE double
// here as there, then rounded to float once.  A step beyond the table leaves the parameters and moments untouched.
__global__ void ge_adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, SegEnds seg,
                               long long n, int ngroups, const double* __restrict__ lr, const int* __restrict__ step, const double* __restrict__ b1pow,
                               const double* __restrict__ b2pow, int n_pow, float b1, float omb1, float b2, float omb2, float eps) {
  pdl_sync();
  const int t = *step + 1;
  if (t > n_pow) return;
  const double bc1 = __dsub_rn(1.0, b1pow[t]);
  const float bc2_sqrt = (float)__dsqrt_rn(__dsub_rn(1.0, b2pow[t]));
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;        // scalars, not an array: a dynamically indexed array would live in local memory
  s0 = (float)__ddiv_rn(lr[0], bc1);
  if (ngroups > 1) s1 = (float)__ddiv_rn(lr[1], bc1);
  if (ngroups > 2) s2 = (float)__ddiv_rn(lr[2], bc1);
  if (ngroups > 3) s3 = (float)__ddiv_rn(lr[3], bc1);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float step_size = (ngroups > 1 && i >= seg.e[0]) ? ((ngroups > 2 && i >= seg.e[1]) ? ((ngroups > 3 && i >= seg.e[2]) ? s3 : s2) : s1) : s0;
    float pi = p[i], mi = m[i], vi = v[i];
    adam_update(pi, mi, vi, g[i], 1.f, b1, omb1, b2, omb2, eps, step_size, bc2_sqrt);
    p[i] = pi; m[i] = mi; v[i] = vi;
  }
}

__global__ void ge_step_count_kernel(int* step) {
  pdl_sync();
  *step += 1;
}

// torch.optim.lr_scheduler.ReduceLROnPlateau(mode='min', threshold_mode='rel', cooldown=0).step(loss), one thread.  Every comparison and
// product is an explicitly rounded double operation, so no contraction changes a decision.
__global__ void ge_plateau_kernel(const float* __restrict__ loss, double* __restrict__ lr, int ngroups, double* __restrict__ best,
                                  int* __restrict__ num_bad, float* __restrict__ hist, double* __restrict__ lr_hist, int* __restrict__ it, int n_hist,
                                  double factor,
                                  int patience, double min_lr, double threshold, double eps) {
  pdl_sync();
  const float l = *loss;
  const int k = *it;
  if (k < n_hist) hist[k] = l;
  *it = k + 1;
  const double a = (double)l;                                  // float(metrics)
  if (a < __dmul_rn(*best, __dsub_rn(1.0, threshold))) {       // _is_better: a < best * (1 - threshold); false for NaN
    *best = a;
    *num_bad = 0;
  } else {
    *num_bad += 1;
  }
  if (*num_bad > patience) {                                   // _reduce_lr
    for (int gi = 0; gi < ngroups; ++gi) {
      const double old_lr = lr[gi];
      const double new_lr = fmax(__dmul_rn(old_lr, factor), min_lr);
      if (__dsub_rn(old_lr, new_lr) > eps) lr[gi] = new_lr;
    }
    *num_bad = 0;
  }
  if (lr_hist && k < n_hist)
    for (int gi = 0; gi < ngroups; ++gi) lr_hist[(long long)k * ngroups + gi] = lr[gi];
}

}  // namespace

// GeOptimizer.assemble_batch_pose_vec (geo_optimizer_both_batch.py:480-485) for both hands in one launch, as loss_fn calls it (:501-513),
// plus the translation views (:531-534).  flat: the optimised variables [hand_tsl B*3 | obj_tsl B*3 | right var B*n_r*4 | left var B*n_l*4];
// gt_r / gt_l: the gt joints [B,16-n_*,4]; joint_src [2][16] (device): k >= 0 selects variable row k, k < 0 gt row -k-1.  Any partition of
// the 16 joints works.  Writes pose_r / pose_l [B,16,4] and tsl_r / tsl_l [B,3].
RIH_API int rih_ge_assemble_fwd(const float* flat, const float* gt_r, const float* gt_l, const int* joint_src, int B, int n_r, int n_l, float* pose_r,
                                float* pose_l, float* tsl_r, float* tsl_l, cudaStream_t s) {
  RIH_REQUIRE(B >= 1 && n_r >= 0 && n_r <= 16 && n_l >= 0 && n_l <= 16, "ge_assemble_fwd: B >= 1 and 0 <= n_r, n_l <= 16 (got B=%d n_r=%d n_l=%d)",
              B, n_r, n_l);
  const long long total = 134LL * B;
  launch_k(ge_assemble_fwd_kernel, (int)min(ew_ctas(s), (total + 255) / 256), 256, 0, s, flat, gt_r, gt_l, joint_src, B, n_r, n_l, pose_r, pose_l,
           tsl_r, tsl_l);
  return check_launch("ge_assemble_fwd");
}

// The backward of rih_ge_assemble_fwd: d_flat (every element written) from d_pose_r / d_pose_l [B,16,4] and d_tsl_r / d_tsl_l [B,3]; the gt rows'
// gradient is dropped, a NULL upstream gradient counts as zero.  var_joint [2][16] (device): the joint of each hand's variable row.
RIH_API int rih_ge_assemble_bwd(const float* d_pose_r, const float* d_pose_l, const float* d_tsl_r, const float* d_tsl_l, const int* var_joint, int B,
                                int n_r, int n_l, float* d_flat, cudaStream_t s) {
  RIH_REQUIRE(B >= 1 && n_r >= 0 && n_r <= 16 && n_l >= 0 && n_l <= 16, "ge_assemble_bwd: B >= 1 and 0 <= n_r, n_l <= 16 (got B=%d n_r=%d n_l=%d)",
              B, n_r, n_l);
  const long long total = 6LL * B + 4LL * B * (n_r + n_l);
  launch_k(ge_assemble_bwd_kernel, (int)min(ew_ctas(s), (total + 255) / 256), 256, 0, s, d_pose_r, d_pose_l, d_tsl_r, d_tsl_l, var_joint, B, n_r,
           n_l, d_flat);
  return check_launch("ge_assemble_bwd");
}

// torch.optim.Adam.step (geo_optimizer_both_batch.py:428, :879; betas, eps, weight_decay 0, amsgrad False) over the flat buffer p with its
// gradient g and moments m, v.  Group k covers [seg_end[k-1], seg_end[k]) of the first ngroups (<= 4) ends and uses lr[k] (double, device);
// *step (device) counts the steps taken and is incremented after the update.  b1pow / b2pow [n_pow + 1] (device, double) hold beta ** t for
// t = 0..n_pow.  The element update is rih_adamw_step's (adam.cuh).
RIH_API int rih_ge_adam_step(float* p, const float* g, float* m, float* v, long long seg_end0, long long seg_end1, long long seg_end2,
                             long long seg_end3, int ngroups, const double* lr, int* step, const double* b1pow, const double* b2pow, int n_pow,
                             double beta1, double beta2, double eps, cudaStream_t s) {
  RIH_REQUIRE(ngroups >= 1 && ngroups <= GE_MAX_GROUPS, "ge_adam_step: 1 <= ngroups <= %d (got %d)", GE_MAX_GROUPS, ngroups);
  SegEnds seg = {{seg_end0, seg_end1, seg_end2, seg_end3}};
  for (int k = 0; k < ngroups; ++k)
    RIH_REQUIRE(seg.e[k] >= (k ? seg.e[k - 1] : 0), "ge_adam_step: segment ends must be non-decreasing and >= 0");
  RIH_REQUIRE(n_pow >= 1, "ge_adam_step: the beta power table must cover t >= 1 (got n_pow=%d)", n_pow);
  const long long n = seg.e[ngroups - 1];
  if (n > 0) {
    launch_k(ge_adam_kernel, (int)min(ew_ctas(s), (n + 255) / 256), 256, 0, s, p, g, m, v, seg, n, ngroups, lr, (const int*)step, b1pow, b2pow, n_pow,
             (float)beta1, (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2), (float)eps);
    if (int e = check_launch("ge_adam")) return e;
  }
  launch_k(ge_step_count_kernel, 1, 1, 0, s, step);
  return check_launch("ge_adam_count");
}

// torch.optim.lr_scheduler.ReduceLROnPlateau(optimizer, mode='min', factor, patience, threshold, threshold_mode='rel', cooldown=0, min_lr, eps)
// .step(loss) (geo_optimizer_both_batch.py:430-432, :880) on the 0-dim fp32 loss, widened to double like float(metrics).  State in device
// memory: best (double, +inf initially), num_bad, and the ngroups learning rates (double).  When *it < n_hist it also stores the loss in
// hist[*it] and, when lr_hist is not NULL, the learning rates after the step in lr_hist[*it][ngroups]; then it increments *it.
RIH_API int rih_ge_plateau_step(const float* loss, double* lr, int ngroups, double* best, int* num_bad, float* hist, double* lr_hist, int* it, int n_hist,
                                double factor, int patience, double min_lr, double threshold, double eps, cudaStream_t s) {
  RIH_REQUIRE(ngroups >= 0 && patience >= 0 && n_hist >= 0, "ge_plateau_step: ngroups, patience and n_hist must be >= 0");
  launch_k(ge_plateau_kernel, 1, 1, 0, s, loss, lr, ngroups, best, num_bad, hist, lr_hist, it, n_hist, factor, patience, min_lr, threshold, eps);
  return check_launch("ge_plateau");
}
