// MANO forward kinematics + linear blend skinning as ONE kernel (one CTA per hand).
// reference: ManoLayer.forward  models/manolayer.py:250-322 ; rodrigues_batch :32-48 ; pca2axis :163-166
// Stage plan inside the CTA (warp roles); S1-S4 are mano_core.cuh's:
//   S0  all warps : betas, root matrix, PCA->axis-angle (45 dots) or the 15 rotation matrices
//   S1  all warps : shape blend v_shaped = T + S*beta (2334 outputs, coalesced [10][2334] table)
//   S2  warp 0    : Rodrigues x15, vec(R - I) ; warps 1.. : joint regression j_tpose = Jreg @ v_shaped (warp per joint row)
//   S3  warp 0    : serial FK chain over the kinematic tree ; warps 1.. : pose blend v_tpose += P*(R-I) ([135][2334] table)
//   S4  all warps : LBS per vertex (16 joint weights as 4x float4), results kept in shared memory
//   S5  21 threads: joints (FK joints + 5 finger tips), reorder, centre
//   S6  all warps : centre / scale / trans, coalesced stores
#include "common.cuh"
#include "mano_core.cuh"
using namespace rih;

struct ManoConsts {
  const float* comps;       // [45,45]  hands_components
  const float* hands_mean;  // [45]
  ManoTables t;             // shapedirsT, posedirsT, v_template, jreg, weights
  int parent[16];
  int new_order[21];
  int tips[5];
};

// S0-S5, shared by both kernels: vl receives the skinned vertices (it may be f.vt), jf the joints in output order and center the
// centre joint (0 when center_idx < 0), all before centre / scale / trans.  Ends with a __syncthreads().
__device__ __forceinline__ void mano_forward(ManoState& f, float* s_axis, float* vl, float (*jf)[3], float* center, const ManoConsts& mc,
                                             const float* __restrict__ root_rot, const float* __restrict__ pose, int use_pca, int ncomps,
                                             const float* __restrict__ shape, int center_idx, int b, int tid) {
  if (tid < 10) f.beta[tid] = shape[(size_t)b * 10 + tid];
  if (tid < 9) f.R[0][tid] = root_rot[(size_t)b * 9 + tid];
  if (use_pca) {
    if (tid < 45) {
      float acc = 0.f;
      for (int i = 0; i < ncomps; ++i) acc = fmaf(pose[(size_t)b * ncomps + i], mc.comps[i * 45 + tid], acc);
      s_axis[tid] = acc + mc.hands_mean[tid];
    }
  } else {
    if (tid < 135) f.R[1 + tid / 9][tid % 9] = pose[(size_t)b * 135 + tid];
  }
  __syncthreads();
  mano_forward_state(f, mc.t, mc.parent, tid, [&](int lane) {
    if (use_pca && lane < 15) {
      float ax = s_axis[lane * 3], ay = s_axis[lane * 3 + 1], az = s_axis[lane * 3 + 2];
      float angle = sqrtf(ax * ax + ay * ay + az * az) + 1e-8f;   // manolayer.py:37 (eps added after the norm)
      float x = ax / angle, y = ay / angle, z = az / angle;
      float sn = sinf(angle), cs = cosf(angle), oc = 1.f - cs;
      // L = [[0,-z,y],[z,0,-x],[-y,x,0]] ; R = I + sin*L + (1-cos)*L@L
      float* R = f.R[1 + lane];
      R[0] = 1.f + oc * (-(z * z) - (y * y)); R[1] = -sn * z + oc * (x * y);        R[2] = sn * y + oc * (x * z);
      R[3] = sn * z + oc * (x * y);         R[4] = 1.f + oc * (-(z * z) - (x * x)); R[5] = -sn * x + oc * (y * z);
      R[6] = -sn * y + oc * (x * z);        R[7] = sn * x + oc * (y * z);           R[8] = 1.f + oc * (-(y * y) - (x * x));
    }
  });
  for (int vtx = tid; vtx < MANO_V; vtx += MANO_THREADS) mano_skin(f, mc.t, vtx, vl);
  __syncthreads();
  if (tid < 21) {
    const int src = mc.new_order[tid];
    const float* p = src < 16 ? f.gt[src] : vl + mc.tips[src - 16] * 3;
    jf[tid][0] = p[0]; jf[tid][1] = p[1]; jf[tid][2] = p[2];
  }
  __syncthreads();
  if (tid < 3) center[tid] = center_idx >= 0 ? jf[center_idx][tid] : 0.f;
  __syncthreads();
}

__global__ void __launch_bounds__(MANO_THREADS)
mano_fwd_kernel(ManoConsts mc, const float* __restrict__ root_rot, const float* __restrict__ pose, int use_pca, int ncomps,
                const float* __restrict__ shape, const float* __restrict__ trans, const float* __restrict__ scale,
                int center_idx, int new_skel, float* __restrict__ v_out, float* __restrict__ j_out) {
  pdl_sync();
  __shared__ ManoState f;               // f.vt: v_shaped -> v_tpose -> v_output
  __shared__ float s_axis[48];
  __shared__ float s_jf[21][3];         // final joints
  __shared__ float s_center[3];
  const int b = blockIdx.x, tid = threadIdx.x;
  mano_forward(f, s_axis, f.vt, s_jf, s_center, mc, root_rot, pose, use_pca, ncomps, shape, center_idx, b, tid);
  // ---- S6: outputs
  float sc = scale ? scale[b] : 1.f;
  float tr[3] = {0.f, 0.f, 0.f};
  if (trans) { tr[0] = trans[(size_t)b * 3]; tr[1] = trans[(size_t)b * 3 + 1]; tr[2] = trans[(size_t)b * 3 + 2]; }
  for (int o = tid; o < MANO_V3; o += MANO_THREADS) {
    int c = o % 3;
    float val = f.vt[o];
    if (center_idx >= 0) val = val - s_center[c];
    if (scale) val = val * sc;
    if (trans) val = val + tr[c];
    f.vt[o] = val;
    v_out[(size_t)b * MANO_V3 + o] = val;
  }
  __syncthreads();
  if (tid < 63) {
    int jt = tid / 3, c = tid % 3;
    float val = s_jf[jt][c];
    if (center_idx >= 0) val = val - s_center[c];
    if (scale) val = val * sc;
    if (trans) val = val + tr[c];
    if (new_skel) {   // manolayer.py:316-320
      if (jt == 5) val = (f.vt[63 * 3 + c] + f.vt[144 * 3 + c]) / 2.f;
      else if (jt == 9) val = (f.vt[271 * 3 + c] + f.vt[220 * 3 + c]) / 2.f;
      else if (jt == 13) val = (f.vt[148 * 3 + c] + f.vt[290 * 3 + c]) / 2.f;
      else if (jt == 17) val = (f.vt[770 * 3 + c] + f.vt[83 * 3 + c]) / 2.f;
    }
    j_out[(size_t)b * 63 + tid] = val;
  }
}

static int fill_consts(ManoConsts& mc, const float* const* const_ptrs, const int* parent, const char* who) {
  mc.comps = const_ptrs[0]; mc.hands_mean = const_ptrs[1];
  mc.t = ManoTables{const_ptrs[2], const_ptrs[3], const_ptrs[4], const_ptrs[5], const_ptrs[6]};
  for (int i = 0; i < 16; ++i) {
    mc.parent[i] = parent[i];
    RIH_REQUIRE(i == 0 || (parent[i] >= 0 && parent[i] < i), "%s: kinematic parent table is not topologically ordered", who);
  }
  static const int order[21] = {0, 13, 14, 15, 16, 1, 2, 3, 17, 4, 5, 6, 18, 10, 11, 12, 19, 7, 8, 9, 20};  // manolayer.py:110-115
  static const int tips[5] = {745, 317, 444, 556, 673};                                                    // manolayer.py:296
  for (int i = 0; i < 21; ++i) mc.new_order[i] = order[i];
  for (int i = 0; i < 5; ++i) mc.tips[i] = tips[i];
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------- backward
// Gradient of ManoLayer.forward w.r.t. root_rotation / pose (PCA coefficients or 15 rotation matrices) / shape / trans / scale,
// as ONE kernel, one CTA per hand.  The reference differentiates this layer with autograd through ~120 torch kernels when the MANO
// tail is trained (common/myhand/decoder_lijun_mano.py:252-262 -> ManoLayer.forward, models/manolayer.py:250-322; SURVEY 8 a3 / f1).
// The CTA first recomputes the forward intermediates into shared memory (cheaper than saving them: 1.2 MFLOP, tables are L2
// resident), then walks the stages in reverse:
//   B1 outputs -> (trans, scale, centre) gradients, new_skel joints back to their vertex pairs        (block reductions)
//   B2 joint reorder / finger tips back to vertices
//   B3-B5 mano_backward and mano_shape_row: LBS, FK chain, pose blend, joint regressor and shape blend adjoints
//   B6 Rodrigues backward (eps added after the norm, manolayer.py:37) and PCA projection
__global__ void __launch_bounds__(MANO_THREADS)
mano_bwd_kernel(ManoConsts mc, const float* __restrict__ root_rot, const float* __restrict__ pose, int use_pca, int ncomps,
                const float* __restrict__ shape, const float* __restrict__ trans, const float* __restrict__ scale,
                int center_idx, int new_skel, const float* __restrict__ g_v, const float* __restrict__ g_j,
                float* __restrict__ d_root, float* __restrict__ d_pose, float* __restrict__ d_shape,
                float* __restrict__ d_trans, float* __restrict__ d_scale) {
  pdl_sync();
  __shared__ ManoState f;               // f.vt: v_shaped -> v_tpose
  __shared__ ManoGrad gs;
  __shared__ float s_vl[MANO_V3];       // skinned vertices (before centre / scale / trans)
  __shared__ float s_g[MANO_V3];        // gradient buffer: g(v_out) -> g(v_lbs) -> g(v_tpose) -> g(v_shaped)
  __shared__ float s_axis[48];
  __shared__ float s_jf[21][3];
  __shared__ float s_center[3];
  __shared__ float s_gjf[21][3], s_gjo[21][3], s_gaxis[48];
  __shared__ float s_red[MANO_WARPS];
  const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  mano_forward(f, s_axis, s_vl, s_jf, s_center, mc, root_rot, pose, use_pca, ncomps, shape, center_idx, b, tid);

  // ================= B1: output affine (centre / scale / trans) and new_skel
  for (int o = tid; o < MANO_V3; o += MANO_THREADS) s_g[o] = g_v ? g_v[(size_t)b * MANO_V3 + o] : 0.f;
  if (tid < 63) {
    const int jt = tid / 3;
    const bool overwritten = new_skel && (jt == 5 || jt == 9 || jt == 13 || jt == 17);   // replaced by vertex midpoints (manolayer.py:316-320)
    s_gjf[jt][tid % 3] = (g_j && !overwritten) ? g_j[(size_t)b * 63 + tid] : 0.f;
  }
  __syncthreads();
  if (new_skel && g_j && tid < 12) {
    const int q = tid / 3, c = tid % 3;
    const int jt = 5 + 4 * q;
    const int va = (q == 0) ? 63 : (q == 1) ? 271 : (q == 2) ? 148 : 770;
    const int vb = (q == 0) ? 144 : (q == 1) ? 220 : (q == 2) ? 290 : 83;
    const float h = 0.5f * g_j[(size_t)b * 63 + jt * 3 + c];
    s_g[va * 3 + c] += h; s_g[vb * 3 + c] += h;
  }
  __syncthreads();
  const float sc = scale ? scale[b] : 1.f;
  float p0 = 0.f, p1 = 0.f, p2 = 0.f, ps = 0.f;   // per-thread partials: sum of output gradients per component, <g, pre-scale value>
  for (int vtx = tid; vtx < MANO_V; vtx += MANO_THREADS) {
    const float gx = s_g[vtx * 3], gy = s_g[vtx * 3 + 1], gz = s_g[vtx * 3 + 2];
    p0 += gx; p1 += gy; p2 += gz;
    ps += gx * (s_vl[vtx * 3] - s_center[0]) + gy * (s_vl[vtx * 3 + 1] - s_center[1]) + gz * (s_vl[vtx * 3 + 2] - s_center[2]);
  }
  if (tid < 21) {
    const float gx = s_gjf[tid][0], gy = s_gjf[tid][1], gz = s_gjf[tid][2];
    p0 += gx; p1 += gy; p2 += gz;
    ps += gx * (s_jf[tid][0] - s_center[0]) + gy * (s_jf[tid][1] - s_center[1]) + gz * (s_jf[tid][2] - s_center[2]);
  }
  const float sum0 = block_sum<MANO_WARPS>(p0, s_red, tid), sum1 = block_sum<MANO_WARPS>(p1, s_red, tid);
  const float sum2 = block_sum<MANO_WARPS>(p2, s_red, tid), sums = block_sum<MANO_WARPS>(ps, s_red, tid);
  if (tid == 0) {
    if (d_trans) { d_trans[(size_t)b * 3] = trans ? sum0 : 0.f; d_trans[(size_t)b * 3 + 1] = trans ? sum1 : 0.f; d_trans[(size_t)b * 3 + 2] = trans ? sum2 : 0.f; }
    if (d_scale) d_scale[b] = scale ? sums : 0.f;
  }
  __syncthreads();
  for (int o = tid; o < MANO_V3; o += MANO_THREADS) s_g[o] *= sc;
  if (tid < 63) s_gjf[tid / 3][tid % 3] *= sc;
  __syncthreads();
  if (center_idx >= 0 && tid < 3) s_gjf[center_idx][tid] -= sc * (tid == 0 ? sum0 : (tid == 1 ? sum1 : sum2));
  __syncthreads();
  // ================= B2: reorder, finger tips
  if (tid < 21) { const int src = mc.new_order[tid]; s_gjo[src][0] = s_gjf[tid][0]; s_gjo[src][1] = s_gjf[tid][1]; s_gjo[src][2] = s_gjf[tid][2]; }
  __syncthreads();
  if (tid < 15) s_g[mc.tips[tid / 3] * 3 + tid % 3] += s_gjo[16 + tid / 3][tid % 3];
  __syncthreads();
  // ================= B3-B5
  mano_backward(f, mc.t, mc.parent, s_g, s_gjo, nullptr, gs, tid);
  // ================= B5c: shape blend (warps 0..9) || B6: rotations (warp 10)
  if (warp < 10) {
    if (d_shape) mano_shape_row(mc.t, s_g, warp, lane, d_shape + (size_t)b * 10 + warp);
  } else if (warp == 10) {
    if (d_root && lane < 9) d_root[(size_t)b * 9 + lane] = gs.gR[0][lane];
    if (d_pose) {
      if (!use_pca) {
        for (int i = lane; i < 135; i += 32) d_pose[(size_t)b * 135 + i] = gs.gR[1 + i / 9][i % 9];
      } else {
        if (lane < 15) {
          const float ax = s_axis[lane * 3], ay = s_axis[lane * 3 + 1], az = s_axis[lane * 3 + 2];
          const float nrm = sqrtf(ax * ax + ay * ay + az * az);
          const float th = nrm + 1e-8f;
          const float x = ax / th, y = ay / th, z = az / th;
          const float sn = sinf(th), cs = cosf(th), oc = 1.f - cs;
          const float* g = gs.gR[1 + lane];
          const float gx = -2.f * oc * x * (g[4] + g[8]) + oc * y * (g[1] + g[3]) + oc * z * (g[2] + g[6]) + sn * (g[7] - g[5]);
          const float gy = -2.f * oc * y * (g[0] + g[8]) + oc * x * (g[1] + g[3]) + oc * z * (g[5] + g[7]) + sn * (g[2] - g[6]);
          const float gz = -2.f * oc * z * (g[0] + g[4]) + oc * x * (g[2] + g[6]) + oc * y * (g[5] + g[7]) + sn * (g[3] - g[1]);
          const float gth = sn * (-(z * z + y * y) * g[0] - (z * z + x * x) * g[4] - (y * y + x * x) * g[8] + x * y * (g[1] + g[3]) + x * z * (g[2] + g[6]) + y * z * (g[5] + g[7]))
                          + cs * (z * (g[3] - g[1]) + y * (g[2] - g[6]) + x * (g[7] - g[5]));
          // u = a / th, th = |a| + eps: d th / d a = a / |a| (0 at a = 0, torch.norm's subgradient)
          const float inv = nrm > 0.f ? 1.f / nrm : 0.f;
          const float nx = ax * inv, ny = ay * inv, nz = az * inv;
          const float dotg = (gx * ax + gy * ay + gz * az) / (th * th);
          s_gaxis[lane * 3] = gx / th + (gth - dotg) * nx;
          s_gaxis[lane * 3 + 1] = gy / th + (gth - dotg) * ny;
          s_gaxis[lane * 3 + 2] = gz / th + (gth - dotg) * nz;
        }
        __syncwarp();
        for (int i = lane; i < ncomps; i += 32) {
          float acc = 0.f;
          for (int t = 0; t < 45; ++t) acc = fmaf(mc.comps[i * 45 + t], s_gaxis[t], acc);
          d_pose[(size_t)b * ncomps + i] = acc;
        }
      }
    }
  }
}

// Backward of rih_mano_fwd: g_v [B,778,3] / g_j [B,21,3] (either may be NULL = zero) -> d_root [B,9], d_pose [B,ncomps | 135],
// d_shape [B,10], d_trans [B,3], d_scale [B] (each may be NULL when not needed).  reference: autograd through models/manolayer.py:250-322.
RIH_API int rih_mano_bwd(const float* const* const_ptrs, const int* parent, const float* root_rot, const float* pose, int use_pca, int ncomps,
                         const float* shape, const float* trans, const float* scale, int center_idx, int new_skel,
                         const float* g_v, const float* g_j, float* d_root, float* d_pose, float* d_shape, float* d_trans, float* d_scale,
                         int B, cudaStream_t s) {
  RIH_REQUIRE(B >= 0, "mano_bwd: negative batch");
  RIH_REQUIRE(!use_pca || (ncomps >= 0 && ncomps <= 45), "mano_bwd: ncomps=%d out of range", ncomps);
  RIH_REQUIRE(center_idx < 21, "mano_bwd: center_idx=%d out of range", center_idx);
  if (B == 0) return 0;
  ManoConsts mc;
  if (int e = fill_consts(mc, const_ptrs, parent, "mano_bwd")) return e;
  launch_k(mano_bwd_kernel, B, MANO_THREADS, 0, s, mc, root_rot, pose, use_pca, ncomps, shape, trans, scale, center_idx, new_skel, g_v, g_j,
                                             d_root, d_pose, d_shape, d_trans, d_scale);
  return check_launch("mano_bwd");
}

// consts: 7 device pointers in the order of ManoConsts; parent[16]
RIH_API int rih_mano_fwd(const float* const* const_ptrs, const int* parent, const float* root_rot, const float* pose, int use_pca, int ncomps,
                         const float* shape, const float* trans, const float* scale, int center_idx, int new_skel,
                         float* v_out, float* j_out, int B, cudaStream_t s) {
  RIH_REQUIRE(B >= 0, "mano_fwd: negative batch");
  RIH_REQUIRE(!use_pca || (ncomps >= 0 && ncomps <= 45), "mano_fwd: ncomps=%d out of range", ncomps);
  RIH_REQUIRE(center_idx < 21, "mano_fwd: center_idx=%d out of range", center_idx);
  if (B == 0) return 0;
  ManoConsts mc;
  if (int e = fill_consts(mc, const_ptrs, parent, "mano_fwd")) return e;
  launch_k(mano_fwd_kernel, B, MANO_THREADS, 0, s, mc, root_rot, pose, use_pca, ncomps, shape, trans, scale, center_idx, new_skel, v_out, j_out);
  return check_launch("mano_fwd");
}
