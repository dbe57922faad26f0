// The pose optimiser's quaternion hand model -- the extended hassony2 `manopth` ManoLayer in quat/quat mode without PCA
// (pose_data_optimize/manopth/manopth/manolayer.py:172-380) -- forward and backward, each ONE kernel with one CTA per hand.
// The MANO stages are those of csrc/mano_core.cuh; what differs is the layer's own conventions:
//   * rotations are unnormalised quaternions (w,x,y,z); each matrix entry is divided by |q|^2 (quatutils.py:188-221), and left hands
//     negate q.y and q.z first (manolayer.py:243-245);
//   * the kinematic chain is the hard-coded three-level chain 0 -> {1,4,7,10,13} -> {2,5,...} -> {3,6,...} (manolayer.py:276-312);
//   * joints: the 16 global translations, joint 0 optionally replaced by the palm (vertices 95, 22; :339-341), finger tips
//     745/317/444|445/556/673 (right|left, :335-338), reordered with the :345 list;
//   * centring (:347-366) is decided over the whole th_trans tensor: a device-side flag (rih_manopth_translate_flag) says whether
//     th_trans is added (norm != 0) or joint `center_idx` is subtracted; the transforms' translation is global t - centre + trans.
// No float atomics: every sum runs in a fixed order, so results are bitwise reproducible.
#include "common.cuh"
#include "hand_pose.cuh"
#include "mano_core.cuh"
using namespace rih;

namespace {

__constant__ int c_parent[16] = {0, 0, 1, 2, 0, 4, 5, 0, 7, 8, 0, 10, 11, 0, 13, 14};                 // manolayer.py:281-310
__constant__ int c_order[21] = {0, 13, 14, 15, 16, 1, 2, 3, 17, 4, 5, 6, 18, 10, 11, 12, 19, 7, 8, 9, 20};  // manolayer.py:345
__constant__ int c_tips[2][5] = {{745, 317, 444, 556, 673}, {745, 317, 445, 556, 673}};                 // manolayer.py:335-338
constexpr int PALM_A = 95, PALM_B = 22;                                                                   // manolayer.py:340

// Everything up to the skinning input (v_posed, A_i, G_i.t); the caller skins.  q receives the quaternions after the left-hand sign flip.
__device__ __forceinline__ void forward_state(ManoState& f, float (*q)[4], const ManoTables& mt, const float* __restrict__ quat,
                                              const float* __restrict__ betas, int betas_shared, int side, int b, int tid) {
  if (tid < 10) f.beta[tid] = betas ? betas[(size_t)(betas_shared ? 0 : b) * 10 + tid] : 0.f;
  __syncthreads();
  mano_forward_state(f, mt, c_parent, tid, [&](int lane) {
    if (lane < 16) {
      const float* p = quat + (size_t)b * 64 + lane * 4;
      const float s = side ? -1.f : 1.f;
      q[lane][0] = p[0]; q[lane][1] = p[1]; q[lane][2] = s * p[2]; q[lane][3] = s * p[3];
      quat_to_R(q[lane][0], q[lane][1], q[lane][2], q[lane][3], f.R[lane]);
    }
  });
}

// joints before centring, in output order (palm, tips, :345 reorder)
__device__ __forceinline__ void output_joint(const ManoState& f, const float* vl, int k, int root_palm, int side, float* o) {
  const int src = c_order[k];
  for (int c = 0; c < 3; ++c) {
    if (src >= 16) o[c] = vl[c_tips[side][src - 16] * 3 + c];
    else if (src == 0 && root_palm) o[c] = (vl[PALM_A * 3 + c] + vl[PALM_B * 3 + c]) / 2.f;
    else o[c] = f.gt[src][c];
  }
}

__global__ void __launch_bounds__(MANO_THREADS)
manopth_fwd_kernel(ManoTables mt, const float* __restrict__ quat, const float* __restrict__ betas, int betas_shared,
                   const float* __restrict__ trans, const int* __restrict__ translate, int center_idx, int root_palm, int side,
                   float* __restrict__ v_out, float* __restrict__ j_out, float* __restrict__ transf_out) {
  pdl_sync();
  __shared__ ManoState f;
  __shared__ float s_q[16][4];
  __shared__ float s_vl[MANO_V3];
  __shared__ float s_jf[21][3];
  __shared__ float s_off[3];           // - centre, or + trans
  const int b = blockIdx.x, tid = threadIdx.x;
  forward_state(f, s_q, mt, quat, betas, betas_shared, side, b, tid);
  for (int vtx = tid; vtx < MANO_V; vtx += MANO_THREADS) mano_skin(f, mt, vtx, s_vl);
  __syncthreads();
  if (tid < 21) output_joint(f, s_vl, tid, root_palm, side, s_jf[tid]);
  __syncthreads();
  const bool add_trans = trans && *translate;
  if (tid < 3) s_off[tid] = add_trans ? trans[(size_t)b * 3 + tid] : (center_idx >= 0 ? -s_jf[center_idx][tid] : 0.f);
  __syncthreads();
  for (int o = tid; o < MANO_V3; o += MANO_THREADS) v_out[(size_t)b * MANO_V3 + o] = s_vl[o] + s_off[o % 3];
  if (tid < 63) j_out[(size_t)b * 63 + tid] = s_jf[tid / 3][tid % 3] + s_off[tid % 3];
  if (transf_out && tid < 256) {
    const int i = tid / 16, r = (tid / 4) % 4, c = tid % 4;
    float val;
    if (r == 3) val = c == 3 ? 1.f : 0.f;
    else if (c < 3) val = f.T[i][r * 4 + c];
    else {   // global t - centre + trans (manolayer.py:363); trans is all zeros whenever the centre is subtracted
      val = f.gt[i][r] + (add_trans ? 0.f : s_off[r]);
      if (trans) val += trans[(size_t)b * 3 + r];
    }
    transf_out[(size_t)b * 256 + tid] = val;
  }
}

// ---------------------------------------------------------------------------------------------------------------- backward
// The CTA recomputes the forward state (cheaper than storing it), then walks back as rih_mano_bwd does:
//   B1 output offset: d_trans, the centre's gradient onto its joint          B2 reorder, palm and tips back to vertices
//   B3-B5 mano_backward, with the transforms' rotation gradient added to gA   B6 quaternion backward
__global__ void __launch_bounds__(MANO_THREADS)
manopth_bwd_kernel(ManoTables mt, const float* __restrict__ quat, const float* __restrict__ betas, int betas_shared,
                   const float* __restrict__ trans, const int* __restrict__ translate, int center_idx, int root_palm, int side,
                   const float* __restrict__ g_v, const float* __restrict__ g_j, const float* __restrict__ g_transf,
                   float* __restrict__ d_quat, float* __restrict__ d_betas_rows, float* __restrict__ d_trans) {
  pdl_sync();
  __shared__ ManoState f;
  __shared__ ManoGrad gs;
  __shared__ float s_q[16][4];
  __shared__ float s_g[MANO_V3];       // g(v_out) -> g(v_lbs) -> g(v_posed) -> g(v_shaped)
  __shared__ float s_gjf[21][3], s_gjo[16][3];
  __shared__ float s_red[MANO_WARPS];
  const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  forward_state(f, s_q, mt, quat, betas, betas_shared, side, b, tid);
  const bool add_trans = trans && *translate;

  // ================= B1
  for (int o = tid; o < MANO_V3; o += MANO_THREADS) s_g[o] = g_v ? g_v[(size_t)b * MANO_V3 + o] : 0.f;
  if (tid < 63) s_gjf[tid / 3][tid % 3] = g_j ? g_j[(size_t)b * 63 + tid] : 0.f;
  __syncthreads();
  float p[3] = {0.f, 0.f, 0.f}, pt[3] = {0.f, 0.f, 0.f};   // per-thread partials over verts + joints, and over the transforms' t
  for (int vtx = tid; vtx < MANO_V; vtx += MANO_THREADS)
    for (int c = 0; c < 3; ++c) p[c] += s_g[vtx * 3 + c];
  if (tid < 21)
    for (int c = 0; c < 3; ++c) p[c] += s_gjf[tid][c];
  if (g_transf && tid < 16)
    for (int c = 0; c < 3; ++c) pt[c] = g_transf[(size_t)b * 256 + tid * 16 + c * 4 + 3];
  float S[3], St[3];
  for (int c = 0; c < 3; ++c) { S[c] = block_sum<MANO_WARPS>(p[c], s_red, tid); St[c] = block_sum<MANO_WARPS>(pt[c], s_red, tid); }
  if (d_trans && tid < 3) d_trans[(size_t)b * 3 + tid] = St[tid] + (add_trans ? S[tid] : 0.f);
  if (!add_trans && center_idx >= 0 && tid < 3) s_gjf[center_idx][tid] -= S[tid] + St[tid];
  __syncthreads();
  // ================= B2
  if (tid < 3) {
    const int c = tid;
    for (int k = 0; k < 21; ++k) {
      const int src = c_order[k];
      const float g = s_gjf[k][c];
      if (src >= 16) s_g[c_tips[side][src - 16] * 3 + c] += g;
      else if (src == 0 && root_palm) { s_g[PALM_A * 3 + c] += g / 2.f; s_g[PALM_B * 3 + c] += g / 2.f; s_gjo[0][c] = 0.f; }
      else s_gjo[src][c] = g;
    }
    for (int i = 0; i < 16; ++i) if (g_transf) s_gjo[i][c] += g_transf[(size_t)b * 256 + i * 16 + c * 4 + 3];
  }
  __syncthreads();
  // ================= B3-B5
  mano_backward(f, mt, c_parent, s_g, s_gjo, g_transf ? g_transf + (size_t)b * 256 : nullptr, gs, tid);
  // ================= B5c: shape blend (warps 0..9) || B6: quaternions (warp 10)
  if (warp < 10) {
    if (d_betas_rows) mano_shape_row(mt, s_g, warp, lane, d_betas_rows + (size_t)b * 10 + warp);
  } else if (warp == 10 && lane < 16 && d_quat) {
    float d[4];
    quat_R_backward(s_q[lane], f.R[lane], gs.gR[lane], d);
    const float s = side ? -1.f : 1.f;          // left hands: q.y, q.z were negated before the conversion
    float* o = d_quat + (size_t)b * 64 + lane * 4;
    o[0] = d[0]; o[1] = d[1]; o[2] = s * d[2]; o[3] = s * d[3];
  }
}

// d_betas of a shared row: the per-hand rows summed over the batch in a fixed order (warp per coefficient)
__global__ void __launch_bounds__(320) manopth_betas_reduce_kernel(const float* __restrict__ rows, int B, float* __restrict__ out) {
  pdl_sync();
  const int k = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float acc = 0.f;
  for (int b = lane; b < B; b += 32) acc += rows[(size_t)b * 10 + k];
  acc = warp_sum(acc);
  if (lane == 0) out[k] = acc;
}

__global__ void __launch_bounds__(1024) manopth_translate_flag_kernel(const float* __restrict__ trans, int n, int* __restrict__ flag) {
  pdl_sync();
  int nz = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) { const float x = trans[i]; nz |= (x * x != 0.f); }   // NaN counts as non-zero
  nz = __syncthreads_or(nz);
  if (threadIdx.x == 0) *flag = nz;
}

int check_args(const float* const* const_ptrs, int B, int center_idx, int side, const char* who) {
  RIH_REQUIRE(B >= 0, "%s: negative batch", who);
  RIH_REQUIRE(center_idx >= -1 && center_idx < 21, "%s: center_idx=%d out of range", who, center_idx);
  RIH_REQUIRE(side == 0 || side == 1, "%s: side=%d (0 = right, 1 = left)", who, side);
  for (int i = 0; i < 5; ++i) RIH_REQUIRE(const_ptrs[i] != nullptr, "%s: constant table %d is NULL", who, i);
  return 0;
}

// left hands: the x rows of shapedirsT are negated by the caller (manolayer.py:169-170)
ManoTables consts(const float* const* p) { return ManoTables{p[0], p[1], p[2], p[3], p[4]}; }

}  // namespace

// flag[0] = 1 if any of trans[0..n) is non-zero (torch.norm(th_trans) != 0, manolayer.py:347), else 0; computed on the device so the
// forward never synchronises.  One CTA.
RIH_API int rih_manopth_translate_flag(const float* trans, int n, int* flag, cudaStream_t s) {
  RIH_REQUIRE(n >= 0 && (n == 0 || trans) && flag, "manopth_translate_flag: bad arguments (n=%d)", n);
  launch_k(manopth_translate_flag_kernel, 1, 1024, 0, s, trans, n, flag);
  return check_launch("manopth_translate_flag");
}

// Forward of the quaternion manopth ManoLayer (pose_data_optimize/manopth/manopth/manolayer.py:172-380, quat/quat, no PCA).
// consts: 5 device pointers shapedirsT [10][2334], posedirsT [135][2334], v_template [2334], J_regressor [16,778], weights [778,16].
// quat [B,16,4] (w,x,y,z); betas [B,10], or one row shared by the batch (betas_shared = 1), or NULL = zeros; trans [B,3] or NULL;
// translate: device int from rih_manopth_translate_flag (read only when trans != NULL); center_idx -1 = none; side 0 right / 1 left.
// -> verts [B,778,3], joints [B,21,3], transf [B,16,4,4] (NULL = not written).
RIH_API int rih_manopth_fwd(const float* const* const_ptrs, const float* quat, const float* betas, int betas_shared, const float* trans,
                            const int* translate, int center_idx, int root_palm, int side, float* verts, float* joints, float* transf,
                            int B, cudaStream_t s) {
  if (int e = check_args(const_ptrs, B, center_idx, side, "manopth_fwd")) return e;
  RIH_REQUIRE(!trans || translate, "manopth_fwd: trans without a translate flag");
  if (B == 0) return 0;
  launch_k(manopth_fwd_kernel, B, MANO_THREADS, 0, s, consts(const_ptrs), quat, betas, betas_shared, trans, translate, center_idx, root_palm, side,
           verts, joints, transf);
  return check_launch("manopth_fwd");
}

// Backward of rih_manopth_fwd (autograd through manolayer.py:172-380).  g_verts [B,778,3], g_joints [B,21,3], g_transf [B,16,4,4]: each
// may be NULL (= zero).  -> d_quat [B,16,4], d_betas [B,10] (or [1,10] summed over the batch when betas_shared; then work must hold
// B*10 floats), d_trans [B,3]; each may be NULL when not needed.
RIH_API int rih_manopth_bwd(const float* const* const_ptrs, const float* quat, const float* betas, int betas_shared, const float* trans,
                            const int* translate, int center_idx, int root_palm, int side, const float* g_verts, const float* g_joints,
                            const float* g_transf, float* d_quat, float* d_betas, float* d_trans, float* work, int B, cudaStream_t s) {
  if (int e = check_args(const_ptrs, B, center_idx, side, "manopth_bwd")) return e;
  RIH_REQUIRE(!trans || translate, "manopth_bwd: trans without a translate flag");
  RIH_REQUIRE(!d_betas || betas, "manopth_bwd: d_betas requested without betas");
  RIH_REQUIRE(!d_trans || trans, "manopth_bwd: d_trans requested without trans");
  RIH_REQUIRE(!(d_betas && betas_shared) || work, "manopth_bwd: a shared betas row needs a B*10 workspace");
  if (B == 0) {
    if (d_betas && betas_shared) RIH_REQUIRE(cudaMemsetAsync(d_betas, 0, 10 * sizeof(float), s) == cudaSuccess, "manopth_bwd: memset failed");
    return 0;
  }
  float* rows = (d_betas && betas_shared) ? work : d_betas;
  launch_k(manopth_bwd_kernel, B, MANO_THREADS, 0, s, consts(const_ptrs), quat, betas, betas_shared, trans, translate, center_idx, root_palm, side,
           g_verts, g_joints, g_transf, d_quat, rows, d_trans);
  if (int e = check_launch("manopth_bwd")) return e;
  if (d_betas && betas_shared) {
    launch_k(manopth_betas_reduce_kernel, 1, 320, 0, s, (const float*)work, B, d_betas);
    return check_launch("manopth_betas_reduce");
  }
  return 0;
}
