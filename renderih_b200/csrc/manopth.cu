// The pose optimiser's quaternion hand model -- the extended hassony2 `manopth` ManoLayer in quat/quat mode without PCA
// (pose_data_optimize/manopth/manopth/manolayer.py:172-380) -- forward and backward, each ONE kernel with one CTA per hand.
// The staging follows csrc/mano.cu; what differs is the layer's own conventions:
//   * rotations are unnormalised quaternions (w,x,y,z); each matrix entry is divided by |q|^2 (quatutils.py:188-221), and left hands
//     negate q.y and q.z first (manolayer.py:243-245);
//   * the kinematic chain is the hard-coded three-level chain 0 -> {1,4,7,10,13} -> {2,5,...} -> {3,6,...} (manolayer.py:276-312);
//   * joints: the 16 global translations, joint 0 optionally replaced by the palm (vertices 95, 22; :339-341), finger tips
//     745/317/444|445/556/673 (right|left, :335-338), reordered with the :345 list;
//   * centring (:347-366) is decided over the whole th_trans tensor: a device-side flag (rih_manopth_translate_flag) says whether
//     th_trans is added (norm != 0) or joint `center_idx` is subtracted; the transforms' translation is global t - centre + trans.
// No float atomics: every sum runs in a fixed order, so results are bitwise reproducible.
#include "common.cuh"
using namespace rih;

namespace {

struct ManopthConsts {
  const float* shapedirsT;  // [10][2334]  (left hands: x rows negated by the caller, manolayer.py:169-170)
  const float* posedirsT;   // [135][2334]
  const float* v_template;  // [2334]
  const float* jreg;        // [16,778]
  const float* weights;     // [778,16]
};

constexpr int V = 778, V3 = 2334, THREADS = 512, NWARPS = THREADS / 32;
__constant__ int c_parent[16] = {0, 0, 1, 2, 0, 4, 5, 0, 7, 8, 0, 10, 11, 0, 13, 14};                 // manolayer.py:281-310
__constant__ int c_order[21] = {0, 13, 14, 15, 16, 1, 2, 3, 17, 4, 5, 6, 18, 10, 11, 12, 19, 7, 8, 9, 20};  // manolayer.py:345
__constant__ int c_tips[2][5] = {{745, 317, 444, 556, 673}, {745, 317, 445, 556, 673}};                 // manolayer.py:335-338
constexpr int PALM_A = 95, PALM_B = 22;                                                                   // manolayer.py:340

// quatutils.py:191-216: entries of the (unnormalised) rotation matrix over |q|^2
__device__ __forceinline__ void quat_to_R(float w, float x, float y, float z, float* R) {
  const float ww = w * w, wx = w * x, wy = w * y, wz = w * z, xx = x * x, xy = x * y, xz = x * z, yy = y * y, yz = y * z, zz = z * z;
  const float n = ww + xx + yy + zz;
  R[0] = (ww + xx - yy - zz) / n; R[1] = 2.f * (xy - wz) / n;       R[2] = 2.f * (wy + xz) / n;
  R[3] = 2.f * (wz + xy) / n;     R[4] = (ww - xx + yy - zz) / n;   R[5] = 2.f * (yz - wx) / n;
  R[6] = 2.f * (xz - wy) / n;     R[7] = 2.f * (wx + yz) / n;       R[8] = (ww - xx - yy + zz) / n;
}

__device__ __forceinline__ float block_sum(float v, float* s_red, int tid) {
  v = warp_sum(v);
  __syncthreads();
  if ((tid & 31) == 0) s_red[tid >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int i = 0; i < NWARPS; ++i) t += s_red[i];
  return t;
}

// Forward state of one hand in shared memory, shared by both kernels.
struct Fwd {
  float vt[V3];        // v_shaped -> v_posed
  float R[16][9];      // joint rotations
  float q[16][4];      // quaternions after the left-hand sign flip
  float ps[136];       // vec(R - I) of joints 1..15
  float beta[10];
  float j[16][3];      // rest joints J_regressor @ v_shaped
  float t[16][3];      // local translations (I - R_i) j_i
  float T[16][12];     // skinning transforms A_i = [G_i.R | G_i.t - G_i.R j_i]
  float gt[16][3];     // global translations G_i.t (joint positions, native order)
};

// Everything up to the skinning input (v_posed, A_i, G_i.t); the caller skins.
__device__ void forward_state(Fwd& f, const ManopthConsts& mc, const float* __restrict__ quat, const float* __restrict__ betas, int betas_shared,
                              int side, int b, int tid) {
  const int warp = tid >> 5, lane = tid & 31;
  if (tid < 10) f.beta[tid] = betas ? betas[(size_t)(betas_shared ? 0 : b) * 10 + tid] : 0.f;
  if (tid < 16) {
    const float* q = quat + (size_t)b * 64 + tid * 4;
    const float s = side ? -1.f : 1.f;
    f.q[tid][0] = q[0]; f.q[tid][1] = q[1]; f.q[tid][2] = s * q[2]; f.q[tid][3] = s * q[3];
    quat_to_R(f.q[tid][0], f.q[tid][1], f.q[tid][2], f.q[tid][3], f.R[tid]);
  }
  __syncthreads();
  for (int o = tid; o < V3; o += THREADS) {
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < 10; ++i) acc = fmaf(mc.shapedirsT[i * V3 + o], f.beta[i], acc);
    f.vt[o] = mc.v_template[o] + acc;
  }
  if (tid < 135) { const int k = tid % 9; f.ps[tid] = f.R[1 + tid / 9][k] - ((k == 0 || k == 4 || k == 8) ? 1.f : 0.f); }
  __syncthreads();
  for (int o = warp; o < 48; o += NWARPS) {
    const int jt = o / 3, c = o % 3;
    float acc = 0.f;
    for (int vtx = lane; vtx < V; vtx += 32) acc = fmaf(mc.jreg[jt * V + vtx], f.vt[vtx * 3 + c], acc);
    acc = warp_sum(acc);
    if (lane == 0) f.j[jt][c] = acc;
  }
  __syncthreads();
  if (warp == 0) {
    if (lane == 0) {
      // G_0 = [R_0 | j_0]; G_i = G_p [R_i | j_i - j_p]  <=>  A_i = A_p [R_i | (I - R_i) j_i] with A_i = G_i - [0 | G_i.R j_i]
      for (int i = 0; i < 16; ++i) {
        const float* R = f.R[i];
        const float jx = f.j[i][0], jy = f.j[i][1], jz = f.j[i][2];
        float t[3];
        t[0] = (1.f - R[0]) * jx + (-R[1]) * jy + (-R[2]) * jz;
        t[1] = (-R[3]) * jx + (1.f - R[4]) * jy + (-R[5]) * jz;
        t[2] = (-R[6]) * jx + (-R[7]) * jy + (1.f - R[8]) * jz;
        f.t[i][0] = t[0]; f.t[i][1] = t[1]; f.t[i][2] = t[2];
        if (i == 0) {
          for (int r = 0; r < 3; ++r) {
            f.T[0][r * 4 + 0] = R[r * 3]; f.T[0][r * 4 + 1] = R[r * 3 + 1]; f.T[0][r * 4 + 2] = R[r * 3 + 2]; f.T[0][r * 4 + 3] = t[r];
            f.gt[0][r] = f.j[0][r];
          }
        } else {
          const float* P = f.T[c_parent[i]];
          for (int r = 0; r < 3; ++r) {
            const float p0 = P[r * 4], p1 = P[r * 4 + 1], p2 = P[r * 4 + 2], p3 = P[r * 4 + 3];
            f.T[i][r * 4 + 0] = p0 * R[0] + p1 * R[3] + p2 * R[6];
            f.T[i][r * 4 + 1] = p0 * R[1] + p1 * R[4] + p2 * R[7];
            f.T[i][r * 4 + 2] = p0 * R[2] + p1 * R[5] + p2 * R[8];
            f.T[i][r * 4 + 3] = p0 * t[0] + p1 * t[1] + p2 * t[2] + p3;
            f.gt[i][r] = p0 * jx + p1 * jy + p2 * jz + p3;
          }
        }
      }
    }
  } else {
    for (int o = tid - 32; o < V3; o += THREADS - 32) {
      float acc = 0.f;
#pragma unroll 9
      for (int i = 0; i < 135; ++i) acc = fmaf(mc.posedirsT[i * V3 + o], f.ps[i], acc);
      f.vt[o] += acc;
    }
  }
  __syncthreads();
}

__device__ __forceinline__ void skin(const Fwd& f, const ManopthConsts& mc, int vtx, float* out) {
  const float4* w4 = reinterpret_cast<const float4*>(mc.weights + (size_t)vtx * 16);
  float w[16];
#pragma unroll
  for (int i = 0; i < 4; ++i) { float4 t = __ldg(w4 + i); w[4 * i] = t.x; w[4 * i + 1] = t.y; w[4 * i + 2] = t.z; w[4 * i + 3] = t.w; }
  float T[12];
#pragma unroll
  for (int e = 0; e < 12; ++e) T[e] = 0.f;
#pragma unroll
  for (int jt = 0; jt < 16; ++jt)
#pragma unroll
    for (int e = 0; e < 12; ++e) T[e] = fmaf(w[jt], f.T[jt][e], T[e]);
  const float x = f.vt[vtx * 3], y = f.vt[vtx * 3 + 1], z = f.vt[vtx * 3 + 2];
  out[vtx * 3] = T[0] * x + T[1] * y + T[2] * z + T[3];
  out[vtx * 3 + 1] = T[4] * x + T[5] * y + T[6] * z + T[7];
  out[vtx * 3 + 2] = T[8] * x + T[9] * y + T[10] * z + T[11];
}

// joints before centring, in output order (palm, tips, :345 reorder)
__device__ __forceinline__ void output_joint(const Fwd& f, const float* vl, int k, int root_palm, int side, float* o) {
  const int src = c_order[k];
  for (int c = 0; c < 3; ++c) {
    if (src >= 16) o[c] = vl[c_tips[side][src - 16] * 3 + c];
    else if (src == 0 && root_palm) o[c] = (vl[PALM_A * 3 + c] + vl[PALM_B * 3 + c]) / 2.f;
    else o[c] = f.gt[src][c];
  }
}

__global__ void __launch_bounds__(THREADS)
manopth_fwd_kernel(ManopthConsts mc, const float* __restrict__ quat, const float* __restrict__ betas, int betas_shared,
                   const float* __restrict__ trans, const int* __restrict__ translate, int center_idx, int root_palm, int side,
                   float* __restrict__ v_out, float* __restrict__ j_out, float* __restrict__ transf_out) {
  pdl_sync();
  __shared__ Fwd f;
  __shared__ float s_vl[V3];
  __shared__ float s_jf[21][3];
  __shared__ float s_off[3];           // - centre, or + trans
  const int b = blockIdx.x, tid = threadIdx.x;
  forward_state(f, mc, quat, betas, betas_shared, side, b, tid);
  for (int vtx = tid; vtx < V; vtx += THREADS) skin(f, mc, vtx, s_vl);
  __syncthreads();
  if (tid < 21) output_joint(f, s_vl, tid, root_palm, side, s_jf[tid]);
  __syncthreads();
  const bool add_trans = trans && *translate;
  if (tid < 3) s_off[tid] = add_trans ? trans[(size_t)b * 3 + tid] : (center_idx >= 0 ? -s_jf[center_idx][tid] : 0.f);
  __syncthreads();
  for (int o = tid; o < V3; o += THREADS) v_out[(size_t)b * V3 + o] = s_vl[o] + s_off[o % 3];
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
//   B3 skinning: gA_i = sum_v w[v,i] g_v (x) [v_posed; 1], g_vposed = T_v.R^T g_v ; B4 chain backward (one thread)
//   B5 pose blend, joint regressor, shape blend                               B6 quaternion backward
__global__ void __launch_bounds__(THREADS)
manopth_bwd_kernel(ManopthConsts mc, const float* __restrict__ quat, const float* __restrict__ betas, int betas_shared,
                   const float* __restrict__ trans, const int* __restrict__ translate, int center_idx, int root_palm, int side,
                   const float* __restrict__ g_v, const float* __restrict__ g_j, const float* __restrict__ g_transf,
                   float* __restrict__ d_quat, float* __restrict__ d_betas_rows, float* __restrict__ d_trans) {
  pdl_sync();
  __shared__ Fwd f;
  __shared__ float s_g[V3];            // g(v_out) -> g(v_lbs) -> g(v_posed) -> g(v_shaped)
  __shared__ float s_gjf[21][3], s_gjo[16][3], s_gj[16][3], s_gG[16][12], s_gR[16][9], s_gps[136];
  __shared__ float s_red[NWARPS];
  const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  forward_state(f, mc, quat, betas, betas_shared, side, b, tid);
  const bool add_trans = trans && *translate;

  // ================= B1
  for (int o = tid; o < V3; o += THREADS) s_g[o] = g_v ? g_v[(size_t)b * V3 + o] : 0.f;
  if (tid < 63) s_gjf[tid / 3][tid % 3] = g_j ? g_j[(size_t)b * 63 + tid] : 0.f;
  __syncthreads();
  float p[3] = {0.f, 0.f, 0.f}, pt[3] = {0.f, 0.f, 0.f};   // per-thread partials over verts + joints, and over the transforms' t
  for (int vtx = tid; vtx < V; vtx += THREADS)
    for (int c = 0; c < 3; ++c) p[c] += s_g[vtx * 3 + c];
  if (tid < 21)
    for (int c = 0; c < 3; ++c) p[c] += s_gjf[tid][c];
  if (g_transf && tid < 16)
    for (int c = 0; c < 3; ++c) pt[c] = g_transf[(size_t)b * 256 + tid * 16 + c * 4 + 3];
  float S[3], St[3];
  for (int c = 0; c < 3; ++c) { S[c] = block_sum(p[c], s_red, tid); St[c] = block_sum(pt[c], s_red, tid); }
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
  // ================= B3a (warp i <-> joint i)
  {
    const int jt = warp;
    float a[12];
#pragma unroll
    for (int e = 0; e < 12; ++e) a[e] = 0.f;
    for (int vtx = lane; vtx < V; vtx += 32) {
      const float w = __ldg(mc.weights + (size_t)vtx * 16 + jt);
      const float gx = w * s_g[vtx * 3], gy = w * s_g[vtx * 3 + 1], gz = w * s_g[vtx * 3 + 2];
      const float x = f.vt[vtx * 3], y = f.vt[vtx * 3 + 1], z = f.vt[vtx * 3 + 2];
      a[0] = fmaf(gx, x, a[0]); a[1] = fmaf(gx, y, a[1]); a[2] = fmaf(gx, z, a[2]); a[3] += gx;
      a[4] = fmaf(gy, x, a[4]); a[5] = fmaf(gy, y, a[5]); a[6] = fmaf(gy, z, a[6]); a[7] += gy;
      a[8] = fmaf(gz, x, a[8]); a[9] = fmaf(gz, y, a[9]); a[10] = fmaf(gz, z, a[10]); a[11] += gz;
    }
#pragma unroll
    for (int e = 0; e < 12; ++e) a[e] = warp_sum(a[e]);
    if (lane == 0) {
#pragma unroll
      for (int e = 0; e < 12; ++e)   // A_i.R = G_i.R: the transforms' rotation gradient adds here
        s_gG[jt][e] = a[e] + ((g_transf && (e & 3) != 3) ? g_transf[(size_t)b * 256 + jt * 16 + e] : 0.f);
    }
  }
  __syncthreads();
  // ================= B3b (warps 1..) || B4 (thread 0)
  if (warp == 0) {
    if (lane == 0) {
      // global translations: gt_0 = j_0 ; gt_i = A_p.R j_i + A_p.t
      for (int c = 0; c < 3; ++c) s_gj[0][c] = s_gjo[0][c];
      for (int i = 1; i < 16; ++i) {
        const int pa = c_parent[i];
        const float* P = f.T[pa];
        const float g[3] = {s_gjo[i][0], s_gjo[i][1], s_gjo[i][2]};
        for (int c = 0; c < 3; ++c) s_gj[i][c] = P[0 * 4 + c] * g[0] + P[1 * 4 + c] * g[1] + P[2 * 4 + c] * g[2];
        for (int r = 0; r < 3; ++r) {
          s_gG[pa][r * 4 + 0] += g[r] * f.j[i][0]; s_gG[pa][r * 4 + 1] += g[r] * f.j[i][1]; s_gG[pa][r * 4 + 2] += g[r] * f.j[i][2];
          s_gG[pa][r * 4 + 3] += g[r];
        }
      }
      // chain: A_i.R = A_p.R R_i ; A_i.t = A_p.R t_i + A_p.t (children carry larger indices than their parents)
      for (int i = 15; i >= 0; --i) {
        const float* gG = s_gG[i];
        const float* R = f.R[i];
        float gR[9], gt[3];
        if (i > 0) {
          const int pa = c_parent[i];
          const float* P = f.T[pa];
          float* gP = s_gG[pa];
          for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c)
              gP[r * 4 + c] += gG[r * 4 + 0] * R[c * 3 + 0] + gG[r * 4 + 1] * R[c * 3 + 1] + gG[r * 4 + 2] * R[c * 3 + 2] + gG[r * 4 + 3] * f.t[i][c];
            gP[r * 4 + 3] += gG[r * 4 + 3];
          }
          for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c) gR[r * 3 + c] = P[0 * 4 + r] * gG[0 * 4 + c] + P[1 * 4 + r] * gG[1 * 4 + c] + P[2 * 4 + r] * gG[2 * 4 + c];
            gt[r] = P[0 * 4 + r] * gG[3] + P[1 * 4 + r] * gG[7] + P[2 * 4 + r] * gG[11];
          }
        } else {
          for (int r = 0; r < 3; ++r) { gR[r * 3] = gG[r * 4]; gR[r * 3 + 1] = gG[r * 4 + 1]; gR[r * 3 + 2] = gG[r * 4 + 2]; gt[r] = gG[r * 4 + 3]; }
        }
        // t_i = (I - R_i) j_i
        for (int c = 0; c < 3; ++c) s_gj[i][c] += gt[c] - (R[0 * 3 + c] * gt[0] + R[1 * 3 + c] * gt[1] + R[2 * 3 + c] * gt[2]);
        for (int r = 0; r < 3; ++r)
          for (int c = 0; c < 3; ++c) s_gR[i][r * 3 + c] = gR[r * 3 + c] - gt[r] * f.j[i][c];
      }
    }
  } else {
    for (int vtx = tid - 32; vtx < V; vtx += THREADS - 32) {
      const float4* w4 = reinterpret_cast<const float4*>(mc.weights + (size_t)vtx * 16);
      float w[16];
#pragma unroll
      for (int i = 0; i < 4; ++i) { float4 t = __ldg(w4 + i); w[4 * i] = t.x; w[4 * i + 1] = t.y; w[4 * i + 2] = t.z; w[4 * i + 3] = t.w; }
      float T[9];
#pragma unroll
      for (int e = 0; e < 9; ++e) T[e] = 0.f;
#pragma unroll
      for (int jt = 0; jt < 16; ++jt)
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
          for (int c = 0; c < 3; ++c) T[r * 3 + c] = fmaf(w[jt], f.T[jt][r * 4 + c], T[r * 3 + c]);
      const float gx = s_g[vtx * 3], gy = s_g[vtx * 3 + 1], gz = s_g[vtx * 3 + 2];
      s_g[vtx * 3] = T[0] * gx + T[3] * gy + T[6] * gz;
      s_g[vtx * 3 + 1] = T[1] * gx + T[4] * gy + T[7] * gz;
      s_g[vtx * 3 + 2] = T[2] * gx + T[5] * gy + T[8] * gz;
    }
  }
  __syncthreads();
  // ================= B5a: pose blend rows (warp per k)
  for (int k = warp; k < 135; k += NWARPS) {
    float acc = 0.f;
    const float* row = mc.posedirsT + (size_t)k * V3;
    for (int o = lane; o < V3; o += 32) acc = fmaf(__ldg(row + o), s_g[o], acc);
    acc = warp_sum(acc);
    if (lane == 0) s_gps[k] = acc;
  }
  __syncthreads();
  if (tid < 135) s_gR[1 + tid / 9][tid % 9] += s_gps[tid];
  // ================= B5b: g_vshaped = g_vposed + Jreg^T g_j
  for (int o = tid; o < V3; o += THREADS) {
    const int vtx = o / 3, c = o - vtx * 3;
    float acc = s_g[o];
#pragma unroll
    for (int jt = 0; jt < 16; ++jt) acc = fmaf(__ldg(mc.jreg + jt * V + vtx), s_gj[jt][c], acc);
    s_g[o] = acc;
  }
  __syncthreads();
  // ================= B5c: shape blend (warps 0..9) || B6: quaternions (warp 10)
  if (warp < 10) {
    if (d_betas_rows) {
      float acc = 0.f;
      const float* row = mc.shapedirsT + (size_t)warp * V3;
      for (int o = lane; o < V3; o += 32) acc = fmaf(__ldg(row + o), s_g[o], acc);
      acc = warp_sum(acc);
      if (lane == 0) d_betas_rows[(size_t)b * 10 + warp] = acc;
    }
  } else if (warp == 10 && lane < 16 && d_quat) {
    // R = M(q) / n, n = |q|^2:  dL/dq = sum_ab gR_ab (dM_ab/dq) / n - 2 q (sum_ab gR_ab R_ab) / n
    const float* g = s_gR[lane];
    const float* R = f.R[lane];
    const float w = f.q[lane][0], x = f.q[lane][1], y = f.q[lane][2], z = f.q[lane][3];
    const float n = w * w + x * x + y * y + z * z;
    float gRR = 0.f;
    for (int e = 0; e < 9; ++e) gRR += g[e] * R[e];
    const float dw = 2.f * (w * (g[0] + g[4] + g[8]) + z * (g[3] - g[1]) + y * (g[2] - g[6]) + x * (g[7] - g[5]));
    const float dx = 2.f * (x * (g[0] - g[4] - g[8]) + y * (g[1] + g[3]) + z * (g[2] + g[6]) + w * (g[7] - g[5]));
    const float dy = 2.f * (y * (-g[0] + g[4] - g[8]) + x * (g[1] + g[3]) + z * (g[5] + g[7]) + w * (g[2] - g[6]));
    const float dz = 2.f * (z * (-g[0] - g[4] + g[8]) + x * (g[2] + g[6]) + y * (g[5] + g[7]) + w * (g[3] - g[1]));
    const float s = side ? -1.f : 1.f;          // left hands: q.y, q.z were negated before the conversion
    float* d = d_quat + (size_t)b * 64 + lane * 4;
    d[0] = (dw - 2.f * w * gRR) / n;
    d[1] = (dx - 2.f * x * gRR) / n;
    d[2] = s * (dy - 2.f * y * gRR) / n;
    d[3] = s * (dz - 2.f * z * gRR) / n;
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

ManopthConsts consts(const float* const* p) { return ManopthConsts{p[0], p[1], p[2], p[3], p[4]}; }

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
  launch_k(manopth_fwd_kernel, B, THREADS, 0, s, consts(const_ptrs), quat, betas, betas_shared, trans, translate, center_idx, root_palm, side,
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
  launch_k(manopth_bwd_kernel, B, THREADS, 0, s, consts(const_ptrs), quat, betas, betas_shared, trans, translate, center_idx, root_palm, side,
           g_verts, g_joints, g_transf, d_quat, rows, d_trans);
  if (int e = check_launch("manopth_bwd")) return e;
  if (d_betas && betas_shared) {
    launch_k(manopth_betas_reduce_kernel, 1, 320, 0, s, (const float*)work, B, d_betas);
    return check_launch("manopth_betas_reduce");
  }
  return 0;
}
