// The MANO stages shared by the axis-angle ManoLayer (mano.cu) and the pose optimiser's quaternion manopth ManoLayer (manopth.cu):
// shape blend, joint regression, the pose feature vec(R - I), the kinematic chain, pose blend and linear-blend skinning, and their
// adjoints.  One CTA of MANO_THREADS threads runs one hand; its state lives in shared memory.  The layers differ only in where the joint
// rotations come from and in what they do with the outputs, which stays in their own files.  Every sum runs in a fixed order and no stage
// uses float atomics, so results are bitwise reproducible.
#pragma once
#include "common.cuh"

namespace rih {

// The backward's skinning adjoint maps warp i to joint i: 16 warps.
constexpr int MANO_V = 778, MANO_V3 = 2334, MANO_THREADS = 512, MANO_WARPS = MANO_THREADS / 32;

struct ManoTables {
  const float* shapedirsT;  // [10][2334]
  const float* posedirsT;   // [135][2334]
  const float* v_template;  // [2334]
  const float* jreg;        // [16,778]
  const float* weights;     // [778,16]
};

// Forward state of one hand.
struct ManoState {
  float vt[MANO_V3];   // v_shaped -> v_posed
  float R[16][9];      // joint rotations, 0 = root
  float ps[136];       // vec(R - I) of joints 1..15
  float beta[10];
  float j[16][3];      // rest joints J_regressor @ v_shaped
  float t[16][3];      // local translations (I - R_i) j_i
  float T[16][12];     // skinning transforms A_i = [G_i.R | G_i.t - G_i.R j_i], top three rows
  float gt[16][3];     // global joint translations G_i.t, native order
};

// Gradients of the backward's middle stages.
struct ManoGrad {
  float gj[16][3];     // rest joints
  float gG[16][12];    // skinning transforms
  float gR[16][9];     // joint rotations
};

// Shape blend, joint regression, pose feature, chain and pose blend: f.vt ends as v_posed, f.T / f.gt hold the chain.
// On entry f.beta, and whatever `rotations` reads, are written behind a __syncthreads().  `rotations(lane)` runs on warp 0 while warps
// 1.. regress the joints and must leave f.R[0..15] complete.  parent[i] < i for i > 0.  Ends with a __syncthreads().
template <class Rotations>
__device__ __forceinline__ void mano_forward_state(ManoState& f, const ManoTables& mt, const int* parent, int tid, Rotations rotations) {
  const int warp = tid >> 5, lane = tid & 31;
  for (int o = tid; o < MANO_V3; o += MANO_THREADS) {
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < 10; ++i) acc = fmaf(mt.shapedirsT[i * MANO_V3 + o], f.beta[i], acc);
    f.vt[o] = mt.v_template[o] + acc;
  }
  __syncthreads();
  if (warp == 0) {
    rotations(lane);
    __syncwarp();
    for (int k = lane; k < 135; k += 32) { const int e = k % 9; f.ps[k] = f.R[1 + k / 9][e] - ((e == 0 || e == 4 || e == 8) ? 1.f : 0.f); }
  } else {
    for (int o = warp - 1; o < 48; o += MANO_WARPS - 1) {
      const int jt = o / 3, c = o % 3;
      float acc = 0.f;
      for (int vtx = lane; vtx < MANO_V; vtx += 32) acc = fmaf(mt.jreg[jt * MANO_V + vtx], f.vt[vtx * 3 + c], acc);
      acc = warp_sum(acc);
      if (lane == 0) f.j[jt][c] = acc;
    }
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
          const float* P = f.T[parent[i]];
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
    for (int o = tid - 32; o < MANO_V3; o += MANO_THREADS - 32) {
      float acc = 0.f;
#pragma unroll 9
      for (int i = 0; i < 135; ++i) acc = fmaf(mt.posedirsT[i * MANO_V3 + o], f.ps[i], acc);
      f.vt[o] += acc;
    }
  }
  __syncthreads();
}

// Linear-blend skinning of vertex vtx: out[vtx] = (sum_i w[vtx,i] A_i) [v_posed; 1].  out may be f.vt.
__device__ __forceinline__ void mano_skin(const ManoState& f, const ManoTables& mt, int vtx, float* out) {
  const float4* w4 = reinterpret_cast<const float4*>(mt.weights + (size_t)vtx * 16);
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

// Backward of mano_forward_state and the skinning, from the gradients on the skinned vertices (g [2334], shared) and on the 16 native
// joint positions G_i.t (gjo), plus an optional gradient gA on the transforms A_i ([16][4][4] row-major; only the rotation blocks are
// read, NULL = none).  gs.gR receives the rotation gradients and g is overwritten with the gradient on v_shaped, for mano_shape_row.
// Ends with a __syncthreads().
//   B3a gA_i = sum_v w[v,i] g_v (x) [v_posed; 1]  (warp i <-> joint i)
//   B3b g_vposed = T_v.R^T g_v  (warps 1..)  ||  B4 global joints and chain backward, children before parents (thread 0)
//   B5a pose blend rows (warp per row) into gR ; B5b g_vshaped = g_vposed + Jreg^T g_j
__device__ __forceinline__ void mano_backward(const ManoState& f, const ManoTables& mt, const int* parent, float* g, const float (*gjo)[3],
                                              const float* gA, ManoGrad& gs, int tid) {
  const int warp = tid >> 5, lane = tid & 31;
  {
    const int jt = warp;
    float a[12];
#pragma unroll
    for (int e = 0; e < 12; ++e) a[e] = 0.f;
    for (int vtx = lane; vtx < MANO_V; vtx += 32) {
      const float w = __ldg(mt.weights + (size_t)vtx * 16 + jt);
      const float gx = w * g[vtx * 3], gy = w * g[vtx * 3 + 1], gz = w * g[vtx * 3 + 2];
      const float x = f.vt[vtx * 3], y = f.vt[vtx * 3 + 1], z = f.vt[vtx * 3 + 2];
      a[0] = fmaf(gx, x, a[0]); a[1] = fmaf(gx, y, a[1]); a[2] = fmaf(gx, z, a[2]); a[3] += gx;
      a[4] = fmaf(gy, x, a[4]); a[5] = fmaf(gy, y, a[5]); a[6] = fmaf(gy, z, a[6]); a[7] += gy;
      a[8] = fmaf(gz, x, a[8]); a[9] = fmaf(gz, y, a[9]); a[10] = fmaf(gz, z, a[10]); a[11] += gz;
    }
#pragma unroll
    for (int e = 0; e < 12; ++e) a[e] = warp_sum(a[e]);
    if (lane == 0) {
#pragma unroll
      for (int e = 0; e < 12; ++e) gs.gG[jt][e] = (gA && (e & 3) != 3) ? a[e] + gA[jt * 16 + e] : a[e];   // A_i.R = G_i.R
    }
  }
  __syncthreads();
  if (warp == 0) {
    if (lane == 0) {
      // global joints: G_0.t = j_0 ; G_i.t = A_p.R j_i + A_p.t
      for (int c = 0; c < 3; ++c) gs.gj[0][c] = gjo[0][c];
      for (int i = 1; i < 16; ++i) {
        const int p = parent[i];
        const float* P = f.T[p];
        const float gv[3] = {gjo[i][0], gjo[i][1], gjo[i][2]};
        for (int c = 0; c < 3; ++c) gs.gj[i][c] = P[0 * 4 + c] * gv[0] + P[1 * 4 + c] * gv[1] + P[2 * 4 + c] * gv[2];
        for (int r = 0; r < 3; ++r) {
          gs.gG[p][r * 4 + 0] += gv[r] * f.j[i][0]; gs.gG[p][r * 4 + 1] += gv[r] * f.j[i][1]; gs.gG[p][r * 4 + 2] += gv[r] * f.j[i][2];
          gs.gG[p][r * 4 + 3] += gv[r];
        }
      }
      // chain: A_i.R = A_p.R R_i ; A_i.t = A_p.R t_i + A_p.t  (children carry larger indices than their parents)
      for (int i = 15; i >= 0; --i) {
        const float* gG = gs.gG[i];
        const float* R = f.R[i];
        float gR[9], gt[3];
        if (i > 0) {
          const int p = parent[i];
          const float* P = f.T[p];
          float* gP = gs.gG[p];
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
        for (int c = 0; c < 3; ++c) gs.gj[i][c] += gt[c] - (R[0 * 3 + c] * gt[0] + R[1 * 3 + c] * gt[1] + R[2 * 3 + c] * gt[2]);
        for (int r = 0; r < 3; ++r)
          for (int c = 0; c < 3; ++c) gs.gR[i][r * 3 + c] = gR[r * 3 + c] - gt[r] * f.j[i][c];
      }
    }
  } else {
    for (int vtx = tid - 32; vtx < MANO_V; vtx += MANO_THREADS - 32) {
      const float4* w4 = reinterpret_cast<const float4*>(mt.weights + (size_t)vtx * 16);
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
      const float gx = g[vtx * 3], gy = g[vtx * 3 + 1], gz = g[vtx * 3 + 2];
      g[vtx * 3] = T[0] * gx + T[3] * gy + T[6] * gz;
      g[vtx * 3 + 1] = T[1] * gx + T[4] * gy + T[7] * gz;
      g[vtx * 3 + 2] = T[2] * gx + T[5] * gy + T[8] * gz;
    }
  }
  __syncthreads();
  for (int k = warp; k < 135; k += MANO_WARPS) {
    float acc = 0.f;
    const float* row = mt.posedirsT + (size_t)k * MANO_V3;
    for (int o = lane; o < MANO_V3; o += 32) acc = fmaf(__ldg(row + o), g[o], acc);
    acc = warp_sum(acc);
    if (lane == 0) gs.gR[1 + k / 9][k % 9] += acc;
  }
  __syncthreads();
  for (int o = tid; o < MANO_V3; o += MANO_THREADS) {
    const int vtx = o / 3, c = o - vtx * 3;
    float acc = g[o];
#pragma unroll
    for (int jt = 0; jt < 16; ++jt) acc = fmaf(__ldg(mt.jreg + jt * MANO_V + vtx), gs.gj[jt][c], acc);
    g[o] = acc;
  }
  __syncthreads();
}

// B5c: shape-blend row k, <shapedirsT[k], g_vshaped> for g as mano_backward leaves it (one warp; lane 0 writes *d).
__device__ __forceinline__ void mano_shape_row(const ManoTables& mt, const float* g, int k, int lane, float* d) {
  float acc = 0.f;
  const float* row = mt.shapedirsT + (size_t)k * MANO_V3;
  for (int o = lane; o < MANO_V3; o += 32) acc = fmaf(__ldg(row + o), g[o], acc);
  acc = warp_sum(acc);
  if (lane == 0) *d = acc;
}

}  // namespace rih
