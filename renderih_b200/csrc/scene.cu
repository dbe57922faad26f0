// The mocap driver's scene preparation on the device (pose_data_optimize/batch_optimize_mocap_origin.py): update_scene's anchor and normal
// geometry (:256-270) and search_anchors (:62-130) for a whole batch of frames in one launch, one CTA per frame and one thread per anchor.
//
// Every floating-point operation is an explicit _rn intrinsic so that nvcc cannot contract it into an FMA: the results are the ones numpy
// computes in the same order (float32 normals, float64 anchors and distances), which oracle/mocap_ref.py restates bit for bit.
#include "common.cuh"
using namespace rih;

namespace {

constexpr int SCENE_MAX_ANCHORS = 128;
constexpr int SCENE_DIM = 4;                    // search_anchors' `dim`

struct Geo {
  double a[3];        // recover_anchor (anchorutils.py:51-62), float64
  float n[3];         // the unnormalised-then-divided face normal, float32
};

// One anchor of one hand: the face's vertices plus the translation (float32, :256-257), the anchor v0 + (w1 (v1 - v0) + w2 (v2 - v0)) with
// float32 edges and float64 weights, and the face normal cross(v1 - v0, v2 - v0) / |.| (numpy's cross, then norm, then divide).
__device__ __forceinline__ Geo anchor_geo(const float* __restrict__ verts, const float* __restrict__ tsl, const int* __restrict__ fvi,
                                          const double* __restrict__ aw, int a) {
  float v[3][3];
  for (int k = 0; k < 3; ++k) {
    const int vi = fvi[a * 3 + k];
    for (int c = 0; c < 3; ++c) v[k][c] = __fadd_rn(verts[vi * 3 + c], tsl[c]);
  }
  float e1[3], e2[3];
  for (int c = 0; c < 3; ++c) {
    e1[c] = __fsub_rn(v[1][c], v[0][c]);
    e2[c] = __fsub_rn(v[2][c], v[0][c]);
  }
  const double w1 = aw[a * 2], w2 = aw[a * 2 + 1];
  Geo g;
  for (int c = 0; c < 3; ++c)
    g.a[c] = __dadd_rn(__dadd_rn(__dmul_rn(w1, (double)e1[c]), __dmul_rn(w2, (double)e2[c])), (double)v[0][c]);
  const float c0 = __fsub_rn(__fmul_rn(e1[1], e2[2]), __fmul_rn(e1[2], e2[1]));
  const float c1 = __fsub_rn(__fmul_rn(e1[2], e2[0]), __fmul_rn(e1[0], e2[2]));
  const float c2 = __fsub_rn(__fmul_rn(e1[0], e2[1]), __fmul_rn(e1[1], e2[0]));
  const float nrm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(c0, c0), __fmul_rn(c1, c1)), __fmul_rn(c2, c2)));
  g.n[0] = __fdiv_rn(c0, nrm);
  g.n[1] = __fdiv_rn(c1, nrm);
  g.n[2] = __fdiv_rn(c2, nrm);
  return g;
}

// |s - m| in float64: the differences squared, summed left to right, square-rooted (np.linalg.norm over the last axis of length 3).
__device__ __forceinline__ double dist(const double* s, const double* m) {
  const double d0 = __dsub_rn(s[0], m[0]), d1 = __dsub_rn(s[1], m[1]), d2 = __dsub_rn(s[2], m[2]);
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(d0, d0), __dmul_rn(d1, d1)), __dmul_rn(d2, d2)));
}

// contact_able * (0.5 cos(pi d / t) + 0.5), rounded to float32 as the float32 anchor_elasti array stores it (:86, :103, :121).
__device__ __forceinline__ float elasticity(double d, double t) {
  if (!(d < t)) return 0.f;
  return (float)__dadd_rn(__dmul_rn(0.5, cos(__ddiv_rn(__dmul_rn(3.141592653589793, d), t))), 0.5);
}

// grid = B frames, block = 128 threads; thread a handles sub (left) anchor a.  prev_id == nullptr selects the fresh branch.
__global__ void __launch_bounds__(SCENE_MAX_ANCHORS) scene_search_anchors_kernel(
    const float* __restrict__ verts_main, const float* __restrict__ verts_sub, const float* __restrict__ tsl_main,
    const float* __restrict__ tsl_sub, const int* __restrict__ fvi, const double* __restrict__ aw, const int* __restrict__ cls, int A,
    const long long* __restrict__ prev_id, long long* __restrict__ anchor_id, float* __restrict__ anchor_elasti,
    long long* __restrict__ padding_mask, long long* __restrict__ vertex_contact, bool* __restrict__ optimize_it,
    float* __restrict__ sub_anchors, float* __restrict__ sub_normals) {
  __shared__ double s_anchor[SCENE_MAX_ANCHORS][3];
  __shared__ float s_normal[SCENE_MAX_ANCHORS][3];
  pdl_sync();
  const int b = blockIdx.x, a = threadIdx.x;
  const long long vo = (long long)b * 778 * 3;
  Geo sub;
  if (a < A) {
    const Geo m = anchor_geo(verts_main + vo, tsl_main + b * 3, fvi, aw, a);
    sub = anchor_geo(verts_sub + vo, tsl_sub + b * 3, fvi, aw, a);
    for (int c = 0; c < 3; ++c) {
      s_anchor[a][c] = m.a[c];
      s_normal[a][c] = m.n[c];
      sub.n[c] = -sub.n[c];                                               // obj_normals = -cross / norm (:266)
      sub_anchors[((long long)b * A + a) * 3 + c] = (float)sub.a[c];
      sub_normals[((long long)b * A + a) * 3 + c] = sub.n[c];
    }
  }
  __syncthreads();
  int contact = 0;
  if (a < A) {
    int id[SCENE_DIM];
    float el[SCENE_DIM];
    const long long o = ((long long)b * A + a) * SCENE_DIM;
    if (prev_id) {                    // :75-91: distances at the given ids only, no `against` mask, threshold 0.02
#pragma unroll
      for (int k = 0; k < SCENE_DIM; ++k) {
        id[k] = (int)prev_id[o + k];
        const double d = dist(sub.a, s_anchor[id[k]]);
        el[k] = elasticity(d, 0.02);
        contact |= d < 0.02;
      }
    } else {                          // :116-127: masked distances are 1000; the 4 smallest, ties to the lowest index
      double best[SCENE_DIM];
#pragma unroll
      for (int k = 0; k < SCENE_DIM; ++k) best[k] = INFINITY, id[k] = 0;
      for (int j = 0; j < A; ++j) {
        const float dot = __fadd_rn(__fadd_rn(__fmul_rn(sub.n[0], s_normal[j][0]), __fmul_rn(sub.n[1], s_normal[j][1])),
                                    __fmul_rn(sub.n[2], s_normal[j][2]));
        const double d = dot > -0.6f ? 1000.0 : dist(sub.a, s_anchor[j]);
        contact |= d < 0.015;
        if (d < best[SCENE_DIM - 1]) {          // strict: an equal distance keeps the earlier (lower) index ahead of it
          best[SCENE_DIM - 1] = d, id[SCENE_DIM - 1] = j;
#pragma unroll
          for (int k = SCENE_DIM - 1; k > 0; --k) {
            if (best[k] < best[k - 1]) {
              const double td = best[k]; best[k] = best[k - 1]; best[k - 1] = td;
              const int ti = id[k]; id[k] = id[k - 1]; id[k - 1] = ti;
            }
          }
        }
      }
#pragma unroll
      for (int k = 0; k < SCENE_DIM; ++k) el[k] = elasticity(best[k], 0.015);
    }
    // :129 -- the elasticity is scaled by 0.3 unless this anchor's or the partner's class is 4
#pragma unroll
    for (int k = 0; k < SCENE_DIM; ++k) {
      const float e = (cls[a] != 4 && cls[id[k]] != 4) ? __fmul_rn(el[k], 0.3f) : el[k];
      anchor_id[o + k] = id[k];
      anchor_elasti[o + k] = e;
      padding_mask[o + k] = el[k] > 0.f;
    }
    vertex_contact[(long long)b * A + a] = contact;
  }
  const int any = __syncthreads_or(contact);
  if (a == 0) optimize_it[b] = any != 0;                                   // :533-538
}

}  // namespace

// search_anchors + update_scene's geometry (batch_optimize_mocap_origin.py:62-130, :256-273) for B frames.  verts_main / verts_sub [B,778,3]
// are the centred MANO vertices of the main (right) and sub (left) hand, tsl_main / tsl_sub [B,3] their translations (float32).  fvi [A,3]
// (int32), aw [A,2] (float64) and cls [A] (int32) are face_vertex_idx, anchor_weight and merged_vertex_assignment, A <= 128.  prev_id
// [B,A,4] (int64, each in [0,A)) selects the previous-id branch, NULL the fresh one.  Writes anchor_id / padding_mask [B,A,4] (int64),
// anchor_elasti [B,A,4] (float32), vertex_contact [B,A] (int64), optimize_it [B] (bool), sub_anchors / sub_normals [B,A,3] (float32).
RIH_API int rih_mocap_search_anchors(const float* verts_main, const float* verts_sub, const float* tsl_main, const float* tsl_sub, const int* fvi,
                                     const double* aw, const int* cls, int A, const long long* prev_id, int B, long long* anchor_id,
                                     float* anchor_elasti, long long* padding_mask, long long* vertex_contact, bool* optimize_it,
                                     float* sub_anchors, float* sub_normals, cudaStream_t s) {
  RIH_REQUIRE(B >= 1 && A >= SCENE_DIM && A <= SCENE_MAX_ANCHORS, "mocap_search_anchors: B >= 1 and %d <= A <= %d (got B=%d A=%d)", SCENE_DIM,
              SCENE_MAX_ANCHORS, B, A);
  launch_k(scene_search_anchors_kernel, B, SCENE_MAX_ANCHORS, 0, s, verts_main, verts_sub, tsl_main, tsl_sub, fvi, aw, cls, A, prev_id, anchor_id,
           anchor_elasti, padding_mask, vertex_contact, optimize_it, sub_anchors, sub_normals);
  return check_launch("mocap_search_anchors");
}
