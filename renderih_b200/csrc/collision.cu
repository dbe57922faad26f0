// Two-hand mesh collision count: the contact stage of the pose data pipeline's collision filter (pose_data_optimize/collision/
// CollisionFilter.py:93-124, CollisionCheck.py), for every frame of a batch in one launch.  For each frame the kernel counts the
// (face of hand A, face of hand B) pairs whose closed triangles intersect.
//
// The narrow phase is Guigue and Devillers' triangle-triangle test ("Faster triangle-triangle intersection tests", 2002/2003): signs of
// 3x3 orientation determinants, and for exactly coplanar pairs its 2-D branch on the projection that keeps the larger normal component.
// Every determinant is evaluated in float64 by one fixed formula with explicit _rn intrinsics, so nvcc cannot contract anything into an
// FMA: oracle/collision_ref.py performs the same IEEE operations in the same order and the counts agree exactly.  A face whose computed
// normal is exactly (0, 0, 0) has zero area and intersects nothing.
//
// Broad phase, one CTA per frame: the float64 coordinates of both hands go to shared memory; both hands' boxes come from a block
// reduction; each hand's faces are compacted to those whose box overlaps the other hand's box; then each thread takes one compacted face
// of hand B and sweeps the compacted faces of hand A, box test first, exact test on overlap.  Every box is float32 rounded outward
// (__double2float_rd / _ru) and the overlap tests are closed, so the culling never drops a pair the exact test accepts.
#include "common.cuh"
using namespace rih;

namespace {

constexpr int COL_THREADS = 256;
constexpr int COL_MAX_V = 1024;
constexpr int COL_MAX_F = 2048;

struct D3 { double x, y, z; };

__device__ __forceinline__ D3 sub(const D3& a, const D3& b) { return {__dsub_rn(a.x, b.x), __dsub_rn(a.y, b.y), __dsub_rn(a.z, b.z)}; }
__device__ __forceinline__ D3 cross(const D3& a, const D3& b) {
  return {__dsub_rn(__dmul_rn(a.y, b.z), __dmul_rn(a.z, b.y)), __dsub_rn(__dmul_rn(a.z, b.x), __dmul_rn(a.x, b.z)),
          __dsub_rn(__dmul_rn(a.x, b.y), __dmul_rn(a.y, b.x))};
}
__device__ __forceinline__ double dot(const D3& a, const D3& b) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a.x, b.x), __dmul_rn(a.y, b.y)), __dmul_rn(a.z, b.z));
}
__device__ __forceinline__ int sgn(double d) { return (d > 0.0) - (d < 0.0); }

// (a - c) x (b - c) in 2-D
__device__ __forceinline__ double orient2d(const double* a, const double* b, const double* c) {
  return __dsub_rn(__dmul_rn(__dsub_rn(a[0], c[0]), __dsub_rn(b[1], c[1])), __dmul_rn(__dsub_rn(a[1], c[1]), __dsub_rn(b[0], c[0])));
}

// INTERSECTION_TEST_VERTEX of the 2-D test
__device__ bool test_vertex(const double* P1, const double* Q1, const double* R1, const double* P2, const double* Q2, const double* R2) {
  if (orient2d(R2, P2, Q1) >= 0.0) {
    if (orient2d(R2, Q2, Q1) <= 0.0) {
      if (orient2d(P1, P2, Q1) > 0.0) return orient2d(P1, Q2, Q1) <= 0.0;
      return orient2d(P1, P2, R1) >= 0.0 && orient2d(Q1, R1, P2) >= 0.0;
    }
    return orient2d(P1, Q2, Q1) <= 0.0 && orient2d(R2, Q2, R1) <= 0.0 && orient2d(Q1, R1, Q2) >= 0.0;
  }
  if (orient2d(R2, P2, R1) >= 0.0) {
    if (orient2d(Q1, R1, R2) >= 0.0) return orient2d(P1, P2, R1) >= 0.0;
    return orient2d(Q1, R1, Q2) >= 0.0 && orient2d(R2, R1, Q2) >= 0.0;
  }
  return false;
}

// INTERSECTION_TEST_EDGE of the 2-D test
__device__ bool test_edge(const double* P1, const double* Q1, const double* R1, const double* P2, const double* /*Q2*/, const double* R2) {
  if (orient2d(R2, P2, Q1) >= 0.0) {
    if (orient2d(P1, P2, Q1) >= 0.0) return orient2d(P1, Q1, R2) >= 0.0;
    return orient2d(Q1, R1, P2) >= 0.0 && orient2d(R1, P1, P2) >= 0.0;
  }
  if (orient2d(R2, P2, R1) >= 0.0) {
    if (orient2d(P1, P2, R1) < 0.0) return false;
    return orient2d(P1, R1, R2) >= 0.0 || orient2d(Q1, R1, R2) >= 0.0;
  }
  return false;
}

// ccw_tri_tri_intersection_2d: both triangles counter-clockwise
__device__ bool ccw_2d(const double* p1, const double* q1, const double* r1, const double* p2, const double* q2, const double* r2) {
  if (orient2d(p2, q2, p1) >= 0.0) {
    if (orient2d(q2, r2, p1) >= 0.0) {
      if (orient2d(r2, p2, p1) >= 0.0) return true;
      return test_edge(p1, q1, r1, p2, q2, r2);
    }
    if (orient2d(r2, p2, p1) >= 0.0) return test_edge(p1, q1, r1, r2, p2, q2);
    return test_vertex(p1, q1, r1, p2, q2, r2);
  }
  if (orient2d(q2, r2, p1) >= 0.0) {
    if (orient2d(r2, p2, p1) >= 0.0) return test_edge(p1, q1, r1, q2, r2, p2);
    return test_vertex(p1, q1, r1, q2, r2, p2);
  }
  return test_vertex(p1, q1, r1, r2, p2, q2);
}

// coplanar_tri_tri3d: project on the axis plane that drops the largest |N1| component, orient both triangles counter-clockwise, 2-D test.
__device__ __noinline__ bool coplanar(const D3* t1, const D3* t2, D3 n) {
  const double nx = fabs(n.x), ny = fabs(n.y), nz = fabs(n.z);
  double a[6][2];      // P1 Q1 R1 P2 Q2 R2
  const D3* src[6] = {&t1[0], &t1[1], &t1[2], &t2[0], &t2[1], &t2[2]};
  if (nx > nz && nx >= ny) {           // YZ, with p and q exchanged
    for (int k = 0; k < 6; ++k) { const D3& s = *src[(k % 3 == 2) ? k : (k % 3 == 0 ? k + 1 : k - 1)]; a[k][0] = s.z; a[k][1] = s.y; }
  } else if (ny > nz && ny >= nx) {    // XZ, with p and q exchanged
    for (int k = 0; k < 6; ++k) { const D3& s = *src[(k % 3 == 2) ? k : (k % 3 == 0 ? k + 1 : k - 1)]; a[k][0] = s.x; a[k][1] = s.z; }
  } else {                             // XY
    for (int k = 0; k < 6; ++k) { a[k][0] = src[k]->x; a[k][1] = src[k]->y; }
  }
  const double *p1 = a[0], *q1 = a[1], *r1 = a[2], *p2 = a[3], *q2 = a[4], *r2 = a[5];
  if (orient2d(p1, q1, r1) < 0.0) { const double* t = q1; q1 = r1; r1 = t; }
  if (orient2d(p2, q2, r2) < 0.0) { const double* t = q2; q2 = r2; r2 = t; }
  return ccw_2d(p1, q1, r1, p2, q2, r2);
}

// The permutation rule shared by both levels of the 3-D test: from the signs of one triangle's vertices against the other's plane, the
// rotation that puts the lone vertex first (0: pqr, 1: qrp, 2: rpq) and whether the other triangle's last two vertices swap.
// Returns false when all three signs are zero (coplanar).
__device__ __forceinline__ bool order(int sp, int sq, int sr, int& rot, bool& swp) {
  if (sp > 0) {
    if (sq > 0) { rot = 2; swp = true; } else if (sr > 0) { rot = 1; swp = true; } else { rot = 0; swp = false; }
  } else if (sp < 0) {
    if (sq < 0) { rot = 2; swp = false; } else if (sr < 0) { rot = 1; swp = false; } else { rot = 0; swp = true; }
  } else if (sq < 0) {
    if (sr >= 0) { rot = 1; swp = true; } else { rot = 0; swp = false; }
  } else if (sq > 0) {
    if (sr > 0) { rot = 0; swp = true; } else { rot = 1; swp = false; }
  } else {
    if (sr > 0) { rot = 2; swp = false; } else if (sr < 0) { rot = 2; swp = true; } else return false;
  }
  return true;
}

__device__ __forceinline__ bool is_zero(const D3& n) { return n.x == 0.0 && n.y == 0.0 && n.z == 0.0; }

// tri_tri_overlap_test_3d on closed triangles t1 = (p1, q1, r1), t2 = (p2, q2, r2).
__device__ __noinline__ bool tri_tri(const D3* t1, const D3* t2) {
  const D3 n1 = cross(sub(t1[0], t1[2]), sub(t1[1], t1[2]));
  const D3 n2 = cross(sub(t2[0], t2[2]), sub(t2[1], t2[2]));
  if (is_zero(n1) || is_zero(n2)) return false;
  int s1[3], s2[3];
  for (int k = 0; k < 3; ++k) s1[k] = sgn(dot(sub(t1[k], t2[2]), n2));
  if (s1[0] == s1[1] && s1[0] == s1[2] && s1[0] != 0) return false;
  for (int k = 0; k < 3; ++k) s2[k] = sgn(dot(sub(t2[k], t1[2]), n1));
  if (s2[0] == s2[1] && s2[0] == s2[2] && s2[0] != 0) return false;
  int rot;
  bool swp;
  if (!order(s1[0], s1[1], s1[2], rot, swp)) return coplanar(t1, t2, n1);
  D3 a[3], b[3];
  for (int k = 0; k < 3; ++k) a[k] = t1[(k + rot) % 3];
  int i2[3] = {0, 1, 2};
  if (swp) { i2[1] = 2; i2[2] = 1; }
  if (!order(s2[i2[0]], s2[i2[1]], s2[i2[2]], rot, swp)) return coplanar(t1, t2, n1);
  for (int k = 0; k < 3; ++k) b[k] = t2[i2[(k + rot) % 3]];
  if (swp) { const D3 t = a[1]; a[1] = a[2]; a[2] = t; }
  // CHECK_MIN_MAX(p1, q1, r1, p2, q2, r2)
  if (dot(sub(b[1], a[1]), cross(sub(b[0], a[1]), sub(a[0], a[1]))) > 0.0) return false;
  return !(dot(sub(b[2], a[0]), cross(sub(b[0], a[0]), sub(a[2], a[0]))) > 0.0);
}

__device__ __forceinline__ D3 vert(const double* X, int v) { return {X[v * 3], X[v * 3 + 1], X[v * 3 + 2]}; }

// Face box rounded outward to float32: lo / hi of the face's three float64 vertices.
__device__ __forceinline__ void face_box(const double* X, int a, int b, int c, float* lo, float* hi) {
  for (int k = 0; k < 3; ++k) {
    const double u = X[a * 3 + k], v = X[b * 3 + k], w = X[c * 3 + k];
    lo[k] = __double2float_rd(fmin(fmin(u, v), w));
    hi[k] = __double2float_ru(fmax(fmax(u, v), w));
  }
}

__device__ __forceinline__ bool overlap(const float* alo, const float* ahi, const float* blo, const float* bhi) {
  return alo[0] <= bhi[0] && blo[0] <= ahi[0] && alo[1] <= bhi[1] && blo[1] <= ahi[1] && alo[2] <= bhi[2] && blo[2] <= ahi[2];
}

size_t col_smem(int V, int F) { return (size_t)V * 6 * sizeof(double) + (size_t)F * (2 * sizeof(float4) + sizeof(int)); }

// grid = B frames, block = COL_THREADS.  Shared: X[2][V*3] doubles, A-face boxes (lo.w = face index) and the compacted B faces.
template <typename T>
__global__ void __launch_bounds__(COL_THREADS) collision_count_kernel(const T* __restrict__ va, const T* __restrict__ vb,
                                                                      const double* __restrict__ ta, const double* __restrict__ tb,
                                                                      const int* __restrict__ faces, int V, int F,
                                                                      long long* __restrict__ count, long long* __restrict__ stats) {
  extern __shared__ __align__(16) unsigned char col_smem_raw[];
  float4* a_lo = reinterpret_cast<float4*>(col_smem_raw);
  float4* a_hi = a_lo + F;
  double* X = reinterpret_cast<double*>(a_hi + F);           // hand A at X, hand B at X + 3V
  int* b_list = reinterpret_cast<int*>(X + 6 * V);
  __shared__ float s_box[COL_THREADS / 32][12];              // per warp: lo A, hi A, lo B, hi B
  __shared__ float h_box[12];
  __shared__ int s_na, s_nb, s_bad, s_hits;
  __shared__ unsigned long long s_exact;
  pdl_sync();
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) { s_na = 0; s_nb = 0; s_bad = 0; s_hits = 0; s_exact = 0; }

  // float64 coordinates (vertex + translation, added in float64) and the hands' outward-rounded boxes
  float bx[12];
  for (int k = 0; k < 3; ++k) { bx[k] = bx[6 + k] = INFINITY; bx[3 + k] = bx[9 + k] = -INFINITY; }
  const long long vo = (long long)b * V * 3;
  for (int i = tid; i < 2 * V * 3; i += COL_THREADS) {
    const int h = i >= V * 3, o = i - h * V * 3;
    const double* t = h ? tb : ta;
    double x = (double)(h ? vb : va)[vo + o];
    if (t) x = __dadd_rn(x, t[b * 3 + o % 3]);
    X[i] = x;
    const int k = h * 6 + o % 3;
    bx[k] = fminf(bx[k], __double2float_rd(x));
    bx[k + 3] = fmaxf(bx[k + 3], __double2float_ru(x));
  }
#pragma unroll
  for (int k = 0; k < 12; ++k) {
    const bool mx = (k % 6) >= 3;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float w = __shfl_xor_sync(0xffffffffu, bx[k], o);
      bx[k] = mx ? fmaxf(bx[k], w) : fminf(bx[k], w);
    }
  }
  if (lane == 0)
    for (int k = 0; k < 12; ++k) s_box[warp][k] = bx[k];
  __syncthreads();
  if (tid < 12) {
    const bool mx = (tid % 6) >= 3;
    float r = s_box[0][tid];
    for (int w = 1; w < COL_THREADS / 32; ++w) r = mx ? fmaxf(r, s_box[w][tid]) : fminf(r, s_box[w][tid]);
    h_box[tid] = r;
  }
  __syncthreads();

  // face validation and compaction: A faces overlapping hand B's box, B faces overlapping hand A's box
  const double* XB = X + 3 * V;
  for (int f = tid; f < F; f += COL_THREADS) {
    const int i0 = faces[f * 3], i1 = faces[f * 3 + 1], i2 = faces[f * 3 + 2];
    if ((unsigned)i0 >= (unsigned)V || (unsigned)i1 >= (unsigned)V || (unsigned)i2 >= (unsigned)V) { s_bad = 1; continue; }
    float lo[3], hi[3];
    face_box(X, i0, i1, i2, lo, hi);
    if (overlap(lo, hi, h_box + 6, h_box + 9)) {
      const int s = atomicAdd(&s_na, 1);
      a_lo[s] = make_float4(lo[0], lo[1], lo[2], __int_as_float(f));
      a_hi[s] = make_float4(hi[0], hi[1], hi[2], 0.f);
    }
    face_box(XB, i0, i1, i2, lo, hi);
    if (overlap(lo, hi, h_box, h_box + 3)) b_list[atomicAdd(&s_nb, 1)] = f;
  }
  __syncthreads();
  if (s_bad) {                     // an index outside [0, V): nothing is read through it, the frame reports -1
    if (tid == 0) {
      count[b] = -1;
      if (stats) stats[2 * b] = stats[2 * b + 1] = 0;
    }
    return;
  }

  // candidate pairs: thread -> one B face, all compacted A faces
  const int na = s_na, nb = s_nb;
  int hits = 0, exact = 0;
  for (int j = tid; j < nb; j += COL_THREADS) {
    const int f = b_list[j];
    const int j0 = faces[f * 3], j1 = faces[f * 3 + 1], j2 = faces[f * 3 + 2];
    float lo[3], hi[3];
    face_box(XB, j0, j1, j2, lo, hi);
    const D3 t2[3] = {vert(XB, j0), vert(XB, j1), vert(XB, j2)};
    for (int i = 0; i < na; ++i) {
      const float4 l = a_lo[i], h = a_hi[i];
      if (l.x <= hi[0] && lo[0] <= h.x && l.y <= hi[1] && lo[1] <= h.y && l.z <= hi[2] && lo[2] <= h.z) {
        const int g = __float_as_int(l.w);
        const D3 t1[3] = {vert(X, faces[g * 3]), vert(X, faces[g * 3 + 1]), vert(X, faces[g * 3 + 2])};
        ++exact;
        hits += tri_tri(t1, t2);
      }
    }
  }
  hits = __reduce_add_sync(0xffffffffu, hits);
  exact = __reduce_add_sync(0xffffffffu, exact);
  if (lane == 0) {
    atomicAdd(&s_hits, hits);
    atomicAdd(&s_exact, (unsigned long long)exact);
  }
  __syncthreads();
  if (tid == 0) {
    count[b] = s_hits;
    if (stats) {
      stats[2 * b] = (long long)na * nb;
      stats[2 * b + 1] = (long long)s_exact;
    }
  }
}

}  // namespace

// CollisionFilter.py:93-124 / CollisionCheck.py for B frames: count[b] = the number of (face of hand A, face of hand B) pairs of frame b
// whose closed triangles intersect.  verts_a / verts_b [B,V,3] are float32 (is_f64 = 0) or float64 (is_f64 = 1); trans_a / trans_b [B,3]
// float64 translations added in float64 to every vertex, or NULL.  faces [F,3] int32 is the face table of both meshes, V <= 1024,
// F <= 2048.  A frame whose face table indexes outside [0, V) gets count -1.  stats [B,2] (or NULL): box tests and exact tests per frame.
RIH_API int rih_hand_collision_count(const void* verts_a, const void* verts_b, int is_f64, const double* trans_a, const double* trans_b,
                                     const int* faces, int V, int F, int B, long long* count, long long* stats, cudaStream_t s) {
  RIH_REQUIRE(verts_a && verts_b && faces && count, "hand_collision_count: NULL argument");
  RIH_REQUIRE(B >= 1 && V >= 3 && V <= COL_MAX_V && F >= 1 && F <= COL_MAX_F,
              "hand_collision_count: need B >= 1, 3 <= V <= %d, 1 <= F <= %d (got B=%d V=%d F=%d)", COL_MAX_V, COL_MAX_F, B, V, F);
  const size_t smem = col_smem(V, F);
  if (is_f64) {
    RIH_CUDA(cudaFuncSetAttribute(collision_count_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)col_smem(COL_MAX_V, COL_MAX_F)));
    launch_k(collision_count_kernel<double>, B, COL_THREADS, smem, s, (const double*)verts_a, (const double*)verts_b, trans_a, trans_b, faces,
             V, F, count, stats);
  } else {
    RIH_CUDA(cudaFuncSetAttribute(collision_count_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)col_smem(COL_MAX_V, COL_MAX_F)));
    launch_k(collision_count_kernel<float>, B, COL_THREADS, smem, s, (const float*)verts_a, (const float*)verts_b, trans_a, trans_b, faces,
             V, F, count, stats);
  }
  return check_launch("hand_collision_count");
}
