// Two-hand anti-penetration SDF loss of the reference's pose optimiser: the dense grid of lib/sdf (sdf_cuda_kernel.cu:243-304) and the
// `NewLoss` of code_sdf/sdf_template.py:57-157, sampled with grid_sample(align_corners=True).  Conventions (voxel centres, inside test,
// distance, sampling, outputs) are written out in renderih_b200/sdf.py; oracle/sdf_ref.py is the float64 reference the tests hold these
// kernels to.
//
//   grid_kernel          one thread per voxel of the dense grid [B,G,G,G]; the sample's face records are staged in shared memory.
//   penetration_kernel   one CTA per (sample, grid hand h): the bounding box of hand h gives its frame (centre, scale); the other hand's
//                        vertices, mapped into that frame, mark the <= 8 cell corners each touches in a G^3 bit mask in shared memory; the
//                        marked voxels are compacted (bit-mask prefix counts), their phi computed exactly as grid_kernel computes it, and
//                        each vertex's trilinear sample, its gradient and the per-vertex loss terms are written.  The loss only ever reads
//                        those corners, so the result equals sampling the dense grid while computing at most 8 V of its G^3 voxels.
//   loss_sum_kernel      one warp per sample: loss[b] = sum of the 2 V per-vertex terms in a fixed order (no float atomics).
//   penetration_bwd_kernel  elementwise: each output depends on its own vertex only, so the backward scales the stored gradient.
//
// Voxel phi: parity of the ray hits first (Moller-Trumbore); the point-triangle distances only for voxels that are inside.  Both loops
// visit the faces in chunks of the same shared-memory records, and min / xor do not depend on the order, so the two kernels agree bitwise.
#include <math.h>

#include "common.cuh"
using namespace rih;

namespace {

constexpr int GRID_THREADS = 256;
constexpr int PEN_THREADS = 512;
constexpr int SUM_THREADS = 256;
constexpr int kSmemBudget = 110 * 1024;     // per CTA: two resident CTAs per SM
constexpr int kMinChunk = 128;              // fewest faces staged at a time

// Face records: the three corners in the grid's normalised frame, 9 floats per face.  A face naming a vertex outside [0,V) gets NaN
// corners, which neither ray test nor distance can accept (the host validates indices; this only keeps the kernel in bounds).
__device__ __forceinline__ void stage_faces(float* sf, const int* __restrict__ faces, int f0, int n, const float* __restrict__ verts, int V,
                                            float c0, float c1, float c2, float s) {
  for (int i = threadIdx.x; i < n * 3; i += blockDim.x) {
    const int vi = faces[3 * f0 + i];
    float x = __int_as_float(0x7fc00000), y = x, z = x;
    if (vi >= 0 && vi < V) {
      const float* p = verts + 3 * (size_t)vi;
      x = __fdiv_rn(p[0] - c0, s); y = __fdiv_rn(p[1] - c1, s); z = __fdiv_rn(p[2] - c2, s);
    }
    sf[3 * i] = x; sf[3 * i + 1] = y; sf[3 * i + 2] = z;
  }
}

// Moller-Trumbore from o along the unnormalised direction d: |det| < 1e-6 rejected, u in [0,1], v >= 0, u + v <= 1, t >= 0.
__device__ __forceinline__ int ray_hit(const float* f, float ox, float oy, float oz, float dx, float dy, float dz) {
  const float e1x = f[3] - f[0], e1y = f[4] - f[1], e1z = f[5] - f[2];
  const float e2x = f[6] - f[0], e2y = f[7] - f[1], e2z = f[8] - f[2];
  const float px = dy * e2z - dz * e2y, py = dz * e2x - dx * e2z, pz = dx * e2y - dy * e2x;
  const float det = e1x * px + e1y * py + e1z * pz;
  if (!(fabsf(det) >= 1e-6f)) return 0;
  const float inv = 1.f / det;
  const float tx = ox - f[0], ty = oy - f[1], tz = oz - f[2];
  const float u = (tx * px + ty * py + tz * pz) * inv;
  if (!(u >= 0.f && u <= 1.f)) return 0;
  const float qx = ty * e1z - tz * e1y, qy = tz * e1x - tx * e1z, qz = tx * e1y - ty * e1x;
  const float v = (dx * qx + dy * qy + dz * qz) * inv;
  if (!(v >= 0.f && u + v <= 1.f)) return 0;
  return (e2x * qx + e2y * qy + e2z * qz) * inv >= 0.f;
}

__device__ __forceinline__ float seg_dist2(float px, float py, float pz, const float* a, const float* b) {
  const float ex = b[0] - a[0], ey = b[1] - a[1], ez = b[2] - a[2];
  const float wx = px - a[0], wy = py - a[1], wz = pz - a[2];
  const float ee = ex * ex + ey * ey + ez * ez;
  float t = ee > 0.f ? (wx * ex + wy * ey + wz * ez) / ee : 0.f;
  t = fminf(fmaxf(t, 0.f), 1.f);
  const float rx = wx - t * ex, ry = wy - t * ey, rz = wz - t * ez;
  return rx * rx + ry * ry + rz * rz;
}

__device__ __forceinline__ float edge_side(const float* u, const float* w, float px, float py, float pz, float nx, float ny, float nz) {
  const float ux = w[0] - u[0], uy = w[1] - u[1], uz = w[2] - u[2];
  const float vx = px - u[0], vy = py - u[1], vz = pz - u[2];
  return (uy * vz - uz * vy) * nx + (uz * vx - ux * vz) * ny + (ux * vy - uy * vx) * nz;
}

// Squared distance from p to the closed triangle f: the plane distance when p projects inside it, else the nearest of its three edges
// (which is also the answer for a zero-area face).
__device__ __forceinline__ float tri_dist2(const float* f, float px, float py, float pz) {
  const float* a = f; const float* b = f + 3; const float* c = f + 6;
  const float e0x = b[0] - a[0], e0y = b[1] - a[1], e0z = b[2] - a[2];
  const float e1x = c[0] - a[0], e1y = c[1] - a[1], e1z = c[2] - a[2];
  const float nx = e0y * e1z - e0z * e1y, ny = e0z * e1x - e0x * e1z, nz = e0x * e1y - e0y * e1x;
  const float nn = nx * nx + ny * ny + nz * nz;
  // orientation of each sub-triangle (edge, p) against n; all >= 0: p projects into the triangle
  if (nn > 0.f && edge_side(a, b, px, py, pz, nx, ny, nz) >= 0.f && edge_side(b, c, px, py, pz, nx, ny, nz) >= 0.f &&
      edge_side(c, a, px, py, pz, nx, ny, nz) >= 0.f) {
    const float h = (px - a[0]) * nx + (py - a[1]) * ny + (pz - a[2]) * nz;
    return h * h / nn;
  }
  return fminf(seg_dist2(px, py, pz, a, b), fminf(seg_dist2(px, py, pz, b, c), seg_dist2(px, py, pz, c, a)));
}

// phi of one voxel per thread (threads with active = false compute nothing).  Every thread of the CTA calls this (it synchronises).
// resident: all F face records are already in sf; otherwise they are staged chunk by chunk (fc faces at a time) from verts in the frame
// (c, s).  Voxel (i,j,k) has its centre at -1 + (idx + 0.5) * 2 / (G - 1) per axis.
__device__ float block_voxel_phi(bool active, int vox, int G, float* sf, int F, int fc, bool resident, const int* __restrict__ faces,
                                 const float* __restrict__ verts, int V, float c0, float c1, float c2, float s) {
  const float d = 2.f / (float)(G - 1);
  const int i = vox % G, j = (vox / G) % G, k = vox / (G * G);
  const float ox = -1.f + ((float)i + 0.5f) * d, oy = -1.f + ((float)j + 0.5f) * d, oz = -1.f + ((float)k + 0.5f) * d;
  const float dx = -1.f - ox, dy = -1.f - oy, dz = -1.f - oz;
  int hits = 0;
  for (int f0 = 0; f0 < F; f0 += fc) {
    const int n = min(fc, F - f0);
    if (!resident) { __syncthreads(); stage_faces(sf, faces, f0, n, verts, V, c0, c1, c2, s); __syncthreads(); }
    if (active)
      for (int f = 0; f < n; ++f) hits ^= ray_hit(sf + 9 * f, ox, oy, oz, dx, dy, dz);
  }
  const bool inside = active && (hits & 1);
  float best = INFINITY;
  if (__syncthreads_or(inside)) {
    for (int f0 = 0; f0 < F; f0 += fc) {
      const int n = min(fc, F - f0);
      if (!resident) { __syncthreads(); stage_faces(sf, faces, f0, n, verts, V, c0, c1, c2, s); __syncthreads(); }
      if (inside)
        for (int f = 0; f < n; ++f) best = fminf(best, tri_dist2(sf + 9 * f, ox, oy, oz));
    }
  }
  return inside ? sqrtf(best) : 0.f;
}

__global__ void __launch_bounds__(GRID_THREADS) grid_kernel(const int* __restrict__ faces, int F, const float* __restrict__ verts, int V, int G,
                                                            int fc, float* __restrict__ phi) {
  extern __shared__ float sf[];
  pdl_sync();
  const int b = blockIdx.y, G3 = G * G * G;
  const int vox = blockIdx.x * GRID_THREADS + threadIdx.x;
  const float* X = verts + (size_t)b * V * 3;
  const bool resident = fc >= F;
  if (resident) { stage_faces(sf, faces, 0, F, X, V, 0.f, 0.f, 0.f, 1.f); __syncthreads(); }
  const float p = block_voxel_phi(vox < G3, vox, G, sf, F, fc, resident, faces, X, V, 0.f, 0.f, 0.f, 1.f);
  if (vox < G3) phi[(size_t)b * G3 + vox] = p;
}

// Shared-memory layout of penetration_kernel: [fc * 9 floats faces | G^3/32 mask words | G^3/32 prefix counts | nmax list / phi slots]
struct PenLayout {
  int fc, words, nmax;
  size_t bytes() const { return sizeof(float) * 9 * (size_t)fc + sizeof(unsigned) * 2 * (size_t)words + sizeof(float) * (size_t)nmax; }
};

// Trilinear sample of the compacted grid at the normalised point (x,y,z), grid_sample(align_corners=True, padding_mode='zeros'):
// ix = (x + 1) / 2 * (G - 1), cell = floor, a corner outside the grid counts 0.  -> value, d(value)/d(ix, iy, iz).
__device__ __forceinline__ float sample_corner(const unsigned* mask, const unsigned* prefix, const float* vals, int G, int i, int j, int k) {
  if (i < 0 || i >= G || j < 0 || j >= G || k < 0 || k >= G) return 0.f;
  const int vox = (k * G + j) * G + i, w = vox >> 5, bit = vox & 31;
  return vals[prefix[w] + __popc(mask[w] & ((1u << bit) - 1u))];
}

__device__ __forceinline__ bool grid_coords(const float* p, float c0, float c1, float c2, float s, int G, float (&g)[3]) {
  const float x[3] = {__fdiv_rn(p[0] - c0, s), __fdiv_rn(p[1] - c1, s), __fdiv_rn(p[2] - c2, s)};
  bool any = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    g[a] = (x[a] + 1.f) / 2.f * (float)(G - 1);
    any = any && (g[a] >= -1.f && g[a] < (float)G);       // otherwise every corner is outside (also rejects NaN)
  }
  return any;
}

__global__ void __launch_bounds__(PEN_THREADS, 2) penetration_kernel(const float* __restrict__ verts, int B, int V, const int* __restrict__ faces,
                                                                     int F, const int* __restrict__ mult, int G, float box_scale, PenLayout lay,
                                                                     float* __restrict__ L, float* __restrict__ O, float* __restrict__ dLdv,
                                                                     float* __restrict__ center, float* __restrict__ scale) {
  extern __shared__ float smem[];
  float* sf = smem;
  unsigned* mask = (unsigned*)(smem + 9 * (size_t)lay.fc);
  unsigned* prefix = mask + lay.words;
  float* slots = (float*)(prefix + lay.words);
  __shared__ float red[6][PEN_THREADS / 32];
  __shared__ int wsum[PEN_THREADS / 32];
  pdl_sync();
  const int h = blockIdx.x, b = blockIdx.y, q = 1 - h;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* Xh = verts + ((size_t)b * 2 + h) * V * 3;
  const float* Xq = verts + ((size_t)b * 2 + q) * V * 3;

  // frame of hand h: centre of its bounding box, scale (1 + scale_factor) / 2 * its longest side
  float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int v = tid; v < V; v += PEN_THREADS)
    for (int a = 0; a < 3; ++a) { const float x = Xh[3 * v + a]; mn[a] = fminf(mn[a], x); mx[a] = fmaxf(mx[a], x); }
  for (int a = 0; a < 3; ++a) {
    float lo = mn[a], hi = mx[a];
    for (int o = 16; o > 0; o >>= 1) { lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o)); hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o)); }
    if (lane == 0) { red[a][warp] = lo; red[3 + a][warp] = hi; }
  }
  for (int w = tid; w < lay.words; w += PEN_THREADS) mask[w] = 0u;
  __syncthreads();
  float c[3], ext = 0.f;
  for (int a = 0; a < 3; ++a) {
    float lo = red[a][0], hi = red[3 + a][0];
    for (int w = 1; w < PEN_THREADS / 32; ++w) { lo = fminf(lo, red[a][w]); hi = fmaxf(hi, red[3 + a][w]); }
    c[a] = (lo + hi) / 2.f;
    ext = fmaxf(ext, hi - lo);
  }
  const float s = box_scale * ext;
  if (tid == 0) {
    for (int a = 0; a < 3; ++a) center[((size_t)b * 2 + h) * 3 + a] = c[a];
    scale[(size_t)b * 2 + h] = s;
  }

  // mark the cell corners the other hand's vertices touch
  for (int v = tid; v < V; v += PEN_THREADS) {
    float g[3];
    if (!grid_coords(Xq + 3 * v, c[0], c[1], c[2], s, G, g)) continue;
    const int i0 = (int)floorf(g[0]), j0 = (int)floorf(g[1]), k0 = (int)floorf(g[2]);
    for (int n = 0; n < 8; ++n) {
      const int i = i0 + (n & 1), j = j0 + ((n >> 1) & 1), k = k0 + (n >> 2);
      if (i < 0 || i >= G || j < 0 || j >= G || k < 0 || k >= G) continue;
      const int vox = (k * G + j) * G + i;
      atomicOr(mask + (vox >> 5), 1u << (vox & 31));
    }
  }
  __syncthreads();

  // exclusive prefix counts of the mask words: each thread owns a contiguous run of words
  const int per = (lay.words + PEN_THREADS - 1) / PEN_THREADS, w0 = min(tid * per, lay.words), w1 = min(w0 + per, lay.words);
  int cnt = 0;
  for (int w = w0; w < w1; ++w) cnt += __popc(mask[w]);
  int incl = cnt;
  for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  int base = 0, total = 0;
  for (int w = 0; w < PEN_THREADS / 32; ++w) { if (w < warp) base += wsum[w]; total += wsum[w]; }
  int run = base + incl - cnt;
  for (int w = w0; w < w1; ++w) {
    prefix[w] = run;
    unsigned m = mask[w];
    while (m) { const int bit = __ffs(m) - 1; m &= m - 1u; slots[run++] = __int_as_float(w * 32 + bit); }
  }
  if (lay.fc >= F) stage_faces(sf, faces, 0, F, Xh, V, c[0], c[1], c[2], s);
  __syncthreads();

  // phi of every marked voxel, written over its own list slot
  for (int r0 = 0; r0 < total; r0 += PEN_THREADS) {
    const int r = r0 + tid;
    const bool active = r < total;
    const int vox = active ? __float_as_int(slots[r]) : 0;
    const float p = block_voxel_phi(active, vox, G, sf, F, lay.fc, lay.fc >= F, faces, Xh, V, c[0], c[1], c[2], s);
    if (active) slots[r] = p;
  }
  __syncthreads();

  // per-vertex sample, loss terms and gradient of the other hand
  const float gs = 0.5f * (float)(G - 1) / s;        // d(ix)/d(vertex)
  for (int v = tid; v < V; v += PEN_THREADS) {
    const size_t o = ((size_t)b * 2 + q) * V + v;
    float g[3], p = 0.f, dp[3] = {0.f, 0.f, 0.f};
    if (grid_coords(Xq + 3 * v, c[0], c[1], c[2], s, G, g)) {
      const int i0 = (int)floorf(g[0]), j0 = (int)floorf(g[1]), k0 = (int)floorf(g[2]);
      const float fx = g[0] - (float)i0, fy = g[1] - (float)j0, fz = g[2] - (float)k0;
      const float wx[2] = {1.f - fx, fx}, wy[2] = {1.f - fy, fy}, wz[2] = {1.f - fz, fz};
      for (int n = 0; n < 8; ++n) {
        const int a = n & 1, bb = (n >> 1) & 1, cc = n >> 2;
        const float val = sample_corner(mask, prefix, slots, G, i0 + a, j0 + bb, k0 + cc);
        p += val * wx[a] * wy[bb] * wz[cc];
        dp[0] += val * (a ? 1.f : -1.f) * wy[bb] * wz[cc];
        dp[1] += val * wx[a] * (bb ? 1.f : -1.f) * wz[cc];
        dp[2] += val * wx[a] * wy[bb] * (cc ? 1.f : -1.f);
      }
    }
    const float m = (float)mult[v];
    L[o] = m * p * 0.25f;
    O[o] = m * p * s;
    for (int a = 0; a < 3; ++a) dLdv[3 * o + a] = m * 0.25f * dp[a] * gs;
  }
}

__global__ void __launch_bounds__(SUM_THREADS) loss_sum_kernel(const float* __restrict__ L, int B, int n, float* __restrict__ loss) {
  pdl_sync();
  const int b = blockIdx.x * (SUM_THREADS / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (b >= B) return;
  const float* x = L + (size_t)b * n;
  float acc = 0.f;
  for (int i = lane; i < n; i += 32) acc += x[i];
  acc = warp_sum(acc);
  if (lane == 0) loss[b] = acc;
}

__global__ void __launch_bounds__(SUM_THREADS) penetration_bwd_kernel(const float* __restrict__ dLdv, const float* __restrict__ scale, int B, int V,
                                                                      const float* __restrict__ g_loss, const float* __restrict__ g_L,
                                                                      const float* __restrict__ g_O, float* __restrict__ dv) {
  pdl_sync();
  const long long i = (long long)blockIdx.x * SUM_THREADS + threadIdx.x;
  if (i >= 2LL * B * V) return;
  const int b = (int)(i / (2LL * V)), h = (int)((i / V) % 2);
  float g = g_loss ? g_loss[b] : 0.f;
  if (g_L) g += g_L[i];
  if (g_O) g += 4.f * scale[(size_t)b * 2 + (1 - h)] * g_O[i];      // O = 4 s_o L: the grid hand's scale
  for (int a = 0; a < 3; ++a) dv[3 * i + a] = g * dLdv[3 * i + a];
}

int max_smem_optin() {
  int dev = 0, v = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess) return 48 * 1024;
  return v;
}

int check_sizes(const char* what, int B, int V, int F, int G) {
  RIH_REQUIRE(B > 0, "%s: batch %d must be positive", what, B);
  RIH_REQUIRE(V >= 3 && F >= 1, "%s: need V >= 3 vertices and F >= 1 faces (got V=%d F=%d)", what, V, F);
  RIH_REQUIRE(G >= 2 && G <= 64, "%s: grid size %d outside 2..64", what, G);
  return 0;
}

}  // namespace

// lib/sdf/sdf/sdf.py SDF / sdf_cuda_kernel.cu:243-304: phi [B,G,G,G] (x fastest) of the closed mesh faces [F,3] (int32, shared by the
// batch) over verts [B,V,3] in the normalised frame [-1,1]^3.  Voxel (i,j,k) has its centre at -1 + (idx + 0.5) * 2 / (G - 1); phi is
// its distance to the nearest face when the ray towards (-1,-1,-1) hits an odd number of faces, else 0.  Every voxel is written.
RIH_API int rih_sdf_grid(const int* faces, int F, const float* verts, int B, int V, int G, float* phi, cudaStream_t stream) {
  if (check_sizes("sdf_grid", B, V, F, G)) return 1;
  RIH_REQUIRE(faces && verts && phi, "sdf_grid: null pointer");
  const int fc = min(F, kSmemBudget / (9 * (int)sizeof(float)));
  const size_t smem = sizeof(float) * 9 * (size_t)fc;
  RIH_CUDA(cudaFuncSetAttribute(grid_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int G3 = G * G * G;
  launch_k(grid_kernel, dim3(cdiv(G3, GRID_THREADS), B), GRID_THREADS, smem, stream, faces, F, verts, V, G, fc, phi);
  return check_launch("sdf_grid");
}

// pose_data_optimize/code_sdf/sdf_template.py:57-157 (NewLoss.forward) with its gradient, for verts [B,2,V,3] (hand 0 = right, 1 = left),
// closed faces [F,3] and mult [V] (int32: the number of the 16 parts containing each vertex).  Per sample and hand h: centre c_h and scale
// s_h = box_scale * longest side of its bounding box; the other hand's vertex v is sampled at (v - c_h) / s_h in the SDF of hand h
// (grid size G) with grid_sample(align_corners=True) -> p.  Writes L [B,2,V] = mult * p / 4, O [B,2,V] = mult * p * s_h, loss [B] = sum
// of L per sample, dLdv [B,2,V,3] = dL/dv (the frames are constants), center [B,2,3] and scale [B,2] of each hand's own frame.
RIH_API int rih_sdf_penetration(const float* verts, int B, int V, const int* faces, int F, const int* mult, int G, float box_scale, float* loss,
                                float* L, float* O, float* dLdv, float* center, float* scale, cudaStream_t stream) {
  if (check_sizes("sdf_penetration", B, V, F, G)) return 1;
  RIH_REQUIRE(verts && faces && mult && loss && L && O && dLdv && center && scale, "sdf_penetration: null pointer");
  PenLayout lay;
  lay.words = (G * G * G + 31) / 32;
  lay.nmax = min(8 * V, G * G * G);
  lay.fc = F;
  const int budget = min(kSmemBudget, max_smem_optin() - 4096);     // static shared memory of the kernel is below 4 KB
  if ((long long)lay.bytes() > budget) {
    lay.fc = 0;
    const long long room = (long long)budget - (long long)lay.bytes();
    lay.fc = (int)(room / (9 * (long long)sizeof(float)));
    RIH_REQUIRE(lay.fc >= kMinChunk, "sdf_penetration: V=%d G=%d leave no shared memory for the face records", V, G);
  }
  RIH_CUDA(cudaFuncSetAttribute(penetration_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lay.bytes()));
  launch_k(penetration_kernel, dim3(2, B), PEN_THREADS, lay.bytes(), stream, verts, B, V, faces, F, mult, G, box_scale, lay, L, O, dLdv, center,
           scale);
  if (int rc = check_launch("sdf_penetration")) return rc;
  launch_k(loss_sum_kernel, dim3(cdiv(B, SUM_THREADS / 32)), SUM_THREADS, 0, stream, (const float*)L, B, 2 * V, loss);
  return check_launch("sdf_penetration loss");
}

// Backward of rih_sdf_penetration: dv [B,2,V,3] = (g_loss[b] + g_L + 4 * s_o * g_O) * dLdv, where s_o is the scale of the grid hand
// (the other hand).  Any of g_loss [B], g_L [B,2,V], g_O [B,2,V] may be NULL (zero).
RIH_API int rih_sdf_penetration_bwd(const float* dLdv, const float* scale, int B, int V, const float* g_loss, const float* g_L, const float* g_O,
                                    float* dv, cudaStream_t stream) {
  RIH_REQUIRE(B > 0 && V > 0, "sdf_penetration_bwd: bad sizes B=%d V=%d", B, V);
  RIH_REQUIRE(dLdv && scale && dv, "sdf_penetration_bwd: null pointer");
  launch_k(penetration_bwd_kernel, dim3(cdiv(2LL * B * V, SUM_THREADS)), SUM_THREADS, 0, stream, dLdv, scale, B, V, g_loss, g_L, g_O, dv);
  return check_launch("sdf_penetration_bwd");
}
