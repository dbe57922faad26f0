// Mesh rasteriser and shader of the reference's two-hand renderer (utils/vis_utils.py:39-100,153-289: pytorch3d MeshRasterizer with
// blur_radius 0 and faces_per_pixel 1, HardPhongShader, hard blend on a white background) and the per-sample mask IoU of
// utils/compute_maskiou.py:59-64,250-263.  Conventions (camera maps, coverage rule, lighting constants) are written out in
// renderih_b200/render.py; oracle/render_ref.py is the float64 reference the tests hold these kernels to.
//
//   raster_kernel<false>  one warp per (sample, face): lanes stride over the face's pixel bounding box, clamped to the image, and
//                         atomicMin a 64-bit key (order-preserving fp32 depth << 32 | face index) into a [B,S,S] workspace.  The
//                         minimum does not depend on launch order, so the result is bitwise deterministic; equal depths go to the
//                         lower face index.
//   raster_kernel<true>   the same traversal, coverage only: atomicOr into a [2,B,S,ceil(S/32)] bit mask (one plane per hand).
//   shade_kernel          one thread per pixel: decode the face, recompute its barycentrics, interpolate colour (and world position and
//                         vertex normal for Phong), light, blend; optional pix_to_face / zbuf / bary fragments.
//   vertex_normals_kernel one thread per (sample, vertex): sums the corner cross products of its faces in the fixed order of a
//                         vertex -> face CSR (no float atomics), then normalises.
//   mask_iou_kernel       one CTA per sample: popcounts of L&R, L and R -> |L n R| / |L u R| (NaN for an empty union).
//
// Projection, edge functions, barycentrics and shading are evaluated in fp64 from the fp32 inputs: the pixel coordinates of a vertex
// are O(S), where an fp32 rounding is ~1e-5 px -- enough to move a barycentric by 1e-6 and a colour past the tolerance the tests use.
// fp64 costs little here (a few dozen operations per covered pixel).  Only the depth stored in the key is fp32.
#include "common.cuh"
using namespace rih;

namespace {

constexpr int RS_THREADS = 256;
constexpr unsigned long long kEmptyKey = ~0ull;

// Pixel coordinates (u: column, v: row, pixel (r,c) has its centre at (c+0.5, r+0.5)) and depth of one vertex.
//   orthographic  cam = (scale, tx, ty, -):   u = S*scale*x + S/2*(tx+1),  v = S*scale*y + S/2*(ty+1),  depth = z + 10
//   perspective   cam = (fx, fy, cx, cy):     u = fx*x/z + cx,             v = fy*y/z + cy,             depth = z
__device__ __forceinline__ void project(const float* p, const float* cam, int persp, int S, double& u, double& v, double& d) {
  const double x = p[0], y = p[1], z = p[2];
  if (persp) {
    u = (double)cam[0] * x / z + (double)cam[2];
    v = (double)cam[1] * y / z + (double)cam[3];
    d = z;
  } else {
    const double a = (double)S * (double)cam[0], h = 0.5 * (double)S;
    u = a * x + h * ((double)cam[1] + 1.0);
    v = a * y + h * ((double)cam[2] + 1.0);
    d = z + 10.0;
  }
}

struct Tri {
  double u[3], v[3], d[3];
  int idx[3];
};

// Projects face f of one sample; false when the face is not drawn (index out of range, non-finite coordinates, a vertex at z <= 0
// under the perspective camera, zero area).
__device__ __forceinline__ bool setup_tri(const float* verts, int V, const int* faces, int f, const float* cam, int persp, int S, Tri& t) {
  for (int k = 0; k < 3; ++k) {
    const int vi = faces[3 * f + k];
    if (vi < 0 || vi >= V) return false;
    t.idx[k] = vi;
    project(verts + 3 * (size_t)vi, cam, persp, S, t.u[k], t.v[k], t.d[k]);
    if (!isfinite(t.u[k]) || !isfinite(t.v[k]) || !isfinite(t.d[k])) return false;
    if (persp && !(t.d[k] > 0.0)) return false;
  }
  const double area = (t.u[1] - t.u[0]) * (t.v[2] - t.v[0]) - (t.v[1] - t.v[0]) * (t.u[2] - t.u[0]);
  return area != 0.0;
}

// Edge functions at (px,py): w[k] is the (doubled, signed) area of the sub-triangle opposite vertex k.  The centre is covered when all
// three are strictly of one sign: a centre exactly on an edge is outside.
__device__ __forceinline__ bool edge_test(const Tri& t, double px, double py, double (&w)[3]) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int a = (k + 1) % 3, b = (k + 2) % 3;
    w[k] = (t.u[b] - t.u[a]) * (py - t.v[a]) - (t.v[b] - t.v[a]) * (px - t.u[a]);
  }
  return (w[0] > 0.0 && w[1] > 0.0 && w[2] > 0.0) || (w[0] < 0.0 && w[1] < 0.0 && w[2] < 0.0);
}

// Barycentrics (perspective-correct under the perspective camera) and depth of a covered centre.
__device__ __forceinline__ double barycentric(const Tri& t, int persp, const double (&w)[3], double (&b)[3]) {
  const double s = w[0] + w[1] + w[2];
  for (int k = 0; k < 3; ++k) b[k] = w[k] / s;
  if (!persp) return b[0] * t.d[0] + b[1] * t.d[1] + b[2] * t.d[2];
  double q[3], qs = 0.0;
  for (int k = 0; k < 3; ++k) { q[k] = b[k] / t.d[k]; qs += q[k]; }
  for (int k = 0; k < 3; ++k) b[k] = q[k] / qs;
  return 1.0 / qs;
}

__device__ __forceinline__ uint32_t depth_bits(float d) {     // order-preserving map of fp32 onto uint32
  const uint32_t u = __float_as_uint(d);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float depth_float(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// kCover = false: keys[B,S,S] (verts0 only); kCover = true: bits[nsets,B,S,W] for hand planes verts0 / verts1.
template <bool kCover>
__global__ void __launch_bounds__(RS_THREADS) raster_kernel(const float* __restrict__ verts0, const float* __restrict__ verts1, int nsets, int B,
                                                            int V, const int* __restrict__ faces, int F, const float* __restrict__ cam, int persp,
                                                            int S, unsigned long long* keys, unsigned* bits) {
  pdl_sync();
  const long long gw = (long long)blockIdx.x * (RS_THREADS / 32) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (gw >= (long long)nsets * B * F) return;
  const int f = (int)(gw % F);
  const int b = (int)((gw / F) % B);
  const int set = (int)(gw / ((long long)F * B));
  const float* verts = (set ? verts1 : verts0) + (size_t)b * V * 3;
  Tri t;
  if (!setup_tri(verts, V, faces, f, cam + 4 * b, persp, S, t)) return;
  const double umin = fmin(t.u[0], fmin(t.u[1], t.u[2])), umax = fmax(t.u[0], fmax(t.u[1], t.u[2]));
  const double vmin = fmin(t.v[0], fmin(t.v[1], t.v[2])), vmax = fmax(t.v[0], fmax(t.v[1], t.v[2]));
  // centres c + 0.5 in [umin, umax]; clamp in fp64 before converting so that far off-screen faces cannot overflow an int
  const int c0 = (int)ceil(fmax(umin - 0.5, 0.0)), c1 = (int)floor(fmin(umax - 0.5, (double)(S - 1)));
  const int r0 = (int)ceil(fmax(vmin - 0.5, 0.0)), r1 = (int)floor(fmin(vmax - 0.5, (double)(S - 1)));
  if (c0 > c1 || r0 > r1) return;
  const int w = c1 - c0 + 1, n = w * (r1 - r0 + 1);
  const int W = (S + 31) >> 5;
  for (int i = lane; i < n; i += 32) {
    const int r = r0 + i / w, c = c0 + i % w;
    double e[3];
    if (!edge_test(t, c + 0.5, r + 0.5, e)) continue;
    if (kCover) {
      atomicOr(bits + (((size_t)set * B + b) * S + r) * W + (c >> 5), 1u << (c & 31));
    } else {
      double bc[3];
      const float d = (float)barycentric(t, persp, e, bc);
      if (!isfinite(d)) continue;
      atomicMin(keys + ((size_t)b * S + r) * S + c, ((unsigned long long)depth_bits(d) << 32) | (unsigned)f);
    }
  }
}

__device__ __forceinline__ void normalize_eps(double (&x)[3]) {     // torch.nn.functional.normalize(x, eps=1e-6)
  const double n = fmax(sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]), 1e-6);
  for (int k = 0; k < 3; ++k) x[k] /= n;
}

__global__ void __launch_bounds__(RS_THREADS) vertex_normals_kernel(const float* __restrict__ verts, int B, int V, const int* __restrict__ faces,
                                                                    const int* __restrict__ vf_ptr, const int* __restrict__ vf_corner,
                                                                    float* __restrict__ normals) {
  pdl_sync();
  const long long i = (long long)blockIdx.x * RS_THREADS + threadIdx.x;
  if (i >= (long long)B * V) return;
  const int b = (int)(i / V), v = (int)(i % V);
  const float* X = verts + (size_t)b * V * 3;
  double n[3] = {0.0, 0.0, 0.0};
  for (int j = vf_ptr[v]; j < vf_ptr[v + 1]; ++j) {
    // corner k of face f: cross(x[k+1] - x[k], x[k+2] - x[k]) (pytorch3d Meshes.verts_normals; all three corners give 2 * area * normal)
    const int f = vf_corner[j] / 3, k = vf_corner[j] % 3;
    const float* p0 = X + 3 * (size_t)faces[3 * f + k];
    const float* p1 = X + 3 * (size_t)faces[3 * f + (k + 1) % 3];
    const float* p2 = X + 3 * (size_t)faces[3 * f + (k + 2) % 3];
    const double a[3] = {(double)p1[0] - p0[0], (double)p1[1] - p0[1], (double)p1[2] - p0[2]};
    const double c[3] = {(double)p2[0] - p0[0], (double)p2[1] - p0[1], (double)p2[2] - p0[2]};
    n[0] += a[1] * c[2] - a[2] * c[1];
    n[1] += a[2] * c[0] - a[0] * c[2];
    n[2] += a[0] * c[1] - a[1] * c[0];
  }
  normalize_eps(n);
  for (int k = 0; k < 3; ++k) normals[i * 3 + k] = (float)n[k];
}

// pytorch3d defaults (PointLights / Materials / BlendParams): ambient 0.5, diffuse 0.3, specular 0.2, shininess 64, light at (0,0,-1);
// AmbientLights: ambient 1, no diffuse or specular.
constexpr double kAmbient = 0.5, kDiffuse = 0.3, kSpecular = 0.2, kLightZ = -1.0;

__global__ void __launch_bounds__(RS_THREADS) shade_kernel(const unsigned long long* __restrict__ keys, const float* __restrict__ verts,
                                                           const float* __restrict__ normals, int B, int V, const int* __restrict__ faces,
                                                           const float* __restrict__ cam, int persp, int S, const float* __restrict__ colors,
                                                           float* __restrict__ img, float* __restrict__ alpha, int* __restrict__ pix_to_face,
                                                           float* __restrict__ zbuf, float* __restrict__ bary) {
  pdl_sync();
  const long long i = (long long)blockIdx.x * RS_THREADS + threadIdx.x;
  if (i >= (long long)B * S * S) return;
  const unsigned long long key = keys[i];
  if (key == kEmptyKey) {
    if (img) for (int k = 0; k < 3; ++k) img[i * 3 + k] = 1.f / 255.f;
    if (alpha) alpha[i] = 0.f;
    if (pix_to_face) pix_to_face[i] = -1;
    if (zbuf) zbuf[i] = -1.f;
    if (bary) for (int k = 0; k < 3; ++k) bary[i * 3 + k] = -1.f;
    return;
  }
  const int b = (int)(i / ((long long)S * S)), rc = (int)(i % ((long long)S * S));
  const int r = rc / S, c = rc % S;
  const int f = (int)(unsigned)(key & 0xffffffffu);
  const float* X = verts + (size_t)b * V * 3;
  Tri t;
  setup_tri(X, V, faces, f, cam + 4 * b, persp, S, t);      // the raster pass accepted this face and covered this centre
  double e[3], bc[3];
  edge_test(t, c + 0.5, r + 0.5, e);
  barycentric(t, persp, e, bc);
  if (alpha) alpha[i] = 1.f;
  if (pix_to_face) pix_to_face[i] = f;
  if (zbuf) zbuf[i] = depth_float((uint32_t)(key >> 32));
  if (bary) for (int k = 0; k < 3; ++k) bary[i * 3 + k] = (float)bc[k];
  if (!img) return;
  double tex[3] = {0.0, 0.0, 0.0};
  for (int j = 0; j < 3; ++j)
    for (int k = 0; k < 3; ++k) tex[k] += bc[j] * (double)colors[3 * t.idx[j] + k];
  double rgb[3];
  if (!normals) {
    for (int k = 0; k < 3; ++k) rgb[k] = tex[k];
  } else {
    const float* N = normals + (size_t)b * V * 3;
    double p[3] = {0.0, 0.0, 0.0}, n[3] = {0.0, 0.0, 0.0};
    for (int j = 0; j < 3; ++j)
      for (int k = 0; k < 3; ++k) {
        p[k] += bc[j] * (double)X[3 * t.idx[j] + k];
        n[k] += bc[j] * (double)N[3 * t.idx[j] + k];
      }
    normalize_eps(n);
    double l[3] = {-p[0], -p[1], kLightZ - p[2]};
    normalize_eps(l);
    const double cz = persp ? 0.0 : -10.0;      // camera centre in world coordinates
    double vw[3] = {-p[0], -p[1], cz - p[2]};
    normalize_eps(vw);
    const double cosl = n[0] * l[0] + n[1] * l[1] + n[2] * l[2];
    double rv = 0.0;
    for (int k = 0; k < 3; ++k) rv += vw[k] * (-l[k] + 2.0 * cosl * n[k]);
    const double spec = cosl > 0.0 ? kSpecular * pow(fmax(rv, 0.0), 64.0) : 0.0;
    const double shade = kAmbient + kDiffuse * fmax(cosl, 0.0);
    for (int k = 0; k < 3; ++k) rgb[k] = shade * tex[k] + spec;
  }
  for (int k = 0; k < 3; ++k) img[i * 3 + k] = (float)(rgb[k] / 255.0);
}

__global__ void __launch_bounds__(RS_THREADS) mask_iou_kernel(const unsigned* __restrict__ bits, int B, int S, float* __restrict__ iou) {
  pdl_sync();
  const int b = blockIdx.x, W = (S + 31) >> 5;
  const unsigned* L = bits + (size_t)b * S * W;
  const unsigned* R = bits + ((size_t)B + b) * S * W;
  long long cnt[3] = {0, 0, 0};        // |L n R|, |L|, |R|
  for (long long j = threadIdx.x; j < (long long)S * W; j += RS_THREADS) {
    const unsigned l = L[j], r = R[j];
    cnt[0] += __popc(l & r); cnt[1] += __popc(l); cnt[2] += __popc(r);
  }
  __shared__ long long red[3][RS_THREADS / 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int k = 0; k < 3; ++k) {
    long long x = cnt[k];
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    if (lane == 0) red[k][warp] = x;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    long long t[3] = {0, 0, 0};
    for (int k = 0; k < 3; ++k)
      for (int w = 0; w < RS_THREADS / 32; ++w) t[k] += red[k][w];
    const long long uni = t[1] + t[2] - t[0];
    iou[b] = uni > 0 ? (float)((double)t[0] / (double)uni) : __int_as_float(0x7fc00000);
  }
}

int check_dims(int B, int V, int F, int persp, int S) {
  RIH_REQUIRE(B > 0 && V > 0 && F > 0, "render: bad sizes B=%d V=%d F=%d", B, V, F);
  RIH_REQUIRE(S > 0 && S <= 8192, "render: image size %d outside 1..8192", S);
  RIH_REQUIRE(persp == 0 || persp == 1, "render: perspective flag must be 0 or 1 (got %d)", persp);
  return 0;
}

}  // namespace

// utils/vis_utils.py:89-97 (MeshRasterizer, blur_radius 0, faces_per_pixel 1): rasterise faces [F,3] (int32, shared by the batch) of
// verts [B,V,3] through per-sample cameras cam [B,4] (orthographic (scale, tx, ty, 0) or perspective (fx, fy, cx, cy)) into
// keys [B,S,S] (uint64: fp32 depth mapped to an order-preserving uint32 << 32 | face index; ~0 = background).  Fills keys first.
RIH_API int rih_render_raster(const float* verts, int B, int V, const int* faces, int F, const float* cam, int perspective, int S,
                              unsigned long long* keys, cudaStream_t stream) {
  if (check_dims(B, V, F, perspective, S)) return 1;
  RIH_REQUIRE(verts && faces && cam && keys, "render_raster: null pointer");
  RIH_CUDA(cudaMemsetAsync(keys, 0xff, sizeof(unsigned long long) * B * S * S, stream));
  const long long warps = (long long)B * F;
  launch_k(raster_kernel<false>, dim3(cdiv(warps, RS_THREADS / 32)), RS_THREADS, 0, stream, verts, verts, 1, B, V, faces, F, cam, perspective, S,
           keys, (unsigned*)nullptr);
  return check_launch("render_raster");
}

// pytorch3d Meshes.verts_normals (used by HardPhongShader, utils/vis_utils.py:56): normals [B,V,3] = normalised sum of the corner cross
// products of each vertex's faces, taken in the order of the vertex -> face CSR vf_ptr [V+1] / vf_corner (entries 3 * face + corner).
RIH_API int rih_render_vertex_normals(const float* verts, int B, int V, const int* faces, const int* vf_ptr, const int* vf_corner, float* normals,
                                      cudaStream_t stream) {
  RIH_REQUIRE(B > 0 && V > 0, "render_vertex_normals: bad sizes B=%d V=%d", B, V);
  RIH_REQUIRE(verts && faces && vf_ptr && vf_corner && normals, "render_vertex_normals: null pointer");
  launch_k(vertex_normals_kernel, dim3(cdiv((long long)B * V, RS_THREADS)), RS_THREADS, 0, stream, verts, B, V, faces, vf_ptr, vf_corner, normals);
  return check_launch("render_vertex_normals");
}

// utils/vis_utils.py:89-100 (HardPhongShader + hard blend, then / 255): resolve keys [B,S,S] of rih_render_raster into img [B,S,S,3]
// and alpha [B,S,S].  colors [V,3] (0..255, shared by the batch).  normals [B,V,3] selects Phong shading with pytorch3d's default
// PointLights at (0,0,-1); NULL selects AmbientLights.  Background: img 1/255, alpha 0.  Every output is optional (NULL = skipped; colors
// is needed with img): pix_to_face [B,S,S] int32 (-1 background), zbuf [B,S,S] (-1 background), bary [B,S,S,3] (-1 background).
RIH_API int rih_render_shade(const unsigned long long* keys, const float* verts, const float* normals, int B, int V, const int* faces, int F,
                             const float* cam, int perspective, int S, const float* colors, float* img, float* alpha, int* pix_to_face,
                             float* zbuf, float* bary, cudaStream_t stream) {
  if (check_dims(B, V, F, perspective, S)) return 1;
  RIH_REQUIRE(keys && verts && faces && cam && (colors || !img), "render_shade: null pointer");
  launch_k(shade_kernel, dim3(cdiv((long long)B * S * S, RS_THREADS)), RS_THREADS, 0, stream, keys, verts, normals, B, V, faces, cam, perspective,
           S, colors, img, alpha, pix_to_face, zbuf, bary);
  return check_launch("render_shade");
}

// utils/compute_maskiou.py:250-263 (render_single_mask per hand, bm0): per-sample IoU [B] of the coverage masks of verts_l and verts_r
// [B,V,3], each rasterised alone with faces [F,3] through the shared cameras cam [B,4]; NaN when both masks are empty.
// bits: workspace of 2 * B * S * ceil(S/32) uint32 (cleared here).
RIH_API int rih_render_mask_iou(const float* verts_l, const float* verts_r, int B, int V, const int* faces, int F, const float* cam, int perspective,
                                int S, unsigned* bits, float* iou, cudaStream_t stream) {
  if (check_dims(B, V, F, perspective, S)) return 1;
  RIH_REQUIRE(verts_l && verts_r && faces && cam && bits && iou, "render_mask_iou: null pointer");
  RIH_CUDA(cudaMemsetAsync(bits, 0, sizeof(unsigned) * 2 * B * S * ((S + 31) / 32), stream));
  const long long warps = 2LL * B * F;
  launch_k(raster_kernel<true>, dim3(cdiv(warps, RS_THREADS / 32)), RS_THREADS, 0, stream, verts_l, verts_r, 2, B, V, faces, F, cam, perspective, S,
           (unsigned long long*)nullptr, bits);
  if (int rc = check_launch("render_mask_iou raster")) return rc;
  launch_k(mask_iou_kernel, dim3(B), RS_THREADS, 0, stream, bits, B, S, iou);
  return check_launch("render_mask_iou reduce");
}
