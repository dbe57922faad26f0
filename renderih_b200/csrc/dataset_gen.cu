// Dataset preparation of the reference on the GPU (utils/dataset_gen/interhand.py, rendering_code/step7_gen_annotations.py), batched over
// frames: the camera geometry and crop box of both hands, the 256x256 crop with the frame mean, the joint heatmaps and the uint8
// conversion cv.imwrite applies to float images.  No kernel synchronises with the host or allocates memory.
//
// dtypes follow the reference step by step (numpy 2 promotion rules):
//   MANO verts / joints, cam_R, cam_t              float32
//   v @ cam_R.T + cam_t                            float32; each output is ((v0*R0 + v1*R1) + v2*R2) + t, rounded per operation, no FMA
//                                                  (numpy hands `@` to a BLAS whose summation order is its own: last-bit differences)
//   cameraIn, v @ cameraIn.T, [:, :2] / [:, 2:]     float64 (cameraIn is built from float32 scalars and Python ints: float64), same order
//   |left_i - right_i| (the `dist` test)            float32, sqrt((dx*dx + dy*dy) + dz*dz); its minimum propagates NaN, so only NaN
//                                                  (or a distance >= 9999999) fails `dist < 9999999`
//   cut_img: Min, Max, mid, L, M, x @ M.T, camera  float64; min / max propagate NaN like np.min / np.max
#include "common.cuh"
using namespace rih;

namespace {

constexpr int HAND_V = 778, HAND_J = 21;

__device__ __forceinline__ double nanmin2(double a, double b) { return (isnan(a) || isnan(b)) ? __longlong_as_double(0x7ff8000000000000LL) : fmin(a, b); }
__device__ __forceinline__ double nanmax2(double a, double b) { return (isnan(a) || isnan(b)) ? __longlong_as_double(0x7ff8000000000000LL) : fmax(a, b); }
__device__ __forceinline__ float nanminf(float a, float b) { return (isnan(a) || isnan(b)) ? __int_as_float(0x7fc00000) : fminf(a, b); }

// p @ R.T + t in float32, one row
__device__ __forceinline__ void cam_xform(const float* p, const float* R, const float* t, float* o) {
#pragma unroll
  for (int r = 0; r < 3; ++r)
    o[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(p[0], R[3 * r]), __fmul_rn(p[1], R[3 * r + 1])), __fmul_rn(p[2], R[3 * r + 2])), t[r]);
}

// (p @ K.T)[:2] / (p @ K.T)[2:] in float64
__device__ __forceinline__ void project(const float* p, const double* K, double* uv) {
  double h[3];
  const double x = p[0], y = p[1], z = p[2];
#pragma unroll
  for (int r = 0; r < 3; ++r) h[r] = __dadd_rn(__dadd_rn(__dmul_rn(x, K[3 * r]), __dmul_rn(y, K[3 * r + 1])), __dmul_rn(z, K[3 * r + 2]));
  uv[0] = __ddiv_rn(h[0], h[2]);
  uv[1] = __ddiv_rn(h[1], h[2]);
}

template <typename T>
__device__ __forceinline__ T warp_reduce(T v, T (*op)(T, T)) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// cut_img (dataset/dataset_utils.py:12-42) for one frame, one warp: box of the n points pts [n,2], M [6], the mapped points
// [x, y, 1] @ M.T (cut, may be NULL) and the camera update (K [9] in place, may be NULL).
__device__ void cut_frame(const double* pts, int n, double radio, int img_size, double* M, double* cut, double* K) {
  const int lane = threadIdx.x & 31;
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  double mn0 = INFINITY, mn1 = INFINITY, mx0 = -INFINITY, mx1 = -INFINITY;
  for (int i = lane; i < n; i += 32) {
    const double a = pts[2 * i], b = pts[2 * i + 1];
    mn0 = nanmin2(mn0, a); mn1 = nanmin2(mn1, b); mx0 = nanmax2(mx0, a); mx1 = nanmax2(mx1, b);
  }
  if (n == 0) mn0 = mn1 = mx0 = mx1 = nan;
  mn0 = warp_reduce<double>(mn0, nanmin2); mn1 = warp_reduce<double>(mn1, nanmin2);
  mx0 = warp_reduce<double>(mx0, nanmax2); mx1 = warp_reduce<double>(mx1, nanmax2);
  const double mid0 = __dmul_rn(__dadd_rn(mn0, mx0), 0.5), mid1 = __dmul_rn(__dadd_rn(mn1, mx1), 0.5);
  const double L = __ddiv_rn(__ddiv_rn(nanmax2(__dsub_rn(mx0, mn0), __dsub_rn(mx1, mn1)), 2.0), radio);
  const double s = __ddiv_rn((double)img_size / 2.0, L);
  const double m[6] = {__dmul_rn(s, 1.0), __dmul_rn(s, 0.0), __dmul_rn(s, __dsub_rn(L, mid0)),
                       __dmul_rn(s, 0.0), __dmul_rn(s, 1.0), __dmul_rn(s, __dsub_rn(L, mid1))};
  if (cut) {
    for (int i = lane; i < n; i += 32) {
      const double a = pts[2 * i], b = pts[2 * i + 1];
      cut[2 * i] = __dadd_rn(__dadd_rn(__dmul_rn(a, m[0]), __dmul_rn(b, m[1])), m[2]);
      cut[2 * i + 1] = __dadd_rn(__dadd_rn(__dmul_rn(a, m[3]), __dmul_rn(b, m[4])), m[5]);
    }
  }
  if (lane == 0) {
    for (int k = 0; k < 6; ++k) M[k] = m[k];
    if (K) {
      K[0] = __dmul_rn(K[0], m[0]);
      K[4] = __dmul_rn(K[4], m[4]);
      K[2] = __dadd_rn(__dmul_rn(K[2], m[0]), m[2]);
      K[5] = __dadd_rn(__dmul_rn(K[5], m[4]), m[5]);
    }
  }
}

__global__ void __launch_bounds__(256)
dsgen_geometry_kernel(const float* __restrict__ vl, const float* __restrict__ vr, const float* __restrict__ jl, const float* __restrict__ jr,
                      const float* __restrict__ Rm, const float* __restrict__ tv, const double* __restrict__ Kin, int B, int crop, double radio,
                      int img_size, float* __restrict__ v3d, float* __restrict__ j3d, double* __restrict__ v2d, double* __restrict__ j2d,
                      int* __restrict__ valid, double* __restrict__ Mout, double* __restrict__ Kout, double* __restrict__ cut2d) {
  pdl_sync();
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (b >= B) return;
  float R[9], t[3];
  double K[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) { R[k] = Rm[(size_t)b * 9 + k]; K[k] = Kin[(size_t)b * 9 + k]; }
#pragma unroll
  for (int k = 0; k < 3; ++k) t[k] = tv[(size_t)b * 3 + k];
  // the dist test of interhand.py:198-201 on the MANO output (before the camera transform)
  if (valid) {
    float dmin = INFINITY;
    for (int i = lane; i < HAND_V; i += 32) {
      const float* a = vl + ((size_t)b * HAND_V + i) * 3;
      const float* c = vr + ((size_t)b * HAND_V + i) * 3;
      const float dx = __fsub_rn(a[0], c[0]), dy = __fsub_rn(a[1], c[1]), dz = __fsub_rn(a[2], c[2]);
      dmin = nanminf(dmin, __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz))));
    }
    dmin = warp_reduce<float>(dmin, nanminf);
    if (lane == 0) valid[b] = dmin < 9999999.f;
  }
  for (int h = 0; h < 2; ++h) {
    const float* vs = (h ? vr : vl) + (size_t)b * HAND_V * 3;
    for (int i = lane; i < HAND_V; i += 32) {
      float p[3];
      double uv[2];
      cam_xform(vs + 3 * i, R, t, p);
      project(p, K, uv);
      const size_t o = ((size_t)b * 2 + h) * HAND_V + i;
      if (v3d) { v3d[3 * o] = p[0]; v3d[3 * o + 1] = p[1]; v3d[3 * o + 2] = p[2]; }
      v2d[2 * o] = uv[0]; v2d[2 * o + 1] = uv[1];
    }
    const float* js = h ? jr : jl;
    if (js && lane < HAND_J) {
      float p[3];
      double uv[2];
      cam_xform(js + ((size_t)b * HAND_J + lane) * 3, R, t, p);
      project(p, K, uv);
      const size_t o = ((size_t)b * 2 + h) * HAND_J + lane;
      if (j3d) { j3d[3 * o] = p[0]; j3d[3 * o + 1] = p[1]; j3d[3 * o + 2] = p[2]; }
      if (j2d) { j2d[2 * o] = uv[0]; j2d[2 * o + 1] = uv[1]; }
    }
  }
  double* Kb = Kout ? Kout + (size_t)b * 9 : nullptr;
  if (Kb && lane == 0)
    for (int k = 0; k < 9; ++k) Kb[k] = K[k];
  __syncwarp();
  if (crop) cut_frame(v2d + (size_t)b * 2 * HAND_V * 2, 2 * HAND_V, radio, img_size, Mout + (size_t)b * 6, cut2d ? cut2d + (size_t)b * 2 * HAND_V * 2 : nullptr, Kb);
}

__global__ void __launch_bounds__(256)
dsgen_cut_kernel(const double* __restrict__ pts, int B, int N, double radio, int img_size, double* __restrict__ Mout, double* __restrict__ cut,
                 double* __restrict__ K) {
  pdl_sync();
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  cut_frame(pts + (size_t)b * N * 2, N, radio, img_size, Mout + (size_t)b * 6, cut ? cut + (size_t)b * N * 2 : nullptr, K ? K + (size_t)b * 9 : nullptr);
}

// saturate_cast<int>((my*y + mc) * 1024) + 16 + saturate_cast<int>(mx*x*1024) >> 5: OpenCV's fixed-point source coordinate in 1/32 pixel
// (csrc/augment.cu states the rule); double products and sums rounded one at a time
__device__ __forceinline__ int fixed_coord(double mx, double my, double mc, int x, int y) {
  const int base = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(my, (double)y), mc), 1024.0)) + 16;
  const int delta = __double2int_rn(__dmul_rn(__dmul_rn(mx, (double)x), 1024.0));
  return (base + delta) >> 5;
}

__global__ void __launch_bounds__(256)
dsgen_crop_kernel(const unsigned char* __restrict__ src, int Hs, int Ws, const double* __restrict__ Mfwd, int S, unsigned char* __restrict__ dst,
                  unsigned long long* __restrict__ sums) {
  pdl_sync();
  const int b = blockIdx.y;
  const unsigned char* img = src + (size_t)b * Hs * Ws * 3;
  // cv::warpAffine inverts the forward matrix in double (imgwarp.cpp, without WARP_INVERSE_MAP)
  const double* f = Mfwd + (size_t)b * 6;
  double D = __dsub_rn(__dmul_rn(f[0], f[4]), __dmul_rn(f[1], f[3]));
  D = D != 0.0 ? __drcp_rn(D) : 0.0;
  const double a11 = __dmul_rn(f[4], D), a22 = __dmul_rn(f[0], D), a12 = __dmul_rn(f[1], -D), a21 = __dmul_rn(f[3], -D);
  const double b1 = __dsub_rn(__dmul_rn(-a11, f[2]), __dmul_rn(a12, f[5]));
  const double b2 = __dsub_rn(__dmul_rn(-a21, f[2]), __dmul_rn(a22, f[5]));
  const int total = S * S;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int x = i % S, y = i / S;
    const int X = fixed_coord(a11, a12, b1, x, y), Y = fixed_coord(a21, a22, b2, x, y);
    const int sx = max(-32768, min(32767, X >> 5)), sy = max(-32768, min(32767, Y >> 5)), fx = X & 31, fy = Y & 31;
    const int w[4] = {(32 - fy) * (32 - fx), (32 - fy) * fx, fy * (32 - fx), fy * fx};
    int acc[3] = {0, 0, 0};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int yy = sy + (k >> 1), xx = sx + (k & 1);
      if (yy >= 0 && yy < Hs && xx >= 0 && xx < Ws && w[k]) {
        const unsigned char* p = img + ((size_t)yy * Ws + xx) * 3;
        acc[0] += w[k] * p[0]; acc[1] += w[k] * p[1]; acc[2] += w[k] * p[2];
      }
    }
    unsigned char* q = dst + ((size_t)b * total + i) * 3;
    q[0] = (unsigned char)((acc[0] + 512) >> 10); q[1] = (unsigned char)((acc[1] + 512) >> 10); q[2] = (unsigned char)((acc[2] + 512) >> 10);
  }
  if (sums) {     // the exact integer sum of the source frame: img.mean() is this over Hs*Ws*3, divided in float64 (interhand.py:203)
    const long long nbytes = (long long)Hs * Ws * 3;
    unsigned long long acc = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nbytes; i += (long long)gridDim.x * blockDim.x) acc += img[i];
#pragma unroll
    for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    __shared__ unsigned long long part[8];
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long s = 0;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += part[w];
      atomicAdd(sums + b, s);
    }
  }
}

__device__ __forceinline__ unsigned char sat_u8(float v) {    // saturate_cast<uchar>(float): round half to even, NaN -> 0
  if (!(v == v)) return 0;
  return (unsigned char)fminf(fmaxf(rintf(v), 0.f), 255.f);
}

__global__ void __launch_bounds__(256)
dsgen_heatmap_kernel(const double* __restrict__ joints, long long B, int N, int res, double denom, float* __restrict__ hms,
                     unsigned char* __restrict__ planes) {
  pdl_sync();
  const long long plane = (long long)res * res, total = B * N * plane;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int col = (int)(i % res), row = (int)((i / res) % res);
    const long long bn = i / plane;
    const double* pt = joints + bn * 3;
    float v = 0.f;
    const double x = pt[0], y = pt[1];
    if (pt[2] > 0 && !(x < 0 || y < 0 || x >= res || y >= res)) {
      const double dx = __dsub_rn((double)col, x), dy = __dsub_rn((double)row, y);
      v = (float)exp(__ddiv_rn(-__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), denom));
    }
    if (hms) hms[i] = v;
    if (planes) {     // hms[k].transpose(1, 2, 0) * 255 for k = n / 3, channel n % 3
      const long long b = bn / N;
      const int n = (int)(bn % N);
      planes[(((b * (N / 3) + n / 3) * res + row) * res + col) * 3 + n % 3] = sat_u8(__fmul_rn(v, 255.f));
    }
  }
}

__global__ void __launch_bounds__(256) dsgen_scale_u8_kernel(const float* __restrict__ x, long long n, float scale, unsigned char* __restrict__ out) {
  pdl_sync();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) out[i] = sat_u8(__fmul_rn(x[i], scale));
}

}  // namespace

// interhand.py:198-215 / :268-280 and step7_gen_annotations.py:260-272 for B frames, one warp per frame, both hands.  vl, vr [B,778,3] and
// jl, jr [B,21,3] (jl / jr may be NULL) float32 MANO output; R [B,3,3] float32 cam_R, t [B,3] float32 cam_t, K [B,3,3] float64 cameraIn.
// Writes v2d [B,2,778,2] float64 (left hand first, always), and when not NULL: v3d [B,2,778,3] / j3d [B,2,21,3] float32 camera-frame
// coordinates, j2d [B,2,21,2] float64, valid [B] int32 (the dist test: 1 unless the minimum |left_i - right_i| is NaN or >= 9999999),
// Kout [B,3,3] float64 (K, updated by cut_img when crop).  crop = 1: cut_img(radio, img_size) over both hands' 2-D verts also writes
// M [B,6] float64 (the forward 2x3 matrix) and, when not NULL, cut2d [B,2,778,2] float64 (the 2-D verts mapped by M).
RIH_API int rih_dsgen_geometry(const float* vl, const float* vr, const float* jl, const float* jr, const float* R, const float* t, const double* K, int B,
                               int crop, double radio, int img_size, float* v3d, float* j3d, double* v2d, double* j2d, int* valid, double* M, double* Kout,
                               double* cut2d, cudaStream_t s) {
  RIH_REQUIRE(B >= 0 && vl && vr && R && t && K && v2d && (!crop || M) && (!(j3d || j2d) || (jl && jr)), "dsgen_geometry: bad arguments");
  if (B == 0) return 0;
  launch_k(dsgen_geometry_kernel, (B + 7) / 8, 256, 0, s, vl, vr, jl, jr, R, t, K, B, crop, radio, img_size, v3d, j3d, v2d, j2d, valid, M, Kout, cut2d);
  return check_launch("dsgen_geometry");
}

// dataset/dataset_utils.py:12-42 (cut_img) without the image: pts [B,N,2] float64 labels of a frame (every list concatenated) -> M [B,6]
// float64, cut [B,N,2] float64 mapped labels (may be NULL), and K [B,3,3] float64 updated in place (may be NULL).
RIH_API int rih_dsgen_cut(const double* pts, int B, int N, double radio, int img_size, double* M, double* cut, double* K, cudaStream_t s) {
  RIH_REQUIRE(B >= 0 && N >= 0 && pts && M, "dsgen_cut: bad arguments");
  if (B == 0) return 0;
  launch_k(dsgen_cut_kernel, (B + 7) / 8, 256, 0, s, pts, B, N, radio, img_size, M, cut, K);
  return check_launch("dsgen_cut");
}

// cv.warpAffine(img, M, (S, S)) (INTER_LINEAR, BORDER_CONSTANT 0; dataset_utils.py:28) for B frames, bit-exact with OpenCV's 8-bit path.
// src [B,Hs,Ws,3] uint8; M [B,6] float64 forward matrices; dst [B,S,S,3] uint8.  sums [B] (may be NULL): the exact integer sum of each
// source frame's bytes (img.mean() * Hs*Ws*3, interhand.py:203); the buffer is zeroed here before the launch.
RIH_API int rih_dsgen_crop_u8(const unsigned char* src, int B, int Hs, int Ws, const double* M, int S, unsigned char* dst, long long* sums, cudaStream_t s) {
  RIH_REQUIRE(B >= 0 && Hs > 0 && Ws > 0 && Hs <= 32767 && Ws <= 32767 && S > 0 && S <= 16384 && B <= 65535 && src && M && dst, "dsgen_crop_u8: bad arguments");
  if (B == 0) return 0;
  if (sums) RIH_REQUIRE(cudaMemsetAsync(sums, 0, (size_t)B * sizeof(long long), s) == cudaSuccess, "dsgen_crop_u8: memset failed");
  const long long work = std::max((long long)S * S, sums ? (long long)Hs * Ws * 3 / 4 : 0LL);
  const int gx = (int)std::min(64LL, (work + 255) / 256);
  launch_k(dsgen_crop_kernel, dim3(gx, B), 256, 0, s, src, Hs, Ws, M, S, dst, (unsigned long long*)sums);
  return check_launch("dsgen_crop_u8");
}

// HeatmapGenerator(res, sigma)(joints, scale) (dataset/heatmap.py:4-39).  joints [B,N,3] float64 (x, y, visibility); denom = 2 * sigma**2
// of the scaled sigma, evaluated by the caller as Python does.  A joint with visibility <= 0, or x < 0, y < 0, x >= res, y >= res, has an
// all-zero map; otherwise hm[row, col] = exp(-((col - x)**2 + (row - y)**2) / denom) in float64, stored as float32.  hms [B,N,res,res]
// float32 (may be NULL); planes [B,N/3,res,res,3] uint8 (may be NULL, N a multiple of 3): cv.imwrite's conversion of
// hms[k].transpose(1, 2, 0) * 255 (step7_gen_annotations.py:275-278; float32 product, round half to even, saturate).
RIH_API int rih_dsgen_heatmaps(const double* joints, long long B, int N, int res, double denom, float* hms, unsigned char* planes, cudaStream_t s) {
  RIH_REQUIRE(B >= 0 && N >= 0 && res > 0 && joints && (hms || planes) && (!planes || N % 3 == 0), "dsgen_heatmaps: bad arguments");
  const long long total = B * N * (long long)res * res;
  if (total == 0) return 0;
  const int grid = (int)std::min(ew_ctas(s), (total + 255) / 256);
  launch_k(dsgen_heatmap_kernel, grid, 256, 0, s, joints, B, N, res, denom, hms, planes);
  return check_launch("dsgen_heatmaps");
}

// cv.imwrite's conversion of a float32 image to 8 bits after `* scale` (step7_gen_annotations.py:282-288: the mask and dense map * 255):
// out[i] = saturate_cast<uchar>(x[i] * scale), the product in float32, round half to even, NaN -> 0.
RIH_API int rih_dsgen_scale_u8(const float* x, long long n, float scale, unsigned char* out, cudaStream_t s) {
  RIH_REQUIRE(n >= 0 && x && out, "dsgen_scale_u8: bad arguments");
  if (n == 0) return 0;
  const int grid = (int)std::min(ew_ctas(s), (n + 255) / 256);
  launch_k(dsgen_scale_u8_kernel, grid, 256, 0, s, x, n, scale, out);
  return check_launch("dsgen_scale_u8");
}
