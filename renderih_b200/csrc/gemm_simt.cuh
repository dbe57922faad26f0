// SIMT fp32 tiled GEMM core with pluggable operand loaders (dense / implicit-conv gathers).
//   C[m,n] (+)= sum_k A(m,k) * B(n,k)
// This is the exact-fp32 path (parity reference mode + shapes the wgmma path does not take).
#pragma once
#include "common.cuh"

namespace rih {
namespace tc { extern long long g_launch_counts[3]; }   // launch bookkeeping shared with the tensor-core path (gemm_tc.cu)

constexpr int GEMM_BK = 16;
constexpr int GEMM_THREADS = 256;

// ------------------------------------------------------------------ loaders
// K-contiguous dense operand: element(row,k) = p[row*ld + k]
struct DenseK {
  static constexpr bool K_CONTIG = true;
  const float* p; int ld; int rows; int vec;
  __device__ __forceinline__ float4 ld4(int row, int k, int klim) const {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row >= rows) return v;
    const float* q = p + (size_t)row * ld + k;
    if (vec && k + 3 < klim) return __ldg(reinterpret_cast<const float4*>(q));
    if (k < klim) v.x = __ldg(q);
    if (k + 1 < klim) v.y = __ldg(q + 1);
    if (k + 2 < klim) v.z = __ldg(q + 2);
    if (k + 3 < klim) v.w = __ldg(q + 3);
    return v;
  }
};
// MN-contiguous dense operand: element(row,k) = p[k*ld + row]; returns rows row..row+3
struct DenseMN {
  static constexpr bool K_CONTIG = false;
  const float* p; int ld; int rows; int vec;
  __device__ __forceinline__ float4 ld4(int row, int k, int klim) const {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (k >= klim || row >= rows) return v;
    const float* q = p + (size_t)k * ld + row;
    if (vec && row + 3 < rows) return __ldg(reinterpret_cast<const float4*>(q));
    v.x = __ldg(q);
    if (row + 1 < rows) v.y = __ldg(q + 1);
    if (row + 2 < rows) v.z = __ldg(q + 2);
    if (row + 3 < rows) v.w = __ldg(q + 3);
    return v;
  }
};

struct ConvGeom {
  int N, H, W, Cin, Ho, Wo, Cout, R, S, stride, pad;
  int ldx;   // row stride (floats) of the NHWC input  (>= Cin)
  int ldy;   // row stride (floats) of the NHWC output (>= Cout)
};

// forward A: rows = output pixels, k = (r,s,c); gathers the NHWC input.
struct ConvFwdA {
  static constexpr bool K_CONTIG = true;
  const float* x; ConvGeom g; int rows; int vec;
  __device__ __forceinline__ float ld1(int n, int oh, int ow, int k) const {
    int c = k % g.Cin; int rs = k / g.Cin; int s = rs % g.S; int r = rs / g.S;
    int ih = oh * g.stride - g.pad + r, iw = ow * g.stride - g.pad + s;
    if ((unsigned)ih >= (unsigned)g.H || (unsigned)iw >= (unsigned)g.W) return 0.f;
    return __ldg(x + ((size_t)(n * g.H + ih) * g.W + iw) * g.ldx + c);
  }
  __device__ __forceinline__ float4 ld4(int row, int k, int klim) const {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row >= rows || k >= klim) return v;
    int ow = row % g.Wo; int t = row / g.Wo; int oh = t % g.Ho; int n = t / g.Ho;
    if (vec && k + 3 < klim) {
      int c = k % g.Cin; int rs = k / g.Cin; int s = rs % g.S; int r = rs / g.S;
      int ih = oh * g.stride - g.pad + r, iw = ow * g.stride - g.pad + s;
      if ((unsigned)ih >= (unsigned)g.H || (unsigned)iw >= (unsigned)g.W) return v;
      return __ldg(reinterpret_cast<const float4*>(x + ((size_t)(n * g.H + ih) * g.W + iw) * g.ldx + c));
    }
    v.x = ld1(n, oh, ow, k);
    if (k + 1 < klim) v.y = ld1(n, oh, ow, k + 1);
    if (k + 2 < klim) v.z = ld1(n, oh, ow, k + 2);
    if (k + 3 < klim) v.w = ld1(n, oh, ow, k + 3);
    return v;
  }
};

// dgrad A: rows = input pixels, k = (r,s,co); gathers dY.
struct ConvDgradA {
  static constexpr bool K_CONTIG = true;
  const float* dy; ConvGeom g; int rows; int vec;
  __device__ __forceinline__ const float* addr(int n, int ih, int iw, int k) const {
    int co = k % g.Cout; int rs = k / g.Cout; int s = rs % g.S; int r = rs / g.S;
    int a = ih + g.pad - r, b = iw + g.pad - s;
    if (a < 0 || b < 0) return nullptr;
    int oh = a / g.stride, ow = b / g.stride;
    if (oh * g.stride != a || ow * g.stride != b || oh >= g.Ho || ow >= g.Wo) return nullptr;
    return dy + ((size_t)(n * g.Ho + oh) * g.Wo + ow) * g.ldy + co;
  }
  __device__ __forceinline__ float ld1(int n, int ih, int iw, int k) const {
    const float* q = addr(n, ih, iw, k);
    return q ? __ldg(q) : 0.f;
  }
  __device__ __forceinline__ float4 ld4(int row, int k, int klim) const {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row >= rows || k >= klim) return v;
    int iw = row % g.W; int t = row / g.W; int ih = t % g.H; int n = t / g.H;
    if (vec && k + 3 < klim) {
      const float* q = addr(n, ih, iw, k);
      if (!q) return v;
      return __ldg(reinterpret_cast<const float4*>(q));
    }
    v.x = ld1(n, ih, iw, k);
    if (k + 1 < klim) v.y = ld1(n, ih, iw, k + 1);
    if (k + 2 < klim) v.z = ld1(n, ih, iw, k + 2);
    if (k + 3 < klim) v.w = ld1(n, ih, iw, k + 3);
    return v;
  }
};
// dgrad B: rows = c (contiguous), k = (r,s,co); weights are [Cout][R][S][Cin].
struct ConvDgradB {
  static constexpr bool K_CONTIG = false;
  const float* w; ConvGeom g; int rows; int vec;
  __device__ __forceinline__ float4 ld4(int row, int k, int klim) const {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (k >= klim || row >= rows) return v;
    int co = k % g.Cout; int rs = k / g.Cout;  // rs = r*S+s
    const float* q = w + ((size_t)co * g.R * g.S + rs) * g.Cin + row;
    if (vec && row + 3 < rows) return __ldg(reinterpret_cast<const float4*>(q));
    v.x = __ldg(q);
    if (row + 1 < rows) v.y = __ldg(q + 1);
    if (row + 2 < rows) v.z = __ldg(q + 2);
    if (row + 3 < rows) v.w = __ldg(q + 3);
    return v;
  }
};
// wgrad B: rows = (r,s,c) (c contiguous), k = output pixel; gathers the NHWC input.
struct ConvWgradB {
  static constexpr bool K_CONTIG = false;
  const float* x; ConvGeom g; int rows; int vec;
  __device__ __forceinline__ float4 ld4(int row, int k, int klim) const {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (k >= klim || row >= rows) return v;
    int ow = k % g.Wo; int t = k / g.Wo; int oh = t % g.Ho; int n = t / g.Ho;
    if (vec) {
      int c = row % g.Cin; int rs = row / g.Cin; int s = rs % g.S; int r = rs / g.S;
      int ih = oh * g.stride - g.pad + r, iw = ow * g.stride - g.pad + s;
      if ((unsigned)ih >= (unsigned)g.H || (unsigned)iw >= (unsigned)g.W) return v;
      return __ldg(reinterpret_cast<const float4*>(x + ((size_t)(n * g.H + ih) * g.W + iw) * g.ldx + c));
    }
    float* pv = reinterpret_cast<float*>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int rr = row + i;
      if (rr >= rows) break;
      int c = rr % g.Cin; int rs = rr / g.Cin; int s = rs % g.S; int r = rs / g.S;
      int ih = oh * g.stride - g.pad + r, iw = ow * g.stride - g.pad + s;
      if ((unsigned)ih < (unsigned)g.H && (unsigned)iw < (unsigned)g.W)
        pv[i] = __ldg(x + ((size_t)(n * g.H + ih) * g.W + iw) * g.ldx + c);
    }
    return v;
  }
};

// ------------------------------------------------------------------ epilogue
struct Epilogue {
  float* c; int ldc; int M, N;
  const float* bias;  // per-n, may be null
  int relu;
  int mode;  // 0 = store, 1 = accumulate (c += v), 2 = atomicAdd (split-K)
  const float* res; int ldres;                 // optional residual added after activation/dropout
  const unsigned long long* seed_ptr;          // dropout: device-resident base seed (CUDA-graph friendly)
  unsigned long long site; uint32_t thresh; float inv_keep;
  float scale;                                 // accumulator scale applied first (1 = none; bias-compensated truncating TF32 uses 1 + 7.05e-4)
  double* stats;                               // optional [2*N] column sum / sum of squares of the stored values (fused BatchNorm statistics)
  int s2_w2, s2_h2, s2_ph, s2_pw;              // tensor-core stride-2 dgrad (s2_w2 > 0): the tile's 128 rows are pixels (n, i, j) of the half-resolution grid
                                               // s2_h2 x s2_w2; they are stored to input pixels (2 i + s2_ph, 2 j + s2_pw) through an element-strided 4-D map
  int nv_pad, nv_real;                         // tensor-core wgrad with Cin % BN != 0: column n of the (virtual) tile grid is (tap = n / nv_pad, c = n % nv_pad), stored iff c < nv_real
  const float* col_scale; const float* col_shift;   // optional per-column affine (an eval-mode BatchNorm folded into the producing convolution):
  int affine_post;                             //   0: applied to the accumulator BEFORE bias / ReLU (torchvision order Conv -> BN -> (+res) -> ReLU)
                                               //   1: applied AFTER the ReLU (repo order Conv -> ReLU -> BN)
  int relu_post;                               // ReLU after the residual add (the block's final activation)
  int opt;                                     // tensor-core persistent epilogue: bit 0 = residual rows prefetched a chunk ahead, bit 1 = column vectors cached in shared memory, bit 2 = the producer warp issues a k-block's TMA boxes from all lanes (rih_set_epilogue_opt)
  __device__ __forceinline__ void store4(int m, int n, float4 v) const {
    if (m >= M || n >= N) return;
    float* q = c + (size_t)m * ldc + n;
    float r[4] = {v.x, v.y, v.z, v.w};
    unsigned long long seed = thresh ? (*seed_ptr + site * 0xD1B54A32D192ED03ull) : 0ull;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (n + i >= N) break;
      float t = r[i] * scale;
      if (col_scale && !affine_post) t = fmaf(t, __ldg(col_scale + n + i), __ldg(col_shift + n + i));
      if (bias) t += __ldg(bias + n + i);
      if (relu) t = fmaxf(t, 0.f);
      if (col_scale && affine_post) t = fmaf(t, __ldg(col_scale + n + i), __ldg(col_shift + n + i));
      if (thresh) t *= dropout_scale(seed, (uint64_t)m * N + n + i, thresh, inv_keep);
      if (res) t += __ldg(res + (size_t)m * ldres + n + i);
      if (relu_post) t = fmaxf(t, 0.f);
      if (mode == 0) q[i] = t;
      else if (mode == 1) q[i] += t;
      else atomicAdd(q + i, t);
    }
  }
};
static inline Epilogue make_epilogue(float* c, int ldc, int M, int N, const float* bias, int relu, int mode) {
  Epilogue e; e.c = c; e.ldc = ldc; e.M = M; e.N = N; e.bias = bias; e.relu = relu; e.mode = mode;
  e.res = nullptr; e.ldres = 0; e.seed_ptr = nullptr; e.site = 0; e.thresh = 0; e.inv_keep = 1.f; e.stats = nullptr; e.scale = 1.f; e.nv_pad = 0; e.nv_real = 0; e.s2_w2 = 0; e.s2_h2 = 0; e.s2_ph = 0; e.s2_pw = 0;
  e.col_scale = nullptr; e.col_shift = nullptr; e.affine_post = 0; e.relu_post = 0; e.opt = 7;
  return e;
}

// ------------------------------------------------------------------ kernel
template <int BM, int BN, int TM, int TN, class AL, class BL>
__global__ void __launch_bounds__(GEMM_THREADS)
gemm_simt_kernel(AL al, BL bl, Epilogue ep, int K, int k_per_split) {
  pdl_sync();
  static_assert((BM / TM) * (BN / TN) == GEMM_THREADS, "tile/thread mismatch");
  static_assert(TM == 4 || TM == 8, "TM");
  static_assert(TN == 4 || TN == 8, "TN");
  constexpr int BK = GEMM_BK;
  constexpr int PAD = 4;
  __shared__ __align__(16) float As[2][BK][BM + PAD];
  __shared__ __align__(16) float Bs[2][BK][BN + PAD];

  const int tid = threadIdx.x;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int kbeg = blockIdx.z * k_per_split;
  const int kend = min(K, kbeg + k_per_split);
  const int ntiles = (kend - kbeg + BK - 1) / BK;

  // loader thread mappings
  constexpr int A_PASSES_K = BM / 64;                                  // K-contig: 64 rows/pass
  constexpr int A_TPK = BM / 4, A_KPP = GEMM_THREADS / A_TPK, A_PASSES_MN = BK / A_KPP;
  constexpr int B_PASSES_K = BN / 64;
  constexpr int B_TPK = BN / 4, B_KPP = GEMM_THREADS / B_TPK, B_PASSES_MN = BK / B_KPP;
  constexpr int A_NREG = AL::K_CONTIG ? A_PASSES_K : A_PASSES_MN;
  constexpr int B_NREG = BL::K_CONTIG ? B_PASSES_K : B_PASSES_MN;
  float4 ra[A_NREG], rb[B_NREG];

  auto gload = [&](int kt) {
    const int k0 = kbeg + kt * BK;
    if constexpr (AL::K_CONTIG) {
#pragma unroll
      for (int p = 0; p < A_PASSES_K; ++p)
        ra[p] = al.ld4(m0 + p * 64 + (tid >> 2), k0 + (tid & 3) * 4, kend);
    } else {
#pragma unroll
      for (int p = 0; p < A_PASSES_MN; ++p)
        ra[p] = al.ld4(m0 + (tid % A_TPK) * 4, k0 + p * A_KPP + tid / A_TPK, kend);
    }
    if constexpr (BL::K_CONTIG) {
#pragma unroll
      for (int p = 0; p < B_PASSES_K; ++p)
        rb[p] = bl.ld4(n0 + p * 64 + (tid >> 2), k0 + (tid & 3) * 4, kend);
    } else {
#pragma unroll
      for (int p = 0; p < B_PASSES_MN; ++p)
        rb[p] = bl.ld4(n0 + (tid % B_TPK) * 4, k0 + p * B_KPP + tid / B_TPK, kend);
    }
  };
  auto sstore = [&](int buf) {
    if constexpr (AL::K_CONTIG) {
#pragma unroll
      for (int p = 0; p < A_PASSES_K; ++p) {
        int r = p * 64 + (tid >> 2), kq = (tid & 3) * 4;
        As[buf][kq + 0][r] = ra[p].x; As[buf][kq + 1][r] = ra[p].y;
        As[buf][kq + 2][r] = ra[p].z; As[buf][kq + 3][r] = ra[p].w;
      }
    } else {
#pragma unroll
      for (int p = 0; p < A_PASSES_MN; ++p)
        *reinterpret_cast<float4*>(&As[buf][p * A_KPP + tid / A_TPK][(tid % A_TPK) * 4]) = ra[p];
    }
    if constexpr (BL::K_CONTIG) {
#pragma unroll
      for (int p = 0; p < B_PASSES_K; ++p) {
        int r = p * 64 + (tid >> 2), kq = (tid & 3) * 4;
        Bs[buf][kq + 0][r] = rb[p].x; Bs[buf][kq + 1][r] = rb[p].y;
        Bs[buf][kq + 2][r] = rb[p].z; Bs[buf][kq + 3][r] = rb[p].w;
      }
    } else {
#pragma unroll
      for (int p = 0; p < B_PASSES_MN; ++p)
        *reinterpret_cast<float4*>(&Bs[buf][p * B_KPP + tid / B_TPK][(tid % B_TPK) * 4]) = rb[p];
    }
  };

  const int tx = tid % (BN / TN), ty = tid / (BN / TN);
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  if (ntiles > 0) {
    gload(0);
    sstore(0);
  }
  __syncthreads();
  for (int kt = 0; kt < ntiles; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < ntiles) gload(kt + 1);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[TM], b[TN];
      *reinterpret_cast<float4*>(&a[0]) = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      if constexpr (TM == 8)
        *reinterpret_cast<float4*>(&a[4]) = *reinterpret_cast<const float4*>(&As[buf][k][BM / 2 + ty * 4]);
      *reinterpret_cast<float4*>(&b[0]) = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      if constexpr (TN == 8)
        *reinterpret_cast<float4*>(&b[4]) = *reinterpret_cast<const float4*>(&Bs[buf][k][BN / 2 + tx * 4]);
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < ntiles) sstore(buf ^ 1);
    __syncthreads();
  }

#pragma unroll
  for (int i = 0; i < TM; ++i) {
    int m = m0 + ((i < 4) ? ty * 4 + i : BM / 2 + ty * 4 + (i - 4));
#pragma unroll
    for (int jj = 0; jj < TN / 4; ++jj) {
      int n = n0 + (jj == 0 ? tx * 4 : BN / 2 + tx * 4);
      ep.store4(m, n, make_float4(acc[i][jj * 4 + 0], acc[i][jj * 4 + 1], acc[i][jj * 4 + 2], acc[i][jj * 4 + 3]));
    }
  }
}

// Host-side launcher: picks the tile config and split-K.
template <class AL, class BL>
int launch_gemm_simt(const AL& al, const BL& bl, Epilogue ep, int M, int N, int K, int allow_splitk,
                     cudaStream_t stream, const char* what) {
  if (M <= 0 || N <= 0) return 0;
  tc::g_launch_counts[2]++;
  long long tiles_big = (long long)cdiv(M, 128) * cdiv(N, 128);
  bool big = (tiles_big >= 120) && N >= 96;
  int BM = big ? 128 : 64, BN = big ? 128 : 64;
  long long tiles = (long long)cdiv(M, BM) * cdiv(N, BN);
  int splits = 1;
  if (allow_splitk && tiles < 296 && K >= 512) {
    splits = (int)((296 + tiles - 1) / tiles);
    int maxs = K / 256;
    if (splits > maxs) splits = maxs;
    if (splits > 64) splits = 64;
    if (splits < 1) splits = 1;
  }
  int kps = cdiv(K, splits);
  kps = ((kps + GEMM_BK - 1) / GEMM_BK) * GEMM_BK;
  splits = cdiv(K, kps);
  if (splits > 1) {
    if (ep.mode == 0) {
      // zero then atomically accumulate (bias/relu are not allowed with split-K)
      if (ep.ldc == N) {
        cudaMemsetAsync(ep.c, 0, (size_t)M * N * sizeof(float), stream);
      } else {
        cudaMemset2DAsync(ep.c, (size_t)ep.ldc * sizeof(float), 0, (size_t)N * sizeof(float), M, stream);
      }
    }
    ep.mode = 2;
  }
  dim3 grid(cdiv(N, BN), cdiv(M, BM), splits);
  if (grid.y > 65535) { set_error("%s: M too large for grid.y", what); return 1; }
  if (big)
    launch_k(gemm_simt_kernel<128, 128, 8, 8, AL, BL>, grid, GEMM_THREADS, 0, stream, al, bl, ep, K, kps);
  else
    launch_k(gemm_simt_kernel<64, 64, 4, 4, AL, BL>, grid, GEMM_THREADS, 0, stream, al, bl, ep, K, kps);
  return check_launch(what);
}

}  // namespace rih
