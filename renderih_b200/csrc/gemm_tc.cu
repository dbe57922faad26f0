// Host launchers + C-ABI for the wgmma TF32 GEMM / implicit-GEMM convolution (see gemm_tc.cuh).
#include "gemm_tc.cuh"

namespace rih {
namespace tc {

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
      return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

int make_tmap_2d(CUtensorMap* map, const float* base, long long rows, long long cols, long long ld, int box_rows, bool atom32) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return 1; }
  if ((reinterpret_cast<uintptr_t>(base) & 15) || (ld % 4)) { set_error("tensor map: base/ld not 16-byte aligned"); return 1; }
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * sizeof(float)};
  cuuint32_t box[2] = {32u, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1u, 1u};
  CUresult r = CUDA_SUCCESS;
  for (int attempt = 0; attempt < 2; ++attempt) {
    r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
           CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_ERROR_INVALID_CONTEXT) break;
    cudaFree(0);   // this thread (e.g. an autograd worker) has no driver context bound yet: let the runtime bind the primary one
  }
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%lld ld=%lld", (int)r, rows, cols, ld); return 1; }
  return 0;
}

int make_tmap_2d_grouped(CUtensorMap* map, const float* base, long long rows, long long cols, long long ld, int groups) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return 1; }
  if ((reinterpret_cast<uintptr_t>(base) & 15) || (ld % 4) || (cols % 32)) { set_error("tensor map (grouped): base/ld not 16-byte aligned or cols %% 32 != 0"); return 1; }
  cuuint64_t dims[3] = {32u, (cuuint64_t)rows, (cuuint64_t)(cols / 32)};
  cuuint64_t strides[2] = {(cuuint64_t)ld * sizeof(float), 128u};
  cuuint32_t box[3] = {32u, 32u, (cuuint32_t)groups};
  cuuint32_t estr[3] = {1u, 1u, 1u};
  CUresult r = CUDA_SUCCESS;
  for (int attempt = 0; attempt < 2; ++attempt) {
    r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, estr,
           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_ERROR_INVALID_CONTEXT) break;
    cudaFree(0);
  }
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(grouped) failed (%d) rows=%lld cols=%lld ld=%lld groups=%d", (int)r, rows, cols, ld, groups); return 1; }
  return 0;
}

int make_tmap_nhwc(CUtensorMap* map, const float* base, int N, int H, int W, int C, long long ld, int bw, int bh, int bn, bool atom32, int estride) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return 1; }
  if ((reinterpret_cast<uintptr_t>(base) & 15) || (ld % 4)) { set_error("tensor map: base/ld not 16-byte aligned"); return 1; }
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)ld * 4, (cuuint64_t)W * ld * 4, (cuuint64_t)H * W * ld * 4};
  // with a traversal stride e the box extent is given in traversed elements: bw * e positions yield bw fetched pixels
  cuuint32_t box[4] = {32u, (cuuint32_t)(bw * estride), (cuuint32_t)(bh * estride), (cuuint32_t)bn};
  cuuint32_t estr[4] = {1u, (cuuint32_t)estride, (cuuint32_t)estride, 1u};
  if (box[1] > 256u || box[2] > 256u) { set_error("tensor map (nhwc, element stride %d): box %u x %u exceeds 256", estride, box[1], box[2]); return 1; }
  CUresult r = CUDA_SUCCESS;
  for (int attempt = 0; attempt < 2; ++attempt) {
    r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(base), dims, strides, box, estr,
           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
           CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_ERROR_INVALID_CONTEXT) break;
    cudaFree(0);
  }
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(4d) failed (%d) N=%d H=%d W=%d C=%d ld=%lld box=%d,%d,%d", (int)r, N, H, W, C, ld, bw, bh, bn); return 1; }
  return 0;
}

int make_tmap_nhwc_grouped(CUtensorMap* map, const float* base, int N, int H, int W, int C, long long ld, int bw, int bh, int estride, int groups) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return 1; }
  if ((reinterpret_cast<uintptr_t>(base) & 15) || (ld % 4) || (C % 32)) { set_error("tensor map (nhwc grouped): base/ld not 16-byte aligned or C %% 32 != 0"); return 1; }
  cuuint64_t dims[5] = {32u, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N, (cuuint64_t)(C / 32)};
  cuuint64_t strides[4] = {(cuuint64_t)ld * 4, (cuuint64_t)W * ld * 4, (cuuint64_t)H * W * ld * 4, 128u};
  cuuint32_t box[5] = {32u, (cuuint32_t)(bw * estride), (cuuint32_t)(bh * estride), 1u, (cuuint32_t)groups};
  cuuint32_t estr[5] = {1u, (cuuint32_t)estride, (cuuint32_t)estride, 1u, 1u};
  if (box[1] > 256u || box[2] > 256u) { set_error("tensor map (nhwc grouped, element stride %d): box %u x %u exceeds 256", estride, box[1], box[2]); return 1; }
  CUresult r = CUDA_SUCCESS;
  for (int attempt = 0; attempt < 2; ++attempt) {
    r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, const_cast<float*>(base), dims, strides, box, estr,
           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_ERROR_INVALID_CONTEXT) break;
    cudaFree(0);
  }
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(5d grouped) failed (%d) N=%d H=%d W=%d C=%d ld=%lld box=%d,%d groups=%d", (int)r, N, H, W, C, ld, bw, bh, groups); return 1; }
  return 0;
}

int make_tmap_stem(CUtensorMap* map, const float* base, int N, int Hp, int Wp, int Wo, int box_ow, bool atom32) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return 1; }
  if (reinterpret_cast<uintptr_t>(base) & 15) { set_error("tensor map (stem): base not 16-byte aligned"); return 1; }
  cuuint64_t dims[4] = {32u, (cuuint64_t)Wo, (cuuint64_t)Hp, (cuuint64_t)N};
  cuuint64_t strides[3] = {32u, (cuuint64_t)Wp * 16u, (cuuint64_t)Hp * Wp * 16u};     // bytes: 2 padded pixels, one padded row, one padded image
  cuuint32_t box[4] = {32u, (cuuint32_t)box_ow, 1u, 1u};
  cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
  CUresult r = CUDA_SUCCESS;
  for (int attempt = 0; attempt < 2; ++attempt) {
    r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
           CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_ERROR_INVALID_CONTEXT) break;
    cudaFree(0);
  }
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(stem, overlapping strides) failed (%d) N=%d Hp=%d Wp=%d Wo=%d", (int)r, N, Hp, Wp, Wo); return 1; }
  return 0;
}

// wgrad output dW[Cout][taps][Cin] as a 3-D map, box {32 channels, 1 tap, 128 filters}: a channel chunk is clipped at its own tap
int make_tmap_wgrad_out(CUtensorMap* map, const float* base, int Cout, int taps, int Cin) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return 1; }
  if ((reinterpret_cast<uintptr_t>(base) & 15) || (Cin % 4)) { set_error("tensor map (wgrad out): base/Cin not 16-byte aligned"); return 1; }
  cuuint64_t dims[3] = {(cuuint64_t)Cin, (cuuint64_t)taps, (cuuint64_t)Cout};
  cuuint64_t strides[2] = {(cuuint64_t)Cin * 4, (cuuint64_t)taps * Cin * 4};
  cuuint32_t box[3] = {32u, 1u, (cuuint32_t)BM};
  cuuint32_t estr[3] = {1u, 1u, 1u};
  CUresult r = CUDA_SUCCESS;
  for (int attempt = 0; attempt < 2; ++attempt) {
    r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
           CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_ERROR_INVALID_CONTEXT) break;
    cudaFree(0);
  }
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(wgrad out) failed (%d) Cout=%d taps=%d Cin=%d", (int)r, Cout, taps, Cin); return 1; }
  return 0;
}

int g_stats_fused = 0;            // set by the launcher when the epilogue accumulated ep.stats (fused BatchNorm statistics)
long long g_launch_counts[3] = {0, 0, 0};   // tensor-core launches with the TMA-store epilogue / with per-thread stores / SIMT GEMM launches (rih_gemm_launch_counts)
long long g_dgrad_t_launches = 0;           // transposed-output (OUT_T) launches (rih_gemm_dgrad_t_launches)
static int g_epi_opt = 7;        // Epilogue::opt of every launch (rih_set_epilogue_opt)
void set_epilogue_opt(int v) { g_epi_opt = v & 7; }
static int g_gemm_rs = 3;        // register-A main loops (rih_set_gemm_rs): bit 0 = the 3x3 / strided convolution weight gradients and the stem's,
                                 // bit 1 = transposed-output input gradients (dgrad_t) and every other MN-major A operand
void set_gemm_rs(int bits) { g_gemm_rs = bits & 3; }
template <int BN, bool A_MN, bool B_MN, class Producer, int NSPLIT, bool A_RS, bool OUT_T>
static int launch_one(const CUtensorMap& ta, const CUtensorMap& tb, Epilogue ep, const Producer& prod, int M, int N, int num_kb, int splits,
                      int kb_per_split, cudaStream_t s, const CUtensorMap* c_map = nullptr) {
  // TMA-store epilogue whenever the output is a 16-byte aligned matrix (a residual is read back row-wise by the epilogue threads when it is aligned too)
  CUtensorMap tc_;
  int tma_epi = 0;
  if (c_map) {       // caller-built output map (3-D wgrad view)
    tc_ = *c_map;
    tma_epi = 1;
  } else if ((!ep.res || (splits == 1 && ((reinterpret_cast<uintptr_t>(ep.res) & 15) == 0) && ep.ldres % 4 == 0 && N % 4 == 0)) &&
             ((reinterpret_cast<uintptr_t>(ep.c) & 15) == 0) && (ep.ldc % 4 == 0)) {
    if (make_tmap_2d(&tc_, ep.c, M, N, ep.ldc, BM)) return 1;
    tma_epi = 1;
  } else {
    tc_ = ta;
  }
  if (ep.col_scale && ep.bias) { set_error("gemm_tc: a folded per-column affine and a bias cannot be combined (fold the bias into the shift)"); return 1; }
  if (OUT_T && (!c_map || ep.bias || ep.relu || ep.res || ep.stats || ep.thresh || ep.col_scale || ep.relu_post || ep.mode > 1 || ep.nv_pad ||
                splits != 1)) {
    set_error("gemm_tc: the transposed-output epilogue only scales and stores / accumulates (no bias, activation, residual, dropout, statistics, split-K)");
    return 1;
  }
  g_launch_counts[tma_epi ? 0 : 1]++;
  if (OUT_T) g_dgrad_t_launches++;
  auto pk = gemm_tc_persistent_kernel<BN, A_MN, B_MN, Producer, NSPLIT, A_RS, OUT_T>;
  static bool pattr = false;
  if (!pattr) {
    if (cudaFuncSetAttribute(pk, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes<BN, NSPLIT>()) != cudaSuccess) {
      set_error("gemm_tc: cannot raise dynamic shared memory to %d", smem_bytes<BN, NSPLIT>());
      return 2;
    }
    pattr = true;
  }
  const int tiles_n = cdiv(N, BN), tiles_m = cdiv(M, BM);
  const long long total = (long long)tiles_n * tiles_m * splits;
  // persistent: at most one CTA per SM (fewer on a CTA-capped stream)
  const long long cap = stream_cta_limit(s, sm_count());
  const int ctas = (int)(total < cap ? total : cap);
  if (ep.stats && !(tma_epi && splits == 1)) ep.stats = nullptr;
  g_stats_fused = ep.stats != nullptr;
  launch_k(pk, dim3(ctas), dim3(persistent_threads<A_MN, B_MN, NSPLIT, A_RS>()), (size_t)smem_bytes<BN, NSPLIT>(), s, ta, tb, tc_, ep, prod, num_kb, kb_per_split,
           tiles_m, tiles_n, splits, tma_epi);
  return check_launch("gemm_tc_persistent");
}
static int g_nsplit = 1;   // set per call by the dispatchers below (1 = TF32, 2 = TF32 rn, 3 = 3xTF32)
static float g_scale = 1.f; // accumulator scale (bias-compensated truncating TF32)
void set_acc_scale(float s) { g_scale = s; }
template <int BN, bool A_MN, bool B_MN, class Producer, bool A_RS = false, bool OUT_T = false>
static int launch_cfg(const CUtensorMap& ta, const CUtensorMap& tb, Epilogue ep, const Producer& prod, int M, int N, int num_kb, int splits,
                      int kb_per_split, cudaStream_t s, const CUtensorMap* c_map = nullptr) {
  ep.scale = g_scale;
  ep.opt = g_epi_opt;
  if (g_nsplit == 3) return launch_one<BN, A_MN, B_MN, Producer, 3, A_RS, OUT_T>(ta, tb, ep, prod, M, N, num_kb, splits, kb_per_split, s, c_map);
  if (g_nsplit == 2) return launch_one<BN, A_MN, B_MN, Producer, 2, A_RS, OUT_T>(ta, tb, ep, prod, M, N, num_kb, splits, kb_per_split, s, c_map);
  return launch_one<BN, A_MN, B_MN, Producer, 1, A_RS, OUT_T>(ta, tb, ep, prod, M, N, num_kb, splits, kb_per_split, s, c_map);
}
void set_nsplit(int n) { g_nsplit = (n == 3) ? 3 : (n == 2 ? 2 : 1); }

// split-K planning over k-blocks of 32; switches the epilogue to atomic accumulation when splitting
static void plan_splitk(Epilogue& ep, int M, int N, int BN, int num_kb, int allow, int& splits, int& kb_per_split, cudaStream_t s, int N_grid = 0) {
  // N = real width of the output rows (what a split-K run has to zero); N_grid = width of the tile grid when it differs (padded wgrad taps)
  long long tiles = (long long)cdiv(M, BM) * cdiv(N_grid ? N_grid : N, BN);
  splits = 1;
  if (allow && tiles < sm_count() && num_kb >= 32) {
    splits = (int)((2 * sm_count() + tiles - 1) / tiles);
    int maxs = num_kb / 4;      // >= 4 k-blocks (128 reduction rows) per slice: these GEMMs are latency bound, so many short slices win
    if (splits > maxs) splits = maxs;
    if (splits > 128) splits = 128;
    if (splits < 1) splits = 1;
  }
  kb_per_split = cdiv(num_kb, splits);
  splits = cdiv(num_kb, kb_per_split);
  if (splits > 1) {
    if (ep.mode == 0) {
      if (ep.ldc == N) cudaMemsetAsync(ep.c, 0, (size_t)M * N * sizeof(float), s);
      else cudaMemset2DAsync(ep.c, (size_t)ep.ldc * sizeof(float), 0, (size_t)N * sizeof(float), M, s);
    }
    ep.mode = 2;
  }
}

// Transposed-output input gradients (rih_set_gemm_rs bit 1): c[rows, cols] (+)= dY . W computed as c^T = W^T dY^T, so that the weights are
// an MN-major A operand read into registers and dY a K-major B operand (see OUT_T in gemm_tc.cuh).  The 128 rows of such a tile are output
// columns (input channels / in-features): narrower outputs would leave rows empty and keep the untransposed product (measured per shape:
// tools/bench_dgrad.py).  The epilogue of the transposed form only scales and stores / accumulates into a 16-byte aligned output.
static bool dgrad_t(const Epilogue& ep, int cols) {
  return (g_gemm_rs & 2) && cols >= 128 &&
         ep.mode <= 1 && !ep.bias && !ep.relu && !ep.res && !ep.stats && !ep.thresh && !ep.col_scale && !ep.relu_post &&
         (reinterpret_cast<uintptr_t>(ep.c) & 15) == 0 && ep.ldc % 4 == 0;
}

// c[M, N] (+)= a[M, K] . b[K, N] (a K-major, b MN-major) as c^T = b^T a^T: b is the MN-major A operand of a register-A, transposed-output launch
static int gemm_tf32_t(const float* a, long long lda, const float* b, long long ldb, Epilogue ep, int M, int N, int K, cudaStream_t s) {
  CUtensorMap ta, tb, tcm;
  const int a_grp = N % 32 == 0 ? 1 : 0;
  if (a_grp ? make_tmap_2d_grouped(&ta, b, K, N, ldb, BM / 32) : make_tmap_2d(&ta, b, K, N, ldb, 32, true)) return 1;
  if (make_tmap_2d(&tb, a, M, K, lda, 128)) return 1;
  if (make_tmap_2d(&tcm, ep.c, M, N, ep.ldc, 128)) return 1;
  const int num_kb = cdiv(K, BK);
  DenseProducer<128, true, false> prod{0, 0ull, a_grp, 0};
  return launch_cfg<128, true, false, DenseProducer<128, true, false>, true, true>(ta, tb, ep, prod, N, M, num_kb, 1, num_kb, s, &tcm);
}

// a: K-major [M,K] (a_mn=0) or MN-major [K,M] (a_mn=1); b likewise with N.
int gemm_tf32(const float* a, long long lda, int a_mn, const float* b, long long ldb, int b_mn, Epilogue ep, int M, int N, int K,
              int allow_splitk, cudaStream_t s) {
  if (M <= 0 || N <= 0) return 0;
  if (a_mn == 0 && b_mn == 1 && !allow_splitk && dgrad_t(ep, N)) return gemm_tf32_t(a, lda, b, ldb, ep, M, N, K, s);
  CUtensorMap ta, tb;
  const int BN = (N > 64) ? 128 : 64;
  // MN-major operands with a multiple of 32 columns: ONE grouped box per k-block instead of BM / 32 (BN / 32) four-KB boxes
  const int a_grp = (a_mn && M % 32 == 0) ? 1 : 0, b_grp = (b_mn && N % 32 == 0) ? 1 : 0;
  if (a_mn ? (a_grp ? make_tmap_2d_grouped(&ta, a, K, M, lda, BM / 32) : make_tmap_2d(&ta, a, K, M, lda, 32, true)) : make_tmap_2d(&ta, a, M, K, lda, BM)) return 1;
  if (b_mn ? (b_grp ? make_tmap_2d_grouped(&tb, b, K, N, ldb, BN / 32) : make_tmap_2d(&tb, b, K, N, ldb, 32, true)) : make_tmap_2d(&tb, b, N, K, ldb, BN)) return 1;
  int num_kb = cdiv(K, BK), splits, kps;
  plan_splitk(ep, M, N, BN, num_kb, allow_splitk, splits, kps, s);
#define RIH_TC_CASE(bn, am, bm)                                                              \
  if (BN == bn && a_mn == am && b_mn == bm) {                                                \
    DenseProducer<bn, am != 0, bm != 0> prod{0, 0ull, a_grp, b_grp};                                             \
    return launch_cfg<bn, am != 0, bm != 0>(ta, tb, ep, prod, M, N, num_kb, splits, kps, s); \
  }
  // MN-major A (the weight gradients): read into registers by the consumers (rih_set_gemm_rs bit 1)
#define RIH_TC_CASE_RS(bn)                                                                                        \
  if ((g_gemm_rs & 2) && BN == bn && a_mn == 1 && b_mn == 1) {                                                    \
    DenseProducer<bn, true, true> prod{0, 0ull, a_grp, b_grp};                                                    \
    return launch_cfg<bn, true, true, DenseProducer<bn, true, true>, true>(ta, tb, ep, prod, M, N, num_kb, splits, kps, s); \
  }
  RIH_TC_CASE_RS(128) RIH_TC_CASE_RS(64)
#undef RIH_TC_CASE_RS
  RIH_TC_CASE(128, 0, 0) RIH_TC_CASE(64, 0, 0)
  RIH_TC_CASE(128, 0, 1) RIH_TC_CASE(64, 0, 1)
  RIH_TC_CASE(128, 1, 1) RIH_TC_CASE(64, 1, 1)
#undef RIH_TC_CASE
  set_error("gemm_tf32: unsupported configuration");
  return 1;
}

static int g_s2_direct = 1;      // stride-2 convolutions through element-strided tensor maps (no parity-stacked / zero-inserted copies); rih_set_s2_direct
void set_s2_direct(int on) { g_s2_direct = on ? 1 : 0; }
int s2_direct() { return g_s2_direct; }
static bool pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }

// Can the convolution run on the tensor-core implicit-GEMM path?
// stride 2 is supported for even H, W through a parity-stacked copy of the input (fwd, wgrad) and a zero-inserted copy of
// dY (dgrad); both need caller-provided workspace (conv_tc_workspace).
bool conv_tc_supported(const ConvGeom& g, int which /*0 fwd, 1 dgrad, 2 wgrad*/) {
  if (g.stride != 1 && g.stride != 2) return false;
  if (g.stride == 2 && ((g.H | g.W) & 1 || g.Ho * 2 != g.H || g.Wo * 2 != g.W || g.R != g.S || (g.R != 1 && g.R != 3) || g.pad != g.R / 2)) return false;
  // channel counts: multiples of 16 from 32 up (HRNet-w48's 48 / 96-wide branches included): a K block / N chunk that sticks out of the
  // tensor is zero-filled on load and clipped on store by the TMA unit
  if (g.Cin % 16 || g.Cout % 16 || g.Cin < 32 || g.Cout < 32) return false;
  if (g.ldx % 4 || g.ldy % 4) return false;
  if (which == 0) return pow2(g.Wo) && pow2(g.Ho) && g.Wo <= 128 && ((long long)g.N * g.Ho * g.Wo) % BM == 0 && (g.Wo * g.Ho >= BM || BM % (g.Wo * g.Ho) == 0);
  if (which == 1 && g.stride == 2 && g_s2_direct)     // four parity-class GEMMs over the half-resolution (= output) grid
    return pow2(g.Wo) && pow2(g.Ho) && g.Wo <= 128 && ((long long)g.N * g.Ho * g.Wo) % BM == 0 && (g.Wo * g.Ho >= BM || BM % (g.Wo * g.Ho) == 0);
  if (which == 1) return pow2(g.W) && pow2(g.H) && g.W <= 128 && ((long long)g.N * g.H * g.W) % BM == 0 && (g.W * g.H >= BM || BM % (g.W * g.H) == 0);
  return pow2(g.Wo) && pow2(g.Ho) && (g.Ho * g.Wo) % 32 == 0;
}

long long conv_tc_workspace(const ConvGeom& g, int which) {
  if (g.stride != 2 || g_s2_direct) return 0;
  if (which == 1) return (long long)g.N * g.H * g.W * g.Cout;   // zero-inserted dY
  return (long long)g.N * g.H * g.W * g.Cin;                    // parity-stacked x
}
extern "C" int rih_parity_stack(const float* x, int ldx, float* xp, int N, int H, int W, int C, cudaStream_t s);
extern "C" int rih_dilate2x(const float* y, int ldy, float* yd, int N, int Ho, int Wo, int C, cudaStream_t s);

int conv_fwd_tf32(const float* x, const float* w, Epilogue ep, const ConvGeom& g, float* ws, cudaStream_t s) {
  const int M = g.N * g.Ho * g.Wo;
  int BN = (g.Cout > 64) ? 128 : 64;
  const int tile_h = (BM / g.Wo) < g.Ho ? (BM / g.Wo) : g.Ho;
  const int tile_n = BM / (g.Wo * tile_h);
  CUtensorMap ta, tb;
  if (g.stride == 2 && g_s2_direct) {
    if (make_tmap_nhwc(&ta, x, g.N, g.H, g.W, g.Cin, g.ldx, g.Wo, tile_h, tile_n, false, 2)) return 1;
  } else if (g.stride == 2) {
    if (!ws) { set_error("conv_fwd_tf32: stride-2 path needs workspace"); return 1; }
    if (int e = rih_parity_stack(x, g.ldx, ws, g.N, g.H, g.W, g.Cin, s)) return e;
    if (make_tmap_nhwc(&ta, ws, 4 * g.N, g.H / 2, g.W / 2, g.Cin, g.Cin, g.Wo, tile_h, tile_n, false)) return 1;
  } else {
    if (make_tmap_nhwc(&ta, x, g.N, g.H, g.W, g.Cin, g.ldx, g.Wo, tile_h, tile_n, false)) return 1;
  }
  if (make_tmap_2d(&tb, w, g.Cout, (long long)g.R * g.S * g.Cin, (long long)g.R * g.S * g.Cin, BN)) return 1;
  ConvTcGeom cg{g.Cin, g.Cout, g.R, g.S, g.pad, g.H, g.W, g.Ho, g.Wo, tile_h, g.stride == 2 ? (g_s2_direct ? -1 : g.N) : 0, g.Cin};
  const int num_kb = g.R * g.S * cdiv(g.Cin, BK);
  if (BN == 128) { ConvFwdProducer<128> p{cg, 0ull}; return launch_cfg<128, false, false>(ta, tb, ep, p, M, g.Cout, num_kb, 1, num_kb, s); }
  ConvFwdProducer<64> p{cg, 0ull};
  return launch_cfg<64, false, false>(ta, tb, ep, p, M, g.Cout, num_kb, 1, num_kb, s);
}

// stride-2 dgrad as four dense parity-class GEMMs over the half-resolution grid (ConvDgradS2Producer), stored / accumulated in place through an
// element-strided map of dx.  Classes without a contributing tap (1x1 convolutions: three of four) are zero-filled unless the caller accumulates.
static int conv_dgrad_s2_direct(const float* dy, const float* w, Epilogue ep, const ConvGeom& g, cudaStream_t s) {
  const int H2 = g.Ho, W2 = g.Wo;                       // class grid == output grid (even H, W)
  const int M = g.N * H2 * W2;
  int BN = (g.Cin > 64) ? 128 : 64;
  const int tile_h = (BM / W2) < H2 ? (BM / W2) : H2;
  const int tile_n = BM / (W2 * tile_h);
  CUtensorMap ta, tb, tcm;
  if (make_tmap_nhwc(&ta, dy, g.N, g.Ho, g.Wo, g.Cout, g.ldy, W2, tile_h, tile_n, false)) return 1;
  // weights [Cout][R*S*Cin] as the MN-major B operand: one grouped box per k-block when Cin % 32 == 0
  const int b_grp = g.Cin % 32 == 0 ? 1 : 0;
  if (b_grp ? make_tmap_2d_grouped(&tb, w, g.Cout, (long long)g.R * g.S * g.Cin, (long long)g.R * g.S * g.Cin, BN / 32)
            : make_tmap_2d(&tb, w, g.Cout, (long long)g.R * g.S * g.Cin, (long long)g.R * g.S * g.Cin, 32, true)) return 1;
  if (make_tmap_nhwc(&tcm, ep.c, g.N, g.H, g.W, g.Cin, ep.ldc, W2, tile_h, tile_n, false, 2)) return 1;
  const int accumulate = ep.mode != 0;
  if (accumulate) { set_error("conv_dgrad_s2_direct: accumulation through an element-strided map is not supported (use the copy-based path)"); return 1; }
  // transposed form (dgrad_t): the weight map is the A operand, its grouped box holds the BM / 32 chunks of an m tile
  const bool tr = dgrad_t(ep, g.Cin);
  CUtensorMap tw;
  if (tr && (b_grp ? make_tmap_2d_grouped(&tw, w, g.Cout, (long long)g.R * g.S * g.Cin, (long long)g.R * g.S * g.Cin, BM / 32)
                   : make_tmap_2d(&tw, w, g.Cout, (long long)g.R * g.S * g.Cin, (long long)g.R * g.S * g.Cin, 32, true))) return 1;
  bool zeroed = false;
  for (int ph = 0; ph < 2; ++ph) for (int pw = 0; pw < 2; ++pw) {
    int nr = 0, ns = 0;
    for (int r = 0; r < g.R; ++r) if (((ph + g.pad - r) & 1) == 0) ++nr;
    for (int q = 0; q < g.S; ++q) if (((pw + g.pad - q) & 1) == 0) ++ns;
    if (nr * ns == 0) {
      if (!accumulate && !zeroed) {      // this class receives no gradient: zero the whole tensor once, the other classes overwrite their pixels
        if (ep.ldc == g.Cin) cudaMemsetAsync(ep.c, 0, (size_t)g.N * g.H * g.W * g.Cin * sizeof(float), s);
        else cudaMemset2DAsync(ep.c, (size_t)ep.ldc * sizeof(float), 0, (size_t)g.Cin * sizeof(float), (size_t)g.N * g.H * g.W, s);
        zeroed = true;
      }
      continue;
    }
  }
  for (int ph = 0; ph < 2; ++ph) for (int pw = 0; pw < 2; ++pw) {
    ConvTcGeom cg{g.Cin, g.Cout, g.R, g.S, g.pad, H2, W2, g.Ho, g.Wo, tile_h, 0, g.Cin};
    int nt = 0, tap[4], dr[4], ds[4];
    for (int r = 0; r < g.R; ++r) if (((ph + g.pad - r) & 1) == 0)
      for (int q = 0; q < g.S; ++q) if (((pw + g.pad - q) & 1) == 0) {
        if (nt >= 4) { set_error("conv_dgrad_s2: more than 4 taps per parity class (kernel %dx%d)", g.R, g.S); return 1; }
        tap[nt] = r * g.S + q; dr[nt] = (ph + g.pad - r) / 2; ds[nt] = (pw + g.pad - q) / 2; ++nt;
      }
    if (nt == 0) continue;
    Epilogue e2 = ep;
    e2.M = M; e2.s2_w2 = W2; e2.s2_h2 = H2; e2.s2_ph = ph; e2.s2_pw = pw;
    const int num_kb = nt * cdiv(g.Cout, BK);
    int rc;
#define RIH_S2_CASE(bn, t)                                                                                                        \
    ConvDgradS2Producer<bn, t> p{cg, nt, {tap[0], tap[1], tap[2], tap[3]}, {dr[0], dr[1], dr[2], dr[3]}, {ds[0], ds[1], ds[2], ds[3]}, b_grp};
    if (tr) {
      RIH_S2_CASE(128, true)
      rc = launch_cfg<128, true, false, ConvDgradS2Producer<128, true>, true, true>(tw, ta, e2, p, g.Cin, M, num_kb, 1, num_kb, s, &tcm);
    } else if (BN == 128) {
      RIH_S2_CASE(128, false)
      rc = launch_cfg<128, false, true>(ta, tb, e2, p, M, g.Cin, num_kb, 1, num_kb, s, &tcm);
    } else {
      RIH_S2_CASE(64, false)
      rc = launch_cfg<64, false, true>(ta, tb, e2, p, M, g.Cin, num_kb, 1, num_kb, s, &tcm);
    }
#undef RIH_S2_CASE
    if (rc) return rc;
  }
  return 0;
}

int conv_dgrad_tf32(const float* dy, const float* w, Epilogue ep, const ConvGeom& g0, float* ws, cudaStream_t s) {
  ConvGeom g = g0;
  if (g0.stride == 2 && g_s2_direct) return conv_dgrad_s2_direct(dy, w, ep, g0, s);
  if (g0.stride == 2) {   // zero-insert dY, then it is a stride-1 dgrad over an H x W "output"
    if (!ws) { set_error("conv_dgrad_tf32: stride-2 path needs workspace"); return 1; }
    if (int e = rih_dilate2x(dy, g0.ldy, ws, g0.N, g0.Ho, g0.Wo, g0.Cout, s)) return e;
    dy = ws; g.stride = 1; g.Ho = g0.H; g.Wo = g0.W; g.ldy = g0.Cout;
  }
  const int M = g.N * g.H * g.W;
  int BN = (g.Cin > 64) ? 128 : 64;
  const int tile_h = (BM / g.W) < g.H ? (BM / g.W) : g.H;
  const int tile_n = BM / (g.W * tile_h);
  CUtensorMap ta, tb;
  if (make_tmap_nhwc(&ta, dy, g.N, g.Ho, g.Wo, g.Cout, g.ldy, g.W, tile_h, tile_n, false)) return 1;
  // weights [Cout][R*S*Cin] as the MN-major B operand: one grouped box per k-block when Cin % 32 == 0
  const int b_grp = g.Cin % 32 == 0 ? 1 : 0;
  if (b_grp ? make_tmap_2d_grouped(&tb, w, g.Cout, (long long)g.R * g.S * g.Cin, (long long)g.R * g.S * g.Cin, BN / 32)
            : make_tmap_2d(&tb, w, g.Cout, (long long)g.R * g.S * g.Cin, (long long)g.R * g.S * g.Cin, 32, true)) return 1;
  ConvTcGeom cg{g.Cin, g.Cout, g.R, g.S, g.pad, g.H, g.W, g.Ho, g.Wo, tile_h, 0, g.Cin};
  const int num_kb = g.R * g.S * cdiv(g.Cout, BK);
  if (dgrad_t(ep, g.Cin)) {     // transposed form: A = the weight chunks of an m tile of input channels, B = the dY pixel box
    CUtensorMap tw, tcm;
    if (b_grp ? make_tmap_2d_grouped(&tw, w, g.Cout, (long long)g.R * g.S * g.Cin, (long long)g.R * g.S * g.Cin, BM / 32)
              : make_tmap_2d(&tw, w, g.Cout, (long long)g.R * g.S * g.Cin, (long long)g.R * g.S * g.Cin, 32, true)) return 1;
    if (make_tmap_2d(&tcm, ep.c, M, g.Cin, ep.ldc, 128)) return 1;
    ConvDgradProducer<128, true> p{cg, b_grp};
    return launch_cfg<128, true, false, ConvDgradProducer<128, true>, true, true>(tw, ta, ep, p, g.Cin, M, num_kb, 1, num_kb, s, &tcm);
  }
  if (BN == 128) { ConvDgradProducer<128> p{cg, b_grp}; return launch_cfg<128, false, true>(ta, tb, ep, p, M, g.Cin, num_kb, 1, num_kb, s); }
  ConvDgradProducer<64> p{cg, b_grp};
  return launch_cfg<64, false, true>(ta, tb, ep, p, M, g.Cin, num_kb, 1, num_kb, s);
}

// RGB stem as an implicit GEMM over the zero-bordered NHWC4 image xp[N][H+6][W+8][4] (see StemFwdProducer): y[N*Ho*Wo, 64] = X'[., 224] . w224^T
int stem_fwd_tf32(const float* xp, const float* w224, Epilogue ep, int N, int H, int W, cudaStream_t s) {
  const int Ho = H / 2, Wo = W / 2, M = N * Ho * Wo;
  if (Wo != BM || (H & 1) || (W & 1)) { set_error("stem_fwd_tf32: needs an even image with W / 2 == 128 (got %d x %d)", H, W); return 1; }
  CUtensorMap ta, tb;
  if (make_tmap_stem(&ta, xp, N, H + 6, W + 8, Wo, BM, false)) return 1;
  if (make_tmap_2d(&tb, w224, 64, 224, 224, 64)) return 1;
  StemFwdProducer<64> p{Ho, Wo};
  return launch_cfg<64, false, false>(ta, tb, ep, p, M, 64, 7, 1, 7, s);
}
// dw224[64, 224] (+)= dY[N*Ho*Wo, 64]^T . X'
int stem_wgrad_tf32(const float* dy, int lddy, const float* xp, Epilogue ep, int N, int H, int W, cudaStream_t s) {
  const int Ho = H / 2, Wo = W / 2, P = N * Ho * Wo;
  if (Wo % 32 || (H & 1) || (W & 1)) { set_error("stem_wgrad_tf32: needs an even image with W / 2 a multiple of 32"); return 1; }
  CUtensorMap ta, tb;
  if (make_tmap_2d(&ta, dy, P, 64, lddy, 32, true)) return 1;
  if (make_tmap_stem(&tb, xp, N, H + 6, W + 8, Wo, 32, true)) return 1;
  int num_kb = P / BK, splits, kps;
  plan_splitk(ep, 64, 224, 128, num_kb, 1, splits, kps, s);
  StemWgradProducer<128> p{Ho, Wo};
  if (g_gemm_rs & 1) return launch_cfg<128, true, true, StemWgradProducer<128>, true>(ta, tb, ep, p, 64, 224, num_kb, splits, kps, s);
  return launch_cfg<128, true, true>(ta, tb, ep, p, 64, 224, num_kb, splits, kps, s);
}

int conv_wgrad_tf32(const float* dy, const float* x, Epilogue ep, const ConvGeom& g, float* ws, cudaStream_t s) {
  const int P = g.N * g.Ho * g.Wo, taps = g.R * g.S, Nn = taps * g.Cin;
  // Cin a multiple of 32: the 32-column chunks of an N tile never straddle a tap, so 128-wide tiles may span several taps (Cin = 32, 64:
  // the dY operand is re-read once per N tile instead of once per tap and channel block).
  // Channel counts that are not multiples of 32 (HRNet's 48, 80, 208 ...) take the wide tiles too, on a "virtual" grid of cin32 = ceil32(Cin)
  // columns per tap: 48-channel convolutions would otherwise run nine 64-wide tiles (dY re-read 9 times); five 128-wide tiles over 9 x 64
  // virtual columns instead.
  const int cin32 = cdiv(g.Cin, 32) * 32;
  const bool wide_pad = g.Cin % 32 != 0 && g.Cin % 4 == 0 && taps * cin32 >= 128;
  const bool wide = (g.Cin % 32 == 0 || wide_pad) && Nn >= 128;
  const int BN = wide ? 128 : ((g.Cin % 128 == 0) ? 128 : 64);
  // N tiles never straddle a tap: each tap owns ceil(Cin / BN) tiles; when BN does not divide Cin (48, 96, ...) the tile grid is
  // "virtual" (cin_pad columns per tap) and the epilogue stores through a 3-D map [Cout][taps][Cin] that clips at the tap's edge
  const int cin_pad = wide ? cin32 : cdiv(g.Cin, BN) * BN, Ngrid = taps * cin_pad;
  const int bw = g.Wo < 32 ? g.Wo : 32, bh = 32 / bw;
  CUtensorMap ta, tb, tcm;
  const int a_grp = g.Cout % 32 == 0 ? 1 : 0;
  if (a_grp ? make_tmap_2d_grouped(&ta, dy, P, g.Cout, g.ldy, BM / 32) : make_tmap_2d(&ta, dy, P, g.Cout, g.ldy, 32, true)) return 1;
  // input chunks of one tap merged into grouped rank-5 boxes: b_grp = gcd(chunks per tap, 4) consecutive chunks per box
  int b_grp = 0;
  if (wide && !wide_pad && (g.stride == 1 || g_s2_direct)) {
    const int per_tap = g.Cin / 32;
    b_grp = (per_tap % 4 == 0) ? 4 : ((per_tap % 2 == 0) ? 2 : 0);
  }
  if (b_grp) {
    if (make_tmap_nhwc_grouped(&tb, x, g.N, g.H, g.W, g.Cin, g.ldx, bw, bh, g.stride == 2 ? 2 : 1, b_grp)) return 1;
  } else if (g.stride == 2 && g_s2_direct) {
    if (make_tmap_nhwc(&tb, x, g.N, g.H, g.W, g.Cin, g.ldx, bw, bh, 1, true, 2)) return 1;
  } else if (g.stride == 2) {
    if (!ws) { set_error("conv_wgrad_tf32: stride-2 path needs workspace"); return 1; }
    if (int e = rih_parity_stack(x, g.ldx, ws, g.N, g.H, g.W, g.Cin, s)) return e;
    if (make_tmap_nhwc(&tb, ws, 4 * g.N, g.H / 2, g.W / 2, g.Cin, g.Cin, bw, bh, 1, true)) return 1;
  } else {
    if (make_tmap_nhwc(&tb, x, g.N, g.H, g.W, g.Cin, g.ldx, bw, bh, 1, true)) return 1;
  }
  ConvTcGeom cg{g.Cin, g.Cout, g.R, g.S, g.pad, g.H, g.W, g.Ho, g.Wo, 0, g.stride == 2 ? (g_s2_direct ? -1 : g.N) : 0, cin_pad};
  int num_kb = P / BK, splits, kps;
  plan_splitk(ep, g.Cout, Nn, BN, num_kb, 1, splits, kps, s, Ngrid);
  const CUtensorMap* cmap = nullptr;
  if (cin_pad != g.Cin) {
    if (ep.ldc != Nn) { set_error("conv_wgrad_tf32: padded-tap path needs a dense dW"); return 1; }
    if (make_tmap_wgrad_out(&tcm, ep.c, g.Cout, taps, g.Cin)) return 1;
    cmap = &tcm; ep.nv_pad = cin_pad; ep.nv_real = g.Cin;
  }
  if (BN == 128) {
    ConvWgradProducer<128> p{cg, a_grp, wide ? b_grp : 0};
    if (g_gemm_rs & 1) return launch_cfg<128, true, true, ConvWgradProducer<128>, true>(ta, tb, ep, p, g.Cout, Ngrid, num_kb, splits, kps, s, cmap);
    return launch_cfg<128, true, true>(ta, tb, ep, p, g.Cout, Ngrid, num_kb, splits, kps, s, cmap);
  }
  ConvWgradProducer<64> p{cg, a_grp, 0};
  if (g_gemm_rs & 1) return launch_cfg<64, true, true, ConvWgradProducer<64>, true>(ta, tb, ep, p, g.Cout, Ngrid, num_kb, splits, kps, s, cmap);
  return launch_cfg<64, true, true>(ta, tb, ep, p, g.Cout, Ngrid, num_kb, splits, kps, s, cmap);
}

}  // namespace tc
}  // namespace rih

using namespace rih;

// Raw tensor-core GEMM entry point (testing / benchmarking of the tensor-core path in isolation):
//   c[M,N] (+)= op(a) * op(b)^T ; a_mn/b_mn select MN-major ([K,M] / [K,N] row-major) operands.
RIH_API int rih_gemm_tf32(const float* a, long long lda, int a_mn, const float* b, long long ldb, int b_mn, float* c, int ldc,
                          int M, int N, int K, const float* bias, int relu, int accumulate, int allow_splitk, int nsplit, cudaStream_t stream) {
  RIH_REQUIRE(M >= 0 && N > 0 && K > 0, "gemm_tf32: bad shape");
  RIH_REQUIRE(nsplit == 1 || nsplit == 2 || nsplit == 3, "gemm_tf32: nsplit must be 1 (TF32, truncating), 2 (TF32, round-to-nearest) or 3 (3xTF32)");
  tc::set_nsplit(nsplit);
  Epilogue ep = make_epilogue(c, ldc, M, N, bias, relu, accumulate ? 1 : 0);
  return tc::gemm_tf32(a, lda, a_mn, b, ldb, b_mn, ep, M, N, K, allow_splitk, stream);
}
