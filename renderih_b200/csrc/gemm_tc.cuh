// Hopper (sm_90a) TF32 GEMM: TMA -> 128B-swizzled shared memory -> wgmma.mma_async with the fp32 accumulator in registers of the
// consumer warpgroups -> shared-memory staging -> TMA-store epilogue.  Hand-written PTX, no CUTLASS.
//   D[M,N] (+)= A(M x K) * B(N x K)^T,  fp32 storage, TF32 multiplicands, fp32 accumulation.
// Operand tiles are [rows x 128 bytes] TMA boxes with SWIZZLE_128B; the same box format serves
//   K-major  operands (rows = M/N index, 32 consecutive k per row)          and
//   MN-major operands (rows = k index, 32 consecutive m/n per row; one box per 32-wide m/n chunk).
// wgmma reads TF32 shared-memory operands K-major only, so MN-major tiles are transposed in shared memory by a preparation warpgroup (which
// also rounds / splits the operands of the TF32-rn and 3xTF32 kernels) before the consumers multiply them -- except an MN-major A tile of an
// A_RS kernel, which the consumers load into registers for the register-A form of wgmma.
#pragma once
#include <cuda.h>
#include "common.cuh"
#include "gemm_simt.cuh"   // Epilogue

namespace rih {
namespace tc {

constexpr int BM = 128;          // two consumer warpgroups x wgmma M = 64
constexpr int BK = 32;           // fp32 elements per stage row = 128 bytes = one swizzle span
constexpr int WG_K = 8;          // tf32: 32 bytes per wgmma instruction

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {}
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, int c4, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, %6}], [%7];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4), "r"(smem_u32(bar))
      : "memory");
}
// L2 eviction-priority hints for streamed operands: an activation tile a GEMM reads once should not push the output of the previous
// kernel (which the next kernel is about to read) out of the 50 MB L2.
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void tma_load_2d_hint(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3}], [%4], %5;"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d_hint(void* dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, uint64_t* bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3, %4, %5}], [%6], %7;"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(smem_u32(bar))
      : "memory");
}
// TMA store of a [rows x 128 B] shared-memory tile (plain or += reduction); bulk-group completion.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(src)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_reduce_add_2d(const CUtensorMap* map, const void* src, int c0, int c1) {
  asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(src)), "r"(c0), "r"(c1) : "memory");
}
// 3-D variants (wgrad output viewed as [Cout][taps][Cin] so that a channel chunk is clipped at ITS tap's edge)
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, const void* src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_reduce_add_3d(const CUtensorMap* map, const void* src, int c0, int c1, int c2) {
  asm volatile("cp.reduce.async.bulk.tensor.3d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_reduce_add_4d(const CUtensorMap* map, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.reduce.async.bulk.tensor.4d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N> __device__ __forceinline__ void tma_store_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void epi_bar_sync(int wg = 0) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }

__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

// wgmma shared-memory matrix descriptor (sm_90), K-major SWIZZLE_128B: 8-row groups of 128-byte rows are 1024 B apart (stride byte
// offset); the leading byte offset is unused for swizzled K-major layouts.  A K step of 8 tf32 advances the start address by 32 B.
__device__ __forceinline__ uint64_t make_wgmma_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;          // layout type 1 = SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// d[64 x BN] += A(64 x 8, K-major smem) * B(BN x 8, K-major smem)^T; per thread BN / 2 fp32 accumulators in the wgmma D fragment layout
template <int BN> __device__ __forceinline__ void wgmma_tf32(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc);
template <> __device__ __forceinline__ void wgmma_tf32<64>(float (&d)[32], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc) : "memory");
}
template <> __device__ __forceinline__ void wgmma_tf32<128>(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc) : "memory");
}
// The same with A (64 x 8) from registers: per thread a[0..3] = rows (warp q) * 16 + lane / 4 + {0, 8, 0, 8}, k = lane % 4 + {0, 0, 4, 4}
template <int BN> __device__ __forceinline__ void wgmma_tf32_rs(float (&d)[BN / 2], const uint32_t (&a)[4], uint64_t bdesc);
template <> __device__ __forceinline__ void wgmma_tf32_rs<64>(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc) : "memory");
}
template <> __device__ __forceinline__ void wgmma_tf32_rs<128>(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc) : "memory");
}

// NSPLIT = 1: single-pass TF32 (the tensor core ignores the low mantissa bits of the fp32 operands).  NSPLIT = 2: single-pass TF32 with the
// operands rounded to nearest in shared memory first (unbiased, what cuDNN/cuBLAS TF32 do).  NSPLIT = 3: error-compensated "3xTF32": every
// operand tile is split in shared memory into hi = value rounded to TF32 and lo = value - hi (exact in fp32), and D += hi*hi + lo*hi + hi*lo
// (fp32-faithful).
template <int BN, int NSPLIT> __host__ __device__ constexpr int stage_bytes() { return (BM * 128 + BN * 128) * (NSPLIT == 3 ? 2 : 1); }
// accumulator staging: the consumers park the 128 x BN tile as BN / 32 SWIZZLE_128B [128 rows x 128 B] chunks, each the source of one TMA store
template <int BN> __host__ __device__ constexpr int acc_bytes() { return BM * BN * 4; }
// as many stages as fit next to the accumulator staging in the 227 KB an H100 CTA may use (at most 8)
template <int BN, int NSPLIT> __host__ __device__ constexpr int num_stages() {
  return (227 * 1024 - acc_bytes<BN>() - 3 * 1024) / stage_bytes<BN, NSPLIT>() > 8 ? 8 : (227 * 1024 - acc_bytes<BN>() - 3 * 1024) / stage_bytes<BN, NSPLIT>();
}
// Per-column epilogue vectors of the tile's BN columns cached in shared memory: [0] = multiplicative (folded BatchNorm scale), [1] = additive
// (bias or folded BatchNorm shift).  Every epilogue thread needs all 32 values of a chunk: 16 broadcast LDS.128 instead of 64 broadcast LDG.32.
template <int BN> __host__ __device__ constexpr int colvec_bytes() { return 2 * BN * 4; }
template <int BN, int NSPLIT> __host__ __device__ constexpr int smem_bytes() {
  return num_stages<BN, NSPLIT>() * stage_bytes<BN, NSPLIT>() + acc_bytes<BN>() + 256 + colvec_bytes<BN>() + 1024;
}

// ---------------------------------------------------------------- producers (TMA issue logic, one elected lane)
// Each producer loads, for k-block `kb`, the A tile (BM x 32) to `sa` and the B tile (BN x 32) to `sb`.
// Tiles are made of 128-byte rows; MN-major operands are split into 32-wide chunks of BK rows (4 KB apart).
template <int BN, bool A_MN, bool B_MN>
struct DenseProducer {
  // WIDE_OK: an MN-major operand is fetched as BM / 32 (or BN / 32) four-KB boxes per k-block; load<true> issues them from different lanes of
  // the producer warp (lanes 0 .. 3: A boxes, lanes 4 ..: B boxes) instead of one after the other from a single thread.  load<false>(.., 0) is the
  // single-thread form (fully unrolled).  K-major operands are one box each and stay with lane 0 / lane 1.
  static constexpr bool WIDE_OK = A_MN || B_MN;
  int kbeg;
  unsigned long long a_policy;   // L2 evict-first policy of the streamed activation operand (K-major A; K-major B = dY when A is MN-major, the transposed dgrad)
  // a_grp / b_grp != 0: the MN-major operand comes through a "grouped" rank-3 tensor map {32 columns of a group, k rows, column groups} whose box
  // {32, 32, BM/32 or BN/32} lands in shared memory as the same [group][k row][32] chunks -- ONE TMA operation per operand and k-block
  // instead of one per 32-column chunk (make_tmap_2d_grouped; needs a column count that is a multiple of 32)
  int a_grp, b_grp;
  __device__ __forceinline__ void set_policy(unsigned long long p) { a_policy = p; }
  template <bool W>
  __device__ __forceinline__ void load(const CUtensorMap* ta, const CUtensorMap* tb, int kb, int m0, int n0, int z, uint8_t* sa, uint8_t* sb, uint64_t* bar, int lane) const {
    const int k0 = kb * BK;
    if constexpr (!A_MN) { if (!W || lane == 0) tma_load_2d_hint(sa, ta, k0, m0, bar, a_policy); }
    else if (a_grp) { if (!W || lane == 0) tma_load_3d(sa, ta, 0, k0, m0 >> 5, bar); }
    else if constexpr (W) { if (lane < BM / 32) tma_load_2d(sa + lane * (BK * 128), ta, m0 + lane * 32, k0, bar); }
    else {
#pragma unroll
      for (int c = 0; c < BM / 32; ++c) tma_load_2d(sa + c * (BK * 128), ta, m0 + c * 32, k0, bar);
    }
    if constexpr (!B_MN) {
      if (!W || lane == BM / 32) { if (A_MN) tma_load_2d_hint(sb, tb, k0, n0, bar, a_policy); else tma_load_2d(sb, tb, k0, n0, bar); }
    }
    else if (b_grp) { if (!W || lane == BM / 32) tma_load_3d(sb, tb, 0, k0, n0 >> 5, bar); }
    else if constexpr (W) { const int c = lane - BM / 32; if (c >= 0 && c < BN / 32) tma_load_2d(sb + c * (BK * 128), tb, n0 + c * 32, k0, bar); }
    else {
#pragma unroll
      for (int c = 0; c < BN / 32; ++c) tma_load_2d(sb + c * (BK * 128), tb, n0 + c * 32, k0, bar);
    }
  }
};

struct ConvTcGeom {
  int Cin, Cout, R, S, pad;
  int H, W, Ho, Wo;        // input / output spatial size (stride 1 only)
  int tile_h;              // fwd/dgrad: rows of the 128-pixel tile (tile_w == full width); tile images = 128/(tile_w*tile_h)
  int s2_images;           // > 0: stride-2 convolution reading the parity-stacked input [4*N, H/2, W/2, C]; value = N
                           // -1 : stride-2 convolution reading the input IN PLACE through a tensor map with element strides {1, 2, 2, 1}
                           //      (the TMA unit fetches every second pixel of a box): coordinates are plain input pixels, no copy of the input
  int cin_pad;             // wgrad: columns per tap in the (virtual) N tile grid = ceil(Cin / BN) * BN (== Cin when BN divides Cin)
};
// stride 2: input row 2*o + r - pad = 2*(o + shift) + parity
__device__ __forceinline__ void s2_tap(int r, int pad, int& parity, int& shift) {
  const int t = r - pad;
  parity = t & 1;
  shift = (t - parity) >> 1;
}

// forward: A = shifted NHWC input boxes (4-D map {C,W,H,N}), B = weights [Cout][R*S*Cin] (K-major 2-D map)
template <int BN>
struct ConvFwdProducer {
  static constexpr bool WIDE_OK = false;     // one or two large boxes per k-block (+ a few weight chunks): issued by lane 0
  ConvTcGeom g;
  unsigned long long a_policy;
  __device__ __forceinline__ void set_policy(unsigned long long p) { a_policy = p; }
  template <bool W>
  __device__ __forceinline__ void load(const CUtensorMap* ta, const CUtensorMap* tb, int kb, int m0, int n0, int z, uint8_t* sa, uint8_t* sb, uint64_t* bar, int lane) const {
    // channel blocks per tap; when Cin % 32 != 0 the last block of a tap is partly out of bounds in the activation map (TMA zero
    // fill), which also cancels whatever the weight box picks up from the next tap's columns
    const int cpb = (g.Cin + BK - 1) / BK;
    const int tap = kb / cpb, c0 = (kb - tap * cpb) * BK;
    const int r = tap / g.S, s = tap - r * g.S;
    const int P = g.Ho * g.Wo;
    const int n = m0 / P, oh0 = (m0 - n * P) / g.Wo;
    if (g.s2_images < 0) {
      tma_load_4d(sa, ta, c0, s - g.pad, 2 * oh0 + r - g.pad, n, bar);
    } else if (g.s2_images > 0) {
      int ph, dh, pw, dw_;
      s2_tap(r, g.pad, ph, dh);
      s2_tap(s, g.pad, pw, dw_);
      tma_load_4d(sa, ta, c0, dw_, oh0 + dh, (ph * 2 + pw) * g.s2_images + n, bar);
    } else if (g.R == 1) {
      tma_load_4d_hint(sa, ta, c0, s - g.pad, oh0 + r - g.pad, n, bar, a_policy);    // single-tap only: a 3x3 re-reads every input tile nine times
    } else {
      tma_load_4d(sa, ta, c0, s - g.pad, oh0 + r - g.pad, n, bar);
    }
    tma_load_2d(sb, tb, tap * g.Cin + c0, n0, bar);
  }
};
// dgrad (stride 1): A = shifted dY boxes (4-D map over [N,Ho,Wo,Cout]), B = weights as MN-major chunks {32 c, 32 co}
// T (transposed output, dX^T = W^T dY^T): the same boxes with the roles swapped -- ta = the weight map, its chunks go to `sa` (A rows = m0 +
// 0..127 = input channels, an MN-major A tile that the consumers read into registers), tb = the dY map, its pixel box goes to `sb` (B rows =
// n0 + 0..127 = pixels, K-major: nothing to transpose).
template <int BN, bool T = false>
struct ConvDgradProducer {
  static constexpr bool WIDE_OK = false;     // one or two large boxes per k-block (+ a few weight chunks): issued by lane 0
  ConvTcGeom g;
  int b_grp;                                 // weights through a grouped rank-3 map: the 128 / 32 (T) or BN / 32 chunks of a k-block in ONE box (Cin % 32 == 0)
  __device__ __forceinline__ void set_policy(unsigned long long) {}
  template <bool W>
  __device__ __forceinline__ void load(const CUtensorMap* ta, const CUtensorMap* tb, int kb, int m0, int n0, int z, uint8_t* sa, uint8_t* sb, uint64_t* bar, int lane) const {
    const int cpb = (g.Cout + BK - 1) / BK;
    const int tap = kb / cpb, co0 = (kb - tap * cpb) * BK;
    const int r = tap / g.S, s = tap - r * g.S;
    const int P = g.H * g.W;
    const int p0 = T ? n0 : m0, c0 = T ? m0 : n0;       // first pixel / first input channel of the tile
    const int n = p0 / P, ih0 = (p0 - n * P) / g.W;
    tma_load_4d(T ? sb : sa, T ? tb : ta, co0, g.pad - s, ih0 + g.pad - r, n, bar);
    uint8_t* sw = T ? sa : sb;
    const CUtensorMap* tw = T ? ta : tb;
    if (b_grp) { tma_load_3d(sw, tw, 0, co0, (tap * g.Cin + c0) >> 5, bar); return; }
#pragma unroll
    for (int c = 0; c < (T ? BM : BN) / 32; ++c) tma_load_2d(sw + c * (BK * 128), tw, tap * g.Cin + c0 + c * 32, co0, bar);
  }
};
// dgrad of a stride-2 convolution, one PARITY CLASS of input pixels (ih, iw) = (2 i + ph, 2 j + pw): only the taps r = ph + pad (mod 2),
// s = pw + pad (mod 2) reach those pixels, from output pixel (i + dr, j + ds) with dr = (ph + pad - r) / 2.  Each class is a dense
// stride-1 problem over the half-resolution grid: A = dY boxes shifted by (dr, ds), B = that tap's weights (MN-major chunks), K = ntaps * Cout;
// the four classes together do a quarter of the multiply-adds of "zero-insert dY, then a stride-1 dgrad" and need no dilated copy.
// T: transposed output, operands swapped as in ConvDgradProducer.
template <int BN, bool T = false>
struct ConvDgradS2Producer {
  static constexpr bool WIDE_OK = false;     // one or two large boxes per k-block (+ a few weight chunks): issued by lane 0
  ConvTcGeom g;            // H, W = half-resolution grid of the class (= Ho, Wo of the convolution); tile_h as usual
  int ntaps;
  int tap[4], dr[4], ds[4];
  int b_grp;               // see ConvDgradProducer
  __device__ __forceinline__ void set_policy(unsigned long long) {}
  template <bool W>
  __device__ __forceinline__ void load(const CUtensorMap* ta, const CUtensorMap* tb, int kb, int m0, int n0, int z, uint8_t* sa, uint8_t* sb, uint64_t* bar, int lane) const {
    const int cpb = (g.Cout + BK - 1) / BK;
    const int ti = kb / cpb, co0 = (kb - ti * cpb) * BK;
    const int P = g.H * g.W;
    const int p0 = T ? n0 : m0, c0 = T ? m0 : n0;
    const int n = p0 / P, i0 = (p0 - n * P) / g.W;
    tma_load_4d(T ? sb : sa, T ? tb : ta, co0, ds[ti], i0 + dr[ti], n, bar);
    uint8_t* sw = T ? sa : sb;
    const CUtensorMap* tw = T ? ta : tb;
    if (b_grp) { tma_load_3d(sw, tw, 0, co0, (tap[ti] * g.Cin + c0) >> 5, bar); return; }
#pragma unroll
    for (int c = 0; c < (T ? BM : BN) / 32; ++c) tma_load_2d(sw + c * (BK * 128), tw, tap[ti] * g.Cin + c0 + c * 32, co0, bar);
  }
};
// wgrad: A = dY as MN-major chunks {32 co, 32 pixels}, B = shifted input boxes of 32 pixels as MN-major chunks {32 c, 32 pixels}.
// The N axis enumerates (tap, channel) in cin_pad-wide groups; every 32-column chunk of the N tile finds its OWN tap, so a tile may span
// several taps (Cin = 64: a 256-wide tile covers 4 taps and the dY tile is fetched 3 times instead of 9).
template <int BN>
struct ConvWgradProducer {
  static constexpr bool WIDE_OK = true;      // 4 dY boxes + BN / 32 input boxes (own tap, own coordinates each) of 4 KB per k-block: one lane per box
  ConvTcGeom g;
  int a_grp;                                 // dY through a grouped rank-3 map (one box per k-block), see DenseProducer
  int b_grp;                                 // > 0: the input through a grouped rank-5 map {32, W, H, N, Cin / 32}: one box fetches b_grp consecutive 32-channel
                                             // chunks of ONE tap (b_grp divides both the chunks per tap and the 8 chunks of a tile): BN / 32 / b_grp boxes per k-block
  __device__ __forceinline__ void set_policy(unsigned long long) {}
  template <bool W>
  __device__ __forceinline__ void load(const CUtensorMap* ta, const CUtensorMap* tb, int kb, int m0, int n0, int z, uint8_t* sa, uint8_t* sb, uint64_t* bar, int lane) const {
    const int p0 = kb * BK;
    const int P = g.Ho * g.Wo;
    const int n = p0 / P, rem = p0 - n * P;
    const int oh = rem / g.Wo, ow = rem - oh * g.Wo;
    const int taps = g.R * g.S;
    if (a_grp) { if (!W || lane == 0) tma_load_3d(sa, ta, 0, p0, m0 >> 5, bar); }
    else if constexpr (W) { if (lane < BM / 32) tma_load_2d(sa + lane * (BK * 128), ta, m0 + lane * 32, p0, bar); }
    else {
#pragma unroll
      for (int c = 0; c < BM / 32; ++c) tma_load_2d(sa + c * (BK * 128), ta, m0 + c * 32, p0, bar);
    }
    const int G = b_grp > 0 ? b_grp : 1;                  // chunks per box
#pragma unroll
    for (int c0 = 0; c0 < (W ? 1 : BN / 32); ++c0) {
      const int c = (W ? lane - BM / 32 : c0) * (W ? G : 1);
      if (W && (c < 0 || c >= BN / 32)) break;
      if (!W && (c % G) != 0) continue;
      const int col = n0 + c * 32;
      int tap = col / g.cin_pad, cbase = col - tap * g.cin_pad;
      if (tap >= taps) { tap = 0; cbase = g.cin_pad + 64; }      // beyond the last tap: a channel coordinate outside the tensor -> the TMA unit zero-fills
      const int r = tap / g.S, s = tap - r * g.S;
      int cw = ow + s - g.pad, ch = oh + r - g.pad, cn = n;
      if (g.s2_images < 0) { cw = 2 * ow + s - g.pad; ch = 2 * oh + r - g.pad; }
      else if (g.s2_images > 0) {
        int ph, dh, pw, dw_;
        s2_tap(r, g.pad, ph, dh);
        s2_tap(s, g.pad, pw, dw_);
        cw = ow + dw_; ch = oh + dh; cn = (ph * 2 + pw) * g.s2_images + n;
      }
      if (b_grp > 0) tma_load_5d(sb + c * (BK * 128), tb, 0, cw, ch, cn, cbase >> 5, bar);
      else tma_load_4d(sb + c * (BK * 128), tb, cbase, cw, ch, cn, bar);
    }
  }
};

// ---- RGB stem (conv1 7x7 / stride 2 / pad 3, 3 -> 64; torchvision ResNet, models/encoder.py:108) as an implicit GEMM without an im2col buffer.
// The image is stored once as zero-bordered NHWC4 P[n][H+6][W+8][4] (3 rows / columns of padding in front, RGB + one zero channel).  The 8
// horizontally adjacent padded pixels that filter row r sees for output pixel (oh, ow) -- columns 2 ow .. 2 ow + 7 of padded row 2 oh + r, i.e.
// taps s = 0 .. 6 plus one extra column that meets a zero weight -- are 32 CONTIGUOUS floats.  A 4-D tensor map with the (overlapping) strides
// {4 B, 32 B (= 2 pixels), row pitch, image pitch} and dims {32, Wo, H + 6, N} therefore presents them as a "virtual" NHWC tensor with 32
// channels per (row, ow), and the convolution becomes a 7-tap (R = 7, S = 1) implicit GEMM with K = 7 x 32 = 224 against weights repacked
// as [64][7][8][4]: one TMA box {32, 128 ow, 1, 1} per k-block, 128-byte rows, SWIZZLE_128B -- the same machinery as every other
// convolution.  An output tile is one output row (Wo = 128).
template <int BN>
struct StemFwdProducer {
  static constexpr bool WIDE_OK = false;     // one or two large boxes per k-block (+ a few weight chunks): issued by lane 0
  int Ho, Wo;
  __device__ __forceinline__ void set_policy(unsigned long long) {}
  template <bool W>
  __device__ __forceinline__ void load(const CUtensorMap* ta, const CUtensorMap* tb, int kb, int m0, int n0, int z, uint8_t* sa, uint8_t* sb, uint64_t* bar, int lane) const {
    const int P = Ho * Wo;
    const int n = m0 / P, oh = (m0 - n * P) / Wo;
    tma_load_4d(sa, ta, 0, 0, 2 * oh + kb, n, bar);       // filter row r = kb
    tma_load_2d(sb, tb, kb * 32, n0, bar);
  }
};
// weight gradient of the stem: dW[64][7 x 32] = sum over pixels dY^T . X', k-block = 32 consecutive output pixels of one output row
template <int BN>
struct StemWgradProducer {
  static constexpr bool WIDE_OK = true;
  int Ho, Wo;
  __device__ __forceinline__ void set_policy(unsigned long long) {}
  template <bool W>
  __device__ __forceinline__ void load(const CUtensorMap* ta, const CUtensorMap* tb, int kb, int m0, int n0, int z, uint8_t* sa, uint8_t* sb, uint64_t* bar, int lane) const {
    const int p0 = kb * BK;
    const int P = Ho * Wo;
    const int n = p0 / P, rem = p0 - n * P;
    const int oh = rem / Wo, ow = rem - oh * Wo;
    if constexpr (W) { if (lane < BM / 32) tma_load_2d(sa + lane * (BK * 128), ta, m0 + lane * 32, p0, bar); }
    else {
#pragma unroll
      for (int c = 0; c < BM / 32; ++c) tma_load_2d(sa + c * (BK * 128), ta, m0 + c * 32, p0, bar);
    }
#pragma unroll
    for (int c0 = 0; c0 < (W ? 1 : BN / 32); ++c0) {
      const int c = W ? lane - BM / 32 : c0;
      if (W && (c < 0 || c >= BN / 32)) break;
      const int r = (n0 >> 5) + c;                         // filter row of this 32-column chunk; rows >= 7 do not exist -> out-of-range row coordinate, zero fill
      tma_load_4d(sb + c * (BK * 128), tb, 0, ow, r < 7 ? 2 * oh + r : (1 << 20), n, bar);
    }
  }
};

// Epilogue arithmetic of one 32-column chunk held in registers (row m, columns nb .. nb+31): the same sequence as Epilogue::store4.
//   pre  : the residual row chunk already in registers (prefetched by the caller) or nullptr = load it here
//   cmul / cadd : this chunk's 32 multiplicative / additive column values in shared memory (see colvec_bytes) or nullptr = global loads
__device__ __forceinline__ void epilogue_math(float (&v)[32], const Epilogue& ep, int m, int nb, unsigned long long dseed,
                                              const float4* pre = nullptr, const float* cmul = nullptr, const float* cadd = nullptr) {
  if (ep.scale != 1.f) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] *= ep.scale;
  }
  const bool affine = ep.col_scale != nullptr;
  if (cadd) {                       // cached column vectors: columns beyond N hold 1 / 0
    if (affine && !ep.affine_post) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 a = *reinterpret_cast<const float4*>(cmul + 4 * j), b = *reinterpret_cast<const float4*>(cadd + 4 * j);
        v[4 * j] = fmaf(v[4 * j], a.x, b.x); v[4 * j + 1] = fmaf(v[4 * j + 1], a.y, b.y);
        v[4 * j + 2] = fmaf(v[4 * j + 2], a.z, b.z); v[4 * j + 3] = fmaf(v[4 * j + 3], a.w, b.w);
      }
    } else if (ep.bias) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 b = *reinterpret_cast<const float4*>(cadd + 4 * j);
        v[4 * j] += b.x; v[4 * j + 1] += b.y; v[4 * j + 2] += b.z; v[4 * j + 3] += b.w;
      }
    }
  } else {
    if (affine && !ep.affine_post) {
#pragma unroll
      for (int j = 0; j < 32; ++j) if (nb + j < ep.N) v[j] = fmaf(v[j], __ldg(ep.col_scale + nb + j), __ldg(ep.col_shift + nb + j));
    }
    if (ep.bias) {
#pragma unroll
      for (int j = 0; j < 32; ++j) if (nb + j < ep.N) v[j] += __ldg(ep.bias + nb + j);
    }
  }
  if (ep.relu) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
  }
  if (affine && ep.affine_post) {
    if (cadd) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 a = *reinterpret_cast<const float4*>(cmul + 4 * j), b = *reinterpret_cast<const float4*>(cadd + 4 * j);
        v[4 * j] = fmaf(v[4 * j], a.x, b.x); v[4 * j + 1] = fmaf(v[4 * j + 1], a.y, b.y);
        v[4 * j + 2] = fmaf(v[4 * j + 2], a.z, b.z); v[4 * j + 3] = fmaf(v[4 * j + 3], a.w, b.w);
      }
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j) if (nb + j < ep.N) v[j] = fmaf(v[j], __ldg(ep.col_scale + nb + j), __ldg(ep.col_shift + nb + j));
    }
  }
  if (ep.thresh) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] *= dropout_scale(dseed, (uint64_t)m * ep.N + nb + j, ep.thresh, ep.inv_keep);
  }
  if (pre) {
#pragma unroll
    for (int j = 0; j < 8; ++j) { v[4 * j] += pre[j].x; v[4 * j + 1] += pre[j].y; v[4 * j + 2] += pre[j].z; v[4 * j + 3] += pre[j].w; }
  } else if (ep.res && m < ep.M) {        // residual row: 128 contiguous bytes per thread (host checked 16-byte alignment and N % 4 == 0)
    const float4* r4 = reinterpret_cast<const float4*>(ep.res + (size_t)m * ep.ldres + nb);
#pragma unroll
    for (int j = 0; j < 8; ++j) if (nb + 4 * j < ep.N) {
      const float4 q = __ldg(r4 + j);
      v[4 * j] += q.x; v[4 * j + 1] += q.y; v[4 * j + 2] += q.z; v[4 * j + 3] += q.w;
    }
  }
  if (ep.relu_post) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
  }
}
// residual row chunk (row m, columns nb .. nb+31) into registers; zeros outside the matrix
__device__ __forceinline__ void load_res_chunk(float4 (&r)[8], const Epilogue& ep, int m, int nb) {
  if (m < ep.M) {
    const float4* p = reinterpret_cast<const float4*>(ep.res + (size_t)m * ep.ldres + nb);
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = (nb + 4 * j < ep.N) ? __ldg(p + j) : make_float4(0.f, 0.f, 0.f, 0.f);
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}


// ---------------------------------------------------------------- operand preparation (transpose / round / split in shared memory)
__device__ __forceinline__ void prep_bar_sync() { asm volatile("bar.sync 3, 128;" ::: "memory"); }
__device__ __forceinline__ void cons_bar_sync() { asm volatile("bar.sync 4, 256;" ::: "memory"); }
template <int NSPLIT> __device__ __forceinline__ void split_tf32(float4 v, float4& h, float4& l) {
  if constexpr (NSPLIT == 1) { h = v; return; }
  // hi = round-to-nearest TF32 (10-bit mantissa): unbiased, so the dropped lo*lo term and the tensor core's truncation of lo do not
  // accumulate coherently over K
  h.x = __uint_as_float((__float_as_uint(v.x) + 0x1000u) & 0xFFFFE000u);
  h.y = __uint_as_float((__float_as_uint(v.y) + 0x1000u) & 0xFFFFE000u);
  h.z = __uint_as_float((__float_as_uint(v.z) + 0x1000u) & 0xFFFFE000u);
  h.w = __uint_as_float((__float_as_uint(v.w) + 0x1000u) & 0xFFFFE000u);
  l = make_float4(v.x - h.x, v.y - h.y, v.z - h.z, v.w - h.w);
}
// One operand tile of R rows (m or n) by BK k.  MN-major: the TMA delivered R / 32 chunks of [32 k rows x 128 B]; they are rewritten in place
// as the K-major [R rows x 128 B] tile wgmma reads (both SWIZZLE_128B: 16-byte unit j of row r sits at unit j ^ (r & 7)).  Every one of the
// 128 preparation threads gathers its units into registers before any thread writes.  lo != nullptr: NSPLIT == 3 low parts.
template <int R, bool MN, int NSPLIT>
__device__ __forceinline__ void prep_operand(uint8_t* hi, uint8_t* lo, int p) {
  if constexpr (MN) {
    constexpr int U = R * 8 / 128;
    float4 g[U];
#pragma unroll
    for (int i = 0; i < U; ++i) {
      const int u = p + i * 128, m = u % R, kq = u / R;
      const uint8_t* src = hi + (m >> 5) * (BK * 128);
      const int mm = m & 31;
      float x[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int k = kq * 4 + e;
        x[e] = *reinterpret_cast<const float*>(src + k * 128 + ((((mm >> 2) ^ (k & 7)) << 4) | ((mm & 3) << 2)));
      }
      g[i] = make_float4(x[0], x[1], x[2], x[3]);
    }
    prep_bar_sync();
#pragma unroll
    for (int i = 0; i < U; ++i) {
      const int u = p + i * 128, m = u % R, kq = u / R;
      const int off = m * 128 + ((kq ^ (m & 7)) << 4);
      float4 h, l;
      split_tf32<NSPLIT>(g[i], h, l);
      *reinterpret_cast<float4*>(hi + off) = h;
      if constexpr (NSPLIT == 3) *reinterpret_cast<float4*>(lo + off) = l;
    }
  } else if constexpr (NSPLIT >= 2) {
#pragma unroll 4
    for (int i = p; i < R * 8; i += 128) {
      float4 h, l;
      split_tf32<NSPLIT>(reinterpret_cast<float4*>(hi)[i], h, l);
      reinterpret_cast<float4*>(hi)[i] = h;
      if constexpr (NSPLIT == 3) reinterpret_cast<float4*>(lo)[i] = l;
    }
  }
}

// ---------------------------------------------------------------- register-A operand (A_RS kernels)
// An MN-major A tile is not transposed in shared memory: each consumer thread loads its wgmma A fragment straight from the BM / 32 TMA chunks
// of [32 k rows x 128 B] with ld.shared.  Warp q of consumer warpgroup wg owns tile rows m = 64 wg + 16 q + g + {0, 8} (g = lane / 4), and
// per k8 step ks the k = 8 ks + t + {0, 4} (t = lane % 4).
// Banks: element (k, m) is word 32 k + 4 ((m' >> 2) ^ (k & 7)) + (m' & 3) of chunk m / 32, m' = m % 32 = 16 (q & 1) + g (+ 8).  If every lane
// loaded the same one of its two k, the warp would cover m' >> 2 in {4h, 4h + 1} (+ 2) and k & 7 = t in 0..3: 4 distinct 16-byte units,
// 16 banks, 2-way conflicts.  So lanes 16..31 (g >= 4) load their k + 4 element first and lanes 0..15 their k element: the two halves of the
// warp then hit the two disjoint unit groups (k & 7 < 4 and k & 7 >= 4), every 32-bit load is conflict-free (one wavefront per warp and
// load), and two selects per row put the values back into fragment order.
struct RsFrag {
  uint32_t off[4];   // byte offsets in the stage for k step 0: (row g, first k), (row g, second k), (row g + 8, first k), (row g + 8, second k)
  bool swap;         // lanes 16..31: the first load is k + 4
  __device__ __forceinline__ void init(int wg, int q, int lane) {
    const int g = lane >> 2, t = lane & 3, hsel = lane >> 4;
    const uint32_t chunk = (uint32_t)(2 * wg + (q >> 1)) * (BK * 128);
    swap = hsel != 0;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int mm = 16 * (q & 1) + g + 8 * r;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int k = t + 4 * (i ^ hsel);
        off[2 * r + i] = chunk + k * 128 + ((((mm >> 2) ^ (k & 7)) << 4) | ((mm & 3) << 2));
      }
    }
  }
  // fragment of k step ks (8 k rows = 1024 B further; k & 7 and so the swizzle are unchanged) from the A tile at `st`
  __device__ __forceinline__ void load(uint32_t (&a)[4], const uint8_t* st, int ks) const {
    uint32_t x[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) x[i] = *reinterpret_cast<const uint32_t*>(st + off[i] + ks * 1024);
    a[0] = swap ? x[1] : x[0]; a[2] = swap ? x[0] : x[1];
    a[1] = swap ? x[3] : x[2]; a[3] = swap ? x[2] : x[3];
  }
};
// register form of split_tf32: the same rounding (NSPLIT >= 2) and hi / lo split (NSPLIT == 3) of one A fragment
template <int NSPLIT> __device__ __forceinline__ void split_frag(const uint32_t (&a)[4], uint32_t (&h)[4], uint32_t (&l)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    h[i] = NSPLIT == 1 ? a[i] : ((a[i] + 0x1000u) & 0xFFFFE000u);
    if constexpr (NSPLIT == 3) l[i] = __float_as_uint(__uint_as_float(a[i]) - __uint_as_float(h[i]));
  }
}

// ---------------------------------------------------------------- the kernel
// Persistent: the grid is at most one CTA per SM and loops over output tiles (static round-robin).  The shared-memory stage ring runs
// continuously across tiles, so the TMA loads of tile i+1 overlap the epilogue of tile i.
//   warpgroup 0: warp 0 = TMA producer (warps 1-3 idle)
//   warpgroup 1 (only when an operand needs a transpose, rounding or a split in shared memory): operand preparation (prep_operand)
//   last two warpgroups: consumers -- wgmma over rows [64 wg, 64 wg + 64) of the tile, then the epilogue of the chunks c with c % 2 == wg
// A_RS (MN-major A only): the consumers read A from the TMA chunks into registers (RsFrag) and round / split it there; the preparation
// warpgroup handles B alone and is dropped when B needs nothing.
// tma_epi != 0: the epilogue writes 32-column chunks with TMA stores (cp.reduce.async.bulk ... .add for accumulate / split-K), fully coalesced
// and clipped at the tensor edge by the hardware.
// OUT_T (transposed output; A_RS, K-major B, BN == 128): the kernel computes D^T of the output it stores.  The input gradients run this way,
// dX^T[channels, pixels] = W^T dY^T, so that the weights are the MN-major A operand the consumers read into registers and dY a K-major B
// operand -- no operand is transposed in shared memory.  The accumulator is staged transposed (BM / 32 chunks of [BN rows x 128 B], one per
// 32 output columns) and stored with tmap_c / ep over the [pixels x channels] output; only ep.scale and store / accumulate (mode 0 / 1) apply.
// Tile order: the m tiles (channels) of one n tile (pixels) run on neighbouring CTAs, so a dY tile is fetched from HBM once and then hit in L2.
// Every tile runs its k-blocks in ascending order, so both forms accumulate each output element in the same k order.
template <bool A_MN, bool B_MN, int NSPLIT, bool A_RS = false> __host__ __device__ constexpr bool has_prep() { return (A_MN && !A_RS) || B_MN || NSPLIT >= 2; }
template <bool A_MN, bool B_MN, int NSPLIT, bool A_RS = false> __host__ __device__ constexpr int persistent_threads() { return (has_prep<A_MN, B_MN, NSPLIT, A_RS>() ? 4 : 3) * 128; }

template <int BN, bool A_MN, bool B_MN, class Producer, int NSPLIT, bool A_RS = false, bool OUT_T = false>
__global__ void __launch_bounds__(persistent_threads<A_MN, B_MN, NSPLIT, A_RS>(), 1)
gemm_tc_persistent_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, const __grid_constant__ CUtensorMap tmap_c,
                          Epilogue ep, Producer prod, int num_kb_total, int kb_per_split, int tiles_m, int tiles_n, int splits, int tma_epi) {
  constexpr int STAGES = num_stages<BN, NSPLIT>();
  constexpr int A_BYTES = BM * 128, B_BYTES = BN * 128, AB_BYTES = A_BYTES + B_BYTES;
  constexpr int STAGE_BYTES = stage_bytes<BN, NSPLIT>();
  static_assert(!A_RS || A_MN, "the register-A main loop reads MN-major A tiles");
  static_assert(!OUT_T || (A_RS && !B_MN && BN == BM), "transposed output: register-A main loop, K-major B, square 128 x 128 tiles");
  constexpr bool PREP = has_prep<A_MN, B_MN, NSPLIT, A_RS>();
  constexpr int CONS_WARP0 = PREP ? 8 : 4;
  constexpr int EPI_WG = 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* accbuf = smem + STAGES * STAGE_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(accbuf + acc_bytes<BN>());
  uint64_t* full = bars;                 // [STAGES] TMA bytes landed
  uint64_t* empty = bars + STAGES;       // [STAGES] consumers finished reading the stage
  uint64_t* ready = bars + 2 * STAGES;   // [STAGES] operands prepared (PREP only)
  float* const colvec = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars) + 256);      // [2][BN]

  pdl_launch_dependents();     // the stream successor may start its own prologue now; it blocks in its pdl_wait() until this grid is done
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int total_tiles = tiles_m * tiles_n * splits;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if (tma_epi) tma_prefetch_desc(&tmap_c);
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); mbar_init(&ready[s], 128); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();                  // prologue done (barriers, descriptors): from here on the kernel reads what its stream predecessor wrote

  // third tile coordinate z: split-K slice (kb_beg = z * kb_per_split)
  auto tile_coords = [&](int t, int& m0, int& n0, int& kb_beg, int& nkb, int& z) {
    int mi, ni;
    if constexpr (OUT_T) {                            // the output's columns (m tiles) fastest, as for the untransposed product
      mi = t % tiles_m;
      const int r = t / tiles_m;
      ni = r % tiles_n;
      z = r / tiles_n;
    } else {
      ni = t % tiles_n;
      const int r = t / tiles_n;
      mi = r % tiles_m;
      z = r / tiles_m;
    }
    m0 = mi * BM; n0 = ni * BN;
    kb_beg = z * kb_per_split;
    nkb = min(num_kb_total - kb_beg, kb_per_split);
  };

  if (warp == 0) {
    // Producers with many small boxes per k-block (MN-major operands: the weight-gradient GEMMs) produce with the whole warp: lane 0 waits for
    // the stage and arms its barrier, then every lane issues its box (Producer::load<true>).  ep.opt bit 2 = 0 keeps the single-thread issue.
    const bool wide_issue = Producer::WIDE_OK && (ep.opt & 4) != 0;
    if (lane == 0 || wide_issue) {
      uint32_t it = 0;
      Producer pr = prod;
      pr.set_policy(l2_policy_evict_first());
      for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        int m0, n0, kb_beg, nkb, z;
        tile_coords(t, m0, n0, kb_beg, nkb, z);
        for (int kb = 0; kb < nkb; ++kb, ++it) {
          const int s = it % STAGES;
          const uint32_t ph = (it / STAGES) & 1;
          if (lane == 0) {
            mbar_wait(&empty[s], ph ^ 1);
            mbar_expect_tx(&full[s], AB_BYTES);
          }
          if (wide_issue) __syncwarp();
          uint8_t* sa = smem + s * STAGE_BYTES;
          if constexpr (Producer::WIDE_OK) {
            if (wide_issue) pr.template load<true>(&tmap_a, &tmap_b, kb_beg + kb, m0, n0, z, sa, sa + A_BYTES, &full[s], lane);
            else pr.template load<false>(&tmap_a, &tmap_b, kb_beg + kb, m0, n0, z, sa, sa + A_BYTES, &full[s], 0);
          } else {
            pr.template load<false>(&tmap_a, &tmap_b, kb_beg + kb, m0, n0, z, sa, sa + A_BYTES, &full[s], 0);
          }
        }
      }
    }
  } else if (warp < 4) {
    // idle warps of the producer warpgroup
  } else if (PREP && warp < CONS_WARP0) {
    const int p = threadIdx.x - 128;
    uint32_t it = 0;
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
      int m0, n0, kb_beg, nkb, z;
      tile_coords(t, m0, n0, kb_beg, nkb, z);
      for (int kb = 0; kb < nkb; ++kb, ++it) {
        const int s = it % STAGES;
        const uint32_t ph = (it / STAGES) & 1;
        mbar_wait(&full[s], ph);
        uint8_t* st = smem + s * STAGE_BYTES;
        if constexpr (!A_RS) prep_operand<BM, A_MN, NSPLIT>(st, st + AB_BYTES, p);
        prep_operand<BN, B_MN, NSPLIT>(st + A_BYTES, st + AB_BYTES + A_BYTES, p);
        fence_proxy_async();     // generic-proxy smem writes -> visible to the tensor core (async proxy)
        mbar_arrive(&ready[s]);
      }
    }
  } else {
    const int wg = (warp - CONS_WARP0) >> 2;        // consumer warpgroup: MMA rows [64 wg, 64 wg + 64); epilogue chunks c with c % 2 == wg
    const int q = warp & 3;                         // warp inside the warpgroup
    const int rr = q * 32 + lane;                   // epilogue row of this thread inside the tile
    const bool elected = (threadIdx.x == (CONS_WARP0 + 4 * wg) * 32);
    const unsigned long long dseed = ep.thresh ? (*ep.seed_ptr + ep.site * 0xD1B54A32D192ED03ull) : 0ull;
    constexpr int NCHUNK = (OUT_T ? BM : BN) / 32;     // 32-column chunks of the stored tile
    constexpr int CHUNK_ROWS = OUT_T ? BN : BM;       // rows of the stored tile
    // fused BatchNorm statistics: per-thread fp64 accumulators (lane = column of a chunk, warp = row quarter), carried ACROSS the tiles of this
    // persistent CTA and flushed with one atomic pair per column when the CTA moves to another column block / at the end: flushing per tile
    // put ~10^6 fp64 atomics per convolution onto 2 N addresses, serialised in the L2.
    constexpr int NCH_WG = (NCHUNK + EPI_WG - 1) / EPI_WG;
    double racc1[NCH_WG], racc2[NCH_WG];
#pragma unroll
    for (int k = 0; k < NCH_WG; ++k) { racc1[k] = 0.0; racc2[k] = 0.0; }
    int acc_n0 = -1;
    auto flush_stats = [&]() {
      if (acc_n0 >= 0) {
#pragma unroll
        for (int k = 0; k < NCH_WG; ++k) {
          const int col = acc_n0 + (k * EPI_WG + wg) * 32 + lane;
          if (col < ep.N && (k * EPI_WG + wg) < NCHUNK) { atomicAdd(ep.stats + col, racc1[k]); atomicAdd(ep.stats + ep.N + col, racc2[k]); }
          racc1[k] = 0.0; racc2[k] = 0.0;
        }
      }
    };
    const bool do_stats = !OUT_T && ep.stats != nullptr;
    const bool use_res = !OUT_T && tma_epi && ep.res != nullptr && !ep.nv_pad && (ep.opt & 1);
    const bool use_cv = !OUT_T && tma_epi && !ep.nv_pad && (ep.bias != nullptr || ep.col_scale != nullptr) && (ep.opt & 2);
    float4 rcur[8], rnext[8];
    int cv_n0 = -1;
    uint32_t it = 0;
    float acc[BN / 2];
    RsFrag frag;
    if constexpr (A_RS) frag.init(wg, q, lane);
    // the producer's tile walk, written with a tile counter: with `t += gridDim.x` ptxas spills more of the epilogue's registers
    for (int i = 0; ; ++i) {
      const int t = blockIdx.x + i * gridDim.x;
      if (t >= total_tiles) break;
      int m0, n0, kb_beg, nkb, z;
      tile_coords(t, m0, n0, kb_beg, nkb, z);
      const int m = m0 + rr;
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      int prev_s = -1;
      if constexpr (A_RS) {
        // ---- register-A main loop: one wgmma group per k8 step; the fragments alternate between two register sets (ahi / alo [ks & 1]).
        // Before a set is reloaded, wgmma_wait<1> retires the group that read it two steps earlier, so one group stays in flight while the
        // next fragment loads.  The stage of k-block kb - 1 is released at step 1 of k-block kb: by then its last group has completed, and
        // so have all of its fragment loads, which every lane finished before the warpgroup issued the group.
        constexpr int KS = BK / WG_K;
        uint32_t ahi[2][4], alo[2][4];
        for (int kb = 0; kb < nkb; ++kb, ++it) {
          const int s = it % STAGES;
          const uint32_t ph = (it / STAGES) & 1;
          if constexpr (PREP) mbar_wait(&ready[s], ph);     // B prepared
          mbar_wait(&full[s], ph);                          // A landed (already observed through ready[s] when PREP)
          const uint8_t* st = smem + s * STAGE_BYTES;
          const uint32_t sb = smem_u32(st) + A_BYTES;
#pragma unroll
          for (int ks = 0; ks < KS; ++ks) {
            wgmma_wait<1>();
            if (ks == 1 && prev_s >= 0 && lane == 0) mbar_arrive(&empty[prev_s]);
            uint32_t a[4];
            frag.load(a, st, ks);
            split_frag<NSPLIT>(a, ahi[ks & 1], alo[ks & 1]);
            wgmma_fence();
            const uint64_t bd = make_wgmma_desc(sb + ks * 32);
            wgmma_tf32_rs<BN>(acc, ahi[ks & 1], bd);
            if constexpr (NSPLIT == 3 && !OUT_T) {
              wgmma_tf32_rs<BN>(acc, alo[ks & 1], bd);                              // lo(A) * hi(B)
              wgmma_tf32_rs<BN>(acc, ahi[ks & 1], bd + (uint64_t)(AB_BYTES >> 4));  // hi(A) * lo(B)
            } else if constexpr (NSPLIT == 3) {
              // the untransposed product's order: lo of the output's row operand (here B) times hi of its column operand first
              wgmma_tf32_rs<BN>(acc, ahi[ks & 1], bd + (uint64_t)(AB_BYTES >> 4));  // hi(A) * lo(B)
              wgmma_tf32_rs<BN>(acc, alo[ks & 1], bd);                              // lo(A) * hi(B)
            }
            wgmma_commit();
          }
          prev_s = s;
        }
      } else {
        // ---- main loop: one wgmma group per k-block; the stage of k-block kb - 1 is released once its group has completed
        for (int kb = 0; kb < nkb; ++kb, ++it) {
          const int s = it % STAGES;
          const uint32_t ph = (it / STAGES) & 1;
          mbar_wait(PREP ? &ready[s] : &full[s], ph);
          const uint32_t sa = smem_u32(smem + s * STAGE_BYTES) + wg * (64 * 128);
          const uint32_t sb = smem_u32(smem + s * STAGE_BYTES) + A_BYTES;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / WG_K; ++k) {
            const uint64_t ad = make_wgmma_desc(sa + k * 32), bd = make_wgmma_desc(sb + k * 32);
            wgmma_tf32<BN>(acc, ad, bd);
            if constexpr (NSPLIT == 3) {
              const uint64_t lo_off = (uint64_t)(AB_BYTES >> 4);      // descriptors address in 16-byte units: the lo copies sit AB_BYTES after the hi tiles
              wgmma_tf32<BN>(acc, ad + lo_off, bd);   // lo(A) * hi(B)
              wgmma_tf32<BN>(acc, ad, bd + lo_off);   // hi(A) * lo(B)
            }
          }
          wgmma_commit();
          wgmma_wait<1>();
          if (prev_s >= 0 && lane == 0) mbar_arrive(&empty[prev_s]);
          prev_s = s;
        }
      }
      wgmma_wait<0>();
      if (prev_s >= 0 && lane == 0) mbar_arrive(&empty[prev_s]);

      // ---- accumulator -> staging chunks.  The TMA stores of the previous tile must have finished reading them.
      if (use_res) load_res_chunk(rcur, ep, m, n0 + wg * 32);
      if (elected && tma_epi) tma_store_wait_read<0>();
      cons_bar_sync();
      if constexpr (OUT_T) {
        // Transposed: element (m, n) of the tile goes to chunk m / 32, row n, column m % 32.  Thread (g, t) = (lane / 4, lane % 4) stores
        // 32-bit words: for register 4 j + 2 h + i, m = r0 + 8 h and n = 8 j + 2 t + i, at unit ((m % 32) >> 2) ^ (n & 7) = ((m' >> 2) ^ (2 t + i))
        // of row n, word m & 3.  Per store instruction (j, h, i fixed) the warp's m' >> 2 = u0 + (g >> 2) with u0 even, so the unit is
        // (u0 ^ 2 t) | ((g >> 2) ^ i): 4 values of t x 2 of g >> 2 = 8 distinct units, times 4 words (g & 3) = all 32 banks -- conflict-free
        // (the row adds a multiple of 128 B and does not move the bank).
        const int r0 = wg * 64 + q * 16 + (lane >> 2);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int mm = r0 + 8 * h;
          uint8_t* chunk = accbuf + (mm >> 5) * (BN * 128);
          const int un = (mm & 31) >> 2, wo = (mm & 3) << 2;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              const int nn = 8 * j + 2 * (lane & 3) + i;
              *reinterpret_cast<float*>(chunk + nn * 128 + ((un ^ (nn & 7)) << 4) + wo) = acc[4 * j + 2 * h + i];
            }
        }
      } else {
        // wgmma D fragment: register 4 j + {0, 1} = row (warp q) * 16 + lane / 4, columns 8 j + 2 (lane % 4) + {0, 1}; + {2, 3} = 8 rows below
        const int r0 = wg * 64 + q * 16 + (lane >> 2);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int col = 8 * j + 2 * (lane & 3);
          uint8_t* chunk = accbuf + (col >> 5) * (BM * 128);
          const int un = (col & 31) >> 2, wo = (col & 3) << 2;
          *reinterpret_cast<float2*>(chunk + r0 * 128 + ((un ^ (r0 & 7)) << 4) + wo) = make_float2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<float2*>(chunk + (r0 + 8) * 128 + ((un ^ ((r0 + 8) & 7)) << 4) + wo) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
      }
      if (use_cv && n0 != cv_n0) {       // this warpgroup's chunks of the tile's column vectors -> shared memory (every consumer is past the last read)
        const int tw = threadIdx.x - (CONS_WARP0 + 4 * wg) * 32;      // 0..127 inside the warpgroup
        for (int i = tw; i < NCH_WG * 32; i += 128) {
          const int col = n0 + ((i >> 5) * EPI_WG + wg) * 32 + (i & 31);
          const bool in = col < ep.N;
          float mul = 1.f, add = 0.f;
          if (ep.col_scale) { if (in) { mul = __ldg(ep.col_scale + col); add = __ldg(ep.col_shift + col); } }
          else if (in) add = __ldg(ep.bias + col);
          colvec[wg * NCH_WG * 32 + i] = mul;
          colvec[BN + wg * NCH_WG * 32 + i] = add;
        }
        cv_n0 = n0;
      }
      cons_bar_sync();
      if (do_stats && n0 != acc_n0) { flush_stats(); acc_n0 = n0; }

      // ---- epilogue of this warpgroup's chunks: thread = row rr, 32 columns
#pragma unroll 1
      for (int c = wg; c < NCHUNK; c += EPI_WG) {
        if (use_res) {
          if (c != wg) {
#pragma unroll
            for (int j = 0; j < 8; ++j) rcur[j] = rnext[j];
          }
          if (c + EPI_WG < NCHUNK) load_res_chunk(rnext, ep, m, n0 + (c + EPI_WG) * 32);
        }
        uint8_t* buf = accbuf + c * (CHUNK_ROWS * 128);
        float v[32];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float4 x = *reinterpret_cast<const float4*>(buf + rr * 128 + ((j ^ (rr & 7)) << 4));
          v[4 * j] = x.x; v[4 * j + 1] = x.y; v[4 * j + 2] = x.z; v[4 * j + 3] = x.w;
        }
        const int nb = (OUT_T ? m0 : n0) + c * 32;       // first output column of the chunk
        const int row0 = OUT_T ? n0 : m0;                // first output row of the tile
        if (OUT_T && nb >= ep.N) continue;               // rows of A beyond the output's columns (e.g. the next tap's weights): never stored
        int sc0 = nb, sc1 = 0;
        if (ep.nv_pad) {               // virtual wgrad column -> (channel, tap); chunks wholly beyond Cin are skipped (warp-uniform)
          sc1 = nb / ep.nv_pad; sc0 = nb - sc1 * ep.nv_pad;
          if (sc0 >= ep.nv_real || sc1 * ep.nv_real >= ep.N) continue;      // beyond the tap's channels / beyond the last tap (wide tiles over a padded grid)
        }
        if (tma_epi) {
          const float* cmul = use_cv ? colvec + (wg * NCH_WG + (c - wg) / EPI_WG) * 32 : nullptr;
          epilogue_math(v, ep, m, nb, dseed, use_res ? rcur : nullptr, cmul, use_cv ? cmul + BN : nullptr);
#pragma unroll
          for (int j = 0; j < 8; ++j)      // back into the same (swizzled) place: the chunk is the TMA store's source
            *reinterpret_cast<float4*>(buf + rr * 128 + ((j ^ (rr & 7)) << 4)) = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
          fence_proxy_async();
          epi_bar_sync(wg);
          if (elected) {
            if (ep.s2_w2) {           // stride-2 dgrad parity class: rows (n, i, j) -> input pixels (2 i + ph, 2 j + pw), element-strided 4-D map
              const int P2 = ep.s2_h2 * ep.s2_w2;
              const int n_ = row0 / P2, i0 = (row0 - n_ * P2) / ep.s2_w2;
              if (ep.mode == 0) tma_store_4d(&tmap_c, buf, nb, ep.s2_pw, 2 * i0 + ep.s2_ph, n_);
              else tma_reduce_add_4d(&tmap_c, buf, nb, ep.s2_pw, 2 * i0 + ep.s2_ph, n_);
            } else if (ep.nv_pad) {
              if (ep.mode == 0) tma_store_3d(&tmap_c, buf, sc0, sc1, m0);
              else tma_reduce_add_3d(&tmap_c, buf, sc0, sc1, m0);
            } else if (ep.mode == 0) tma_store_2d(&tmap_c, buf, nb, row0);
            else tma_reduce_add_2d(&tmap_c, buf, nb, row0);
            tma_store_commit();
          }
          if (do_stats) {
            // fused BatchNorm statistics: column sums / sums of squares of the chunk over this warp's 32 rows.  Each lane holds one ROW
            // (32 columns) in registers: a halving butterfly over the lanes (16 + 8 + 4 + 2 + 1 = 31 exchanges per quantity) leaves lane l with
            // the totals of column l.  Then one fp64 atomic pair per column per warp when the column block changes.
            const int rows_valid = min(32, ep.M - (m0 + q * 32));
            float s1[32], s2[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) { const float x = (lane < rows_valid) ? v[j] : 0.f; s1[j] = x; s2[j] = x * x; }
#pragma unroll
            for (int w = 16; w >= 1; w >>= 1) {
              const bool up = (lane & w) != 0;
#pragma unroll
              for (int j = 0; j < w; ++j) {
                // keep the half of the columns whose bit `w` equals this lane's bit `w`, hand the other half to the partner lane
                const float keep1 = up ? s1[j + w] : s1[j], give1 = up ? s1[j] : s1[j + w];
                const float keep2 = up ? s2[j + w] : s2[j], give2 = up ? s2[j] : s2[j + w];
                s1[j] = keep1 + __shfl_xor_sync(0xffffffffu, give1, w);
                s2[j] = keep2 + __shfl_xor_sync(0xffffffffu, give2, w);
              }
            }
            // after the butterfly lane l holds column l of the chunk (bit w of the column index = bit w of the lane)
            const int ci = (c - wg) / EPI_WG;
#pragma unroll
            for (int k = 0; k < NCH_WG; ++k) if (k == ci) { racc1[k] += (double)s1[0]; racc2[k] += (double)s2[0]; }
          }
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j)
            ep.store4(m, nb + j * 4, make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]));
        }
      }
    }
    if (do_stats) flush_stats();
    if (elected && tma_epi) tma_store_wait<0>();
  }
}
// ---------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode_fn();

// 2-D fp32 tensor map over a row-major [rows, cols] matrix with row stride ld (elements); box = {32 cols, box_rows}.
int make_tmap_2d(CUtensorMap* map, const float* base, long long rows, long long cols, long long ld, int box_rows, bool atom32 = false);
// MN-major operand [rows (k), cols] with cols % 32 == 0 as a rank-3 map {32, rows, cols / 32}: box {32, 32, groups} = `groups` chunks in one operation
int make_tmap_2d_grouped(CUtensorMap* map, const float* base, long long rows, long long cols, long long ld, int groups);
// 4-D fp32 tensor map over an NHWC tensor [N,H,W,C] with pixel stride ld; box = {32 channels, bw, bh, bn}.
// estride = 2: the box visits every second pixel in W and H (stride-2 convolutions read / write the full-resolution tensor in place);
// bw / bh stay the numbers of pixels FETCHED
int make_tmap_nhwc(CUtensorMap* map, const float* base, int N, int H, int W, int C, long long ld, int bw, int bh, int bn, bool atom32, int estride = 1);
// NHWC tensor with C % 32 == 0 as a rank-5 map {32, W, H, N, C / 32}: box {32, bw, bh, 1, groups} = `groups` consecutive 32-channel chunks of one pixel window
int make_tmap_nhwc_grouped(CUtensorMap* map, const float* base, int N, int H, int W, int C, long long ld, int bw, int bh, int estride, int groups);
// overlapping-stride view of the zero-bordered NHWC4 stem input (see StemFwdProducer); box = {32, box_ow, 1, 1}
int make_tmap_stem(CUtensorMap* map, const float* base, int N, int Hp, int Wp, int Wo, int box_ow, bool atom32);

}  // namespace tc
}  // namespace rih
