// Batched per-head GEMM of the attention core on the wgmma path (implemented in gemm_tc.cu, used by attention.cu).
#pragma once
#include <cuda_runtime.h>

namespace rih {
namespace tc {

// token matrix: element (b, h, s, k) at p + (b * rows + s) * ld + h * cols + k   (rows = tokens per batch image, cols = head dim)
// score matrix: element (z, r, c)    at p + (z * rows + r) * ld + c              (z = b * H + h, ld = padded row stride)
struct BOperand { const float* p; int tok; int rows; int cols; long long ld; };

// C[z] = scale * op(A[z]) op(B[z])^T for all z = b * H + h in one persistent launch.  *_mn = 0: operand stored [M|N rows, K cols];
// 1: stored [K rows, M|N cols].  Supported (a_mn, b_mn): (0,0), (0,1), (1,1).  Arithmetic (TF32 / 3xTF32) = current set_nsplit().
int bgemm_tf32(const BOperand& a, int a_mn, const BOperand& b, int b_mn, const BOperand& c, int B, int H, int M, int N, int K, float scale,
               cudaStream_t s);
void set_nsplit(int n);
void set_acc_scale(float s);
int set_stream_cta_limit(cudaStream_t s, int ctas);   // cap the persistent grid of GEMMs launched on stream s (0 = no cap)

}  // namespace tc
}  // namespace rih
