// fp32 products of the training backward (motion_train.cu owns the kernels; nets_train.cu shares them).
#pragma once
#include "common.cuh"

namespace dyn {

// C[m, n] (+)= sum_k A(m, k) B(k, n) s(k);  A(m, k) = A[m * sam + k * sak],
// B(k, n) = B[(k / bdiv) * sbk + n * sbn] (bdiv > 1: one B row serves `bdiv` consecutive k -- a per-point
// tensor against per-(point, view) rows), s(k) = kscale ? kscale[k] : 1 (the row scale of a layer input).
// gridDim.z splits K (split_k: a number of splits that depends on the shape alone); each split writes its partial
// product to `red` and launch_red_add adds the partials in split order.  No float atomics anywhere in the training
// backward: the same inputs give the same bits.
struct GemmArgs {
  const float *A, *B;
  float* C;
  long long M, N, K;
  long long sam, sak, sbk, sbn;
  long long ldc;
  int accumulate;
  long long k_per_split;
  long long bdiv = 1;
  const float* kscale = nullptr;
  float* red = nullptr;  // partials of a split product (kRedFloats floats)
};

// Fixed-order reductions: a product that splits its reduction over rows writes one partial per slab into a
// reduction scratch of kRedFloats floats (part of the caller's scratch), then adds the partials in slab order, once,
// into its accumulator.  The slab partitions depend on the shapes alone (never on the SM count).
constexpr long long kRedFloats = 128LL * 128 * 128;  // 8 MiB
inline size_t red_scratch_bytes() { return (size_t)kRedFloats * sizeof(float); }
// C[m * ldc + n] (+)= sum_{s < slabs} part[s * sstride + m * N + n], s in increasing order
int launch_red_add(const float* part, int slabs, long long sstride, long long M, long long N, float* C, long long ldc,
                   bool accumulate, cudaStream_t st);

int launch_gemm(GemmArgs a, bool split_k, cudaStream_t st);
// db[c] += sum_r g[r * ldg + c], c < width (red: reduction scratch)
int launch_colsum(const float* g, long long ldg, int width, long long N, float* db, float* red, cudaStream_t st);

// tensor-core versions (train_tc.cu; bf16 operands, fp32 accumulation); *_ok tells whether a shape is supported
bool tc_grad_w_ok(int out, int width, long long rows);
bool tc_grad_in_ok(int out, int width, long long rows);
size_t tc_grad_in_scratch_bytes();
// dW[out, width] (ld ldw) += dz[rows, out]^T (x[rows, width] * kscale[rows])   (red: reduction scratch)
int tc_grad_w(const float* dz, long long lddz, int out, long long rows, const float* x, long long ldx, int width,
              const float* kscale, float* dW, long long ldw, float* red, cudaStream_t st);
// din[rows, width] (ld ldd) = dz[rows, out] W[out, 0:width] (W row-major, ldw columns; pass W + column offset)
int tc_grad_in(const float* dz, long long lddz, int out, long long rows, const float* W, long long ldw, int width,
               float* din, long long ldd, void* img_scratch, cudaStream_t st);

}  // namespace dyn
