// Tensor-core products of the training backward (bf16 operands, fp32 accumulation, fp32 master
// weights and gradients): the two GEMMs per linear layer that dominate a training step,
//
//   dW[out, width] += dZ^T X      (tc_grad_w)   reduction over the ROWS: both operands are read exactly as they lie
//                                               in HBM (row-major, the reduction index is the slow one) and staged as
//                                               MN-major wgmma operands -- no transposition anywhere
//   dIn[rows, width] = dZ W[:, c0:c0+width]  (tc_grad_in)  == a forward linear layer whose weight is a transposed
//                                               slice of W: packed on the fly, then linear_tc.cu's kernel
//
// tc_grad_w: a CTA owns a slab of rows and a 128 x 128 tile of dW; warps 0-7 stage 64 rows at a time (one 16 B chunk =
// 8 consecutive columns of one row per store; 8 consecutive rows form one 128-byte core matrix whose CONTIGUOUS
// dimension is M / N, i.e. the canonical MN-major no-swizzle layout: LBO = 128 B between 8-row groups along K,
// SBO = 64 * 16 B between 8-column groups along M / N); warpgroup g multiplies rows 64 g .. of the tile with wgmma (both
// operands MN-major) over a 2-stage ring; its accumulators live in registers for the whole slab and are stored as
// that slab's partial dW tile.  A second pass (launch_red_add) adds the slabs' partials into dW in slab order.  The
// slab count is a function of the shape alone: the same inputs give the same bits on every H100.
#include "linear_tc.cuh"
#include "tc.cuh"
#include "train_gemm.cuh"

namespace dyn {

using namespace tc;

namespace {

constexpr int kRowsStage = 64;   // K per stage
constexpr int kTileM = 128, kTileN = 128;
constexpr int kStageBytes = (kTileM + kTileN) * kRowsStage * 2;  // 32 KB
constexpr int kGwSmem = 2 * kStageBytes;

struct GradWArgs {
  const float* dz; long long lddz; int out;
  const float* x; long long ldx; int width;
  const float* kscale;
  long long rows, rows_per_cta;
  float* part;  // [slab, out, width] partials
  int mtiles, nblocks;
};

// 8 consecutive columns [c, c + 8) of row `row` (zero outside the matrix), scaled, as 8 bf16
__device__ __forceinline__ uint4 load8_bf16(const float* __restrict__ p, long long ld, long long row, long long rows,
                                            int c, int width, float scale, bool vec_ok) {
  float v[8];
  if (row < rows && vec_ok && c + 8 <= width) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(p + row * ld + c));
    const float4 b = __ldg(reinterpret_cast<const float4*>(p + row * ld + c + 4));
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = (row < rows && c + i < width) ? __ldg(p + row * ld + c + i) : 0.f;
  }
  uint4 q;
  q.x = pack_bf16x2(v[0] * scale, v[1] * scale);
  q.y = pack_bf16x2(v[2] * scale, v[3] * scale);
  q.z = pack_bf16x2(v[4] * scale, v[5] * scale);
  q.w = pack_bf16x2(v[6] * scale, v[7] * scale);
  return q;
}

__device__ __forceinline__ void mma_block_mn(float* d, int w, uint64_t ad, uint64_t bd, uint32_t sc) {
  switch (w) {
    case 16: Wgmma<16, 1, 1>::mma(d, ad, bd, sc); break;
    case 32: Wgmma<32, 1, 1>::mma(d, ad, bd, sc); break;
    case 48: Wgmma<48, 1, 1>::mma(d, ad, bd, sc); break;
    default: Wgmma<64, 1, 1>::mma(d, ad, bd, sc); break;
  }
}

// grid: x = slab, y = M tile * nblocks + N block
__global__ void __launch_bounds__(256, 1) grad_w_tc_kernel(const __grid_constant__ GradWArgs a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
  const int mt = blockIdx.y / a.nblocks, nbk = blockIdx.y % a.nblocks;
  const int m0 = mt * kTileM, n0 = nbk * kTileN;
  const int nw = min(kTileN, ((a.width - n0) + 15) / 16 * 16);  // columns of this N block (multiple of 16)
  const long long r_lo = (long long)blockIdx.x * a.rows_per_cta;
  const long long r_hi = r_lo + a.rows_per_cta < a.rows ? r_lo + a.rows_per_cta : a.rows;
  const int nstages = (int)((r_hi - r_lo + kRowsStage - 1) / kRowsStage);

  // loaders: four lanes read 4 x 32 B = one 128-byte line of a row (8 lines per warp instruction instead of 32);
  // a warp owns 8 rows of the stage.  Groups g < 16 are 8 columns of dZ (M), g >= 16 of X (N).
  const int srow = warp * 8 + (lane >> 2), gsel = lane & 3;
  const bool dz_vec = (a.lddz & 3) == 0 && (reinterpret_cast<uintptr_t>(a.dz) & 15) == 0;
  const bool x_vec = (a.ldx & 3) == 0 && (reinterpret_cast<uintptr_t>(a.x) & 15) == 0;
  const int ngroups = 16 + nw / 8;
  uint4 q[8];
  auto fetch = [&](int s) {
    const long long row = r_lo + (long long)s * kRowsStage + srow;
    const bool row_in = row < r_hi;
    const long long rows_lim = row_in ? a.rows : 0;  // rows of the next CTA's slab read as zero
    const float sc = (row_in && a.kscale != nullptr) ? __ldg(a.kscale + row) : 1.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int g = gsel + 4 * j;
      if (g < 16) q[j] = load8_bf16(a.dz, a.lddz, row, rows_lim, m0 + 8 * g, a.out, 1.f, dz_vec);
      else if (g < ngroups) q[j] = load8_bf16(a.x, a.ldx, row, rows_lim, n0 + 8 * (g - 16), a.width, sc, x_vec);
    }
  };
  auto stash = [&](int sb) {
    uint8_t* base = smem + sb * kStageBytes + srow * 16;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int g = gsel + 4 * j;
      if (g < ngroups) *reinterpret_cast<uint4*>(base + g * (kRowsStage * 16)) = q[j];
    }
  };

  float acc[2][32];
  if (nstages > 0) fetch(0);
  for (int s = 0; s < nstages; ++s) {
    const int sb = s & 1;
    stash(sb);
    fence_proxy_async_smem();
    __syncthreads();  // stage s is complete; the wgmmas of stage s - 1 (other buffer) have retired
    if (s + 1 < nstages) fetch(s + 1);
    const uint32_t a_addr = smem_u32(smem + sb * kStageBytes) + wg * 8 * (kRowsStage * 16);
    const uint32_t b_addr = smem_u32(smem + sb * kStageBytes) + 16 * (kRowsStage * 16);
    fence_regs<32>(acc[0]);
    fence_regs<32>(acc[1]);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      // 16 rows of the reduction = two 8-row core-matrix groups (LBO = 128 B apart); 8-column groups along M / N
      // at SBO = 64 rows * 16 B
      const uint64_t ad = smem_desc(a_addr + ks * 256, 128, kRowsStage * 16);
      const uint32_t sc = (s > 0 || ks > 0) ? 1u : 0u;
#pragma unroll
      for (int b = 0; b < 2; ++b)
        if (64 * b < nw)
          mma_block_mn(acc[b], min(64, nw - 64 * b), ad,
                       smem_desc(b_addr + 64 * b / 8 * (kRowsStage * 16) + ks * 256, 128, kRowsStage * 16), sc);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<32>(acc[0]);
    fence_regs<32>(acc[1]);
  }
  if (nstages == 0) return;

  // ---------------- epilogue: fragment -> this slab's partial ----------------
  float* part = a.part + (long long)blockIdx.x * a.out * a.width;
  const int w = warp & 3;
#pragma unroll
  for (int b = 0; b < 2; ++b) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (64 * b + 8 * j >= nw) continue;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int o = m0 + 64 * wg + 16 * w + (lane >> 2) + 8 * h;
        if (o >= a.out) continue;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = n0 + 64 * b + 8 * j + 2 * (lane & 3) + e;
          if (c < a.width) part[(long long)o * a.width + c] = acc[b][4 * j + 2 * h + e];
        }
      }
    }
  }
}

// W'(n, k) = W[k * ldw + n] for n < N (= width), k < K (= out): the transposed slice as linear_tc chunk images
__global__ void pack_wt_tc_kernel(const float* __restrict__ W, long long ldw, int N, int K, int Npad, int nchunks,
                                  __nv_bfloat16* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long tot = (long long)nchunks * Npad * 64;
  if (idx >= tot) return;
  const int c = (int)(idx / ((long long)Npad * 64));
  const int rem = (int)(idx % ((long long)Npad * 64));
  // consecutive threads run along n (the unit-stride dimension of W)
  const int kk = rem / Npad, n = rem % Npad;
  const int k = c * 64 + kk;
  const float v = (n < N && k < K) ? W[(long long)k * ldw + n] : 0.f;
  const size_t off = (size_t)c * Npad * 64 * 2 + tile_off((uint32_t)Npad, (uint32_t)n, (uint32_t)kk);
  *reinterpret_cast<__nv_bfloat16*>(reinterpret_cast<uint8_t*>(out) + off) = __float2bfloat16_rn(v);
}

}  // namespace

bool tc_grad_w_ok(int out, int width, long long rows) { return out >= 1 && out <= 256 && width >= 1 && width <= 256 && rows >= 2048; }
bool tc_grad_in_ok(int out, int width, long long rows) { return width >= 16 && width <= 256 && out >= 16 && rows >= 2048; }
size_t tc_grad_in_scratch_bytes() { return tc_packed_bytes(256, 320); }

int tc_grad_w(const float* dz, long long lddz, int out, long long rows, const float* x, long long ldx, int width,
              const float* kscale, float* dW, long long ldw, float* red, cudaStream_t st) {
  if (rows == 0) return DYN_OK;
  if (!tc_grad_w_ok(out, width, rows)) return fail(DYN_E_INVALID, "tc_grad_w: unsupported shape %d x %d", out, width);
  if (red == nullptr) return fail(DYN_E_INVALID, "tc_grad_w: no reduction scratch");
  GradWArgs a;
  a.dz = dz; a.lddz = lddz; a.out = out; a.x = x; a.ldx = ldx; a.width = width; a.kscale = kscale;
  a.rows = rows; a.part = red;
  a.mtiles = (out + kTileM - 1) / kTileM;
  a.nblocks = (width + kTileN - 1) / kTileN;
  // slabs: about one wave of kGwCtas CTAs (an H100 has 132 SMs) over all dW tiles, at least 1024 rows each.  tiles is
  // 1, 2 or 4, so slabs * out * width <= kGwCtas * 128 * 128 = kRedFloats.
  constexpr int kGwCtas = 128;
  const int tiles = a.mtiles * a.nblocks;
  long long slabs = kGwCtas / tiles;
  long long per = (rows + slabs - 1) / slabs;
  per = per < 1024 ? 1024 : per;
  per = (per + kRowsStage - 1) / kRowsStage * kRowsStage;
  a.rows_per_cta = per;
  static bool attr_set = false;
  if (!attr_set) {
    DYN_CUDA(cudaFuncSetAttribute(grad_w_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kGwSmem));
    attr_set = true;
  }
  const long long nslabs = (rows + per - 1) / per;
  if (nslabs * out * width > kRedFloats) return fail(DYN_E_INVALID, "tc_grad_w: partials exceed the reduction scratch");
  const dim3 grid((unsigned)nslabs, (unsigned)tiles);
  grad_w_tc_kernel<<<grid, 256, kGwSmem, st>>>(a);
  DYN_LAUNCH_CHECK();
  return launch_red_add(red, (int)nslabs, (long long)out * width, out, width, dW, ldw, true, st);
}

int tc_grad_in(const float* dz, long long lddz, int out, long long rows, const float* W, long long ldw, int width,
               float* din, long long ldd, void* img_scratch, cudaStream_t st) {
  if (rows == 0) return DYN_OK;
  if (!tc_grad_in_ok(out, width, rows)) return fail(DYN_E_INVALID, "tc_grad_in: unsupported shape %d x %d", out, width);
  const int Npad = (width + 15) / 16 * 16;
  const int nchunks = (out + 63) / 64;
  if (tc_packed_bytes(width, out) > tc_grad_in_scratch_bytes()) return fail(DYN_E_INVALID, "tc_grad_in: image too large");
  const long long tot = (long long)nchunks * Npad * 64;
  pack_wt_tc_kernel<<<cdiv(tot, 256), 256, 0, st>>>(W, ldw, width, out, Npad, nchunks,
                                                    reinterpret_cast<__nv_bfloat16*>(img_scratch));
  DYN_LAUNCH_CHECK();
  LinArgs a = lin1(dz, (int)lddz, nullptr, nullptr, din, (int)ldd, rows, width, out, ACT_NONE);
  return launch_linear_tc(a, img_scratch, st);
}

}  // namespace dyn

using namespace dyn;

// unit-test hooks (tests/test_train_gpu.py): plain fp32 matrices in and out
// The slab partials live in a stream-ordered allocation of this hook's own (the library's entry points take them from
// the caller's scratch).
extern "C" int dyn_debug_tc_grad_w(const float* dz, int lddz, int out, int rows, const float* x, int ldx, int width,
                                   const float* kscale, float* dW, int ldw, void* stream) {
  DYN_CHECK_ARG(dz && x && dW);
  cudaStream_t st = (cudaStream_t)stream;
  void* red = nullptr;
  DYN_CUDA(cudaMallocAsync(&red, red_scratch_bytes(), st));
  const int rc = tc_grad_w(dz, lddz, out, rows, x, ldx, width, kscale, dW, ldw, (float*)red, st);
  DYN_CUDA(cudaFreeAsync(red, st));
  return rc;
}

extern "C" int dyn_debug_tc_grad_in(const float* dz, int lddz, int out, int rows, const float* W, int ldw, int width,
                                    float* din, int ldd, void* scratch, size_t scratch_bytes, void* stream) {
  DYN_CHECK_ARG(dz && W && din && scratch && scratch_bytes >= tc_grad_in_scratch_bytes());
  return tc_grad_in(dz, lddz, out, rows, W, ldw, width, din, ldd, scratch, (cudaStream_t)stream);
}

extern "C" size_t dyn_debug_tc_grad_in_scratch_bytes(void) { return tc_grad_in_scratch_bytes(); }
