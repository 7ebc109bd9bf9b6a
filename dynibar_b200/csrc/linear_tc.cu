// Generic tensor-core linear layer  Y = act(concat(segments) * W^T + b)
// on wgmma (bf16 operands, fp32 accumulation in registers).
//
// One CTA computes a 128-row slab for the full output width N <= 256: two warpgroups of 64 rows, K in
// chunks of 64; per chunk every thread loads its share of the slab (global fp32 -> bf16 -> canonical smem
// tile, the next chunk's loads in flight during the MMAs) and thread 0 lands the weight chunk by cp.async.bulk.
// Used for the per-point layers of the aggregation networks and, until the
// fused per-view kernels take over, for every large layer in DYN_PREC_BF16 mode.
#include "linear_tc.cuh"
#include "tc.cuh"

namespace dyn {

using namespace tc;

namespace {

constexpr int kKC = 64;                   // K per chunk
constexpr int kRows = 128;                // rows per CTA
constexpr int kATile = kRows * kKC * 2;   // one A chunk: 16 KB
__host__ __device__ constexpr int smem_bytes(int Npad) { return 2 * kATile + 2 * Npad * kKC * 2 + 64; }

__device__ __forceinline__ float act_f(float v, int act) {
  switch (act) {
    case ACT_ELU: return elu_f(v);
    case ACT_RELU: return fmaxf(v, 0.f);
    case ACT_SIGMOID: return sigmoid_f(v);
    default: return v;
  }
}

__device__ __forceinline__ float seg_value(const TcLinArgs& a, long long row, int col) {
  int c = col;
#pragma unroll
  for (int s = 0; s < 4; ++s) {
    if (s < a.nseg) {
      if (c < a.seg[s].width) return a.seg[s].p[(row / a.seg[s].div) * a.seg[s].ld + c];
      c -= a.seg[s].width;
    }
  }
  return 0.f;
}

// D[64 x w] (+)= A * B for one N-block of w <= 64 columns
__device__ __forceinline__ void mma_block(float* d, int w, uint64_t ad, uint64_t bd, uint32_t sc) {
  switch (w) {
    case 16: Wgmma<16, 0, 0>::mma(d, ad, bd, sc); break;
    case 32: Wgmma<32, 0, 0>::mma(d, ad, bd, sc); break;
    case 48: Wgmma<48, 0, 0>::mma(d, ad, bd, sc); break;
    default: Wgmma<64, 0, 0>::mma(d, ad, bd, sc); break;
  }
}

__global__ void __launch_bounds__(256, 1) linear_tc_kernel(const __grid_constant__ TcLinArgs a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int wsb = a.Npad * kKC * 2;  // bytes per weight chunk
  uint8_t* a_buf = smem;             // 2 x 16 KB
  uint8_t* w_buf = smem + 2 * kATile;
  const uint32_t bar0 = smem_u32(w_buf + 2 * wsb);  // [0,1]: weight chunk of stage s has landed
  const int tid = threadIdx.x, wg = tid >> 7;
  const long long m0 = (long long)blockIdx.x * kRows;
  const int nchunks = a.nchunks;
  const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(a.Wp);
  if (tid == 0) {
    mbar_init(bar0, 1);
    mbar_init(bar0 + 8, 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(bar0, (uint32_t)wsb);
    bulk_g2s(smem_u32(w_buf), wsrc, (uint32_t)wsb, bar0);
  }

  // operand loads: thread -> k-group kg (8 columns) of slab rows lr0 + 32 i
  const int kg = tid & 7, lr0 = tid >> 3;
  const bool dense = a.nseg == 1 && a.seg[0].div == 1 && (a.seg[0].ld & 3) == 0 &&
                     ((reinterpret_cast<uintptr_t>(a.seg[0].p) & 15) == 0);
  float v[4][8];
  auto fetch = [&](int kc) {
    const int k0 = kc * kKC + 8 * kg;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const long long row = m0 + lr0 + 32 * i;
      const bool ok = row < a.M;
      const float rs = (ok && a.row_scale) ? __ldg(a.row_scale + row) : 1.f;
      if (ok && dense && k0 + 8 <= a.K) {
        const float4* src = reinterpret_cast<const float4*>(a.seg[0].p + row * a.seg[0].ld + k0);
        const float4 q0 = __ldg(src), q1 = __ldg(src + 1);
        v[i][0] = q0.x * rs; v[i][1] = q0.y * rs; v[i][2] = q0.z * rs; v[i][3] = q0.w * rs;
        v[i][4] = q1.x * rs; v[i][5] = q1.y * rs; v[i][6] = q1.z * rs; v[i][7] = q1.w * rs;
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[i][j] = (ok && k0 + j < a.K) ? seg_value(a, row, k0 + j) * rs : 0.f;
      }
    }
  };
  auto stash = [&](int s) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      uint4 q;
      q.x = pack_bf16x2(v[i][0], v[i][1]); q.y = pack_bf16x2(v[i][2], v[i][3]);
      q.z = pack_bf16x2(v[i][4], v[i][5]); q.w = pack_bf16x2(v[i][6], v[i][7]);
      *reinterpret_cast<uint4*>(a_buf + s * kATile + tile_off(kRows, lr0 + 32 * i, 8 * kg)) = q;
    }
  };

  float acc[4][32];
  fetch(0);
  for (int kc = 0; kc < nchunks; ++kc) {
    const int s = kc & 1;
    stash(s);
    fence_proxy_async_smem();
    __syncthreads();  // A chunk kc is complete; every warpgroup has retired its wgmmas of chunk kc - 1
    if (tid == 0 && kc + 1 < nchunks) {  // stage s ^ 1 held chunk kc - 1
      mbar_arrive_expect_tx(bar0 + 8u * (s ^ 1), (uint32_t)wsb);
      bulk_g2s(smem_u32(w_buf + (s ^ 1) * wsb), wsrc + (size_t)(kc + 1) * wsb, (uint32_t)wsb, bar0 + 8u * (s ^ 1));
    }
    if (kc + 1 < nchunks) fetch(kc + 1);
    mbar_wait(bar0 + 8u * s, (kc >> 1) & 1);
    int ksteps = (a.K - kc * kKC + 15) / 16;
    if (ksteps > 4) ksteps = 4;
    const uint32_t a_addr = smem_u32(a_buf + s * kATile) + wg * 1024u;
    const uint32_t w_addr = smem_u32(w_buf + s * wsb);
#pragma unroll
    for (int b = 0; b < 4; ++b) fence_regs<32>(acc[b]);
    wgmma_fence();
    for (int ks = 0; ks < ksteps; ++ks) {
      const uint64_t ad = smem_desc(a_addr + ks * 2 * (kRows * 16), kRows * 16, 128);
      const uint32_t sc = (kc > 0 || ks > 0) ? 1u : 0u;
#pragma unroll
      for (int b = 0; b < 4; ++b)
        if (64 * b < a.Npad)
          mma_block(acc[b], min(64, a.Npad - 64 * b),
                    ad, smem_desc(w_addr + 64 * b * 16 + ks * 2 * (a.Npad * 16), a.Npad * 16, 128), sc);
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int b = 0; b < 4; ++b) fence_regs<32>(acc[b]);
  }

  // ---------------- epilogue: bias, activation, fp32 out ----------------
  const int w = (tid >> 5) & 3, l = tid & 31;
#pragma unroll
  for (int b = 0; b < 4; ++b) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col0 = 64 * b + 8 * j + 2 * (l & 3);
      if (64 * b + 8 * j >= a.Npad) continue;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long row = m0 + 64 * wg + 16 * w + (l >> 2) + 8 * h;
        if (row >= a.M) continue;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = col0 + e;
          if (col < a.N) a.Y[row * a.ldy + col] = act_f(acc[b][4 * j + 2 * h + e] + (a.b ? __ldg(a.b + col) : 0.f), a.act);
        }
      }
    }
  }
}

// W fp32 [N,K] row-major -> bf16 chunk images: chunk c holds k in [64c, 64c+64)
// as an [Npad x 64] K-major interleaved tile (zero padded).
__global__ void pack_w_tc_kernel(const float* __restrict__ W, int N, int K, int Npad, int nchunks,
                                 __nv_bfloat16* __restrict__ out) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long tot = (long long)nchunks * Npad * kKC;
  if (idx >= tot) return;
  int c = (int)(idx / ((long long)Npad * kKC));
  int rem = (int)(idx % ((long long)Npad * kKC));
  int n = rem / kKC, kk = rem % kKC;
  int k = c * kKC + kk;
  float v = (n < N && k < K) ? W[(long long)n * K + k] : 0.f;
  size_t off = (size_t)c * Npad * kKC * 2 + tile_off((uint32_t)Npad, (uint32_t)n, (uint32_t)kk);
  *reinterpret_cast<__nv_bfloat16*>(reinterpret_cast<uint8_t*>(out) + off) = __float2bfloat16_rn(v);
}

}  // namespace

size_t tc_packed_bytes(int N, int K) {
  int Npad = (N + 15) / 16 * 16;
  int nchunks = (K + kKC - 1) / kKC;
  return (size_t)nchunks * Npad * kKC * 2;
}

int tc_pack_weight(const float* W, int N, int K, void* out, cudaStream_t st) {
  int Npad = (N + 15) / 16 * 16;
  int nchunks = (K + kKC - 1) / kKC;
  long long tot = (long long)nchunks * Npad * kKC;
  pack_w_tc_kernel<<<cdiv(tot, 256), 256, 0, st>>>(W, N, K, Npad, nchunks,
                                                   reinterpret_cast<__nv_bfloat16*>(out));
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int launch_linear_tc(const LinArgs& f, const void* packed_w, cudaStream_t st) {
  if (f.M == 0) return DYN_OK;
  if (f.N > 256) return fail(DYN_E_INVALID, "linear_tc: N %d > 256", f.N);
  int ksum = 0;
  for (int s = 0; s < f.nseg; ++s) ksum += f.seg[s].width;
  if (ksum != f.K) return fail(DYN_E_INVALID, "linear_tc: segment widths %d != K %d", ksum, f.K);
  TcLinArgs a;
  memset(&a, 0, sizeof(a));
  for (int s = 0; s < 4; ++s) a.seg[s] = f.seg[s];
  a.nseg = f.nseg; a.row_scale = f.row_scale;
  a.Wp = packed_w; a.b = f.b; a.Y = f.Y; a.ldy = f.ldy;
  a.M = f.M; a.N = f.N; a.K = f.K; a.act = f.act;
  a.Npad = (f.N + 15) / 16 * 16;
  a.nchunks = (f.K + kKC - 1) / kKC;
  static bool attr_set = false;
  if (!attr_set) {
    DYN_CUDA(cudaFuncSetAttribute(linear_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes(256)));
    attr_set = true;
  }
  linear_tc_kernel<<<cdiv(f.M, kRows), 256, smem_bytes(a.Npad), st>>>(a);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

}  // namespace dyn

using namespace dyn;

extern "C" int dyn_linear_tc(const float* X, int ldx, const float* W, const float* b, int M, int N,
                             int K, int act, float* Y, int ldy, void* packed_ws, size_t packed_ws_bytes,
                             void* stream) {
  DYN_CHECK_ARG(X && W && Y && packed_ws && M >= 0 && N >= 1 && N <= 256 && K >= 1);
  DYN_CHECK_ARG(packed_ws_bytes >= tc_packed_bytes(N, K));
  cudaStream_t st = (cudaStream_t)stream;
  int rc = tc_pack_weight(W, N, K, packed_ws, st);
  if (rc) return rc;
  LinArgs a = lin1(X, ldx, W, b, Y, ldy, M, N, K, act);
  return launch_linear_tc(a, packed_ws, st);
}

extern "C" size_t dyn_linear_tc_packed_bytes(int N, int K) { return tc_packed_bytes(N, K); }
