// Training slice of the MotionMLP (row f2): forward that keeps its activations, and the backward.
//
//   MotionMLP.forward (ibrnet/mlp_network.py:605-618):
//     x0 = PeriodicEmbed(xyzt) [N,132];  h = x0
//     for i in 0..7:  h = relu(pts_linears[i](h));  if i == 4: h = cat([x0, h])
//     coeff = coeff_linear(h)                                            [N, 3 nb]
//
//   backward, fp32, one GEMM per product:
//     dZ_i = dH_{i+1} * (out_i > 0)                    relu_mask_kernel
//     dW_i += dZ_i^T in_i, db_i += colsum(dZ_i)        gemm_f32_kernel (split-K over the rows: partials in order)
//     dIn_i = dZ_i W_i                                  gemm_f32_kernel
//     layer 5 reads cat([x0, out_4]): its dIn splits into a contribution to dx0 and dH
//     d xyzt = PeriodicEmbed backward of dx0
//
// The gradients are ACCUMULATED into d_params (the caller zeroes it), in the same flat layout as the
// parameter blob of the forward (motion_layout).  Split-K partials are added in split order (train_gemm.cuh), no
// float atomics: the same inputs give the same bits.  tests/test_backward_gpu.py checks them against autograd
// through the oracle.
#include "common.cuh"
#include "linear_f32.cuh"
#include "linear_tc.cuh"
#include "nets.cuh"
#include "train_gemm.cuh"

namespace dyn {

namespace {

// the product kernel behind launch_gemm (train_gemm.cuh): 64 x 64 x 16 tiles, 256 threads, 4 x 4 outputs per thread
__global__ void __launch_bounds__(256) gemm_f32_kernel(const GemmArgs a) {
  __shared__ float As[16][64 + 4];
  __shared__ float Bs[16][64 + 4];
  const int tid = threadIdx.x;
  const long long m0 = (long long)blockIdx.x * 64, n0 = (long long)blockIdx.y * 64;
  const long long k_lo = (long long)blockIdx.z * a.k_per_split;
  const long long k_hi = k_lo + a.k_per_split < a.K ? k_lo + a.k_per_split : a.K;
  const int tm = (tid >> 4) * 4, tn = (tid & 15) * 4;
  float acc[4][4] = {};
  // loader mapping: consecutive threads run along the unit-stride dimension of each operand
  const bool a_kfast = a.sak == 1, b_nfast = a.sbn == 1;
  for (long long k0 = k_lo; k0 < k_hi; k0 += 16) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int idx = tid + e * 256;  // 0..1023
      {
        const int kk = a_kfast ? (idx & 15) : (idx >> 6), mm = a_kfast ? (idx >> 4) : (idx & 63);
        const long long m = m0 + mm, k = k0 + kk;
        As[kk][mm] = (m < a.M && k < k_hi) ? a.A[m * a.sam + k * a.sak] : 0.f;
      }
      {
        const int kk = b_nfast ? (idx >> 6) : (idx & 15), nn = b_nfast ? (idx & 63) : (idx >> 4);
        const long long n = n0 + nn, k = k0 + kk;
        float bv = (n < a.N && k < k_hi) ? a.B[(a.bdiv > 1 ? k / a.bdiv : k) * a.sbk + n * a.sbn] : 0.f;
        if (a.kscale != nullptr && k < k_hi) bv *= a.kscale[k];
        Bs[kk][nn] = bv;
      }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      const float4 av = *reinterpret_cast<const float4*>(&As[kk][tm]);
      const float4 bv = *reinterpret_cast<const float4*>(&Bs[kk][tn]);
      const float ar[4] = {av.x, av.y, av.z, av.w}, br[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
    }
    __syncthreads();
  }
  // one split: every element has one owner (written, or added once); several: a dense [split, M, N] partial
  const bool split = gridDim.z > 1;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long m = m0 + tm + i, n = n0 + tn + j;
      if (m < a.M && n < a.N) {
        if (split) {
          a.red[((long long)blockIdx.z * a.M + m) * a.N + n] = acc[i][j];
        } else {
          float* c = a.C + m * a.ldc + n;
          *c = a.accumulate ? *c + acc[i][j] : acc[i][j];
        }
      }
    }
}

// C[m * ldc + n] (+)= sum_s part[s * sstride + m * N + n], s = 0, 1, ... in order
__global__ void red_add_kernel(const float* __restrict__ part, int slabs, long long sstride, long long M, long long N,
                               float* __restrict__ C, long long ldc, int accumulate) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * N) return;
  const long long m = idx / N, n = idx - m * N;
  float s = part[idx];
  for (int k = 1; k < slabs; ++k) s += part[k * sstride + idx];
  float* c = C + m * ldc + n;
  *c = accumulate ? *c + s : s;
}

}  // namespace

int launch_red_add(const float* part, int slabs, long long sstride, long long M, long long N, float* C, long long ldc,
                   bool accumulate, cudaStream_t st) {
  if (M == 0 || N == 0 || slabs == 0) return DYN_OK;
  red_add_kernel<<<cdiv(M * N, 256), 256, 0, st>>>(part, slabs, sstride, M, N, C, ldc, accumulate ? 1 : 0);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int launch_gemm(GemmArgs a, bool split_k, cudaStream_t st) {
  if (a.M == 0 || a.N == 0) return DYN_OK;
  int splits = 1;
  if (split_k) {
    // a split per 4096 rows, at most 128 and at most as many partials as the reduction scratch holds
    const long long want = (a.K + 4095) / 4096;
    const long long fit = kRedFloats / (a.M * a.N);
    splits = (int)(want < 1 ? 1 : (want > 128 ? 128 : want));
    if (splits > fit) splits = (int)(fit < 1 ? 1 : fit);
  }
  a.k_per_split = ((a.K + splits - 1) / splits + 15) / 16 * 16;
  if (a.k_per_split == 0) a.k_per_split = 16;
  splits = (int)((a.K + a.k_per_split - 1) / a.k_per_split);
  if (splits < 1) splits = 1;
  if (splits > 1 && a.red == nullptr) return fail(DYN_E_INVALID, "launch_gemm: a split product needs reduction scratch");
  dim3 grid((unsigned)((a.M + 63) / 64), (unsigned)((a.N + 63) / 64), (unsigned)splits);
  gemm_f32_kernel<<<grid, 256, 0, st>>>(a);
  DYN_LAUNCH_CHECK();
  if (splits > 1) return launch_red_add(a.red, splits, a.M * a.N, a.M, a.N, a.C, a.ldc, a.accumulate != 0, st);
  return DYN_OK;
}

namespace {

// g[r, c] *= (out[r, c] > 0)   (ReLU backward; g has leading dimension ldg, out is dense [N, width])
__global__ void relu_mask_kernel(float* __restrict__ g, long long ldg, const float* __restrict__ out, int width,
                                 long long N) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N * width) return;
  const long long r = idx / width;
  const int c = (int)(idx - r * width);
  if (!(out[idx] > 0.f)) g[r * ldg + c] = 0.f;
}

// sum_r g[r, c] over a slab of rows: a block owns 32 columns x one slab; one slab adds into db[c], several write
// part[slab, c] for launch_red_add
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ g, long long ldg, int width,
                                                     long long N, long long rows_per_block, float* __restrict__ db,
                                                     float* __restrict__ part) {
  __shared__ float red[8][32];
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  const int ry = threadIdx.x >> 5;
  const long long r0 = (long long)blockIdx.y * rows_per_block;
  const long long r1 = r0 + rows_per_block < N ? r0 + rows_per_block : N;
  float s = 0.f;
  if (c < width)
    for (long long r = r0 + ry; r < r1; r += 8) s += g[r * ldg + c];
  red[ry][threadIdx.x & 31] = s;
  __syncthreads();
  if (ry == 0 && c < width) {
#pragma unroll
    for (int i = 1; i < 8; ++i) s += red[i][threadIdx.x & 31];
    if (gridDim.y == 1) db[c] += s;
    else part[(long long)blockIdx.y * width + c] = s;
  }
}

}  // namespace

int launch_colsum(const float* g, long long ldg, int width, long long N, float* db, float* red, cudaStream_t st) {
  if (N == 0) return DYN_OK;
  // slabs of 2048 rows: a call on rows [0, N) and calls on ray slices that start at multiples of 2048 rows form the
  // same slab sums
  const long long rows_per_block = 2048;
  const long long slabs = (N + rows_per_block - 1) / rows_per_block;
  if (slabs > 1 && (red == nullptr || slabs * width > kRedFloats))
    return fail(DYN_E_INVALID, "launch_colsum: %lld slabs of %d columns need reduction scratch", slabs, width);
  dim3 grid((unsigned)((width + 31) / 32), (unsigned)slabs);
  colsum_kernel<<<grid, 256, 0, st>>>(g, ldg, width, N, rows_per_block, db, red);
  DYN_LAUNCH_CHECK();
  if (slabs > 1) return launch_red_add(red, (int)slabs, width, 1, width, db, width, true, st);
  return DYN_OK;
}

namespace {

// PeriodicEmbed backward (mlp_network.py:530-555, layout of pe_kernel in nets_f32.cu):
// x0 = [x, cos(f_k x) (k = 0..n-1), sin(f_k x) (k = 0..n-1)], each block D = 4 wide
struct MotionFreqs {
  float f[16];
};

__global__ void pe_backward_kernel(const float* __restrict__ xyzt, const float* __restrict__ dx0,
                                   const float* __restrict__ dx0_skip, MotionFreqs q, long long N,
                                   float* __restrict__ dxyzt) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N * 4) return;
  const long long r = idx >> 2;
  const int d = (int)(idx & 3);
  const float x = xyzt[idx];
  const float* g = dx0 + r * 132;
  const float* h = dx0_skip + r * 132;  // the part that arrived through the skip connection of layer 5
  float s = g[d] + h[d];
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    float sn, cs;
    sincosf(q.f[k] * x, &sn, &cs);
    s += q.f[k] * (cs * (g[(17 + k) * 4 + d] + h[(17 + k) * 4 + d]) - sn * (g[(1 + k) * 4 + d] + h[(1 + k) * 4 + d]));
  }
  dxyzt[idx] = s;
}

struct TrainBufs {
  float* x0;       // [N,132]
  float* out[8];   // [N,256] post-ReLU outputs of pts_linears
  float* ga;       // [N,256] gradient ping
  float* gb;       // [N,256] gradient pong
  float* gw;       // [N,388] dIn of layer 5 (cat([x0, out_4])); reused for the [N,132] dIn of layer 0
  float* gx0;      // [N,132] gradient of x0 through the skip connection
  float* img;      // transposed weight image of the tensor-core dIn product
  float* red;      // partials of the fixed-order reductions (train_gemm.cuh)
};

size_t train_alloc(char* base, long long N, TrainBufs* t) {
  size_t off = 0;
  auto take = [&](size_t n) {
    off = (off + 255) & ~(size_t)255;
    float* p = base ? reinterpret_cast<float*>(base + off) : nullptr;
    off += n * sizeof(float);
    return p;
  };
  t->x0 = take((size_t)N * 132);
  for (int i = 0; i < 8; ++i) t->out[i] = take((size_t)N * 256);
  t->ga = take((size_t)N * 256);
  t->gb = take((size_t)N * 256);
  t->gw = take((size_t)N * 388);
  t->gx0 = take((size_t)N * 132);
  t->img = take(tc_grad_in_scratch_bytes() / sizeof(float));
  t->red = take((size_t)kRedFloats);
  return off;
}

}  // namespace

size_t motion_train_workspace(long long N) {
  TrainBufs t;
  return train_alloc(nullptr, N, &t);
}

int motion_train_forward(const dyn_net* n, const float* xyzt, long long N, float* coeff, void* ws,
                         size_t ws_bytes, int prec, cudaStream_t st) {
  const bool tc = prec == DYN_PREC_BF16;
  if (tc && n->packed == nullptr) return fail(DYN_E_INVALID, "bf16 training needs a net created with layer images");
  const MotionLayout& L = n->ml;
  TrainBufs t;
  if (train_alloc((char*)ws, N, &t) > ws_bytes)
    return fail(DYN_E_WORKSPACE, "motion train: workspace %zu < %zu", ws_bytes, motion_train_workspace(N));
  int rc = motion_embed(xyzt, N, t.x0, st);
  if (rc) return rc;
  auto P = [&](int off) { return off < 0 ? nullptr : n->params + off; };
  for (int i = 0; i < 8; ++i) {
    const LinearP& l = L.pts[i];
    LinArgs a = lin1(i == 0 ? t.x0 : t.out[i - 1], l.in, P(l.w), P(l.b), t.out[i], 256, N, 256, l.in, ACT_RELU);
    if (i == 5) {  // skip connection: input is cat([x0, out_4]) (:612-613)
      a.seg[0] = Seg{t.x0, 132, 132, 1};
      a.seg[1] = Seg{t.out[4], 256, 256, 1};
      a.nseg = 2;
    }
    rc = (tc && N >= 128) ? launch_linear_tc(a, reinterpret_cast<const char*>(n->packed) + l.tc, st)
                          : launch_linear(a, st);
    if (rc) return rc;
  }
  const LinearP& lc = L.coeff;
  return launch_linear(lin1(t.out[7], 256, P(lc.w), P(lc.b), coeff, lc.out, N, lc.out, 256, ACT_NONE), st);
}

int motion_train_backward(const dyn_net* n, const float* xyzt, const float* d_coeff, long long N, void* ws,
                          size_t ws_bytes, float* d_params, float* d_xyzt, int prec, cudaStream_t st) {
  const bool tc = prec == DYN_PREC_BF16;
  const MotionLayout& L = n->ml;
  TrainBufs t;
  if (train_alloc((char*)ws, N, &t) > ws_bytes)
    return fail(DYN_E_WORKSPACE, "motion train: workspace %zu < %zu", ws_bytes, motion_train_workspace(N));
  if (N == 0) return DYN_OK;
  int rc;
#define MT_RUN(e) do { rc = (e); if (rc) return rc; } while (0)
  // product helpers on row-major operands
  auto grad_w = [&](const float* dz, long long lddz, int out, const float* in, long long ldin, int width,
                    float* dW, long long lddw) {  // dW[out, width] += dz^T in
    if (tc && tc_grad_w_ok(out, width, N))
      return tc_grad_w(dz, lddz, out, N, in, ldin, width, nullptr, dW, lddw, t.red, st);
    GemmArgs g{dz, in, dW, out, width, N, 1, lddz, ldin, 1, lddw, 1, 0};
    g.red = t.red;
    return launch_gemm(g, true, st);
  };
  auto grad_in = [&](const float* dz, long long lddz, int out, const float* W, int in, float* din, long long ldd) {
    if (tc && in <= 256 && tc_grad_in_ok(out, in, N)) return tc_grad_in(dz, lddz, out, N, W, in, in, din, ldd, t.img, st);
    if (tc && in > 256 && tc_grad_in_ok(out, 256, N) && tc_grad_in_ok(out, in - 256, N)) {  // 388 = 256 + 132
      int rc2 = tc_grad_in(dz, lddz, out, N, W, in, 256, din, ldd, t.img, st);
      if (rc2) return rc2;
      return tc_grad_in(dz, lddz, out, N, W + 256, in, in - 256, din + 256, ldd, t.img, st);
    }
    GemmArgs g{dz, W, din, N, in, out, lddz, 1, in, 1, ldd, 0, 0};  // din[N, in] = dz[N, out] W[out, in]
    return launch_gemm(g, false, st);
  };
  const LinearP& lc = L.coeff;
  MT_RUN(grad_w(d_coeff, lc.out, lc.out, t.out[7], 256, 256, d_params + lc.w, 256));
  MT_RUN(launch_colsum(d_coeff, lc.out, lc.out, N, d_params + lc.b, t.red, st));
  float *g = t.ga, *g2 = t.gb;  // dense [N,256]
  MT_RUN(grad_in(d_coeff, lc.out, lc.out, n->params + lc.w, 256, g, 256));
  for (int i = 7; i >= 0; --i) {
    const LinearP& l = L.pts[i];
    relu_mask_kernel<<<(unsigned)((N * 256 + 255) / 256), 256, 0, st>>>(g, 256, t.out[i], 256, N);
    DYN_LAUNCH_CHECK();
    MT_RUN(launch_colsum(g, 256, 256, N, d_params + l.b, t.red, st));
    if (i == 5) {  // input cat([x0, out_4]): W is [256, 388]
      MT_RUN(grad_w(g, 256, 256, t.x0, 132, 132, d_params + l.w, 388));
      MT_RUN(grad_w(g, 256, 256, t.out[4], 256, 256, d_params + l.w + 132, 388));
      MT_RUN(grad_in(g, 256, 256, n->params + l.w, 388, t.gw, 388));
      DYN_CUDA(cudaMemcpy2DAsync(t.gx0, 132 * sizeof(float), t.gw, 388 * sizeof(float), 132 * sizeof(float),
                                 (size_t)N, cudaMemcpyDeviceToDevice, st));
      DYN_CUDA(cudaMemcpy2DAsync(g2, 256 * sizeof(float), t.gw + 132, 388 * sizeof(float), 256 * sizeof(float),
                                 (size_t)N, cudaMemcpyDeviceToDevice, st));
    } else if (i > 0) {
      MT_RUN(grad_w(g, 256, 256, t.out[i - 1], 256, 256, d_params + l.w, 256));
      MT_RUN(grad_in(g, 256, 256, n->params + l.w, 256, g2, 256));
    } else {
      MT_RUN(grad_w(g, 256, 256, t.x0, 132, 132, d_params + l.w, 132));
      if (d_xyzt != nullptr) {
        MT_RUN(grad_in(g, 256, 256, n->params + l.w, 132, t.gw, 132));
        MotionFreqs q;
        motion_freqs(q.f);
        pe_backward_kernel<<<(unsigned)((N * 4 + 255) / 256), 256, 0, st>>>(xyzt, t.gw, t.gx0, q, N, d_xyzt);
        DYN_LAUNCH_CHECK();
      }
    }
    float* tmp = g; g = g2; g2 = tmp;
  }
#undef MT_RUN
  return DYN_OK;
}

}  // namespace dyn
