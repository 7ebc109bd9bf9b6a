// 2-D feature encoder, the part of ibrnet/feature_network.py the reference actually executes
// (ResNet.forward, feature_network.py:302-311):
//
//   conv1 7x7 stride 2 (3 -> 64, reflect padding, no bias) -> InstanceNorm(affine) -> ReLU
//   layer1: 3 BasicBlocks (64 -> 64; the first with stride 2 and a 1x1 stride-2 + InstanceNorm shortcut):
//           conv3x3 (reflect) -> IN -> ReLU -> conv3x3 -> IN -> (+ identity) -> ReLU     (:42-84)
//   out_conv 1x1 (64 -> 64, bias) -> split into coarse (first 32) and fine (last 32) channels
//
// It runs once per frame on the <= 25 source images (eval_nvidia.py:335-358), ~2.5 GMAC per 288x512 image:
// fp32 SIMT kernels with register tiling (a few ms per frame against > 400 ms of ray rendering; bf16
// tensor-core convolutions would buy < 1 % of the frame).  All statistics in fp64 accumulators.
#include "common.cuh"
#include "train_gemm.cuh"

namespace dyn {

namespace {

__device__ __forceinline__ int reflect_idx(int i, int n) {
  // torch 'reflect' padding: -1 -> 1, n -> n - 2 (pads here are < n).  The tile loaders of the forward convolutions
  // stage the input window of a whole 8 x 16 output tile; on images smaller than a tile (H <= 17 or W <= 33) its rows
  // and columns past the image reach i >= 2n - 1, which reflects to a negative index.  Those values feed only
  // outputs that are never stored; the clamp keeps their loads inside the image.
  i = i < 0 ? -i : i;
  i = i >= n ? 2 * n - 2 - i : i;
  return min(max(i, 0), n - 1);
}

// ---------------------------------------------------------------------------
// conv1: 7x7, stride 2, pad 3 (reflect), 3 -> 64.  Block = 8 x 16 output pixels, thread = 1 pixel x 64
// channels; weights in shared memory as [tap][co] so four output channels come with one 16-byte read.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(128) enc_conv7_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                        int H, int W, int Ho, int Wo, float* __restrict__ y) {
  __shared__ __align__(16) float sw[147 * 64];
  __shared__ float sx[3][21][38];
  const int n = blockIdx.z, ox0 = blockIdx.x * 16, oy0 = blockIdx.y * 8;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  for (int i = tid; i < 147 * 64; i += 128) {
    const int co = i / 147, tap = i % 147;  // w is [co][ci][ky][kx]
    sw[tap * 64 + co] = w[i];
  }
  const int ix0 = ox0 * 2 - 3, iy0 = oy0 * 2 - 3;
  for (int i = tid; i < 3 * 21 * 37; i += 128) {
    const int ci = i / (21 * 37), r = (i / 37) % 21, c = i % 37;
    sx[ci][r][c] = x[((long long)(n * 3 + ci) * H + reflect_idx(iy0 + r, H)) * W + reflect_idx(ix0 + c, W)];
  }
  __syncthreads();
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  for (int ci = 0; ci < 3; ++ci)
    for (int ky = 0; ky < 7; ++ky)
#pragma unroll
      for (int kx = 0; kx < 7; ++kx) {
        const float v = sx[ci][2 * ty + ky][2 * tx + kx];
        const float4* wp = reinterpret_cast<const float4*>(sw + ((ci * 7 + ky) * 7 + kx) * 64);
#pragma unroll
        for (int q = 0; q < 16; ++q) {
          const float4 ww = wp[q];
          acc[4 * q] = fmaf(v, ww.x, acc[4 * q]); acc[4 * q + 1] = fmaf(v, ww.y, acc[4 * q + 1]);
          acc[4 * q + 2] = fmaf(v, ww.z, acc[4 * q + 2]); acc[4 * q + 3] = fmaf(v, ww.w, acc[4 * q + 3]);
        }
      }
  const int ox = ox0 + tx, oy = oy0 + ty;
  if (ox < Wo && oy < Ho) {
#pragma unroll
    for (int co = 0; co < 64; ++co) y[((long long)(n * 64 + co) * Ho + oy) * Wo + ox] = acc[co];
  }
}

// ---------------------------------------------------------------------------
// conv3x3, pad 1 (reflect), 64 -> 64, stride S in {1, 2}, no bias.  Block = 8 x 16 output pixels x 64 output
// channels, 128 threads; thread = 4 consecutive pixels of a row x 16 output channels (64 accumulators);
// input channels in chunks of 8 staged in shared memory with their weights ([ci][tap][co]).
// ---------------------------------------------------------------------------
template <int S>
__global__ void __launch_bounds__(128) enc_conv3_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                        int H, int W, int Ho, int Wo, float* __restrict__ y) {
  constexpr int TH = 8, TW = 16, IH = (TH - 1) * S + 3, IW = (TW - 1) * S + 3, IWP = IW + 1;
  __shared__ __align__(16) float sw[8 * 9 * 64];
  __shared__ float sx[8][IH][IWP];
  const int n = blockIdx.z, ox0 = blockIdx.x * TW, oy0 = blockIdx.y * TH;
  const int tid = threadIdx.x;
  const int cg = tid & 3;          // output channels 16 cg .. 16 cg + 15
  const int pg = tid >> 2;         // pixel group: row pg / 4, columns 4 (pg % 4) .. + 3
  const int py = pg >> 2, px = (pg & 3) * 4;
  float acc[4][16];
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int c = 0; c < 16; ++c) acc[p][c] = 0.f;
  const int ix0 = ox0 * S - 1, iy0 = oy0 * S - 1;
  for (int c0 = 0; c0 < 64; c0 += 8) {
    __syncthreads();
    for (int i = tid; i < 8 * 9 * 64; i += 128) {
      const int co = i & 63, tap = (i >> 6) % 9, ci = i / (9 * 64);
      sw[i] = w[((long long)co * 64 + (c0 + ci)) * 9 + tap];  // w is [co][ci][3][3]
    }
    for (int i = tid; i < 8 * IH * IW; i += 128) {
      const int ci = i / (IH * IW), r = (i / IW) % IH, c = i % IW;
      sx[ci][r][c] = x[((long long)(n * 64 + c0 + ci) * H + reflect_idx(iy0 + r, H)) * W + reflect_idx(ix0 + c, W)];
    }
    __syncthreads();
#pragma unroll 1
    for (int ci = 0; ci < 8; ++ci)
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          float v[4];
#pragma unroll
          for (int p = 0; p < 4; ++p) v[p] = sx[ci][py * S + ky][(px + p) * S + kx];
          const float4* wp = reinterpret_cast<const float4*>(sw + (ci * 9 + ky * 3 + kx) * 64 + 16 * cg);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float4 ww = wp[q];
#pragma unroll
            for (int p = 0; p < 4; ++p) {
              acc[p][4 * q] = fmaf(v[p], ww.x, acc[p][4 * q]); acc[p][4 * q + 1] = fmaf(v[p], ww.y, acc[p][4 * q + 1]);
              acc[p][4 * q + 2] = fmaf(v[p], ww.z, acc[p][4 * q + 2]); acc[p][4 * q + 3] = fmaf(v[p], ww.w, acc[p][4 * q + 3]);
            }
          }
        }
  }
  const int oy = oy0 + py;
  if (oy < Ho) {
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      float* dst = y + ((long long)(n * 64 + 16 * cg + c) * Ho + oy) * Wo + ox0 + px;
#pragma unroll
      for (int p = 0; p < 4; ++p)
        if (ox0 + px + p < Wo) dst[p] = acc[p][c];
    }
  }
}

// 1x1 convolution 64 -> 64 with stride S and optional bias: thread = 1 output pixel x 16 channels
template <int S>
__global__ void __launch_bounds__(256) enc_conv1_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                        const float* __restrict__ bias, int H, int W, int Ho, int Wo,
                                                        int N, float* __restrict__ y) {
  __shared__ __align__(16) float sw[64 * 64];  // [ci][co]
  for (int i = threadIdx.x; i < 4096; i += 256) sw[(i & 63) * 64 + (i >> 6)] = w[i];  // w is [co][ci]
  __syncthreads();
  const long long total = (long long)N * Ho * Wo * 4;
  const long long e = (long long)blockIdx.x * 256 + threadIdx.x;
  if (e >= total) return;
  const int cg = (int)(e & 3);
  const long long pix = e >> 2;
  const int ox = (int)(pix % Wo), oy = (int)((pix / Wo) % Ho), n = (int)(pix / ((long long)Wo * Ho));
  float acc[16];
#pragma unroll
  for (int c = 0; c < 16; ++c) acc[c] = bias ? bias[16 * cg + c] : 0.f;
  const float* xp = x + ((long long)n * 64 * H + (long long)oy * S) * W + (long long)ox * S;
  for (int ci = 0; ci < 64; ++ci) {
    const float v = xp[(long long)ci * H * W];
    const float4* wp = reinterpret_cast<const float4*>(sw + ci * 64 + 16 * cg);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 ww = wp[q];
      acc[4 * q] = fmaf(v, ww.x, acc[4 * q]); acc[4 * q + 1] = fmaf(v, ww.y, acc[4 * q + 1]);
      acc[4 * q + 2] = fmaf(v, ww.z, acc[4 * q + 2]); acc[4 * q + 3] = fmaf(v, ww.w, acc[4 * q + 3]);
    }
  }
#pragma unroll
  for (int c = 0; c < 16; ++c) y[((long long)(n * 64 + 16 * cg + c) * Ho + oy) * Wo + ox] = acc[c];
}

// InstanceNorm2d statistics (biased variance, eps 1e-5): one block per (image, channel) plane
__global__ void __launch_bounds__(256) enc_in_stats_kernel(const float* __restrict__ x, int hw,
                                                           float* __restrict__ mean, float* __restrict__ rstd) {
  const float* p = x + (long long)blockIdx.x * hw;
  double s = 0.0, q = 0.0;
  for (int i = threadIdx.x; i < hw; i += 256) {
    const double v = p[i];
    s += v; q += v * v;
  }
  __shared__ double ss[256], sq[256];
  ss[threadIdx.x] = s; sq[threadIdx.x] = q;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) { ss[threadIdx.x] += ss[threadIdx.x + o]; sq[threadIdx.x] += sq[threadIdx.x + o]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double m = ss[0] / hw;
    const double var = fmax(sq[0] / hw - m * m, 0.0);
    mean[blockIdx.x] = (float)m;
    rstd[blockIdx.x] = (float)(1.0 / sqrt(var + 1e-5));
  }
}

// y = (x - mean) * rstd * gamma + beta [+ residual] [ReLU]; in place when y == x
__global__ void enc_in_apply_kernel(const float* __restrict__ x, const float* __restrict__ mean,
                                    const float* __restrict__ rstd, const float* __restrict__ gamma,
                                    const float* __restrict__ beta, const float* __restrict__ residual, int relu,
                                    int hw, int C, long long total, float* __restrict__ y) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long plane = i / hw;
  const int c = (int)(plane % C);
  float v = (x[i] - mean[plane]) * rstd[plane] * gamma[c] + beta[c];
  if (residual) v += residual[i];
  if (relu) v = fmaxf(v, 0.f);
  y[i] = v;
}

// parameter offsets (floats) inside the blob, in the reference's state_dict order restricted to the
// executed modules: conv1.weight, bn1.{weight,bias}, layer1.{0,1,2}.{conv1.weight, bn1.*, conv2.weight, bn2.*}
// (+ layer1.0.downsample.{0.weight, 1.weight, 1.bias} after layer1.0.bn2), out_conv.{weight,bias}
struct EncLayout {
  int conv1, bn1w, bn1b;
  struct Block { int c1, b1w, b1b, c2, b2w, b2b, dsw, dsbw, dsbb; } blk[3];
  int outw, outb, total;
};
EncLayout enc_layout() {
  EncLayout L;
  int o = 0;
  auto take = [&](int n) { int r = o; o += n; return r; };
  L.conv1 = take(64 * 3 * 49); L.bn1w = take(64); L.bn1b = take(64);
  for (int b = 0; b < 3; ++b) {
    L.blk[b].c1 = take(64 * 64 * 9); L.blk[b].b1w = take(64); L.blk[b].b1b = take(64);
    L.blk[b].c2 = take(64 * 64 * 9); L.blk[b].b2w = take(64); L.blk[b].b2b = take(64);
    if (b == 0) { L.blk[b].dsw = take(64 * 64); L.blk[b].dsbw = take(64); L.blk[b].dsbb = take(64); }
    else { L.blk[b].dsw = L.blk[b].dsbw = L.blk[b].dsbb = -1; }
  }
  L.outw = take(64 * 64); L.outb = take(64);
  L.total = o;
  return L;
}

int in_norm(const float* x, const float* P, int gw, int gb, const float* residual, int relu, int N, int hw,
            float* stats, float* y, cudaStream_t st) {
  enc_in_stats_kernel<<<N * 64, 256, 0, st>>>(x, hw, stats, stats + N * 64);
  DYN_LAUNCH_CHECK();
  const long long total = (long long)N * 64 * hw;
  enc_in_apply_kernel<<<cdiv(total, 256), 256, 0, st>>>(x, stats, stats + N * 64, P + gw, P + gb, residual, relu, hw,
                                                        64, total, y);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}


// ---------------------------------------------------------------------------
// training (row f2): backward of the executed encoder.  Every convolution is differentiated through its im2col
// form so that the two products run on the shared training GEMMs (tensor cores in bf16 mode):
//   dYt [rows, 64]       = dY (NCHW) with rows = (n, oy, ox)
//   col [rows, Cin k k]  = im2col(X) with the forward's reflect padding / stride, column = ci k k + ky k + kx
//                          (the layout of conv.weight [co][ci][ky][kx], so dW = dYt^T col is the weight gradient as is)
//   dcol = dYt W  ->  col2im: scatter-add through the SAME index map (the adjoint of reflect padding for free)
// ---------------------------------------------------------------------------
__global__ void enc_nchw_to_rows_kernel(const float* __restrict__ x, int C, int hw, long long rows,
                                        float* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * C) return;
  const long long r = idx / C;
  const int c = (int)(idx - r * C);
  const long long n = r / hw, pix = r - n * hw;
  out[idx] = x[(n * C + c) * hw + pix];
}

// mode 0: col[r, j] = X[...];  mode 1: atomicAdd(dX[...], col[r, j])
__global__ void enc_im2col_kernel(float* __restrict__ x, int Cin, int H, int W, int Ho, int Wo, int k, int stride,
                                  int pad, long long rows, float* __restrict__ col, int mode) {
  const int K = Cin * k * k;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * K) return;
  const long long r = idx / K;
  const int j = (int)(idx - r * K);
  const int ci = j / (k * k), t = j - ci * k * k, ky = t / k, kx = t - ky * k;
  const int ox = (int)(r % Wo), oy = (int)((r / Wo) % Ho);
  const long long n = r / ((long long)Wo * Ho);
  const int iy = reflect_idx(oy * stride + ky - pad, H), ix = reflect_idx(ox * stride + kx - pad, W);
  float* p = x + ((n * Cin + ci) * H + iy) * W + ix;
  if (mode == 0) col[idx] = *p;
  else atomicAdd(p, col[idx]);
}

__global__ void enc_relu_mask_kernel(float* __restrict__ g, const float* __restrict__ y, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && !(y[i] > 0.f)) g[i] = 0.f;
}

// InstanceNorm2d backward, one block per (image, channel) plane: xh = (x - mean) rstd,
// dx = rstd gamma (dy - mean(dy) - xh mean(dy xh)); dgamma += sum dy xh, dbeta += sum dy.  dx may alias dy.
__global__ void __launch_bounds__(256) enc_in_bwd_kernel(const float* __restrict__ x, const float* dy,
                                                         const float* __restrict__ mean,
                                                         const float* __restrict__ rstd,
                                                         const float* __restrict__ gamma, int hw, int C, float* dx,
                                                         float* __restrict__ dgamma, float* __restrict__ dbeta) {
  const long long plane = blockIdx.x;
  const int c = (int)(plane % C);
  const float* xp = x + plane * hw;
  const float* gp = dy + plane * hw;
  const float m = mean[plane], rs = rstd[plane];
  double s1 = 0.0, s2 = 0.0;
  for (int i = threadIdx.x; i < hw; i += 256) {
    const double g = gp[i];
    s1 += g;
    s2 += g * (double)((xp[i] - m) * rs);
  }
  __shared__ double a1[256], a2[256];
  a1[threadIdx.x] = s1; a2[threadIdx.x] = s2;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) { a1[threadIdx.x] += a1[threadIdx.x + o]; a2[threadIdx.x] += a2[threadIdx.x + o]; }
    __syncthreads();
  }
  const float mg = (float)(a1[0] / hw), mgx = (float)(a2[0] / hw);
  const float k = rs * gamma[c];
  float* op = dx + plane * hw;
  for (int i = threadIdx.x; i < hw; i += 256) {
    const float xh = (xp[i] - m) * rs;
    op[i] = k * (gp[i] - mg - xh * mgx);
  }
  if (threadIdx.x == 0) {
    atomicAdd(dgamma + c, (float)a2[0]);
    atomicAdd(dbeta + c, (float)a1[0]);
  }
}

// saved activations of the training forward (floats)
struct EncSaved {
  float *c1, *a1;                         // half resolution: conv1 output, relu(IN(.))
  struct B { float *cA, *aA, *cB, *o; } b[3];
  float* cds;                             // block 0 shortcut conv output (before its InstanceNorm)
  float* stats[8];                        // mean | rstd per InstanceNorm: bn1, b0.bn1, b0.bn2, b0.ds, b1.bn1, b1.bn2, b2.*
};

size_t enc_saved_alloc(char* base, int N, int H2, int W2, int H4, int W4, EncSaved* s) {
  size_t off = 0;
  auto take = [&](size_t n) {
    off = (off + 255) & ~(size_t)255;
    float* p = base ? reinterpret_cast<float*>(base + off) : nullptr;
    off += n * sizeof(float);
    return p;
  };
  const size_t n2 = (size_t)N * 64 * H2 * W2, n4 = (size_t)N * 64 * H4 * W4;
  s->c1 = take(n2); s->a1 = take(n2);
  for (int i = 0; i < 3; ++i) { s->b[i].cA = take(n4); s->b[i].aA = take(n4); s->b[i].cB = take(n4); s->b[i].o = take(n4); }
  s->cds = take(n4);
  for (int i = 0; i < 8; ++i) s->stats[i] = take((size_t)2 * N * 64);
  return off;
}

struct EncScratch {
  float *g2a, *g2b;        // half-resolution gradients
  float *g4a, *g4b, *g4c;  // quarter-resolution gradients
  float *dyt, *col, *img;
};

size_t enc_scratch_alloc(char* base, int N, int H, int W, int H2, int W2, int H4, int W4, EncScratch* q) {
  size_t off = 0;
  auto take = [&](size_t n) {
    off = (off + 255) & ~(size_t)255;
    float* p = base ? reinterpret_cast<float*>(base + off) : nullptr;
    off += n * sizeof(float);
    return p;
  };
  (void)H; (void)W;
  const size_t n2 = (size_t)N * 64 * H2 * W2, n4 = (size_t)N * 64 * H4 * W4;
  const size_t r2 = (size_t)N * H2 * W2, r4 = (size_t)N * H4 * W4;
  q->g2a = take(n2); q->g2b = take(n2);
  q->g4a = take(n4); q->g4b = take(n4); q->g4c = take(n4);
  q->dyt = take(r2 * 64 > r4 * 64 ? r2 * 64 : r4 * 64);
  const size_t c_stem = r2 * 147, c_33 = r4 * 576;
  q->col = take(c_stem > c_33 ? c_stem : c_33);
  q->img = take(tc_grad_in_scratch_bytes() / sizeof(float));
  return off;
}

// backward of one convolution (see the header of this section).  dX: null = not needed; acc_dx: add to dX
struct ConvBwd {
  cudaStream_t st;
  bool tc;
  EncScratch q;
  int N;
  int run(const float* dY, int Ho, int Wo, const float* Wt, float* dW, float* X, int Cin, int H, int W, int k,
          int stride, int pad, float* dX, bool zero_dx) const {
    const long long rows = (long long)N * Ho * Wo;
    const int K = Cin * k * k;
    enc_nchw_to_rows_kernel<<<cdiv(rows * 64, 256), 256, 0, st>>>(dY, 64, Ho * Wo, rows, q.dyt);
    DYN_LAUNCH_CHECK();
    enc_im2col_kernel<<<cdiv(rows * K, 256), 256, 0, st>>>(X, Cin, H, W, Ho, Wo, k, stride, pad, rows, q.col, 0);
    DYN_LAUNCH_CHECK();
    for (int c0 = 0; c0 < K; c0 += 256) {  // dW[64, K] += dYt^T col
      const int wd = K - c0 < 256 ? K - c0 : 256;
      int rc;
      if (tc && tc_grad_w_ok(64, wd, rows)) {
        rc = tc_grad_w(q.dyt, 64, 64, rows, q.col + c0, K, wd, nullptr, dW + c0, K, st);
      } else {
        GemmArgs g{q.dyt, q.col + c0, dW + c0, 64, wd, rows, 1, 64, K, 1, K, 1, 0};
        rc = launch_gemm(g, true, st);
      }
      if (rc) return rc;
    }
    if (dX == nullptr) return DYN_OK;
    for (int c0 = 0; c0 < K; c0 += 256) {  // dcol[rows, K] = dYt W  (overwrites col)
      const int wd = K - c0 < 256 ? K - c0 : 256;
      int rc;
      if (tc && tc_grad_in_ok(64, wd, rows)) {
        rc = tc_grad_in(q.dyt, 64, 64, rows, Wt + c0, K, wd, q.col + c0, K, q.img, st);
      } else {
        GemmArgs g{q.dyt, Wt + c0, q.col + c0, rows, wd, 64, 64, 1, K, 1, K, 0, 0};
        rc = launch_gemm(g, false, st);
      }
      if (rc) return rc;
    }
    if (zero_dx) DYN_CUDA(cudaMemsetAsync(dX, 0, (size_t)N * Cin * H * W * sizeof(float), st));
    enc_im2col_kernel<<<cdiv(rows * K, 256), 256, 0, st>>>(dX, Cin, H, W, Ho, Wo, k, stride, pad, rows, q.col, 1);
    DYN_LAUNCH_CHECK();
    return DYN_OK;
  }
};

}  // namespace
}  // namespace dyn

using namespace dyn;

extern "C" {

size_t dyn_encoder_param_count(void) { return (size_t)enc_layout().total; }

// workspace: 64-channel maps at half resolution (1) and at quarter resolution (4) + statistics
size_t dyn_encoder_workspace_bytes(int N, int H, int W) {
  const long long H2 = (H + 6 - 7) / 2 + 1, W2 = (W + 6 - 7) / 2 + 1;
  const long long H4 = (H2 + 2 - 3) / 2 + 1, W4 = (W2 + 2 - 3) / 2 + 1;
  return (size_t)(((long long)N * 64 * H2 * W2 + 4LL * N * 64 * H4 * W4 + 2LL * N * 64) * sizeof(float) + 1024);
}

int dyn_encoder_forward(const float* params, size_t n_params, const float* images, int N, int H, int W,
                        float* coarse, float* fine, void* workspace, size_t workspace_bytes, void* stream) {
  const EncLayout L = enc_layout();
  DYN_CHECK_ARG(params && images && coarse && fine && workspace && N >= 1 && H >= 8 && W >= 8);
  if (n_params != (size_t)L.total)
    return fail(DYN_E_INVALID, "encoder: got %zu parameters, expected %d", n_params, L.total);
  if (workspace_bytes < dyn_encoder_workspace_bytes(N, H, W))
    return fail(DYN_E_WORKSPACE, "encoder: workspace %zu < %zu", workspace_bytes, dyn_encoder_workspace_bytes(N, H, W));
  cudaStream_t st = (cudaStream_t)stream;
  const int H2 = (H + 6 - 7) / 2 + 1, W2 = (W + 6 - 7) / 2 + 1;
  const int H4 = (H2 + 2 - 3) / 2 + 1, W4 = (W2 + 2 - 3) / 2 + 1;
  float* a2 = reinterpret_cast<float*>(workspace);          // [N,64,H2,W2]
  const long long n4 = (long long)N * 64 * H4 * W4;
  float* b0 = a2 + (long long)N * 64 * H2 * W2;               // [N,64,H4,W4] x 4
  float *b1 = b0 + n4, *b2 = b1 + n4, *b3 = b2 + n4;
  float* stats = b3 + n4;
  const float* P = params;
  // stem (feature_network.py:303)
  enc_conv7_kernel<<<dim3(cdiv(W2, 16), cdiv(H2, 8), N), 128, 0, st>>>(images, P + L.conv1, H, W, H2, W2, a2);
  DYN_LAUNCH_CHECK();
  int rc = in_norm(a2, P, L.bn1w, L.bn1b, nullptr, 1, N, H2 * W2, stats, a2, st);
  if (rc) return rc;
  // layer1.0: stride 2, shortcut = IN(conv1x1 stride 2)
  const dim3 g4(cdiv(W4, 16), cdiv(H4, 8), N);
  enc_conv3_kernel<2><<<g4, 128, 0, st>>>(a2, P + L.blk[0].c1, H2, W2, H4, W4, b0);
  DYN_LAUNCH_CHECK();
  if ((rc = in_norm(b0, P, L.blk[0].b1w, L.blk[0].b1b, nullptr, 1, N, H4 * W4, stats, b0, st))) return rc;
  enc_conv3_kernel<1><<<g4, 128, 0, st>>>(b0, P + L.blk[0].c2, H4, W4, H4, W4, b1);
  DYN_LAUNCH_CHECK();
  enc_conv1_kernel<2><<<cdiv((long long)N * H4 * W4 * 4, 256), 256, 0, st>>>(a2, P + L.blk[0].dsw, nullptr, H2, W2, H4,
                                                                               W4, N, b2);
  DYN_LAUNCH_CHECK();
  if ((rc = in_norm(b2, P, L.blk[0].dsbw, L.blk[0].dsbb, nullptr, 0, N, H4 * W4, stats, b2, st))) return rc;
  if ((rc = in_norm(b1, P, L.blk[0].b2w, L.blk[0].b2b, b2, 1, N, H4 * W4, stats, b1, st))) return rc;
  // layer1.1, layer1.2: identity shortcuts (x in `cur`)
  float *cur = b1, *t0 = b0, *t1 = b2;
  for (int b = 1; b < 3; ++b) {
    enc_conv3_kernel<1><<<g4, 128, 0, st>>>(cur, P + L.blk[b].c1, H4, W4, H4, W4, t0);
    DYN_LAUNCH_CHECK();
    if ((rc = in_norm(t0, P, L.blk[b].b1w, L.blk[b].b1b, nullptr, 1, N, H4 * W4, stats, t0, st))) return rc;
    enc_conv3_kernel<1><<<g4, 128, 0, st>>>(t0, P + L.blk[b].c2, H4, W4, H4, W4, t1);
    DYN_LAUNCH_CHECK();
    if ((rc = in_norm(t1, P, L.blk[b].b2w, L.blk[b].b2b, cur, 1, N, H4 * W4, stats, t1, st))) return rc;
    float* tmp = cur; cur = t1; t1 = tmp;
  }
  // out_conv (1x1, bias) -> coarse | fine (feature_network.py:306-309)
  enc_conv1_kernel<1><<<cdiv((long long)N * H4 * W4 * 4, 256), 256, 0, st>>>(cur, P + L.outw, P + L.outb, H4, W4, H4, W4,
                                                                               N, b3);
  DYN_LAUNCH_CHECK();
  const size_t plane = (size_t)H4 * W4 * sizeof(float);
  DYN_CUDA(cudaMemcpy2DAsync(coarse, 32 * plane, b3, 64 * plane, 32 * plane, N, cudaMemcpyDeviceToDevice, st));
  DYN_CUDA(cudaMemcpy2DAsync(fine, 32 * plane, reinterpret_cast<char*>(b3) + 32 * plane, 64 * plane, 32 * plane, N,
                             cudaMemcpyDeviceToDevice, st));
  return DYN_OK;
}

// ---- training (row f2) -------------------------------------------------------------------------
static void enc_dims(int H, int W, int* H2, int* W2, int* H4, int* W4) {
  *H2 = (H + 6 - 7) / 2 + 1; *W2 = (W + 6 - 7) / 2 + 1;
  *H4 = (*H2 + 2 - 3) / 2 + 1; *W4 = (*W2 + 2 - 3) / 2 + 1;
}

size_t dyn_encoder_train_workspace_bytes(int N, int H, int W) {
  int H2, W2, H4, W4;
  enc_dims(H, W, &H2, &W2, &H4, &W4);
  EncSaved s;
  return enc_saved_alloc(nullptr, N, H2, W2, H4, W4, &s) + (size_t)N * 64 * H4 * W4 * sizeof(float) + 256;
}

size_t dyn_encoder_backward_scratch_bytes(int N, int H, int W) {
  int H2, W2, H4, W4;
  enc_dims(H, W, &H2, &W2, &H4, &W4);
  EncScratch q;
  return enc_scratch_alloc(nullptr, N, H, W, H2, W2, H4, W4, &q);
}

int dyn_encoder_train_forward(const float* params, size_t n_params, const float* images, int N, int H, int W,
                              float* coarse, float* fine, void* saved, size_t saved_bytes, void* stream) {
  const EncLayout L = enc_layout();
  DYN_CHECK_ARG(params && images && coarse && fine && saved && N >= 1 && H >= 8 && W >= 8);
  if (n_params != (size_t)L.total)
    return fail(DYN_E_INVALID, "encoder: got %zu parameters, expected %d", n_params, L.total);
  if (saved_bytes < dyn_encoder_train_workspace_bytes(N, H, W))
    return fail(DYN_E_WORKSPACE, "encoder: saved workspace %zu < %zu", saved_bytes, dyn_encoder_train_workspace_bytes(N, H, W));
  cudaStream_t st = (cudaStream_t)stream;
  int H2, W2, H4, W4;
  enc_dims(H, W, &H2, &W2, &H4, &W4);
  EncSaved s;
  const size_t used = enc_saved_alloc((char*)saved, N, H2, W2, H4, W4, &s);
  float* outb = reinterpret_cast<float*>((char*)saved + ((used + 255) & ~(size_t)255));  // out_conv result [N,64,h,w]
  const float* P = params;
  int rc;
  enc_conv7_kernel<<<dim3(cdiv(W2, 16), cdiv(H2, 8), N), 128, 0, st>>>(images, P + L.conv1, H, W, H2, W2, s.c1);
  DYN_LAUNCH_CHECK();
  if ((rc = in_norm(s.c1, P, L.bn1w, L.bn1b, nullptr, 1, N, H2 * W2, s.stats[0], s.a1, st))) return rc;
  const dim3 g4(cdiv(W4, 16), cdiv(H4, 8), N);
  const float* xin = s.a1;
  for (int b = 0; b < 3; ++b) {
    if (b == 0) enc_conv3_kernel<2><<<g4, 128, 0, st>>>(xin, P + L.blk[0].c1, H2, W2, H4, W4, s.b[0].cA);
    else enc_conv3_kernel<1><<<g4, 128, 0, st>>>(xin, P + L.blk[b].c1, H4, W4, H4, W4, s.b[b].cA);
    DYN_LAUNCH_CHECK();
    if ((rc = in_norm(s.b[b].cA, P, L.blk[b].b1w, L.blk[b].b1b, nullptr, 1, N, H4 * W4,
                      s.stats[b == 0 ? 1 : 2 * b + 2], s.b[b].aA, st))) return rc;
    enc_conv3_kernel<1><<<g4, 128, 0, st>>>(s.b[b].aA, P + L.blk[b].c2, H4, W4, H4, W4, s.b[b].cB);
    DYN_LAUNCH_CHECK();
    const float* resid = xin;
    if (b == 0) {
      enc_conv1_kernel<2><<<cdiv((long long)N * H4 * W4 * 4, 256), 256, 0, st>>>(s.a1, P + L.blk[0].dsw, nullptr, H2, W2,
                                                                                   H4, W4, N, s.cds);
      DYN_LAUNCH_CHECK();
      // the normalised shortcut lives in block 0's output buffer until the sum replaces it
      if ((rc = in_norm(s.cds, P, L.blk[0].dsbw, L.blk[0].dsbb, nullptr, 0, N, H4 * W4, s.stats[3], s.b[0].o, st))) return rc;
      resid = s.b[0].o;
    }
    if ((rc = in_norm(s.b[b].cB, P, L.blk[b].b2w, L.blk[b].b2b, resid, 1, N, H4 * W4,
                      s.stats[b == 0 ? 2 : 2 * b + 3], s.b[b].o, st))) return rc;
    xin = s.b[b].o;
  }
  enc_conv1_kernel<1><<<cdiv((long long)N * H4 * W4 * 4, 256), 256, 0, st>>>(xin, P + L.outw, P + L.outb, H4, W4, H4, W4,
                                                                               N, outb);
  DYN_LAUNCH_CHECK();
  const size_t plane = (size_t)H4 * W4 * sizeof(float);
  DYN_CUDA(cudaMemcpy2DAsync(coarse, 32 * plane, outb, 64 * plane, 32 * plane, N, cudaMemcpyDeviceToDevice, st));
  DYN_CUDA(cudaMemcpy2DAsync(fine, 32 * plane, reinterpret_cast<char*>(outb) + 32 * plane, 64 * plane, 32 * plane, N,
                             cudaMemcpyDeviceToDevice, st));
  return DYN_OK;
}

int dyn_encoder_backward(const float* params, size_t n_params, const float* images, int N, int H, int W,
                         const float* d_coarse, const float* d_fine, void* saved, size_t saved_bytes, void* scratch,
                         size_t scratch_bytes, float* d_params, int precision, void* stream) {
  const EncLayout L = enc_layout();
  DYN_CHECK_ARG(params && images && saved && scratch && d_params && (d_coarse || d_fine) && N >= 1);
  DYN_CHECK_ARG(precision == DYN_PREC_FP32 || precision == DYN_PREC_BF16);
  if (n_params != (size_t)L.total)
    return fail(DYN_E_INVALID, "encoder: got %zu parameters, expected %d", n_params, L.total);
  if (saved_bytes < dyn_encoder_train_workspace_bytes(N, H, W) || scratch_bytes < dyn_encoder_backward_scratch_bytes(N, H, W))
    return fail(DYN_E_WORKSPACE, "encoder backward: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  int H2, W2, H4, W4;
  enc_dims(H, W, &H2, &W2, &H4, &W4);
  EncSaved s;
  enc_saved_alloc((char*)saved, N, H2, W2, H4, W4, &s);
  EncScratch q;
  enc_scratch_alloc((char*)scratch, N, H, W, H2, W2, H4, W4, &q);
  const float* P = params;
  float* dP = d_params;
  const int hw4 = H4 * W4, hw2 = H2 * W2;
  const long long n4 = (long long)N * 64 * hw4, n2 = (long long)N * 64 * hw2;
  const size_t plane = (size_t)hw4 * sizeof(float);
  const ConvBwd cb{st, precision == DYN_PREC_BF16, q, N};
  int rc;
  auto in_bwd = [&](const float* x, float* g, const float* stats, int gw, int gb, int hw) {
    enc_in_bwd_kernel<<<N * 64, 256, 0, st>>>(x, g, stats, stats + N * 64, P + gw, hw, 64, g, dP + gw, dP + gb);
    DYN_LAUNCH_CHECK();
    return DYN_OK;
  };
  auto relu_mask = [&](float* g, const float* y, long long n) {
    enc_relu_mask_kernel<<<cdiv(n, 256), 256, 0, st>>>(g, y, n);
    DYN_LAUNCH_CHECK();
    return DYN_OK;
  };
  // d(out_conv output) [N,64,h,w] = [d_coarse | d_fine]
  float* g = q.g4a;
  DYN_CUDA(cudaMemsetAsync(g, 0, (size_t)n4 * sizeof(float), st));
  if (d_coarse) DYN_CUDA(cudaMemcpy2DAsync(g, 64 * plane, d_coarse, 32 * plane, 32 * plane, N, cudaMemcpyDeviceToDevice, st));
  if (d_fine) DYN_CUDA(cudaMemcpy2DAsync(reinterpret_cast<char*>(g) + 32 * plane, 64 * plane, d_fine, 32 * plane, 32 * plane, N,
                                         cudaMemcpyDeviceToDevice, st));
  // out_conv (1x1, bias): db = sum over pixels; dW, d(o2)
  float* d_o = q.g4b;
  if ((rc = cb.run(g, H4, W4, P + L.outw, dP + L.outw, s.b[2].o, 64, H4, W4, 1, 1, 0, d_o, true))) return rc;
  if ((rc = launch_colsum(q.dyt, 64, 64, (long long)N * hw4, dP + L.outb, st))) return rc;  // q.dyt = rows of g
  // blocks 2, 1 (identity shortcuts), then block 0
  float* t = q.g4a;   // free again
  float* u = q.g4c;
  for (int b = 2; b >= 1; --b) {
    float* xin = s.b[b - 1].o;
    if ((rc = relu_mask(d_o, s.b[b].o, n4))) return rc;                       // d_sum in d_o
    DYN_CUDA(cudaMemcpyAsync(t, d_o, (size_t)n4 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    if ((rc = in_bwd(s.b[b].cB, t, s.stats[2 * b + 3], L.blk[b].b2w, L.blk[b].b2b, hw4))) return rc;   // d cB
    if ((rc = cb.run(t, H4, W4, P + L.blk[b].c2, dP + L.blk[b].c2, s.b[b].aA, 64, H4, W4, 3, 1, 1, u, true))) return rc;
    if ((rc = relu_mask(u, s.b[b].aA, n4))) return rc;
    if ((rc = in_bwd(s.b[b].cA, u, s.stats[2 * b + 2], L.blk[b].b1w, L.blk[b].b1b, hw4))) return rc;   // d cA
    // d xin = d_sum (identity shortcut, already in d_o) + conv1 backward, accumulated in place
    if ((rc = cb.run(u, H4, W4, P + L.blk[b].c1, dP + L.blk[b].c1, xin, 64, H4, W4, 3, 1, 1, d_o, false))) return rc;
  }
  // block 0: stride 2, shortcut = IN(conv1x1 stride 2)
  if ((rc = relu_mask(d_o, s.b[0].o, n4))) return rc;
  DYN_CUDA(cudaMemcpyAsync(t, d_o, (size_t)n4 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if ((rc = in_bwd(s.b[0].cB, t, s.stats[2], L.blk[0].b2w, L.blk[0].b2b, hw4))) return rc;
  if ((rc = cb.run(t, H4, W4, P + L.blk[0].c2, dP + L.blk[0].c2, s.b[0].aA, 64, H4, W4, 3, 1, 1, u, true))) return rc;
  if ((rc = relu_mask(u, s.b[0].aA, n4))) return rc;
  if ((rc = in_bwd(s.b[0].cA, u, s.stats[1], L.blk[0].b1w, L.blk[0].b1b, hw4))) return rc;
  float* d_a1 = q.g2a;
  if ((rc = cb.run(u, H4, W4, P + L.blk[0].c1, dP + L.blk[0].c1, s.a1, 64, H2, W2, 3, 2, 1, d_a1, true))) return rc;
  if ((rc = in_bwd(s.cds, d_o, s.stats[3], L.blk[0].dsbw, L.blk[0].dsbb, hw4))) return rc;           // d cds (in d_o)
  if ((rc = cb.run(d_o, H4, W4, P + L.blk[0].dsw, dP + L.blk[0].dsw, s.a1, 64, H2, W2, 1, 2, 0, d_a1, false))) return rc;
  // stem: relu, InstanceNorm, conv1 (only its weight gradient: the images carry none)
  if ((rc = relu_mask(d_a1, s.a1, n2))) return rc;
  if ((rc = in_bwd(s.c1, d_a1, s.stats[0], L.bn1w, L.bn1b, hw2))) return rc;
  return cb.run(d_a1, H2, W2, P + L.conv1, dP + L.conv1, const_cast<float*>(images), 3, H, W, 7, 2, 3, nullptr, false);
}

}  // extern "C"
