// Masked PSNR and SSIM of rendered views (eval_nvidia.py: calculate_psnr:201, calculate_ssim:228, the per-camera
// scoring block :380-457), with skimage 0.19.3 structural_similarity(multichannel=True, full=True) restated on the
// device.  DESIGN §3.6 gives the semantics and the reference lines.
//
//   dyn_image_scores_workspace_bytes   per-CTA partial sums of K images
//   dyn_image_scores                   scores [K, M, 2] = (PSNR, SSIM) per image and mask row, on the device
//
// Two launches, no float atomics, no host synchronisation.  ssim_tile_kernel writes one row of fp64 partial sums per
// output tile; scores_finish_kernel adds an image's rows in a fixed order.  The same inputs give the same bits, and an
// image's scores do not depend on K or on the other images of the call.
#include "common.cuh"

namespace dyn {
namespace {

constexpr int kTileW = 32, kTileH = 16, kHalo = 3, kWin = 2 * kHalo + 1;
constexpr int kInW = kTileW + 2 * kHalo, kInH = kTileH + 2 * kHalo;
constexpr int kThreads = 256, kWarps = kThreads / 32;
constexpr int kMaxRows = 3, kSums = 3 * kMaxRows;  // per mask row m: sum S w_m, sum w_m, sum (x - y)^2 w_m

// skimage 0.19.3: cov_norm = NP / (NP - 1), C1 = (K1 R)^2, C2 = (K2 R)^2 with R = 2 (dtype_range[float32] = (-1, 1)).
// Python floats meeting float32 arrays, so numpy rounds them to float32.
constexpr float kCov = (float)(49.0 / 48.0);
constexpr float kC1 = (float)((0.01 * 2.0) * (0.01 * 2.0));
constexpr float kC2 = (float)((0.03 * 2.0) * (0.03 * 2.0));
constexpr double kCountEps = 1e-8;  // np.sum(mask) + 1e-8

// scipy.ndimage mode 'reflect' (d c b a | a b c d); the clamp only keeps the unused rows / columns of a partial tile in
// bounds
__device__ __forceinline__ int reflect(int i, int n) {
  if (i < 0) i = -i - 1;
  if (i >= n) i = 2 * n - 1 - i;
  return min(max(i, 0), n - 1);
}

// One CTA per kTileW x kTileH output tile of image blockIdx.z, all 3 channels.  The tile plus a 3-pixel reflected halo
// is staged in shared memory (EVAL: both images times the valid mask of the prediction); per channel a vertical then a
// horizontal 7-tap pass gives the 5 moments, each pass a direct fp64 sum / 7 rounded to float32 as scipy's
// uniform_filter1d stores it; S follows skimage's float32 expression order.  Partial sums per mask row go to
// partial[(blockIdx.z * tiles + tile) * kSums + j].
//   plain: row 0 weighted by mask (1 when mask is NULL), on the given images.
//   EVAL:  rows valid, mask, 1 - mask (eval_nvidia.py:395-448), on the masked images; one S map for all rows.
template <bool EVAL>
__global__ void __launch_bounds__(kThreads) ssim_tile_kernel(const float* __restrict__ pred,
                                                             const float* __restrict__ gt,
                                                             const float* __restrict__ mask, int H, int W,
                                                             float* __restrict__ smap, double* __restrict__ partial) {
  __shared__ float xs[3][kInH * kInW], ys[3][kInH * kInW];
  __shared__ float vert[5][kTileH * kInW];
  __shared__ double red[kWarps][kSums];
  const int x0 = blockIdx.x * kTileW, y0 = blockIdx.y * kTileH;
  const size_t img = (size_t)blockIdx.z * H * W * 3;
  const float* P = pred + img;
  const float* G = gt + img;
  for (int i = threadIdx.x; i < kInH * kInW; i += kThreads) {
    const int gy = reflect(y0 + i / kInW - kHalo, H), gx = reflect(x0 + i % kInW - kHalo, W);
    const size_t o = ((size_t)gy * W + gx) * 3;
    float a[3] = {P[o], P[o + 1], P[o + 2]}, b[3] = {G[o], G[o + 1], G[o + 2]};
    if (EVAL) {
      const float v = valid_pixel(a[0], a[1], a[2]) ? 1.f : 0.f;
#pragma unroll
      for (int c = 0; c < 3; ++c) a[c] = __fmul_rn(a[c], v), b[c] = __fmul_rn(b[c], v);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) xs[c][i] = a[c], ys[c][i] = b[c];
  }
  __syncthreads();

  double acc[kSums];
#pragma unroll
  for (int j = 0; j < kSums; ++j) acc[j] = 0.0;
  for (int ch = 0; ch < 3; ++ch) {
    const float* X = xs[ch];
    const float* Y = ys[ch];
    for (int i = threadIdx.x; i < kTileH * kInW; i += kThreads) {
      const int r = i / kInW, c = i % kInW;
      double s[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
      for (int t = 0; t < kWin; ++t) {
        const float x = X[(r + t) * kInW + c], y = Y[(r + t) * kInW + c];
        s[0] += x;
        s[1] += y;
        s[2] += __fmul_rn(x, x);
        s[3] += __fmul_rn(y, y);
        s[4] += __fmul_rn(x, y);
      }
#pragma unroll
      for (int m = 0; m < 5; ++m) vert[m][i] = __double2float_rn(__ddiv_rn(s[m], (double)kWin));
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kTileH * kTileW; i += kThreads) {
      const int r = i / kTileW, c = i % kTileW;
      float u[5];
#pragma unroll
      for (int m = 0; m < 5; ++m) {
        double s = 0.0;
#pragma unroll
        for (int t = 0; t < kWin; ++t) s += vert[m][r * kInW + c + t];
        u[m] = __double2float_rn(__ddiv_rn(s, (double)kWin));
      }
      const float ux = u[0], uy = u[1];
      const float vx = __fmul_rn(kCov, __fsub_rn(u[2], __fmul_rn(ux, ux)));
      const float vy = __fmul_rn(kCov, __fsub_rn(u[3], __fmul_rn(uy, uy)));
      const float vxy = __fmul_rn(kCov, __fsub_rn(u[4], __fmul_rn(ux, uy)));
      const float A1 = __fadd_rn(__fmul_rn(__fmul_rn(2.f, ux), uy), kC1);
      const float A2 = __fadd_rn(__fmul_rn(2.f, vxy), kC2);
      const float B1 = __fadd_rn(__fadd_rn(__fmul_rn(ux, ux), __fmul_rn(uy, uy)), kC1);
      const float B2 = __fadd_rn(__fadd_rn(vx, vy), kC2);
      const float S = __fdiv_rn(__fmul_rn(A1, A2), __fmul_rn(B1, B2));
      const int gy = y0 + r, gx = x0 + c;
      if (gy >= H || gx >= W) continue;
      const size_t o = img + ((size_t)gy * W + gx) * 3 + ch;
      if (smap) smap[o] = S;
      const int ci = (r + kHalo) * kInW + c + kHalo;
      const double d = (double)X[ci] - (double)Y[ci];
      const double d2 = d * d, s = (double)S;
      float w[kMaxRows];
      if (EVAL) {
        w[0] = valid_pixel(xs[0][ci], xs[1][ci], xs[2][ci]) ? 1.f : 0.f;  // masked == raw where valid
        w[1] = mask ? mask[o] : 0.f;
        w[2] = mask ? __fsub_rn(1.f, w[1]) : 0.f;
      } else {
        w[0] = mask ? mask[o] : 1.f;
        w[1] = w[2] = 0.f;
      }
#pragma unroll
      for (int m = 0; m < kMaxRows; ++m) {
        const double wm = (double)w[m];
        acc[3 * m] += s * wm;
        acc[3 * m + 1] += wm;
        acc[3 * m + 2] += d2 * wm;
      }
    }
    __syncthreads();
  }

  block_sum<kSums, kWarps>(acc, red);
  if (threadIdx.x == 0) {
    const size_t tile = ((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
#pragma unroll
    for (int j = 0; j < kSums; ++j) partial[tile * kSums + j] = acc[j];
  }
}

// One block per image: its tiles' partial rows summed in a fixed order (thread t takes tiles t, t + kThreads, ...,
// then the CTA tree), then per mask row m: den = sum w + 1e-8, mse = sum d^2 w / den, PSNR = mse == 0 ? 0 :
// 10 log10(1 / mse), SSIM = sum S w / den (eval_nvidia.py:218-225, :245-247).
__global__ void __launch_bounds__(kThreads) scores_finish_kernel(const double* __restrict__ partial, int tiles, int M,
                                                                 double* __restrict__ scores) {
  __shared__ double red[kWarps][kSums];
  const double* p = partial + (size_t)blockIdx.x * tiles * kSums;
  double acc[kSums];
#pragma unroll
  for (int j = 0; j < kSums; ++j) acc[j] = 0.0;
  for (int t = threadIdx.x; t < tiles; t += kThreads)
#pragma unroll
    for (int j = 0; j < kSums; ++j) acc[j] += p[(size_t)t * kSums + j];
  block_sum<kSums, kWarps>(acc, red);
  if (threadIdx.x != 0) return;
  double* out = scores + (size_t)blockIdx.x * M * 2;
#pragma unroll
  for (int m = 0; m < kMaxRows; ++m) {
    if (m >= M) break;
    const double den = acc[3 * m + 1] + kCountEps;
    const double mse = acc[3 * m + 2] / den;
    out[2 * m] = mse == 0.0 ? 0.0 : 10.0 * log10(1.0 / mse);
    out[2 * m + 1] = acc[3 * m] / den;
  }
}

bool scores_shape_ok(long long K, long long H, long long W) {
  // skimage: win_size 7 may not exceed the image; images are grid.z
  return K >= 1 && K < 65536 && H >= kWin && W >= kWin && H * W < (1ll << 31);
}

size_t scores_ws_bytes(int K, int H, int W) {
  return (size_t)K * cdiv(W, kTileW) * cdiv(H, kTileH) * kSums * sizeof(double);
}

}  // namespace
}  // namespace dyn

using namespace dyn;

extern "C" {

size_t dyn_image_scores_workspace_bytes(int K, int H, int W) {
  return scores_shape_ok(K, H, W) ? scores_ws_bytes(K, H, W) : 0;
}

int dyn_image_scores(const float* pred, const float* gt, const float* mask, int K, int H, int W, int mode,
                     double* scores, float* ssim_map, void* workspace, size_t workspace_bytes, void* stream) {
  DYN_CHECK_ARG(pred && gt && scores && scores_shape_ok(K, H, W));
  DYN_CHECK_ARG(mode == DYN_SCORES_PLAIN || mode == DYN_SCORES_EVAL);
  const size_t need = scores_ws_bytes(K, H, W);
  if (workspace == nullptr || workspace_bytes < need)
    return fail(DYN_E_WORKSPACE, "image_scores: workspace of %zu bytes, %zu needed", workspace_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  double* partial = (double*)workspace;
  const dim3 grid(cdiv(W, kTileW), cdiv(H, kTileH), K);
  int M = 1;
  if (mode == DYN_SCORES_EVAL) {
    M = mask ? 3 : 1;
    ssim_tile_kernel<true><<<grid, kThreads, 0, st>>>(pred, gt, mask, H, W, ssim_map, partial);
  } else {
    ssim_tile_kernel<false><<<grid, kThreads, 0, st>>>(pred, gt, mask, H, W, ssim_map, partial);
  }
  DYN_LAUNCH_CHECK();
  scores_finish_kernel<<<K, kThreads, 0, st>>>(partial, (int)(grid.x * grid.y), M, scores);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

}  // extern "C"
