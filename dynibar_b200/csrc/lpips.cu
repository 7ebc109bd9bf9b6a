// LPIPS v0.1 'alex' of rendered views (eval_nvidia.py:289-291, :402-452), fp32 FFMA products with fp32 accumulation
// (no TF32) and fp64 masked sums.  DESIGN §3.6 gives the definition, the mask rule and the measurements.
//
//   dyn_lpips_param_count       the weight blob's length in floats
//   dyn_lpips_workspace_bytes   the network's activations and the score's partial sums for K cameras of H x W
//   dyn_lpips                   scores [K, M] per camera and mask row, on the device
//
// Launches of one call, each over all 2K images (pred 0..K-1, gt K..2K-1) or all K cameras:
//   lpips_prep_kernel      valid mask, masking, 2x - 1 and the ScalingLayer; channels-last in, [2K, 3, H, W] out, and
//                          the per-pixel weight of every mask row [K, M, H, W]
//   lpips_conv_kernel      the five convolutions as implicit GEMMs with a bias + ReLU epilogue (one launch each)
//   lpips_pool_kernel      the two 3 / 2 max pools
//   lpips_tap_kernel       per tap: unit-normalised channel vectors, squared difference, lin dot product -> d_l
//   lpips_reduce_kernel    per (camera, tile of d_l pixels): the area-pooled mask rows on the fly, fp64 partial sums
//   lpips_finish_kernel    per camera: the tiles of each tap in a fixed order, sum_l (sum m_l d_l / sum m_l)
// No float atomics, no host synchronisation: the same inputs give the same bits, and a camera's scores do not depend
// on K or on the other cameras.
#include "common.cuh"

namespace dyn {
namespace {

constexpr int kTaps = 5, kMaxRows = 3, kSums = 2 * kMaxRows;  // per row m: sum m_l d_l, sum m_l
constexpr int kMinSide = 31;  // the smallest side whose second max pool still has an output (DESIGN §3.6)
// torchvision alexnet().features: conv l maps kCin[l] -> kCout[l] channels with a kKs[l]^2 kernel
constexpr int kCin[kTaps] = {3, 64, 192, 384, 256};
constexpr int kCout[kTaps] = {64, 192, 384, 256, 256};
constexpr int kKs[kTaps] = {11, 5, 3, 3, 3};
// LPIPS v0.1 ScalingLayer (float32 buffers)
__constant__ float kShift[3] = {-.030f, -.088f, -.188f};
__constant__ float kScale[3] = {.458f, .448f, .450f};
constexpr float kNormEps = 1e-10f;  // lpips normalize_tensor: x / (sqrt(sum x^2) + eps)

// ---- shapes ------------------------------------------------------------------------------------------------------

struct Geom {
  int K, H, W, M;
  int h1, w1, h2, w2, h3, w3;  // conv1 (tap 1), pool1 = conv2 (tap 2), pool2 = conv3..5 (taps 3-5)
  int th[kTaps], tw[kTaps];    // tap sizes
  int doff[kTaps + 1];         // offset of tap l in a camera's row of d, doff[kTaps] = its length
  int tile0[kTaps + 1];        // first reduce tile of tap l, tile0[kTaps] = tiles per camera
};

constexpr int kRedThreads = 256, kRedWarps = kRedThreads / 32;

inline int pool_out(int n) { return (n - 3) / 2 + 1; }  // max pool 3 / 2, floor mode, n >= 3

Geom geom(int K, int H, int W, int M) {
  Geom g;
  g.K = K, g.H = H, g.W = W, g.M = M;
  g.h1 = (H + 4 - 11) / 4 + 1, g.w1 = (W + 4 - 11) / 4 + 1;
  g.h2 = pool_out(g.h1), g.w2 = pool_out(g.w1);
  g.h3 = pool_out(g.h2), g.w3 = pool_out(g.w2);
  const int th[kTaps] = {g.h1, g.h2, g.h3, g.h3, g.h3}, tw[kTaps] = {g.w1, g.w2, g.w3, g.w3, g.w3};
  g.doff[0] = g.tile0[0] = 0;
  for (int l = 0; l < kTaps; ++l) {
    g.th[l] = th[l], g.tw[l] = tw[l];
    g.doff[l + 1] = g.doff[l] + th[l] * tw[l];
    g.tile0[l + 1] = g.tile0[l] + cdiv(th[l] * tw[l], kRedThreads);
  }
  return g;
}

bool lpips_shape_ok(long long K, long long H, long long W) {
  return K >= 1 && K <= 65535 && H >= kMinSide && W >= kMinSide && K * H * W <= (1ll << 28);
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// workspace carve-up, in order; every part 256-byte aligned
struct Carve {
  float *x0, *a1, *p1, *a2, *p2, *a3, *a4, *a5, *d, *rw;
  double* partial;
  size_t bytes;
};

Carve carve(const Geom& g, char* base) {
  const size_t n = 2 * (size_t)g.K, hw1 = (size_t)g.h1 * g.w1, hw2 = (size_t)g.h2 * g.w2, hw3 = (size_t)g.h3 * g.w3;
  const size_t sizes[11] = {n * 3 * g.H * g.W * 4, n * 64 * hw1 * 4, n * 64 * hw2 * 4, n * 192 * hw2 * 4,
                            n * 192 * hw3 * 4,     n * 384 * hw3 * 4, n * 256 * hw3 * 4, n * 256 * hw3 * 4,
                            (size_t)g.K * g.doff[kTaps] * 4, (size_t)g.K * kMaxRows * g.H * g.W * 4,
                            (size_t)g.K * g.tile0[kTaps] * kSums * sizeof(double)};
  void* ptrs[11];
  size_t off = 0;
  for (int i = 0; i < 11; ++i) {
    ptrs[i] = base ? base + off : nullptr;
    off += align256(sizes[i]);
  }
  Carve c;
  c.x0 = (float*)ptrs[0], c.a1 = (float*)ptrs[1], c.p1 = (float*)ptrs[2], c.a2 = (float*)ptrs[3];
  c.p2 = (float*)ptrs[4], c.a3 = (float*)ptrs[5], c.a4 = (float*)ptrs[6], c.a5 = (float*)ptrs[7];
  c.d = (float*)ptrs[8], c.rw = (float*)ptrs[9], c.partial = (double*)ptrs[10];
  c.bytes = off;
  return c;
}

// offsets (floats) of the weight blob: conv l weight [kCout, kCin, k, k] then its bias, l = 0..4; then lin l [kCout]
struct Offsets {
  size_t w[kTaps], b[kTaps], lin[kTaps], total;
};

Offsets offsets() {
  Offsets o;
  size_t off = 0;
  for (int l = 0; l < kTaps; ++l) {
    o.w[l] = off, off += (size_t)kCout[l] * kCin[l] * kKs[l] * kKs[l];
    o.b[l] = off, off += kCout[l];
  }
  for (int l = 0; l < kTaps; ++l) o.lin[l] = off, off += kCout[l];
  o.total = off;
  return o;
}

// ---- kernels -----------------------------------------------------------------------------------------------------

// One thread per pixel of camera k: x0[k] = scaled pred, x0[K + k] = scaled gt ([2K, 3, H, W]); rw[k, m] = the
// weight of mask row m at the pixel: the sum of the row's three channels ((c0 + c1) + c2), which area pooling and the
// row's normalisation turn into the pooled 3-channel mask broadcast over d_l.  The valid row is eval_nvidia.py's valid
// mask tiled over 3 channels, and an absent mask is 1 in each of them: both weigh 3.
//   EVAL:  valid = ((r + g) + b of pred) > 1e-3; x = 2 (img * valid) - 1; rows valid, mask, 1 - mask (M = 3)
//          or valid alone (M = 1).
//   PLAIN: x = img (already in [-1, 1]); row 0 = mask, all ones where mask is NULL.
// Then (x - shift) / scale per channel, float32 as the ScalingLayer computes it.
template <bool EVAL>
__global__ void __launch_bounds__(256) lpips_prep_kernel(const float* __restrict__ pred, const float* __restrict__ gt,
                                                          const float* __restrict__ mask, int K, int HW, int M,
                                                          float* __restrict__ x0, float* __restrict__ rw) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)K * HW) return;
  const int k = (int)(i / HW), p = (int)(i - (long long)k * HW);
  float a[3] = {pred[3 * i], pred[3 * i + 1], pred[3 * i + 2]}, b[3] = {gt[3 * i], gt[3 * i + 1], gt[3 * i + 2]};
  float v = 1.f;
  if (EVAL) {
    v = valid_pixel(a[0], a[1], a[2]) ? 1.f : 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      a[c] = __fsub_rn(__fmul_rn(__fmul_rn(a[c], v), 2.f), 1.f);  // im2tensor: image / 0.5 - 1
      b[c] = __fsub_rn(__fmul_rn(__fmul_rn(b[c], v), 2.f), 1.f);
    }
  }
  float* xp = x0 + (size_t)k * 3 * HW + p;
  float* xg = x0 + ((size_t)K + k) * 3 * HW + p;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    xp[(size_t)c * HW] = __fdiv_rn(__fsub_rn(a[c], kShift[c]), kScale[c]);
    xg[(size_t)c * HW] = __fdiv_rn(__fsub_rn(b[c], kShift[c]), kScale[c]);
  }
  float* r = rw + (size_t)k * M * HW + p;
  const float m = mask ? __fadd_rn(__fadd_rn(mask[3 * i], mask[3 * i + 1]), mask[3 * i + 2]) : 0.f;
  if (EVAL) {
    r[0] = 3.f * v;
    if (M == 3) {
      r[HW] = m;
      r[2 * (size_t)HW] = __fadd_rn(__fadd_rn(__fsub_rn(1.f, mask[3 * i]), __fsub_rn(1.f, mask[3 * i + 1])),
                                    __fsub_rn(1.f, mask[3 * i + 2]));
    }
  } else {
    r[0] = mask ? m : 3.f;
  }
}

// Implicit-GEMM convolution, zero padding PAD, stride S, KS x KS kernel, + bias, ReLU: out[n, co, oy, ox] over the
// npix = nimg Ho Wo output pixels of all images.  GEMM rows are output channels (A = the weights [Cout, Cin KS KS] as
// torch stores them), columns output pixels (B = the im2col of the input, gathered by the tile loader, 0 outside the
// image).  A CTA computes a kBM x kBN tile, staging kBK-deep slices of A and B in shared memory; each thread owns
// kBM / 16 x kBN / 16 outputs (rows ty + 16 i, columns tx + 16 j) and accumulates over k in order with FFMA, so an
// output's value does not depend on its tile or on the other images.
constexpr int kBM = 64, kBN = 128, kBK = 16, kConvThreads = 256;
constexpr int kTM = kBM / 16, kTN = kBN / 16;

template <int KS, int S, int PAD>
__global__ void __launch_bounds__(kConvThreads) lpips_conv_kernel(const float* __restrict__ in,
                                                                   const float* __restrict__ w,
                                                                   const float* __restrict__ bias,
                                                                   float* __restrict__ out, int Cin, int Cout, int Hi,
                                                                   int Wi, int Ho, int Wo, int npix) {
  __shared__ float As[kBK][kBM + 1];
  __shared__ float Bs[kBK][kBN];
  constexpr int KK = KS * KS;
  const int Kd = Cin * KK;
  const int co0 = blockIdx.y * kBM, p0 = blockIdx.x * kBN;
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  const int hwo = Ho * Wo;
  // the B column this thread loads: one output pixel, rows bk0, bk0 + 2, ...
  const int bn = tid % kBN, bk0 = tid / kBN;
  const int pl = p0 + bn;
  const bool pin = pl < npix;
  int img = 0, oy = 0, ox = 0;
  if (pin) {
    img = pl / hwo;
    const int r = pl - img * hwo;
    oy = r / Wo, ox = r - oy * Wo;
  }
  const float* src = in + (size_t)img * Cin * Hi * Wi;
  const int iy0 = oy * S - PAD, ix0 = ox * S - PAD;

  float acc[kTM][kTN];
#pragma unroll
  for (int i = 0; i < kTM; ++i)
#pragma unroll
    for (int j = 0; j < kTN; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < Kd; k0 += kBK) {
#pragma unroll
    for (int i = 0; i < kBM * kBK / kConvThreads; ++i) {
      const int e = tid + kConvThreads * i, am = e / kBK, ak = e % kBK;
      const int co = co0 + am, k = k0 + ak;
      As[ak][am] = (co < Cout && k < Kd) ? w[(size_t)co * Kd + k] : 0.f;
    }
#pragma unroll
    for (int i = 0; i < kBK * kBN / kConvThreads; ++i) {
      const int kl = bk0 + (kConvThreads / kBN) * i, k = k0 + kl;
      float v = 0.f;
      if (pin && k < Kd) {
        const int ci = k / KK, r = k - ci * KK, ky = r / KS, kx = r - ky * KS;
        const int iy = iy0 + ky, ix = ix0 + kx;
        if (iy >= 0 && iy < Hi && ix >= 0 && ix < Wi) v = src[((size_t)ci * Hi + iy) * Wi + ix];
      }
      Bs[kl][bn] = v;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kBK; ++k) {
      float a[kTM], b[kTN];
#pragma unroll
      for (int i = 0; i < kTM; ++i) a[i] = As[k][ty + 16 * i];
#pragma unroll
      for (int j = 0; j < kTN; ++j) b[j] = Bs[k][tx + 16 * j];
#pragma unroll
      for (int i = 0; i < kTM; ++i)
#pragma unroll
        for (int j = 0; j < kTN; ++j) acc[i][j] = __fmaf_rn(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }

#pragma unroll
  for (int i = 0; i < kTM; ++i) {
    const int co = co0 + ty + 16 * i;
    if (co >= Cout) continue;
    const float bv = bias[co];
#pragma unroll
    for (int j = 0; j < kTN; ++j) {
      const int p = p0 + tx + 16 * j;
      if (p >= npix) continue;
      const int n = p / hwo, r = p - n * hwo;
      out[((size_t)n * Cout + co) * hwo + r] = fmaxf(__fadd_rn(acc[i][j], bv), 0.f);
    }
  }
}

// max pool 3 / 2, floor mode, no padding: [nc, Hi, Wi] -> [nc, Ho, Wo], one thread per output
__global__ void __launch_bounds__(256) lpips_pool_kernel(const float* __restrict__ in, long long nc, int Hi, int Wi,
                                                          int Ho, int Wo, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nc * Ho * Wo) return;
  const long long c = i / ((long long)Ho * Wo);
  const int r = (int)(i - c * Ho * Wo), oy = r / Wo, ox = r - oy * Wo;
  const float* s = in + ((size_t)c * Hi + 2 * oy) * Wi + 2 * ox;
  float m = s[0];
#pragma unroll
  for (int dy = 0; dy < 3; ++dy)
#pragma unroll
    for (int dx = 0; dx < 3; ++dx) m = fmaxf(m, s[dy * Wi + dx]);
  out[i] = m;
}

// One thread per (camera k, pixel p) of a tap of C channels and hw pixels (features [2K, C, hw], pred then gt):
// d[k * ld + p] = sum_c lin[c] (f0_c / (|f0| + eps) - f1_c / (|f1| + eps))^2, channels in order, fp32.
__global__ void __launch_bounds__(256) lpips_tap_kernel(const float* __restrict__ f, const float* __restrict__ lin,
                                                         int K, int C, int hw, float* __restrict__ d, int ld) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= K * hw) return;
  const int k = i / hw, p = i - k * hw;
  const float* f0 = f + (size_t)k * C * hw + p;
  const float* f1 = f + ((size_t)K + k) * C * hw + p;
  float s0 = 0.f, s1 = 0.f;
  for (int c = 0; c < C; ++c) {
    const float a = f0[(size_t)c * hw], b = f1[(size_t)c * hw];
    s0 = __fmaf_rn(a, a, s0), s1 = __fmaf_rn(b, b, s1);
  }
  const float n0 = __fadd_rn(__fsqrt_rn(s0), kNormEps), n1 = __fadd_rn(__fsqrt_rn(s1), kNormEps);
  float acc = 0.f;
  for (int c = 0; c < C; ++c) {
    const float t = __fsub_rn(__fdiv_rn(f0[(size_t)c * hw], n0), __fdiv_rn(f1[(size_t)c * hw], n1));
    acc = __fmaf_rn(lin[c], __fmul_rn(t, t), acc);
  }
  d[(size_t)k * ld + p] = acc;
}

// One CTA per (tile of kRedThreads pixels of one tap, camera blockIdx.y), one thread per pixel (i, j) of the tap's
// h x w map: m_l = adaptive_avg_pool2d's bin mean of each row's weights over rows [floor(i H / h), ceil((i + 1) H / h))
// and the matching columns, in fp64; partial[(k * tiles + tile) * kSums + 2m (+1)] = sum m_l d_l (sum m_l).
__global__ void __launch_bounds__(kRedThreads) lpips_reduce_kernel(const float* __restrict__ d,
                                                                   const float* __restrict__ rw, Geom g,
                                                                   double* __restrict__ partial) {
  __shared__ double red[kRedWarps][kSums];
  const int tile = blockIdx.x, k = blockIdx.y, H = g.H, W = g.W;
  int l = 0;
  while (l < kTaps - 1 && tile >= g.tile0[l + 1]) ++l;
  const int h = g.th[l], w = g.tw[l];
  const int p = (tile - g.tile0[l]) * kRedThreads + threadIdx.x;
  double acc[kSums];
#pragma unroll
  for (int j = 0; j < kSums; ++j) acc[j] = 0.0;
  if (p < h * w) {
    const int i = p / w, j = p - i * w;
    const int ys = (i * H) / h, ye = ((i + 1) * H + h - 1) / h;
    const int xs = (j * W) / w, xe = ((j + 1) * W + w - 1) / w;
    const double dv = (double)d[(size_t)k * g.doff[kTaps] + g.doff[l] + p];
    const double cnt = (double)((ye - ys) * (xe - xs));
#pragma unroll
    for (int m = 0; m < kMaxRows; ++m) {
      if (m >= g.M) break;
      const float* r = rw + ((size_t)k * g.M + m) * H * W;
      double s = 0.0;
      for (int y = ys; y < ye; ++y)
        for (int x = xs; x < xe; ++x) s += (double)r[(size_t)y * W + x];
      const double ml = s / cnt;
      acc[2 * m] = ml * dv;
      acc[2 * m + 1] = ml;
    }
  }
  block_sum<kSums, kRedWarps>(acc, red);
  if (threadIdx.x == 0) {
    double* o = partial + ((size_t)k * g.tile0[kTaps] + tile) * kSums;
#pragma unroll
    for (int j = 0; j < kSums; ++j) o[j] = acc[j];
  }
}

// One thread per camera: per row m and tap l, the tap's tiles added in order; scores[k, m] = sum_l num_l / den_l over
// the taps with den_l > 0.
__global__ void __launch_bounds__(64) lpips_finish_kernel(const double* __restrict__ partial, Geom g,
                                                           double* __restrict__ scores) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= g.K) return;
  const double* p = partial + (size_t)k * g.tile0[kTaps] * kSums;
  for (int m = 0; m < g.M; ++m) {
    double s = 0.0;
    for (int l = 0; l < kTaps; ++l) {
      double num = 0.0, den = 0.0;
      for (int t = g.tile0[l]; t < g.tile0[l + 1]; ++t) num += p[t * kSums + 2 * m], den += p[t * kSums + 2 * m + 1];
      if (den > 0.0) s += num / den;
    }
    scores[(size_t)k * g.M + m] = s;
  }
}

template <int KS, int S, int PAD>
int conv(const float* in, const float* w, const float* b, float* out, int nimg, int Cin, int Cout, int Hi, int Wi,
         int Ho, int Wo, cudaStream_t st) {
  const int npix = nimg * Ho * Wo;
  const dim3 grid(cdiv(npix, kBN), Cout / kBM);
  lpips_conv_kernel<KS, S, PAD><<<grid, kConvThreads, 0, st>>>(in, w, b, out, Cin, Cout, Hi, Wi, Ho, Wo, npix);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int pool(const float* in, long long nc, int Hi, int Wi, int Ho, int Wo, float* out, cudaStream_t st) {
  const long long n = nc * Ho * Wo;
  lpips_pool_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(in, nc, Hi, Wi, Ho, Wo, out);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

}  // namespace
}  // namespace dyn

using namespace dyn;

extern "C" {

size_t dyn_lpips_param_count(void) { return offsets().total; }

size_t dyn_lpips_workspace_bytes(int K, int H, int W) {
  return lpips_shape_ok(K, H, W) ? carve(geom(K, H, W, kMaxRows), nullptr).bytes : 0;
}

int dyn_lpips(const float* pred, const float* gt, const float* mask, int K, int H, int W, int mode,
              const float* weights, double* scores, void* workspace, size_t workspace_bytes, void* stream) {
  DYN_CHECK_ARG(pred && gt && weights && scores && lpips_shape_ok(K, H, W));
  DYN_CHECK_ARG(mode == DYN_SCORES_PLAIN || mode == DYN_SCORES_EVAL);
  const int M = (mode == DYN_SCORES_EVAL && mask) ? 3 : 1;
  const Geom g = geom(K, H, W, M);
  const size_t need = carve(geom(K, H, W, kMaxRows), nullptr).bytes;
  if (workspace == nullptr || workspace_bytes < need)
    return fail(DYN_E_WORKSPACE, "lpips: workspace of %zu bytes, %zu needed", workspace_bytes, need);
  const Carve c = carve(geom(K, H, W, kMaxRows), (char*)workspace);
  const Offsets o = offsets();
  cudaStream_t st = (cudaStream_t)stream;
  const int n = 2 * K, HW = H * W;

  const long long np = (long long)K * HW;
  if (mode == DYN_SCORES_EVAL)
    lpips_prep_kernel<true><<<(unsigned)((np + 255) / 256), 256, 0, st>>>(pred, gt, mask, K, HW, M, c.x0, c.rw);
  else
    lpips_prep_kernel<false><<<(unsigned)((np + 255) / 256), 256, 0, st>>>(pred, gt, mask, K, HW, M, c.x0, c.rw);
  DYN_LAUNCH_CHECK();

  const float* P = weights;
  int rc;
  if ((rc = conv<11, 4, 2>(c.x0, P + o.w[0], P + o.b[0], c.a1, n, 3, 64, H, W, g.h1, g.w1, st))) return rc;
  if ((rc = pool(c.a1, (long long)n * 64, g.h1, g.w1, g.h2, g.w2, c.p1, st))) return rc;
  if ((rc = conv<5, 1, 2>(c.p1, P + o.w[1], P + o.b[1], c.a2, n, 64, 192, g.h2, g.w2, g.h2, g.w2, st))) return rc;
  if ((rc = pool(c.a2, (long long)n * 192, g.h2, g.w2, g.h3, g.w3, c.p2, st))) return rc;
  if ((rc = conv<3, 1, 1>(c.p2, P + o.w[2], P + o.b[2], c.a3, n, 192, 384, g.h3, g.w3, g.h3, g.w3, st))) return rc;
  if ((rc = conv<3, 1, 1>(c.a3, P + o.w[3], P + o.b[3], c.a4, n, 384, 256, g.h3, g.w3, g.h3, g.w3, st))) return rc;
  if ((rc = conv<3, 1, 1>(c.a4, P + o.w[4], P + o.b[4], c.a5, n, 256, 256, g.h3, g.w3, g.h3, g.w3, st))) return rc;

  const float* taps[kTaps] = {c.a1, c.a2, c.a3, c.a4, c.a5};
  for (int l = 0; l < kTaps; ++l) {
    const int hw = g.th[l] * g.tw[l];
    lpips_tap_kernel<<<cdiv((long long)K * hw, 256), 256, 0, st>>>(taps[l], P + o.lin[l], K, kCout[l], hw,
                                                                   c.d + g.doff[l], g.doff[kTaps]);
    DYN_LAUNCH_CHECK();
  }
  lpips_reduce_kernel<<<dim3(g.tile0[kTaps], K), kRedThreads, 0, st>>>(c.d, c.rw, g, c.partial);
  DYN_LAUNCH_CHECK();
  lpips_finish_kernel<<<cdiv(K, 64), 64, 0, st>>>(c.partial, g, scores);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

}  // extern "C"
