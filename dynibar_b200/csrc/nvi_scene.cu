// An Nvidia-benchmark scene resident on the device (eval_nvidia.py DynamicVideoDataset.__getitem__ and the ground
// truth / mask reads of its __main__ block, restated).  DESIGN §3.8 gives the semantics.
//
//   dyn_area_resize      at load: cv2.resize(INTER_AREA) uint8 -> uint8 of many images (the ground truth)
//   dyn_nearest_resize   at load: cv2.resize(INTER_NEAREST) uint8 -> uint8, optionally thresholded (> 0)
//   dyn_nvi_time_step    per time step: source stacks, static masks, the masked static stack, ground truth, masks
//   dyn_nvi_rays         per time step: every pixel's ray of the K target cameras, and camera_index
//
// The per-time-step calls read their view table and cameras from device memory the caller filled with one
// asynchronous copy, so a time step makes no host synchronisation.  No float atomics: the same inputs give the same
// bits.
#include <math.h>

#include "common.cuh"
#include "scene_common.cuh"

namespace dyn {
namespace {

constexpr int kThreads = 256;
constexpr int kTileW = 32, kTileH = kThreads / kTileW;  // area resize: one 32 x 8 output tile per CTA
constexpr int kMaxC = 4;
constexpr int kMaxCams = 16;

// One axis of OpenCV's computeResizeAreaTab for destination index d: the entries (source index, float32 weight) in
// table order, computed in double as OpenCV does (scale = 1 / (dst / src)); slivers of <= 1e-3 are dropped.
struct AreaCell {
  double f1, f2, cell;
  int s1, s2;
  __device__ AreaCell(int d, int ssize, double scale) {
    f1 = d * scale;
    f2 = f1 + scale;
    cell = fmin(scale, ssize - f1);
    s2 = min((int)floor(f2), ssize - 1);
    s1 = min((int)ceil(f1), s2);
  }
  __device__ bool head() const { return s1 - f1 > 1e-3; }
  __device__ float head_w() const { return (float)((s1 - f1) / cell); }
  __device__ float body_w() const { return (float)(1.0 / cell); }
  __device__ bool tail() const { return f2 - s2 > 1e-3; }
  __device__ float tail_w() const { return (float)(fmin(fmin(f2 - s2, 1.0), cell) / cell); }
};

// The horizontal pass of one source row at one destination column: buf = (((0 + s a0) + s a1) + ...), rounded
// products, no contraction.
__device__ __forceinline__ void area_row(const uint8_t* __restrict__ row, const AreaCell& x, int C, float* buf) {
  for (int c = 0; c < C; ++c) buf[c] = 0.f;
  if (x.head()) {
    const float a = x.head_w();
    for (int c = 0; c < C; ++c) buf[c] = __fadd_rn(buf[c], __fmul_rn((float)row[(x.s1 - 1) * C + c], a));
  }
  const float a = x.body_w();
  for (int sx = x.s1; sx < x.s2; ++sx)
    for (int c = 0; c < C; ++c) buf[c] = __fadd_rn(buf[c], __fmul_rn((float)row[sx * C + c], a));
  if (x.tail()) {
    const float t = x.tail_w();
    for (int c = 0; c < C; ++c) buf[c] = __fadd_rn(buf[c], __fmul_rn((float)row[x.s2 * C + c], t));
  }
}

// OpenCV's resizeArea for one output pixel: the vertical weights in table order over the horizontal passes, the first
// term a product (sum = beta * buf), the rest accumulated; rounded to nearest even at the end.
__device__ __forceinline__ void area_generic(const uint8_t* __restrict__ img, int sh, int sw, int C, int dy, int dx,
                                             double sy_scale, double sx_scale, float* acc) {
  const AreaCell y(dy, sh, sy_scale), x(dx, sw, sx_scale);
  float buf[kMaxC];
  bool first = true;
  auto add = [&](int sy, float beta) {
    area_row(img + (size_t)sy * sw * C, x, C, buf);
    for (int c = 0; c < C; ++c) acc[c] = first ? __fmul_rn(beta, buf[c]) : __fadd_rn(acc[c], __fmul_rn(beta, buf[c]));
    first = false;
  };
  if (y.head()) add(y.s1 - 1, y.head_w());
  const float b = y.body_w();
  for (int sy = y.s1; sy < y.s2; ++sy) add(sy, b);
  if (y.tail()) add(y.s2, y.tail_w());
}

// blockIdx.z: image; one 32 x 8 output tile per CTA, one output pixel (all channels) per thread.
__global__ void __launch_bounds__(kThreads) area_kernel(const uint8_t* __restrict__ src, int sh, int sw, int C, int dh,
                                                        int dw, uint8_t* __restrict__ dst) {
  const int dx = blockIdx.x * kTileW + (threadIdx.x % kTileW), dy = blockIdx.y * kTileH + threadIdx.x / kTileW;
  if (dx >= dw || dy >= dh) return;
  const uint8_t* img = src + (size_t)blockIdx.z * sh * sw * C;
  uint8_t* out = dst + (((size_t)blockIdx.z * dh + dy) * dw + dx) * C;
  const int fy = sh / dh, fx = sw / dw;
  if (fy * dh == sh && fx * dw == sw) {
    // resizeAreaFast: the integer box sum; (s + 2) >> 2 at 2 x 2 (its vector path), else
    // saturate_cast<uchar>(s * (1.f / area)) in float32
    const float scale = __fdiv_rn(1.f, (float)(fy * fx));
    for (int c = 0; c < C; ++c) {
      int s = 0;
      for (int i = 0; i < fy; ++i) {
        const uint8_t* row = img + ((size_t)(dy * fy + i) * sw + dx * fx) * C + c;
        for (int j = 0; j < fx; ++j) s += row[j * C];
      }
      const int v = (fy == 2 && fx == 2) ? (s + 2) >> 2 : __float2int_rn(__fmul_rn((float)s, scale));
      out[c] = (uint8_t)min(max(v, 0), 255);
    }
    return;
  }
  float acc[kMaxC];
  area_generic(img, sh, sw, C, dy, dx, 1.0 / ((double)dh / sh), 1.0 / ((double)dw / sw), acc);
  for (int c = 0; c < C; ++c) out[c] = (uint8_t)min(max(__float2int_rn(acc[c]), 0), 255);
}

__global__ void __launch_bounds__(kThreads) nearest_kernel(const uint8_t* __restrict__ src, int sh, int sw, int C,
                                                           int dh, int dw, int threshold, uint8_t* __restrict__ dst) {
  const long long p = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (p >= (long long)dh * dw) return;
  const int y = (int)(p / dw), x = (int)(p - (long long)y * dw);
  const uint8_t* s = src + (((size_t)blockIdx.y * sh + nn_index(y, dh, sh)) * sw + nn_index(x, dw, sw)) * C;
  uint8_t* d = dst + ((size_t)blockIdx.y * dh * dw + p) * C;
  for (int c = 0; c < C; ++c) d[c] = threshold ? (s[c] > 0 ? 1 : 0) : s[c];
}

struct StepOut {
  float *src, *st, *st_mask, *st_masked, *gt, *dmask;
};

// blockIdx.y = plane: [0, nd) dynamic source views, [nd, nd + ns) static source views (image, coarse mask, masked
// image), [nd + ns, nd + ns + K) ground truth and dynamic mask of target camera k.  table[plane] names the frame
// (source views) or the row t * S + s of the ground-truth store; rows outside the scene write nothing.
__global__ void __launch_bounds__(kThreads) time_step_kernel(dyn_nvi_scene_t s, const int* __restrict__ table, int nd,
                                                             int ns, int K, StepOut o) {
  const int HW = s.H * s.W;
  const int p = blockIdx.x * kThreads + threadIdx.x;
  if (p >= HW) return;
  const int plane = blockIdx.y, f = table[plane];
  if (plane < nd + ns) {
    if (f < 0 || f >= s.N) return;
    const uint8_t* px = s.frames + ((size_t)f * HW + p) * 3;
    const float r = u8f(px[0]), g = u8f(px[1]), b = u8f(px[2]);
    const bool dyn = plane < nd;
    const size_t q = (size_t)(dyn ? plane : plane - nd) * HW + p;
    float* d = (dyn ? o.src : o.st) + q * 3;
    d[0] = r;
    d[1] = g;
    d[2] = b;
    if (dyn) return;
    const float m = u8f(s.smask[(size_t)f * HW + p]);
    o.st_mask[q] = m;
    float* dm = o.st_masked + q * 3;
    dm[0] = __fmul_rn(r, m);
    dm[1] = __fmul_rn(g, m);
    dm[2] = __fmul_rn(b, m);
    return;
  }
  if (f < 0 || f >= s.T * s.S) return;
  const size_t src = ((size_t)f * HW + p) * 3, dst = ((size_t)(plane - nd - ns) * HW + p) * 3;
  for (int c = 0; c < 3; ++c) {
    o.gt[dst + c] = u8f(s.gt[src + c]);
    o.dmask[dst + c] = (float)s.dmask[src + c];
  }
}

// One thread per ray of K cameras of H x W: ray k * H * W + p is camera k's pixel p; cams (device) [K, 12].
__global__ void __launch_bounds__(kThreads) nvi_rays_kernel(const float* __restrict__ cams, int K, int H, int W,
                                                            float* __restrict__ ray_o, float* __restrict__ ray_d,
                                                            float* __restrict__ uv, int* __restrict__ camera_index) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  const int HW = H * W;
  if (i >= (long long)K * HW) return;
  const int k = (int)(i / HW), p = (int)(i - (long long)k * HW);
  const float u = (float)(p % W), v = (float)(p / W);
  pixel_ray(cams + 12 * k, u, v, ray_o + 3 * i, ray_d + 3 * i);
  uv[2 * i] = u;
  uv[2 * i + 1] = v;
  camera_index[i] = k;
}

bool nvi_scene_ok(const dyn_nvi_scene_t* s) {
  return s && s->frames && s->smask && s->gt && s->dmask && s->N >= 1 && s->H >= 1 && s->W >= 1 &&
         (long long)s->H * s->W < (1ll << 31) / 16 && s->T >= 0 && s->S >= 0;
}

}  // namespace
}  // namespace dyn

using namespace dyn;

extern "C" {

int dyn_area_resize(const uint8_t* src, int N, int sh, int sw, int C, int dh, int dw, uint8_t* dst, void* stream) {
  DYN_CHECK_ARG(src && dst && N >= 0 && N < 65536 && C >= 1 && C <= kMaxC);
  DYN_CHECK_ARG(dh >= 1 && dw >= 1 && sh >= dh && sw >= dw && (long long)sh * sw * C < (1ll << 31));
  if (N == 0) return DYN_OK;
  area_kernel<<<dim3(cdiv(dw, kTileW), cdiv(dh, kTileH), N), kThreads, 0, (cudaStream_t)stream>>>(src, sh, sw, C, dh,
                                                                                                  dw, dst);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int dyn_nearest_resize(const uint8_t* src, int N, int sh, int sw, int C, int dh, int dw, int threshold, uint8_t* dst,
                       void* stream) {
  DYN_CHECK_ARG(src && dst && N >= 0 && N < 65536 && C >= 1 && sh >= 1 && sw >= 1 && dh >= 1 && dw >= 1);
  DYN_CHECK_ARG((long long)dh * dw < (1ll << 31) - kThreads);
  if (N == 0) return DYN_OK;
  nearest_kernel<<<dim3(cdiv((long long)dh * dw, kThreads), N), kThreads, 0, (cudaStream_t)stream>>>(
      src, sh, sw, C, dh, dw, threshold, dst);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int dyn_nvi_time_step(const dyn_nvi_scene_t* scene, const int* table, int nd, int ns, int K, float* src_rgbs,
                      float* static_src_rgbs, float* static_src_masks, float* static_masked, float* gt,
                      float* dynamic_mask, void* stream) {
  DYN_CHECK_ARG(nvi_scene_ok(scene) && table && nd >= 0 && ns >= 0 && K >= 0 && nd + ns + K <= 65535);
  DYN_CHECK_ARG((nd == 0 || src_rgbs) && (ns == 0 || (static_src_rgbs && static_src_masks && static_masked)));
  DYN_CHECK_ARG(K == 0 || (gt && dynamic_mask));
  if (nd + ns + K == 0) return DYN_OK;
  StepOut o{src_rgbs, static_src_rgbs, static_src_masks, static_masked, gt, dynamic_mask};
  time_step_kernel<<<dim3(cdiv((long long)scene->H * scene->W, kThreads), nd + ns + K), kThreads, 0,
                      (cudaStream_t)stream>>>(*scene, table, nd, ns, K, o);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int dyn_nvi_rays(const float* cams, int K, int H, int W, float* ray_o, float* ray_d, float* uv_grid, int* camera_index,
                 void* stream) {
  DYN_CHECK_ARG(cams && ray_o && ray_d && uv_grid && camera_index && K >= 1 && K <= kMaxCams && H >= 1 && W >= 1);
  DYN_CHECK_ARG((long long)K * H * W < (1ll << 31) / 3);
  nvi_rays_kernel<<<cdiv((long long)K * H * W, kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      cams, K, H, W, ray_o, ray_d, uv_grid, camera_index);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

}  // extern "C"
