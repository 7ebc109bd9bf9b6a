// A monocular training scene resident on the device (ibrnet/data_loaders/monocular.py MonocularDataset.__getitem__
// and ibrnet/sample_ray.py RaySamplerSingleImage.random_sample, restated).  DESIGN §3.7 gives the semantics.
//
//   dyn_scene_masks      once per scene: motion, static and source masks of all frames (two launches)
//   dyn_scene_views      per step: the three float source-view stacks and the target's full-frame supervision
//   dyn_scene_rays       per step: the selected pixels' rays and supervision (or every pixel's rays)
//
// Per step everything the kernels need to know (view table, target frame, camera matrix) sits in device memory the
// caller filled with one asynchronous copy, so a step makes no host synchronisation.  No float atomics; every float
// is the reference's float32 expression rounded as numpy rounds it (__fdiv_rn / __fmul_rn / __fsub_rn, no
// contraction): the same inputs give the same bits.
#include <math.h>

#include "common.cuh"
#include "scene_common.cuh"

namespace dyn {
namespace {

constexpr int kMaxRadius = 16;           // erosion radius limit (disk of 33 x 33)
constexpr int kTileW = 32, kTileH = 16;  // erosion output tile
constexpr int kThreads = 256;
constexpr int kStacks = 3;
constexpr int kMaxTableViews = 3 * kMaxViews;

// scipy.ndimage mode 'reflect' (d c b a | a b c d), periodic with period 2n for offsets beyond the image
__device__ __forceinline__ int reflect(int i, int n) {
  const int p = 2 * n;
  i %= p;
  if (i < 0) i += p;
  return i < n ? i : p - 1 - i;
}

// 1 - m / 255 > 1e-3 in float32 (monocular.py:168 / :174, :194 / :204)
__device__ __forceinline__ bool mask_on(uint8_t m) {
  return __fsub_rn(1.0f, __fdiv_rn((float)m, 255.0f)) > 1e-3f;
}

// Threshold + erosion at eh x ew (the motion mask resized to height 288): one 32 x 16 output tile of one frame per
// CTA.  The tile and its reflected halo are thresholded into shared memory straight from the nearest-resized
// dynamic mask (thresholding before a nearest resize equals thresholding after it), then each output takes the
// minimum over the disk X^2 + Y^2 <= r^2.
__global__ void __launch_bounds__(kThreads) erode_kernel(const uint8_t* __restrict__ dyn, int mh, int mw, int mc,
                                                         int eh, int ew, int r, uint8_t* __restrict__ eroded) {
  __shared__ uint8_t tile[kTileH + 2 * kMaxRadius][kTileW + 2 * kMaxRadius];
  const int n = blockIdx.z, y0 = blockIdx.y * kTileH, x0 = blockIdx.x * kTileW;
  const int th = kTileH + 2 * r, tw = kTileW + 2 * r;
  const uint8_t* m = dyn + (size_t)n * mh * mw * mc;
  for (int i = threadIdx.x; i < th * tw; i += kThreads) {
    const int ty = i / tw, tx = i - ty * tw;
    const int y = reflect(y0 - r + ty, eh), x = reflect(x0 - r + tx, ew);
    const int sy = nn_index(y, eh, mh), sx = nn_index(x, ew, mw);
    tile[ty][tx] = mask_on(m[((size_t)sy * mw + sx) * mc]) ? 1 : 0;
  }
  __syncthreads();
  const int tx = threadIdx.x & (kTileW - 1);
  for (int ty = threadIdx.x / kTileW; ty < kTileH; ty += kThreads / kTileW) {
    const int y = y0 + ty, x = x0 + tx;
    if (y >= eh || x >= ew) continue;
    uint8_t v = 1;
    for (int dy = -r; dy <= r && v; ++dy)
      for (int dx = -r; dx <= r; ++dx)
        if (dx * dx + dy * dy <= r * r) v &= tile[ty + r + dy][tx + r + dx];
    eroded[((size_t)n * eh + y) * ew + x] = v;
  }
}

// Per frame pixel: motion = eroded at the nearest (eh, ew) pixel; static = threshold of the nearest static-mask
// pixel; srcmask = the nearest dynamic-mask pixel's raw channels (load_src_view: m / 255, not thresholded).
__global__ void __launch_bounds__(kThreads) frame_masks_kernel(const uint8_t* __restrict__ eroded, int eh, int ew,
                                                               const uint8_t* __restrict__ dyn, int mh, int mw, int mc,
                                                               const uint8_t* __restrict__ st, int sh, int sw, int H,
                                                               int W, uint8_t* __restrict__ motion,
                                                               uint8_t* __restrict__ stat,
                                                               uint8_t* __restrict__ srcmask) {
  const int n = blockIdx.y;
  const int p = blockIdx.x * kThreads + threadIdx.x;
  if (p >= H * W) return;
  const int y = p / W, x = p - y * W;
  const size_t o = (size_t)n * H * W + p;
  motion[o] = eroded[((size_t)n * eh + nn_index(y, H, eh)) * ew + nn_index(x, W, ew)];
  stat[o] = mask_on(st[((size_t)n * sh + nn_index(y, H, sh)) * sw + nn_index(x, W, sw)]) ? 1 : 0;
  const uint8_t* m = dyn + (((size_t)n * mh + nn_index(y, H, mh)) * mw + nn_index(x, W, mw)) * mc;
  for (int c = 0; c < mc; ++c) srcmask[o * mc + c] = m[c];
}

struct Stacks {
  float* out[kStacks];
  int views[kStacks];
};

struct Target {
  float *rgb, *disp, *motion, *stat, *flows, *masks;
};

// blockIdx.y < V: view row (frame, vv, masked, stack << 8 | slot) of the table -> float32 [H, W, 3] of its stack;
// blockIdx.y == V: the target frame (row V: frame) -> rgb, disp, motion_mask, static_mask, flows [6, H, W, 2],
// masks [6, H, W].  Rows that name no valid frame / slot write nothing (the host checks the table before the copy).
__global__ void __launch_bounds__(kThreads) views_kernel(dyn_scene_t s, const int* __restrict__ table, int V,
                                                         Stacks stk, Target tg) {
  const int HW = s.H * s.W;
  const int p = blockIdx.x * kThreads + threadIdx.x;
  if (p >= HW) return;
  const int v = blockIdx.y;
  if (v < V) {
    const int4 row = reinterpret_cast<const int4*>(table)[v];
    const int f = row.x, vv = row.y, stack = row.w >> 8, slot = row.w & 255;
    // selects, not a dynamic index into the by-value struct (which would put it on the stack)
    const int nviews = stack == 0 ? stk.views[0] : stack == 1 ? stk.views[1] : stk.views[2];
    float* out = stack == 0 ? stk.out[0] : stack == 1 ? stk.out[1] : stk.out[2];
    if (f < 0 || f >= s.N || vv >= 8 || stack < 0 || stack >= kStacks || slot >= nviews) return;
    const uint8_t* src = vv < 0 ? s.frames + ((size_t)f * HW + p) * 3 : s.vviews + (((size_t)f * 8 + vv) * HW + p) * 3;
    float* dst = out + ((size_t)slot * HW + p) * 3;
    const float r = u8f(src[0]), g = u8f(src[1]), b = u8f(src[2]);
    if (row.z && s.srcmask != nullptr) {  // src_rgb * st_mask (monocular.py:142): 1 or 3 mask channels
      const uint8_t* m = s.srcmask + ((size_t)f * HW + p) * s.mc;
      const int c1 = s.mc == 3 ? 1 : 0, c2 = s.mc == 3 ? 2 : 0;
      dst[0] = __fmul_rn(r, u8f(m[0]));
      dst[1] = __fmul_rn(g, u8f(m[c1]));
      dst[2] = __fmul_rn(b, u8f(m[c2]));
    } else {
      dst[0] = r;
      dst[1] = g;
      dst[2] = b;
    }
    return;
  }
  const int f = table[4 * V];
  if (f < 0 || f >= s.N) return;
  const size_t o = (size_t)f * HW + p;
  const uint8_t* src = s.frames + o * 3;
  for (int c = 0; c < 3; ++c) tg.rgb[(size_t)p * 3 + c] = u8f(src[c]);
  tg.disp[p] = s.disp[o];
  tg.motion[p] = (float)s.motion[o];
  tg.stat[p] = (float)s.stat[o];
  const int fr = f - s.flow_base;
  if (fr < 0 || fr >= s.NF) return;
  for (int k = 0; k < 6; ++k) {
    const size_t q = ((size_t)fr * 6 + k) * HW + p;
    const float2 fl = reinterpret_cast<const float2*>(s.flows)[q];
    reinterpret_cast<float2*>(tg.flows)[(size_t)k * HW + p] = fl;
    tg.masks[(size_t)k * HW + p] = (float)s.flow_masks[q];
  }
}

// One thread per ray (pixel_ray: cam = M | t, M = R_c2w K^-1 formed on the host in float32).  sel == NULL: ray i is
// pixel i.
// Supervision pointers may be NULL (get_all: rays only).
__global__ void __launch_bounds__(kThreads) rays_kernel(dyn_scene_t s, const float* __restrict__ cam,
                                                        const int* __restrict__ target, const int* __restrict__ sel,
                                                        int R, float* __restrict__ ray_o, float* __restrict__ ray_d,
                                                        float* __restrict__ uv, Target tg) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= R) return;
  const int HW = s.H * s.W;
  const int p = sel ? sel[i] : i;
  if (p < 0 || p >= HW) return;
  const float u = (float)(p % s.W), v = (float)(p / s.W);
  pixel_ray(cam, u, v, ray_o + 3 * i, ray_d + 3 * i);
  uv[2 * i] = u;
  uv[2 * i + 1] = v;
  if (tg.rgb == nullptr) return;
  const int f = *target;
  if (f < 0 || f >= s.N) return;
  const size_t o = (size_t)f * HW + p;
  for (int c = 0; c < 3; ++c) tg.rgb[3 * i + c] = u8f(s.frames[o * 3 + c]);
  tg.disp[i] = s.disp[o];
  tg.motion[i] = (float)s.motion[o];
  tg.stat[i] = (float)s.stat[o];
  const int fr = f - s.flow_base;
  if (fr < 0 || fr >= s.NF) return;
  for (int k = 0; k < 6; ++k) {
    const size_t q = ((size_t)fr * 6 + k) * HW + p;
    reinterpret_cast<float2*>(tg.flows)[(size_t)k * R + i] = reinterpret_cast<const float2*>(s.flows)[q];
    tg.masks[(size_t)k * R + i] = (float)s.flow_masks[q];
  }
}

bool scene_ok(const dyn_scene_t* s) {
  return s && s->frames && s->vviews && s->motion && s->stat && s->disp && s->flows && s->flow_masks &&
         s->N >= 1 && s->H >= 1 && s->W >= 1 && (long long)s->H * s->W < (1ll << 31) / 8 && s->NF >= 0 &&
         (s->srcmask == nullptr || s->mc == 1 || s->mc == 3);
}

}  // namespace
}  // namespace dyn

using namespace dyn;

extern "C" {

size_t dyn_scene_masks_workspace_bytes(int N, int eh, int ew) {
  if (N < 1 || eh < 1 || ew < 1) return 0;
  return (size_t)N * eh * ew;
}

int dyn_scene_masks(const uint8_t* dyn, int mh, int mw, int mc, const uint8_t* st, int sh, int sw, int N, int H, int W,
                    int eh, int ew, int radius, uint8_t* motion, uint8_t* stat, uint8_t* srcmask, void* workspace,
                    size_t workspace_bytes, void* stream) {
  DYN_CHECK_ARG(dyn && st && motion && stat && srcmask);
  DYN_CHECK_ARG(N >= 1 && N < 65536 && mh >= 1 && mw >= 1 && (mc == 1 || mc == 3) && sh >= 1 && sw >= 1);
  DYN_CHECK_ARG(H >= 1 && W >= 1 && eh >= 1 && ew >= 1 && eh < 65536 * kTileH && ew < (1 << 30));
  DYN_CHECK_ARG(radius >= 0 && radius <= kMaxRadius);
  const size_t need = dyn_scene_masks_workspace_bytes(N, eh, ew);
  if (workspace == nullptr || workspace_bytes < need)
    return fail(DYN_E_WORKSPACE, "scene_masks: workspace of %zu bytes, %zu needed", workspace_bytes, need);
  cudaStream_t s = (cudaStream_t)stream;
  uint8_t* eroded = (uint8_t*)workspace;
  erode_kernel<<<dim3(cdiv(ew, kTileW), cdiv(eh, kTileH), N), kThreads, 0, s>>>(dyn, mh, mw, mc, eh, ew, radius,
                                                                                 eroded);
  DYN_LAUNCH_CHECK();
  frame_masks_kernel<<<dim3(cdiv((long long)H * W, kThreads), N), kThreads, 0, s>>>(
      eroded, eh, ew, dyn, mh, mw, mc, st, sh, sw, H, W, motion, stat, srcmask);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int dyn_scene_views(const dyn_scene_t* scene, const int* table, int V, float* src_rgbs, int n_src,
                    float* anchor_src_rgbs, int n_anchor, float* static_src_rgbs, int n_static, float* rgb, float* disp,
                    float* motion_mask, float* static_mask, float* flows, float* masks, void* stream) {
  DYN_CHECK_ARG(scene_ok(scene) && table && V >= 0 && V <= kMaxTableViews);
  DYN_CHECK_ARG(n_src >= 0 && n_anchor >= 0 && n_static >= 0 && n_src + n_anchor + n_static == V);
  DYN_CHECK_ARG((n_src == 0 || src_rgbs) && (n_anchor == 0 || anchor_src_rgbs) && (n_static == 0 || static_src_rgbs));
  DYN_CHECK_ARG(rgb && disp && motion_mask && static_mask && flows && masks);
  Stacks stk{{src_rgbs, anchor_src_rgbs, static_src_rgbs}, {n_src, n_anchor, n_static}};
  Target tg{rgb, disp, motion_mask, static_mask, flows, masks};
  views_kernel<<<dim3(cdiv((long long)scene->H * scene->W, kThreads), V + 1), kThreads, 0, (cudaStream_t)stream>>>(
      *scene, table, V, stk, tg);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int dyn_scene_rays(const dyn_scene_t* scene, const float* cam, const int* target, const int* sel, int R, float* ray_o,
                   float* ray_d, float* uv_grid, float* rgb, float* disp, float* motion_mask, float* static_mask,
                   float* flows, float* masks, void* stream) {
  DYN_CHECK_ARG(scene_ok(scene) && cam && ray_o && ray_d && uv_grid && R >= 0);
  DYN_CHECK_ARG(sel || R == scene->H * scene->W);
  const bool sup = rgb != nullptr;
  DYN_CHECK_ARG(!sup || (target && disp && motion_mask && static_mask && flows && masks));
  if (R == 0) return DYN_OK;
  Target tg{rgb, disp, motion_mask, static_mask, flows, masks};
  rays_kernel<<<cdiv(R, kThreads), kThreads, 0, (cudaStream_t)stream>>>(*scene, cam, target, sel, R, ray_o, ray_d,
                                                                         uv_grid, tg);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

}  // extern "C"
