// Deterministic softmax forward splatting and the virtual-source-view product of a monocular frame
// (render_source_vv.py: render_forward_splat:15, sobel_fg_alpha:118, the per-frame loop :253-330).
//
//   dyn_splat_softmax        splatting_function('softmax', frame, flow, metric) of the external extension
//   dyn_forward_splat        render_forward_splat: reproject RGB-D pixels, weight by inverse depth, splat
//   dyn_sobel_alpha          exp(-beta |sobel(x)|), replicate border
//   dyn_virtual_views        one frame's V virtual views as uint8 RGB: alpha, splat, threshold, erode, quantise
//
// No float atomics.  Each source pixel gets the key of its north-west cell; a stable radix sort groups sources by
// cell in source order; one thread per target pixel then reads the four cells that can reach it in a fixed order.
// The same inputs give the same bits, whatever the pile-up.
#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"

namespace dyn {
namespace {

constexpr float kSplatEps = 1e-7f;    // splatting_function's eps: out = sum / (sum_e + eps)
constexpr float kZClamp = 1e-8f;      // render_forward_splat: p /= clamp(p_z, 1e-8)
constexpr float kWeightEps = 1e-6f;   // (imp - min) / (max - min + 1e-6) * 20 - 10
constexpr int kMaxValues = 8;         // splatted channels per source (metric excluded)
constexpr int kCamFloats = 30;        // K_src^-1 (9) | R (9) | t (3) | K_dst (9), row-major

// key space of item b: (H+1)(W+1) cells whose NW corner is in [-1, W-1] x [-1, H-1]; B * cells marks "reaches no pixel"
__device__ __forceinline__ unsigned cell_key(float ox, float oy, int b, int B, int H, int W) {
  const unsigned cells = (unsigned)(H + 1) * (W + 1);
  // compared in float first: NaN, inf and far-off taps never reach the int conversion
  if (!(ox >= -1.f && ox < (float)W && oy >= -1.f && oy < (float)H)) return cells * B;
  const int cx = (int)floorf(ox), cy = (int)floorf(oy);
  return (unsigned)b * cells + (unsigned)(cy + 1) * (W + 1) + (unsigned)(cx + 1);
}

// splatting_function: target = pixel + flow, e = exp(metric).  grid (cdiv(HW), B)
__global__ void flow_prep_kernel(const float* __restrict__ flow, const float* __restrict__ metric, int H, int W,
                                 float* __restrict__ ox, float* __restrict__ oy, float* __restrict__ e,
                                 unsigned* __restrict__ keys, unsigned* __restrict__ idx) {
  const int HW = H * W, b = blockIdx.y;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  const long long s = (long long)b * HW + p;
  const float x = (float)(p % W) + flow[(long long)b * 2 * HW + p];
  const float y = (float)(p / W) + flow[(long long)b * 2 * HW + HW + p];
  ox[s] = x;
  oy[s] = y;
  e[s] = expf(metric[s]);
  keys[s] = cell_key(x, y, b, gridDim.y, H, W);
  idx[s] = (unsigned)s;
}

// render_forward_splat:15-48: p = K_dst (R ((d K_src^-1) [x y 1]^T) + t) in fp32, with the reference's operation
// order (each 3-term product summed left to right, no contraction); target = pixel + (p_xy / clamp(p_z) - pixel);
// importance 1 / p_z.  depth item stride 0 = one depth map shared by all items.  grid (cdiv(HW), B)
__global__ void project_kernel(const float* __restrict__ depth, long long depth_stride, const float* __restrict__ cams,
                               int H, int W, float* __restrict__ ox, float* __restrict__ oy, float* __restrict__ imp,
                               unsigned* __restrict__ keys, unsigned* __restrict__ idx) {
  const int HW = H * W, b = blockIdx.y;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  const float* c = cams + b * kCamFloats;
  const float* ki = c;
  const float* r = c + 9;
  const float* t = c + 18;
  const float* kd = c + 21;
  const float d = depth[b * depth_stride + p];
  const float x = (float)(p % W), y = (float)(p / W);
  float q[3], g[3], o[3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
    q[i] = __fadd_rn(__fadd_rn(__fmul_rn(__fmul_rn(d, ki[3 * i]), x), __fmul_rn(__fmul_rn(d, ki[3 * i + 1]), y)),
                     __fmul_rn(d, ki[3 * i + 2]));
#pragma unroll
  for (int i = 0; i < 3; ++i)
    g[i] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(r[3 * i], q[0]), __fmul_rn(r[3 * i + 1], q[1])),
                               __fmul_rn(r[3 * i + 2], q[2])), t[i]);
#pragma unroll
  for (int i = 0; i < 3; ++i)
    o[i] = __fadd_rn(__fadd_rn(__fmul_rn(kd[3 * i], g[0]), __fmul_rn(kd[3 * i + 1], g[1])), __fmul_rn(kd[3 * i + 2], g[2]));
  const float z = o[2];
  const float zc = z < kZClamp ? kZClamp : z;  // torch.clamp(min=): NaN stays NaN
  const float tx = __fadd_rn(x, __fsub_rn(__fdiv_rn(o[0], zc), x));
  const float ty = __fadd_rn(y, __fsub_rn(__fdiv_rn(o[1], zc), y));
  const long long s = (long long)b * HW + p;
  ox[s] = tx;
  oy[s] = ty;
  imp[s] = __fdiv_rn(1.f, z);
  keys[s] = cell_key(tx, ty, b, gridDim.y, H, W);
  idx[s] = (unsigned)s;
}

// per-item min / max of the importance (exact in any order), then e = exp((imp - min) / (max - min + 1e-6) * 20 - 10).
// One block per item: no cross-block reduction, no atomics.
constexpr int kMinMaxThreads = 1024;
__global__ void __launch_bounds__(kMinMaxThreads) importance_exp_kernel(const float* __restrict__ imp, int HW,
                                                                        float* __restrict__ e) {
  __shared__ float smin[kMinMaxThreads / 32], smax[kMinMaxThreads / 32];
  const long long base = (long long)blockIdx.x * HW;
  float mn = INFINITY, mx = -INFINITY;
  for (int p = threadIdx.x; p < HW; p += kMinMaxThreads) {
    const float v = imp[base + p];
    mn = fminf(mn, v);
    mx = fmaxf(mx, v);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) smin[warp] = mn, smax[warp] = mx;
  __syncthreads();
  mn = smin[0];
  mx = smax[0];
  for (int i = 1; i < kMinMaxThreads / 32; ++i) mn = fminf(mn, smin[i]), mx = fmaxf(mx, smax[i]);
  const float den = __fadd_rn(__fsub_rn(mx, mn), kWeightEps);
  for (int p = threadIdx.x; p < HW; p += kMinMaxThreads) {
    const float w = __fsub_rn(__fmul_rn(__fdiv_rn(__fsub_rn(imp[base + p], mn), den), 20.f), 10.f);
    e[base + p] = expf(w);
  }
}

// first / one-past-last sorted position of every occupied cell (both zeroed beforehand: empty cells are [0, 0))
__global__ void cell_ranges_kernel(const unsigned* __restrict__ keys, long long n, unsigned invalid,
                                   unsigned* __restrict__ start, unsigned* __restrict__ end) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned k = keys[i];
  if (k >= invalid) return;
  if (i == 0 || keys[i - 1] != k) start[k] = (unsigned)i;
  if (i == n - 1 || keys[i + 1] != k) end[k] = (unsigned)(i + 1);
}

struct Values {
  const float* v;         // channel c of source p of item b: v[b * item + p * pix + c * ch], c < C
  long long item;
  int pix, ch, C;
  const float* extra;     // optional channel C: extra[b * HW + p] (the importance 1 / p_z)
};

// One thread per target pixel.  Cells (tx, ty), (tx-1, ty), (tx, ty-1), (tx-1, ty-1) reach it through their NW, NE,
// SW, SE corner; within a cell, sources come in source order.  Per source: acc_c += (v_c e) w, acc_e += e w
// (the extension multiplies frame by exp(metric) before splatting).  out [B, NV, H, W] = acc / (acc_e + eps).
template <int NV>
__global__ void splat_gather_kernel(const float* __restrict__ ox, const float* __restrict__ oy,
                                    const float* __restrict__ e, const unsigned* __restrict__ order,
                                    const unsigned* __restrict__ start, const unsigned* __restrict__ end, Values val,
                                    int H, int W, float* __restrict__ out) {
  const int HW = H * W, b = blockIdx.y;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  const int tx = p % W, ty = p / W;
  const unsigned cells = (unsigned)(H + 1) * (W + 1);
  float acc[NV + 1];
#pragma unroll
  for (int c = 0; c <= NV; ++c) acc[c] = 0.f;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int cx = tx - (q & 1), cy = ty - (q >> 1);
    const unsigned key = (unsigned)b * cells + (unsigned)(cy + 1) * (W + 1) + (unsigned)(cx + 1);
    const unsigned i1 = end[key];
    const float fx0 = (float)cx, fx1 = (float)(cx + 1), fy0 = (float)cy, fy1 = (float)(cy + 1);
    for (unsigned i = start[key]; i < i1; ++i) {
      const unsigned s = order[i];
      const float x = ox[s], y = oy[s], ee = e[s];
      const float wx = (q & 1) ? __fsub_rn(x, fx0) : __fsub_rn(fx1, x);
      const float wy = (q >> 1) ? __fsub_rn(y, fy0) : __fsub_rn(fy1, y);
      const float w = __fmul_rn(wx, wy);
      const long long sp = (long long)s - (long long)b * HW;
      const float* v = val.v + b * val.item + sp * val.pix;
#pragma unroll
      for (int c = 0; c < NV; ++c) {
        const float vc = (val.extra && c == val.C) ? val.extra[s] : (c < val.C ? v[c * val.ch] : 0.f);
        acc[c] = __fadd_rn(acc[c], __fmul_rn(__fmul_rn(vc, ee), w));
      }
      acc[NV] = __fadd_rn(acc[NV], __fmul_rn(ee, w));
    }
  }
  const float den = __fadd_rn(acc[NV], kSplatEps);
  float* o = out + (long long)b * NV * HW + p;
#pragma unroll
  for (int c = 0; c < NV; ++c) o[(long long)c * HW] = __fdiv_rn(acc[c], den);
}

// kornia.filters.spatial_gradient(mode='sobel', normalized=False) on a replicate-padded plane, then
// exp(-beta sqrt(gx^2 + gy^2)).  FROM_DISP: the plane is (1 / disp) / 10 (render_source_vv.py:285-287), and the
// kernel also writes the splat's source: rgba = [img * 255, alpha] and depth = 1 / disp.  grid (cdiv(HW), N)
template <bool FROM_DISP>
__global__ void sobel_kernel(const float* __restrict__ x, int H, int W, float beta, float* __restrict__ alpha,
                             const float* __restrict__ img, float4* __restrict__ rgba, float* __restrict__ depth) {
  const int HW = H * W;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  const int px = p % W, py = p / W;
  const float* plane = x + (long long)blockIdx.y * HW;
  float a[3][3];
#pragma unroll
  for (int j = 0; j < 3; ++j)
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const int yy = min(max(py + j - 1, 0), H - 1), xx = min(max(px + i - 1, 0), W - 1);
      const float v = plane[yy * W + xx];
      a[j][i] = FROM_DISP ? __fdiv_rn(__fdiv_rn(1.f, v), 10.f) : v;
    }
  const float gx = (a[0][2] - a[0][0]) + 2.f * (a[1][2] - a[1][0]) + (a[2][2] - a[2][0]);
  const float gy = (a[2][0] - a[0][0]) + 2.f * (a[2][1] - a[0][1]) + (a[2][2] - a[0][2]);
  const float al = expf(-beta * sqrtf(gx * gx + gy * gy));
  if (FROM_DISP) {
    rgba[p] = make_float4(__fmul_rn(img[3 * p], 255.f), __fmul_rn(img[3 * p + 1], 255.f),
                          __fmul_rn(img[3 * p + 2], 255.f), al);
    depth[p] = __fdiv_rn(1.f, x[p]);
  } else {
    alpha[(long long)blockIdx.y * HW + p] = al;
  }
}

// render_source_vv.py:313-329 on the splatted rgba F [V, 4, H, W]: mask = erosion(F_a > 0.5) with the 3x3 cross
// (edge replicated), out [V, H, W, 3] = uint8(255 clip(clip(F_rgb / 255, 0, 1) mask, 0, 1)), truncating.
__global__ void quantise_kernel(const float* __restrict__ F, int H, int W, uint8_t* __restrict__ out) {
  const int HW = H * W;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  const int px = p % W, py = p / W;
  const float* f = F + (long long)blockIdx.y * 4 * HW;
  const float* fa = f + 3 * HW;
  const bool m = fa[p] > 0.5f && fa[max(py - 1, 0) * W + px] > 0.5f && fa[min(py + 1, H - 1) * W + px] > 0.5f &&
                 fa[py * W + max(px - 1, 0)] > 0.5f && fa[py * W + min(px + 1, W - 1)] > 0.5f;
  uint8_t* o = out + ((long long)blockIdx.y * HW + p) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float r = fminf(fmaxf(__fdiv_rn(f[c * HW + p], 255.f), 0.f), 1.f);
    o[c] = m ? (uint8_t)__fmul_rn(255.f, r) : (uint8_t)0;
  }
}

// ---- workspace: per-source arrays, two key / index buffers, cell ranges, the sort's temporary storage -----------
int key_bits(long long invalid) {
  int bits = 1;
  while ((1ll << bits) <= invalid) ++bits;
  return bits;
}

size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }

struct SplatWs {
  float *ox, *oy, *imp, *e;
  unsigned *keys, *keys_sorted, *idx, *order, *start, *end;
  void* sort_tmp;
  size_t sort_bytes, total;
};

// NULL base: sizes only
int splat_ws(int B, int H, int W, void* base, SplatWs* w) {
  const size_t n = (size_t)B * H * W, cells = (size_t)B * (H + 1) * (W + 1);
  size_t sort_bytes = 0;
  cudaError_t err = cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (unsigned*)nullptr, (unsigned*)nullptr,
                                                    (unsigned*)nullptr, (unsigned*)nullptr, (int)n, 0,
                                                    key_bits((long long)cells));
  if (err != cudaSuccess) return fail(DYN_E_CUDA, "splat: radix sort size query: %s", cudaGetErrorString(err));
  char* p = (char*)base;
  size_t off = 0;
  auto take = [&](size_t bytes) { void* r = p ? p + off : nullptr; off += align256(bytes); return r; };
  w->ox = (float*)take(n * 4);
  w->oy = (float*)take(n * 4);
  w->imp = (float*)take(n * 4);
  w->e = (float*)take(n * 4);
  w->keys = (unsigned*)take(n * 4);
  w->keys_sorted = (unsigned*)take(n * 4);
  w->idx = (unsigned*)take(n * 4);
  w->order = (unsigned*)take(n * 4);
  w->start = (unsigned*)take(cells * 4 * 2);
  w->end = w->start ? w->start + cells : nullptr;
  w->sort_tmp = take(sort_bytes);
  w->sort_bytes = sort_bytes;
  w->total = off;
  return DYN_OK;
}

bool splat_shape_ok(long long B, long long H, long long W) {
  // keys, source indices and sorted positions are 32-bit; the sort takes an int count; items are grid.y
  return B >= 1 && B < 65536 && H >= 1 && W >= 1 && B * (H + 1) * (W + 1) < (1ll << 31) && B * H * W < (1ll << 31);
}

// sort + ranges + gather, after a front kernel filled ox, oy, e, keys, idx
int splat_tail(const SplatWs& w, int B, int H, int W, const Values& val, int NV, float* out, cudaStream_t st) {
  const long long n = (long long)B * H * W, cells = (long long)B * (H + 1) * (W + 1);
  size_t tmp = w.sort_bytes;
  DYN_CUDA(cub::DeviceRadixSort::SortPairs(w.sort_tmp, tmp, w.keys, w.keys_sorted, w.idx, w.order, (int)n, 0,
                                           key_bits(cells), st));
  ++g_launches;
  DYN_CUDA(cudaMemsetAsync(w.start, 0, (size_t)cells * 2 * sizeof(unsigned), st));
  cell_ranges_kernel<<<cdiv(n, 256), 256, 0, st>>>(w.keys_sorted, n, (unsigned)cells, w.start, w.end);
  DYN_LAUNCH_CHECK();
  const dim3 grid(cdiv((long long)H * W, 128), B);
  switch (NV) {
#define DYN_SPLAT_CASE(k) \
  case k: splat_gather_kernel<k><<<grid, 128, 0, st>>>(w.ox, w.oy, w.e, w.order, w.start, w.end, val, H, W, out); break;
    DYN_SPLAT_CASE(1) DYN_SPLAT_CASE(2) DYN_SPLAT_CASE(3) DYN_SPLAT_CASE(4)
    DYN_SPLAT_CASE(5) DYN_SPLAT_CASE(6) DYN_SPLAT_CASE(7) DYN_SPLAT_CASE(8)
#undef DYN_SPLAT_CASE
    default: return fail(DYN_E_INVALID, "splat: %d channels (1..%d supported)", NV, kMaxValues);
  }
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int check_ws(const char* what, void* workspace, size_t have, size_t need) {
  if (workspace == nullptr || have < need)
    return fail(DYN_E_WORKSPACE, "%s: workspace of %zu bytes, %zu needed", what, have, need);
  return DYN_OK;
}

}  // namespace
}  // namespace dyn

using namespace dyn;

extern "C" {

size_t dyn_splat_workspace_bytes(int B, int H, int W) {
  if (!splat_shape_ok(B, H, W)) return 0;
  SplatWs w;
  return splat_ws(B, H, W, nullptr, &w) == DYN_OK ? w.total : 0;
}

int dyn_splat_softmax(const float* frame, const float* flow, const float* metric, int B, int C, int H, int W,
                      float* out, void* workspace, size_t workspace_bytes, void* stream) {
  DYN_CHECK_ARG(frame && flow && metric && out && splat_shape_ok(B, H, W));
  DYN_CHECK_ARG(C >= 1 && C <= kMaxValues);
  SplatWs w;
  int rc = splat_ws(B, H, W, nullptr, &w);
  if (rc) return rc;
  if ((rc = check_ws("splat_softmax", workspace, workspace_bytes, w.total))) return rc;
  splat_ws(B, H, W, workspace, &w);
  cudaStream_t st = (cudaStream_t)stream;
  flow_prep_kernel<<<dim3(cdiv((long long)H * W, 256), B), 256, 0, st>>>(flow, metric, H, W, w.ox, w.oy, w.e, w.keys,
                                                                         w.idx);
  DYN_LAUNCH_CHECK();
  const long long HW = (long long)H * W;
  return splat_tail(w, B, H, W, Values{frame, C * HW, 1, (int)HW, C, nullptr}, C, out, st);
}

int dyn_forward_splat(const float* imgs, const float* depths, const float* cams, int B, int C, int H, int W, float* out,
                      void* workspace, size_t workspace_bytes, void* stream) {
  DYN_CHECK_ARG(imgs && depths && cams && out && splat_shape_ok(B, H, W));
  DYN_CHECK_ARG(C >= 1 && C + 1 <= kMaxValues);
  SplatWs w;
  int rc = splat_ws(B, H, W, nullptr, &w);
  if (rc) return rc;
  if ((rc = check_ws("forward_splat", workspace, workspace_bytes, w.total))) return rc;
  splat_ws(B, H, W, workspace, &w);
  cudaStream_t st = (cudaStream_t)stream;
  const long long HW = (long long)H * W;
  project_kernel<<<dim3(cdiv(HW, 256), B), 256, 0, st>>>(depths, HW, cams, H, W, w.ox, w.oy, w.imp, w.keys, w.idx);
  DYN_LAUNCH_CHECK();
  importance_exp_kernel<<<B, kMinMaxThreads, 0, st>>>(w.imp, (int)HW, w.e);
  DYN_LAUNCH_CHECK();
  return splat_tail(w, B, H, W, Values{imgs, C * HW, C, 1, C, w.imp}, C + 1, out, st);
}

int dyn_sobel_alpha(const float* x, int N, int H, int W, float beta, float* alpha, void* stream) {
  DYN_CHECK_ARG(x && alpha && N >= 1 && H >= 1 && W >= 1 && (long long)H * W < (1ll << 31) && N < 65536);
  sobel_kernel<false><<<dim3(cdiv((long long)H * W, 256), N), 256, 0, (cudaStream_t)stream>>>(
      x, H, W, beta, alpha, nullptr, nullptr, nullptr);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

size_t dyn_virtual_views_workspace_bytes(int V, int H, int W) {
  const size_t splat = dyn_splat_workspace_bytes(V, H, W);
  if (splat == 0) return 0;
  const size_t HW = (size_t)H * W;
  return splat + align256(HW * 16) + align256(HW * 4) + align256((size_t)V * 4 * HW * 4);
}

int dyn_virtual_views(const float* img, const float* disp, const float* cams, int V, int H, int W, uint8_t* out,
                      void* workspace, size_t workspace_bytes, void* stream) {
  DYN_CHECK_ARG(img && disp && cams && out && splat_shape_ok(V, H, W));
  SplatWs w;
  int rc = splat_ws(V, H, W, nullptr, &w);
  if (rc) return rc;
  const size_t HW = (size_t)H * W;
  if ((rc = check_ws("virtual_views", workspace, workspace_bytes,
                     w.total + align256(HW * 16) + align256(HW * 4) + align256((size_t)V * 4 * HW * 4))))
    return rc;
  splat_ws(V, H, W, workspace, &w);
  char* p = (char*)workspace + w.total;
  float4* rgba = (float4*)p;
  float* depth = (float*)(p + align256(HW * 16));
  float* F = (float*)(p + align256(HW * 16) + align256(HW * 4));
  cudaStream_t st = (cudaStream_t)stream;
  const int gx = cdiv((long long)HW, 256);
  sobel_kernel<true><<<dim3(gx, 1), 256, 0, st>>>(disp, H, W, 0.5f, nullptr, img, rgba, depth);
  DYN_LAUNCH_CHECK();
  project_kernel<<<dim3(gx, V), 256, 0, st>>>(depth, 0, cams, H, W, w.ox, w.oy, w.imp, w.keys, w.idx);
  DYN_LAUNCH_CHECK();
  importance_exp_kernel<<<V, kMinMaxThreads, 0, st>>>(w.imp, (int)HW, w.e);
  DYN_LAUNCH_CHECK();
  // the splat's 1 / p_z channel has no use here: only rgba is splatted (each channel's sums are independent)
  rc = splat_tail(w, V, H, W, Values{(const float*)rgba, 0, 4, 1, 4, nullptr}, 4, F, st);
  if (rc) return rc;
  quantise_kernel<<<dim3(gx, V), 256, 0, st>>>(F, H, W, out);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

}  // extern "C"
