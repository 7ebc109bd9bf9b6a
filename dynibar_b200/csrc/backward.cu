// First slice of the training backward (row f2): the two non-MLP ends of the path.
//
//   dyn_composite_backward       raw2outputs (render_ray.py:214-330): gradients of the 11-key output dict
//                                 w.r.t. raw_dy / raw_st [R,S,4] (colours and densities of both nets)
//   dyn_project_gather_backward  Projector.compute_with_motions (projection.py:103-176): gradient of the
//                                 gathered rgb_feat w.r.t. the source feature maps (F.grid_sample backward,
//                                 bilinear, zero padding, align_corners=True) and w.r.t. the (motion-displaced)
//                                 sample points through the projection
//   dyn_traj_combine_grad_d      gradient of the trajectory displacements w.r.t. the trajectory-basis rows
//                                 (deterministic two-stage reduction over all points)
//   dyn_expected_scene_flow      exp_sf of the mv fine pass (render_ray.py:585-595), forward and backward
//
// fp32 throughout; one warp per ray for the compositing scan (reverse multiplicative scan for the
// transmittance), atomicAdd scatter for the feature-map gradient.  The MLP / ray-transformer backward is not
// built yet (DESIGN.md, "next").
#include "common.cuh"
#include "geometry.cuh"

namespace dyn {

namespace {

__device__ __forceinline__ float warp_sum_b(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// exclusive suffix sum inside the warp: lane i gets sum_{j > i} v_j
__device__ __forceinline__ float warp_suffix_excl(float v, int lane) {
  float s = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_down_sync(0xffffffffu, s, o);
    if (lane + o < 32) s += t;
  }
  return s - v;
}
__device__ __forceinline__ float warp_scan_mul_b(float v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v *= t;
  }
  return v;
}

constexpr int kMaxSeg = 8;  // S <= 256

// g_rays [R,11]: d/d(rgb 3, rgb_static 3, rgb_dy 3, depth, mask(ignored)); g_samples [5,R,S]:
// d/d(alpha_dy, weights_dy, weights_st, alpha, weights) or null.
// vanilla (raw2outputs_vanilla, render_ray.py:134-211 == the same compositing with no second net: raw_b = null):
// g_rays [R,5] = d/d(rgb 3, depth, mask(ignored)), g_samples [2,R,S] = d/d(weights, alpha) or null.
__global__ void composite_backward_kernel(const float* __restrict__ raw_a, const float* __restrict__ raw_b,
                                          const float* __restrict__ z_vals, const float* __restrict__ g_rays,
                                          const float* __restrict__ g_samples, int R, int S,
                                          float* __restrict__ g_raw_a, float* __restrict__ g_raw_b, int vanilla) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= R) return;
  const long long RS = (long long)R * S;
  const int nseg = (S + 31) / 32;
  const float* gr = g_rays + (long long)r * (vanilla ? 5 : 11);
  const float gA[3] = {vanilla ? gr[0] : gr[0] + gr[6], vanilla ? gr[1] : gr[1] + gr[7],
                       vanilla ? gr[2] : gr[2] + gr[8]};  // d/d c_dy weights: rgb + rgb_dy
  const float gB[3] = {vanilla ? 0.f : gr[0] + gr[3], vanilla ? 0.f : gr[1] + gr[4],
                       vanilla ? 0.f : gr[2] + gr[5]};    // rgb + rgb_static
  const float gdepth = vanilla ? gr[3] : gr[9];
  // forward quantities per (segment, lane)
  float aA[kMaxSeg], aB[kMaxSeg], T[kMaxSeg], G[kMaxSeg];
  float carry = 1.f;
  for (int sg = 0; sg < nseg; ++sg) {
    const int s = sg * 32 + lane;
    const bool ok = s < S;
    const long long p = (long long)r * S + (ok ? s : 0);
    const float sa = ok ? raw_a[p * 4 + 3] : 0.f, sb = (ok && !vanilla) ? raw_b[p * 4 + 3] : 0.f;
    const float delta = (s == S - 1) ? 1e10f : 1.f;
    aA[sg] = ok ? 1.f - expf(-softplus_f(sa) * delta) : 0.f;
    aB[sg] = (ok && !vanilla) ? 1.f - expf(-softplus_f(sb) * delta) : 0.f;
    const float al = 1.f - (1.f - aB[sg]) * (1.f - aA[sg]);
    const float f = ok ? (1.f - al + 1e-10f) : 1.f;
    const float inc = warp_scan_mul_b(f, lane);
    const float excl = __shfl_up_sync(0xffffffffu, inc, 1);
    T[sg] = carry * (lane == 0 ? 1.f : excl);
    carry *= __shfl_sync(0xffffffffu, inc, 31);
  }
  // backward: suffix sums of G_s T_s, segments from the last to the first
  float tail = 0.f;  // sum over all samples of later segments
  for (int sg = nseg - 1; sg >= 0; --sg) {
    const int s = sg * 32 + lane;
    const bool ok = s < S;
    const long long p = (long long)r * S + (ok ? s : 0);
    float4 ca = make_float4(0.f, 0.f, 0.f, 0.f), cb = ca;
    float z = 0.f;
    if (ok) {
      ca = reinterpret_cast<const float4*>(raw_a)[p];
      if (!vanilla) cb = reinterpret_cast<const float4*>(raw_b)[p];
      z = z_vals[p];
    }
    const bool gs_ok = ok && g_samples != nullptr;
    const float gs_aA = (gs_ok && !vanilla) ? g_samples[0 * RS + p] : 0.f;
    const float gs_wA = (gs_ok && !vanilla) ? g_samples[1 * RS + p] : 0.f;
    const float gs_wB = (gs_ok && !vanilla) ? g_samples[2 * RS + p] : 0.f;
    const float gs_al = gs_ok ? g_samples[(vanilla ? 1 : 3) * RS + p] : 0.f;
    const float gs_w = gs_ok ? g_samples[(vanilla ? 0 : 4) * RS + p] : 0.f;
    const float al = 1.f - (1.f - aB[sg]) * (1.f - aA[sg]);
    const float dwA = gs_wA + gA[0] * ca.x + gA[1] * ca.y + gA[2] * ca.z;   // dL/d w_dy
    const float dwB = gs_wB + gB[0] * cb.x + gB[1] * cb.y + gB[2] * cb.z;   // dL/d w_st
    const float dw = gs_w + gdepth * z;                                       // dL/d w
    G[sg] = ok ? (dwA * aA[sg] + dwB * aB[sg] + dw * al) : 0.f;              // dL/d T_s
    const float gt = G[sg] * T[sg];
    const float suf = warp_suffix_excl(gt, lane) + tail;  // sum_{s' > s} G T
    tail += warp_sum_b(gt);
    if (ok) {
      const float f = 1.f - al + 1e-10f;
      const float dal = gs_al + dw * T[sg] - suf / f;                          // dL/d alpha
      const float daA = gs_aA + dwA * T[sg] + dal * (1.f - aB[sg]);
      const float daB = dwB * T[sg] + dal * (1.f - aA[sg]);
      const float delta = (s == S - 1) ? 1e10f : 1.f;
      // d alpha / d sigma = exp(-softplus(sigma) delta) * delta * sigmoid(sigma)   (0 where the exp underflows)
      const float ea = 1.f - aA[sg], eb = 1.f - aB[sg];
      const float dsa = ea > 0.f ? daA * ea * delta * sigmoid_f(ca.w) : 0.f;
      const float dsb = eb > 0.f ? daB * eb * delta * sigmoid_f(cb.w) : 0.f;
      const float wA = aA[sg] * T[sg], wB = aB[sg] * T[sg];
      reinterpret_cast<float4*>(g_raw_a)[p] = make_float4(gA[0] * wA, gA[1] * wA, gA[2] * wA, dsa);
      if (!vanilla) reinterpret_cast<float4*>(g_raw_b)[p] = make_float4(gB[0] * wB, gB[1] * wB, gB[2] * wB, dsb);
    }
  }
}

// one thread per (view, point): scatter into the feature-map gradient (reference layout [V,C,h,w]) and
// accumulate d/d(u,v) -> d/d xyz of that view's displaced point.  g_feat [N,V,3+C] (rgb channels first).
__global__ void gather_backward_kernel(const float* __restrict__ xyz, const float* __restrict__ xyz_st,
                                       const float* __restrict__ featmaps, const float* __restrict__ rgbs,
                                       const float* __restrict__ g_feat, const __grid_constant__ ViewCams cams,
                                       int V, long long N, int H, int W, int C, int h, int w,
                                       float* __restrict__ g_maps, float* __restrict__ g_xyz) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N * V) return;
  const int v = (int)(idx / N);
  const long long pt = idx - (long long)v * N;
  const float* q = xyz != nullptr ? xyz + idx * 3 : xyz_st + pt * 3;
  const float* P = cams.P[v];
  const float px = P[0] * q[0] + P[1] * q[1] + P[2] * q[2] + P[3];
  const float py = P[4] * q[0] + P[5] * q[1] + P[6] * q[2] + P[7];
  const float pz = P[8] * q[0] + P[9] * q[1] + P[10] * q[2] + P[11];
  const float d = fmaxf(pz, 1e-8f);
  const float u0 = px / d, v0 = py / d;
  const float u = fminf(fmaxf(u0, -1e6f), 1e6f), vv = fminf(fmaxf(v0, -1e6f), 1e6f);
  const float gx = 2.f * u / (cams.w_img - 1.f) - 1.f, gy = 2.f * vv / (cams.h_img - 1.f) - 1.f;
  const float* g = g_feat + (pt * V + v) * (long long)(3 + C);
  float dfx = 0.f, dfy = 0.f;   // dL/d(feature-map sample coordinates), in image-pixel units (via du, dv below)
  float du = 0.f, dv = 0.f;
  {  // deep features
    const float fx = (gx + 1.f) * 0.5f * (float)(w - 1), fy = (gy + 1.f) * 0.5f * (float)(h - 1);
    const float x0f = floorf(fx), y0f = floorf(fy);
    const int x0 = (int)x0f, y0 = (int)y0f;
    const float ax = fx - x0f, ay = fy - y0f, bx = (x0f + 1.f) - fx, by = (y0f + 1.f) - fy;
    const bool in00 = x0 >= 0 && x0 < w && y0 >= 0 && y0 < h, in01 = x0 + 1 >= 0 && x0 + 1 < w && y0 >= 0 && y0 < h;
    const bool in10 = x0 >= 0 && x0 < w && y0 + 1 >= 0 && y0 + 1 < h, in11 = x0 + 1 >= 0 && x0 + 1 < w && y0 + 1 >= 0 && y0 + 1 < h;
    for (int c = 0; c < C; ++c) {
      const float gc = g[3 + c];
      const long long base = ((long long)v * C + c) * h * w;
      float m00 = 0.f, m01 = 0.f, m10 = 0.f, m11 = 0.f;
      if (in00) { m00 = featmaps[base + (long long)y0 * w + x0]; if (g_maps) atomicAdd(g_maps + base + (long long)y0 * w + x0, gc * bx * by); }
      if (in01) { m01 = featmaps[base + (long long)y0 * w + x0 + 1]; if (g_maps) atomicAdd(g_maps + base + (long long)y0 * w + x0 + 1, gc * ax * by); }
      if (in10) { m10 = featmaps[base + (long long)(y0 + 1) * w + x0]; if (g_maps) atomicAdd(g_maps + base + (long long)(y0 + 1) * w + x0, gc * bx * ay); }
      if (in11) { m11 = featmaps[base + (long long)(y0 + 1) * w + x0 + 1]; if (g_maps) atomicAdd(g_maps + base + (long long)(y0 + 1) * w + x0 + 1, gc * ax * ay); }
      dfx += gc * ((m01 - m00) * by + (m11 - m10) * ay);
      dfy += gc * ((m10 - m00) * bx + (m11 - m01) * ax);
    }
    du += dfx * (float)(w - 1) / (cams.w_img - 1.f);
    dv += dfy * (float)(h - 1) / (cams.h_img - 1.f);
  }
  {  // colours ([V,H,W,3], sampled at image resolution); no gradient to the images themselves
    const float fx = (gx + 1.f) * 0.5f * (float)(W - 1), fy = (gy + 1.f) * 0.5f * (float)(H - 1);
    const float x0f = floorf(fx), y0f = floorf(fy);
    const int x0 = (int)x0f, y0 = (int)y0f;
    const float ax = fx - x0f, ay = fy - y0f, bx = (x0f + 1.f) - fx, by = (y0f + 1.f) - fy;
    float ex = 0.f, ey = 0.f;
    for (int c = 0; c < 3; ++c) {
      const float gc = g[c];
      auto tap = [&](int xi, int yi) {
        return (xi >= 0 && xi < W && yi >= 0 && yi < H) ? rgbs[(((long long)v * H + yi) * W + xi) * 3 + c] : 0.f;
      };
      const float m00 = tap(x0, y0), m01 = tap(x0 + 1, y0), m10 = tap(x0, y0 + 1), m11 = tap(x0 + 1, y0 + 1);
      ex += gc * ((m01 - m00) * by + (m11 - m10) * ay);
      ey += gc * ((m10 - m00) * bx + (m11 - m01) * ax);
    }
    du += ex * (float)(W - 1) / (cams.w_img - 1.f);
    dv += ey * (float)(H - 1) / (cams.h_img - 1.f);
  }
  if (g_xyz != nullptr) {
    // u = clamp(px / clamp(pz, min=1e-8), -1e6, 1e6) (projection.py:51-55): no gradient through an active
    // outer clamp, none through pz where the inner clamp is active
    const float live = pz > 1e-8f ? 1.f : 0.f;
    const float su = fabsf(u0) <= 1e6f ? du / d : 0.f, sv = fabsf(v0) <= 1e6f ? dv / d : 0.f;
    float* o = g_xyz + idx * 3;
#pragma unroll
    for (int k = 0; k < 3; ++k)
      o[k] = su * (P[k] - live * u0 * P[8 + k]) + sv * (P[4 + k] - live * v0 * P[8 + k]);
  }
}

// Trajectory combination (compute_traj_pts + the displacements built from it, render_ray.py:361-369, :462-500,
// :1101-1176): out[i, p, a] = (base ? base[p, a] : 0) + sum_k coeff[p, a nb + k] D[i, k], where a row of D is a
// difference of two rows of the DCT trajectory basis.  Linear in coeff and base.
__global__ void traj_combine_kernel(const float* __restrict__ coeff, const float* __restrict__ D,
                                    const float* __restrict__ base, int n, int nb, long long P,
                                    float* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)n * P * 3) return;
  const int a = (int)(idx % 3);
  const long long t = idx / 3;
  const long long p = t % P;
  const int i = (int)(t / P);
  float s = base != nullptr ? base[p * 3 + a] : 0.f;
  for (int k = 0; k < nb; ++k) s = fmaf(coeff[p * 3 * nb + a * nb + k], D[i * nb + k], s);
  out[idx] = s;
}

__global__ void traj_combine_bwd_kernel(const float* __restrict__ g_out, const float* __restrict__ D, int n, int nb,
                                        long long P, float* __restrict__ g_coeff, float* __restrict__ g_base) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= P * 3) return;
  const long long p = idx / 3;
  const int a = (int)(idx - p * 3);
  float gb = 0.f;
  float gc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int i = 0; i < n; ++i) {
    const float g = g_out[((long long)i * P + p) * 3 + a];
    gb += g;
    for (int k = 0; k < nb; ++k) gc[k] = fmaf(g, D[i * nb + k], gc[k]);
  }
  if (g_base != nullptr) g_base[idx] = gb;
  if (g_coeff != nullptr)
    for (int k = 0; k < nb; ++k) g_coeff[p * 3 * nb + a * nb + k] = gc[k];
}

// Gradient of traj_combine w.r.t. the basis-difference rows: gD[i, k] = sum_p sum_a g_out[i, p, a] coeff[p, a nb + k],
// a reduction over all P points.  Stage 1: block b owns points [b kGdPts, (b + 1) kGdPts) and writes its partial sums
// partial[b, i, k]; stage 2 adds the partials of every block in block order.  Each thread, lane and warp always covers
// the same points in the same order, so the result does not depend on scheduling (no float atomics): two calls on the
// same inputs give the same bits.
constexpr int kGdThreads = 256;
constexpr int kGdPts = 1024;  // points per block (4 per thread)

__global__ void __launch_bounds__(kGdThreads) traj_grad_d_partial_kernel(const float* __restrict__ g_out,
                                                                       const float* __restrict__ coeff, int n, int nb,
                                                                       long long P, float* __restrict__ partial) {
  __shared__ float red[kGdThreads / 32][8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long p0 = (long long)blockIdx.x * kGdPts;
  const long long p1 = min(P, p0 + kGdPts);
  for (int i = 0; i < n; ++i) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (long long p = p0 + tid; p < p1; p += kGdThreads) {
      const float* g = g_out + ((long long)i * P + p) * 3;
      const float* c = coeff + p * 3 * nb;
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        const float ga = g[a];
#pragma unroll
        for (int k = 0; k < 8; ++k)
          if (k < nb) acc[k] = fmaf(ga, c[a * nb + k], acc[k]);
      }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = warp_sum_b(acc[k]);
    if (lane == 0)
#pragma unroll
      for (int k = 0; k < 8; ++k) red[warp][k] = acc[k];
    __syncthreads();
    if (tid < nb) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < kGdThreads / 32; ++w) s += red[w][tid];
      partial[((long long)blockIdx.x * n + i) * nb + tid] = s;
    }
    __syncthreads();
  }
}

__global__ void traj_grad_d_sum_kernel(const float* __restrict__ partial, int blocks, int n, int nb,
                                       float* __restrict__ g_D) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n * nb) return;
  float s = 0.f;
  for (int b = 0; b < blocks; ++b) s += partial[(long long)b * n * nb + j];
  g_D[j] = s;
}

// Expected scene flow (render_ray.py:585-595): exp_sf[r, a] = max(sum_s w[r, s] sf[0, r, s, a],
// sum_s w[r, s] sf[1, r, s, a]) with sf = (traj(f + k) - traj(f), traj(f - k) - traj(f)).  One warp per ray; forward
// and backward form the two sums with the same code, so the backward sees the forward's ties.
__device__ __forceinline__ void exp_sf_sums(const float* __restrict__ w, const float* __restrict__ sf, int r, int R,
                                            int S, int lane, float ep[3], float em[3]) {
  const long long N = (long long)R * S;
  for (int a = 0; a < 3; ++a) ep[a] = em[a] = 0.f;
  for (int s = lane; s < S; s += 32) {
    const long long ps = (long long)r * S + s;
    const float wv = w[ps];
    const float* p = sf + ps * 3;
    const float* m = sf + (N + ps) * 3;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      ep[a] = fmaf(wv, p[a], ep[a]);
      em[a] = fmaf(wv, m[a], em[a]);
    }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    ep[a] = warp_sum_b(ep[a]);
    em[a] = warp_sum_b(em[a]);
  }
}

__global__ void exp_sf_kernel(const float* __restrict__ w, const float* __restrict__ sf, int R, int S,
                              float* __restrict__ exp_sf) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= R) return;
  float ep[3], em[3];
  exp_sf_sums(w, sf, r, R, S, lane, ep, em);
  if (lane < 3) exp_sf[r * 3 + lane] = fmaxf(ep[lane], em[lane]);
}

// torch.max(p, m) backward: the larger side takes the gradient; at a tie each side takes half of it.
__global__ void exp_sf_bwd_kernel(const float* __restrict__ w, const float* __restrict__ sf,
                                  const float* __restrict__ g_exp, int R, int S, float* __restrict__ g_w,
                                  float* __restrict__ g_sf) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= R) return;
  const long long N = (long long)R * S;
  float ep[3], em[3], gp[3], gm[3];
  exp_sf_sums(w, sf, r, R, S, lane, ep, em);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float g = g_exp[r * 3 + a];
    gp[a] = ep[a] > em[a] ? g : (ep[a] == em[a] ? 0.5f * g : 0.f);
    gm[a] = em[a] > ep[a] ? g : (ep[a] == em[a] ? 0.5f * g : 0.f);
  }
  for (int s = lane; s < S; s += 32) {
    const long long ps = (long long)r * S + s;
    const float* p = sf + ps * 3;
    const float* m = sf + (N + ps) * 3;
    if (g_w != nullptr)
      g_w[ps] = gp[0] * p[0] + gp[1] * p[1] + gp[2] * p[2] + gm[0] * m[0] + gm[1] * m[1] + gm[2] * m[2];
    if (g_sf != nullptr) {
      const float wv = w[ps];
      float* op = g_sf + ps * 3;
      float* om = g_sf + (N + ps) * 3;
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        op[a] = wv * gp[a];
        om[a] = wv * gm[a];
      }
    }
  }
}

}  // namespace
}  // namespace dyn

using namespace dyn;

extern "C" {

int dyn_composite_backward(const float* raw_dy, const float* raw_st, const float* z_vals, const float* g_rays,
                           const float* g_samples, int R, int S, float* g_raw_dy, float* g_raw_st, void* stream) {
  if (R == 0) return DYN_OK;
  DYN_CHECK_ARG(raw_dy && raw_st && z_vals && g_rays && g_raw_dy && g_raw_st && S >= 1);
  if (S > 32 * kMaxSeg) return fail(DYN_E_INVALID, "composite backward supports S <= %d (got %d)", 32 * kMaxSeg, S);
  composite_backward_kernel<<<cdiv((long long)R * 32, 128), 128, 0, (cudaStream_t)stream>>>(
      raw_dy, raw_st, z_vals, g_rays, g_samples, R, S, g_raw_dy, g_raw_st, 0);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int dyn_composite_vanilla_backward(const float* raw, const float* z_vals, const float* g_rays, const float* g_samples,
                                   int R, int S, float* g_raw, void* stream) {
  if (R == 0) return DYN_OK;
  DYN_CHECK_ARG(raw && z_vals && g_rays && g_raw && S >= 1);
  if (S > 32 * kMaxSeg) return fail(DYN_E_INVALID, "composite backward supports S <= %d (got %d)", 32 * kMaxSeg, S);
  composite_backward_kernel<<<cdiv((long long)R * 32, 128), 128, 0, (cudaStream_t)stream>>>(
      raw, nullptr, z_vals, g_rays, g_samples, R, S, g_raw, nullptr, 1);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int dyn_project_gather_backward(const float* xyz_st, const float* xyz, const float* src_rgbs, const float* src_cams,
                                const float* featmaps, const float* g_rgb_feat, int V, int R, int S, int H, int W, int C,
                                int h, int w, float* g_featmaps, float* g_xyz, void* stream) {
  if (R == 0) return DYN_OK;
  DYN_CHECK_ARG(xyz_st && src_rgbs && src_cams && featmaps && g_rgb_feat && (g_featmaps || g_xyz));
  cudaStream_t st = (cudaStream_t)stream;
  ViewCams vc;
  int rc = build_view_cams(src_cams, V, nullptr, st, &vc);
  if (rc) return rc;
  const long long N = (long long)R * S;
  if (g_featmaps) DYN_CUDA(cudaMemsetAsync(g_featmaps, 0, (size_t)V * C * h * w * sizeof(float), st));
  gather_backward_kernel<<<cdiv(N * V, 256), 256, 0, st>>>(xyz, xyz_st, featmaps, src_rgbs, g_rgb_feat, vc, V, N, H, W,
                                                           C, h, w, g_featmaps, g_xyz);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int dyn_traj_combine(const float* coeff, const float* D, const float* base, int n, int nb, int P, float* out,
                     void* stream) {
  if (P == 0 || n == 0) return DYN_OK;
  DYN_CHECK_ARG(coeff && D && out && n >= 1 && nb >= 1 && nb <= 8 && P >= 0);
  traj_combine_kernel<<<cdiv((long long)n * P * 3, 256), 256, 0, (cudaStream_t)stream>>>(coeff, D, base, n, nb, P, out);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int dyn_traj_combine_backward(const float* g_out, const float* D, int n, int nb, int P, float* g_coeff, float* g_base,
                              void* stream) {
  if (P == 0) return DYN_OK;
  DYN_CHECK_ARG(g_out && D && n >= 1 && nb >= 1 && nb <= 8 && P >= 0 && (g_coeff || g_base));
  traj_combine_bwd_kernel<<<cdiv((long long)P * 3, 256), 256, 0, (cudaStream_t)stream>>>(g_out, D, n, nb, P, g_coeff,
                                                                                       g_base);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

size_t dyn_traj_combine_grad_d_workspace_bytes(int n, int nb, int P) {
  if (n <= 0 || nb <= 0 || P <= 0) return 0;
  return (size_t)cdiv((long long)P, kGdPts) * n * nb * sizeof(float);
}

int dyn_traj_combine_grad_d(const float* g_out, const float* coeff, int n, int nb, int P, float* g_D, void* workspace,
                            size_t workspace_bytes, void* stream) {
  DYN_CHECK_ARG(g_D && n >= 1 && nb >= 1 && nb <= 8 && P >= 0);
  cudaStream_t st = (cudaStream_t)stream;
  if (P == 0) {
    DYN_CUDA(cudaMemsetAsync(g_D, 0, (size_t)n * nb * sizeof(float), st));
    return DYN_OK;
  }
  DYN_CHECK_ARG(g_out && coeff && workspace);
  if (workspace_bytes < dyn_traj_combine_grad_d_workspace_bytes(n, nb, P))
    return fail(DYN_E_INVALID, "traj_combine_grad_d: workspace of %zu bytes, %zu needed", workspace_bytes,
                dyn_traj_combine_grad_d_workspace_bytes(n, nb, P));
  const int blocks = (int)cdiv((long long)P, kGdPts);
  float* partial = (float*)workspace;
  traj_grad_d_partial_kernel<<<blocks, kGdThreads, 0, st>>>(g_out, coeff, n, nb, P, partial);
  DYN_LAUNCH_CHECK();
  traj_grad_d_sum_kernel<<<cdiv((long long)n * nb, 128), 128, 0, st>>>(partial, blocks, n, nb, g_D);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int dyn_expected_scene_flow(const float* weights, const float* sf, int R, int S, float* exp_sf, void* stream) {
  if (R == 0) return DYN_OK;
  DYN_CHECK_ARG(weights && sf && exp_sf && R > 0 && S >= 1);
  exp_sf_kernel<<<cdiv((long long)R * 32, 256), 256, 0, (cudaStream_t)stream>>>(weights, sf, R, S, exp_sf);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int dyn_expected_scene_flow_backward(const float* weights, const float* sf, const float* g_exp_sf, int R, int S,
                                     float* g_weights, float* g_sf, void* stream) {
  if (R == 0) return DYN_OK;
  DYN_CHECK_ARG(weights && sf && g_exp_sf && (g_weights || g_sf) && R > 0 && S >= 1);
  exp_sf_bwd_kernel<<<cdiv((long long)R * 32, 256), 256, 0, (cudaStream_t)stream>>>(weights, sf, g_exp_sf, R, S,
                                                                                    g_weights, g_sf);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

}  // extern "C"
