// The monocular training criterion (row f2): every loss term of a DynibarMono step (train.py:187-196, :300-456;
// ibrnet/criterion.py; utils.py:32-39) as one forward and one backward entry point.
//
//   dyn_mono_loss           pass 1: one warp per ray adds the ray's share of every numerator and denominator; a block
//                           of 8 rays writes one row of partial sums.  pass 2: one block adds the rows in block order,
//                           forms component = numerator / denominator, applies the weights and writes the nine logged
//                           scalars, the components and the table weight / denominator for the backward.
//   dyn_mono_loss_rows / dyn_mono_loss_finish  the two passes as separate calls, so that a batch can be evaluated in
//                           ray slices: each slice writes its rows into one batch-wide buffer, finish runs once with
//                           the batch's dimensions (the same bits as dyn_mono_loss when slices start on a block).
//   dyn_mono_loss_backward  one warp per ray writes every requested gradient element exactly once; the upstream
//                           gradient is read from device memory.
//
// Each term has ONE device function giving the value and the derivative of an element's contribution; the forward
// uses the value, the backward the derivative, and the single-term entry points of dynibar_b200/criterion.py are
// the same kernels with one bit of `terms` set.  fp32, no float atomics: sums are shuffle trees inside a warp, warp
// order inside a block and block order across blocks, so the same inputs give the same bits.
#include "common.cuh"

namespace dyn {

namespace {

enum Term { T_RGB0 = 0, T_STATIC = 5, T_DISP = 6, T_FLOW = 7, T_CYCLE = 8, T_REG_ABS = 9, T_REG_TIME = 10,
            T_REG_SPACE = 11, T_ENTROPY = 12, T_DIST = 13, T_STATIC_DY = 14, kTerms = DYN_LOSS_TERMS };
constexpr int kAcc = 2 * kTerms;  // numerator 2k, denominator 2k + 1 of term k
constexpr int kWarps = 8;         // rays per block
constexpr int kOutComp = 9, kOutScale = 9 + kTerms;  // offsets in `out`, after the nine logged scalars
constexpr int kMaxDistSamples = 256;  // dist_n limit of the distortion term

struct Dims { int R, S, K, n_sf; };

__device__ __forceinline__ bool on(unsigned terms, int k) { return (terms >> k) & 1u; }
__device__ __forceinline__ float sgn(float x) { return (float)(x > 0.f) - (float)(x < 0.f); }
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_scan_add(float v, int lane) {  // inclusive
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  return v;
}

// ---- one function per term: v = the element's value, dv = d v / d (first argument) ---------------------------------
// utils.py:32-39 with eps = 0.001
__device__ __forceinline__ void charbonnier(float pred, float gt, float& v, float& dv) {
  const float d = pred - gt;
  v = sqrtf(d * d + 1e-6f);
  dv = d / v;
}
__device__ __forceinline__ void l1(float x, float y, float& v, float& dv) {
  const float d = x - y;
  v = fabsf(d);
  dv = sgn(d);
}
__device__ __forceinline__ void sq(float x, float y, float& v, float& dv) {
  const float d = x - y;
  v = d * d;
  dv = 2.f * d;
}
// train.py:332-340: |1 / clamp(depth, min=1e-2) - gt|; no gradient where the clamp is active
__device__ __forceinline__ void disparity(float depth, float gt, float& v, float& dv) {
  const float p = 1.f / fmaxf(depth, 1e-2f);
  const float d = p - gt;
  v = fabsf(d);
  dv = depth >= 1e-2f ? -sgn(d) * p * p : 0.f;
}
// train.py:406-408: rho = a / clamp(a + b, min=1e-9) and its derivatives (a, b: the ray's summed dynamic / static weights)
struct Ratio { float rho, d_dy, d_st; };
__device__ __forceinline__ Ratio weights_ratio(float a, float b) {
  const float c = fmaxf(a + b, 1e-9f);
  const float dc = (a + b >= 1e-9f) ? a / (c * c) : 0.f;
  return Ratio{a / c, 1.f / c - dc, -dc};
}
// train.py:409-412
__device__ __forceinline__ void entropy(float rho, float& v, float& dv) {
  const float p = rho + 1e-9f, q = 1.f - rho + 1e-9f;
  v = -(rho * logf(p) + (1.f - rho) * logf(q));
  dv = -(logf(p) + rho / p - logf(q) - (1.f - rho) / q);
}
// distortion (train.py:416-423) of sample i of a ray in its cumulative-sum form: exW / exWM are the exclusive, inW /
// inWM the inclusive prefix sums of w and w m at i, totW / totWM the ray's totals (the derivative needs the suffix
// sums: total - inclusive prefix)
__device__ __forceinline__ void distortion(float w, float m, float iv, float exW, float exWM, float inW, float inWM,
                                           float totW, float totWM, float& v, float& dv) {
  const float before = m * exW - exWM;  // sum_{j<i} w_j (m_i - m_j)
  v = 2.f * w * before + (1.f / 3.f) * iv * w * w;
  dv = 2.f * (before + (totWM - inWM) - m * (totW - inW)) + (2.f / 3.f) * iv * w;
}

// per-ray weight of an rgb slot
__device__ __forceinline__ float slot_weight(const dyn_loss_rgb_slot& sl, int r, float rho) {
  float m = sl.mask ? (sl.mask[r] ? 1.f : 0.f) : 1.f;
  if (sl.w0) m *= (sl.flags & DYN_LOSS_SLOT_COMPLEMENT_W0) ? 1.f - sl.w0[r] : sl.w0[r];
  if (sl.w1) m *= sl.w1[r];
  if (sl.flags & DYN_LOSS_SLOT_TIMES_ONE_MINUS_RATIO) m *= 1.f - rho;
  return m;
}
__device__ __forceinline__ float ray_mask(const dyn_mono_loss_inputs& in, int r) {
  return in.ray_mask ? (in.ray_mask[r] ? 1.f : 0.f) : 1.f;
}
// mid-point and interval of distortion sample i (either given or formed from s_vals, train.py:416-418)
__device__ __forceinline__ void dist_sample(const dyn_mono_loss_inputs& in, int r, int i, float& m, float& iv) {
  if (in.s_vals) {
    const float* s = in.s_vals + (long long)r * (in.dist_n + 1) + i;
    m = (s[1] + s[0]) * 0.5f;
    iv = s[1] - s[0];
  } else {
    m = in.dist_m[(long long)r * in.dist_n + i];
    iv = in.dist_interval[(long long)r * in.dist_n + i];
  }
}

// the ray's summed dynamic and static weights (each lane returns the warp's sums)
__device__ __forceinline__ void summed_weights(const dyn_mono_loss_inputs& in, int r, int lane, float& a, float& b) {
  a = b = 0.f;
  if (in.weights_dy == nullptr) return;
  for (int s = lane; s < in.S; s += 32) {
    a += in.weights_dy[(long long)r * in.S + s];
    if (in.weights_st) b += in.weights_st[(long long)r * in.S + s];
  }
  a = warp_sum(a);
  b = warp_sum(b);
}

__global__ void __launch_bounds__(kWarps * 32) mono_loss_kernel(const __grid_constant__ dyn_mono_loss_inputs in,
                                                                unsigned terms, float* __restrict__ partial) {
  __shared__ float sh[kWarps][kAcc];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * kWarps + warp;
  float* acc = sh[warp];
  for (int k = lane; k < kAcc; k += 32) acc[k] = 0.f;
  __syncwarp();
  if (r < in.R) {
    const int S = in.S, S3 = in.S * 3, R = in.R;
    float sum_dy, sum_st;
    summed_weights(in, r, lane, sum_dy, sum_st);
    const Ratio rt = weights_ratio(sum_dy, sum_st);
    // ---- the six rgb slots: lane k takes slot k
#pragma unroll
    for (int k = 0; k < DYN_LOSS_RGB_SLOTS; ++k) {
      if (lane == k && (on(terms, k) || (k == T_STATIC && on(terms, T_STATIC_DY)))) {
        const float m = slot_weight(in.rgb[k], r, rt.rho);
        if (on(terms, k)) {
          float num = 0.f, v, dv;
          for (int c = 0; c < 3; ++c) {
            charbonnier(in.rgb[k].pred[(long long)r * in.rgb[k].ld + c], in.gt_rgb[r * 3 + c], v, dv);
            num += v;
          }
          acc[2 * k] = m * num;
          acc[2 * k + 1] = m;
        }
        if (k == T_STATIC && on(terms, T_STATIC_DY)) {  // train.py:437-445
          const float m2 = rt.rho < 0.1f ? m : 0.f;
          acc[2 * T_STATIC_DY] = fabsf(sum_dy * m2);
          acc[2 * T_STATIC_DY + 1] = m2 + 1e-8f;
        }
      }
    }
    if (on(terms, T_DISP) && lane == 6) {
      float v, dv;
      disparity(in.depth[(long long)r * in.depth_ld], in.gt_disp[r], v, dv);
      const float m = ray_mask(in, r);
      acc[2 * T_DISP] = v * m;
      acc[2 * T_DISP + 1] = m;
    }
    if (on(terms, T_ENTROPY) && lane == 7) {
      float v, dv;
      entropy(rt.rho, v, dv);
      acc[2 * T_ENTROPY] = v;
    }
    if (on(terms, T_FLOW)) {
      const float mr = ray_mask(in, r);
      float num = 0.f, den = 0.f;
      for (int i = lane; i < in.n_flow * 2; i += 32) {
        const long long p = (long long)(i >> 1) * R + r;
        const float fm = mr * in.flow_masks[p];
        float v, dv;
        l1(in.flows[p * 2 + (i & 1)], in.gt_flows[p * 2 + (i & 1)], v, dv);
        num += v * fm;
        if ((i & 1) == 0) den += fm;
      }
      num = warp_sum(num);
      den = warp_sum(den);
      if (lane == 0) { acc[2 * T_FLOW] = num; acc[2 * T_FLOW + 1] = den; }
    }
    if (on(terms, T_CYCLE)) {
      float num = 0.f, den = 0.f;
      for (int k = 0; k < in.K; ++k) {
        const long long base = ((long long)k * R + r) * S3;
        for (int i = lane; i < S3; i += 32) {
          float v, dv;
          l1(in.traj_ref[base + i], in.traj_anchor[base + i], v, dv);
          num += v * in.occ_weights[(long long)r * S + i / 3];
        }
      }
      for (int s = lane; s < S; s += 32) den += in.occ_weights[(long long)r * S + s];
      num = warp_sum(num);
      den = warp_sum(den);
      if (lane == 0) { acc[2 * T_CYCLE] = num; acc[2 * T_CYCLE + 1] = den; }
    }
    if (on(terms, T_REG_ABS) || on(terms, T_REG_TIME) || on(terms, T_REG_SPACE)) {
      float n_abs = 0.f, n_time = 0.f, n_space = 0.f;
      for (int f = 0; f < in.n_sf; ++f) {
        const float* x = in.sf_seq + ((long long)f * R + r) * S3;
        const float* xn = x + (long long)R * S3;  // the next time step
        for (int i = lane; i < S3; i += 32) {
          float v, dv;
          const float xi = x[i];
          l1(xi, 0.f, v, dv);
          n_abs += v;
          if (f + 1 < in.n_sf) { sq(xi, xn[i], v, dv); n_time += v; }
          if (i + 3 < S3) { l1(x[i + 3], xi, v, dv); n_space += v; }
        }
      }
      n_abs = warp_sum(n_abs);
      n_time = warp_sum(n_time);
      n_space = warp_sum(n_space);
      if (lane == 0) { acc[2 * T_REG_ABS] = n_abs; acc[2 * T_REG_TIME] = n_time; acc[2 * T_REG_SPACE] = n_space; }
    }
    if (on(terms, T_DIST)) {
      float num = 0.f, carryW = 0.f, carryWM = 0.f;
      for (int i0 = 0; i0 < in.dist_n; i0 += 32) {
        const int i = i0 + lane;
        float w = 0.f, m = 0.f, iv = 0.f;
        if (i < in.dist_n) {
          w = in.dist_w[(long long)r * in.dist_ld + i];
          dist_sample(in, r, i, m, iv);
        }
        const float inW = carryW + warp_scan_add(w, lane), inWM = carryWM + warp_scan_add(w * m, lane);
        float exW = __shfl_up_sync(0xffffffffu, inW, 1), exWM = __shfl_up_sync(0xffffffffu, inWM, 1);
        if (lane == 0) { exW = carryW; exWM = carryWM; }
        float v, dv;
        distortion(w, m, iv, exW, exWM, inW, inWM, 0.f, 0.f, v, dv);
        num += v;
        carryW = __shfl_sync(0xffffffffu, inW, 31);
        carryWM = __shfl_sync(0xffffffffu, inWM, 31);
      }
      num = warp_sum(num);
      if (lane == 0) acc[2 * T_DIST] = num;
    }
  }
  __syncthreads();
  if (threadIdx.x < kAcc) {
    float s = 0.f;
    for (int w = 0; w < kWarps; ++w) s += sh[w][threadIdx.x];
    partial[(long long)blockIdx.x * kAcc + threadIdx.x] = s;
  }
}

__device__ __forceinline__ float denominator(int k, float den, const dyn_mono_loss_weights& wt, const Dims& d) {
  const float RS3 = (float)d.R * (float)d.S * 3.f;
  if (k < DYN_LOSS_RGB_SLOTS) return 3.f * den + wt.rgb_eps[k];
  switch (k) {
    case T_DISP: return den + 1e-8f;
    case T_FLOW: return 2.f * den + 1e-8f;
    case T_CYCLE: return 3.f * (float)d.K * den + 1e-8f;
    case T_REG_ABS: return (float)d.n_sf * RS3;
    case T_REG_TIME: return (float)(d.n_sf - 1) * RS3;
    case T_REG_SPACE: return (float)d.n_sf * (float)d.R * (float)(d.S - 1) * 3.f;
    case T_STATIC_DY: return den;
    default: return (float)d.R;  // entropy, distortion: means over the rays
  }
}

__global__ void mono_loss_finish_kernel(const float* __restrict__ partial, int nblocks,
                                        const __grid_constant__ dyn_mono_loss_weights wt, Dims d,
                                        float* __restrict__ out) {
  __shared__ float tot[kAcc];
  if (threadIdx.x < kAcc) {
    float s = 0.f;
    for (int b = 0; b < nblocks; ++b) s += partial[(long long)b * kAcc + threadIdx.x];
    tot[threadIdx.x] = s;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  float t[kTerms];  // weighted terms
#pragma unroll
  for (int k = 0; k < kTerms; ++k) {
    float comp = 0.f, scale = 0.f;
    if (on(wt.terms, k)) {
      const float den = denominator(k, tot[2 * k + 1], wt, d);
      comp = tot[2 * k] / den;
      scale = wt.w[k] / den;
    }
    t[k] = on(wt.terms, k) ? wt.w[k] * comp : 0.f;
    out[kOutComp + k] = comp;
    out[kOutScale + k] = scale;
  }
  const float rgb = (((t[0] + t[1]) + t[2]) + t[3]) + t[4];  // train.py:304-328
  const float reg = (t[T_REG_ABS] + t[T_REG_TIME]) + t[T_REG_SPACE];
  const float stat = t[T_STATIC] + t[T_STATIC_DY];
  // train.py:447-456
  out[0] = ((((((rgb + t[T_CYCLE]) + t[T_FLOW]) + t[T_DISP]) + reg) + t[T_ENTROPY]) + t[T_DIST]) + stat;
  out[1] = t[T_FLOW];
  out[2] = t[T_DISP];
  out[3] = rgb;
  out[4] = t[T_DIST];
  out[5] = t[T_ENTROPY];
  out[6] = stat;
  out[7] = t[T_CYCLE];
  out[8] = reg;
  out[kOutScale + kTerms] = 0.f;
}

__global__ void __launch_bounds__(kWarps * 32)
mono_loss_backward_kernel(const __grid_constant__ dyn_mono_loss_inputs in, unsigned terms,
                          const float* __restrict__ out, const float* __restrict__ g_loss,
                          const __grid_constant__ dyn_mono_loss_grads gr) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (r >= in.R) return;
  const int S = in.S, S3 = in.S * 3, R = in.R;
  const float g = *g_loss;
  const float* scale = out + kOutScale;  // weight / denominator of each term (0 for an absent term)
  float sum_dy, sum_st;
  summed_weights(in, r, lane, sum_dy, sum_st);
  const Ratio rt = weights_ratio(sum_dy, sum_st);
#pragma unroll
  for (int k = 0; k < DYN_LOSS_RGB_SLOTS; ++k) {
    if (gr.rgb[k] && lane < 3) {
      float v, dv;
      charbonnier(in.rgb[k].pred[(long long)r * in.rgb[k].ld + lane], in.gt_rgb[r * 3 + lane], v, dv);
      gr.rgb[k][r * 3 + lane] = g * scale[k] * slot_weight(in.rgb[k], r, rt.rho) * dv;
    }
  }
  if (gr.depth && lane == 3) {
    float v, dv;
    disparity(in.depth[(long long)r * in.depth_ld], in.gt_disp[r], v, dv);
    gr.depth[r] = g * scale[T_DISP] * ray_mask(in, r) * dv;
  }
  if (gr.flows) {
    const float mr = ray_mask(in, r);
    for (int i = lane; i < in.n_flow * 2; i += 32) {
      const long long p = (long long)(i >> 1) * R + r;
      float v, dv;
      l1(in.flows[p * 2 + (i & 1)], in.gt_flows[p * 2 + (i & 1)], v, dv);
      gr.flows[p * 2 + (i & 1)] = g * scale[T_FLOW] * mr * in.flow_masks[p] * dv;
    }
  }
  if (gr.weights_dy || gr.weights_st) {
    float e_dy = 0.f, e_st = 0.f;
    if (on(terms, T_ENTROPY)) {
      float v, dv;
      entropy(rt.rho, v, dv);
      e_dy = g * scale[T_ENTROPY] * dv * rt.d_dy;
      e_st = g * scale[T_ENTROPY] * dv * rt.d_st;
    }
    if (on(terms, T_STATIC_DY)) {
      const float m5 = slot_weight(in.rgb[T_STATIC], r, rt.rho);
      const float m2 = rt.rho < 0.1f ? m5 : 0.f;
      e_dy += g * scale[T_STATIC_DY] * sgn(sum_dy * m2) * m2;
    }
    for (int s = lane; s < S; s += 32) {
      if (gr.weights_dy) gr.weights_dy[(long long)r * S + s] = e_dy;
      if (gr.weights_st) gr.weights_st[(long long)r * S + s] = e_st;
    }
  }
  if (gr.traj_ref || gr.traj_anchor) {
    for (int k = 0; k < in.K; ++k) {
      const long long base = ((long long)k * R + r) * S3;
      for (int i = lane; i < S3; i += 32) {
        float v, dv;
        l1(in.traj_ref[base + i], in.traj_anchor[base + i], v, dv);
        const float gi = g * scale[T_CYCLE] * in.occ_weights[(long long)r * S + i / 3] * dv;
        if (gr.traj_ref) gr.traj_ref[base + i] = gi;
        if (gr.traj_anchor) gr.traj_anchor[base + i] = -gi;
      }
    }
  }
  if (gr.sf_seq) {
    const float s_abs = g * scale[T_REG_ABS], s_time = g * scale[T_REG_TIME], s_space = g * scale[T_REG_SPACE];
    const long long step = (long long)R * S3;
    for (int f = 0; f < in.n_sf; ++f) {
      const float* x = in.sf_seq + ((long long)f * R + r) * S3;
      for (int i = lane; i < S3; i += 32) {
        float v, dv, acc;
        const float xi = x[i];
        l1(xi, 0.f, v, dv);
        acc = s_abs * dv;
        if (f + 1 < in.n_sf) { sq(xi, x[i + step], v, dv); acc += s_time * dv; }
        if (f > 0) { sq(x[i - step], xi, v, dv); acc -= s_time * dv; }
        if (i >= 3) { l1(xi, x[i - 3], v, dv); acc += s_space * dv; }
        if (i + 3 < S3) { l1(x[i + 3], xi, v, dv); acc -= s_space * dv; }
        gr.sf_seq[((long long)f * R + r) * S3 + i] = acc;
      }
    }
  }
  if (gr.weights) {
    float totW = 0.f, totWM = 0.f;
    for (int i = lane; i < in.dist_n; i += 32) {
      float m, iv;
      const float w = in.dist_w[(long long)r * in.dist_ld + i];
      dist_sample(in, r, i, m, iv);
      totW += w;
      totWM += w * m;
    }
    totW = warp_sum(totW);
    totWM = warp_sum(totWM);
    float carryW = 0.f, carryWM = 0.f;
    for (int i0 = 0; i0 < in.dist_ld; i0 += 32) {
      const int i = i0 + lane;
      float w = 0.f, m = 0.f, iv = 0.f;
      if (i < in.dist_n) {
        w = in.dist_w[(long long)r * in.dist_ld + i];
        dist_sample(in, r, i, m, iv);
      }
      const float inW = carryW + warp_scan_add(w, lane), inWM = carryWM + warp_scan_add(w * m, lane);
      float exW = __shfl_up_sync(0xffffffffu, inW, 1), exWM = __shfl_up_sync(0xffffffffu, inWM, 1);
      if (lane == 0) { exW = carryW; exWM = carryWM; }
      float v, dv;
      distortion(w, m, iv, exW, exWM, inW, inWM, totW, totWM, v, dv);
      if (i < in.dist_ld) gr.weights[(long long)r * in.dist_ld + i] = i < in.dist_n ? g * scale[T_DIST] * dv : 0.f;
      carryW = __shfl_sync(0xffffffffu, inW, 31);
      carryWM = __shfl_sync(0xffffffffu, inWM, 31);
    }
  }
}

int check_inputs(const dyn_mono_loss_inputs& in, const dyn_mono_loss_weights& wt) {
  const unsigned t = wt.terms;
  auto has = [t](int k) { return ((t >> k) & 1u) != 0; };
  DYN_CHECK_ARG(in.R > 0 && in.S >= 2 && (t >> kTerms) == 0);
  bool any_rgb = false;
  for (int k = 0; k < DYN_LOSS_RGB_SLOTS; ++k) {
    if (!has(k)) continue;
    any_rgb = true;
    DYN_CHECK_ARG(in.rgb[k].pred != nullptr && in.rgb[k].ld >= 3);
  }
  bool needs_ratio = has(T_ENTROPY) || has(T_STATIC_DY);
  for (int k = 0; k < DYN_LOSS_RGB_SLOTS; ++k)
    needs_ratio = needs_ratio || (has(k) && (in.rgb[k].flags & DYN_LOSS_SLOT_TIMES_ONE_MINUS_RATIO));
  DYN_CHECK_ARG(!any_rgb || in.gt_rgb != nullptr);
  DYN_CHECK_ARG(!needs_ratio || (in.weights_dy != nullptr && in.weights_st != nullptr));
  DYN_CHECK_ARG(!has(T_DISP) || (in.depth != nullptr && in.gt_disp != nullptr && in.depth_ld >= 1));
  DYN_CHECK_ARG(!has(T_FLOW) || (in.flows != nullptr && in.gt_flows != nullptr && in.flow_masks != nullptr &&
                                 in.n_flow > 0));
  DYN_CHECK_ARG(!has(T_CYCLE) || (in.traj_ref != nullptr && in.traj_anchor != nullptr &&
                                  in.occ_weights != nullptr && in.K > 0));
  DYN_CHECK_ARG(!(has(T_REG_ABS) || has(T_REG_TIME) || has(T_REG_SPACE)) || (in.sf_seq != nullptr && in.n_sf >= 2));
  DYN_CHECK_ARG(!has(T_DIST) || (in.dist_w != nullptr && in.dist_n > 0 && in.dist_ld >= in.dist_n &&
                                 (in.s_vals != nullptr || (in.dist_m != nullptr && in.dist_interval != nullptr))));
  if (has(T_DIST) && in.dist_n > kMaxDistSamples)
    return fail(DYN_E_INVALID, "dyn_mono_loss: the distortion term supports at most %d samples per ray, got %d",
                kMaxDistSamples, in.dist_n);
  return DYN_OK;
}

}  // namespace

}  // namespace dyn

using namespace dyn;

extern "C" size_t dyn_mono_loss_workspace_bytes(int R) {
  return R > 0 ? (size_t)cdiv(R, kWarps) * kAcc * sizeof(float) : 0;
}

extern "C" int dyn_mono_loss_rows(const dyn_mono_loss_inputs* in_host, const dyn_mono_loss_weights* weights_host,
                                  float* partial, int first_block, void* stream) {
  DYN_CHECK_ARG(in_host != nullptr && weights_host != nullptr && partial != nullptr && first_block >= 0);
  const int rc = check_inputs(*in_host, *weights_host);
  if (rc != DYN_OK) return rc;
  // in.R is the slice's ray count and the stride of its [n, R, ...] inputs; the block rows land at first_block
  mono_loss_kernel<<<cdiv(in_host->R, kWarps), kWarps * 32, 0, (cudaStream_t)stream>>>(
      *in_host, weights_host->terms, partial + (long long)first_block * kAcc);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

extern "C" int dyn_mono_loss_finish(const float* partial, int nblocks, const dyn_mono_loss_weights* weights_host,
                                    int R, int S, int K, int n_sf, float* out, void* stream) {
  DYN_CHECK_ARG(partial != nullptr && weights_host != nullptr && out != nullptr);
  const unsigned t = weights_host->terms;
  auto has = [t](int k) { return ((t >> k) & 1u) != 0; };
  DYN_CHECK_ARG(R > 0 && S >= 2 && K >= 0 && n_sf >= 0 && (t >> kTerms) == 0);
  DYN_CHECK_ARG(!has(T_CYCLE) || K > 0);
  DYN_CHECK_ARG(!(has(T_REG_ABS) || has(T_REG_TIME) || has(T_REG_SPACE)) || n_sf >= 2);
  if (nblocks != cdiv(R, kWarps))
    return fail(DYN_E_INVALID, "dyn_mono_loss_finish: %d rows given for %d rays, %d expected", nblocks, R,
                cdiv(R, kWarps));
  const Dims d{R, S, K, n_sf};
  mono_loss_finish_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(partial, nblocks, *weights_host, d, out);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

extern "C" int dyn_mono_loss(const dyn_mono_loss_inputs* in_host, const dyn_mono_loss_weights* weights_host,
                             float* out, void* workspace, size_t workspace_bytes, void* stream) {
  DYN_CHECK_ARG(in_host != nullptr && weights_host != nullptr && out != nullptr && workspace != nullptr);
  const int rc = check_inputs(*in_host, *weights_host);
  if (rc != DYN_OK) return rc;
  if (workspace_bytes < dyn_mono_loss_workspace_bytes(in_host->R))
    return fail(DYN_E_WORKSPACE, "dyn_mono_loss: workspace of %zu bytes, %zu needed", workspace_bytes,
                dyn_mono_loss_workspace_bytes(in_host->R));
  const int rc_rows = dyn_mono_loss_rows(in_host, weights_host, (float*)workspace, 0, stream);
  if (rc_rows != DYN_OK) return rc_rows;
  return dyn_mono_loss_finish((const float*)workspace, cdiv(in_host->R, kWarps), weights_host, in_host->R, in_host->S,
                              in_host->K, in_host->n_sf, out, stream);
}

extern "C" int dyn_mono_loss_backward(const dyn_mono_loss_inputs* in_host, const dyn_mono_loss_weights* weights_host,
                                      const float* out, const float* g_loss, const dyn_mono_loss_grads* grads_host,
                                      void* stream) {
  DYN_CHECK_ARG(in_host != nullptr && weights_host != nullptr && out != nullptr && g_loss != nullptr &&
                grads_host != nullptr);
  const int rc = check_inputs(*in_host, *weights_host);
  if (rc != DYN_OK) return rc;
  // a gradient can only be asked for an input of a term that is present
  const unsigned t = weights_host->terms;
  auto has = [t](int k) { return ((t >> k) & 1u) != 0; };
  const dyn_mono_loss_grads& gr = *grads_host;
  for (int k = 0; k < DYN_LOSS_RGB_SLOTS; ++k) DYN_CHECK_ARG(gr.rgb[k] == nullptr || has(k));
  DYN_CHECK_ARG(gr.depth == nullptr || has(T_DISP));
  DYN_CHECK_ARG(gr.flows == nullptr || has(T_FLOW));
  DYN_CHECK_ARG(gr.weights == nullptr || has(T_DIST));
  DYN_CHECK_ARG(gr.weights_dy == nullptr || has(T_ENTROPY) || has(T_STATIC_DY));
  DYN_CHECK_ARG(gr.weights_st == nullptr || has(T_ENTROPY));
  DYN_CHECK_ARG((gr.traj_ref == nullptr && gr.traj_anchor == nullptr) || has(T_CYCLE));
  DYN_CHECK_ARG(gr.sf_seq == nullptr || has(T_REG_ABS) || has(T_REG_TIME) || has(T_REG_SPACE));
  mono_loss_backward_kernel<<<cdiv(in_host->R, kWarps), kWarps * 32, 0, (cudaStream_t)stream>>>(
      *in_host, t, out, g_loss, gr);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}
