// Training backward of the two aggregation networks (row f2): DynibarDynamic.forward
// (ibrnet/mlp_network.py:236-316) and DynibarStatic.forward (:423-527), including the ray transformer
// (:13-31, :56-104), as torch.autograd would differentiate them.
//
// Forward = the staged fp32 evaluation of nets_f32.cu run with `train = true` (one internal chunk, nothing
// updated in place), whose workspace the caller keeps: every activation the backward needs is found again by
// replaying the same bump allocation (nets_f32_bufs.cuh).  Backward, fp32:
//
//   per linear layer    dZ = dY * act'(Y) (from the stored post-activation), dW += dZ^T In, db += colsum dZ,
//                       dIn = dZ W  -- the strided split-K product of motion_train.cu (train_gemm.cuh); inputs
//                       that the forward concatenates / broadcasts / row-scales (Seg, linear_f32.cuh) are
//                       handled per segment (group sums over the views of a point, per-row scale)
//   glue                view pooling (weighted mean / variance and their weight normalisations: mask, anti-alias
//                       exp(|s|(cos - 1)) - min, visibility), visibility gating, LayerNorm, softmax attention
//                       with the query-row mask quirk, positional encodings, both output heads
//
// Gradients of the parameters are ACCUMULATED into d_params (flat, the layout of the blob given to
// dyn_net_create; the caller zeroes it).  Float atomics: reproducible to rounding, not bit-exact between runs.
// tests/test_train_gpu.py checks everything against torch autograd through the oracle.
#include <math.h>

#include "common.cuh"
#include "linear_f32.cuh"
#include "nets.cuh"
#include "nets_f32_bufs.cuh"
#include "train_gemm.cuh"

namespace dyn {

namespace {

__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// g[r, c] *= ELU'(pre) from the stored post-activation y: y > 0 ? 1 : y + 1.  posenc_S > 0: `out` had the
// sinusoid table added after the activation (mlp_network.py:286); it is subtracted again first.
__global__ void elu_bwd_kernel(float* __restrict__ g, long long ldg, const float* __restrict__ out, long long ldo,
                               int width, long long N, int posenc_S) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N * width) return;
  const long long r = idx / width;
  const int c = (int)(idx - r * width);
  float y = out[r * ldo + c];
  if (posenc_S > 0) {
    const int s = (int)(r % posenc_S);
    const double ang = (double)s / pow(10000.0, 2.0 * (double)(c / 2) / 128.0);
    y -= (float)((c & 1) ? cos(ang) : sin(ang));
  }
  if (!(y > 0.f)) g[r * ldg + c] *= (y + 1.f);
}

// out[p, c] = sum_v in[(p V + v) ldin + c]
__global__ void groupsum_kernel(const float* __restrict__ in, long long ldin, int width, long long P, int V,
                                float* __restrict__ out, long long ldo) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= P * width) return;
  const long long p = idx / width;
  const int c = (int)(idx - p * width);
  float s = 0.f;
  for (int v = 0; v < V; ++v) s += in[(p * V + v) * ldin + c];
  out[p * ldo + c] = s;
}

// Backward of fused_mean_variance (mlp_network.py:115-119) for one pooled tensor:
//   mean_c = sum_v w_v x_vc,  var_c = sum_v w_v (x_vc - mean_c)^2   (w need not sum to one)
//   dx_vc (+)= w_v (dmean_c + 2 dvar_c (x_vc - mean_c - A_c)),  A_c = mean_c (1 - sum_v w_v)
//   dw_v  (+)= sum_c dmean_c x_vc + dvar_c ((x_vc - mean_c)^2 - 2 A_c x_vc)
// One warp per point; mv = [mean(C) | var(C)] of the forward, dmv likewise.
__global__ void pool_bwd_kernel(const float* __restrict__ x, long long ldx, int C, const float* __restrict__ w,
                                const float* __restrict__ mv, long long ldmv, const float* __restrict__ dmv,
                                long long lddmv, long long P, int V, float* __restrict__ dx, long long lddx,
                                int acc_dx, float* __restrict__ dw, int acc_dw) {
  const long long p = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (p >= P) return;
  float wv[kMaxViews], part[kMaxViews];
  float W = 0.f;
  for (int v = 0; v < V; ++v) { wv[v] = w[p * V + v]; W += wv[v]; part[v] = 0.f; }
  for (int c = lane; c < C; c += 32) {
    const float mu = mv[p * ldmv + c];
    const float dmu = dmv[p * lddmv + c], dvar = dmv[p * lddmv + C + c];
    const float A = mu * (1.f - W);
    for (int v = 0; v < V; ++v) {
      const long long m = p * V + v;
      const float xv = x[m * ldx + c];
      const float g = wv[v] * (dmu + 2.f * dvar * (xv - mu - A));
      float* o = dx + m * lddx + c;
      *o = acc_dx ? *o + g : g;
      const float t = xv - mu;
      part[v] += dmu * xv + dvar * (t * t - 2.f * A * xv);
    }
  }
  for (int v = 0; v < V; ++v) {
    const float s = wsum(part[v]);
    if (lane == 0) {
      float* o = dw + p * V + v;
      *o = acc_dw ? *o + s : s;
    }
  }
}

// w2[m] = vis2[m] mask[m] / (sum_v vis2 mask + 1e-8)   (pool2_kernel of the forward)
__global__ void w2_kernel(const float* __restrict__ vis2, const float* __restrict__ mask, long long P, int V,
                          float* __restrict__ w2) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  float sum = 0.f;
  for (int v = 0; v < V; ++v) sum += vis2[p * V + v] * mask[p * V + v];
  const float den = sum + 1e-8f;
  for (int v = 0; v < V; ++v) w2[p * V + v] = vis2[p * V + v] * mask[p * V + v] / den;
}

// second pooling weights (mlp_network.py:276-281): u_v = vis2_v (already masked), w = u / (sum u + 1e-8),
// G[256] = mean_v w.  In: dw [M] (from the pooled statistics), dG256 = d/dG[:,256], extra [M] or null (the
// static blending head reads the masked visibility too).  Out: d/d(sigmoid output of vis_fc2) [M], already
// multiplied by sigmoid' = s (1 - s) and the mask.
__global__ void pool2_w_bwd_kernel(const float* __restrict__ vis2, const float* __restrict__ mask,
                                   const float* __restrict__ dw, const float* __restrict__ dG, long long lddg,
                                   const float* __restrict__ extra, long long P, int V, float* __restrict__ dz) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  float sum = 0.f;
  for (int v = 0; v < V; ++v) sum += vis2[p * V + v] * mask[p * V + v];
  const float den = sum + 1e-8f;
  const float dwm = dG[p * lddg + 256] / (float)V;
  float dot = 0.f;
  for (int v = 0; v < V; ++v) {
    const long long m = p * V + v;
    dot += (dw[m] + dwm) * (vis2[m] * mask[m] / den);
  }
  for (int v = 0; v < V; ++v) {
    const long long m = p * V + v;
    const float s = vis2[m];  // == sigmoid output where mask = 1
    float du = (dw[m] + dwm - dot) / den;
    if (extra != nullptr) du += extra[m];
    dz[m] = du * mask[m] * s * (1.f - s);
  }
}

// static first pooling weights with anti-aliasing (mlp_network.py:461-467): e_v = exp(|s| (cos_v - 1)),
// u_v = (e_v - min_v e) mask_v, w = u / (sum u + 1e-8).  In: dw [M].  Out: d/ds accumulated into ds.
__global__ void aa_w_bwd_kernel(const float* __restrict__ ray_diff, const float* __restrict__ meff,
                                const float* __restrict__ s_param, const float* __restrict__ dw, long long P,
                                int V, float* __restrict__ ds) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  float contrib = 0.f;
  if (p < P) {
    const float sabs = fabsf(*s_param);
    float e[kMaxViews];
    float emin = INFINITY;
    int amin = 0;
    for (int v = 0; v < V; ++v) {
      e[v] = expf(sabs * (ray_diff[(p * V + v) * 4 + 3] - 1.f));
      if (e[v] < emin) { emin = e[v]; amin = v; }
    }
    float sum = 0.f;
    for (int v = 0; v < V; ++v) sum += (e[v] - emin) * meff[p * V + v];
    const float den = sum + 1e-8f;
    float dot = 0.f;
    for (int v = 0; v < V; ++v) dot += dw[p * V + v] * ((e[v] - emin) * meff[p * V + v] / den);
    // d|s| = sum_v de_v (g_v - g_min), g_v = de_v/d|s| = e_v (cos_v - 1), the min's share folded in view by view.
    // Summing de_v g_v and the min's -sum_v de_v g_min separately cancels terms of size |dw| / den, and den = 1e-8
    // at a point whose valid views are all the argmin (every u = 0, where the exact contribution is 0); an FMA
    // contraction of that cancellation leaves a product's rounding error 1e8 times amplified.  The argmin's own
    // term is skipped and the g are rounded products (__fmul_rn: no contraction), so such a point adds exactly 0.
    const float gmin = __fmul_rn(e[amin], ray_diff[(p * V + amin) * 4 + 3] - 1.f);
    float acc = 0.f;
    for (int v = 0; v < V; ++v) {
      if (v == amin) continue;
      const float de = (dw[p * V + v] - dot) / den * meff[p * V + v];
      acc += de * (__fmul_rn(e[v], ray_diff[(p * V + v) * 4 + 3] - 1.f) - gmin);
    }
    const float sv = *s_param;
    contrib = sv > 0.f ? acc : (sv < 0.f ? -acc : 0.f);  // d|s|/ds, 0 at s = 0 like torch.abs
  }
  contrib = wsum(contrib);
  if ((threadIdx.x & 31) == 0 && contrib != 0.f) atomicAdd(ds, contrib);
}

// y = x * scale[row] fed a layer: dx[m, c] (+)= ds[m, c] scale[m];  dscale[m] (=) sum_c ds[m, c] x[m, c].  Warp per row.
__global__ void rowscale_bwd_kernel(const float* __restrict__ dsx, const float* __restrict__ x,
                                    const float* __restrict__ scale, long long M, float* __restrict__ dx,
                                    int acc_dx, float* __restrict__ dscale) {
  const long long m = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (m >= M) return;
  const float sc = scale[m];
  float dot = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = lane + 32 * i;
    const float g = dsx[m * 128 + c];
    dot = fmaf(g, x[m * 128 + c], dot);
    float* o = dx + m * 128 + c;
    *o = acc_dx ? *o + g * sc : g * sc;
  }
  dot = wsum(dot);
  if (lane == 0) dscale[m] = dot;
}

// x2 = x + xv[:, :128], vis1 = sigmoid(xv[:, 128]) mask, xv = ELU(vis_fc.2 h)  (mlp_network.py:273-275):
// dz[m, c] = d/d(pre-activation of vis_fc.2)
__global__ void xv_bwd_kernel(const float* __restrict__ dx2, const float* __restrict__ dvis1,
                              const float* __restrict__ xv, const float* __restrict__ mask, long long M,
                              float* __restrict__ dz) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * 129) return;
  const long long m = idx / 129;
  const int c = (int)(idx - m * 129);
  const float y = xv[idx];
  float g;
  if (c < 128) {
    g = dx2[m * 128 + c];
  } else {
    const float s = sigmoid_f(y);
    g = dvis1[m] * mask[m] * s * (1.f - s);
  }
  dz[idx] = y > 0.f ? g : g * (y + 1.f);
}

// out = LayerNorm(a + resid) w + b (mlp_network.py:100-102), eps 1e-6: dv = d/d(a + resid); dw, db accumulated
// per block and added once.  A warp walks rows r, r + nwarps, ...
__global__ void __launch_bounds__(256) ln_bwd_kernel(const float* __restrict__ a, const float* __restrict__ resid,
                                                      const float* __restrict__ w, const float* __restrict__ dy,
                                                      long long P, float* __restrict__ dv, float* __restrict__ dw,
                                                      float* __restrict__ db) {
  __shared__ float sw[8][128], sb[8][128];
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const long long nw = (long long)gridDim.x * 8;
  float aw[4] = {0.f, 0.f, 0.f, 0.f}, ab[4] = {0.f, 0.f, 0.f, 0.f};
  for (long long row = (long long)blockIdx.x * 8 + wp; row < P; row += nw) {
    float v[4], g[4];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = lane + 32 * i;
      v[i] = a[row * 128 + c] + resid[row * 128 + c];
      s += v[i];
    }
    const float mean = wsum(s) / 128.f;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) { const float t = v[i] - mean; q += t * t; }
    const float rstd = rsqrtf(wsum(q) / 128.f + 1e-6f);
    float sg = 0.f, sgx = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = lane + 32 * i;
      const float xh = (v[i] - mean) * rstd;
      const float d = dy[row * 128 + c];
      aw[i] += d * xh;
      ab[i] += d;
      g[i] = d * w[c];
      v[i] = xh;
      sg += g[i];
      sgx += g[i] * xh;
    }
    sg = wsum(sg) / 128.f;
    sgx = wsum(sgx) / 128.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) dv[row * 128 + lane + 32 * i] = rstd * (g[i] - sg - v[i] * sgx);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) { sw[wp][lane + 32 * i] = aw[i]; sb[wp][lane + 32 * i] = ab[i]; }
  __syncthreads();
  if (threadIdx.x < 128) {
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) { s1 += sw[k][threadIdx.x]; s2 += sb[k][threadIdx.x]; }
    atomicAdd(dw + threadIdx.x, s1);
    atomicAdd(db + threadIdx.x, s2);
  }
}

// Backward of softmax(q k^T / sqrt(32)) v per ray and head (mlp_network.py:19-31), with the reference's
// QUERY-row mask (rows with <= 1 valid views attend uniformly and pass no gradient to q / k).  One block per
// (ray, head); phase A: a thread per query row (row statistics, D_i = sum_j p_ij dP_ij, dQ_i); phase B: a thread
// per key row (dK_j, dV_j).  Q, K, V, dO, dQ, dK, dV are [P,128] rows; the head owns columns 32 h .. 32 h + 31.
// Shared memory: (4 S 33 + 4 S) floats.
__device__ __forceinline__ void attention_bwd_body(const float* __restrict__ Q, const float* __restrict__ K,
                                                   const float* __restrict__ Vv, const float* __restrict__ dO,
                                                   const float* __restrict__ nvalid, int S, float* __restrict__ dQ,
                                                   float* __restrict__ dK, float* __restrict__ dV) {
  extern __shared__ __align__(16) float sm[];
  float* Qs = sm;               // [S][33] (scaled by 1/sqrt(32)); padded rows: conflict-free per-thread rows
  float* Ks = Qs + S * 33;
  float* Vs = Ks + S * 33;
  float* Gs = Vs + S * 33;      // dO
  float* mx = Gs + S * 33;      // [S] row max
  float* dn = mx + S;           // [S] row sum
  float* Dd = dn + S;           // [S] D_i
  float* ok = Dd + S;           // [S] 1 = unmasked query row
  const int ray = blockIdx.x >> 2, h = blockIdx.x & 3;
  const long long base = (long long)ray * S;
  const float inv_temp = 1.f / sqrtf(32.f);
  for (int e = threadIdx.x; e < S * 32; e += blockDim.x) {
    const int j = e >> 5, d = e & 31;
    const long long g = (base + j) * 128 + h * 32 + d;
    Qs[j * 33 + d] = Q[g] * inv_temp;
    Ks[j * 33 + d] = K[g];
    Vs[j * 33 + d] = Vv[g];
    Gs[j * 33 + d] = dO[g];
  }
  __syncthreads();
  const int i = threadIdx.x;
  if (i < S) {
    const bool row_ok = nvalid[base + i] > 1.f;
    float q[32], g[32];
#pragma unroll
    for (int d = 0; d < 32; ++d) { q[d] = Qs[i * 33 + d]; g[d] = Gs[i * 33 + d]; }
    float m = -INFINITY;
    for (int j = 0; j < S; ++j) {
      float l = 0.f;
#pragma unroll
      for (int d = 0; d < 32; ++d) l = fmaf(q[d], Ks[j * 33 + d], l);
      m = fmaxf(m, l);
    }
    float den = 0.f, D = 0.f;
    for (int j = 0; j < S; ++j) {
      float l = 0.f, dp = 0.f;
#pragma unroll
      for (int d = 0; d < 32; ++d) {
        l = fmaf(q[d], Ks[j * 33 + d], l);
        dp = fmaf(g[d], Vs[j * 33 + d], dp);
      }
      const float e = expf(l - m);
      den += e;
      D += e * dp;
    }
    D /= den;
    float dq[32];
#pragma unroll
    for (int d = 0; d < 32; ++d) dq[d] = 0.f;
    if (row_ok) {
      for (int j = 0; j < S; ++j) {
        float l = 0.f, dp = 0.f;
#pragma unroll
        for (int d = 0; d < 32; ++d) {
          l = fmaf(q[d], Ks[j * 33 + d], l);
          dp = fmaf(g[d], Vs[j * 33 + d], dp);
        }
        const float ds = expf(l - m) / den * (dp - D);
#pragma unroll
        for (int d = 0; d < 32; ++d) dq[d] = fmaf(ds, Ks[j * 33 + d], dq[d]);
      }
    }
#pragma unroll
    for (int d = 0; d < 32; ++d) dQ[(base + i) * 128 + h * 32 + d] = dq[d] * inv_temp;
    mx[i] = m; dn[i] = den; Dd[i] = D; ok[i] = row_ok ? 1.f : 0.f;
  }
  __syncthreads();
  if (i < S) {
    const int j = i;
    float k[32], v[32], dk[32], dv[32];
#pragma unroll
    for (int d = 0; d < 32; ++d) { k[d] = Ks[j * 33 + d]; v[d] = Vs[j * 33 + d]; dk[d] = 0.f; dv[d] = 0.f; }
    const float unif = 1.f / (float)S;
    for (int r = 0; r < S; ++r) {
      float l = 0.f, dp = 0.f;
#pragma unroll
      for (int d = 0; d < 32; ++d) {
        l = fmaf(Qs[r * 33 + d], k[d], l);
        dp = fmaf(Gs[r * 33 + d], v[d], dp);
      }
      const bool rok = ok[r] > 0.5f;
      const float p = rok ? expf(l - mx[r]) / dn[r] : unif;
      const float ds = rok ? p * (dp - Dd[r]) : 0.f;
#pragma unroll
      for (int d = 0; d < 32; ++d) {
        dk[d] = fmaf(ds, Qs[r * 33 + d], dk[d]);  // Qs carries the 1/sqrt(32)
        dv[d] = fmaf(p, Gs[r * 33 + d], dv[d]);
      }
    }
#pragma unroll
    for (int d = 0; d < 32; ++d) {
      dK[(base + j) * 128 + h * 32 + d] = dk[d];
      dV[(base + j) * 128 + h * 32 + d] = dv[d];
    }
  }
}

// Unbounded instance: its register count (about 210) limits a block to 288 threads, so it runs S <= 288.
__global__ void attention_bwd_kernel(const float* __restrict__ Q, const float* __restrict__ K,
                                     const float* __restrict__ Vv, const float* __restrict__ dO,
                                     const float* __restrict__ nvalid, int S, float* __restrict__ dQ,
                                     float* __restrict__ dK, float* __restrict__ dV) {
  attention_bwd_body(Q, K, Vv, dO, nvalid, S, dQ, dK, dV);
}

// The same body bounded to kAttnBwdMaxS threads (at most 168 registers, the rest spills to local memory), for the
// sample counts above the unbounded instance's block limit.
constexpr int kAttnBwdMaxS = 384;
__global__ void __launch_bounds__(kAttnBwdMaxS) attention_bwd_wide_kernel(
    const float* __restrict__ Q, const float* __restrict__ K, const float* __restrict__ Vv,
    const float* __restrict__ dO, const float* __restrict__ nvalid, int S, float* __restrict__ dQ,
    float* __restrict__ dK, float* __restrict__ dV) {
  attention_bwd_body(Q, K, Vv, dO, nvalid, S, dQ, dK, dV);
}

static size_t attention_bwd_smem(int S) { return (size_t)(4 * S * 33 + 4 * S) * sizeof(float); }

// Which attention-backward instance runs S samples per ray: the unbounded kernel while S fits its block limit,
// the bounded one up to kAttnBwdMaxS; limits queried once per process.  *wide = -1: S is not supported (the
// error is set).
static int attention_bwd_select(int S, int* wide) {
  static int max_plain = 0, max_wide = 0, smem_optin = 0;
  *wide = -1;
  if (max_plain == 0) {
    cudaFuncAttributes fa;
    DYN_CUDA(cudaFuncGetAttributes(&fa, attention_bwd_kernel));
    const int plain = fa.maxThreadsPerBlock;
    DYN_CUDA(cudaFuncGetAttributes(&fa, attention_bwd_wide_kernel));
    const int wide_threads = fa.maxThreadsPerBlock;
    int dev = 0, optin = 0;
    DYN_CUDA(cudaGetDevice(&dev));
    DYN_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    max_wide = wide_threads;
    smem_optin = optin;
    max_plain = plain;
  }
  const int by_threads = max_wide > max_plain ? max_wide : max_plain;  // a multiple of 32
  const int by_smem = smem_optin / (int)attention_bwd_smem(1);
  const int limit = by_threads < by_smem ? by_threads : by_smem;
  if (S > limit)
    return fail(DYN_E_INVALID, "training: the attention backward supports S <= %d samples per ray (got %d)", limit, S);
  *wide = ((S + 31) / 32) * 32 > max_plain ? 1 : 0;
  return DYN_OK;
}

// PeriodicEmbed backward for 3 inputs with frequencies 2^k, k < n (layout of pe_kernel): dpe rows have `ld` floats
__global__ void pe3_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dpe, long long ld, int n,
                               long long N, float* __restrict__ dx) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N * 3) return;
  const long long r = idx / 3;
  const int d = (int)(idx - r * 3);
  const float xv = x[idx];
  const float* g = dpe + r * ld;
  float s = g[d];
  for (int k = 0; k < n; ++k) {
    const float f = (float)(1 << k);
    float sn, cs;
    sincosf(f * xv, &sn, &cs);
    s += f * (cs * g[(1 + n + k) * 3 + d] - sn * g[(1 + k) * 3 + d]);
  }
  dx[idx] = s;
}

// dynamic head (mlp_network.py:294-315): raw = [sigmoid(rgb_fc) (0 where no valid view), sigma - shift (-1e9 ...)]
// -> dz3 = d/d(pre-sigmoid colour) [P,3], dsig [P]
__global__ void dyn_out_bwd_kernel(const float* __restrict__ draw, const float* __restrict__ nvalid,
                                   const float* __restrict__ rgb, long long P, float* __restrict__ dz3,
                                   float* __restrict__ dsig) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const bool none = nvalid[p] < 1.f;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float s = rgb[p * 3 + k];
    dz3[p * 3 + k] = none ? 0.f : draw[p * 4 + k] * s * (1.f - s);
  }
  dsig[p] = none ? 0.f : draw[p * 4 + 3];
}

// static head (mlp_network.py:503-526): blending = softmax_v(masked_fill(logit, mask == 0, -1e9)),
// rgb = sum_v blending_v rgb_in_v -> dlogit [M], d rgb_in (first 3 of the 35 gathered channels; the other 32
// columns of d_rgb_feat are written by the pooling backward), dsig [P]
__global__ void st_out_bwd_kernel(const float* __restrict__ draw, const float* __restrict__ logit,
                                  const float* __restrict__ meff, const float* __restrict__ rgb_feat,
                                  const float* __restrict__ nvalid, long long P, int V,
                                  float* __restrict__ dlogit, float* __restrict__ d_rgb_feat,
                                  float* __restrict__ dsig) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  float l[kMaxViews], db[kMaxViews];
  float mx = -INFINITY;
  for (int v = 0; v < V; ++v) {
    const float t = meff[p * V + v] == 0.f ? -1e9f : logit[p * V + v];
    l[v] = t;
    mx = fmaxf(mx, t);
  }
  float den = 0.f;
  for (int v = 0; v < V; ++v) { l[v] = expf(l[v] - mx); den += l[v]; }
  const float g0 = draw[p * 4], g1 = draw[p * 4 + 1], g2 = draw[p * 4 + 2];
  float dot = 0.f;
  for (int v = 0; v < V; ++v) {
    l[v] /= den;
    const float* c = rgb_feat + (p * V + v) * kF;
    db[v] = g0 * c[0] + g1 * c[1] + g2 * c[2];
    dot += l[v] * db[v];
  }
  for (int v = 0; v < V; ++v) {
    const long long m = p * V + v;
    dlogit[m] = meff[m] == 0.f ? 0.f : l[v] * (db[v] - dot);
    if (d_rgb_feat != nullptr) {
      d_rgb_feat[m * kF] = l[v] * g0; d_rgb_feat[m * kF + 1] = l[v] * g1; d_rgb_feat[m * kF + 2] = l[v] * g2;
    }
  }
  dsig[p] = nvalid[p] < 1.f ? 0.f : draw[p * 4 + 3];
}

// dynamic time feature ray_dir_fc(PE(t)) (mlp_network.py:240-244; dyn_time_feat_kernel with keep = 1):
// saved = [dfeat 35 .. | hidden 256 at 64 | PE(t) 21 at 320], ddfeat[35] = column sums of d feat.  One block.
__global__ void dyn_time_feat_bwd_kernel(const float* __restrict__ prm, DynamicLayout L,
                                         const float* __restrict__ saved, const float* __restrict__ ddfeat,
                                         float* __restrict__ dprm) {
  __shared__ float dz2[kF];
  __shared__ float dz0[256];
  const int tid = threadIdx.x;
  if (tid < kF) {
    const float y = saved[tid];
    dz2[tid] = ddfeat[tid] * (y > 0.f ? 1.f : y + 1.f);
  }
  __syncthreads();
  {
    const float hk = saved[64 + tid];
    float dh = 0.f;
    for (int c = 0; c < kF; ++c) {
      dh = fmaf(dz2[c], prm[L.ray_dir2.w + c * 256 + tid], dh);
      atomicAdd(dprm + L.ray_dir2.w + c * 256 + tid, dz2[c] * hk);
    }
    dz0[tid] = dh * (hk > 0.f ? 1.f : hk + 1.f);
    if (tid < kF) atomicAdd(dprm + L.ray_dir2.b + tid, dz2[tid]);
  }
  __syncthreads();
  for (int j = 0; j < 21; ++j) atomicAdd(dprm + L.ray_dir0.w + tid * 21 + j, dz0[tid] * saved[320 + j]);
  atomicAdd(dprm + L.ray_dir0.b + tid, dz0[tid]);
}

// static: feat70[:, 35:70] = src_feat * ref_feat[ray] (mlp_network.py:450-452): d src_feat [M,35] and
// d ref_feat [R,35].  One block per ray, a thread per channel walks the S V rows of the ray.
__global__ void sfprod_bwd_kernel(const float* __restrict__ dfeat70, const float* __restrict__ SF,
                                  const float* __restrict__ reff, int rows_per_ray, float* __restrict__ dSF,
                                  float* __restrict__ dreff) {
  const int ray = blockIdx.x, c = threadIdx.x;
  if (c >= kF) return;
  const float rf = reff[ray * kF + c];
  float acc = 0.f;
  const long long m0 = (long long)ray * rows_per_ray;
  for (int i = 0; i < rows_per_ray; ++i) {
    const long long m = m0 + i;
    const float g = dfeat70[m * 2 * kF + kF + c];
    dSF[m * kF + c] = g * rf;
    acc = fmaf(g, SF[m * kF + c], acc);
  }
  dreff[ray * kF + c] = acc;
}

// d_rgb_feat[m, c] (c0 <= c < 35) = dfeat[m * ld + c]  (columns below c0 were written by the head backward and are
// ADDED to)
__global__ void feat_out_kernel(const float* __restrict__ dfeat, long long ld, long long M, int c_add,
                                float* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * kF) return;
  const long long m = idx / kF;
  const int c = (int)(idx - m * kF);
  const float g = dfeat[m * ld + c];
  out[idx] = c < c_add ? out[idx] + g : g;
}

#define TR(expr)             \
  do {                       \
    int rc_ = (expr);        \
    if (rc_) return rc_;     \
  } while (0)

// the products of one layer's backward on row-major operands
struct Prod {
  cudaStream_t st;
  const float* prm;
  float* dprm;
  bool tc;      // large products on the tensor cores (train_tc.cu)
  void* img;    // scratch of tc_grad_in
  // dW[out, width] (leading dimension ldw, column offset applied by the caller) += dz^T in;
  // in[(row / bdiv) * ldin + c], optionally scaled per row
  int grad_w(const float* dz, long long lddz, int out, long long rows, const float* in, long long ldin, int width,
             float* dW, long long ldw, long long bdiv = 1, const float* kscale = nullptr) const {
    if (tc && bdiv == 1 && width > 256 && tc_grad_w_ok(out, 256, rows)) {  // 257 = 256 + 1: two passes over dz
      int rc = tc_grad_w(dz, lddz, out, rows, in, ldin, 256, kscale, dW, ldw, st);
      if (rc) return rc;
      return grad_w(dz, lddz, out, rows, in + 256, ldin, width - 256, dW + 256, ldw, 1, kscale);
    }
    if (tc && bdiv == 1 && tc_grad_w_ok(out, width, rows))
      return tc_grad_w(dz, lddz, out, rows, in, ldin, width, kscale, dW, ldw, st);
    GemmArgs g{dz, in, dW, out, width, rows, 1, lddz, ldin, 1, ldw, 1, 0};
    g.bdiv = bdiv;
    g.kscale = kscale;
    return launch_gemm(g, true, st);
  }
  // din[rows, width] (+)= dz[rows, out] W[out, coloff : coloff + width]   (W row-major with ldw columns)
  int grad_in(const float* dz, long long lddz, int out, long long rows, const float* W, long long ldw, int width,
              float* din, long long ldd, bool accumulate = false) const {
    if (tc && !accumulate && width > 256 && tc_grad_in_ok(out, 256, rows)) {
      int rc = tc_grad_in(dz, lddz, out, rows, W, ldw, 256, din, ldd, img, st);
      if (rc) return rc;
      return grad_in(dz, lddz, out, rows, W + 256, ldw, width - 256, din + 256, ldd, false);
    }
    if (tc && !accumulate && tc_grad_in_ok(out, width, rows))
      return tc_grad_in(dz, lddz, out, rows, W, ldw, width, din, ldd, img, st);
    GemmArgs g{dz, W, din, rows, width, out, lddz, 1, ldw, 1, ldd, accumulate ? 1 : 0, 0};
    return launch_gemm(g, false, st);
  }
  int bias(const float* dz, long long lddz, int out, long long rows, int b_off) const {
    if (b_off < 0) return DYN_OK;
    return launch_colsum(dz, lddz, out, rows, dprm + b_off, st);
  }
  int elu(float* g, long long ldg, const float* out, long long ldo, int width, long long rows, int posenc_S = 0) const {
    if (rows == 0) return DYN_OK;
    elu_bwd_kernel<<<cdiv(rows * width, 256), 256, 0, st>>>(g, ldg, out, ldo, width, rows, posenc_S);
    DYN_LAUNCH_CHECK();
    return DYN_OK;
  }
  int gsum(const float* in, long long ldin, int width, long long P, int V, float* out, long long ldo) const {
    groupsum_kernel<<<cdiv(P * width, 256), 256, 0, st>>>(in, ldin, width, P, V, out, ldo);
    DYN_LAUNCH_CHECK();
    return DYN_OK;
  }
  // plain dense layer: dz [rows, out] holds dY on entry -> act' applied in place, dW / db accumulated,
  // din = dz W (unless null)
  int dense(const LinearP& l, float* dz, long long rows, const float* y_out, const float* in, float* din,
            bool elu_act, bool acc_in = false) const {
    if (elu_act) { int rc = elu(dz, l.out, y_out, l.out, l.out, rows); if (rc) return rc; }
    int rc = grad_w(dz, l.out, l.out, rows, in, l.in, l.in, dprm + l.w, l.in);
    if (rc) return rc;
    rc = bias(dz, l.out, l.out, rows, l.b);
    if (rc) return rc;
    if (din != nullptr) return grad_in(dz, l.out, l.out, rows, prm + l.w, l.in, l.in, din, l.in, acc_in);
    return DYN_OK;
  }
};

// scratch of the backward
struct BwdBufs {
  float *mA, *mB, *mC, *mD, *mE, *mF, *mS1, *mS2, *mS3;            // per (point, view)
  float *mCh, *mCh2, *mLog, *mXe, *mVe, *mSF;                      // static only
  float *pA, *pB, *pC, *pD, *pE, *pF, *pG, *pMV, *pX, *pY, *p64, *p33, *p3, *pS;  // per point
  float *rA, *rB;                                                  // per ray
  float* small;
  float* img;                                                      // tc_grad_in weight image
};

size_t bwd_alloc(Bump& b, bool st_net, int R, int S, int V, BwdBufs* q) {
  const long long P = (long long)R * S, M = P * V;
  q->mA = b.f(M * 128); q->mB = b.f(M * 128); q->mC = b.f(M * 128); q->mD = b.f(M * 129);
  q->mE = b.f(M * 256); q->mF = b.f(M * 2 * kF); q->mS1 = b.f(M); q->mS2 = b.f(M); q->mS3 = b.f(M);
  if (st_net) {
    q->mCh = b.f(M * 128); q->mCh2 = b.f(M * 64); q->mLog = b.f(M); q->mXe = b.f(M * 128); q->mVe = b.f(M);
    q->mSF = b.f(M * kF);
  } else {
    q->mCh = q->mCh2 = q->mLog = q->mXe = q->mVe = q->mSF = nullptr;
  }
  q->pA = b.f(P * 128); q->pB = b.f(P * 128); q->pC = b.f(P * 128); q->pD = b.f(P * 128); q->pE = b.f(P * 128);
  q->pF = b.f(P * 256); q->pG = b.f(P * 257); q->pMV = b.f(P * 4 * kF); q->pX = b.f(P * 128);
  q->pY = b.f(P * 256); q->p64 = b.f(P * 64); q->p33 = b.f(P * 33); q->p3 = b.f(P * 3); q->pS = b.f(P);
  q->rA = b.f((long long)R * 128); q->rB = b.f((long long)R * 2 * kF);
  q->small = b.f(64);
  q->img = b.f(tc_grad_in_scratch_bytes() / sizeof(float));
  return b.off;
}

// Backward of the shared trunk (base_fc ... ray transformer; run_trunk + run_point_tail of nets_f32.cu).
//   in : q.pA = d/dG3 [P,128];  static: q.mXe = extra d/dX2 [M,128], q.mVe = extra d/d(masked vis2) [M] (else null)
//   out: q.pMV = d/d[mean | var] of the first pooling [P, 2 C],  q.mF = d/dfeat [M, C] (leading dimension C),
//        q.mS2 = d/dw1 [M] (through vis_fc's row scale only; the pooling adds its share later)
template <class Layout>
int trunk_backward(const dyn_net* n, const Layout& L, const Prod& pr, const TrunkBufs& t, BwdBufs& q,
                   const float* mv, int C, const float* feat, const float* w1, const float* mask, long long M,
                   long long P, int R, int S, int V, bool posenc, bool have_extra, cudaStream_t st) {
  float* dprm = pr.dprm;
  const float* prm = pr.prm;
  // LayerNorm(fc(O) + G2) (mlp_network.py:99-102)
  int ln_blocks = cdiv(P, 64);
  ln_blocks = ln_blocks < 1 ? 1 : (ln_blocks > 1184 ? 1184 : ln_blocks);
  ln_bwd_kernel<<<ln_blocks, 256, 0, st>>>(
      t.O2, t.G2, prm + L.ln_w, q.pA, P, q.pB, dprm + L.ln_w, dprm + L.ln_b);
  DYN_LAUNCH_CHECK();
  // q.pB = d/d(O2 + G2): fc has no bias
  TR(pr.grad_w(q.pB, 128, 128, P, t.O, 128, 128, dprm + L.fc.w, 128));
  TR(pr.grad_in(q.pB, 128, 128, P, prm + L.fc.w, 128, 128, q.pA, 128));  // q.pA = dO
  {
    int wide;
    TR(attention_bwd_select(S, &wide));
    const int threads = ((S + 31) / 32) * 32;
    const size_t smem = attention_bwd_smem(S);
    auto kernel = wide ? attention_bwd_wide_kernel : attention_bwd_kernel;
    if (smem > 48 * 1024)
      DYN_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<R * 4, threads, smem, st>>>(t.Q, t.K, t.V, q.pA, t.nvalid, S, q.pC, q.pD, q.pE);
    DYN_LAUNCH_CHECK();
  }
  // q/k/v projections of G2 (no bias): dG2 = d(resid) + dQ Wq + dK Wk + dV Wv   (accumulated into q.pB)
  TR(pr.grad_w(q.pC, 128, 128, P, t.G2, 128, 128, dprm + L.wq.w, 128));
  TR(pr.grad_w(q.pD, 128, 128, P, t.G2, 128, 128, dprm + L.wk.w, 128));
  TR(pr.grad_w(q.pE, 128, 128, P, t.G2, 128, 128, dprm + L.wv.w, 128));
  TR(pr.grad_in(q.pC, 128, 128, P, prm + L.wq.w, 128, 128, q.pB, 128, true));
  TR(pr.grad_in(q.pD, 128, 128, P, prm + L.wk.w, 128, 128, q.pB, 128, true));
  TR(pr.grad_in(q.pE, 128, 128, P, prm + L.wv.w, 128, 128, q.pB, 128, true));
  // geometry_fc (:283 / :496): G2 = ELU(geo2(GH)) (+ sinusoid), GH = ELU(geo0(G))
  TR(pr.elu(q.pB, 128, t.G2, 128, 128, P, posenc ? S : 0));
  TR(pr.grad_w(q.pB, 128, 128, P, t.GH, 256, 256, dprm + L.geo2.w, 256));
  TR(pr.bias(q.pB, 128, 128, P, L.geo2.b));
  TR(pr.grad_in(q.pB, 128, 128, P, prm + L.geo2.w, 256, 256, q.pF, 256));
  TR(pr.elu(q.pF, 256, t.GH, 256, 256, P));
  TR(pr.grad_w(q.pF, 256, 256, P, t.G, 257, 257, dprm + L.geo0.w, 257));
  TR(pr.bias(q.pF, 256, 256, P, L.geo0.b));
  TR(pr.grad_in(q.pF, 256, 256, P, prm + L.geo0.w, 257, 257, q.pG, 257));  // q.pG = dG [P,257]
  // second pooling (:276-281 / :489-494): statistics of X2 under w2 = vis2 / (sum + 1e-8); w2 is rebuilt
  w2_kernel<<<cdiv(P, 256), 256, 0, st>>>(t.vis2, mask, P, V, q.mS3);
  DYN_LAUNCH_CHECK();
  pool_bwd_kernel<<<cdiv(P * 32, 256), 256, 0, st>>>(t.X2, 128, 128, q.mS3, t.G, 257, q.pG, 257, P, V, q.mA, 128,
                                                     have_extra ? 1 : 0, q.mS1, 0);
  DYN_LAUNCH_CHECK();
  pool2_w_bwd_kernel<<<cdiv(P, 256), 256, 0, st>>>(t.vis2, mask, q.mS1, q.pG, 257, have_extra ? q.mVe : nullptr, P, V,
                                                   q.mS2);
  DYN_LAUNCH_CHECK();
  // vis_fc2 (:276 / :489): vis2 = sigmoid(vis2_2(H3)), H3 = ELU(vis2_0(X2 vis1));  q.mS2 = d/d(pre-sigmoid)
  TR(pr.grad_w(q.mS2, 1, 1, M, t.H3, 128, 128, dprm + L.vis2_2.w, 128));
  TR(pr.bias(q.mS2, 1, 1, M, L.vis2_2.b));
  TR(pr.grad_in(q.mS2, 1, 1, M, prm + L.vis2_2.w, 128, 128, q.mB, 128));
  TR(pr.elu(q.mB, 128, t.H3, 128, 128, M));
  TR(pr.grad_w(q.mB, 128, 128, M, t.X2, 128, 128, dprm + L.vis2_0.w, 128, 1, t.vis1));
  TR(pr.bias(q.mB, 128, 128, M, L.vis2_0.b));
  TR(pr.grad_in(q.mB, 128, 128, M, prm + L.vis2_0.w, 128, 128, q.mC, 128));
  rowscale_bwd_kernel<<<cdiv(M * 32, 256), 256, 0, st>>>(q.mC, t.X2, t.vis1, M, q.mA, 1, q.mS1);  // q.mS1 = dvis1
  DYN_LAUNCH_CHECK();
  // x2 = x + x_res, vis1 = sigmoid(x_vis[128]) mask, [x_res | x_vis] = ELU(vis_fc.2(H2)) (:272-275 / :485-488)
  xv_bwd_kernel<<<cdiv(M * 129, 256), 256, 0, st>>>(q.mA, q.mS1, t.XV, mask, M, q.mD);
  DYN_LAUNCH_CHECK();
  TR(pr.grad_w(q.mD, 129, 129, M, t.H2, 128, 128, dprm + L.vis2.w, 128));
  TR(pr.bias(q.mD, 129, 129, M, L.vis2.b));
  TR(pr.grad_in(q.mD, 129, 129, M, prm + L.vis2.w, 128, 128, q.mB, 128));
  TR(pr.elu(q.mB, 128, t.H2, 128, 128, M));
  TR(pr.grad_w(q.mB, 128, 128, M, t.X, 128, 128, dprm + L.vis0.w, 128, 1, w1));
  TR(pr.bias(q.mB, 128, 128, M, L.vis0.b));
  TR(pr.grad_in(q.mB, 128, 128, M, prm + L.vis0.w, 128, 128, q.mC, 128));
  rowscale_bwd_kernel<<<cdiv(M * 32, 256), 256, 0, st>>>(q.mC, t.X, w1, M, q.mA, 1, q.mS2);  // q.mA = dX, q.mS2 = dw1
  DYN_LAUNCH_CHECK();
  // base_fc (:270 / :483) on [mean | var (per point) , feat (per view)]
  TR(pr.elu(q.mA, 128, t.X, 128, 128, M));
  TR(pr.grad_w(q.mA, 128, 128, M, t.H1, 256, 256, dprm + L.base2.w, 256));
  TR(pr.bias(q.mA, 128, 128, M, L.base2.b));
  TR(pr.grad_in(q.mA, 128, 128, M, prm + L.base2.w, 256, 256, q.mE, 256));
  TR(pr.elu(q.mE, 256, t.H1, 256, 256, M));
  TR(pr.gsum(q.mE, 256, 256, P, V, q.pY, 256));
  const int K0 = 3 * C;
  TR(pr.grad_w(q.pY, 256, 256, P, mv, 2 * C, 2 * C, dprm + L.base0.w, K0));
  TR(pr.grad_w(q.mE, 256, 256, M, feat, C, C, dprm + L.base0.w + 2 * C, K0));
  TR(pr.bias(q.mE, 256, 256, M, L.base0.b));
  TR(pr.grad_in(q.pY, 256, 256, P, prm + L.base0.w, K0, 2 * C, q.pMV, 2 * C));
  TR(pr.grad_in(q.mE, 256, 256, M, prm + L.base0.w + 2 * C, K0, C, q.mF, C));
  return DYN_OK;
}

}  // namespace

// The training forward calls this at entry, so that no forward work is done for an S its backward cannot run.
int check_attention_backward(int S) {
  int wide;
  return attention_bwd_select(S, &wide);
}

size_t net_train_workspace(int kind, int R, int S, int V) {
  Bump b{nullptr, 0};
  if (kind == DYN_NET_DYNAMIC) { DynBufs d; return dyn_alloc(b, R, S, V, &d, true); }
  StBufs d;
  return st_alloc(b, R, S, V, &d, true);
}

size_t net_backward_scratch(int kind, int R, int S, int V) {
  Bump b{nullptr, 0};
  BwdBufs q;
  return bwd_alloc(b, kind == DYN_NET_STATIC, R, S, V, &q);
}

int net_dynamic_backward(const dyn_net* n, const float* pts, const float* rgb_feat, const float* ray_dir,
                         const float* mask, int R, int S, int V, const float* d_raw, void* ws, size_t ws_bytes,
                         void* scratch, size_t scratch_bytes, float* d_params, float* d_rgb_feat, float* d_pts,
                         int prec, cudaStream_t st) {
  (void)rgb_feat; (void)ray_dir;
  const DynamicLayout& L = n->dl;
  const long long P = (long long)R * S, M = P * V;
  Bump b{(char*)ws, 0};
  DynBufs d;
  if (dyn_alloc(b, R, S, V, &d, true) > ws_bytes) return fail(DYN_E_WORKSPACE, "net backward: saved workspace too small");
  Bump b2{(char*)scratch, 0};
  BwdBufs q;
  if (bwd_alloc(b2, false, R, S, V, &q) > scratch_bytes) return fail(DYN_E_WORKSPACE, "net backward: scratch too small");
  const Prod pr{st, n->params, d_params, prec == DYN_PREC_BF16, q.img};
  const float* prm = n->params;
  float* dprm = d_params;
  // heads (mlp_network.py:294-315)
  dyn_out_bwd_kernel<<<cdiv(P, 256), 256, 0, st>>>(d_raw, d.t.nvalid, d.rgb, P, q.p3, q.pS);
  DYN_LAUNCH_CHECK();
  TR(pr.grad_w(q.p3, 3, 3, P, d.ch2, 64, 64, dprm + L.rgb4.w, 64));
  TR(pr.bias(q.p3, 3, 3, P, L.rgb4.b));
  TR(pr.grad_in(q.p3, 3, 3, P, prm + L.rgb4.w, 64, 64, q.p64, 64));
  TR(pr.dense(L.rgb2, q.p64, P, d.ch2, d.ch, q.pX, true));
  TR(pr.elu(q.pX, 128, d.ch, 128, 128, P));
  TR(pr.grad_w(q.pX, 128, 128, P, d.G4, 128, 128, dprm + L.rgb0.w, 155));
  // the direction encoding is per ray: sum dz over the samples of a ray first, then a product over R rows
  TR(pr.gsum(q.pX, 128, 128, R, S, q.rA, 128));
  TR(pr.grad_w(q.rA, 128, 128, R, d.dirpe, 27, 27, dprm + L.rgb0.w + 128, 155));
  TR(pr.bias(q.pX, 128, 128, P, L.rgb0.b));
  TR(pr.grad_in(q.pX, 128, 128, P, prm + L.rgb0.w, 155, 128, q.pA, 128));  // q.pA = dG4
  TR(pr.grad_w(q.pS, 1, 1, P, d.sh, 128, 128, dprm + L.outgeo2.w, 128));
  TR(pr.bias(q.pS, 1, 1, P, L.outgeo2.b));
  TR(pr.grad_in(q.pS, 1, 1, P, prm + L.outgeo2.w, 128, 128, q.pB, 128));
  TR(pr.dense(L.outgeo0, q.pB, P, d.sh, d.G4, q.pA, true, true));
  // ref_pts_fc(cat[g, PE(pts)]) (:291-292)
  TR(pr.dense(L.refpts2, q.pA, P, d.G4, d.G4h, q.pF, true));
  TR(pr.elu(q.pF, 256, d.G4h, 256, 256, P));
  TR(pr.grad_w(q.pF, 256, 256, P, d.t.G3, 128, 128, dprm + L.refpts0.w, 161));
  TR(pr.grad_w(q.pF, 256, 256, P, d.ptspe, 33, 33, dprm + L.refpts0.w + 128, 161));
  TR(pr.bias(q.pF, 256, 256, P, L.refpts0.b));
  if (d_pts != nullptr) {
    TR(pr.grad_in(q.pF, 256, 256, P, prm + L.refpts0.w + 128, 161, 33, q.p33, 33));
    pe3_bwd_kernel<<<cdiv(P * 3, 256), 256, 0, st>>>(pts, q.p33, 33, 5, P, d_pts);
    DYN_LAUNCH_CHECK();
  }
  TR(pr.grad_in(q.pF, 256, 256, P, prm + L.refpts0.w, 161, 128, q.pA, 128));  // q.pA = dG3
  TR(trunk_backward(n, L, pr, d.t, q, d.mv, kF, d.feat, d.w1, mask, M, P, R, S, V, /*posenc=*/true, false, st));
  // first pooling (:244-262): feat = rgb_feat + dfeat, w1 = mask / (sum mask + 1e-8) (no gradient)
  pool_bwd_kernel<<<cdiv(P * 32, 256), 256, 0, st>>>(d.feat, kF, kF, d.w1, d.mv, 2 * kF, q.pMV, 2 * kF, P, V, q.mF, kF,
                                                     1, q.mS1, 0);
  DYN_LAUNCH_CHECK();
  if (d_rgb_feat != nullptr) {
    feat_out_kernel<<<cdiv(M * kF, 256), 256, 0, st>>>(q.mF, kF, M, 0, d_rgb_feat);
    DYN_LAUNCH_CHECK();
  }
  DYN_CUDA(cudaMemsetAsync(q.small, 0, 64 * sizeof(float), st));
  TR(launch_colsum(q.mF, kF, kF, M, q.small, st));
  dyn_time_feat_bwd_kernel<<<1, 256, 0, st>>>(prm, L, d.dfeat, q.small, dprm);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int net_static_backward(const dyn_net* n, const float* rgb_feat, const float* ray_diff, int R, int S, int V,
                        const float* d_raw, void* ws, size_t ws_bytes, void* scratch, size_t scratch_bytes,
                        float* d_params, float* d_rgb_feat, int prec, cudaStream_t st) {
  const StaticLayout& L = n->sl;
  const long long P = (long long)R * S, M = P * V;
  Bump b{(char*)ws, 0};
  StBufs d;
  if (st_alloc(b, R, S, V, &d, true) > ws_bytes) return fail(DYN_E_WORKSPACE, "net backward: saved workspace too small");
  Bump b2{(char*)scratch, 0};
  BwdBufs q;
  if (bwd_alloc(b2, true, R, S, V, &q) > scratch_bytes) return fail(DYN_E_WORKSPACE, "net backward: scratch too small");
  const Prod pr{st, n->params, d_params, prec == DYN_PREC_BF16, q.img};
  const float* prm = n->params;
  float* dprm = d_params;
  // blending head (mlp_network.py:508-526)
  st_out_bwd_kernel<<<cdiv(P, 256), 256, 0, st>>>(d_raw, d.logit, d.meff, rgb_feat, d.t.nvalid, P, V, q.mLog,
                                                  d_rgb_feat, q.pS);
  DYN_LAUNCH_CHECK();
  TR(pr.grad_w(q.mLog, 1, 1, M, d.ch2, 64, 64, dprm + L.rgb4.w, 64));
  TR(pr.bias(q.mLog, 1, 1, M, L.rgb4.b));
  TR(pr.grad_in(q.mLog, 1, 1, M, prm + L.rgb4.w, 64, 64, q.mCh2, 64));
  TR(pr.dense(L.rgb2, q.mCh2, M, d.ch2, d.ch, q.mCh, true));
  TR(pr.elu(q.mCh, 128, d.ch, 128, 128, M));
  TR(pr.gsum(q.mCh, 128, 128, P, V, q.pX, 128));
  TR(pr.grad_w(q.pX, 128, 128, P, d.t.G3, 128, 128, dprm + L.rgb0.w, 261));
  TR(pr.grad_w(q.mCh, 128, 128, M, d.t.X2, 128, 128, dprm + L.rgb0.w + 128, 261));
  TR(pr.grad_w(q.mCh, 128, 128, M, d.t.vis2, 1, 1, dprm + L.rgb0.w + 256, 261));
  TR(pr.grad_w(q.mCh, 128, 128, M, ray_diff, 4, 4, dprm + L.rgb0.w + 257, 261));
  TR(pr.bias(q.mCh, 128, 128, M, L.rgb0.b));
  TR(pr.grad_in(q.pX, 128, 128, P, prm + L.rgb0.w, 261, 128, q.pA, 128));        // dG3
  TR(pr.grad_in(q.mCh, 128, 128, M, prm + L.rgb0.w + 128, 261, 128, q.mA, 128));  // extra dX2
  TR(pr.grad_in(q.mCh, 128, 128, M, prm + L.rgb0.w + 256, 261, 1, q.mVe, 1));     // extra d(masked vis2)
  // density head (:503-506) on G3
  TR(pr.grad_w(q.pS, 1, 1, P, d.sh, 128, 128, dprm + L.outgeo2.w, 128));
  TR(pr.bias(q.pS, 1, 1, P, L.outgeo2.b));
  TR(pr.grad_in(q.pS, 1, 1, P, prm + L.outgeo2.w, 128, 128, q.pB, 128));
  TR(pr.dense(L.outgeo0, q.pB, P, d.sh, d.t.G3, q.pA, true, true));
  TR(trunk_backward(n, L, pr, d.t, q, d.mv, 2 * kF, d.feat70, d.w1, d.meff, M, P, R, S, V, /*posenc=*/false, true, st));
  // first pooling (:452-477) on feat70 = [rgb_feat | src_feat * ref_feat]
  pool_bwd_kernel<<<cdiv(P * 32, 256), 256, 0, st>>>(d.feat70, 2 * kF, 2 * kF, d.w1, d.mv, 4 * kF, q.pMV, 4 * kF, P, V,
                                                     q.mF, 2 * kF, 1, q.mS2, 1);
  DYN_LAUNCH_CHECK();
  if (n->anti_alias) {
    aa_w_bwd_kernel<<<cdiv(P, 256), 256, 0, st>>>(ray_diff, d.meff, prm + L.s, q.mS2, P, V, dprm + L.s);
    DYN_LAUNCH_CHECK();
  }
  if (d_rgb_feat != nullptr) {
    feat_out_kernel<<<cdiv(M * kF, 256), 256, 0, st>>>(q.mF, 2 * kF, M, 3, d_rgb_feat);
    DYN_LAUNCH_CHECK();
  }
  sfprod_bwd_kernel<<<R, 64, 0, st>>>(q.mF, d.SF, d.reff, S * V, q.mSF, q.rB);
  DYN_LAUNCH_CHECK();
  // src_feat = ray_dir_fc([PE(pts) | PE(plucker) | ray_diff]) (:441-449); no activation after the last layer
  TR(pr.dense(L.ray_dir2, q.mSF, M, nullptr, d.H0, q.mE, false));
  TR(pr.elu(q.mE, 256, d.H0, 256, 256, M));
  TR(pr.gsum(q.mE, 256, 256, P, V, q.pY, 256));
  TR(pr.grad_w(q.pY, 256, 256, P, d.ptspe, 33, 33, dprm + L.ray_dir0.w, 103));
  TR(pr.grad_w(q.mE, 256, 256, M, d.srcpe, 66, 66, dprm + L.ray_dir0.w + 33, 103));
  TR(pr.grad_w(q.mE, 256, 256, M, ray_diff, 4, 4, dprm + L.ray_dir0.w + 99, 103));
  TR(pr.bias(q.mE, 256, 256, M, L.ray_dir0.b));
  // ref_feat = ref_feature_fc(PE(target-ray plucker)) per ray (:450)
  TR(pr.dense(L.ref_feat, q.rB, R, nullptr, d.refpe, nullptr, false));
  return DYN_OK;
}

}  // namespace dyn
