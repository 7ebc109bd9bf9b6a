// Geometry kernels: ray sampling (a2), trajectory displacement (a3 tail),
// projection + bilinear gather + view-angle difference (a4-a6), Plucker
// coordinates (a7), optical flow / expected scene flow (a14).
// All fp32.  Reference file:line citations are relative to the reference checkout's root.
#include <cuda_bf16.h>

#include "common.cuh"
#include "geometry.cuh"

namespace dyn {

// ---------------------------------------------------------------------------
// a2  sample_along_camera_ray (render_ray.py:67-131)
// The reference evaluates start + i*step with separate fp32 mul and add and
// z = 1/inv_z; the explicit _rn intrinsics stop nvcc contracting them into
// FMAs so z_vals agree bit-for-bit with the reference.
// ---------------------------------------------------------------------------
__device__ __forceinline__ float depth_at(int i, float start, float step, bool inv) {
  float v = __fadd_rn(start, __fmul_rn((float)i, step));
  return inv ? __fdiv_rn(1.0f, v) : v;
}

__global__ void sample_rays_kernel(const float* __restrict__ ray_o, const float* __restrict__ ray_d,
                                   float near_d, float far_d, int R, int S, int inv_uniform,
                                   const float* __restrict__ jitter, float* __restrict__ pts,
                                   float* __restrict__ z_vals, float* __restrict__ s_vals) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)R * S) return;
  int r = (int)(idx / S), i = (int)(idx % S);
  float start, step;
  if (inv_uniform) {
    start = __fdiv_rn(1.0f, near_d);
    step = __fdiv_rn(__fsub_rn(__fdiv_rn(1.0f, far_d), start), (float)(S - 1));
  } else {
    start = near_d;
    step = __fdiv_rn(__fsub_rn(far_d, near_d), (float)(S - 1));
  }
  float z = depth_at(i, start, step, inv_uniform);
  if (jitter != nullptr) {  // render_ray.py:113-120 (z-space mid points)
    float zl = i > 0 ? depth_at(i - 1, start, step, inv_uniform) : z;
    float zu = i < S - 1 ? depth_at(i + 1, start, step, inv_uniform) : z;
    float lower = i > 0 ? __fmul_rn(0.5f, __fadd_rn(z, zl)) : z;
    float upper = i < S - 1 ? __fmul_rn(0.5f, __fadd_rn(zu, z)) : z;
    z = __fadd_rn(lower, __fmul_rn(__fsub_rn(upper, lower), jitter[idx]));
  }
  z_vals[idx] = z;
#pragma unroll
  for (int a = 0; a < 3; ++a)
    pts[idx * 3 + a] = __fadd_rn(__fmul_rn(z, ray_d[r * 3 + a]), ray_o[r * 3 + a]);
  if (s_vals != nullptr) {
    float inv_near = __fdiv_rn(1.0f, near_d), inv_far = __fdiv_rn(1.0f, far_d);
    s_vals[idx] = __fdiv_rn(__fsub_rn(__fdiv_rn(1.0f, z), inv_near), __fsub_rn(inv_far, inv_near));
  }
}

__global__ void points_from_depths_kernel(const float* __restrict__ ray_o,
                                          const float* __restrict__ ray_d,
                                          const float* __restrict__ z_vals, float near_d,
                                          float far_d, int R, int S, float* __restrict__ pts,
                                          float* __restrict__ s_vals) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)R * S) return;
  int r = (int)(idx / S);
  float z = z_vals[idx];
#pragma unroll
  for (int a = 0; a < 3; ++a)
    pts[idx * 3 + a] = __fadd_rn(__fmul_rn(z, ray_d[r * 3 + a]), ray_o[r * 3 + a]);
  if (s_vals != nullptr) {
    float inv_near = __fdiv_rn(1.0f, near_d), inv_far = __fdiv_rn(1.0f, far_d);
    s_vals[idx] = __fdiv_rn(__fsub_rn(__fdiv_rn(1.0f, z), inv_near), __fsub_rn(inv_far, inv_near));
  }
}

// ---------------------------------------------------------------------------
// a3 tail: pts_o = pts + (traj(f+o) - traj(f))  (render_ray.py:479-497)
// brows[v][k] = basis[f+off_v][k] - is NOT pre-subtracted: the reference
// forms the two sums separately and subtracts the 3-vectors.
// ---------------------------------------------------------------------------
struct TrajArgs {
  float b_off[kMaxViews][8];  // basis rows of the displaced frames
  float b_ref[8];             // basis row of the reference frame
  int n_off, num_vv, nb;
};

__global__ void traj_displace_kernel(const float* __restrict__ pts, const float* __restrict__ coeff,
                                     TrajArgs a, long long N, float* __restrict__ pts_seq) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N) return;
  const int nb = a.nb;
  float c[24];
  for (int j = 0; j < 3 * nb; ++j) c[j] = coeff[idx * 3 * nb + j];
  float p[3] = {pts[idx * 3], pts[idx * 3 + 1], pts[idx * 3 + 2]};
  float t0[3];
  for (int ax = 0; ax < 3; ++ax) {
    float s = 0.f;
    for (int k = 0; k < nb; ++k) s += c[ax * nb + k] * a.b_ref[k];
    t0[ax] = s;
  }
  for (int v = 0; v < a.n_off; ++v) {
    for (int ax = 0; ax < 3; ++ax) {
      float s = 0.f;
      for (int k = 0; k < nb; ++k) s += c[ax * nb + k] * a.b_off[v][k];
      pts_seq[((long long)v * N + idx) * 3 + ax] = p[ax] + (s - t0[ax]);
    }
  }
  for (int v = a.n_off; v < a.n_off + a.num_vv; ++v)
    for (int ax = 0; ax < 3; ++ax) pts_seq[((long long)v * N + idx) * 3 + ax] = p[ax];
}

// scene-flow deltas traj(frame_a) - traj(frame_b) (render_ray.py:1101-1105)
struct DeltaArgs {
  float ba[8][8], bb[8][8];
  int n, nb;
};
__global__ void traj_delta_kernel(const float* __restrict__ coeff, DeltaArgs a, long long N,
                                  float* __restrict__ out) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N) return;
  const int nb = a.nb;
  float c[24];
  for (int j = 0; j < 3 * nb; ++j) c[j] = coeff[idx * 3 * nb + j];
  for (int v = 0; v < a.n; ++v)
    for (int ax = 0; ax < 3; ++ax) {
      float sa = 0.f, sb = 0.f;
      for (int k = 0; k < nb; ++k) { sa += c[ax * nb + k] * a.ba[v][k]; sb += c[ax * nb + k] * a.bb[v][k]; }
      out[((long long)v * N + idx) * 3 + ax] = sa - sb;
    }
}

// occlusion weights of the cross-time branch (render_ray.py:1224-1257); warp per ray
__global__ void occlusion_kernel(const float* __restrict__ w_ref, const float* __restrict__ w_anc, int R,
                                 int S, float* __restrict__ occ, float* __restrict__ occ_map) {
  int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (r >= R) return;
  float acc = 0.f;
  for (int s = lane; s < S; s += 32) {
    const float d = w_ref[(long long)r * S + s] - w_anc[(long long)r * S + s];
    occ[(long long)r * S + s] = 1.f - fabsf(d);
    acc += d;
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) occ_map[r] = 1.f - fabsf(acc);
}

// ---------------------------------------------------------------------------
// a4-a6 projection + gather
// ---------------------------------------------------------------------------
// featmaps [V,C,h,w] -> channels-last [V,h,w,C] so one bilinear tap is 128
// contiguous bytes.
__global__ void to_channels_last_kernel(const float* __restrict__ in, float* __restrict__ out, int C,
                                        int hw) {
  __shared__ float tile[32][33];
  int v = blockIdx.z;
  int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const float* src = in + (long long)v * C * hw;
  float* dst = out + (long long)v * C * hw;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    int c = c0 + j, p = p0 + threadIdx.x;
    if (c < C && p < hw) tile[j][threadIdx.x] = src[(long long)c * hw + p];
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    int p = p0 + j, c = c0 + threadIdx.x;
    if (c < C && p < hw) dst[(long long)p * C + c] = tile[threadIdx.x][j];
  }
}

// The fused per-view kernels read the source views in two packed per-frame layouts:
//   feature maps [V,C,h,w] fp32 -> channels-last bf16 [V,h,w,C]: one bilinear tap of all 32 channels
//     = 64 contiguous bytes (the operands of the per-view layers are bf16 anyway);
//   source images [V,H,W,3] fp32 -> [V,H,W,4] fp32 (alpha = 0): one tap = ONE aligned 16-byte load
//     instead of three 4-byte loads (colours stay fp32: the blending head outputs them directly).
__global__ void to_channels_last_bf16_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out,
                                             int C, int hw) {
  __shared__ float tile[32][33];
  int v = blockIdx.z;
  int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const float* src = in + (long long)v * C * hw;
  __nv_bfloat16* dst = out + (long long)v * C * hw;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    int c = c0 + j, p = p0 + threadIdx.x;
    if (c < C && p < hw) tile[j][threadIdx.x] = src[(long long)c * hw + p];
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    int p = p0 + j, c = c0 + threadIdx.x;
    if (c < C && p < hw) dst[(long long)p * C + c] = __float2bfloat16_rn(tile[threadIdx.x][j]);
  }
}

__global__ void rgb_to_rgba_kernel(const float* __restrict__ in, float4* __restrict__ out, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = make_float4(in[3 * i], in[3 * i + 1], in[3 * i + 2], 0.f);
}

// Stand-alone projection + gather (Projector.compute_with_motions).
// A 256-thread block owns 256 consecutive (point, view) pairs = 256 x 35 floats of
// contiguous rgb_feat output: one projection per thread, then 8 lanes per pair for the
// taps (lane j gathers feature channels 4j..4j+3 with float4 loads from the channels-last
// map, lanes 0..2 one RGB channel each); results are staged in shared memory and written
// with coalesced 16-byte stores.
// Bilinear, zero padding, align_corners=True, coordinates normalised by the
// SOURCE IMAGE size for both maps (projection.py:22-30, :143-158).
// tgt_idx [R] (multi-camera launches, else null): ray r's target camera centre is cams.tgts[tgt_idx[r]].
__global__ void __launch_bounds__(256)
project_gather_kernel(const float* __restrict__ xyz_st, const float* __restrict__ xyz,
                      const float* __restrict__ rgbs, const float* __restrict__ feat_cl,
                      const __grid_constant__ ViewCams cams, const int* __restrict__ tgt_idx, int S, int V,
                      long long N /* R*S */, int H, int W, int h, int w, float* __restrict__ rgb_feat,
                      float* __restrict__ ray_diff, float* __restrict__ mask) {
  // A block owns 256 consecutive (point, view) pairs.  Phase 1: every thread projects ONE pair (all lanes
  // busy; coalesced mask / ray_diff stores) and leaves the sampling position in shared memory.  Phase 2:
  // eight rounds of 32 pairs, eight lanes per pair (four channels each from the channels-last map, lanes
  // 0..2 one RGB channel), staged and written with coalesced 16-byte stores.
  __shared__ __align__(16) float stage[2][32 * kF];
  __shared__ float s_gx[256], s_gy[256];
  __shared__ int s_v[256];
  const long long pair0 = (long long)blockIdx.x * 256;
  const long long total = N * V;
  {
    const long long gid = pair0 + threadIdx.x;
    // (point, view) without a per-thread 64-bit division: one uniform division per block
    const long long q0 = pair0 / V;
    const int t0 = (int)(pair0 - q0 * V) + (int)threadIdx.x;
    float gx = 0.f, gy = 0.f;
    const int v = t0 % V;
    if (gid < total) {
      const long long pt = q0 + t0 / V;
      const float sx = xyz_st[pt * 3], sy = xyz_st[pt * 3 + 1], sz = xyz_st[pt * 3 + 2];
      float x = sx, y = sy, z = sz;
      if (xyz != nullptr) {
        const float* q = xyz + ((long long)v * N + pt) * 3;
        x = q[0]; y = q[1]; z = q[2];
      }
      float u, vv;
      bool front;
      project_point(cams.P[v], x, y, z, u, vv, front);
      gx = 2.f * u / (cams.w_img - 1.f) - 1.f;
      gy = 2.f * vv / (cams.h_img - 1.f) - 1.f;
      const bool inb = (u <= cams.w_img - 1.f) && (u >= 0.f) && (vv <= cams.h_img - 1.f) && (vv >= 0.f);
      mask[gid] = (inb && front) ? 1.f : 0.f;
      // compute_angle, projection.py:61-101
      const float* tgt = tgt_idx != nullptr ? cams.tgts[tgt_idx[pt / S]] : cams.tgt;
      float a0 = tgt[0] - sx, a1 = tgt[1] - sy, a2 = tgt[2] - sz;
      normalize3(a0, a1, a2);
      float b0 = cams.center[v][0] - x, b1 = cams.center[v][1] - y, b2 = cams.center[v][2] - z;
      normalize3(b0, b1, b2);
      float d0 = a0 - b0, d1 = a1 - b1, d2 = a2 - b2;
      const float dot = a0 * b0 + a1 * b1 + a2 * b2;
      normalize3(d0, d1, d2);
      reinterpret_cast<float4*>(ray_diff)[gid] = make_float4(d0, d1, d2, dot);
    }
    s_gx[threadIdx.x] = gx; s_gy[threadIdx.x] = gy; s_v[threadIdx.x] = v;
  }
  __syncthreads();
  const int lp = threadIdx.x >> 3;  // pair inside the round
  const int lane8 = threadIdx.x & 7;
#pragma unroll 1
  for (int round = 0; round < 8; ++round) {
    const long long base_pair = pair0 + round * 32;
    if (base_pair >= total) break;
    float* stg = stage[round & 1];
    const int sp = round * 32 + lp;
    if (base_pair + lp < total) {
      const float gx = s_gx[sp], gy = s_gy[sp];
      const int v = s_v[sp];
      {  // deep features, channels 4*lane8 .. +3
        const float fx = (gx + 1.f) * 0.5f * (float)(w - 1);
        const float fy = (gy + 1.f) * 0.5f * (float)(h - 1);
        const float x0f = floorf(fx), y0f = floorf(fy);
        const int x0 = (int)x0f, y0 = (int)y0f;
        const float ax = fx - x0f, ay = fy - y0f;                  // ATen grid_sampler weights:
        const float bx = (x0f + 1.f) - fx, by = (y0f + 1.f) - fy;  // (ix_se - ix) etc.
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        const float* base = feat_cl + (size_t)v * (size_t)(h * w * kC) + lane8 * 4;
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
          for (int dx = 0; dx < 2; ++dx) {
            const int xi = x0 + dx, yi = y0 + dy;
            const float wgt = (dx ? ax : bx) * (dy ? ay : by);
            if (xi >= 0 && xi < w && yi >= 0 && yi < h) {
              const float4 t = __ldg(reinterpret_cast<const float4*>(base + (yi * w + xi) * kC));
              acc.x += t.x * wgt; acc.y += t.y * wgt; acc.z += t.z * wgt; acc.w += t.w * wgt;
            }
          }
        float* o = stg + lp * kF + 3 + lane8 * 4;
        o[0] = acc.x; o[1] = acc.y; o[2] = acc.z; o[3] = acc.w;
      }
      if (lane8 < 3) {  // RGB channel lane8 from [V,H,W,3]
        const float fx = (gx + 1.f) * 0.5f * (float)(W - 1);
        const float fy = (gy + 1.f) * 0.5f * (float)(H - 1);
        const float x0f = floorf(fx), y0f = floorf(fy);
        const int x0 = (int)x0f, y0 = (int)y0f;
        const float ax = fx - x0f, ay = fy - y0f;
        const float bx = (x0f + 1.f) - fx, by = (y0f + 1.f) - fy;
        float acc = 0.f;
        const float* base = rgbs + (size_t)v * (size_t)(H * W * 3) + lane8;
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
          for (int dx = 0; dx < 2; ++dx) {
            const int xi = x0 + dx, yi = y0 + dy;
            const float wgt = (dx ? ax : bx) * (dy ? ay : by);
            if (xi >= 0 && xi < W && yi >= 0 && yi < H)
              acc += __ldg(base + (yi * W + xi) * 3) * wgt;
          }
        stg[lp * kF + lane8] = acc;
      }
    }
    __syncthreads();  // the two stage buffers alternate: the next round writes the other one
    // 32 pairs x 35 floats = 1120 contiguous floats (base_pair * 35 floats is 16-byte aligned)
    const long long n_out = (total - base_pair < 32 ? total - base_pair : 32) * kF;
    float* dst = rgb_feat + base_pair * kF;
    for (int i = threadIdx.x * 4; i < n_out; i += 256 * 4) {
      if (i + 4 <= n_out) {
        *reinterpret_cast<float4*>(dst + i) = *reinterpret_cast<const float4*>(stg + i);
      } else {
        for (int j = i; j < n_out; ++j) dst[j] = stg[j];
      }
    }
  }
}

__global__ void compute_projections_kernel(const float* __restrict__ xyz,
                                           const __grid_constant__ ViewCams cams, int V,
                                           long long N, float* __restrict__ pix,
                                           uint8_t* __restrict__ front_out) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N * V) return;
  int v = (int)(idx / N);
  float u, vv;
  bool front;
  project_point(cams.P[v], xyz[idx * 3], xyz[idx * 3 + 1], xyz[idx * 3 + 2], u, vv, front);
  pix[idx * 2] = u;
  pix[idx * 2 + 1] = vv;
  front_out[idx] = front ? 1 : 0;
}

// ---------------------------------------------------------------------------
// a7 Plucker coordinates (render_ray.py:372-396); cross over the last dim.
// ---------------------------------------------------------------------------
__global__ void plucker_ref_kernel(const float* __restrict__ ray_o, const float* __restrict__ ray_d,
                                   int R, float* __restrict__ out) {
  int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  float dx = ray_d[r * 3], dy = ray_d[r * 3 + 1], dz = ray_d[r * 3 + 2];
  normalize3(dx, dy, dz);
  float ox = ray_o[r * 3], oy = ray_o[r * 3 + 1], oz = ray_o[r * 3 + 2];
  float* o = out + r * 6;
  o[0] = dx; o[1] = dy; o[2] = dz;
  o[3] = oy * dz - oz * dy;
  o[4] = oz * dx - ox * dz;
  o[5] = ox * dy - oy * dx;
}

__global__ void plucker_src_kernel(const float* __restrict__ pts,
                                   const __grid_constant__ ViewCams cams, int V, long long N,
                                   float* __restrict__ out) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N * V) return;
  long long pt = idx / V;
  int v = (int)(idx % V);
  float ox = cams.center[v][0], oy = cams.center[v][1], oz = cams.center[v][2];
  float dx = pts[pt * 3] - ox, dy = pts[pt * 3 + 1] - oy, dz = pts[pt * 3 + 2] - oz;
  normalize3(dx, dy, dz);
  float* o = out + idx * 6;
  o[0] = dx; o[1] = dy; o[2] = dz;
  o[3] = oy * dz - oz * dy;
  o[4] = oz * dx - ox * dz;
  o[5] = ox * dy - oy * dx;
}

// ---------------------------------------------------------------------------
// a14 optical flow + expected scene flow
// (render_ray.py:333-358, :585-595, :1086-1096).  One warp per ray.
// ---------------------------------------------------------------------------
struct FlowCams {
  float Kc[kMaxViews][9];    // K[:3,:3]
  float Rw[kMaxViews][9];    // inv(c2w)[:3,:3]
  float tw[kMaxViews][3];    // inv(c2w)[:3,3]
  float b_p[8], b_m[8], b_0[8];  // basis rows f+k, f-k, f
  int nb;
};

__global__ void flow_sf_kernel(const float* __restrict__ weights, const float* __restrict__ pts_seq,
                               const float* __restrict__ uv, const float* __restrict__ coeff,
                               const __grid_constant__ FlowCams fc, int n_flow, int R, int S,
                               float* __restrict__ flows, float* __restrict__ exp_sf) {
  int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (r >= R) return;
  const long long N = (long long)R * S;
  for (int v = 0; v < n_flow; ++v) {
    float e[3] = {0.f, 0.f, 0.f};
    for (int s = lane; s < S; s += 32) {
      float wv = weights[(long long)r * S + s];
      const float* p = pts_seq + ((long long)v * N + (long long)r * S + s) * 3;
      e[0] += wv * p[0]; e[1] += wv * p[1]; e[2] += wv * p[2];
    }
#pragma unroll
    for (int a = 0; a < 3; ++a)
      for (int o = 16; o > 0; o >>= 1) e[a] += __shfl_xor_sync(0xffffffffu, e[a], o);
    if (lane == 0) {
      float c[3], q[3];
      for (int i = 0; i < 3; ++i)
        c[i] = fc.Rw[v][i * 3] * e[0] + fc.Rw[v][i * 3 + 1] * e[1] + fc.Rw[v][i * 3 + 2] * e[2] + fc.tw[v][i];
      for (int i = 0; i < 3; ++i)
        q[i] = fc.Kc[v][i * 3] * c[0] + fc.Kc[v][i * 3 + 1] * c[1] + fc.Kc[v][i * 3 + 2] * c[2];
      flows[((long long)v * R + r) * 2] = q[0] / q[2] - uv[r * 2];
      flows[((long long)v * R + r) * 2 + 1] = q[1] / q[2] - uv[r * 2 + 1];
    }
  }
  if (exp_sf != nullptr) {
    float ep[3] = {0.f, 0.f, 0.f}, em[3] = {0.f, 0.f, 0.f};
    const int nb = fc.nb;
    for (int s = lane; s < S; s += 32) {
      float wv = weights[(long long)r * S + s];
      const float* c = coeff + ((long long)r * S + s) * 3 * nb;
      for (int a = 0; a < 3; ++a) {
        float t0 = 0.f, tp = 0.f, tm = 0.f;
        for (int k = 0; k < nb; ++k) {
          float ck = c[a * nb + k];
          t0 += ck * fc.b_0[k]; tp += ck * fc.b_p[k]; tm += ck * fc.b_m[k];
        }
        ep[a] += wv * (tp - t0);
        em[a] += wv * (tm - t0);
      }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a)
      for (int o = 16; o > 0; o >>= 1) {
        ep[a] += __shfl_xor_sync(0xffffffffu, ep[a], o);
        em[a] += __shfl_xor_sync(0xffffffffu, em[a], o);
      }
    if (lane == 0)
      for (int a = 0; a < 3; ++a) exp_sf[r * 3 + a] = fmaxf(ep[a], em[a]);
  }
}

// Backward of compute_optical_flow (render_ray.py:333-358): flows[v, r] = proj_v(sum_s w[r, s] pts_seq[v, r, s]) - uv
// -> g_weights [R,S] and g_pts_seq [n_flow,R,S,3].  One warp per ray, S <= 256.
__global__ void flow_backward_kernel(const float* __restrict__ weights, const float* __restrict__ pts_seq,
                                     const float* __restrict__ g_flows, const __grid_constant__ FlowCams fc,
                                     int n_flow, int R, int S, float* __restrict__ g_weights,
                                     float* __restrict__ g_pts) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= R) return;
  const long long N = (long long)R * S;
  float gw[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int v = 0; v < n_flow; ++v) {
    float e[3] = {0.f, 0.f, 0.f};
    for (int s = lane; s < S; s += 32) {
      const float wv = weights[(long long)r * S + s];
      const float* p = pts_seq + ((long long)v * N + (long long)r * S + s) * 3;
      e[0] += wv * p[0]; e[1] += wv * p[1]; e[2] += wv * p[2];
    }
#pragma unroll
    for (int a = 0; a < 3; ++a)
      for (int o = 16; o > 0; o >>= 1) e[a] += __shfl_xor_sync(0xffffffffu, e[a], o);
    float c[3], q[3];
    for (int i = 0; i < 3; ++i)
      c[i] = fc.Rw[v][i * 3] * e[0] + fc.Rw[v][i * 3 + 1] * e[1] + fc.Rw[v][i * 3 + 2] * e[2] + fc.tw[v][i];
    for (int i = 0; i < 3; ++i)
      q[i] = fc.Kc[v][i * 3] * c[0] + fc.Kc[v][i * 3 + 1] * c[1] + fc.Kc[v][i * 3 + 2] * c[2];
    const float g0 = g_flows[((long long)v * R + r) * 2], g1 = g_flows[((long long)v * R + r) * 2 + 1];
    const float gq[3] = {g0 / q[2], g1 / q[2], -(g0 * q[0] + g1 * q[1]) / (q[2] * q[2])};
    float gc[3], ge[3];
    for (int j = 0; j < 3; ++j) gc[j] = fc.Kc[v][j] * gq[0] + fc.Kc[v][3 + j] * gq[1] + fc.Kc[v][6 + j] * gq[2];
    for (int j = 0; j < 3; ++j) ge[j] = fc.Rw[v][j] * gc[0] + fc.Rw[v][3 + j] * gc[1] + fc.Rw[v][6 + j] * gc[2];
    int i = 0;
    for (int s = lane; s < S; s += 32, ++i) {
      const long long ps = (long long)r * S + s;
      const float* p = pts_seq + ((long long)v * N + ps) * 3;
      gw[i] += ge[0] * p[0] + ge[1] * p[1] + ge[2] * p[2];
      if (g_pts != nullptr) {
        const float wv = weights[ps];
        float* o = g_pts + ((long long)v * N + ps) * 3;
        o[0] = wv * ge[0]; o[1] = wv * ge[1]; o[2] = wv * ge[2];
      }
    }
  }
  if (g_weights != nullptr) {
    int i = 0;
    for (int s = lane; s < S; s += 32, ++i) g_weights[(long long)r * S + s] = gw[i];
  }
}


// ---------------------------------------------------------------------------
// host helpers
// ---------------------------------------------------------------------------
static bool invert4(const double* m, double* inv) {
  // Gauss-Jordan with partial pivoting on a 4x4 (camera-to-world poses)
  double a[4][8];
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      a[i][j] = m[i * 4 + j];
      a[i][4 + j] = (i == j) ? 1.0 : 0.0;
    }
  for (int c = 0; c < 4; ++c) {
    int piv = c;
    for (int r = c + 1; r < 4; ++r)
      if (fabs(a[r][c]) > fabs(a[piv][c])) piv = r;
    if (fabs(a[piv][c]) < 1e-300) return false;
    if (piv != c)
      for (int j = 0; j < 8; ++j) { double t = a[c][j]; a[c][j] = a[piv][j]; a[piv][j] = t; }
    double d = a[c][c];
    for (int j = 0; j < 8; ++j) a[c][j] /= d;
    for (int r = 0; r < 4; ++r)
      if (r != c) {
        double f = a[r][c];
        for (int j = 0; j < 8; ++j) a[r][j] -= f * a[c][j];
      }
  }
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) inv[i * 4 + j] = a[i][4 + j];
  return true;
}

// Cameras are tiny (34 floats per view); they are read back to the host once
// per call to build the kernel-parameter structs.  `cams_dev` may also be a
// host pointer (cudaMemcpyDefault).
// Small read-back helper: `src` may be a device OR a host pointer.  Host
// pointers (what dynibar_b200/render_ray.py passes for cameras / basis rows) are
// copied directly -- no stream synchronisation, so the kernel pipeline is not
// drained once per call.
int fetch_small(const float* src, size_t n_floats, float* host, cudaStream_t st) {
  cudaPointerAttributes at;
  cudaError_t e = cudaPointerGetAttributes(&at, src);
  if (e != cudaSuccess) { cudaGetLastError(); at.type = cudaMemoryTypeUnregistered; }
  if (at.type == cudaMemoryTypeUnregistered || at.type == cudaMemoryTypeHost) {
    memcpy(host, src, sizeof(float) * n_floats);
    return DYN_OK;
  }
  DYN_CUDA(cudaMemcpyAsync(host, src, sizeof(float) * n_floats, cudaMemcpyDefault, st));
  DYN_CUDA(cudaStreamSynchronize(st));
  return DYN_OK;
}

static int fetch_cams(const float* cams, int V, float* host, cudaStream_t st) {
  return fetch_small(cams, (size_t)34 * V, host, st);
}

int build_view_cams(const float* src_cams, int V, const float* query_cam, cudaStream_t st,
                    ViewCams* vc, int n_query) {
  DYN_CHECK_ARG(V >= 1 && V <= kMaxViews && n_query >= 1 && n_query <= kMaxTargets);
  static thread_local float host[34 * (kMaxViews + kMaxTargets)];
  int rc = fetch_cams(src_cams, V, host, st);
  if (rc) return rc;
  if (query_cam != nullptr) {
    rc = fetch_cams(query_cam, n_query, host + 34 * V, st);
    if (rc) return rc;
    for (int i = 0; i < 3; ++i) vc->tgt[i] = host[34 * V + 18 + i * 4 + 3];
    for (int k = 0; k < n_query; ++k)
      for (int i = 0; i < 3; ++i) vc->tgts[k][i] = host[34 * (V + k) + 18 + i * 4 + 3];
  }
  vc->h_img = host[0];
  vc->w_img = host[1];
  for (int v = 0; v < V; ++v) {
    const float* c = host + 34 * v;
    double K[16], c2w[16], w2c[16];
    for (int i = 0; i < 16; ++i) { K[i] = c[2 + i]; c2w[i] = c[18 + i]; }
    if (!invert4(c2w, w2c)) return fail(DYN_E_INVALID, "singular camera pose for view %d", v);
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 4; ++j) {
        double s = 0;
        for (int k = 0; k < 4; ++k) s += K[i * 4 + k] * w2c[k * 4 + j];
        vc->P[v][i * 4 + j] = (float)s;
      }
    for (int i = 0; i < 3; ++i) vc->center[v][i] = c[18 + i * 4 + 3];
  }
  return DYN_OK;
}

int launch_to_channels_last(const float* featmaps, float* out, int V, int C, int hw, cudaStream_t st) {
  dim3 tb(32, 8), tg(cdiv(hw, 32), cdiv(C, 32), V);
  to_channels_last_kernel<<<tg, tb, 0, st>>>(featmaps, out, C, hw);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int launch_to_channels_last_bf16(const float* featmaps, void* out, int V, int C, int hw, cudaStream_t st) {
  dim3 tb(32, 8), tg(cdiv(hw, 32), cdiv(C, 32), V);
  to_channels_last_bf16_kernel<<<tg, tb, 0, st>>>(featmaps, reinterpret_cast<__nv_bfloat16*>(out), C, hw);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int launch_rgb_to_rgba(const float* rgbs, float* out, long long npix, cudaStream_t st) {
  rgb_to_rgba_kernel<<<cdiv(npix, 256), 256, 0, st>>>(rgbs, reinterpret_cast<float4*>(out), npix);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int build_flow_cams(const float* src_cams, int V, cudaStream_t st, FlowCams* fc) {
  DYN_CHECK_ARG(V >= 1 && V <= kMaxViews);
  static thread_local float host[34 * kMaxViews];
  int rc = fetch_cams(src_cams, V, host, st);
  if (rc) return rc;
  for (int v = 0; v < V; ++v) {
    const float* c = host + 34 * v;
    double c2w[16], w2c[16];
    for (int i = 0; i < 16; ++i) c2w[i] = c[18 + i];
    if (!invert4(c2w, w2c)) return fail(DYN_E_INVALID, "singular camera pose for view %d", v);
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) {
        fc->Kc[v][i * 3 + j] = c[2 + i * 4 + j];
        fc->Rw[v][i * 3 + j] = (float)w2c[i * 4 + j];
      }
      fc->tw[v][i] = (float)w2c[i * 4 + 3];
    }
  }
  return DYN_OK;
}

}  // namespace dyn

using namespace dyn;

extern "C" {

int dyn_sample_rays(const float* ray_o, const float* ray_d, float near_depth, float far_depth, int R,
                    int S, int inv_uniform, const float* jitter, float* pts, float* z_vals,
                    float* s_vals, void* stream) {
  if (R == 0) return DYN_OK;  // empty batch: nothing to do (pointers may be null)
  DYN_CHECK_ARG(ray_o && ray_d && pts && z_vals && R >= 0 && S >= 2);
  DYN_CHECK_ARG(near_depth > 0 && far_depth > near_depth);  // render_ray.py:90-94
  if (R == 0) return DYN_OK;
  long long n = (long long)R * S;
  sample_rays_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(
      ray_o, ray_d, near_depth, far_depth, R, S, inv_uniform, jitter, pts, z_vals, s_vals);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int dyn_points_from_depths(const float* ray_o, const float* ray_d, const float* z_vals,
                           float near_depth, float far_depth, int R, int S, float* pts,
                           float* s_vals, void* stream) {
  if (R == 0) return DYN_OK;  // empty batch: nothing to do (pointers may be null)
  DYN_CHECK_ARG(ray_o && ray_d && z_vals && pts && R >= 0 && S >= 1);
  if (R == 0) return DYN_OK;
  long long n = (long long)R * S;
  points_from_depths_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(
      ray_o, ray_d, z_vals, near_depth, far_depth, R, S, pts, s_vals);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

// trajectory_basis[f] with Python indexing: the reference indexes the [T,nb] basis tensor with
// ref_frame_idx + offset, and negative indices wrap (render_ray.py:479-497); only f < -T or f >= T fail
static inline bool wrap_frame(int f, int T, int* out) {
  if (f < -T || f >= T) return false;
  *out = f < 0 ? f + T : f;
  return true;
}

int dyn_traj_displace(const float* pts, const float* coeff, const float* basis, int T, int nb,
                      int frame_idx, const int* offsets_host, int n_off, int num_vv, int R, int S,
                      float* pts_seq, void* stream) {
  if (R == 0) return DYN_OK;  // empty batch: nothing to do (pointers may be null)
  DYN_CHECK_ARG(pts && coeff && basis && pts_seq && (offsets_host || n_off == 0));
  DYN_CHECK_ARG(nb >= 1 && nb <= 8 && n_off >= 0 && num_vv >= 0 && n_off + num_vv <= kMaxViews);
  if (R == 0) return DYN_OK;
  cudaStream_t st = (cudaStream_t)stream;
  static thread_local float hb[8 * (kMaxViews + 1)];
  TrajArgs a;
  memset(&a, 0, sizeof(a));
  a.n_off = n_off; a.num_vv = num_vv; a.nb = nb;
  int f0 = 0;
  DYN_CHECK_ARG(wrap_frame(frame_idx, T, &f0));
  for (int v = 0; v < n_off; ++v) {
    int f = 0;
    DYN_CHECK_ARG(wrap_frame(frame_idx + offsets_host[v], T, &f));
    int rc = fetch_small(basis + (size_t)f * nb, nb, hb + 8 * v, st);
    if (rc) return rc;
  }
  {
    int rc = fetch_small(basis + (size_t)f0 * nb, nb, hb + 8 * n_off, st);
    if (rc) return rc;
  }
  for (int v = 0; v < n_off; ++v)
    for (int k = 0; k < nb; ++k) a.b_off[v][k] = hb[8 * v + k];
  for (int k = 0; k < nb; ++k) a.b_ref[k] = hb[8 * n_off + k];
  long long N = (long long)R * S;
  traj_displace_kernel<<<cdiv(N, 256), 256, 0, st>>>(pts, coeff, a, N, pts_seq);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int dyn_traj_delta(const float* coeff, const float* basis, int T, int nb, const int* frames_a_host,
                   const int* frames_b_host, int n, int R, int S, float* out, void* stream) {
  if (R == 0) return DYN_OK;
  DYN_CHECK_ARG(coeff && basis && frames_a_host && frames_b_host && out);
  DYN_CHECK_ARG(n >= 1 && n <= 8 && nb >= 1 && nb <= 8);
  cudaStream_t st = (cudaStream_t)stream;
  static thread_local DeltaArgs a;
  a.n = n; a.nb = nb;
  for (int v = 0; v < n; ++v) {
    int fa = 0, fb = 0;
    DYN_CHECK_ARG(wrap_frame(frames_a_host[v], T, &fa) && wrap_frame(frames_b_host[v], T, &fb));
    int rc = fetch_small(basis + (size_t)fa * nb, nb, a.ba[v], st);
    if (!rc) rc = fetch_small(basis + (size_t)fb * nb, nb, a.bb[v], st);
    if (rc) return rc;
  }
  long long N = (long long)R * S;
  traj_delta_kernel<<<cdiv(N, 256), 256, 0, st>>>(coeff, a, N, out);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int dyn_occlusion_weights(const float* w_ref, const float* w_anchor, int R, int S, float* occ,
                          float* occ_map, void* stream) {
  if (R == 0) return DYN_OK;
  DYN_CHECK_ARG(w_ref && w_anchor && occ && occ_map && S >= 1);
  occlusion_kernel<<<cdiv((long long)R * 32, 256), 256, 0, (cudaStream_t)stream>>>(w_ref, w_anchor, R, S,
                                                                                  occ, occ_map);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int dyn_project_gather(const float* xyz_st, const float* xyz, const float* query_cam,
                       const float* src_rgbs, const float* src_cams, const float* featmaps, int V,
                       int R, int S, int H, int W, int C, int h, int w, float* feat_cl_ws,
                       float* rgb_feat, float* ray_diff, float* mask, void* stream) {
  return dyn_project_gather_mc(xyz_st, xyz, query_cam, 1, nullptr, src_rgbs, src_cams, featmaps, V, R, S, H, W, C,
                               h, w, feat_cl_ws, rgb_feat, ray_diff, mask, stream);
}

int dyn_project_gather_mc(const float* xyz_st, const float* xyz, const float* query_cams, int K,
                          const int* query_idx, const float* src_rgbs, const float* src_cams,
                          const float* featmaps, int V, int R, int S, int H, int W, int C, int h, int w,
                          float* feat_cl_ws, float* rgb_feat, float* ray_diff, float* mask, void* stream) {
  if (K < 1 || K > kMaxTargets) return fail(DYN_E_INVALID, "target camera count K = %d outside 1..%d", K, kMaxTargets);
  if (K > 1 && query_idx == nullptr) return fail(DYN_E_INVALID, "K = %d target cameras need a per-ray camera index", K);
  if (R == 0) return DYN_OK;  // empty batch: nothing to do (pointers may be null)
  DYN_CHECK_ARG(xyz_st && query_cams && src_rgbs && src_cams && featmaps && feat_cl_ws);
  DYN_CHECK_ARG(rgb_feat && ray_diff && mask);
  DYN_CHECK_ARG(C == kC && V >= 1 && V <= kMaxViews && H > 1 && W > 1 && h > 1 && w > 1 && (K == 1 || S >= 1));
  if (R == 0) return DYN_OK;
  cudaStream_t st = (cudaStream_t)stream;
  ViewCams vc;
  int rc = build_view_cams(src_cams, V, query_cams, st, &vc, K);
  if (rc) return rc;
  dim3 tb(32, 8), tg(cdiv(h * w, 32), cdiv(C, 32), V);
  to_channels_last_kernel<<<tg, tb, 0, st>>>(featmaps, feat_cl_ws, C, h * w);
  DYN_LAUNCH_CHECK();
  long long N = (long long)R * S;
  ProfScope prof(PROF_GATHER, st);
  project_gather_kernel<<<cdiv(N * V, 256), 256, 0, st>>>(xyz_st, xyz, src_rgbs, feat_cl_ws, vc,
                                                            K > 1 ? query_idx : nullptr, S, V, N, H, W, h,
                                                            w, rgb_feat, ray_diff, mask);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int dyn_compute_projections(const float* xyz, const float* src_cams, int V, int N, float* pix,
                            uint8_t* front, void* stream) {
  DYN_CHECK_ARG(xyz && src_cams && pix && front && N >= 0);
  if (N == 0) return DYN_OK;
  cudaStream_t st = (cudaStream_t)stream;
  ViewCams vc;
  int rc = build_view_cams(src_cams, V, nullptr, st, &vc);
  if (rc) return rc;
  compute_projections_kernel<<<cdiv((long long)N * V, 256), 256, 0, st>>>(xyz, vc, V, N, pix, front);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

// compute_angle (projection.py:61-101): a = normalize(cam_tgt - x_st), b = normalize(cam_src_v - x_v),
// out = [normalize(a - b), a . b]; xyz_st is [N,3] (st_views == 1, broadcast over the views) or [V,N,3]
__global__ void compute_angle_kernel(const float* __restrict__ xyz_st, int st_views,
                                     const float* __restrict__ xyz, const __grid_constant__ ViewCams cams,
                                     int V, long long N, float* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N * V) return;
  const int v = (int)(idx / N);
  const long long pt = idx - (long long)v * N;
  const float* s = xyz_st + ((st_views > 1 ? (long long)v * N : 0) + pt) * 3;
  const float* q = xyz + idx * 3;
  float a0 = cams.tgt[0] - s[0], a1 = cams.tgt[1] - s[1], a2 = cams.tgt[2] - s[2];
  normalize3(a0, a1, a2);
  float b0 = cams.center[v][0] - q[0], b1 = cams.center[v][1] - q[1], b2 = cams.center[v][2] - q[2];
  normalize3(b0, b1, b2);
  float d0 = a0 - b0, d1 = a1 - b1, d2 = a2 - b2;
  const float dot = a0 * b0 + a1 * b1 + a2 * b2;
  normalize3(d0, d1, d2);
  reinterpret_cast<float4*>(out)[idx] = make_float4(d0, d1, d2, dot);
}

int dyn_compute_angle(const float* xyz_st, int st_views, const float* xyz, const float* query_cam,
                      const float* src_cams, int V, int N, float* ray_diff, void* stream) {
  DYN_CHECK_ARG(N >= 0 && V >= 1 && (st_views == 1 || st_views == V));
  if (N == 0) return DYN_OK;
  DYN_CHECK_ARG(xyz_st && xyz && query_cam && src_cams && ray_diff);
  cudaStream_t st = (cudaStream_t)stream;
  ViewCams vc;
  int rc = build_view_cams(src_cams, V, query_cam, st, &vc);
  if (rc) return rc;
  compute_angle_kernel<<<cdiv((long long)N * V, 256), 256, 0, st>>>(xyz_st, st_views, xyz, vc, V, N, ray_diff);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int dyn_plucker_ref(const float* ray_o, const float* ray_d, int R, float* out6, void* stream) {
  if (R == 0) return DYN_OK;  // empty batch: nothing to do (pointers may be null)
  DYN_CHECK_ARG(ray_o && ray_d && out6 && R >= 0);
  if (R == 0) return DYN_OK;
  plucker_ref_kernel<<<cdiv(R, 256), 256, 0, (cudaStream_t)stream>>>(ray_o, ray_d, R, out6);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int dyn_plucker_src(const float* pts, const float* src_cams, int V, int R, int S, float* out,
                    void* stream) {
  if (R == 0) return DYN_OK;  // empty batch: nothing to do (pointers may be null)
  DYN_CHECK_ARG(pts && src_cams && out && R >= 0);
  if (R == 0) return DYN_OK;
  cudaStream_t st = (cudaStream_t)stream;
  ViewCams vc;
  int rc = build_view_cams(src_cams, V, nullptr, st, &vc);
  if (rc) return rc;
  long long N = (long long)R * S;
  plucker_src_kernel<<<cdiv(N * V, 256), 256, 0, st>>>(pts, vc, V, N, out);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int dyn_flow_sceneflow(const float* weights, const float* pts_seq, const float* src_cams,
                       const float* uv, const float* coeff, const float* basis, int T, int nb,
                       int frame_idx, int sf_k, int n_flow, int R, int S, float* flows,
                       float* exp_sf, void* stream) {
  if (R == 0) return DYN_OK;  // empty batch: nothing to do (pointers may be null)
  DYN_CHECK_ARG(weights && pts_seq && src_cams && uv && flows);
  DYN_CHECK_ARG(n_flow >= 0 && n_flow <= kMaxViews && nb >= 1 && nb <= 8);
  if (R == 0) return DYN_OK;
  cudaStream_t st = (cudaStream_t)stream;
  static thread_local FlowCams fc;
  memset(&fc, 0, sizeof(fc));
  fc.nb = nb;
  if (n_flow > 0) {
    int rc = build_flow_cams(src_cams, n_flow, st, &fc);
    if (rc) return rc;
  }
  if (exp_sf != nullptr) {
    int fp = 0, fm = 0, f0 = 0;
    DYN_CHECK_ARG(coeff && basis && wrap_frame(frame_idx + sf_k, T, &fp) && wrap_frame(frame_idx - sf_k, T, &fm) &&
                  wrap_frame(frame_idx, T, &f0));
    float hb[24];
    int rc = fetch_small(basis + (size_t)fp * nb, nb, hb, st);
    if (!rc) rc = fetch_small(basis + (size_t)fm * nb, nb, hb + 8, st);
    if (!rc) rc = fetch_small(basis + (size_t)f0 * nb, nb, hb + 16, st);
    if (rc) return rc;
    for (int k = 0; k < nb; ++k) { fc.b_p[k] = hb[k]; fc.b_m[k] = hb[8 + k]; fc.b_0[k] = hb[16 + k]; }
  }
  flow_sf_kernel<<<cdiv((long long)R * 32, 256), 256, 0, st>>>(weights, pts_seq, uv, coeff, fc,
                                                               n_flow, R, S, flows, exp_sf);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int dyn_flow_backward(const float* weights, const float* pts_seq, const float* src_cams, const float* g_flows,
                      int n_flow, int R, int S, float* g_weights, float* g_pts_seq, void* stream) {
  if (R == 0 || n_flow == 0) return DYN_OK;
  DYN_CHECK_ARG(weights && pts_seq && src_cams && g_flows && (g_weights || g_pts_seq));
  DYN_CHECK_ARG(n_flow >= 1 && n_flow <= kMaxViews && S >= 1 && S <= 256);
  cudaStream_t st = (cudaStream_t)stream;
  static thread_local FlowCams fc;
  memset(&fc, 0, sizeof(fc));
  int rc = build_flow_cams(src_cams, n_flow, st, &fc);
  if (rc) return rc;
  flow_backward_kernel<<<cdiv((long long)R * 32, 256), 256, 0, st>>>(weights, pts_seq, g_flows, fc, n_flow, R, S,
                                                                     g_weights, g_pts_seq);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

}  // extern "C"
