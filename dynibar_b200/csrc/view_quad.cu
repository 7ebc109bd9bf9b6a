// Fused per-(point, view) stage of the two aggregation networks on the tensor cores, "quad" schedule
// (reference: ibrnet/projection.py:103-176, ibrnet/mlp_network.py:236-284 (dynamic) / :423-497 (static)).
//
// Same per-tile work as view_twin.cu (projection, masks, view-angle difference, bilinear gather,
// Plucker / positional encodings, ray_dir_fc, both view poolings, base_fc -> vis_fc -> vis_fc2), but
// scheduled so that the CUDA cores never wait for the tensor pipe:
//
//   * ONE CTA per SM owns TWO 128-row tiles (TMEM 2 x 256 columns, two 64 KB operand tiles);
//   * all 16 row warps serve BOTH tiles: every row has four threads (warps w, w+4, w+8, w+12 share the
//     TMEM lane quadrant w & 3) that split each layer's output columns, the gathered channels and the
//     pooled channels four ways;
//   * the row warps ALTERNATE between the tiles phase by phase:  epilogue_k(tile 0) -> arrive ->
//     epilogue_k(tile 1) -> arrive -> wait(tile 0) ...  While they run tile 1's epilogue the MMA warpgroup
//     (fused_engine.cuh: issuer_loop<PP = true>) runs tile 0's next layer on the tensor cores, and vice
//     versa, so an accumulator is normally complete by the time its epilogue starts.
//   * the bilinear taps of a tile are issued one phase before they are consumed: their L2 latency is
//     covered by the other tile's phase.
//
// warps 0-15 : row warps (quad index q = warp >> 2, TMEM lane quadrant = warp & 3)
// warps 16-19 : MMA warpgroup (wgmma)             warp 20 : weight producer (cp.async.bulk ring)
#include <cstdlib>
#include "fused_engine.cuh"
#include "geometry.cuh"
#include "nets.cuh"

namespace dyn {

using namespace tc;
using namespace fe;

namespace {

constexpr int kQATile = 65536;   // K <= 256: 32 k-groups of 2 KB
constexpr int kQStage = 16384;
constexpr int kQRing = 4;
// constants (floats)
constexpr int Q_B2 = 0, Q_B4 = 48, Q_B5 = 176, Q_B6 = 304, Q_W6V = 432, Q_B7 = 560, Q_W8 = 688,
              Q_MISC = 816, Q_DFEAT = 832, Q_XCH5 = 880, Q_XCH7 = Q_XCH5 + 1024, kQConst = Q_XCH7 + 1024;
constexpr int kQSmem = 2 * kQATile + kQRing * kQStage + kQConst * 4 + 256;
constexpr int W_ISSUE = 16, W_PROD = 16 + kIssuerWarps;  // MMA warpgroup, weight producer
constexpr int kQThreads = 32 * (W_PROD + 1);

__device__ __forceinline__ void quad_sync(int quadrant) {
  asm volatile("bar.sync %0, 128;" ::"r"(quadrant + 1) : "memory");
}

__device__ __forceinline__ void tmem_ld8(uint32_t taddr, float* v) { tmem_ld<8>(taddr, v); }

// 11 values of one PE component: [x, cos(2^k x) k=0..4, sin(2^k x) k=0..4]
__device__ __forceinline__ void pe_comp11(float x, float* o) {
  float s, c;
  __sincosf(x, &s, &c);
  o[0] = x;
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    o[1 + k] = c;
    o[6 + k] = s;
    const float s2 = 2.f * s * c, c2 = 1.f - 2.f * s * s;
    s = s2; c = c2;
  }
}

// 32 accumulator columns [col0, col0+32) -> ELU on the exp2 scale -> bf16 operand columns
__device__ __forceinline__ void elu_log2_32_to_A(uint8_t* arow, uint32_t tacc, int col0) {
  float acc[32];
  tmem_ld32(tacc + col0, acc);
  tmem_wait_ld();
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = elu_log2(acc[i]);
#pragma unroll
  for (int g = 0; g < 4; ++g) store8(arow, col0 + 8 * g, acc + 8 * g);
}

// per-tile state of one row thread
struct QCtx {
  uint8_t* arow;
  uint32_t tacc, b_ready, b_acc, acc_cnt;
  long long pl, m;
  bool pt_ok, valid;
  float pu, pv, mask_proj, mask, w1, vis1, rd[4];
  float ch[24];   // pooled channels of this quad (slot layout in view_quad_build)
  // bilinear taps in flight
  uint4 tf[4];    // 4 taps x 16 B (8 bf16 feature channels)
  float tw[4];    // tap weights (feature map)
  float4 tr[4];   // 4 taps x RGBA
  float twr[4];   // tap weights (image)
};

__device__ __forceinline__ void q_ready(const QCtx& c) {
  fence_proxy_async_smem();
  tc_fence_before_sync();
  mbar_arrive(c.b_ready);
}
__device__ __forceinline__ void q_wait(QCtx& c) {
  mbar_wait(c.b_acc, c.acc_cnt & 1);
  ++c.acc_cnt;
  tc_fence_after_sync();
}

template <int VP, bool ST>
struct QuadOps {
  const ViewFusedArgs& a;
  float* cst;
  int q, quadrant, r, v, gl;
  float wh, hh;
  bool want_rgb;

  // ---- geometry (every quad thread; cheap) + [static] this quad's part of the ray_dir_fc.0 operand ----
  __device__ __forceinline__ void geometry(QCtx& c, int it, int T) const {
    const long long row = (long long)it * 256 + T * 128 + r;
    c.pl = row / VP;
    c.pt_ok = c.pl < a.P;
    c.valid = c.pt_ok && v < a.V;
    c.m = c.pl * a.V + v;
    float p3[3] = {0.f, 0.f, 0.f}, q3[3];
    if (c.pt_ok) { p3[0] = a.pts[c.pl * 3]; p3[1] = a.pts[c.pl * 3 + 1]; p3[2] = a.pts[c.pl * 3 + 2]; }
    q3[0] = p3[0]; q3[1] = p3[1]; q3[2] = p3[2];
    if (!ST && c.valid) {
      const float* qq = a.pts_seq + ((long long)v * a.seq_stride + c.pl) * 3;
      q3[0] = qq[0]; q3[1] = qq[1]; q3[2] = qq[2];
    }
    const int vc = c.valid ? v : 0;
    bool front;
    project_point(a.cams.P[vc], q3[0], q3[1], q3[2], c.pu, c.pv, front);
    const bool inb = (c.pu <= wh - 1.f) && (c.pu >= 0.f) && (c.pv <= hh - 1.f) && (c.pv >= 0.f);
    c.mask_proj = (c.valid && inb && front) ? 1.f : 0.f;
    {
      float a0 = a.cams.tgt[0] - p3[0], a1 = a.cams.tgt[1] - p3[1], a2 = a.cams.tgt[2] - p3[2];
      normalize3(a0, a1, a2);
      float b0 = a.cams.center[vc][0] - q3[0], b1 = a.cams.center[vc][1] - q3[1],
            b2 = a.cams.center[vc][2] - q3[2];
      normalize3(b0, b1, b2);
      c.rd[0] = a0 - b0; c.rd[1] = a1 - b1; c.rd[2] = a2 - b2;
      c.rd[3] = a0 * b0 + a1 * b1 + a2 * b2;
      normalize3(c.rd[0], c.rd[1], c.rd[2]);
    }
    if (ST) {
      // ray_dir_fc.0 operand, K = 128: quad q < 3 writes PE components 3q .. 3q+2 (33 values) at
      // columns [40q, 40q+40); quad 3 writes [ray_diff(4), 1, 1, 0, 0] at [120, 128)
      if (q < 3) {
        float comp[3];
        if (q == 0) {
          comp[0] = p3[0]; comp[1] = p3[1]; comp[2] = p3[2];
        } else {
          const float ox = a.cams.center[vc][0], oy = a.cams.center[vc][1], oz = a.cams.center[vc][2];
          float dx = p3[0] - ox, dy = p3[1] - oy, dz = p3[2] - oz;
          normalize3(dx, dy, dz);
          if (q == 1) {
            comp[0] = dx; comp[1] = dy; comp[2] = dz;
          } else {
            comp[0] = oy * dz - oz * dy;
            comp[1] = oz * dx - ox * dz;
            comp[2] = ox * dy - oy * dx;
          }
        }
        float xin[40];
        pe_comp11(comp[0], xin); pe_comp11(comp[1], xin + 11); pe_comp11(comp[2], xin + 22);
#pragma unroll
        for (int i = 33; i < 40; ++i) xin[i] = 0.f;
        if (!c.valid) {
#pragma unroll
          for (int i = 0; i < 33; ++i) xin[i] = 0.f;
        }
#pragma unroll
        for (int g = 0; g < 5; ++g) store8(c.arow, 40 * q + 8 * g, xin + 8 * g);
      } else {
        float t[8] = {c.rd[0], c.rd[1], c.rd[2], c.rd[3], 1.f, 1.f, 0.f, 0.f};
        if (!c.valid) {
#pragma unroll
          for (int i = 0; i < 8; ++i) t[i] = 0.f;
        }
        store8(c.arow, 120, t);
      }
      q_ready(c);
    }
  }

  // ---- issue the bilinear taps of this quad's 8 feature channels (+ rgb): packed per-frame layouts
  //      (bf16 channels-last features: one 16 B load per tap; RGBA fp32 images: one 16 B load per tap) ----
  __device__ __forceinline__ void gather_issue(QCtx& c) const {
    const int vc = c.valid ? v : 0;
    const float gx = 2.f * c.pu / (wh - 1.f) - 1.f, gy = 2.f * c.pv / (hh - 1.f) - 1.f;
    {
      const float fx = (gx + 1.f) * 0.5f * (float)(a.w - 1), fy = (gy + 1.f) * 0.5f * (float)(a.h - 1);
      const float x0f = floorf(fx), y0f = floorf(fy);
      const int x0 = (int)x0f, y0 = (int)y0f;
      const float ax = fx - x0f, ay = fy - y0f, bx = (x0f + 1.f) - fx, by = (y0f + 1.f) - fy;
      const uint16_t* base = a.feat_bf + (long long)vc * a.h * a.w * kC + 8 * q;
#pragma unroll
      for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
          // out-of-range taps (and padding rows) load a clamped texel with weight 0 (no branch)
          const int xi = x0 + dx, yi = y0 + dy;
          const bool in = c.valid && xi >= 0 && xi < a.w && yi >= 0 && yi < a.h;
          c.tw[2 * dy + dx] = in ? (dx ? ax : bx) * (dy ? ay : by) : 0.f;
          const int xc = min(max(xi, 0), a.w - 1), yc = min(max(yi, 0), a.h - 1);
          c.tf[2 * dy + dx] = __ldg(reinterpret_cast<const uint4*>(base + ((long long)yc * a.w + xc) * kC));
        }
    }
    if (want_rgb) {
      const float fx = (gx + 1.f) * 0.5f * (float)(a.W - 1), fy = (gy + 1.f) * 0.5f * (float)(a.H - 1);
      const float x0f = floorf(fx), y0f = floorf(fy);
      const int x0 = (int)x0f, y0 = (int)y0f;
      const float ax = fx - x0f, ay = fy - y0f, bx = (x0f + 1.f) - fx, by = (y0f + 1.f) - fy;
      const float* base = a.rgba + (long long)vc * a.H * a.W * 4;
#pragma unroll
      for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
          const int xi = x0 + dx, yi = y0 + dy;
          const bool in = c.valid && xi >= 0 && xi < a.W && yi >= 0 && yi < a.H;
          c.twr[2 * dy + dx] = in ? (dx ? ax : bx) * (dy ? ay : by) : 0.f;
          const int xc = min(max(xi, 0), a.W - 1), yc = min(max(yi, 0), a.H - 1);
          c.tr[2 * dy + dx] = __ldg(reinterpret_cast<const float4*>(base + ((long long)yc * a.W + xc) * 4));
        }
    }
  }

  // ---- interpolate: ch[0..7] = this quad's feature channels; quad 3: ch[8..10] = rgb; masks / outputs ----
  __device__ __forceinline__ void gather_consume(QCtx& c) const {
#pragma unroll
    for (int i = 0; i < 24; ++i) c.ch[i] = 0.f;
    // same accumulation order as the reference-layout kernels: taps (0,0), (0,1), (1,0), (1,1)
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float wgt = c.tw[t];
      const uint32_t u[4] = {c.tf[t].x, c.tf[t].y, c.tf[t].z, c.tf[t].w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        c.ch[2 * j] += __uint_as_float(u[j] << 16) * wgt;
        c.ch[2 * j + 1] += __uint_as_float(u[j] & 0xffff0000u) * wgt;
      }
    }
    float rgb[3] = {0.f, 0.f, 0.f};
    if (want_rgb) {
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float wgt = c.twr[t];
        rgb[0] += c.tr[t].x * wgt; rgb[1] += c.tr[t].y * wgt; rgb[2] += c.tr[t].z * wgt;
      }
    }
    c.mask = c.mask_proj;
    if (ST && a.mask_rgb) c.mask *= ((rgb[0] + rgb[1] + rgb[2]) > 1e-3f) ? 1.f : 0.f;
    if (q == 3) {
      c.ch[8] = rgb[0]; c.ch[9] = rgb[1]; c.ch[10] = rgb[2];
      if (c.valid) {
        a.mask_proj[c.m] = c.mask_proj;
        if (ST) {
          a.mask_eff[c.m] = c.mask;
          reinterpret_cast<float4*>(a.ray_diff)[c.m] = make_float4(c.rd[0], c.rd[1], c.rd[2], c.rd[3]);
          a.rgb_in[c.m * 3] = rgb[0]; a.rgb_in[c.m * 3 + 1] = rgb[1]; a.rgb_in[c.m * 3 + 2] = rgb[2];
        }
      }
    }
  }

  // ---- F1 epilogue: ELU(ray_dir_fc.0), this quad's 64 of the 256 columns ----
  __device__ __forceinline__ void f1_epilogue(QCtx& c) const {
    q_wait(c);
    elu_log2_32_to_A(c.arow, c.tacc, 64 * q);
    elu_log2_32_to_A(c.arow, c.tacc, 64 * q + 32);
    q_ready(c);
  }

  // ---- [static] F2 epilogue (src_feat * ref_feat) + pooling weights + first pooling; [dynamic] + time feature ----
  __device__ __forceinline__ void pool1(QCtx& c) const {
    if (ST) {
      q_wait(c);
      // ray_dir_fc.2 output channels: quad 0 -> 0..15, quad 1 -> 16..23, quad 2 -> 24..31, quad 3 -> 32..34
      float s[16];
      if (q == 0) tmem_ld16(c.tacc, s);
      else tmem_ld8(c.tacc + 16 + 8 * (q - 1), s);
      tmem_wait_ld();
      const long long ray = c.pt_ok ? c.pl / a.S : 0;
      const float* rf = a.ref_feat + ray * kF;
      if (q == 0) {
#pragma unroll
        for (int i = 0; i < 16; ++i) c.ch[8 + i] = c.valid ? (s[i] + cst[Q_B2 + i]) * __ldg(rf + i) : 0.f;
      } else if (q < 3) {
#pragma unroll
        for (int i = 0; i < 8; ++i)
          c.ch[8 + i] = c.valid ? (s[i] + cst[Q_B2 + 8 + 8 * q + i]) * __ldg(rf + 8 + 8 * q + i) : 0.f;
      } else {
#pragma unroll
        for (int i = 0; i < 3; ++i) c.ch[11 + i] = c.valid ? (s[i] + cst[Q_B2 + 32 + i]) * __ldg(rf + 32 + i) : 0.f;
      }
    } else {
      // dynamic: + time feature on every gathered channel (mlp_network.py:244-247)
#pragma unroll
      for (int i = 0; i < 8; ++i) c.ch[i] = c.valid ? c.ch[i] + cst[Q_DFEAT + 3 + 8 * q + i] : 0.f;
      if (q == 3) {
#pragma unroll
        for (int i = 0; i < 3; ++i) c.ch[8 + i] = c.valid ? c.ch[8 + i] + cst[Q_DFEAT + i] : 0.f;
      }
    }
    // pooling weights (every quad thread)
    float w1;
    if (ST && a.anti_alias) {
      const float e = ex2f(cst[Q_MISC + 2] * (c.rd[3] - 1.f) * 1.4426950408889634f);
      const float emin = group_min<VP>(c.valid ? e : INFINITY);
      w1 = c.valid ? (e - emin) * c.mask : 0.f;
    } else {
      w1 = c.mask;
    }
    w1 = w1 / (group_sum<VP>(w1) + 1e-8f);
    c.w1 = w1;
    // [mean8 | var8 | feat8] per 8-slot group; static: quad 0 owns groups 0-2, quads 1-3 two groups each;
    // dynamic: quads 0-2 one group, quad 3 two
    const int ngroups = ST ? (q == 0 ? 3 : 2) : (q == 3 ? 2 : 1);
    const int gbase = ST ? (q == 0 ? 0 : 1 + 2 * q) : q;
#pragma unroll
    for (int g = 0; g < 3; ++g) {
      if (g >= ngroups) break;
      float o[24];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float fv = c.ch[8 * g + j];
        const float s1 = group_sum<VP>(w1 * fv);
        const float d = fv - s1;
        const float s2 = group_sum<VP>(w1 * d * d);
        o[j] = s1; o[8 + j] = s2; o[16 + j] = fv;
      }
      // bias columns of base_fc.0 (hi, lo): the last (unused) slot of quad 3
      if (q == 3 && g == 1) { o[7] = 1.f; o[15] = 1.f; }
      const int col = 24 * (gbase + g);
      store8(c.arow, col, o);
      store8(c.arow, col + 8, o + 8);
      store8(c.arow, col + 16, o + 16);
    }
    // zero the K padding (static: columns 216..223, dynamic: 120..127)
    if (q == (ST ? 1 : 0)) {
      float z[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      store8(c.arow, ST ? 216 : 120, z);
    }
    q_ready(c);
  }

  // ---- F3: ELU(base_fc.0), this quad's 64 columns ----
  __device__ __forceinline__ void f3_epilogue(QCtx& c) const {
    q_wait(c);
    elu_log2_32_to_A(c.arow, c.tacc, 64 * q);
    elu_log2_32_to_A(c.arow, c.tacc, 64 * q + 32);
    q_ready(c);
  }

  // ---- F4: x = ELU(base_fc.2) -> TMEM [128,256); A = x * w1 ----
  __device__ __forceinline__ void f4_epilogue(QCtx& c) const {
    q_wait(c);
    const int cb = 32 * q;
    float acc[32];
    tmem_ld32(c.tacc + cb, acc);
    tmem_wait_ld();
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = elu_fast(acc[i] + cst[Q_B4 + cb + i]);
    tmem_st32(c.tacc + 128 + cb, acc);
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] *= c.w1;
#pragma unroll
    for (int g = 0; g < 4; ++g) store8(c.arow, cb + 8 * g, acc + 8 * g);
    tmem_wait_st();
    q_ready(c);
  }

  // ---- F5: h = ELU(vis_fc.0) -> A; partial visibility logit ----
  __device__ __forceinline__ void f5_epilogue(QCtx& c, int T) const {
    q_wait(c);
    const int cb = 32 * q;
    float acc[32];
    tmem_ld32(c.tacc + cb, acc);
    tmem_wait_ld();
    float part = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      acc[i] = elu_fast(acc[i] + cst[Q_B5 + cb + i]);
      part = fmaf(acc[i], cst[Q_W6V + cb + i], part);
    }
#pragma unroll
    for (int g = 0; g < 4; ++g) store8(c.arow, cb + 8 * g, acc + 8 * g);
    cst[Q_XCH5 + q * 256 + T * 128 + r] = part;
    q_ready(c);
  }

  // ---- F6: x += ELU(vis_fc.2[:128]); A = x * vis1; [static] spill x for the blending head ----
  __device__ __forceinline__ void f6_epilogue(QCtx& c, int it, int T) const {
    q_wait(c);
    // all four quads arrived on a_ready before this MMA ran: the partial logits are visible
    const int xr = T * 128 + r;
    const float vlogit = cst[Q_MISC + 0] + ((cst[Q_XCH5 + xr] + cst[Q_XCH5 + 256 + xr]) +
                                            (cst[Q_XCH5 + 512 + xr] + cst[Q_XCH5 + 768 + xr]));
    const float vis1 = sigmoid_fast(elu_fast(vlogit)) * c.mask;
    const int cb = 32 * q;
    float acc[32], xs[32];
    tmem_ld32(c.tacc + cb, acc);
    tmem_ld32(c.tacc + 128 + cb, xs);
    tmem_wait_ld();
#pragma unroll
    for (int i = 0; i < 32; ++i) xs[i] += elu_fast(acc[i] + cst[Q_B6 + cb + i]);
    tmem_st32(c.tacc + 128 + cb, xs);
    if (ST) {
      // bf16 tile image in view-slot row order: the blending head lands it with one bulk copy per 128 rows
      uint8_t* xo = reinterpret_cast<uint8_t*>(a.X) +
                    tile_image_off((long long)it * 256 + T * 128 + r, cb >> 3, 16);
#pragma unroll
      for (int i = 0; i < 4; ++i)
        *reinterpret_cast<uint4*>(xo + i * 2048) =
            make_uint4(pack_bf16x2(xs[8 * i], xs[8 * i + 1]), pack_bf16x2(xs[8 * i + 2], xs[8 * i + 3]),
                       pack_bf16x2(xs[8 * i + 4], xs[8 * i + 5]), pack_bf16x2(xs[8 * i + 6], xs[8 * i + 7]));
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) xs[i] *= vis1;
#pragma unroll
    for (int g = 0; g < 4; ++g) store8(c.arow, cb + 8 * g, xs + 8 * g);
    tmem_wait_st();
    q_ready(c);
  }

  // ---- F7: vis2 = sigmoid(vis_fc2.2 . ELU(vis_fc2.0)) * mask; second pooling -> G ----
  __device__ __forceinline__ void f7_pool2(QCtx& c, int T) const {
    q_wait(c);
    const int cb = 32 * q;
    {
      float acc[32];
      tmem_ld32(c.tacc + cb, acc);
      tmem_wait_ld();
      float part = 0.f;
#pragma unroll
      for (int i = 0; i < 32; ++i) part = fmaf(elu_fast(acc[i] + cst[Q_B7 + cb + i]), cst[Q_W8 + cb + i], part);
      cst[Q_XCH7 + q * 256 + T * 128 + r] = part;
    }
    quad_sync(quadrant);
    const int xr = T * 128 + r;
    const float v2 = cst[Q_MISC + 1] + ((cst[Q_XCH7 + xr] + cst[Q_XCH7 + 256 + xr]) +
                                        (cst[Q_XCH7 + 512 + xr] + cst[Q_XCH7 + 768 + xr]));
    const float vis2 = sigmoid_fast(v2) * c.mask;
    if (ST && c.valid && q == 0) a.vis2[c.m] = vis2;
    const float vsum = group_sum<VP>(vis2);
    const float w2 = vis2 / (vsum + 1e-8f);
    const float W = group_sum<VP>(w2);
    const float nval = group_sum<VP>(c.mask);
    // reduce-scatter of sum(w x), sum(w x^2) over the point's view lanes: this quad's 32 channels
    const bool b0 = gl & 1, b1 = gl & 2, b2 = gl & 4, b3 = gl & 8;
    constexpr int NO = VP == 16 ? 2 : 4;
    const int cbase = cb + (b0 ? 16 : 0) + (b1 ? 8 : 0) + (b2 ? 4 : 0) + ((VP == 16 && b3) ? 2 : 0);
    float mean[NO], sq[NO];
    float xs[32];
    tmem_ld32(c.tacc + 128 + cb, xs);
    tmem_wait_ld();
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      float s0[32], s1[16], s2[8], s3[4];
#pragma unroll
      for (int i = 0; i < 32; ++i) s0[i] = k ? w2 * xs[i] * xs[i] : w2 * xs[i];
      rs_step<32>(s0, s1, b0, 1);
      rs_step<16>(s1, s2, b1, 2);
      rs_step<8>(s2, s3, b2, 4);
      float* dst = k ? sq : mean;
      if (VP == 16) {
        float s4[2];
        rs_step<4>(s3, s4, b3, 8);
#pragma unroll
        for (int i = 0; i < NO; ++i) dst[i] = s4[i < 2 ? i : 0];
      } else {
#pragma unroll
        for (int i = 0; i < NO; ++i) dst[i] = s3[i < 4 ? i : 0];
      }
    }
    if (c.pt_ok) {
      // pooled statistics as the bf16 tile image of geometry_fc's operand (34 k-groups:
      // mean 0..127 | var 128..255 | weight 256 | zero pad), rows = points
      uint8_t* gi = reinterpret_cast<uint8_t*>(a.G);
      float mu[NO], vr[NO];
#pragma unroll
      for (int i = 0; i < NO; ++i) {
        mu[i] = mean[i];
        vr[i] = sq[i] - mu[i] * mu[i] * (2.f - W);
      }
      uint8_t* pm = gi + tile_image_off(c.pl, cbase >> 3, 34) + (cbase & 7) * 2;
      uint8_t* pv = gi + tile_image_off(c.pl, 16 + (cbase >> 3), 34) + (cbase & 7) * 2;
      if (NO == 4) {
        *reinterpret_cast<uint2*>(pm) = make_uint2(pack_bf16x2(mu[0], mu[1]), pack_bf16x2(mu[2 % NO], mu[3 % NO]));
        *reinterpret_cast<uint2*>(pv) = make_uint2(pack_bf16x2(vr[0], vr[1]), pack_bf16x2(vr[2 % NO], vr[3 % NO]));
      } else {
        *reinterpret_cast<uint32_t*>(pm) = pack_bf16x2(mu[0], mu[1]);
        *reinterpret_cast<uint32_t*>(pv) = pack_bf16x2(vr[0], vr[1]);
      }
      if (gl == 0 && q == 0) {
        *reinterpret_cast<uint4*>(gi + tile_image_off(c.pl, 32, 34)) =
            make_uint4(pack_bf16x2(W / (float)a.V, 0.f), 0u, 0u, 0u);
        *reinterpret_cast<uint4*>(gi + tile_image_off(c.pl, 33, 34)) = make_uint4(0x3F803F80u, 0u, 0u, 0u);  // 1, 1: bias columns of geometry_fc
        a.nvalid[c.pl] = nval;
      }
    }
    tc_fence_before_sync();
  }
};

template <int VP, bool ST>
__global__ void __launch_bounds__(kQThreads, 1) view_quad_kernel(const __grid_constant__ ViewFusedArgs a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* ring = smem + 2 * kQATile;
  float* cst = reinterpret_cast<float*>(ring + kQRing * kQStage);
  uint64_t* bars = reinterpret_cast<uint64_t*>(cst + kQConst);
  uint32_t* tmem_slot = reinterpret_cast<uint32_t*>(bars + 24);
  const int tid = threadIdx.x, warp = tid >> 5;
  const uint32_t bar0 = smem_u32(bars);
  __shared__ __align__(16) FusedChunk s_tab[kMaxChunks];
  stage_chunks(s_tab, a.chunks, a.nchunks);

  if (tid == 0) init_barriers(bar0, /*pp=*/true, /*arrivals=*/512, kQRing);
  {
    const float* prm = a.params;
    for (int i = tid; i < 128; i += blockDim.x) {
      cst[Q_B4 + i] = prm[a.o_b4 + i];
      cst[Q_B5 + i] = prm[a.o_b5 + i];
      cst[Q_B6 + i] = prm[a.o_b6 + i];
      cst[Q_W6V + i] = prm[a.o_w6 + 128 * 128 + i];
      cst[Q_B7 + i] = prm[a.o_b7 + i];
      cst[Q_W8 + i] = prm[a.o_w8 + i];
    }
    if (tid < 48) cst[Q_B2 + tid] = (ST && tid < kF) ? prm[a.o_b2 + tid] : 0.f;
    if (tid < 40) cst[Q_DFEAT + tid] = (!ST && tid < kF) ? a.dfeat[tid] : 0.f;
    if (tid == 0) {
      cst[Q_MISC + 0] = prm[a.o_b6 + 128];
      cst[Q_MISC + 1] = prm[a.o_b8];
      cst[Q_MISC + 2] = (ST && a.o_s >= 0) ? fabsf(prm[a.o_s]) : 0.f;
    }
  }
  if (warp == W_ISSUE) tmem_alloc(smem_u32(tmem_slot), 512);
  tc_fence_before_sync();
  __syncthreads();
  tc_fence_after_sync();
  const uint32_t tmem_base = *tmem_slot;

  const long long n_rows = a.P * VP;
  const int n_iter = (int)((n_rows + 255) / 256);

  if (warp == W_PROD) {
    if ((tid & 31) < a.producers)
      producer_loop<true, kQRing, kQStage>(s_tab, a.nchunks, a.wimg, n_iter, ring, bar0, tid & 31, a.producers);
  } else if (warp >= W_ISSUE) {
    issuer_loop<true, 2, kQRing, kQStage>(s_tab, a.nchunks, n_iter, smem, ring, bar0, tmem_base, kQATile,
                                          a.dbg ? a.dbg + 256 : nullptr);
  } else {
    QuadOps<VP, ST> ops{a, cst, warp >> 2, warp & 3, (warp & 3) * 32 + (tid & 31), 0, 0, a.w_img, a.h_img, false};
    ops.v = ops.r % VP;
    ops.gl = ops.r & (VP - 1);
    ops.want_rgb = (ops.q == 3) || (ST && a.mask_rgb);
    QCtx c0, c1;
    c0.arow = smem + (ops.r >> 3) * 128 + (ops.r & 7) * 16;
    c1.arow = c0.arow + kQATile;
    c0.tacc = tmem_addr(tmem_base, (uint32_t)(ops.quadrant * 32), 0u);
    c1.tacc = c0.tacc + 256u;
    c0.b_ready = bar_aready(bar0, 0, kQRing); c0.b_acc = bar_acc(bar0, 0, kQRing);
    c1.b_ready = bar_aready(bar0, 1, kQRing); c1.b_acc = bar_acc(bar0, 1, kQRing);
    c0.acc_cnt = 0; c1.acc_cnt = 0;

    // profiling hook (dyn_debug_set_view_timestamps): clock64() of block 0, row 0 of every quad
    int dbg_n = 0;
    const bool dbg_on = a.dbg != nullptr && blockIdx.x == 0 && ops.r == 0;
#define TS()                                                              \
  do {                                                                    \
    if (dbg_on && dbg_n < 64) a.dbg[ops.q * 64 + dbg_n++] = clock64();    \
  } while (0)
    for (int it = blockIdx.x; it < n_iter; it += gridDim.x) {
      TS();  // 0
      if (ST) {
        ops.geometry(c0, it, 0);
        ops.gather_issue(c0);
        TS();  // 1
        ops.geometry(c1, it, 1);     // tile 0: taps in flight, ray_dir_fc.0 on the tensor cores
        TS();  // 2
        ops.gather_consume(c0);
        ops.gather_issue(c1);
        TS();  // 3
        ops.f1_epilogue(c0);         // tile 1: taps in flight
        TS();  // 4
        ops.gather_consume(c1);
        ops.f1_epilogue(c1);
        TS();  // 5
      } else {
        ops.geometry(c0, it, 0);
        ops.gather_issue(c0);
        ops.geometry(c1, it, 1);
        ops.gather_consume(c0);
        ops.gather_issue(c1);
        TS();  // 1
      }
      ops.pool1(c0);
      TS();  // 6 (dynamic: 2)
      if (!ST) ops.gather_consume(c1);
      ops.pool1(c1);
      TS();  // 7
      ops.f3_epilogue(c0);
      TS();  // 8
      ops.f3_epilogue(c1);
      TS();  // 9
      ops.f4_epilogue(c0);
      TS();  // 10
      ops.f4_epilogue(c1);
      TS();  // 11
      ops.f5_epilogue(c0, 0);
      TS();  // 12
      ops.f5_epilogue(c1, 1);
      TS();  // 13
      ops.f6_epilogue(c0, it, 0);
      TS();  // 14
      ops.f6_epilogue(c1, it, 1);
      TS();  // 15
      ops.f7_pool2(c0, 0);
      TS();  // 16
      ops.f7_pool2(c1, 1);
      TS();  // 17
    }
#undef TS
  }
  __syncthreads();
  if (warp == W_ISSUE) {
    tc_fence_after_sync();
    tmem_dealloc(tmem_base, 512);
  }
}

}  // namespace

// ---------------------------------------------------------------------------
// host: weight images in the quad column layouts
// ---------------------------------------------------------------------------
size_t view_quad_bytes(int kind) { (void)kind; return (size_t)(512 * 1024); }

int view_quad_build(dyn_net* n, const float* P, void* dst_dev, size_t dst_bytes, cudaStream_t st) {
  std::vector<uint8_t> img;
  std::vector<FusedChunk> tab;
  constexpr float kLog2e = 1.4426950408889634f, kLn2 = 0.6931471805599453f;
  auto add = [&](const LinearP& l, int N, int Npad, int Kpad, std::vector<int> map, float scale = 1.f,
                 bool fold_bias = false) {
    HostLayer L;
    L.W = P + l.w; L.N = N; L.Kw = l.in; L.Npad = Npad; L.Kpad = Kpad; L.colmap = std::move(map);
    L.scale = scale;
    if (fold_bias) L.bias = P + l.b;
    append_layer(L, img, tab, 0, 0, 9, true, kQStage);
  };
  if (n->kind == DYN_NET_STATIC) {
    const StaticLayout& L = n->sl;
    // layer 1 (K = 128): quad q < 3 holds PE components 3q..3q+2 at [40q, 40q+33); [120,128) = ray_diff, 1, 1
    std::vector<int> m1(128, -1);
    auto comp_col = [](int ci, int j) {  // j: 0 = x, 1..5 = cos f_k, 6..10 = sin f_k
      if (ci < 3) return j == 0 ? ci : (j <= 5 ? 3 + 3 * (j - 1) + ci : 18 + 3 * (j - 6) + ci);
      const int d = ci - 3;
      return j == 0 ? 33 + d : (j <= 5 ? 39 + 6 * (j - 1) + d : 69 + 6 * (j - 6) + d);
    };
    for (int q = 0; q < 3; ++q)
      for (int c = 0; c < 3; ++c)
        for (int j = 0; j < 11; ++j) m1[40 * q + 11 * c + j] = comp_col(3 * q + c, j);
    for (int i = 0; i < 4; ++i) m1[120 + i] = 99 + i;
    m1[124] = kBiasHi; m1[125] = kBiasLo;
    add(L.ray_dir0, 256, 256, 128, m1, kLog2e, true);              // ELU on the exp2 scale
    add(L.ray_dir2, kF, 48, 256, identity_map(256, 256), kLn2);    // consumes log2(e) * ELU
    // layer 3 (K = 224): 9 groups of [mean8 | var8 | feat8]; quad 0 groups 0-2, quad q groups 2q+1, 2q+2
    std::vector<int> m3(224, -1);
    auto chan = [](int q, int s) {  // concat channel (0..69) of a quad's slot, -1 = pad
      if (q == 0) return s < 8 ? 3 + s : 35 + (s - 8);
      if (q == 1) return s < 8 ? 11 + s : 51 + (s - 8);
      if (q == 2) return s < 8 ? 19 + s : 59 + (s - 8);
      return s < 8 ? 27 + s : (s < 11 ? s - 8 : (s < 14 ? 67 + (s - 11) : -1));
    };
    for (int q = 0; q < 4; ++q) {
      const int ns = q == 0 ? 24 : 16, gbase = q == 0 ? 0 : 1 + 2 * q;
      for (int s = 0; s < ns; ++s) {
        const int c = chan(q, s);
        if (c < 0) continue;
        const int base = 24 * (gbase + s / 8) + (s % 8);
        m3[base] = c; m3[base + 8] = 70 + c; m3[base + 16] = 140 + c;
      }
    }
    m3[24 * 8 + 7] = kBiasHi; m3[24 * 8 + 15] = kBiasLo;  // quad 3, slot 15 (unused): mean / var columns
    add(L.base0, 256, 256, 224, m3, kLog2e, true);
    add(L.base2, 128, 128, 256, identity_map(256, 256), kLn2);
    add(L.vis0, 128, 128, 128, identity_map(128, 128));
    add(L.vis2, 128, 128, 128, identity_map(128, 128));
    add(L.vis2_0, 128, 128, 128, identity_map(128, 128));
  } else {
    const DynamicLayout& L = n->dl;
    // K = 128: group q = [mean8 | var8 | feat8] of feature channels 8q..8q+7 (concat channel 3 + 8q + j);
    // group 4 (quad 3): rgb in slots 0..2, bias in slot 7
    std::vector<int> m3(128, -1);
    for (int q = 0; q < 4; ++q)
      for (int j = 0; j < 8; ++j) {
        const int c = 3 + 8 * q + j, b = 24 * q + j;
        m3[b] = c; m3[b + 8] = 35 + c; m3[b + 16] = 70 + c;
      }
    for (int j = 0; j < 3; ++j) { const int b = 24 * 4 + j; m3[b] = j; m3[b + 8] = 35 + j; m3[b + 16] = 70 + j; }
    m3[24 * 4 + 7] = kBiasHi; m3[24 * 4 + 15] = kBiasLo;
    add(L.base0, 256, 256, 128, m3, kLog2e, true);
    add(L.base2, 128, 128, 256, identity_map(256, 256), kLn2);
    add(L.vis0, 128, 128, 128, identity_map(128, 128));
    add(L.vis2, 128, 128, 128, identity_map(128, 128));
    add(L.vis2_0, 128, 128, 128, identity_map(128, 128));
  }
  const size_t img_bytes = (img.size() + 255) & ~(size_t)255;
  const size_t need = img_bytes + tab.size() * sizeof(FusedChunk);
  if (need > dst_bytes) return fail(DYN_E_INVALID, "quad images need %zu bytes, have %zu", need, dst_bytes);
  if (tab.size() > (size_t)kMaxChunks) return fail(DYN_E_INVALID, "chunk table too long (%zu)", tab.size());
  DYN_CUDA(cudaMemcpyAsync(dst_dev, img.data(), img.size(), cudaMemcpyHostToDevice, st));
  DYN_CUDA(cudaMemcpyAsync(reinterpret_cast<char*>(dst_dev) + img_bytes, tab.data(),
                           tab.size() * sizeof(FusedChunk), cudaMemcpyHostToDevice, st));
  DYN_CUDA(cudaStreamSynchronize(st));
  n->quad.img = dst_dev;
  n->quad.tab = reinterpret_cast<const FusedChunk*>(reinterpret_cast<char*>(dst_dev) + img_bytes);
  n->quad.nchunks = (int)tab.size();
  return DYN_OK;
}

int view_quad_prepare() {
#define PREP(VPV, STV) \
  DYN_CUDA(cudaFuncSetAttribute(view_quad_kernel<VPV, STV>, cudaFuncAttributeMaxDynamicSharedMemorySize, kQSmem))
  PREP(8, true); PREP(16, true); PREP(8, false); PREP(16, false);
#undef PREP
  return DYN_OK;
}

int launch_view_quad(const dyn_net* n, ViewFusedArgs& a, int V, cudaStream_t st) {
  if (n->quad.img == nullptr) return fail(DYN_E_INVALID, "net has no quad per-view images");
  a.wimg = n->quad.img;
  a.chunks = n->quad.tab;
  a.nchunks = n->quad.nchunks;
  a.ablate = 0;
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    DYN_CUDA(cudaGetDevice(&dev));
    DYN_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    int rc = view_quad_prepare();
    if (rc) { sms = 0; return rc; }
  }
  const int VP = V <= 8 ? 8 : 16;
  const long long n_iter = (a.P * VP + 255) / 256;
  const int grid = (int)(n_iter < sms ? n_iter : sms);
  if (grid == 0) return DYN_OK;
  const int rc = bind_acc_pool();
  if (rc) return rc;
  const bool st_net = n->kind == DYN_NET_STATIC;
  ProfScope prof(st_net ? PROF_VIEW_ST : PROF_VIEW_DY, st);
  if (st_net) {
    if (VP == 8) view_quad_kernel<8, true><<<grid, kQThreads, kQSmem, st>>>(a);
    else view_quad_kernel<16, true><<<grid, kQThreads, kQSmem, st>>>(a);
  } else {
    if (VP == 8) view_quad_kernel<8, false><<<grid, kQThreads, kQSmem, st>>>(a);
    else view_quad_kernel<16, false><<<grid, kQThreads, kQSmem, st>>>(a);
  }
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

}  // namespace dyn
