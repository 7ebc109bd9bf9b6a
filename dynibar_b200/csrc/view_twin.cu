// Fused per-(point, view) stage of the two aggregation networks on the tensor cores (reference:
// ibrnet/projection.py:103-176, ibrnet/mlp_network.py:236-284 (dynamic) / :423-497 (static)).
// Per 128-row tile, without leaving the SM:
//
//   projection + in-front/in-bounds masks + view-angle difference   (a4, a6)
//   bilinear gather of source RGB + features from L2-resident maps  (a5)
//   [static]  Plucker coords, positional encodings, ray_dir_fc     (a7, a8, a10)
//   pooling weights, weighted mean/var over views (warp shuffles)  (a9/a10)
//   base_fc -> vis_fc -> vis_fc2 (tensor cores, fp32 accum in TMEM)
//   visibility re-weighting and the second mean/var pooling -> G (bf16 tile image) per point
//
// Engine: fused_engine.cuh (operand tile in shared memory written by the epilogues, accumulators
// in TMEM, weights streamed through a cp.async.bulk ring, table-driven MMA warpgroup).  Every row is
// served by TWO threads in twin warps w and w + 4 (same TMEM lane quadrant), which is what the
// latency-bound epilogues need; each twin owns half of every layer's output columns and half of the
// gathered / pooled channels, and the twins exchange only two scalars per row and iteration (the
// partial visibility logits).
//
// One CTA per SM with one 128-row tile:
//   warps 0-3  : twin 0 (quadrant = w & 3)  warps 4-7 : twin 1 of the same rows
//   warps 8-11 : MMA warpgroup (wgmma)      warp 12   : weight producer
//
// Latency hiding inside a CTA: the source views are read in
// their packed per-frame layouts (bf16 channels-last features: 2 x 16-byte loads per tap and twin; RGBA
// fp32 images: 1 load per tap), the taps are ISSUED right after the projection and consumed after the
// positional-encoding operand has been built and handed to the tensor cores, the per-ray reference
// feature is loaded before the wait for ray_dir_fc.2, the next iteration's points before the last wait,
// and the camera matrices sit in shared memory (lanes of a warp index different views).
#include "fused_engine.cuh"
#include "geometry.cuh"
#include "nets.cuh"

namespace dyn {

using namespace tc;
using namespace fe;

namespace {

constexpr int kTwinATile = 69632;  // K <= 256 (+ one k-step of bias columns): 34 k-groups
// T_B5 / T_B7 hold log2(e) * bias, T_W6V / T_W8 hold ln(2) * weight (the hidden activations of vis_fc.0 and
// vis_fc2.0 live on the exp2 scale); the biases of base_fc.2 and vis_fc.2 ride in the MMA
constexpr int T_B2 = 0, T_B5 = 48, T_W6V = 176, T_B7 = 304, T_W8 = 432, T_MISC = 560, T_DFEAT = 576,
              T_CAMS = 624 /* 16 views x (P 12 + centre 3 + pad) */, T_XCH = T_CAMS + 256;  // + 2 x [2][128] exchange
constexpr int kTwinConst = T_XCH + 512;
// two 8 KB weight stages leave room for TMEM in shared memory
constexpr int kTwinStage = 8192;
constexpr int kTwinRing = 2;
constexpr int kTwinThreads = 256 + 32 * (kIssuerWarps + 1);
// shared memory: operand tile | weight ring | constants | barriers (256 B) | accumulator memory (one tile)
constexpr int kTwinSmem = kTwinATile + kTwinRing * kTwinStage + kTwinConst * 4 + 256 + kAccSmemBytes;

__device__ __forceinline__ void pair_sync(int pair) {
  asm volatile("bar.sync %0, 64;" ::"r"(pair + 1) : "memory");
}

// 11 values of one PE component: [x, cos(2^k x) k=0..4, sin(2^k x) k=0..4]
__device__ __forceinline__ void pe_comp(float x, float* o) {
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

// layers whose bias rides in the MMA and whose accumulator is on the exp2 scale (F1, F3)
template <int N>
__device__ __forceinline__ void elu_log2_block_to_A(uint8_t* arow, uint32_t tacc, int col0) {
#pragma unroll 1
  for (int cb = 0; cb < N; cb += 32) {
    float acc[32];
    tmem_ld32(tacc + col0 + cb, acc);
    tmem_wait_ld();
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = elu_log2(acc[i]);
#pragma unroll
    for (int g = 0; g < 4; ++g) store8(arow, col0 + cb + 8 * g, acc + 8 * g);
  }
}

template <int N>
__device__ __forceinline__ void elu_block_to_A(uint8_t* arow, uint32_t tacc, int col0, const float* bias) {
#pragma unroll 1
  for (int cb = 0; cb < N; cb += 32) {
    float acc[32];
    tmem_ld32(tacc + col0 + cb, acc);
    tmem_wait_ld();
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = elu_fast(acc[i] + bias[col0 + cb + i]);
#pragma unroll
    for (int g = 0; g < 4; ++g) store8(arow, col0 + cb + 8 * g, acc + 8 * g);
  }
}

template <int VP, bool ST>
__global__ void __launch_bounds__(kTwinThreads, 1) view_twin_kernel(const __grid_constant__ ViewFusedArgs a) {
  constexpr int ROWS = 128;  // rows per iteration
  constexpr int RING = kTwinRing;
  constexpr int W_ISSUE = 8, W_PROD = 8 + kIssuerWarps;  // MMA warpgroup, weight producer
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* ring = smem + kTwinATile;
  float* cst = reinterpret_cast<float*>(ring + RING * kTwinStage);
  uint64_t* bars = reinterpret_cast<uint64_t*>(cst + kTwinConst);
  uint32_t* tmem_slot = reinterpret_cast<uint32_t*>(bars + 24);
  const int tid = threadIdx.x, warp = tid >> 5;
  const uint32_t bar0 = smem_u32(bars);
  __shared__ __align__(16) FusedChunk s_tab[kMaxChunks];
  stage_chunks(s_tab, a.chunks, a.nchunks);

  if (tid == 0) init_barriers(bar0, /*arrivals=*/256, RING);
  {
    const float* prm = a.params;
    for (int i = tid; i < 256; i += blockDim.x) {  // camera matrices: lanes index them by view
      const int vv = i >> 4, j = i & 15;
      cst[T_CAMS + i] = j < 12 ? a.cams.P[vv][j] : (j < 15 ? a.cams.center[vv][j - 12] : 0.f);
    }
    for (int i = tid; i < 128; i += blockDim.x) {
      cst[T_B5 + i] = prm[a.o_b5 + i] * 1.4426950408889634f;
      cst[T_W6V + i] = prm[a.o_w6 + 128 * 128 + i] * 0.6931471805599453f;
      cst[T_B7 + i] = prm[a.o_b7 + i] * 1.4426950408889634f;
      cst[T_W8 + i] = prm[a.o_w8 + i] * 0.6931471805599453f;
    }
    if (tid < 48) cst[T_B2 + tid] = (ST && tid < kF) ? prm[a.o_b2 + tid] : 0.f;
    if (tid < 40) cst[T_DFEAT + tid] = (!ST && tid < kF) ? a.dfeat[tid] : 0.f;
    if (tid == 0) {
      cst[T_MISC + 0] = prm[a.o_b6 + 128];
      cst[T_MISC + 1] = prm[a.o_b8];
      cst[T_MISC + 2] = (ST && a.o_s >= 0) ? fabsf(prm[a.o_s]) : 0.f;
    }
  }
  if (warp == W_ISSUE) tmem_alloc_smem(smem_u32(tmem_slot), smem + kTwinSmem - kAccSmemBytes);
  tc_fence_before_sync();
  __syncthreads();
  tc_fence_after_sync();
  const uint32_t tmem_base = *tmem_slot;

  const long long n_rows = a.P * VP;
  const int n_iter = (int)((n_rows + ROWS - 1) / ROWS);

  if (warp == W_PROD) {
    if ((tid & 31) == 0) producer_loop<RING, kTwinStage>(s_tab, a.nchunks, a.wimg, n_iter, ring, bar0);
  } else if (warp >= W_ISSUE) {
    issuer_loop<RING, kTwinStage>(s_tab, a.nchunks, n_iter, smem, ring, bar0, tmem_base,
                                  a.dbg ? a.dbg + 128 : nullptr);
  } else {
    const int tw = tid >> 7, t = tid & 127;  // twin index, row of the tile
    uint8_t* arow = smem + (t >> 3) * 128 + (t & 7) * 16;
    const uint32_t tacc = tmem_addr(tmem_base, (uint32_t)((warp & 3) * 32), 0u);
    const int v = t % VP;
    const int gl = t & (VP - 1);
    const int pair = warp & 3;
    float* xch5 = cst + T_XCH;        // [2][128] partial visibility logits of vis_fc
    float* xch7 = cst + T_XCH + 256;  // [2][128] partial logits of vis_fc2
    if (tw == 0) {
      // persistent bias columns of base_fc.2 (K = 256 + 16): k-groups 32, 33 = [1, 1, 0 ...] (hi, lo)
      float o[8] = {1.f, 1.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, z[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      store8(arow, 256, o);
      store8(arow, 264, z);
    }
    uint32_t acc_cnt = 0;
    const float wh = a.w_img, hh = a.h_img;
    int dbg_n = 0;
#define TS()                                                                            \
  do {                                                                                  \
    if (a.dbg != nullptr && blockIdx.x == 0 && t == 0 && dbg_n < 64)                 \
      a.dbg[tw * 64 + dbg_n++] = clock64();                                             \
  } while (0)
    constexpr int NG = ST ? 5 : (0);  // static: 5 channel groups per twin (set below for dynamic)
    (void)NG;

    // the first point of this thread; later ones are fetched one iteration ahead (before the last MMA wait)
    float np3[3], nq3[3];
    auto fetch_point = [&](int it2) {
      const long long pl2 = ((long long)it2 * ROWS + t) / VP;
      np3[0] = 0.f; np3[1] = 0.f; np3[2] = 0.f;
      if (pl2 < a.P) { np3[0] = a.pts[pl2 * 3]; np3[1] = a.pts[pl2 * 3 + 1]; np3[2] = a.pts[pl2 * 3 + 2]; }
      nq3[0] = np3[0]; nq3[1] = np3[1]; nq3[2] = np3[2];
      if (!ST && pl2 < a.P && v < a.V) {
        const float* q = a.pts_seq + ((long long)v * a.seq_stride + pl2) * 3;
        nq3[0] = q[0]; nq3[1] = q[1]; nq3[2] = q[2];
      }
    };
    if ((int)blockIdx.x < n_iter) fetch_point((int)blockIdx.x);
    const bool want_rgb = (tw == 0) || (ST && a.mask_rgb);

    for (int it = blockIdx.x; it < n_iter; it += gridDim.x) {
      const long long pl = ((long long)it * ROWS + t) / VP;
      const bool pt_ok = pl < a.P;
      const bool valid = pt_ok && v < a.V;
      const long long m = pl * a.V + v;
      const long long ray = pt_ok ? pl / a.S : 0;

      TS();  // 0: iteration start
      // ---- geometry (both twins; cheap) ----
      const float p3[3] = {np3[0], np3[1], np3[2]}, q3[3] = {nq3[0], nq3[1], nq3[2]};
      const int vc = valid ? v : 0;
      const float* cam = cst + T_CAMS + 16 * vc;  // P (12) | centre (3)
      float pu, pv;
      bool front;
      project_point(cam, q3[0], q3[1], q3[2], pu, pv, front);
      const bool inb = (pu <= wh - 1.f) && (pu >= 0.f) && (pv <= hh - 1.f) && (pv >= 0.f);
      const float mask_proj = (valid && inb && front) ? 1.f : 0.f;

      // ---- issue the bilinear taps now: 2 x 16 B per tap of this twin's 16 bf16 feature channels
      //      (+ 1 x 16 B RGBA); they are consumed after the ray_dir_fc.0 operand has been built ----
      uint4 tf[8];
      float4 tr[4];
      float tw4[4], twr[4];
      {
        const float gx = 2.f * pu / (wh - 1.f) - 1.f, gy = 2.f * pv / (hh - 1.f) - 1.f;
        {
          const float fx = (gx + 1.f) * 0.5f * (float)(a.w - 1), fy = (gy + 1.f) * 0.5f * (float)(a.h - 1);
          const float x0f = floorf(fx), y0f = floorf(fy);
          const int x0 = (int)x0f, y0 = (int)y0f;
          const float ax = fx - x0f, ay = fy - y0f, bx = (x0f + 1.f) - fx, by = (y0f + 1.f) - fy;
          const uint16_t* base = a.feat_bf + (long long)vc * a.h * a.w * kC + 16 * tw;
#pragma unroll
          for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) {
              // out-of-range taps (and padding rows) load a clamped texel with weight 0: no branch, all loads
              // of this thread are in flight together
              const int xi = x0 + dx, yi = y0 + dy;
              const bool in = valid && xi >= 0 && xi < a.w && yi >= 0 && yi < a.h;
              tw4[2 * dy + dx] = in ? (dx ? ax : bx) * (dy ? ay : by) : 0.f;
              const int xc = min(max(xi, 0), a.w - 1), yc = min(max(yi, 0), a.h - 1);
              const uint4* tp = reinterpret_cast<const uint4*>(base + ((long long)yc * a.w + xc) * kC);
              tf[2 * (2 * dy + dx)] = __ldg(tp);
              tf[2 * (2 * dy + dx) + 1] = __ldg(tp + 1);
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
              const bool in = valid && xi >= 0 && xi < a.W && yi >= 0 && yi < a.H;
              twr[2 * dy + dx] = in ? (dx ? ax : bx) * (dy ? ay : by) : 0.f;
              const int xc = min(max(xi, 0), a.W - 1), yc = min(max(yi, 0), a.H - 1);
              tr[2 * dy + dx] = __ldg(reinterpret_cast<const float4*>(base + ((long long)yc * a.W + xc) * 4));
            }
        }
      }

      float rd[4];
      {
        float a0 = a.cams.tgt[0] - p3[0], a1 = a.cams.tgt[1] - p3[1], a2 = a.cams.tgt[2] - p3[2];
        normalize3(a0, a1, a2);
        float b0 = cam[12] - q3[0], b1 = cam[13] - q3[1], b2 = cam[14] - q3[2];
        normalize3(b0, b1, b2);
        rd[0] = a0 - b0; rd[1] = a1 - b1; rd[2] = a2 - b2;
        rd[3] = a0 * b0 + a1 * b1 + a2 * b2;
        normalize3(rd[0], rd[1], rd[2]);
      }

      if (ST) {
        // ---- layer-1 operand, 56 columns per twin (component-major PE, see view_twin_build); each
        //      8-column group is stored as soon as it is complete (short register live ranges while the
        //      taps are in flight).  Padding rows keep (finite) garbage: every use of their layer outputs
        //      is guarded by `valid` ----
        float pl6[6];
        {
          const float ox = cam[12], oy = cam[13], oz = cam[14];
          float dx = p3[0] - ox, dy = p3[1] - oy, dz = p3[2] - oz;
          normalize3(dx, dy, dz);
          pl6[0] = dx; pl6[1] = dy; pl6[2] = dz;
          pl6[3] = oy * dz - oz * dy;
          pl6[4] = oz * dx - ox * dz;
          pl6[5] = ox * dy - oy * dx;
        }
        float xin[56];
        if (tw == 0) {
          pe_comp(p3[0], xin);         store8(arow, 0, xin);
          pe_comp(p3[1], xin + 11);    store8(arow, 8, xin + 8);
          pe_comp(p3[2], xin + 22);    store8(arow, 16, xin + 16); store8(arow, 24, xin + 24);
          pe_comp(pl6[0], xin + 33);   store8(arow, 32, xin + 32);
          pe_comp(pl6[1], xin + 44);   xin[55] = 0.f;
          store8(arow, 40, xin + 40);  store8(arow, 48, xin + 48);
        } else {
          pe_comp(pl6[2], xin);        store8(arow, 56, xin);
          pe_comp(pl6[3], xin + 11);   store8(arow, 64, xin + 8);
          pe_comp(pl6[4], xin + 22);   store8(arow, 72, xin + 16); store8(arow, 80, xin + 24);
          pe_comp(pl6[5], xin + 33);   store8(arow, 88, xin + 32);
          xin[44] = rd[0]; xin[45] = rd[1]; xin[46] = rd[2]; xin[47] = rd[3];
          xin[48] = 1.f; xin[49] = 1.f;  // bias columns of ray_dir_fc.0 (hi, lo)
#pragma unroll
          for (int i = 50; i < 56; ++i) xin[i] = 0.f;
          store8(arow, 96, xin + 40);  store8(arow, 104, xin + 48);
        }
        fence_proxy_async_smem();
        tc_fence_before_sync();
        mbar_arrive(bar_aready(bar0, RING));
      }

      TS();  // 1: after F1 operand + arrive
      // ---- consume the taps: rgb (twin 0, or both when mask_rgb) + this twin's 16 feature channels ----
      float chv[40];  // this twin's pooled channels (layout in view_twin_build)
#pragma unroll
      for (int i = 0; i < 40; ++i) chv[i] = 0.f;
      float rgb[3] = {0.f, 0.f, 0.f};
      {
        const int fo = tw == 0 ? 3 : 0;  // twin 0 keeps rgb in slots 0..2
#pragma unroll
        for (int tp = 0; tp < 4; ++tp) {
          const float wgt = tw4[tp];
#pragma unroll
          for (int hlf = 0; hlf < 2; ++hlf) {
            const uint4 q = tf[2 * tp + hlf];
            const uint32_t u[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float lo = __uint_as_float(u[j] << 16), hi = __uint_as_float(u[j] & 0xffff0000u);
              if (tw == 0) {
                chv[3 + 8 * hlf + 2 * j] += lo * wgt; chv[3 + 8 * hlf + 2 * j + 1] += hi * wgt;
              } else {
                chv[8 * hlf + 2 * j] += lo * wgt; chv[8 * hlf + 2 * j + 1] += hi * wgt;
              }
            }
          }
        }
        (void)fo;
        if (want_rgb) {
#pragma unroll
          for (int tp = 0; tp < 4; ++tp) {
            rgb[0] += tr[tp].x * twr[tp]; rgb[1] += tr[tp].y * twr[tp]; rgb[2] += tr[tp].z * twr[tp];
          }
        }
      }
      float mask = mask_proj;
      if (ST && a.mask_rgb) mask *= ((rgb[0] + rgb[1] + rgb[2]) > 1e-3f) ? 1.f : 0.f;
      if (tw == 0) {
        chv[0] = rgb[0]; chv[1] = rgb[1]; chv[2] = rgb[2];
        if (valid) {
          a.mask_proj[m] = mask_proj;
          if (ST) {
            a.mask_eff[m] = mask;
            reinterpret_cast<float4*>(a.ray_diff)[m] = make_float4(rd[0], rd[1], rd[2], rd[3]);
            a.rgb_in[m * 3] = rgb[0]; a.rgb_in[m * 3 + 1] = rgb[1]; a.rgb_in[m * 3 + 2] = rgb[2];
          }
        }
      }

      TS();  // 2: after gather
      if (ST) {
        // ---- F1 epilogue: this twin's 128 of the 256 columns ----
        mbar_wait(bar_acc(bar0, RING), acc_cnt & 1); ++acc_cnt;
        TS();  // 3: F1 acc ready
        tc_fence_after_sync();
        elu_log2_block_to_A<128>(arow, tacc, 128 * tw);
        fence_proxy_async_smem();
        tc_fence_before_sync();
        mbar_arrive(bar_aready(bar0, RING));
        TS();  // 4: F1 epilogue done
        // ---- F2: src_feat (35 of 48 columns) * ref_feat; twin 0 keeps 0..17, twin 1 keeps 18..34.
        //      The per-ray reference feature is loaded BEFORE the wait (its L2 latency hides behind the MMA) ----
        float rfv[18];
        {
          const float* rf = a.ref_feat + ray * kF + 18 * tw;
#pragma unroll
          for (int i = 0; i < 18; ++i) rfv[i] = (tw == 0 || i < 17) ? __ldg(rf + i) : 0.f;
        }
        mbar_wait(bar_acc(bar0, RING), acc_cnt & 1); ++acc_cnt;
        TS();  // 5: F2 acc ready
        tc_fence_after_sync();
        float s48[48];
        tmem_ld32(tacc, s48);
        tmem_ld16(tacc + 32, s48 + 32);
        tmem_wait_ld();
        if (tw == 0) {
#pragma unroll
          for (int i = 0; i < 18; ++i) chv[19 + i] = valid ? (s48[i] + cst[T_B2 + i]) * rfv[i] : 0.f;
        } else {
#pragma unroll
          for (int i = 0; i < 17; ++i)
            chv[16 + i] = valid ? (s48[18 + i] + cst[T_B2 + 18 + i]) * rfv[i] : 0.f;
        }
      } else {
        // dynamic: + time feature on this twin's channels (mlp_network.py:244-247)
        if (tw == 0) {
#pragma unroll
          for (int i = 0; i < 19; ++i) chv[i] = valid ? chv[i] + cst[T_DFEAT + i] : 0.f;
        } else {
#pragma unroll
          for (int i = 0; i < 16; ++i) chv[i] = valid ? chv[i] + cst[T_DFEAT + 19 + i] : 0.f;
        }
      }

      // ---- pooling weights (both twins) ----
      float w1;
      if (ST && a.anti_alias) {
        const float e = ex2f(cst[T_MISC + 2] * (rd[3] - 1.f) * 1.4426950408889634f);
        const float emin = group_min<VP>(valid ? e : INFINITY);
        w1 = valid ? (e - emin) * mask : 0.f;
      } else {
        w1 = mask;
      }
      w1 = w1 / (group_sum<VP>(w1) + 1e-8f);

      // ---- first pooling on this twin's channel groups: [mean8 | var8 | feat8] per group ----
      {
        constexpr int ng0 = ST ? 5 : 3, ng1 = ST ? 5 : 2;
        const int col_base = tw == 0 ? 0 : 24 * ng0;
#pragma unroll
        for (int g = 0; g < ng0; ++g) {
          if (tw == 1 && g >= ng1) break;
          float o[24];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float fv = chv[8 * g + j];
            const float s1 = group_sum<VP>(w1 * fv);
            const float d = fv - s1;
            const float s2 = group_sum<VP>(w1 * d * d);
            o[j] = s1; o[8 + j] = s2; o[16 + j] = fv;
          }
          // bias columns of base_fc.0 (hi, lo): the last (unused) channel slot of twin 0
          if (tw == 0 && g == ng0 - 1) { o[7] = 1.f; o[15] = 1.f; }
          store8(arow, col_base + 24 * g, o);
          store8(arow, col_base + 24 * g + 8, o + 8);
          store8(arow, col_base + 24 * g + 16, o + 16);
        }
        if (!ST && tw == 1) {  // dynamic: zero the K padding 120..127
          float z[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
          store8(arow, 120, z);
        }
      }
      fence_proxy_async_smem();
      tc_fence_before_sync();
      mbar_arrive(bar_aready(bar0, RING));

      TS();  // 6: pool1 done + arrive
      // ---- F3: ELU(base_fc.0), this twin's 128 columns ----
      mbar_wait(bar_acc(bar0, RING), acc_cnt & 1); ++acc_cnt;
      TS();  // 7: F3 acc ready
      tc_fence_after_sync();
      elu_log2_block_to_A<128>(arow, tacc, 128 * tw);
      fence_proxy_async_smem();
      tc_fence_before_sync();
      mbar_arrive(bar_aready(bar0, RING));

      const int c0 = 64 * tw;  // this twin's columns of the 128-wide layers
      TS();  // 8: F3 epilogue done
      // ---- F4: x = ELU(base_fc.2) -> TMEM [128,256); A = x (the pooling weight w1 of vis_fc.0's input is applied
      //      to the accumulator in the next epilogue: W (w1 x) = w1 (W x)); bias folded, accumulator on the exp2 scale ----
      mbar_wait(bar_acc(bar0, RING), acc_cnt & 1); ++acc_cnt;
      TS();  // 9: F4 acc ready
      tc_fence_after_sync();
#pragma unroll 1
      for (int cb = c0; cb < c0 + 64; cb += 32) {
        float acc[32];
        tmem_ld32(tacc + cb, acc);
        tmem_wait_ld();
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[i] = elu_from_log2(acc[i]);
        tmem_st32(tacc + 128 + cb, acc);
#pragma unroll
        for (int g = 0; g < 4; ++g) store8(arow, cb + 8 * g, acc + 8 * g);
      }
      if (tw == 1) {
        // bias columns of vis_fc.2 (K = 128 + 16): k-groups 16, 17 (free once this layer's MMA has read them)
        float o[8] = {1.f, 1.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, z[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        store8(arow, 128, o);
        store8(arow, 136, z);
      }
      tmem_wait_st();
      fence_proxy_async_smem();
      tc_fence_before_sync();
      mbar_arrive(bar_aready(bar0, RING));

      TS();  // 10: F4 epilogue done
      // ---- F5: h = ELU(vis_fc.0) -> A; partial visibility logit ----
      mbar_wait(bar_acc(bar0, RING), acc_cnt & 1); ++acc_cnt;
      TS();  // 11: F5 acc ready
      tc_fence_after_sync();
      {
        float part = 0.f;
#pragma unroll 1
        for (int cb = c0; cb < c0 + 64; cb += 32) {
          float acc[32];
          tmem_ld32(tacc + cb, acc);
          tmem_wait_ld();
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            acc[i] = elu_log2(fmaf(acc[i], w1, cst[T_B5 + cb + i]));  // log2(e) * ELU(w1 (W x) + b)
            part = fmaf(acc[i], cst[T_W6V + cb + i], part);
          }
#pragma unroll
          for (int g = 0; g < 4; ++g) store8(arow, cb + 8 * g, acc + 8 * g);
        }
        xch5[tw * 128 + t] = part;
      }
      fence_proxy_async_smem();
      tc_fence_before_sync();
      mbar_arrive(bar_aready(bar0, RING));

      TS();  // 12: F5 epilogue done
      // ---- F6: x += ELU(vis_fc.2[:128]); A = x * vis1 ----
      mbar_wait(bar_acc(bar0, RING), acc_cnt & 1); ++acc_cnt;
      TS();  // 13: F6 acc ready
      tc_fence_after_sync();
      // both twins arrived on a_ready before this MMA ran: the partial logits are visible
      const float vlogit = cst[T_MISC + 0] + xch5[t] + xch5[128 + t];
      const float vis1 = sigmoid_fast(elu_fast(vlogit)) * mask;
#pragma unroll 1
      for (int cb = c0; cb < c0 + 64; cb += 32) {
        float acc[32], xs[32];
        tmem_ld32(tacc + cb, acc);
        tmem_ld32(tacc + 128 + cb, xs);
        tmem_wait_ld();
#pragma unroll
        for (int i = 0; i < 32; ++i) xs[i] += elu_from_log2(acc[i]);
        tmem_st32(tacc + 128 + cb, xs);
        // bf16(x) is both vis_fc2.0's operand (vis1 is applied to its accumulator) and, for the static net,
        // the spill for the blending head (a bf16 tile image in view-slot row order, fused_engine.cuh)
        uint4 pk[4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
          pk[i] = make_uint4(pack_bf16x2(xs[8 * i], xs[8 * i + 1]), pack_bf16x2(xs[8 * i + 2], xs[8 * i + 3]),
                             pack_bf16x2(xs[8 * i + 4], xs[8 * i + 5]), pack_bf16x2(xs[8 * i + 6], xs[8 * i + 7]));
        if (ST) {
          uint8_t* xo = reinterpret_cast<uint8_t*>(a.X) + tile_image_off((long long)it * ROWS + t, cb >> 3, 16);
#pragma unroll
          for (int i = 0; i < 4; ++i) *reinterpret_cast<uint4*>(xo + i * 2048) = pk[i];
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) *reinterpret_cast<uint4*>(arow + ((cb >> 3) + i) * 2048) = pk[i];
      }
      tmem_wait_st();
      fence_proxy_async_smem();
      tc_fence_before_sync();
      mbar_arrive(bar_aready(bar0, RING));

      TS();  // 14: F6 epilogue done
      if (it + (int)gridDim.x < n_iter) fetch_point(it + (int)gridDim.x);  // next iteration's point
      // ---- F7: vis2 = sigmoid(vis_fc2.2 . ELU(vis_fc2.0)) * mask ----
      mbar_wait(bar_acc(bar0, RING), acc_cnt & 1); ++acc_cnt;
      TS();  // 15: F7 acc ready
      tc_fence_after_sync();
      {
        float part = 0.f;
#pragma unroll 1
        for (int cb = c0; cb < c0 + 64; cb += 32) {
          float acc[32];
          tmem_ld32(tacc + cb, acc);
          tmem_wait_ld();
#pragma unroll
          for (int i = 0; i < 32; ++i)
            part = fmaf(elu_log2(fmaf(acc[i], vis1, cst[T_B7 + cb + i])), cst[T_W8 + cb + i], part);
        }
        xch7[tw * 128 + t] = part;
      }
      TS();  // 16: F7 partial done
      pair_sync(pair);
      const float v2 = cst[T_MISC + 1] + xch7[t] + xch7[128 + t];
      const float vis2 = sigmoid_fast(v2) * mask;
      if (ST && valid && tw == 0) a.vis2[m] = vis2;
      const float vsum = group_sum<VP>(vis2);
      const float w2 = vis2 / (vsum + 1e-8f);
      const float W = group_sum<VP>(w2);
      const float nval = group_sum<VP>(mask);

      // ---- second pooling on this twin's 64 channels: reduce-scatter of sum(w x), sum(w x^2) ----
      {
        const bool b0 = gl & 1, b1 = gl & 2, b2 = gl & 4, b3 = gl & 8;
        constexpr int NO = VP == 16 ? 4 : 8;
        const int cbase = c0 + (b0 ? 32 : 0) + (b1 ? 16 : 0) + (b2 ? 8 : 0) + ((VP == 16 && b3) ? 4 : 0);
        float mean[NO], sq[NO];
        float lo[32], hi[32];
        tmem_ld32(tacc + 128 + c0, lo);
        tmem_ld32(tacc + 128 + c0 + 32, hi);
        tmem_wait_ld();
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          float s1[32];
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            const float l = q ? w2 * lo[i] * lo[i] : w2 * lo[i];
            const float h = q ? w2 * hi[i] * hi[i] : w2 * hi[i];
            const float send = b0 ? l : h, keep = b0 ? h : l;
            s1[i] = keep + __shfl_xor_sync(0xffffffffu, send, 1);
          }
          float s2[16], s3[8];
          rs_step<32>(s1, s2, b1, 2);
          rs_step<16>(s2, s3, b2, 4);
          float* dst = q ? sq : mean;
          if (VP == 16) {
            float s4[4];
            rs_step<8>(s3, s4, b3, 8);
#pragma unroll
            for (int i = 0; i < NO; ++i) dst[i] = s4[i < 4 ? i : 0];
          } else {
#pragma unroll
            for (int i = 0; i < NO; ++i) dst[i] = s3[i < 8 ? i : 0];
          }
        }
        if (pt_ok) {
          // pooled statistics as the bf16 tile image of geometry_fc's operand (34 k-groups:
          // mean 0..127 | var 128..255 | weight 256 | zero pad), rows = points
          uint8_t* gi = reinterpret_cast<uint8_t*>(a.G);
          float mu[NO], vr[NO];
#pragma unroll
          for (int i = 0; i < NO; ++i) {
            mu[i] = mean[i];
            vr[i] = sq[i] - mu[i] * mu[i] * (2.f - W);
          }
          uint8_t* pm = gi + tile_image_off(pl, cbase >> 3, 34) + (cbase & 7) * 2;
          uint8_t* pv = gi + tile_image_off(pl, 16 + (cbase >> 3), 34) + (cbase & 7) * 2;
          if (NO == 8) {
            *reinterpret_cast<uint4*>(pm) = make_uint4(pack_bf16x2(mu[0], mu[1]), pack_bf16x2(mu[2], mu[3]),
                                                       pack_bf16x2(mu[4 % NO], mu[5 % NO]), pack_bf16x2(mu[6 % NO], mu[7 % NO]));
            *reinterpret_cast<uint4*>(pv) = make_uint4(pack_bf16x2(vr[0], vr[1]), pack_bf16x2(vr[2], vr[3]),
                                                       pack_bf16x2(vr[4 % NO], vr[5 % NO]), pack_bf16x2(vr[6 % NO], vr[7 % NO]));
          } else {
            *reinterpret_cast<uint2*>(pm) = make_uint2(pack_bf16x2(mu[0], mu[1]), pack_bf16x2(mu[2], mu[3]));
            *reinterpret_cast<uint2*>(pv) = make_uint2(pack_bf16x2(vr[0], vr[1]), pack_bf16x2(vr[2], vr[3]));
          }
          if (gl == 0 && tw == 0) {
            *reinterpret_cast<uint4*>(gi + tile_image_off(pl, 32, 34)) =
                make_uint4(pack_bf16x2(W / (float)a.V, 0.f), 0u, 0u, 0u);
            *reinterpret_cast<uint4*>(gi + tile_image_off(pl, 33, 34)) = make_uint4(0x3F803F80u, 0u, 0u, 0u);  // 1, 1: bias columns of geometry_fc
            a.nvalid[pl] = nval;
          }
        }
      }
      TS();  // 17: pool2 + outputs done
      tc_fence_before_sync();
    }
#undef TS
  }
}

}  // namespace

// ---------------------------------------------------------------------------
// host: weight images in the twin column layouts
// ---------------------------------------------------------------------------
size_t view_twin_bytes(int kind) { (void)kind; return (size_t)(512 * 1024); }

int view_twin_build(dyn_net* n, const float* P, void* dst_dev, size_t dst_bytes, cudaStream_t st) {
  std::vector<uint8_t> img;
  std::vector<FusedChunk> tab;
  constexpr float kLog2e = 1.4426950408889634f, kLn2 = 0.6931471805599453f;
  // fold_bias: the layer's bias rides in the map's kBiasHi / kBiasLo columns
  auto add = [&](const LinearP& l, int N, int Npad, int Kpad, std::vector<int> map, float scale = 1.f,
                 bool fold_bias = false, float bias_scale = -1.f) {
    HostLayer L;
    L.W = P + l.w; L.N = N; L.Kw = l.in; L.Npad = Npad; L.Kpad = Kpad; L.colmap = std::move(map);
    L.scale = scale; L.bias_scale = bias_scale;
    if (fold_bias) L.bias = P + l.b;
    append_layer(L, img, tab, 0, 0, 9, true, kTwinStage);
  };
  // identity columns 0..K-1 followed by one k-step whose first two columns carry the folded bias (hi, lo)
  auto bias_map = [](int K) {
    std::vector<int> m = identity_map(K, K + 16);
    m[K] = kBiasHi; m[K + 1] = kBiasLo;
    return m;
  };
  if (n->kind == DYN_NET_STATIC) {
    const StaticLayout& L = n->sl;
    // layer 1: component-major PE; twin 0 = comps 0..4 (+1 pad), twin 1 = comps 5..8, ray_diff, pad
    std::vector<int> m1(112, -1);
    auto comp_col = [](int ci, int j) {  // j: 0 = x, 1..5 = cos f_k, 6..10 = sin f_k
      if (ci < 3) return j == 0 ? ci : (j <= 5 ? 3 + 3 * (j - 1) + ci : 18 + 3 * (j - 6) + ci);
      const int d = ci - 3;
      return j == 0 ? 33 + d : (j <= 5 ? 39 + 6 * (j - 1) + d : 69 + 6 * (j - 6) + d);
    };
    for (int ci = 0; ci < 5; ++ci)
      for (int j = 0; j < 11; ++j) m1[11 * ci + j] = comp_col(ci, j);
    for (int ci = 5; ci < 9; ++ci)
      for (int j = 0; j < 11; ++j) m1[56 + 11 * (ci - 5) + j] = comp_col(ci, j);
    for (int i = 0; i < 4; ++i) m1[100 + i] = 99 + i;
    m1[104] = kBiasHi; m1[105] = kBiasLo;
    add(L.ray_dir0, 256, 256, 112, m1, kLog2e, true);               // ELU on the exp2 scale
    add(L.ray_dir2, kF, 48, 256, identity_map(256, 256), kLn2);     // consumes log2(e) * ELU
    // layer 3: per twin 5 groups of [mean8 | var8 | feat8]; concat channel c: mean c, var 70+c, feat 140+c
    std::vector<int> m3(240, -1);
    auto chan = [](int tw, int slot) {  // concat channel (0..69) of a twin's slot, -1 = pad
      if (tw == 0) return slot < 19 ? slot : (slot < 37 ? 35 + (slot - 19) : -1);
      return slot < 16 ? 19 + slot : (slot < 33 ? 53 + (slot - 16) : -1);
    };
    for (int tw = 0; tw < 2; ++tw)
      for (int s = 0; s < 40; ++s) {
        const int c = chan(tw, s);
        if (c < 0) continue;
        const int base = 120 * tw + 24 * (s / 8) + (s % 8);
        m3[base] = c; m3[base + 8] = 70 + c; m3[base + 16] = 140 + c;
      }
    m3[103] = kBiasHi; m3[111] = kBiasLo;  // twin 0, slot 39 (unused): mean / var columns of group 4
    add(L.base0, 256, 256, 240, m3, kLog2e, true);
    add(L.base2, 128, 128, 272, bias_map(256), 1.f, true, kLog2e);  // in: log2(e) ELU (x ln2), out: exp2 scale (x log2e)
    add(L.vis0, 128, 128, 128, identity_map(128, 128), kLog2e);     // in: x (true units); w1 and bias in the epilogue
    add(L.vis2, 128, 128, 144, bias_map(128), 1.f, true, kLog2e);   // rows 0..127 of vis_fc.2; in: log2(e) ELU
    add(L.vis2_0, 128, 128, 128, identity_map(128, 128), kLog2e);   // vis1 and bias in the epilogue
  } else {
    const DynamicLayout& L = n->dl;
    // twin 0: channels 0..18 (3 groups, cols 0..71), twin 1: channels 19..34 (2 groups, cols 72..119)
    std::vector<int> m3(128, -1);
    for (int s = 0; s < 24; ++s)
      if (s < 19) { const int b = 24 * (s / 8) + (s % 8); m3[b] = s; m3[b + 8] = 35 + s; m3[b + 16] = 70 + s; }
    for (int s = 0; s < 16; ++s) {
      const int c = 19 + s, b = 72 + 24 * (s / 8) + (s % 8);
      m3[b] = c; m3[b + 8] = 35 + c; m3[b + 16] = 70 + c;
    }
    m3[55] = kBiasHi; m3[63] = kBiasLo;  // twin 0, slot 23 (unused): mean / var columns of group 2
    add(L.base0, 256, 256, 128, m3, kLog2e, true);
    add(L.base2, 128, 128, 272, bias_map(256), 1.f, true, kLog2e);  // in: log2(e) ELU (x ln2), out: exp2 scale (x log2e)
    add(L.vis0, 128, 128, 128, identity_map(128, 128), kLog2e);     // in: x (true units); w1 and bias in the epilogue
    add(L.vis2, 128, 128, 144, bias_map(128), 1.f, true, kLog2e);   // rows 0..127 of vis_fc.2; in: log2(e) ELU
    add(L.vis2_0, 128, 128, 128, identity_map(128, 128), kLog2e);   // vis1 and bias in the epilogue
  }
  const size_t img_bytes = (img.size() + 255) & ~(size_t)255;
  const size_t need = img_bytes + tab.size() * sizeof(FusedChunk);
  if (need > dst_bytes) return fail(DYN_E_INVALID, "twin images need %zu bytes, have %zu", need, dst_bytes);
  DYN_CUDA(cudaMemcpyAsync(dst_dev, img.data(), img.size(), cudaMemcpyHostToDevice, st));
  DYN_CUDA(cudaMemcpyAsync(reinterpret_cast<char*>(dst_dev) + img_bytes, tab.data(),
                           tab.size() * sizeof(FusedChunk), cudaMemcpyHostToDevice, st));
  DYN_CUDA(cudaStreamSynchronize(st));
  n->twin.img = dst_dev;
  n->twin.tab = reinterpret_cast<const FusedChunk*>(reinterpret_cast<char*>(dst_dev) + img_bytes);
  n->twin.nchunks = (int)tab.size();
  if (tab.size() > (size_t)kMaxChunks) return fail(DYN_E_INVALID, "chunk table too long (%zu)", tab.size());
  return DYN_OK;
}

int launch_view_twin(const dyn_net* n, ViewFusedArgs& a, int V, cudaStream_t st) {
  if (n->twin.img == nullptr) return fail(DYN_E_INVALID, "net has no twin-warp view images");
  a.wimg = n->twin.img;
  a.chunks = n->twin.tab;
  a.nchunks = n->twin.nchunks;
  // one-time set-up (SM count, dynamic shared-memory opt-in of every instantiation)
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    DYN_CUDA(cudaGetDevice(&dev));
    DYN_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
#define PREP_VT(VPV, STV) \
    DYN_CUDA(cudaFuncSetAttribute(view_twin_kernel<VPV, STV>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTwinSmem))
    PREP_VT(8, true); PREP_VT(16, true); PREP_VT(8, false); PREP_VT(16, false);
#undef PREP_VT
  }
  const int VP = V <= 8 ? 8 : 16;
  const long long n_iter = (a.P * VP + 127) / 128;
  static_assert(2 * kTwinSmem > 227 * 1024, "one CTA per SM");  // shared memory holds the accumulators
  const long long slots = sms;
  const int grid = (int)(n_iter < slots ? n_iter : slots);
  if (grid == 0) return DYN_OK;
  const bool st_net = n->kind == DYN_NET_STATIC;
  ProfScope prof(st_net ? PROF_VIEW_ST : PROF_VIEW_DY, st);
  if (st_net) {
    if (VP == 8) view_twin_kernel<8, true><<<grid, kTwinThreads, kTwinSmem, st>>>(a);
    else view_twin_kernel<16, true><<<grid, kTwinThreads, kTwinSmem, st>>>(a);
  } else {
    if (VP == 8) view_twin_kernel<8, false><<<grid, kTwinThreads, kTwinSmem, st>>>(a);
    else view_twin_kernel<16, false><<<grid, kTwinThreads, kTwinSmem, st>>>(a);
  }
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

}  // namespace dyn
