// Fused per-(point, view) stage of the two aggregation networks, built for Hopper (reference:
// ibrnet/projection.py:103-176, ibrnet/mlp_network.py:236-284 (dynamic) / :423-497 (static)).
// Same work and outputs as view_twin.cu, per 64-row half-tile:
//
//   projection + masks + view-angle difference, bilinear gather of source RGB + features
//   [static]  positional encodings -> ray_dir_fc (SS wgmma, N = 256) -> ray_dir_fc.2 (RS, N = 48)
//   pooling weights, weighted mean/var over views -> base_fc.0 (SS, N = 256)
//   base_fc.2 -> vis_fc.0 -> vis_fc.2 -> vis_fc2.0 (RS, N = 128), visibility logits, second pooling -> G
//
// Built on the warpgroup engine (wg_engine.cuh): each consumer warpgroup owns 64 rows (view slots) of the CTA's
// 128-row iteration, accumulators stay in registers, and only the two front-end operands (positional encodings,
// pooled features) go through shared memory.  The two issue their layers in turn, so while one warpgroup runs an
// epilogue, the other's wgmmas keep the tensor cores busy.  A point's view slots are 8 or 16 aligned rows of one warp's 16-row slab, so sums over its
// views are shuffles over the row lanes (wg_engine.cuh: views_sum).
// The front end (projection, gather, first pooling of the gathered channels, positional encodings) runs on a
// warpgroup of its own, for consumer 0's rows and then consumer 1's, with two threads per row as in view_twin.cu:
// warps 0-1 ("twin 0") and 2-3 ("twin 1") each take half of the channels.  A full / empty mbarrier pair per
// consumer hands over its operand tiles and per-row pooling weights and masks: the consumer frees them once
// base_fc.0 has retired, so the front end of its next iteration runs behind its remaining layers.
#include "geometry.cuh"
#include "nets.cuh"
#include "wg_engine.cuh"

namespace dyn {

using namespace tc;
using namespace fe;
using namespace wg;

namespace {

// per consumer warpgroup: positional-encoding operand (112 columns) | pooled operand of base_fc.0 (240 columns),
// 64 rows
constexpr int kPeBytes = 14 * 1024, kPoolBytes = 30 * 1024, kWgATile = kPeBytes + kPoolBytes;
// constants (floats): biases in true units; W6V = row 128 of vis_fc.2 (visibility logit), W8 = vis_fc2.2;
// MISC = b(vis_fc.2)[128], b(vis_fc2.2), |s|; W1 / MK = per-row pooling weight and mask of each consumer;
// TGT = the target camera centres of a multi-camera launch (3 floats each)
constexpr int C_B1 = 0, C_B2 = 256, C_B3 = 304, C_B4 = 560, C_B5 = 688, C_B6 = 816, C_W6V = 944, C_B7 = 1072,
              C_W8 = 1200, C_MISC = 1328, C_DFEAT = 1332, C_CAMS = 1372, C_W1 = 1628, C_MK = 1756, C_TGT = 1884;
constexpr int kWgConst = C_TGT + 3 * kMaxTargets;
// mbarriers: the weight ring's full / empty pairs, then per consumer its operand tiles' full and empty
constexpr int kViewBars = 2 * kWgRing + 4;
constexpr int kWgSmem = kWgRing * kWgStage + 2 * kWgATile + kWgConst * 4 + 4 /* align */ + kViewBars * 8;
static_assert(kWgSmem + kWgMaxChunks * 16 <= 227 * 1024, "shared memory of one CTA");
// warpgroups 0, 1: consumers; 2: front end; 3: weight producer.  setmaxnreg splits the 64 K registers:
// 2 x 128 x 208 + 128 x 72 + 128 x 24 = 64 K.  The consumers' peak is a 256-wide epilogue (128 accumulators,
// then 64 A-fragment registers).
constexpr int kViewThreads = 4 * 128;
constexpr int kViewConsumerRegs = 208, kViewFrontRegs = 72, kViewProducerRegs = 24;

// Phase profile of block 0 (dyn_debug_set_view_timestamps).  Thread 0 of each warpgroup charges the cycles since
// its previous mark to one phase, less the weight-ring waits in between, which go to PH_WEIGHTS; the counters sit in
// shared memory while the kernel runs and are copied to dbg[32 wg + phase] at its end.  tools/view_phases.py reads
// them; the indices are its table.
enum Phase {
  PH_FRONT, PH_BAR, PH_WEIGHTS, PH_F1, PH_F1_EPI, PH_F2, PH_F2_EPI, PH_F3, PH_F3_EPI, PH_F4, PH_F4_EPI, PH_F5,
  PH_F5_EPI, PH_F6, PH_F6_EPI, PH_F7, PH_F7_EPI, PH_POOL2, PH_HANDOFF,
  PH_T = 28, PH_W = 29, PH_ITERS = 30, PH_LIFE = 31  // last mark, weight waits at the last mark, iterations, lifetime
};
constexpr int kPhaseSlots = 32;
__shared__ long long s_phase[3][kPhaseSlots];  // consumers 0, 1, front end
struct PhaseClock {
  const ViewFusedArgs& a;  // profiling when a.dbg is set: thread 0 of each warpgroup of block 0
  int wg;
  __device__ __forceinline__ bool on() const { return a.dbg != nullptr && blockIdx.x == 0 && (threadIdx.x & 127) == 0; }
  __device__ __forceinline__ long long* c() const { return s_phase[wg]; }
  __device__ __forceinline__ void start() {
    if (!on()) return;
    for (int i = 0; i < kPhaseSlots; ++i) c()[i] = 0;
    c()[PH_T] = c()[PH_LIFE] = clock64();
  }
  __device__ __forceinline__ void mark(int ph, long long waits) {
    if (!on()) return;
    long long* s = c();
    const long long now = clock64();
    s[ph] += now - s[PH_T] - (waits - s[PH_W]);
    s[PH_WEIGHTS] += waits - s[PH_W];
    s[PH_T] = now;
    s[PH_W] = waits;
  }
  __device__ __forceinline__ void iteration() {
    if (on()) ++c()[PH_ITERS];
  }
  __device__ __forceinline__ void finish() {
    if (!on()) return;
    c()[PH_LIFE] = clock64() - c()[PH_LIFE];
    for (int i = 0; i < kPhaseSlots; ++i) a.dbg[kPhaseSlots * wg + i] = c()[i];
  }
};

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

// layer_ss<256, KS> as two m64n128k16 wgmmas per k-step, columns 0..127 into acc[0..63] and 128..255 into
// acc[64..127] (the fragment layout of one N = 256 wgmma): a single m64n256k16 needs more registers than the
// 128 a 512-thread CTA may launch with.  Rows 128..255 of a weight chunk's k-step start 16 core matrices (2048
// bytes) after rows 0..127.
template <int KS>
__device__ __forceinline__ void layer_ss256(float* acc, uint32_t a_tile, Ring& rg) {
  layer_issue<256, KS>(acc, rg, [&](float* d, int ks, uint64_t bd, uint32_t sc) {
    const uint64_t ad = smem_desc(a_tile + ks * 2048u, 1024u, 128u);
    Wgmma<128, 0, 0>::mma(d, ad, bd, sc);
    Wgmma<128, 0, 0>::mma(d + 64, ad, bd + (2048u >> 4), sc);
  });
}

// layer_rs without its layer_finish
template <int N, int KS>
__device__ __forceinline__ void layer_rs_issue(float* acc, const uint32_t (&af)[KS][4], Ring& rg) {
  layer_issue<N, KS>(acc, rg, [&](float* d, int ks, uint64_t bd, uint32_t sc) { WgmmaRS<N>::mma(d, af[ks], bd, sc); });
}

__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// columns (col, col + 1) of row r of a 64-row operand tile (col even)
__device__ __forceinline__ void store2_64(uint8_t* tile, int r, int col, float x, float y) {
  *reinterpret_cast<uint32_t*>(tile + (col >> 3) * 1024 + (r >> 3) * 128 + (r & 7) * 16 + (col & 7) * 2) =
      pack_bf16x2(x, y);
}

// The front end of the 64 rows from row0 on, row layout (t = thread of the front-end warpgroup: twin tw = t / 64 of
// row t % 64): projection, masks, gather, first pooling into columns 0..119 of pool_tile, [static] positional
// encodings into pe_tile; each row's pooling weight and mask into s_w1 / s_mk; the per-(point, view) outputs.
// MC (static, multi-camera launch): the target camera centre of the row's ray is cst[C_TGT + 3 a.tgt_idx[ray]].
template <int VP, bool ST, bool MC>
__device__ __forceinline__ void front_end(const ViewFusedArgs& a, const float* cst, int t, long long row0,
                                          uint8_t* pe_tile, uint8_t* pool_tile, float* s_w1, float* s_mk) {
  const int tw = t >> 6, r = t & 63, v = r & (VP - 1);
  uint8_t* arow_pe = pe_tile + (r >> 3) * 128 + (r & 7) * 16;
  uint8_t* arow_pool = pool_tile + (r >> 3) * 128 + (r & 7) * 16;
  const float wh = a.w_img, hh = a.h_img;
  const bool want_rgb = (tw == 0) || (ST && a.mask_rgb);

  const long long pl = (row0 + r) / VP;
  const bool pt_ok = pl < a.P;
  const bool valid = pt_ok && v < a.V;
  const long long m = pl * a.V + v;
  float p3[3] = {0.f, 0.f, 0.f};
  if (pt_ok) { p3[0] = a.pts[pl * 3]; p3[1] = a.pts[pl * 3 + 1]; p3[2] = a.pts[pl * 3 + 2]; }
  float q3[3] = {p3[0], p3[1], p3[2]};
  if (!ST && valid) {
    const float* qq = a.pts_seq + ((long long)v * a.seq_stride + pl) * 3;
    q3[0] = qq[0]; q3[1] = qq[1]; q3[2] = qq[2];
  }

  const int vc = valid ? v : 0;
  const float* cam = cst + C_CAMS + 16 * vc;
  float pu, pv;
  bool front;
  project_point(cam, q3[0], q3[1], q3[2], pu, pv, front);
  const bool inb = (pu <= wh - 1.f) && (pu >= 0.f) && (pv <= hh - 1.f) && (pv >= 0.f);
  const float mask_proj = (valid && inb && front) ? 1.f : 0.f;

  // ---- gather: this twin's 16 bf16 feature channels (+ RGB) at the 4 bilinear taps, two taps per round ----
  float chv[24];
#pragma unroll
  for (int i = 0; i < 24; ++i) chv[i] = 0.f;
  float rgb[3] = {0.f, 0.f, 0.f};
  {
    const float gx = 2.f * pu / (wh - 1.f) - 1.f, gy = 2.f * pv / (hh - 1.f) - 1.f;
    const float fx = (gx + 1.f) * 0.5f * (float)(a.w - 1), fy = (gy + 1.f) * 0.5f * (float)(a.h - 1);
    const float x0f = floorf(fx), y0f = floorf(fy);
    const int x0 = (int)x0f, y0 = (int)y0f;
    const float ax = fx - x0f, ay = fy - y0f, bx = (x0f + 1.f) - fx, by = (y0f + 1.f) - fy;
    const uint16_t* base = a.feat_bf + (long long)vc * a.h * a.w * kC + 16 * tw;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
      uint4 tf[4];
      float tw4[2];
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        // out-of-range taps (and padding rows) load a clamped texel with weight 0
        const int xi = x0 + dx, yi = y0 + dy;
        const bool in = valid && xi >= 0 && xi < a.w && yi >= 0 && yi < a.h;
        tw4[dx] = in ? (dx ? ax : bx) * (dy ? ay : by) : 0.f;
        const int xc = min(max(xi, 0), a.w - 1), yc = min(max(yi, 0), a.h - 1);
        const uint4* tp = reinterpret_cast<const uint4*>(base + ((long long)yc * a.w + xc) * kC);
        tf[2 * dx] = __ldg(tp);
        tf[2 * dx + 1] = __ldg(tp + 1);
      }
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
#pragma unroll
        for (int hlf = 0; hlf < 2; ++hlf) {
          const uint4 qv = tf[2 * dx + hlf];
          const uint32_t u[4] = {qv.x, qv.y, qv.z, qv.w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float lo = __uint_as_float(u[j] << 16), hi = __uint_as_float(u[j] & 0xffff0000u);
            if (tw == 0) {
              chv[3 + 8 * hlf + 2 * j] += lo * tw4[dx];  // twin 0 keeps rgb in slots 0..2
              chv[3 + 8 * hlf + 2 * j + 1] += hi * tw4[dx];
            } else {
              chv[8 * hlf + 2 * j] += lo * tw4[dx]; chv[8 * hlf + 2 * j + 1] += hi * tw4[dx];
            }
          }
        }
      }
    }
    if (want_rgb) {
      const float fx = (gx + 1.f) * 0.5f * (float)(a.W - 1), fy = (gy + 1.f) * 0.5f * (float)(a.H - 1);
      const float x0f = floorf(fx), y0f = floorf(fy);
      const int x0 = (int)x0f, y0 = (int)y0f;
      const float ax = fx - x0f, ay = fy - y0f, bx = (x0f + 1.f) - fx, by = (y0f + 1.f) - fy;
      const float* base = a.rgba + (long long)vc * a.H * a.W * 4;
      float4 tr[4];
      float twr[4];
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
#pragma unroll
      for (int tp = 0; tp < 4; ++tp) {
        rgb[0] += tr[tp].x * twr[tp]; rgb[1] += tr[tp].y * twr[tp]; rgb[2] += tr[tp].z * twr[tp];
      }
    }
  }

  float rd[4];
  {
    const float* tgt = a.cams.tgt;
    if (MC) tgt = cst + C_TGT + 3 * (pt_ok ? a.tgt_idx[(int)pl / a.S] : 0);
    float a0 = tgt[0] - p3[0], a1 = tgt[1] - p3[1], a2 = tgt[2] - p3[2];
    normalize3(a0, a1, a2);
    float b0 = cam[12] - q3[0], b1 = cam[13] - q3[1], b2 = cam[14] - q3[2];
    normalize3(b0, b1, b2);
    rd[0] = a0 - b0; rd[1] = a1 - b1; rd[2] = a2 - b2;
    rd[3] = a0 * b0 + a1 * b1 + a2 * b2;
    normalize3(rd[0], rd[1], rd[2]);
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
  if (!ST) {  // dynamic: + time feature on this twin's channels (mlp_network.py:244-247)
    const int c0 = tw == 0 ? 0 : 19, nc = tw == 0 ? 19 : 16;
#pragma unroll
    for (int i = 0; i < 19; ++i)
      if (i < nc) chv[i] = valid ? chv[i] + cst[C_DFEAT + c0 + i] : 0.f;
  }

  // ---- pooling weights (both twins) ----
  float w1;
  if (ST && a.anti_alias) {
    const float e = ex2f(cst[C_MISC + 2] * (rd[3] - 1.f) * 1.4426950408889634f);
    const float emin = group_min<VP>(valid ? e : INFINITY);
    w1 = valid ? (e - emin) * mask : 0.f;
  } else {
    w1 = mask;
  }
  w1 = w1 / (group_sum<VP>(w1) + 1e-8f);
  if (tw == 0) { s_w1[r] = w1; s_mk[r] = mask; }

  // ---- first pooling of the gathered channels (row layout): per twin groups of
  //      [mean8 | var8 | feat8], twin 0 at columns 0..71 (3 groups), twin 1 at 72..119 (2 groups) ----
#pragma unroll
  for (int g = 0; g < 3; ++g) {
    if (tw == 1 && g == 2) break;
    float o[24];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float fv = chv[8 * g + j];
      const float s1 = group_sum<VP>(w1 * fv);
      const float d = fv - s1;
      const float s2 = group_sum<VP>(w1 * d * d);
      o[j] = s1; o[8 + j] = s2; o[16 + j] = fv;
    }
    const int cb = 72 * tw + 24 * g;
    store8_64(arow_pool, cb, o);
    store8_64(arow_pool, cb + 8, o + 8);
    store8_64(arow_pool, cb + 16, o + 16);
  }
  if (!ST && tw == 1) {  // dynamic: K padding 120..127
    const float z[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    store8_64(arow_pool, 120, z);
  }

  if (ST) {
    // ---- ray_dir_fc.0 operand: component-major PE, 56 columns per twin (layout in view_wg_build) ----
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
    // each 8-column group is stored as soon as it is complete (short live ranges)
    float xin[56];
    if (tw == 0) {
      pe_comp(p3[0], xin);         store8_64(arow_pe, 0, xin);
      pe_comp(p3[1], xin + 11);    store8_64(arow_pe, 8, xin + 8);
      pe_comp(p3[2], xin + 22);    store8_64(arow_pe, 16, xin + 16); store8_64(arow_pe, 24, xin + 24);
      pe_comp(pl6[0], xin + 33);   store8_64(arow_pe, 32, xin + 32);
      pe_comp(pl6[1], xin + 44);   xin[55] = 0.f;
      store8_64(arow_pe, 40, xin + 40);  store8_64(arow_pe, 48, xin + 48);
    } else {
      pe_comp(pl6[2], xin);        store8_64(arow_pe, 56, xin);
      pe_comp(pl6[3], xin + 11);   store8_64(arow_pe, 64, xin + 8);
      pe_comp(pl6[4], xin + 22);   store8_64(arow_pe, 72, xin + 16); store8_64(arow_pe, 80, xin + 24);
      pe_comp(pl6[5], xin + 33);   store8_64(arow_pe, 88, xin + 32);
      xin[44] = rd[0]; xin[45] = rd[1]; xin[46] = rd[2]; xin[47] = rd[3];
#pragma unroll
      for (int i = 48; i < 56; ++i) xin[i] = 0.f;
      store8_64(arow_pe, 96, xin + 40);  store8_64(arow_pe, 104, xin + 48);
    }
  }
}

template <int VP, bool ST, bool MC>
__global__ void __launch_bounds__(kViewThreads, 1) view_wg_kernel(const __grid_constant__ ViewFusedArgs a) {
  static_assert(ST || !MC, "multi-camera launches are static-net only");
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* ring = smem;
  uint8_t* atiles = smem + kWgRing * kWgStage;
  float* cst = reinterpret_cast<float*>(atiles + 2 * kWgATile);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + ((kWgRing * kWgStage + 2 * kWgATile + kWgConst * 4 + 7) & ~7));
  __shared__ __align__(16) FusedChunk s_tab[kWgMaxChunks];
  const int tid = threadIdx.x, lane = tid & 31;
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);  // warpgroup index, uniform to the compiler
  const uint32_t bar0 = smem_u32(bars);
  // consumer c's operand tiles: filled by the front end (128 arrivals), free again (4 warps arrive)
  const uint32_t tiles_full = bar0 + 8u * (2 * kWgRing), tiles_empty = tiles_full + 16u;
  stage_chunks(s_tab, a.chunks, a.nchunks);
  if (tid == 0) {
    for (int i = 0; i < kWgRing; ++i) {
      mbar_init(bar0 + 8u * i, 1);
      mbar_init(bar0 + 8u * (kWgRing + i), 8);
    }
    for (int c = 0; c < 2; ++c) {
      mbar_init(tiles_full + 8u * c, 128);
      mbar_init(tiles_empty + 8u * c, 4);
    }
    mbar_fence_init();
  }
  {
    const float* prm = a.params;
    for (int i = tid; i < 256; i += blockDim.x) {
      const int vv = i >> 4, j = i & 15;
      cst[C_CAMS + i] = j < 12 ? a.cams.P[vv][j] : (j < 15 ? a.cams.center[vv][j - 12] : 0.f);
      cst[C_B1 + i] = ST ? prm[a.o_b1 + i] : 0.f;
      cst[C_B3 + i] = prm[a.o_b3 + i];
    }
    for (int i = tid; i < 128; i += blockDim.x) {
      cst[C_B4 + i] = prm[a.o_b4 + i];
      cst[C_B5 + i] = prm[a.o_b5 + i];
      cst[C_B6 + i] = prm[a.o_b6 + i];
      cst[C_W6V + i] = prm[a.o_w6 + 128 * 128 + i];
      cst[C_B7 + i] = prm[a.o_b7 + i];
      cst[C_W8 + i] = prm[a.o_w8 + i];
    }
    if (tid < 48) cst[C_B2 + tid] = (ST && tid < kF) ? prm[a.o_b2 + tid] : 0.f;
    if (tid < 40) cst[C_DFEAT + tid] = (!ST && tid < kF) ? a.dfeat[tid] : 0.f;
    if (tid == 0) {
      cst[C_MISC + 0] = prm[a.o_b6 + 128];
      cst[C_MISC + 1] = prm[a.o_b8];
      cst[C_MISC + 2] = (ST && a.o_s >= 0) ? fabsf(prm[a.o_s]) : 0.f;
    }
    if (MC && tid < 3 * kMaxTargets) cst[C_TGT + tid] = a.cams.tgts[tid / 3][tid % 3];
  }
  __syncthreads();

  const long long n_rows = a.P * VP;
  const int n_iter = (int)((n_rows + 127) / 128);
  const int t = tid & 127;
  if (wg == 3) {
    setmaxnreg_dec<kViewProducerRegs>();
    if (t == 0) producer_loop<kWgRing, kWgStage>(s_tab, a.nchunks, a.wimg, n_iter, ring, bar0);
    return;
  }
  if (wg == 2) {
    setmaxnreg_dec<kViewFrontRegs>();
    PhaseClock pc{a, 2};
    pc.start();
    uint32_t k = 0;  // iterations handed over to each consumer so far
    for (int it = blockIdx.x; it < n_iter; it += gridDim.x, ++k) {
#pragma unroll 1
      for (int c = 0; c < 2; ++c) {
        if (k > 0) mbar_wait(tiles_empty + 8u * c, (k - 1) & 1);
        pc.mark(PH_HANDOFF, 0);
        front_end<VP, ST, MC>(a, cst, t, (long long)it * 128 + 64 * c, atiles + c * kWgATile,
                          atiles + c * kWgATile + kPeBytes, cst + C_W1 + 64 * c, cst + C_MK + 64 * c);
        fence_proxy_async_smem();
        mbar_arrive(tiles_full + 8u * c);
        pc.mark(PH_FRONT, 0);
      }
      pc.iteration();
    }
    pc.finish();
    return;
  }
  setmaxnreg_inc<kViewConsumerRegs>();

  const int ww = t >> 5, q = lane & 3;
  uint8_t* pool_tile = atiles + wg * kWgATile + kPeBytes;
  const uint32_t pe_addr = smem_u32(atiles + wg * kWgATile), pool_addr = smem_u32(pool_tile);
  const float* s_w1 = cst + C_W1 + 64 * wg;
  const float* s_mk = cst + C_MK + 64 * wg;
  // fragment layout: rows fr[h] of the half-tile
  const int fr[2] = {16 * ww + (lane >> 2), 16 * ww + (lane >> 2) + 8};

  PhaseClock pc{a, wg};
  Ring rg{ring, bar0, 0u, pc.on(), 0};
  pc.start();
#define TS(ph) pc.mark(ph, rg.wait_cycles)
  // The consumers issue their layers in turn (named barrier 3 + w: warpgroup w's turn, both warpgroups count), so
  // one warpgroup's epilogue runs while the tensor cores work on the other's layer.  A warpgroup keeps the turn
  // until its layer is issued, all chunks but the last retired.  Consumer 0 starts; consumer 1 does not pass the
  // turn after its very last layer.
  auto in_turn = [&](auto issue, bool pass) {
    named_bar_sync(3 + wg, 256);
    TS(PH_BAR);
    issue();
    if (pass) named_bar_arrive(4 - wg, 256);
  };
  if (wg == 1) named_bar_arrive(3, 256);

  uint32_t k = 0;  // iterations of this warpgroup so far
  for (int it = blockIdx.x; it < n_iter; it += gridDim.x, ++k) {
    const long long row0 = (long long)it * 128 + 64 * wg;  // first row of this warpgroup
    mbar_wait(tiles_full + 8u * wg, k & 1);
    TS(PH_HANDOFF);
    // the rows' pooling weights and masks stay in registers: the front end rewrites them once base_fc.0 has retired
    const float w1r[2] = {s_w1[fr[0]], s_w1[fr[1]]}, mk[2] = {s_mk[fr[0]], s_mk[fr[1]]};

    float acc[128];  // accumulators of the 256-wide layers (the first 64 / 24 for the narrower ones)
    if (ST) {
      in_turn([&] { layer_ss256<7>(acc, pe_addr, rg); }, true);
      layer_finish<256>(acc, rg);
      TS(PH_F1);
      // ---- F1 epilogue -> ray_dir_fc.2 (register A) ----
      {
        uint32_t af[16][4];
        bias_elu<256>(acc, cst + C_B1, q);
        to_afrag<16>(acc, af);
        TS(PH_F1_EPI);
        in_turn([&] { layer_rs_issue<48, 16>(acc, af, rg); }, true);
        layer_finish<48>(acc, rg);
      }
      TS(PH_F2);
      // ---- src_feat * ref_feat (35 channels, fragment columns j < 5) and their pooling over views:
      //      mean at column 120 + n, var at 160 + n, feat at 200 + n ----
      float f[2][10];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long prow = (row0 + fr[h]) / VP;
        const bool ok = prow < a.P && ((fr[h] & (VP - 1)) < a.V);
        const float* rf = a.ref_feat + (ok ? prow / a.S : 0) * kF;
#pragma unroll
        for (int j = 0; j < 5; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int n = 8 * j + 2 * q + e;
            f[h][2 * j + e] = (ok && n < kF) ? (acc[4 * j + 2 * h + e] + cst[C_B2 + n]) * __ldg(rf + n) : 0.f;
          }
      }
#pragma unroll
      for (int j = 0; j < 5; ++j) {
        float mu[2][2], va[2][2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int i = 2 * j + e;
          float tv[2] = {w1r[0] * f[0][i], w1r[1] * f[1][i]}, s1[2], s2[2];
          views_sum<VP>(tv, s1);
          const float d0 = f[0][i] - s1[0], d1 = f[1][i] - s1[1];
          tv[0] = w1r[0] * d0 * d0;
          tv[1] = w1r[1] * d1 * d1;
          views_sum<VP>(tv, s2);
          mu[0][e] = s1[0]; mu[1][e] = s1[1]; va[0][e] = s2[0]; va[1][e] = s2[1];
        }
        const int n = 8 * j + 2 * q;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          store2_64(pool_tile, fr[h], 120 + n, mu[h][0], mu[h][1]);
          store2_64(pool_tile, fr[h], 160 + n, va[h][0], va[h][1]);
          store2_64(pool_tile, fr[h], 200 + n, f[h][2 * j], f[h][2 * j + 1]);
        }
      }
      TS(PH_F2_EPI);
      // every warp's columns 120..239 are in place before base_fc.0 reads them
      fence_proxy_async_smem();
      named_bar_sync(1 + wg, 128);
      TS(PH_BAR);
    }
    in_turn([&] { layer_ss256<ST ? 15 : 8>(acc, pool_addr, rg); }, true);
    layer_finish<256>(acc, rg);
    // both operand tiles and the rows' pooling weights / masks are free for the next iteration's front end
    __syncwarp();
    if (lane == 0) mbar_arrive(tiles_empty + 8u * wg);
    TS(PH_F3);
    // ---- base_fc.0 epilogue -> base_fc.2 (register A) ----
    {
      uint32_t af[16][4];
      bias_elu<256>(acc, cst + C_B3, q);
      to_afrag<16>(acc, af);
      TS(PH_F3_EPI);
      in_turn([&] { layer_rs_issue<128, 16>(acc, af, rg); }, true);
      layer_finish<128>(acc, rg);
    }
    TS(PH_F4);
    // ---- x = ELU(base_fc.2) (fp32 residual); vis_fc.0 on bf16(x): its row scale w1 applies to the accumulator ----
    float x[64];
    bias_elu<128>(acc, cst + C_B4, q);
#pragma unroll
    for (int i = 0; i < 64; ++i) x[i] = acc[i];
    {
      uint32_t af[8][4];
      to_afrag<8>(x, af);
      TS(PH_F4_EPI);
      in_turn([&] { layer_rs_issue<128, 8>(acc, af, rg); }, true);
      layer_finish<128>(acc, rg);
    }
    TS(PH_F5);
    // ---- h = ELU(w1 (W x) + b) and the row's visibility logit (quad sum) -> vis_fc.2 ----
    float part[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float2 b = *reinterpret_cast<const float2*>(cst + C_B5 + 8 * j + 2 * q);
      const float2 wv = *reinterpret_cast<const float2*>(cst + C_W6V + 8 * j + 2 * q);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float& h0 = acc[4 * j + 2 * h];
        float& h1 = acc[4 * j + 2 * h + 1];
        h0 = elu_fast(fmaf(h0, w1r[h], b.x));
        h1 = elu_fast(fmaf(h1, w1r[h], b.y));
        part[h] = fmaf(h1, wv.y, fmaf(h0, wv.x, part[h]));
      }
    }
    part[0] = quad_sum(part[0]);
    part[1] = quad_sum(part[1]);
    {
      uint32_t af[8][4];
      to_afrag<8>(acc, af);
      TS(PH_F5_EPI);
      in_turn([&] { layer_rs_issue<128, 8>(acc, af, rg); }, true);
      layer_finish<128>(acc, rg);
    }
    TS(PH_F6);
    // ---- x += ELU(vis_fc.2); bf16(x) is vis_fc2.0's operand (vis1 applies to its accumulator) and, for the
    //      static net, the blending head's input (X tile image, rows = view slots) ----
    float vis1[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) vis1[h] = sigmoid_fast(elu_fast(cst[C_MISC + 0] + part[h])) * mk[h];
    bias_elu<128>(acc, cst + C_B6, q);
#pragma unroll
    for (int i = 0; i < 64; ++i) x[i] += acc[i];
    {
      uint32_t af[8][4];
      to_afrag<8>(x, af);
      if (ST) {
        uint8_t* xo = reinterpret_cast<uint8_t*>(a.X);
#pragma unroll
        for (int s = 0; s < 8; ++s)
#pragma unroll
          for (int k = 0; k < 4; ++k)  // af[s][k]: row fr[k & 1], 8-column group 2 s + (k >> 1)
            *reinterpret_cast<uint32_t*>(xo + tile_image_off(row0 + fr[k & 1], 2 * s + (k >> 1), 16) + 4 * q) = af[s][k];
      }
      TS(PH_F6_EPI);
      in_turn([&] { layer_rs_issue<128, 8>(acc, af, rg); }, wg == 0 || it + (int)gridDim.x < n_iter);
      layer_finish<128>(acc, rg);
    }
    TS(PH_F7);
    // ---- vis2 = sigmoid(vis_fc2.2 . ELU(vis1 (W x) + b)) * mask ----
    float p7[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float2 b = *reinterpret_cast<const float2*>(cst + C_B7 + 8 * j + 2 * q);
      const float2 wv = *reinterpret_cast<const float2*>(cst + C_W8 + 8 * j + 2 * q);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        p7[h] = fmaf(elu_fast(fmaf(acc[4 * j + 2 * h], vis1[h], b.x)), wv.x, p7[h]);
        p7[h] = fmaf(elu_fast(fmaf(acc[4 * j + 2 * h + 1], vis1[h], b.y)), wv.y, p7[h]);
      }
    }
    float vis2[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      vis2[h] = sigmoid_fast(cst[C_MISC + 1] + quad_sum(p7[h])) * mk[h];
      const long long prow = (row0 + fr[h]) / VP;
      const int vh = fr[h] & (VP - 1);
      if (ST && q == 0 && prow < a.P && vh < a.V) a.vis2[prow * a.V + vh] = vis2[h];
    }
    TS(PH_F7_EPI);

    // ---- second pooling: mean / second moment of x over the point's views, reduce-scattered over the row lanes:
    //      afterwards lane l holds columns 8 j0 + 2 q + {0, 1} and 8 (j0 + 1) + 2 q + {0, 1} ----
    float vsum[2], w2[2], Wsum[2], nval[2];
    views_sum<VP>(vis2, vsum);
#pragma unroll
    for (int h = 0; h < 2; ++h) w2[h] = vis2[h] / (vsum[h] + 1e-8f);
    views_sum<VP>(w2, Wsum);
    views_sum<VP>(mk, nval);
    const bool b4 = lane & 16, b3 = lane & 8, b2 = lane & 4;
    const int j0 = (b4 ? 8 : 0) + (b3 ? 4 : 0) + (b2 ? 2 : 0);
    uint8_t* gi = reinterpret_cast<uint8_t*>(a.G);
#pragma unroll
    for (int pi = 0; pi < (VP == 8 ? 2 : 1); ++pi) {
      float st4[2][4];
#pragma unroll
      for (int qq = 0; qq < 2; ++qq) {
        float s32[32], s16[16], s8[8];
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float x0 = x[4 * j + e], x1 = x[4 * j + 2 + e];
            if (VP == 16)
              s32[2 * j + e] = qq ? w2[0] * x0 * x0 + w2[1] * x1 * x1 : w2[0] * x0 + w2[1] * x1;
            else
              s32[2 * j + e] = pi ? (qq ? w2[1] * x1 * x1 : w2[1] * x1) : (qq ? w2[0] * x0 * x0 : w2[0] * x0);
          }
        rs_step<32>(s32, s16, b4, 16);
        rs_step<16>(s16, s8, b3, 8);
        rs_step<8>(s8, st4[qq], b2, 4);
      }
      const long long prow = (row0 + 16 * ww + 8 * pi) / VP;
      if (prow < a.P) {
        const float W = Wsum[pi];
        float mu4[4], vr4[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          mu4[i] = st4[0][i];
          vr4[i] = st4[1][i] - mu4[i] * mu4[i] * (2.f - W);
        }
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const int c = 8 * (j0 + k) + 2 * q;
          *reinterpret_cast<uint32_t*>(gi + tile_image_off(prow, c >> 3, 34) + (c & 7) * 2) =
              pack_bf16x2(mu4[2 * k], mu4[2 * k + 1]);
          *reinterpret_cast<uint32_t*>(gi + tile_image_off(prow, 16 + (c >> 3), 34) + (c & 7) * 2) =
              pack_bf16x2(vr4[2 * k], vr4[2 * k + 1]);
        }
        if (lane == 0) {
          *reinterpret_cast<uint4*>(gi + tile_image_off(prow, 32, 34)) = make_uint4(pack_bf16x2(W / (float)a.V, 0.f), 0u, 0u, 0u);
          *reinterpret_cast<uint4*>(gi + tile_image_off(prow, 33, 34)) = make_uint4(0x3F803F80u, 0u, 0u, 0u);  // 1, 1: bias columns of geometry_fc
          a.nvalid[prow] = nval[pi];
        }
      }
    }
    TS(PH_POOL2);
    pc.iteration();
  }
#undef TS
  pc.finish();
}

}  // namespace

// ---------------------------------------------------------------------------
// host: weight images, full layer width per chunk, in the order the warpgroups consume them
// ---------------------------------------------------------------------------
size_t view_wg_bytes(int kind) { (void)kind; return (size_t)(512 * 1024); }

int view_wg_build(dyn_net* n, const float* P, void* dst_dev, size_t dst_bytes, cudaStream_t st) {
  std::vector<uint8_t> img;
  std::vector<FusedChunk> tab;
  auto add = [&](const LinearP& l, int N, int Npad, int Kpad, std::vector<int> map) {
    HostLayer L;
    L.W = P + l.w; L.N = N; L.Kw = l.in; L.Npad = Npad; L.Kpad = Kpad; L.colmap = std::move(map);
    append_wg_layer(L, img, tab);
  };
  // base_fc.0 operand columns 0..119: the gathered channels (rgb + 32 features, + the time feature for the
  // dynamic net) as [mean8 | var8 | feat8] groups, twin 0 channels 0..18 at 0..71, twin 1 channels 19..34 at
  // 72..119; the concatenated input has C channels: mean c, var C + c, feat 2 C + c
  auto gathered_map = [](std::vector<int>& m, int C) {
    for (int s = 0; s < 19; ++s) {
      const int b = 24 * (s / 8) + (s % 8);
      m[b] = s; m[b + 8] = C + s; m[b + 16] = 2 * C + s;
    }
    for (int s = 0; s < 16; ++s) {
      const int c = 19 + s, b = 72 + 24 * (s / 8) + (s % 8);
      m[b] = c; m[b + 8] = C + c; m[b + 16] = 2 * C + c;
    }
  };
  if (n->kind == DYN_NET_STATIC) {
    const StaticLayout& L = n->sl;
    // ray_dir_fc.0: component-major PE; twin 0 = comps 0..4 (+1 pad), twin 1 = comps 5..8, ray_diff, pad
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
    add(L.ray_dir0, 256, 256, 112, m1);
    add(L.ray_dir2, kF, 48, 256, identity_map(256, 256));
    // columns 120..239: the 35 channels src_feat * ref_feat (concat channels 35..69) as mean | var | feat blocks
    std::vector<int> m3(240, -1);
    gathered_map(m3, 70);
    for (int c = 0; c < kF; ++c) {
      m3[120 + c] = 35 + c; m3[160 + c] = 70 + 35 + c; m3[200 + c] = 140 + 35 + c;
    }
    add(L.base0, 256, 256, 240, m3);
  } else {
    const DynamicLayout& L = n->dl;
    std::vector<int> m3(128, -1);
    gathered_map(m3, kF);
    add(L.base0, 256, 256, 128, m3);
  }
  const LinearP& base2 = n->kind == DYN_NET_STATIC ? n->sl.base2 : n->dl.base2;
  const LinearP& vis0 = n->kind == DYN_NET_STATIC ? n->sl.vis0 : n->dl.vis0;
  const LinearP& vis2 = n->kind == DYN_NET_STATIC ? n->sl.vis2 : n->dl.vis2;
  const LinearP& vis2_0 = n->kind == DYN_NET_STATIC ? n->sl.vis2_0 : n->dl.vis2_0;
  add(base2, 128, 128, 256, identity_map(256, 256));
  add(vis0, 128, 128, 128, identity_map(128, 128));
  add(vis2, 128, 128, 128, identity_map(128, 128));  // rows 0..127 of vis_fc.2; row 128 (the logit) in the epilogue
  add(vis2_0, 128, 128, 128, identity_map(128, 128));
  return upload_wg_image(img, tab, dst_dev, dst_bytes, "per-view", &n->wg, st);
}

int launch_view_wg(const dyn_net* n, ViewFusedArgs& a, int V, cudaStream_t st) {
  if (n->wg.img == nullptr) return fail(DYN_E_INVALID, "net has no per-view weight images");
  a.wimg = n->wg.img;
  a.chunks = n->wg.tab;
  a.nchunks = n->wg.nchunks;
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    DYN_CUDA(cudaGetDevice(&dev));
    DYN_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
#define PREP_WG(VPV, STV, MCV) \
    DYN_CUDA(cudaFuncSetAttribute(view_wg_kernel<VPV, STV, MCV>, cudaFuncAttributeMaxDynamicSharedMemorySize, kWgSmem))
    PREP_WG(8, true, false); PREP_WG(16, true, false); PREP_WG(8, false, false); PREP_WG(16, false, false);
    PREP_WG(8, true, true); PREP_WG(16, true, true);
#undef PREP_WG
  }
  const bool st_net = n->kind == DYN_NET_STATIC;
  const bool mc = a.tgt_idx != nullptr;
  if (mc && !st_net) return fail(DYN_E_INVALID, "multi-camera per-view launches are for the static net only");
  const int VP = V <= 8 ? 8 : 16;
  const long long n_iter = (a.P * VP + 127) / 128;
  const int grid = (int)(n_iter < sms ? n_iter : sms);
  if (grid == 0) return DYN_OK;
  ProfScope prof(st_net ? PROF_VIEW_ST : PROF_VIEW_DY, st);
  if (st_net && mc) {
    if (VP == 8) view_wg_kernel<8, true, true><<<grid, kViewThreads, kWgSmem, st>>>(a);
    else view_wg_kernel<16, true, true><<<grid, kViewThreads, kWgSmem, st>>>(a);
  } else if (st_net) {
    if (VP == 8) view_wg_kernel<8, true, false><<<grid, kViewThreads, kWgSmem, st>>>(a);
    else view_wg_kernel<16, true, false><<<grid, kViewThreads, kWgSmem, st>>>(a);
  } else {
    if (VP == 8) view_wg_kernel<8, false, false><<<grid, kViewThreads, kWgSmem, st>>>(a);
    else view_wg_kernel<16, false, false><<<grid, kViewThreads, kWgSmem, st>>>(a);
  }
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

}  // namespace dyn
