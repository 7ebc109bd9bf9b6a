// Row-local fused tensor-core chains of the aggregation nets, built for Hopper on the warpgroup engine
// (wg_engine.cuh):
//
//   point_fused_wg_kernel : point1 -> ray-transformer attention -> point2 in one kernel, S dividing 128
//                           (mlp_network.py:13-31, :84-98)
//   point1_wg_kernel  : geometry_fc -> (+ sinusoid) -> Q | K | V projections
//                       (mlp_network.py:283-286 / :496, :84-86)
//   point2_wg_kernel  : attention fc + residual + LayerNorm -> heads
//                       (mlp_network.py:99-102, :291-315 / :503-506, first rgb_fc layer)
//   (point1 and point2 run as separate launches around the SIMT attention for the other S)
//   rgbhead_wg_kernel : static per-view colour-blending head + masked softmax over views
//                       (mlp_network.py:508-526)
//
// One persistent CTA per SM.  Per 128-row iteration a thread of the producer warpgroup lands the input tile (the
// G, O or X tile image) with one bulk copy; both consumer warpgroups read their 64 rows of it as the A operand
// of the first layer, and the tile is refilled for the next iteration as soon as both have retired that layer
// (the blending head instead keeps its weights resident and streams its X tiles through a ring).
// Every later layer takes A from registers (the dynamic point2 also from two small per-warpgroup tiles of
// positional encodings).  Each layer is one wgmma per k-step at its full width (N = 256, 128 or 64).
//
// Hidden activations that only feed another MMA live on the exp2 scale (log2(e) * ELU: fused_engine.cuh:
// elu_log2).  Biases are folded into the weight images as a bf16 hi / lo pair read through two operand columns
// that hold 1; where the operand is a register fragment, that k-step is a constant fragment (bias_afrag).
#include "nets.cuh"
#include "wg_engine.cuh"

namespace dyn {

using namespace tc;
using namespace fe;
using namespace wg;

namespace {

constexpr float kLog2e = 1.4426950408889634f, kLn2 = 0.6931471805599453f;

// barriers: [0, 2 RING) weight ring, then the input tile's full / empty pair
template <int RING>
struct ChainBars {
  static constexpr int kTileFull = 2 * RING, kTileEmpty = 2 * RING + 1, kCount = 2 * RING + 2;
};

// shared memory: weight ring | input tile (128 rows) | per-warpgroup operand tiles | constants | barriers
template <int kTile, int kExtra, int kConst, int RING = kWgRing>
struct ChainSmem {
  static constexpr int kTileOff = RING * kWgStage;
  static constexpr int kExtraOff = kTileOff + kTile;
  static constexpr int kConstOff = kExtraOff + kExtra;
  static constexpr int kBarOff = (kConstOff + kConst * 4 + 7) & ~7;
  static constexpr int kBytes = kBarOff + ChainBars<RING>::kCount * 8;
  static_assert(kBytes + kWgMaxChunks * 16 <= 227 * 1024, "shared memory of one CTA");
};

template <int RING = kWgRing>
__device__ __forceinline__ uint32_t chain_init(uint8_t* smem, int bar_off, FusedChunk* s_tab,
                                               const FusedChunk* chunks, int nchunks) {
  const uint32_t bar0 = smem_u32(smem + bar_off);
  stage_chunks(s_tab, chunks, nchunks);
  if (threadIdx.x == 0) {
    for (int i = 0; i < RING; ++i) {
      mbar_init(bar0 + 8u * i, 1);
      mbar_init(bar0 + 8u * (RING + i), 8);
    }
    mbar_init(bar0 + 8u * ChainBars<RING>::kTileFull, 1);
    mbar_init(bar0 + 8u * ChainBars<RING>::kTileEmpty, 8);  // 4 warps x 2 warpgroups
    mbar_fence_init();
  }
  return bar0;
}

// The producer warpgroup: one thread streams the weight chunks, another the input tiles (tile_bytes per 128 rows
// of `src`, a tile image), each tile once both consumer warpgroups have released the previous one.
template <int RING = kWgRing>
__device__ __forceinline__ void chain_producers(const FusedChunk* s_tab, int nchunks, const void* wimg,
                                                const void* src, uint32_t tile_bytes, int n_iter, uint8_t* smem,
                                                uint32_t bar0) {
  setmaxnreg_dec<kProducerRegs>();
  const int t = threadIdx.x & 127;
  if (t == 0) {
    producer_loop<RING, kWgStage>(s_tab, nchunks, wimg, n_iter, smem, bar0);
  } else if (t == 32) {
    const uint8_t* s = reinterpret_cast<const uint8_t*>(src);
    const uint32_t dst = smem_u32(smem + RING * kWgStage);
    uint32_t k = 0;
    for (int it = blockIdx.x; it < n_iter; it += gridDim.x, ++k) {
      if (k > 0) mbar_wait(bar0 + 8u * ChainBars<RING>::kTileEmpty, (k - 1) & 1);
      mbar_arrive_expect_tx(bar0 + 8u * ChainBars<RING>::kTileFull, tile_bytes);
      bulk_g2s(dst, s + (size_t)it * tile_bytes, tile_bytes, bar0 + 8u * ChainBars<RING>::kTileFull);
    }
  }
}
template <int RING = kWgRing>
__device__ __forceinline__ void tile_wait(uint32_t bar0, uint32_t k) {
  mbar_wait(bar0 + 8u * ChainBars<RING>::kTileFull, k & 1);
}
// this warp's wgmmas that read the input tile have retired
template <int RING = kWgRing>
__device__ __forceinline__ void tile_release(uint32_t bar0) {
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(bar0 + 8u * ChainBars<RING>::kTileEmpty);
}

// A fragment of a k-step whose operand columns c0, c0 + 1 (c0 = 0 or 8) hold 1 and the others 0: the bias columns
__device__ __forceinline__ void bias_afrag(uint32_t* a, int c0, int q) {
  const uint32_t one = q == 0 ? 0x3F803F80u : 0u;
  a[0] = a[1] = c0 == 0 ? one : 0u;
  a[2] = a[3] = c0 == 0 ? 0u : one;
}
template <int NA>
__device__ __forceinline__ void elu_log2_all(float* acc) {
#pragma unroll
  for (int i = 0; i < NA; ++i) acc[i] = elu_log2(acc[i]);
}

// the float pair (row, c .. c + 1) of an fp32 tile-layout array (fused_engine.cuh: tile_f32_off), c even
__device__ __forceinline__ float2* f32_pair(const void* base, long long row, int c) {
  return reinterpret_cast<float2*>(const_cast<uint8_t*>(reinterpret_cast<const uint8_t*>(base)) +
                                   tile_f32_off(row, c >> 2) + (c & 3) * 4);
}

// 128 fragment columns -> bf16 tile image (16 k-groups), rows row0 + fr[h]; rows at or past P get zeros
__device__ __forceinline__ void store_image128(const float* acc, void* img, long long row0, const int* fr, int q,
                                               long long P) {
  uint8_t* o = reinterpret_cast<uint8_t*>(img);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const long long row = row0 + fr[h];
    const bool ok = row < P;
#pragma unroll
    for (int j = 0; j < 16; ++j)
      *reinterpret_cast<uint32_t*>(o + tile_image_off(row, j, 16) + 4 * q) =
          ok ? pack_bf16x2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]) : 0u;
  }
}

__device__ __forceinline__ float rows8_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 4));
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 8));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 16));
}

// ---------------------------------------------------------------------------
// per-point stage 1: G -> geometry_fc -> (+ posenc) -> g2, Q, K, V      (rows = points)
// input tile = the G tile image (34 k-groups: mean 128 | var 128 | weight, 0 x 7 | 0 x 8 with 1, 1 at
// columns 264, 265: the per-view kernels write those ones, geometry_fc.0's bias rides on them)
// ---------------------------------------------------------------------------
constexpr int kP1Tile = 34 * 2048;
using P1Smem = ChainSmem<kP1Tile, 0, 0>;

__global__ void __launch_bounds__(kWgThreads, 1) point1_wg_kernel(const __grid_constant__ Point1Args a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ __align__(16) FusedChunk s_tab[kWgMaxChunks];
  const uint32_t bar0 = chain_init(smem, P1Smem::kBarOff, s_tab, a.chunks, a.nchunks);
  __syncthreads();
  const int n_iter = (int)((a.P + 127) / 128);
  const int tid = threadIdx.x, lane = tid & 31;
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);  // warpgroup index, uniform to the compiler
  if (wg == 2) {
    chain_producers(s_tab, a.nchunks, a.wimg, a.G, (uint32_t)kP1Tile, n_iter, smem, bar0);
    return;
  }
  setmaxnreg_inc<kConsumerRegs>();
  const int q = lane & 3, ww = (tid & 127) >> 5;
  const int fr[2] = {16 * ww + (lane >> 2), 16 * ww + (lane >> 2) + 8};
  Ring rg{smem, bar0, 0u, false, 0};
  const uint32_t tile = smem_u32(smem + P1Smem::kTileOff) + 1024u * wg;  // this warpgroup's 64 rows
  uint32_t k = 0;
  for (int it = blockIdx.x; it < n_iter; it += gridDim.x, ++k) {
    const long long row0 = (long long)it * 128 + 64 * wg;
    float acc[128];
    tile_wait(bar0, k);
    layer_ss<256, 17, 128>(acc, tile, rg);  // geometry_fc.0 (bias folded, exp2 scale)
    layer_finish<256>(acc, rg);
    tile_release(bar0);
    {
      uint32_t af[17][4];
      elu_log2_all<128>(acc);
#pragma unroll
      for (int s = 0; s < 16; ++s) acc_to_afrag(acc, s, af[s]);
      bias_afrag(af[16], 8, q);  // operand columns 264, 265
      layer_rs<128, 17>(acc, af, rg);  // geometry_fc.2 (bias folded, exp2 scale)
    }
    // g2 = ELU(geometry_fc.2) (+ sinusoid): the fp32 residual stream, and as bf16 the operand of Q | K | V
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long row = row0 + fr[h];
      const bool ok = row < a.P;
      const float* pe = a.posenc ? a.posenc + (ok ? row % a.S : 0) * 128 : nullptr;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int c = 8 * j + 2 * q;
        float v0 = elu_from_log2(acc[4 * j + 2 * h]), v1 = elu_from_log2(acc[4 * j + 2 * h + 1]);
        if (pe) {
          const float2 p = __ldg(reinterpret_cast<const float2*>(pe + c));
          v0 += p.x;
          v1 += p.y;
        }
        acc[4 * j + 2 * h] = v0;
        acc[4 * j + 2 * h + 1] = v1;
        if (ok) *f32_pair(a.g2, row, c) = make_float2(v0, v1);
      }
    }
    uint32_t ag[8][4];
    to_afrag<8>(acc, ag);
    layer_rs<128, 8>(acc, ag, rg);  // Wq (no bias)
    store_image128(acc, a.Q, row0, fr, q, a.P);
    layer_rs<128, 8>(acc, ag, rg);  // Wk
    store_image128(acc, a.K, row0, fr, q, a.P);
    layer_rs<128, 8>(acc, ag, rg);  // Wv
    store_image128(acc, a.V, row0, fr, q, a.P);
  }
}

// ---------------------------------------------------------------------------
// per-point stage 2: fc(O) + g2 -> LayerNorm -> heads                    (rows = points)
// input tile = the attention output O (bf16 tile image, 16 k-groups)
// dynamic net: per warpgroup, [PE(pts) 33 | 1, 1 | 0] (operand columns 128..175 of ref_pts_fc.0) and
// [PE(dir) 27 | 1, 1 | 0] (columns 128..159 of out_geometry_fc.0, rgb_fc.0 and rgb_fc.2)
// ---------------------------------------------------------------------------
constexpr int kP2Tile = 16 * 2048;
constexpr int kPePtsBytes = 6 * 1024, kPeDirBytes = 4 * 1024;
// constants (floats): LayerNorm weight and bias; ln 2 x out_geometry_fc.2 and rgb_fc.4 weights; their biases
constexpr int C_LNW = 0, C_LNB = 128, C_WOG2 = 256, C_WRGB4 = 384, C_BOG2 = 576, C_BRGB4 = 577;
constexpr int kP2Const = 580;
using P2Smem = ChainSmem<kP2Tile, 2 * (kPePtsBytes + kPeDirBytes), kP2Const>;

// point2's constants in shared memory (kP2Const floats)
__device__ __forceinline__ void point2_constants(const Point2Args& a, float* cst, bool dynamic) {
  const int tid = threadIdx.x;
  const float* p = a.params;
  for (int i = tid; i < 128; i += blockDim.x) {
    cst[C_LNW + i] = p[a.o_lnw + i];
    cst[C_LNB + i] = p[a.o_lnb + i];
    cst[C_WOG2 + i] = p[a.o_woutgeo2 + i] * kLn2;
  }
  if (dynamic) {
    for (int i = tid; i < 192; i += blockDim.x) cst[C_WRGB4 + i] = p[a.o_wrgb4 + i] * kLn2;
    if (tid < 3) cst[C_BRGB4 + tid] = p[a.o_brgb4 + tid];
  }
  if (tid == 0) cst[C_BOG2] = p[a.o_boutgeo2];
}

// dynamic net: the positional-encoding tiles of rows row0 .. row0 + 63 (thread t of the warpgroup writes row
// t % 64, PE(pts) for t < 64, PE(dir) otherwise).  The caller orders the writes after the wgmmas that read the
// previous contents and before those that read these.
__device__ __forceinline__ void write_pe_tiles(const Point2Args& a, long long row0, uint8_t* pe_pts, uint8_t* pe_dir) {
  const int tw = (threadIdx.x & 127) >> 6, r = threadIdx.x & 63;
  const long long row = row0 + r;
  const bool valid = row < a.P;
  if (tw == 0) {
    float p3[3] = {0.f, 0.f, 0.f};
    if (valid) { p3[0] = a.pts[row * 3]; p3[1] = a.pts[row * 3 + 1]; p3[2] = a.pts[row * 3 + 2]; }
    float pe[48];
    pe_pow2<3, 5>(p3, pe);
    pe[33] = 1.f; pe[34] = 1.f;  // bias columns of ref_pts_fc.0
#pragma unroll
    for (int i = 35; i < 48; ++i) pe[i] = 0.f;
    uint8_t* arow = pe_pts + (r >> 3) * 128 + (r & 7) * 16;
#pragma unroll
    for (int g = 0; g < 6; ++g) store8_64(arow, 8 * g, pe + 8 * g);
  } else {
    const long long ray = valid ? row / a.S : 0;
    float d3[3] = {a.ray_dir[ray * 3], a.ray_dir[ray * 3 + 1], a.ray_dir[ray * 3 + 2]};
    float pe2[32];
    pe_pow2<3, 4>(d3, pe2);
    pe2[27] = 1.f; pe2[28] = 1.f;  // bias columns of the three layers that read this tile
#pragma unroll
    for (int i = 29; i < 32; ++i) pe2[i] = 0.f;
    uint8_t* arow = pe_dir + (r >> 3) * 128 + (r & 7) * 16;
#pragma unroll
    for (int g = 0; g < 4; ++g) store8_64(arow, 8 * g, pe2 + 8 * g);
  }
  fence_proxy_async_smem();
}

// point2 after its first layer: acc[0 .. 63] = fc(O) + g2 of this warpgroup's 64 rows -> LayerNorm -> heads
// (dynamic: raw; static: GW and sigma).  rows / ok / nv: this thread's two rows, whether they exist, their nvalid.
template <bool DYNAMIC, class RG>
__device__ __forceinline__ void point2_heads(float* acc, const Point2Args& a, const float* cst, uint32_t pe_pts,
                                             uint32_t pe_dir, const long long* rows, const bool* ok, const float* nv,
                                             int wg, RG& rg) {
  const int q = threadIdx.x & 3;
  // LayerNorm (eps 1e-6) with two passes over the register-resident row (a row is one quad's values of one h), so
  // that a large mean does not cancel the variance
  uint32_t ay[9][4];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j) s += acc[4 * j + 2 * h] + acc[4 * j + 2 * h + 1];
    const float mean = quad_sum(s) * (1.f / 128.f);
    float d2 = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float d0 = acc[4 * j + 2 * h] - mean, d1 = acc[4 * j + 2 * h + 1] - mean;
      d2 = fmaf(d0, d0, fmaf(d1, d1, d2));
    }
    const float rstd = rsqrtf(quad_sum(d2) * (1.f / 128.f) + 1e-6f);
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float2 w = *reinterpret_cast<const float2*>(cst + C_LNW + 8 * j + 2 * q);
      const float2 b = *reinterpret_cast<const float2*>(cst + C_LNB + 8 * j + 2 * q);
      acc[4 * j + 2 * h] = (acc[4 * j + 2 * h] - mean) * rstd * w.x + b.x;
      acc[4 * j + 2 * h + 1] = (acc[4 * j + 2 * h + 1] - mean) * rstd * w.y + b.y;
    }
  }
#pragma unroll
  for (int s = 0; s < 8; ++s) acc_to_afrag(acc, s, ay[s]);
  float sg[2] = {0.f, 0.f};  // density logit (fp32 dot product of out_geometry_fc.2)
  if (DYNAMIC) {
    named_bar_sync(1 + wg, 128);  // the positional-encoding tiles are complete
    layer_rs_ss<256, 11, 8>(acc, ay, pe_pts, rg);  // ref_pts_fc.0 (bias folded, exp2 scale)
    {
      uint32_t ah[17][4];
      elu_log2_all<128>(acc);
#pragma unroll
      for (int s = 0; s < 16; ++s) acc_to_afrag(acc, s, ah[s]);
      bias_afrag(ah[16], 0, q);  // operand columns 256, 257
      layer_rs<128, 17>(acc, ah, rg);  // ref_pts_fc.2 (bias folded, exp2 scale)
    }
    uint32_t ag[8][4];
    elu_log2_all<64>(acc);
    to_afrag<8>(acc, ag);  // g4
    layer_rs_ss<128, 10, 8>(acc, ag, pe_dir, rg);  // out_geometry_fc.0 (exp2 scale)
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float2 w = *reinterpret_cast<const float2*>(cst + C_WOG2 + 8 * j + 2 * q);
#pragma unroll
      for (int h = 0; h < 2; ++h)
        sg[h] = fmaf(elu_log2(acc[4 * j + 2 * h + 1]), w.y, fmaf(elu_log2(acc[4 * j + 2 * h]), w.x, sg[h]));
    }
    layer_rs_ss<128, 10, 8>(acc, ag, pe_dir, rg);  // rgb_fc.0 (exp2 scale)
    elu_log2_all<64>(acc);
    to_afrag<8>(acc, ag);
    layer_rs_ss<64, 10, 8>(acc, ag, pe_dir, rg);  // rgb_fc.2 (bias folded, exp2 scale) -> rgb_fc.4 dot products
    float pr[3][2] = {{0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float h0 = elu_log2(acc[4 * j + 2 * h]), h1 = elu_log2(acc[4 * j + 2 * h + 1]);
#pragma unroll
        for (int cc = 0; cc < 3; ++cc) {
          const float2 w = *reinterpret_cast<const float2*>(cst + C_WRGB4 + 64 * cc + 8 * j + 2 * q);
          pr[cc][h] = fmaf(h1, w.y, fmaf(h0, w.x, pr[cc][h]));
        }
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float sigma = cst[C_BOG2] + quad_sum(sg[h]);
      const float r0 = cst[C_BRGB4] + quad_sum(pr[0][h]);
      const float r1 = cst[C_BRGB4 + 1] + quad_sum(pr[1][h]);
      const float r2 = cst[C_BRGB4 + 2] + quad_sum(pr[2][h]);
      if (q == 0 && ok[h]) {
        const bool none = nv[h] < 1.f;  // mlp_network.py:297-299, :314
        reinterpret_cast<float4*>(a.raw)[rows[h]] =
            make_float4(none ? 0.f : sigmoid_fast(r0), none ? 0.f : sigmoid_fast(r1),
                        none ? 0.f : sigmoid_fast(r2), none ? -1e9f : sigma - a.shift);
      }
    }
  } else {
    bias_afrag(ay[8], 0, q);  // operand columns 128, 129
    layer_rs<128, 9>(acc, ay, rg);  // out_geometry_fc.0 (bias folded, exp2 scale)
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float2 w = *reinterpret_cast<const float2*>(cst + C_WOG2 + 8 * j + 2 * q);
#pragma unroll
      for (int h = 0; h < 2; ++h)
        sg[h] = fmaf(elu_log2(acc[4 * j + 2 * h + 1]), w.y, fmaf(elu_log2(acc[4 * j + 2 * h]), w.x, sg[h]));
    }
    // per-point part of the blending head, GW = rgb_fc.0[:, :128] y + b (bias folded, true units), fp32 tile layout
    layer_rs<128, 9>(acc, ay, rg);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float sigma = cst[C_BOG2] + quad_sum(sg[h]);
      if (ok[h]) {
#pragma unroll
        for (int j = 0; j < 16; ++j)
          *f32_pair(a.GW, rows[h], 8 * j + 2 * q) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        if (q == 0) a.sigma[rows[h]] = nv[h] < 1.f ? -1e9f : sigma;
      }
    }
  }
}

template <bool DYNAMIC>
__global__ void __launch_bounds__(kWgThreads, 1) point2_wg_kernel(const __grid_constant__ Point2Args a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ __align__(16) FusedChunk s_tab[kWgMaxChunks];
  const uint32_t bar0 = chain_init(smem, P2Smem::kBarOff, s_tab, a.chunks, a.nchunks);
  float* cst = reinterpret_cast<float*>(smem + P2Smem::kConstOff);
  point2_constants(a, cst, DYNAMIC);
  __syncthreads();
  const int tid = threadIdx.x, lane = tid & 31;
  const int n_iter = (int)((a.P + 127) / 128);
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);
  if (wg == 2) {
    chain_producers(s_tab, a.nchunks, a.wimg, a.O, (uint32_t)kP2Tile, n_iter, smem, bar0);
    return;
  }
  setmaxnreg_inc<kConsumerRegs>();
  const int q = lane & 3, ww = (tid & 127) >> 5;
  const int fr[2] = {16 * ww + (lane >> 2), 16 * ww + (lane >> 2) + 8};
  Ring rg{smem, bar0, 0u, false, 0};
  const uint32_t tile = smem_u32(smem + P2Smem::kTileOff) + 1024u * wg;
  uint8_t* pe_pts = smem + P2Smem::kExtraOff + wg * (kPePtsBytes + kPeDirBytes);
  uint8_t* pe_dir = pe_pts + kPePtsBytes;
  uint32_t k = 0;
  for (int it = blockIdx.x; it < n_iter; it += gridDim.x, ++k) {
    const long long row0 = (long long)it * 128 + 64 * wg;
    if (DYNAMIC) {
      named_bar_sync(1 + wg, 128);  // the previous iteration's wgmmas have retired before the tiles are rewritten
      write_pe_tiles(a, row0, pe_pts, pe_dir);
    }
    // residual (fp32 tile layout) and nvalid of this thread's rows: loaded while O lands
    long long rows[2];
    bool ok[2];
    float nv[2];
    float2 res[2][16];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      rows[h] = row0 + fr[h];
      ok[h] = rows[h] < a.P;
      nv[h] = ok[h] ? a.nvalid[rows[h]] : 0.f;
#pragma unroll
      for (int j = 0; j < 16; ++j) res[h][j] = ok[h] ? __ldg(f32_pair(a.g2, rows[h], 8 * j + 2 * q)) : make_float2(0.f, 0.f);
    }
    float acc[128];
    tile_wait(bar0, k);
    layer_ss<128, 8, 128>(acc, tile, rg);  // fc (no bias)
    layer_finish<128>(acc, rg);
    tile_release(bar0);
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        acc[4 * j + 2 * h] += res[h][j].x;
        acc[4 * j + 2 * h + 1] += res[h][j].y;
      }
    point2_heads<DYNAMIC>(acc, a, cst, smem_u32(pe_pts), smem_u32(pe_dir), rows, ok, nv, wg, rg);
  }
}

// ---------------------------------------------------------------------------
// The whole per-point stage in one kernel when S divides 128: point1 -> ray-transformer attention -> point2, with
// g2, Q, K, V and O kept on chip (rows = points; a ray never leaves a 128-row iteration).
//   KEYS = 64 (S divides 64): each warpgroup's 64 rows are whole rays; its keys and values are its own rows.
//   KEYS = 128 (S = 128): the 128 rows are one ray; both warpgroups read all 128 keys and values.
// Q and O stay in registers as A fragments, g2 as the fp32 residual; K and V go to shared memory as K-major
// tiles (k-group stride KEYS x 16 bytes) from the accumulator fragments.  Per head, the logits are one register-A
// wgmma over the keys, the softmax runs on the logit fragment (quad shuffles), P = bf16(e) is the register A of
// O_h = P V_h (V read MN-major), and O_h / den becomes the A fragment of point2's first layer.
// CAPTURE additionally stores g2, Q, K, V and O as point1_wg_kernel and the attention wrote them (test hooks).
// ---------------------------------------------------------------------------
constexpr int kFusedRing = 5;
constexpr int kKvBytes = 2 * 128 * 256;  // K and V of 128 rows, bf16
// the dynamic net's positional-encoding tiles reuse the K / V region once attention is done
using FusedSmem = ChainSmem<kP1Tile, kKvBytes, kP2Const, kFusedRing>;
constexpr float kAttnScale = 0.17677669529663687f;  // 1 / sqrt(32)

// 128 columns of this thread's rows kr[h] -> a K-major key tile of KEYS rows; word(j, h) is the bf16 pair of
// columns 8 j + 2 q, + 1.  Rows that do not exist get zeros: a masked key's P = 0 must not meet a NaN.
template <int KEYS, class W>
__device__ __forceinline__ void store_keys(uint8_t* dst, const int* kr, const bool* ok, int q, W word) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int j = 0; j < 16; ++j)
      *reinterpret_cast<uint32_t*>(dst + j * (KEYS * 16) + (kr[h] >> 3) * 128 + (kr[h] & 7) * 16 + 4 * q) =
          ok[h] ? word(j, h) : 0u;
}

// Attention of this warpgroup's 64 query rows over the key tile kt / value tile vt (KEYS rows each).  Row h of the
// thread attends to keys [lo[h], lo[h] + S) (all KEYS keys when S = KEYS); sc[h] = log2(e) / sqrt(32), or 0 for a
// query row with nvalid <= 1, which attends uniformly (mlp_network.py:23-24, :91-94).
template <int KEYS>
__device__ __forceinline__ void attend(const uint32_t (&qf)[8][4], uint32_t (&of)[8][4], uint32_t kt, uint32_t vt,
                                       const float* sc, const int* lo, int S) {
  constexpr int NL = KEYS / 2, KG = KEYS * 16;
  const int q = threadIdx.x & 3;
  // rows attend to part of the key tile only at KEYS = 64 (S < 64); KEYS = 128 runs S = 128 alone.  Known at compile
  // time, the masks and their key indices cost no registers in the 128-key instantiations, which keeps ptxas from
  // spilling and serializing their wgmmas (C7511).
  const bool part = KEYS == 64 && S < KEYS;
#pragma unroll
  for (int hd = 0; hd < 4; ++hd) {
    float lg[NL];
    fence_regs<NL>(lg);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 2; ++ks)
      WgmmaRS<KEYS>::mma(lg, qf[2 * hd + ks], smem_desc(kt + (2 * hd + ks) * 2 * KG, KG, 128u), ks ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<NL>(lg);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < NL; ++i) {
      const int h = (i >> 1) & 1, key = 8 * (i >> 2) + 2 * q + (i & 1);
      if (!part || (unsigned)(key - lo[h]) < (unsigned)S) mx[h] = fmaxf(mx[h], lg[i]);
    }
    float sh[2], den[2] = {0.f, 0.f};
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
      sh[h] = mx[h] * sc[h];
    }
#pragma unroll
    for (int i = 0; i < NL; ++i) {
      const int h = (i >> 1) & 1, key = 8 * (i >> 2) + 2 * q + (i & 1);
      float e = ex2f(fmaf(lg[i], sc[h], -sh[h]));
      if (part && (unsigned)(key - lo[h]) >= (unsigned)S) e = 0.f;
      lg[i] = e;
      den[h] += e;
    }
    uint32_t pf[KEYS / 16][4];  // P = bf16(e), unnormalised
#pragma unroll
    for (int s = 0; s < KEYS / 16; ++s) acc_to_afrag(lg, s, pf[s]);
    float o[16];
    fence_regs<16>(o);
    wgmma_fence();
    // V_h as MN-major B: dims 32 hd .. (k-groups at stride KG), keys 16 s .. (row groups at stride 128)
#pragma unroll
    for (int s = 0; s < KEYS / 16; ++s)
      WgmmaRS<32, 1>::mma(o, pf[s], smem_desc(vt + 4 * hd * KG + s * 256, 128u, KG), s ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<16>(o);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float inv = 1.f / quad_sum(den[h]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        o[4 * j + 2 * h] *= inv;
        o[4 * j + 2 * h + 1] *= inv;
      }
    }
    acc_to_afrag(o, 0, of[2 * hd]);
    acc_to_afrag(o, 1, of[2 * hd + 1]);
  }
}

// A fragments (k-step s = columns 16 s .. 16 s + 15) of rows row0 + fr[h] <-> bf16 tile image (16 k-groups)
__device__ __forceinline__ void afrag_to_image(const uint32_t (&af)[8][4], void* img, long long row0, const int* fr,
                                               int q, long long P) {
  uint8_t* o = reinterpret_cast<uint8_t*>(img);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const long long row = row0 + fr[h];
    if (row >= P) continue;
#pragma unroll
    for (int s = 0; s < 8; ++s) {
      *reinterpret_cast<uint32_t*>(o + tile_image_off(row, 2 * s, 16) + 4 * q) = af[s][h];
      *reinterpret_cast<uint32_t*>(o + tile_image_off(row, 2 * s + 1, 16) + 4 * q) = af[s][2 + h];
    }
  }
}

template <bool DYNAMIC, int KEYS, bool CAPTURE>
__global__ void __launch_bounds__(kWgThreads, 1) point_fused_wg_kernel(const __grid_constant__ PointFusedArgs a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ __align__(16) FusedChunk s_tab[kWgMaxChunks];
  const Point1Args& p1 = a.p1;
  const Point2Args& p2 = a.p2;
  const uint32_t bar0 = chain_init<kFusedRing>(smem, FusedSmem::kBarOff, s_tab, p1.chunks, p1.nchunks);
  float* cst = reinterpret_cast<float*>(smem + FusedSmem::kConstOff);
  point2_constants(p2, cst, DYNAMIC);
  __syncthreads();
  const long long P = p1.P;
  const int S = p1.S;
  const int n_iter = (int)((P + 127) / 128);
  const int tid = threadIdx.x, lane = tid & 31;
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);
  if (wg == 2) {
    chain_producers<kFusedRing>(s_tab, p1.nchunks, p1.wimg, p1.G, (uint32_t)kP1Tile, n_iter, smem, bar0);
    return;
  }
  setmaxnreg_inc<kConsumerRegs>();
  const int q = lane & 3, ww = (tid & 127) >> 5;
  const int fr[2] = {16 * ww + (lane >> 2), 16 * ww + (lane >> 2) + 8};
  RingN<kFusedRing> rg{smem, bar0, 0u, false, 0};
  const uint32_t tile = smem_u32(smem + FusedSmem::kTileOff) + 1024u * wg;
  uint8_t* kt = smem + FusedSmem::kExtraOff + (KEYS == 64 ? wg * 32768 : 0);
  uint8_t* vt = kt + KEYS * 256;
  const int kr[2] = {(KEYS == 128 ? 64 * wg : 0) + fr[0], (KEYS == 128 ? 64 * wg : 0) + fr[1]};
  uint8_t* pe_pts = smem + FusedSmem::kExtraOff + wg * (KEYS == 64 ? 32768 : kPePtsBytes + kPeDirBytes);
  uint8_t* pe_dir = pe_pts + kPePtsBytes;
  // the warpgroups that share the K / V region
  auto kv_sync = [&]() {
    if (KEYS == 128) named_bar_sync(3, 256);
    else named_bar_sync(1 + wg, 128);
  };
  uint32_t k = 0;
  for (int it = blockIdx.x; it < n_iter; it += gridDim.x, ++k) {
    const long long row0 = (long long)it * 128 + 64 * wg;
    long long rows[2];
    bool ok[2];
    float nv[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      rows[h] = row0 + fr[h];
      ok[h] = rows[h] < P;
      nv[h] = ok[h] ? p2.nvalid[rows[h]] : 0.f;
    }
    float g2[64];
    uint32_t qf[8][4];
    {
      float acc[128];
      tile_wait<kFusedRing>(bar0, k);
      layer_ss<256, 17, 128>(acc, tile, rg);  // geometry_fc.0 (bias folded, exp2 scale)
      layer_finish<256>(acc, rg);
      tile_release<kFusedRing>(bar0);
      {
        uint32_t af[17][4];
        elu_log2_all<128>(acc);
#pragma unroll
        for (int s = 0; s < 16; ++s) acc_to_afrag(acc, s, af[s]);
        bias_afrag(af[16], 8, q);  // operand columns 264, 265
        layer_rs<128, 17>(acc, af, rg);  // geometry_fc.2 (bias folded, exp2 scale)
      }
      // g2 = ELU(geometry_fc.2) (+ sinusoid): the fp32 residual stream, and as bf16 the operand of Q, K, V
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float* pe = p1.posenc ? p1.posenc + (ok[h] ? rows[h] % S : 0) * 128 : nullptr;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int c = 8 * j + 2 * q;
          float v0 = elu_from_log2(acc[4 * j + 2 * h]), v1 = elu_from_log2(acc[4 * j + 2 * h + 1]);
          if (pe) {
            const float2 p = __ldg(reinterpret_cast<const float2*>(pe + c));
            v0 += p.x;
            v1 += p.y;
          }
          g2[4 * j + 2 * h] = v0;
          g2[4 * j + 2 * h + 1] = v1;
          if (CAPTURE && ok[h]) *f32_pair(p1.g2, rows[h], c) = make_float2(v0, v1);
        }
      }
      uint32_t ag[8][4];
      to_afrag<8>(g2, ag);
      layer_rs<128, 8>(acc, ag, rg);  // Wq (no bias)
      to_afrag<8>(acc, qf);
      if (CAPTURE) store_image128(acc, p1.Q, row0, fr, q, P);
      kv_sync();  // every read of the previous iteration's keys, values and encodings is done
      auto pair = [&](int j, int h) { return pack_bf16x2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]); };
      layer_rs<128, 8>(acc, ag, rg);  // Wk
      store_keys<KEYS>(kt, kr, ok, q, pair);
      if (CAPTURE) store_image128(acc, p1.K, row0, fr, q, P);
      layer_rs<128, 8>(acc, ag, rg);  // Wv
      store_keys<KEYS>(vt, kr, ok, q, pair);
      if (CAPTURE) store_image128(acc, p1.V, row0, fr, q, P);
    }
    fence_proxy_async_smem();
    kv_sync();  // keys and values complete
    uint32_t of[8][4];
    {
      float sc[2];
      int lo[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        sc[h] = ok[h] && nv[h] > 1.f ? kAttnScale * kLog2e : 0.f;
        lo[h] = (kr[h] / S) * S;
      }
      attend<KEYS>(qf, of, smem_u32(kt), smem_u32(vt), sc, lo, S);
    }
    if (CAPTURE) afrag_to_image(of, a.O, row0, fr, q, P);
    if (DYNAMIC) {
      kv_sync();  // every read of the keys and values is done
      write_pe_tiles(p2, row0, pe_pts, pe_dir);
    }
    float acc[128];
    layer_rs<128, 8>(acc, of, rg);  // fc (no bias)
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] += g2[i];
    point2_heads<DYNAMIC>(acc, p2, cst, smem_u32(pe_pts), smem_u32(pe_dir), rows, ok, nv, wg, rg);
  }
}

// The attention alone on Q, K, V tile images -> O tile image (the test hook of the fused stage's attention): one CTA
// of two warpgroups per 128-row tile, the same device code as point_fused_wg_kernel.
template <int KEYS>
__global__ void __launch_bounds__(256, 1) attention_wg_kernel(const uint8_t* __restrict__ Q, const uint8_t* __restrict__ K,
                                                              const uint8_t* __restrict__ V,
                                                              const float* __restrict__ nvalid, long long P, int S,
                                                              uint8_t* __restrict__ O) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, lane = tid & 31, wg = tid >> 7;
  const int q = lane & 3, ww = (tid & 127) >> 5;
  const int fr[2] = {16 * ww + (lane >> 2), 16 * ww + (lane >> 2) + 8};
  const long long row0 = (long long)blockIdx.x * 128 + 64 * wg;
  long long rows[2];
  bool ok[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    rows[h] = row0 + fr[h];
    ok[h] = rows[h] < P;
  }
  auto word = [&](const uint8_t* img, int h, int g) {
    return *reinterpret_cast<const uint32_t*>(img + tile_image_off(rows[h], g, 16) + 4 * q);
  };
  uint8_t* kt = smem + (KEYS == 64 ? wg * 32768 : 0);
  uint8_t* vt = kt + KEYS * 256;
  const int kr[2] = {(KEYS == 128 ? 64 * wg : 0) + fr[0], (KEYS == 128 ? 64 * wg : 0) + fr[1]};
  uint32_t qf[8][4], of[8][4];
#pragma unroll
  for (int s = 0; s < 8; ++s)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      qf[s][h] = word(Q, h, 2 * s);
      qf[s][2 + h] = word(Q, h, 2 * s + 1);
    }
  store_keys<KEYS>(kt, kr, ok, q, [&](int j, int h) { return word(K, h, j); });
  store_keys<KEYS>(vt, kr, ok, q, [&](int j, int h) { return word(V, h, j); });
  fence_proxy_async_smem();
  __syncthreads();
  float sc[2];
  int lo[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    sc[h] = ok[h] && nvalid[rows[h]] > 1.f ? kAttnScale * kLog2e : 0.f;
    lo[h] = (kr[h] / S) * S;
  }
  attend<KEYS>(qf, of, smem_u32(kt), smem_u32(vt), sc, lo, S);
  afrag_to_image(of, O, row0, fr, q, P);
}

// ---------------------------------------------------------------------------
// static colour-blending head (rows = (point, view slot), VP slots per point)
// input tile = the X image the per-view kernel writes (16 k-groups); k-step 8 of rgb_fc.0 is a register
// fragment holding [vis2, ray_diff(4), 0 x 11]
// A streaming kernel: its whole weight image (5 chunks, 80 KB) stays in shared memory for the CTA's lifetime, and
// one producer thread keeps kRhDepth iterations in flight, each an X tile plus the GW rows of its 128 / VP points;
// every consumer thread loads the per-row scalars of its next iteration while it finishes the current one, so no
// global load latency sits on the consumers' critical path.
// ---------------------------------------------------------------------------
constexpr int kRhTile = 16 * 2048;
constexpr int kRhChunks = 5;  // rgb_fc.0: 3 chunks (4, 4, 1 k-steps), rgb_fc.2: 2 chunks (8, 1)
constexpr int kRhDepth = 3;   // slots of the X / GW ring: 80 KB + 3 x 40.5 KB
// GW of an iteration's points in a slot: 32 groups of 4 columns (the fp32 tile layout's groups), each group the 16 B
// of every point, group stride padded by 16 B so that the two groups a warp's load touches fall in different banks
template <int VP>
__host__ __device__ constexpr int rh_gw_stride() { return (128 / VP) * 16 + 16; }
constexpr int kRhGw = 32 * rh_gw_stride<8>();
constexpr int C_RW4 = 0, C_RB4 = 64;  // ln 2 x rgb_fc.4 weights, its bias
constexpr int kRhConst = 68;
// shared memory: resident weights | X ring | GW ring | constants | barriers: weights landed, then full / empty per slot
struct RhSmem {
  static constexpr int kXOff = kRhChunks * kWgStage;
  static constexpr int kGwOff = kXOff + kRhDepth * kRhTile;
  static constexpr int kConstOff = kGwOff + kRhDepth * kRhGw;
  static constexpr int kBarOff = (kConstOff + kRhConst * 4 + 7) & ~7;
  static constexpr int kBytes = kBarOff + (1 + 2 * kRhDepth) * 8;
  static_assert(kBytes <= 227 * 1024, "shared memory of one CTA");
};
__device__ __forceinline__ uint32_t rh_full(uint32_t bar0, uint32_t slot) { return bar0 + 8u * (1 + slot); }
__device__ __forceinline__ uint32_t rh_empty(uint32_t bar0, uint32_t slot) {
  return bar0 + 8u * (1 + kRhDepth + slot);
}

// This thread's two rows row0 + fr[h] of an iteration (row0 a multiple of VP): their point, whether it exists,
// whether the view slot holds a view, and the per-view row index m = point * V + view.
template <int VP>
__device__ __forceinline__ void head_rows(const RgbHeadArgs& a, long long row0, const int* fr, long long* pl,
                                          bool* pt_ok, bool* valid, long long* m) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int v = fr[h] & (VP - 1);
    pl[h] = (row0 + fr[h]) / VP;
    pt_ok[h] = pl[h] < a.P;
    valid[h] = pt_ok[h] && v < a.V;
    m[h] = pl[h] * a.V + v;
  }
}

// What an iteration reads from global memory besides the X tile and GW, for this thread's two rows: vis2 and
// ray_diff (operand columns 128..132 of rgb_fc.0; lane q holds columns 2 q, 2 q + 1), the masked-softmax inputs
// and the density passed through to raw.
struct HeadIn {
  float vis[2];
  float4 rd[2];
  float mk[2], c3[2][3], sig[2];
};
// Issues the loads of HeadIn for the iteration whose rows start at row0; rows past the end read zeros.
template <int VP>
__device__ __forceinline__ void head_load(const RgbHeadArgs& a, long long row0, const int* fr, int q, HeadIn& in) {
  long long pl[2], m[2];
  bool pt_ok[2], valid[2];
  head_rows<VP>(a, row0, fr, pl, pt_ok, valid, m);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    in.vis[h] = 0.f;
    in.rd[h] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (valid[h] && q < 3) {
      in.vis[h] = a.vis2[m[h]];
      in.rd[h] = __ldg(reinterpret_cast<const float4*>(a.ray_diff) + m[h]);
    }
    in.mk[h] = 0.f;
    in.c3[h][0] = in.c3[h][1] = in.c3[h][2] = 0.f;
    if (valid[h]) {
      in.mk[h] = a.mask_eff[m[h]];
      in.c3[h][0] = a.rgb_in[m[h] * 3]; in.c3[h][1] = a.rgb_in[m[h] * 3 + 1]; in.c3[h][2] = a.rgb_in[m[h] * 3 + 2];
    }
    in.sig[h] = pt_ok[h] ? a.sigma[pl[h]] : 0.f;
  }
}

template <int VP>
__global__ void __launch_bounds__(kWgThreads, 1) rgbhead_wg_kernel(const __grid_constant__ RgbHeadArgs a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t bar0 = smem_u32(smem + RhSmem::kBarOff);
  float* cst = reinterpret_cast<float*>(smem + RhSmem::kConstOff);
  const int tid = threadIdx.x, lane = tid & 31;
  if (tid == 0) {
    mbar_init(bar0, 1);
    for (int s = 0; s < kRhDepth; ++s) {
      mbar_init(rh_full(bar0, s), 1);
      mbar_init(rh_empty(bar0, s), 8);  // 4 warps x 2 warpgroups
    }
    mbar_fence_init();
  }
  for (int i = tid; i < 64; i += blockDim.x) cst[C_RW4 + i] = a.params[a.o_wrgb4 + i] * kLn2;
  if (tid == 0) cst[C_RB4] = a.params[a.o_brgb4];
  __syncthreads();
  const int n_iter = (int)((a.P * VP + 127) / 128);
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);
  if (wg == 2) {
    setmaxnreg_dec<kProducerRegs>();
    if ((tid & 127) == 0) {
      // the weight image, once
      const uint8_t* w = reinterpret_cast<const uint8_t*>(a.wimg);
      uint32_t bytes = 0;
      for (int c = 0; c < kRhChunks; ++c) bytes += a.chunks[c].bytes;
      mbar_arrive_expect_tx(bar0, bytes);
      for (int c = 0; c < kRhChunks; ++c)
        bulk_g2s(smem_u32(smem + c * kWgStage), w + a.chunks[c].off, a.chunks[c].bytes, bar0);
      // per iteration the X tile and the GW rows of its points, into a slot as soon as both consumer warpgroups have
      // released the slot's previous iteration.  GW is allocated in whole 128-point tiles, so the points of the last
      // iteration that lie past the end can be read too; no output depends on them.
      const uint8_t* x = reinterpret_cast<const uint8_t*>(a.X);
      const uint8_t* gw = reinterpret_cast<const uint8_t*>(a.GW);
      constexpr uint32_t kGwRow = (128 / VP) * 16;  // one group of the iteration's points
      uint32_t k = 0;
      for (int it = blockIdx.x; it < n_iter; it += gridDim.x, ++k) {
        const uint32_t s = k % kRhDepth, full = rh_full(bar0, s);
        if (k >= kRhDepth) mbar_wait(rh_empty(bar0, s), (k / kRhDepth - 1) & 1);
        mbar_arrive_expect_tx(full, kRhTile + 32 * kGwRow);
        bulk_g2s(smem_u32(smem + RhSmem::kXOff + s * kRhTile), x + (size_t)it * kRhTile, kRhTile, full);
        const uint32_t gdst = smem_u32(smem + RhSmem::kGwOff + s * kRhGw);
        const long long p0 = (long long)it * (128 / VP);
        for (int g = 0; g < 32; ++g) bulk_g2s(gdst + g * rh_gw_stride<VP>(), gw + tile_f32_off(p0, g), kGwRow, full);
      }
    }
    return;
  }
  setmaxnreg_inc<kConsumerRegs>();
  const int q = lane & 3, ww = (tid & 127) >> 5;
  const int fr[2] = {16 * ww + (lane >> 2), 16 * ww + (lane >> 2) + 8};
  Resident rg{smem, 0u};
  const uint32_t x0 = smem_u32(smem + RhSmem::kXOff) + 1024u * wg;  // this warpgroup's 64 rows of slot 0
  const uint8_t* gw_slot = smem + RhSmem::kGwOff;
  HeadIn in;
  head_load<VP>(a, (long long)blockIdx.x * 128 + 64 * wg, fr, q, in);
  mbar_wait(bar0, 0);  // the weights have landed
  uint32_t k = 0;
  for (int it = blockIdx.x; it < n_iter; it += gridDim.x, ++k) {
    const long long row0 = (long long)it * 128 + 64 * wg;  // a multiple of VP
    long long pl[2], m[2];
    bool pt_ok[2], valid[2];
    head_rows<VP>(a, row0, fr, pl, pt_ok, valid, m);
    uint32_t a8[4] = {0u, 0u, 0u, 0u};
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float4 rd = in.rd[h];
      a8[h] = q == 0 ? pack_bf16x2(in.vis[h], rd.x) : q == 1 ? pack_bf16x2(rd.y, rd.z)
                                                            : pack_bf16x2(q == 2 ? rd.w : 0.f, 0.f);
    }
    const uint32_t s = k % kRhDepth, tile = x0 + s * kRhTile;
    float acc[64];
    mbar_wait(rh_full(bar0, s), (k / kRhDepth) & 1);
    rg.cnt = 0;
    // rgb_fc.0, per-view part (weights x log2 e): accumulator on the exp2 scale
    layer_issue<128, 9>(acc, rg, [&](float* d, int ks, uint64_t bd, uint32_t sc) {
      if (ks < 8) Wgmma<128, 0, 0>::mma(d, smem_desc(tile + ks * 4096u, 2048u, 128u), bd, sc);
      else WgmmaRS<128>::mma(d, a8, bd, sc);
    });
    // per-point part of rgb_fc.0 (GW, bias included) of this thread's rows, read behind the MMA
    float2 gw[2][16];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint8_t* g = gw_slot + s * kRhGw + ((64 * wg + fr[h]) / VP) * 16 + (q & 1) * 8;
#pragma unroll
      for (int j = 0; j < 16; ++j)
        gw[h][j] = *reinterpret_cast<const float2*>(g + (2 * j + (q >> 1)) * rh_gw_stride<VP>());
    }
    layer_finish<128>(acc, rg);
    __syncwarp();  // this warp's wgmmas that read the slot's X tile have retired, and its GW reads are done
    if (lane == 0) mbar_arrive(rh_empty(bar0, s));
    uint32_t ah[9][4];
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        acc[4 * j + 2 * h] = elu_log2(fmaf(gw[h][j].x, kLog2e, acc[4 * j + 2 * h]));
        acc[4 * j + 2 * h + 1] = elu_log2(fmaf(gw[h][j].y, kLog2e, acc[4 * j + 2 * h + 1]));
      }
    to_afrag<8>(acc, *reinterpret_cast<uint32_t(*)[8][4]>(ah));
    bias_afrag(ah[8], 0, q);  // operand columns 128, 129
    layer_rs<64, 9>(acc, ah, rg);  // rgb_fc.2 (bias folded, exp2 scale) -> rgb_fc.4 logit
    const float mk[2] = {in.mk[0], in.mk[1]}, sig[2] = {in.sig[0], in.sig[1]};
    const float c3[2][3] = {{in.c3[0][0], in.c3[0][1], in.c3[0][2]}, {in.c3[1][0], in.c3[1][1], in.c3[1][2]}};
    head_load<VP>(a, row0 + (long long)gridDim.x * 128, fr, q, in);  // the next iteration's inputs
    float lg[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float2 w = *reinterpret_cast<const float2*>(cst + C_RW4 + 8 * j + 2 * q);
#pragma unroll
      for (int h = 0; h < 2; ++h)
        lg[h] = fmaf(elu_log2(acc[4 * j + 2 * h + 1]), w.y, fmaf(elu_log2(acc[4 * j + 2 * h]), w.x, lg[h]));
    }
    // masked softmax over the views of the point, blend source colours (mlp_network.py:523-525)
    float l[2], mx[2], e[2], den[2], w[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float logit = cst[C_RB4] + quad_sum(lg[h]);
      l[h] = valid[h] ? (mk[h] == 0.f ? -1e9f : logit) : -INFINITY;
    }
    if (VP == 16) {
      mx[0] = mx[1] = rows8_max(fmaxf(l[0], l[1]));
    } else {
      mx[0] = rows8_max(l[0]);
      mx[1] = rows8_max(l[1]);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) e[h] = valid[h] ? __expf(l[h] - mx[h]) : 0.f;
    views_sum<VP>(e, den);
#pragma unroll
    for (int h = 0; h < 2; ++h) w[h] = e[h] / den[h];
    float b[3][2];
#pragma unroll
    for (int cc = 0; cc < 3; ++cc) {
      const float t[2] = {c3[0][cc] * w[0], c3[1][cc] * w[1]};
      views_sum<VP>(t, b[cc]);
    }
    // lane 0 holds view slot 0 of each point: rows 16 ww (+ 8 for the second point of VP = 8)
#pragma unroll
    for (int h = 0; h < (VP == 8 ? 2 : 1); ++h)
      if (lane == 0 && pt_ok[h])
        reinterpret_cast<float4*>(a.raw)[pl[h]] = make_float4(b[0][h], b[1][h], b[2][h], sig[h]);
  }
}

template <class K, class A>
int launch_chain(K kernel, const A& args, long long rows, int smem_bytes, cudaStream_t st) {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    DYN_CUDA(cudaGetDevice(&dev));
    DYN_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  }
  const long long n_iter = (rows + 127) / 128;
  const int grid = (int)(n_iter < sms ? n_iter : sms);  // one persistent CTA per SM
  if (grid == 0) return DYN_OK;
  kernel<<<grid, kWgThreads, smem_bytes, st>>>(args);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

}  // namespace

// ---------------------------------------------------------------------------
// host: weight images of the chains, full layer width per chunk, in the order the warpgroups consume them
// ---------------------------------------------------------------------------
size_t chain_wg_bytes(int kind) { return kind == DYN_NET_MOTION ? 0 : (size_t)(768 * 1024); }

int chain_wg_build(dyn_net* n, const float* P, void* dst_dev, size_t dst_bytes, cudaStream_t st) {
  if (n->kind == DYN_NET_MOTION) return DYN_OK;
  std::vector<uint8_t> img;
  std::vector<FusedChunk> tab;
  char* cur = reinterpret_cast<char*>(dst_dev);
  size_t left = dst_bytes;
  auto add = [&](const LinearP& l, int N, int Kpad, std::vector<int> map, float scale, bool fold_bias,
                 float bias_scale, std::vector<float> colscale = {}) {
    HostLayer L;
    L.W = P + l.w; L.N = N; L.Kw = l.in; L.Npad = N; L.Kpad = Kpad; L.colmap = std::move(map);
    L.scale = scale; L.bias_scale = bias_scale; L.colscale = std::move(colscale);
    if (fold_bias) L.bias = P + l.b;
    append_wg_layer(L, img, tab);
  };
  auto upload = [&](const char* what, ChainImage* out) {
    const int rc = upload_wg_image(img, tab, cur, left, what, out, st);
    if (rc) return rc;
    const size_t used = ((img.size() + 255) & ~(size_t)255) + ((tab.size() * sizeof(FusedChunk) + 255) & ~(size_t)255);
    const size_t step = used < left ? used : left;
    cur += step;
    left -= step;
    img.clear();
    tab.clear();
    return DYN_OK;
  };
  // K columns followed by pad and the folded bias at operand columns hi, hi + 1
  auto with_bias = [](int K, int Kpad, int hi) {
    std::vector<int> m = identity_map(K, Kpad);
    m[hi] = kBiasHi; m[hi + 1] = kBiasLo;
    return m;
  };
  const bool dynamic = n->kind == DYN_NET_DYNAMIC;
  const LinearP &geo0 = dynamic ? n->dl.geo0 : n->sl.geo0, &geo2 = dynamic ? n->dl.geo2 : n->sl.geo2;
  const LinearP &wq = dynamic ? n->dl.wq : n->sl.wq, &wk = dynamic ? n->dl.wk : n->sl.wk;
  const LinearP &wv = dynamic ? n->dl.wv : n->sl.wv, &fc = dynamic ? n->dl.fc : n->sl.fc;
  const LinearP& og0 = dynamic ? n->dl.outgeo0 : n->sl.outgeo0;
  // ---- one image for the per-point stage: point1's layers (its first point1_chunks chunks), then point2's
  // ---- point stage 1: geometry_fc.0 (K = 272: G image, ones at 264, 265), geometry_fc.2 (K = 256 + the
  //      bias k-step, ones at 264, 265), Wq, Wk, Wv as three N = 128 layers
  add(geo0, 256, 272, with_bias(257, 272, 264), kLog2e, true, -1.f);
  add(geo2, 128, 272, with_bias(256, 272, 264), 1.f, true, kLog2e);
  add(wq, 128, 128, identity_map(128, 128), 1.f, false, -1.f);
  add(wk, 128, 128, identity_map(128, 128), 1.f, false, -1.f);
  add(wv, 128, 128, identity_map(128, 128), 1.f, false, -1.f);
  n->point1_chunks = (int)tab.size();
  // ---- point stage 2
  add(fc, 128, 128, identity_map(128, 128), 1.f, false, -1.f);
  if (dynamic) {
    // ref_pts_fc.0 on [y 128 | PE(pts) 33 | 1 1 | 0]; ref_pts_fc.2 consumes the exp2-scale hidden layer
    add(n->dl.refpts0, 256, 176, with_bias(161, 176, 161), kLog2e, true, -1.f);
    add(n->dl.refpts2, 128, 272, with_bias(256, 272, 256), 1.f, true, kLog2e);
    // operand [g4 (exp2 scale) 128 | PE(dir) 27 | 1 1 | 0]: g4 columns x ln2, both outputs on the exp2 scale
    std::vector<float> cs(160, 1.f);
    for (int i = 0; i < 128; ++i) cs[i] = kLn2;
    add(og0, 128, 160, with_bias(128, 160, 155), kLog2e, true, kLog2e, cs);
    add(n->dl.rgb0, 128, 160, with_bias(155, 160, 155), kLog2e, true, kLog2e, cs);
    // rgb_fc.2 on [hidden (exp2 scale) 128 | (PE(dir): zero weights) | 1 1]
    add(n->dl.rgb2, 64, 160, with_bias(128, 160, 155), 1.f, true, kLog2e);
  } else {
    // operand [y 128 | 1 1 | 0]: out_geometry_fc.0 on the exp2 scale, rgb_fc.0[:, :128] + b in true units (= GW)
    add(og0, 128, 144, with_bias(128, 144, 128), kLog2e, true, kLog2e);
    add(n->sl.rgb0, 128, 144, with_bias(128, 144, 128), 1.f, true, 1.f);
  }
  int rc = upload("per-point stage", &n->chain[0]);
  if (rc) return rc;
  if (n->kind == DYN_NET_STATIC) {
    // blending head: operand [x 128 | vis2, ray_diff 4 | pad] <-> rgb_fc.0 columns 128..260 (the per-point
    // columns 0..127 and the bias arrive as GW); rgb_fc.2 on [hidden 128 | 1 1 | 0]
    std::vector<int> m(144, -1);
    for (int i = 0; i < 133; ++i) m[i] = 128 + i;
    add(n->sl.rgb0, 128, 144, m, kLog2e, false, -1.f);
    add(n->sl.rgb2, 64, 144, with_bias(128, 144, 128), 1.f, true, kLog2e);
    rc = upload("blending head", &n->chain[1]);
    if (rc) return rc;
  }
  return DYN_OK;
}

// point2's parameter offsets and density shift
static void point2_layout(const dyn_net* n, Point2Args& a) {
  a.params = n->params;
  a.shift = n->shift;
  if (n->kind == DYN_NET_DYNAMIC) {
    const DynamicLayout& L = n->dl;
    a.o_lnw = L.ln_w; a.o_lnb = L.ln_b; a.o_woutgeo2 = L.outgeo2.w; a.o_boutgeo2 = L.outgeo2.b;
    a.o_wrgb4 = L.rgb4.w; a.o_brgb4 = L.rgb4.b;
  } else {
    const StaticLayout& L = n->sl;
    a.o_lnw = L.ln_w; a.o_lnb = L.ln_b; a.o_woutgeo2 = L.outgeo2.w; a.o_boutgeo2 = L.outgeo2.b;
    a.o_wrgb4 = 0; a.o_brgb4 = 0;
  }
}

int launch_point1_wg(const dyn_net* n, Point1Args& a, cudaStream_t st) {
  if (!n->chain[0].img) return fail(DYN_E_INVALID, "net has no point-stage images");
  a.wimg = n->chain[0].img; a.chunks = n->chain[0].tab; a.nchunks = n->point1_chunks;
  a.params = n->params;
  static bool prepared = false;
  if (!prepared) {
    DYN_CUDA(cudaFuncSetAttribute(point1_wg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, P1Smem::kBytes));
    prepared = true;
  }
  ProfScope prof(PROF_POINT1, st);
  return launch_chain(point1_wg_kernel, a, a.P, P1Smem::kBytes, st);
}

int launch_point2_wg(const dyn_net* n, Point2Args& a, cudaStream_t st) {
  if (!n->chain[0].img) return fail(DYN_E_INVALID, "net has no point-stage images");
  const bool dynamic = n->kind == DYN_NET_DYNAMIC;
  a.wimg = n->chain[0].img; a.chunks = n->chain[0].tab + n->point1_chunks;
  a.nchunks = n->chain[0].nchunks - n->point1_chunks;
  point2_layout(n, a);
  static bool prepared = false;
  if (!prepared) {
    DYN_CUDA(cudaFuncSetAttribute(point2_wg_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, P2Smem::kBytes));
    DYN_CUDA(cudaFuncSetAttribute(point2_wg_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, P2Smem::kBytes));
    prepared = true;
  }
  ProfScope prof(PROF_POINT2, st);
  if (dynamic) return launch_chain(point2_wg_kernel<true>, a, a.P, P2Smem::kBytes, st);
  return launch_chain(point2_wg_kernel<false>, a, a.P, P2Smem::kBytes, st);
}

bool point_fused_supported(int S) { return S >= 1 && S <= 128 && 128 % S == 0; }

namespace {
template <bool DYNAMIC, int KEYS, bool CAPTURE>
int launch_point_fused_t(const PointFusedArgs& a, cudaStream_t st) {
  static bool prepared = false;
  if (!prepared) {
    DYN_CUDA(cudaFuncSetAttribute(point_fused_wg_kernel<DYNAMIC, KEYS, CAPTURE>,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize, FusedSmem::kBytes));
    prepared = true;
  }
  return launch_chain(point_fused_wg_kernel<DYNAMIC, KEYS, CAPTURE>, a, a.p1.P, FusedSmem::kBytes, st);
}
template <bool DYNAMIC, bool CAPTURE>
int launch_point_fused_keys(const PointFusedArgs& a, cudaStream_t st) {
  return a.p1.S == 128 ? launch_point_fused_t<DYNAMIC, 128, CAPTURE>(a, st)
                       : launch_point_fused_t<DYNAMIC, 64, CAPTURE>(a, st);
}
}  // namespace

int launch_point_fused_wg(const dyn_net* n, const Point1Args& p1, const Point2Args& p2, __nv_bfloat16* O_capture,
                          cudaStream_t st) {
  if (!n->chain[0].img) return fail(DYN_E_INVALID, "net has no point-stage images");
  if (!point_fused_supported(p1.S)) return fail(DYN_E_INVALID, "fused point stage: S = %d does not divide 128", p1.S);
  PointFusedArgs a;
  a.p1 = p1;
  a.p2 = p2;
  a.O = O_capture;
  a.p1.wimg = n->chain[0].img; a.p1.chunks = n->chain[0].tab; a.p1.nchunks = n->chain[0].nchunks;
  a.p1.params = n->params;
  point2_layout(n, a.p2);
  const bool dynamic = n->kind == DYN_NET_DYNAMIC;
  ProfScope prof(PROF_POINT1, st);
  if (O_capture)
    return dynamic ? launch_point_fused_keys<true, true>(a, st) : launch_point_fused_keys<false, true>(a, st);
  return dynamic ? launch_point_fused_keys<true, false>(a, st) : launch_point_fused_keys<false, false>(a, st);
}

int launch_attention_wg(const __nv_bfloat16* Q, const __nv_bfloat16* K, const __nv_bfloat16* V, const float* nvalid,
                        long long P, int S, __nv_bfloat16* O, cudaStream_t st) {
  if (!point_fused_supported(S)) return fail(DYN_E_INVALID, "attention: S = %d does not divide 128", S);
  const long long n_tiles = (P + 127) / 128;
  if (n_tiles == 0) return DYN_OK;
  static bool prepared = false;
  if (!prepared) {
    DYN_CUDA(cudaFuncSetAttribute(attention_wg_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, kKvBytes));
    DYN_CUDA(cudaFuncSetAttribute(attention_wg_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, kKvBytes));
    prepared = true;
  }
  ProfScope prof(PROF_ATTENTION, st);
  const uint8_t *q = reinterpret_cast<const uint8_t*>(Q), *k = reinterpret_cast<const uint8_t*>(K),
                *v = reinterpret_cast<const uint8_t*>(V);
  uint8_t* o = reinterpret_cast<uint8_t*>(O);
  if (S == 128) attention_wg_kernel<128><<<(unsigned)n_tiles, 256, kKvBytes, st>>>(q, k, v, nvalid, P, S, o);
  else attention_wg_kernel<64><<<(unsigned)n_tiles, 256, kKvBytes, st>>>(q, k, v, nvalid, P, S, o);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

int launch_rgbhead_wg(const dyn_net* n, RgbHeadArgs& a, cudaStream_t st) {
  if (!n->chain[1].img) return fail(DYN_E_INVALID, "static net has no blending-head images");
  if (n->chain[1].nchunks != kRhChunks)
    return fail(DYN_E_INVALID, "blending-head image has %d chunks, the kernel keeps %d resident", n->chain[1].nchunks,
                kRhChunks);
  a.wimg = n->chain[1].img; a.chunks = n->chain[1].tab; a.nchunks = n->chain[1].nchunks;
  a.params = n->params;
  a.o_wrgb4 = n->sl.rgb4.w; a.o_brgb4 = n->sl.rgb4.b;
  static bool prepared = false;
  if (!prepared) {
    DYN_CUDA(cudaFuncSetAttribute(rgbhead_wg_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, RhSmem::kBytes));
    DYN_CUDA(cudaFuncSetAttribute(rgbhead_wg_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, RhSmem::kBytes));
    prepared = true;
  }
  ProfScope prof(PROF_RGBHEAD, st);
  if (a.V <= 8) return launch_chain(rgbhead_wg_kernel<8>, a, a.P * 8, RhSmem::kBytes, st);
  return launch_chain(rgbhead_wg_kernel<16>, a, a.P * 16, RhSmem::kBytes, st);
}

}  // namespace dyn
