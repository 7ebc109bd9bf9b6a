// Shared machinery of the fused tensor-core kernels (nets_fused.cu, motion_wg.cu, chains_wg.cu,
// view_*.cu): smem budget constants, fast activations, A-tile stores, view-group shuffles, the
// table-driven weight producer and MMA warpgroup, and the host-side packing of weight chunks into
// wgmma B-operand images.
#pragma once
#include <vector>

#include "nets_fused.cuh"
#include "tc.cuh"

namespace dyn {
namespace fe {

using namespace tc;

constexpr int kRing = 4;
constexpr int kStageBytes = 16384;
constexpr int kNB = 64;              // widest N-block of a chunk (accumulator registers of the MMA warpgroup)

__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float elu_fast(float x) {
  float e = ex2f(x * 1.4426950408889634f);
  return x > 0.f ? x : e - 1.f;
}
// ELU on the exp2 scale: x2 = log2(e) * x in, log2(e) * ELU(x) out (4 instructions; the producing layer's
// weights and folded bias carry the log2 e, the consuming layer's weights the ln 2)
__device__ __forceinline__ float elu_log2(float x2) {
  const float e = ex2f(x2);
  return x2 > 0.f ? x2 : fmaf(e, 1.4426950408889634f, -1.4426950408889634f);
}
// ELU in true units from an accumulator on the exp2 scale (x2 = log2(e) * x): 4 instructions
__device__ __forceinline__ float elu_from_log2(float x2) {
  const float e = ex2f(x2);
  return x2 > 0.f ? x2 * 0.6931471805599453f : e - 1.f;
}
__device__ __forceinline__ float sigmoid_fast(float x) {
  return __frcp_rn(1.f + ex2f(-x * 1.4426950408889634f));
}

// 8 consecutive columns [c0, c0+8) of this thread's row -> one 16-byte store
__device__ __forceinline__ void store8(uint8_t* arow, int c0, const float* v) {
  uint4 q;
  q.x = pack_bf16x2(v[0], v[1]);
  q.y = pack_bf16x2(v[2], v[3]);
  q.z = pack_bf16x2(v[4], v[5]);
  q.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(arow + (c0 >> 3) * 2048) = q;
}

// acc[32] (+bias, ELU) -> bf16 columns [c0, c0+32) of the A tile, optional row scale
template <bool kElu>
__device__ __forceinline__ void epi32_to_A(uint8_t* arow, int c0, float* acc, const float* bias,
                                           float scale) {
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    float v = acc[i] + bias[c0 + i];
    if (kElu) v = elu_fast(v);
    acc[i] = v * scale;
  }
#pragma unroll
  for (int g = 0; g < 4; ++g) store8(arow, c0 + 8 * g, acc + 8 * g);
}

// PE with frequencies 2^k via angle doubling: out = [x(D), cos(2^k x)(NF*D), sin(2^k x)(NF*D)]
template <int D, int NF>
__device__ __forceinline__ void pe_pow2(const float* x, float* out) {
#pragma unroll
  for (int d = 0; d < D; ++d) {
    out[d] = x[d];
    float s, c;
    __sincosf(x[d], &s, &c);
#pragma unroll
    for (int k = 0; k < NF; ++k) {
      out[D + k * D + d] = c;
      out[D + NF * D + k * D + d] = s;
      float s2 = 2.f * s * c, c2 = 1.f - 2.f * s * s;
      s = s2; c = c2;
    }
  }
}

template <int VP>
__device__ __forceinline__ float group_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  if (VP == 16) v += __shfl_xor_sync(0xffffffffu, v, 8);
  return v;
}
template <int VP>
__device__ __forceinline__ float group_min(float v) {
  v = fminf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  v = fminf(v, __shfl_xor_sync(0xffffffffu, v, 2));
  v = fminf(v, __shfl_xor_sync(0xffffffffu, v, 4));
  if (VP == 16) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, 8));
  return v;
}

// one reduce-scatter step over N values: lanes with `bit` set keep the upper half
template <int N>
__device__ __forceinline__ void rs_step(const float* in, float* out, bool upper, int xr) {
#pragma unroll
  for (int i = 0; i < N / 2; ++i) {
    float send = upper ? in[i] : in[N / 2 + i];
    float keep = upper ? in[N / 2 + i] : in[i];
    out[i] = keep + __shfl_xor_sync(0xffffffffu, send, xr);
  }
}


// "Tile image": how bf16 activations travel between fused kernels through HBM.  Rows are grouped in
// tiles of 128 and stored exactly as the consumer's wgmma A operand sits in shared memory (K-major
// 8x8 core matrices): element (row r, column k) of a tile with KG 8-column groups lives at byte
//   tile * KG * 2048 + (k / 8) * 2048 + (r % 128) * 16 + (k % 8) * 2.
// The producer's per-row 16-byte stores are therefore warp-coalesced (32 rows x 16 B = 512 B), and
// the consumer lands a whole operand block with ONE cp.async.bulk instead of per-thread loads.
__host__ __device__ __forceinline__ size_t tile_image_off(long long row, int kgroup, int kgroups) {
  return (size_t)(row >> 7) * (size_t)kgroups * 2048u + (size_t)kgroup * 2048u + (size_t)(row & 127) * 16u;
}
__host__ __device__ __forceinline__ size_t tile_image_bytes(long long rows, int kgroups) {
  return (size_t)((rows + 127) >> 7) * (size_t)kgroups * 2048u;
}

// fp32 companion of the tile image for per-point vectors that stay fp32 (residual stream g2, the
// blending head's per-point term GW): 128 columns in groups of 4 floats, element (row r, column c)
// of a 128-row tile at byte  tile * 65536 + (c / 4) * 2048 + (r % 128) * 16 + (c % 4) * 4,
// so that both the producer's and the consumer's per-row float4 accesses are warp-coalesced.
__host__ __device__ __forceinline__ size_t tile_f32_off(long long row, int col4group) {
  return (size_t)(row >> 7) * 65536u + (size_t)col4group * 2048u + (size_t)(row & 127) * 16u;
}

// The chunk table is staged into shared memory once per CTA: the producer and the issuer
// read one entry per chunk on their critical path (a global load there costs an L2 round trip
// per chunk and was the bottleneck of the MMA issue thread).
constexpr int kMaxChunks = 160;
__device__ __forceinline__ void stage_chunks(FusedChunk* s, const FusedChunk* __restrict__ g, int n) {
  static_assert(sizeof(FusedChunk) == 16, "FusedChunk is copied as uint4");
  const uint4* src = reinterpret_cast<const uint4*>(g);
  uint4* dst = reinterpret_cast<uint4*>(s);
  for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
}

// ---- control warps: the weight producer and the MMA warpgroup --------------------
// One 128-row tile served by two threads per row (twin warps), one a_ready / acc_full barrier pair.
// barrier layout for a ring of `ring` slots: [0,ring) w_full, [ring,2 ring) w_empty, then a_ready, acc_full
__device__ __forceinline__ uint32_t bar_aready(uint32_t bar0, int ring = kRing) { return bar0 + 8u * (2 * ring); }
__device__ __forceinline__ uint32_t bar_acc(uint32_t bar0, int ring = kRing) { return bar0 + 8u * (2 * ring + 1); }

// The MMA warpgroup: 4 warps, warp-index aligned (wgmma is issued by a whole warpgroup).  w_empty completes
// when each of its warps has retired the wgmmas that read the slot (one arrival per warp), acc_full when
// all of its threads have stored their accumulator fragments (one arrival per thread).
constexpr int kIssuerWarps = 4;
// `arrivals` = row threads that signal a_ready per 128-row tile
__device__ __forceinline__ void init_barriers(uint32_t bar0, int arrivals, int ring = kRing) {
  for (int i = 0; i < ring; ++i) { mbar_init(bar0 + 8u * i, 1); mbar_init(bar0 + 8u * (ring + i), kIssuerWarps); }
  mbar_init(bar_aready(bar0, ring), arrivals);
  mbar_init(bar_acc(bar0, ring), 32 * kIssuerWarps);
  mbar_fence_init();
}

// Called by one thread: streams the weight chunks of every iteration through the ring.
template <int RING = kRing, int STAGE = kStageBytes>
__device__ __forceinline__ void producer_loop(const FusedChunk* __restrict__ chunks, int nchunks,
                                              const void* wimg, int n_iter, uint8_t* ring, uint32_t bar0) {
  const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(wimg);
  uint32_t cnt = 0;
  for (int it = blockIdx.x; it < n_iter; it += gridDim.x) {
    for (int c = 0; c < nchunks; ++c, ++cnt) {
      const uint32_t st = cnt % RING;
      if (cnt >= RING) mbar_wait(bar0 + 8u * (RING + st), ((cnt / RING) - 1) & 1);
      const FusedChunk ch = chunks[c];
      mbar_arrive_expect_tx(bar0 + 8u * st, ch.bytes);
      bulk_g2s(smem_u32(ring + st * STAGE), wsrc + ch.off, ch.bytes, bar0 + 8u * st);
    }
  }
}

// One N-block of a chunk for the accumulators of the tile: 2 x 64-row wgmmas per k-step.
template <int NB>
__device__ __forceinline__ void mma_chunk(float (&acc)[2][kNB / 2], uint32_t a_addr, const FusedChunk& ch,
                                          uint32_t w_addr) {
  const uint32_t lbo_b = (uint32_t)NB * 16u;
  const uint32_t aa = a_addr + (uint32_t)ch.a_kgroup * 2048u;
  for (int ks = 0; ks < ch.ksteps; ++ks) {
    const uint64_t bd = smem_desc(w_addr + ks * 2u * lbo_b, lbo_b, 128u);
    const uint32_t sc = ((ch.flags & 8) && ks == 0) ? 0u : 1u;
#pragma unroll
    for (int h = 0; h < 2; ++h)
      Wgmma<NB, 0, 0>::mma(acc[h], smem_desc(aa + ks * 4096u + h * 1024u, 2048u, 128u), bd, sc);
  }
}
// accumulators <-> accumulator memory (columns from col0, col0 including d_col)
template <int NB>
__device__ __forceinline__ void acc_chunk_io(float (&acc)[2][kNB / 2], int col0, bool store) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (store) acc_store_frag<NB>(acc[h], 64 * h, col0);
    else acc_load_frag<NB>(acc[h], 64 * h, col0);
  }
}

// one chunk start to finish: resume the N-block from accumulator memory if it continues one, multiply,
// wait for the wgmmas to retire, store the N-block if it ends here
template <int NB>
__device__ __forceinline__ void run_chunk(float (&acc)[2][kNB / 2], uint32_t a_addr, const FusedChunk& ch,
                                          uint32_t w_addr, uint32_t tmem_base) {
  const int col0 = (int)(tmem_base & 0xffffu) + ch.d_col;
  if ((ch.flags & 40) == 32) acc_chunk_io<NB>(acc, col0, false);
  fence_regs<NB / 2>(acc[0]); fence_regs<NB / 2>(acc[1]);
  wgmma_fence();
  mma_chunk<NB>(acc, a_addr, ch, w_addr);
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs<NB / 2>(acc[0]); fence_regs<NB / 2>(acc[1]);
  if (ch.flags & 16) acc_chunk_io<NB>(acc, col0, true);
}

// Called by ALL 128 threads of the MMA warpgroup (warps 4k .. 4k + 3 of the CTA).
// FusedChunk.flags: 1 = wait for a_ready before this chunk, 2 = last chunk of a
// round (signal acc_full), 8 = first k-step overwrites D (start of a layer),
// 16 / 32 = last / first chunk of an N-block (store it to TMEM / without 8: continue from TMEM);
// d_col = accumulator column offset inside the tile's 256-column TMEM region.
// RING = weight-ring slots in use.
template <int RING = kRing, int STAGE = kStageBytes>
__device__ __forceinline__ void issuer_loop(const FusedChunk* __restrict__ chunks, int nchunks, int n_iter,
                                            uint8_t* smem, uint8_t* ring, uint32_t bar0,
                                            uint32_t tmem_base, long long* dbg = nullptr) {
  // wgmma is issued by the whole warpgroup; the accumulators of one N-block (<= kNB columns) stay in
  // registers across the N-block's chunks
  {
    float acc[2][kNB / 2];
    const bool lead = threadIdx.x % 128 == 0;
    uint32_t cnt = 0, a_cnt = 0;
    long long t_a = 0, t_w = 0, t_begin = clock64();
    const uint32_t a_addr = smem_u32(smem);
    for (int it = blockIdx.x; it < n_iter; it += gridDim.x) {
      for (int c = 0; c < nchunks; ++c, ++cnt) {
        const FusedChunk ch = chunks[c];
        long long t0 = dbg ? clock64() : 0;
        if (ch.flags & 1) {
          mbar_wait(bar_aready(bar0, RING), a_cnt & 1);
          ++a_cnt;
        }
        long long t1 = dbg ? clock64() : 0;
        const uint32_t st = cnt % RING;
        mbar_wait(bar0 + 8u * st, (cnt / RING) & 1);
        tc_fence_after_sync();
        long long t2 = 0;
        if (dbg) {
          t2 = clock64();
          t_a += t1 - t0;
          t_w += t2 - t1;
        }
        const uint32_t w_addr = smem_u32(ring + st * STAGE);
        switch (ch.npad) {
          case 16: run_chunk<16>(acc, a_addr, ch, w_addr, tmem_base); break;
          case 32: run_chunk<32>(acc, a_addr, ch, w_addr, tmem_base); break;
          case 48: run_chunk<48>(acc, a_addr, ch, w_addr, tmem_base); break;
          case 64: run_chunk<64>(acc, a_addr, ch, w_addr, tmem_base); break;
          default: __trap();  // the host packer emits N-blocks of 16, 32, 48 or 64 columns only
        }
        __syncwarp();
        if ((threadIdx.x & 31) == 0) mbar_arrive(bar0 + 8u * (RING + st));  // this warp's wgmmas have retired
        if (ch.flags & 2) mbar_arrive(bar_acc(bar0, RING));
        if (dbg && blockIdx.x == 0 && lead && cnt < 120) {
          dbg[8 + 4 * cnt + 0] = t0; dbg[8 + 4 * cnt + 1] = t1;
          dbg[8 + 4 * cnt + 2] = t2; dbg[8 + 4 * cnt + 3] = clock64();
        }
      }
    }
    if (dbg != nullptr && blockIdx.x == 0 && lead) {
      dbg[0] = clock64() - t_begin;  // issuer lifetime
      dbg[1] = t_a;                  // waiting for A operands (epilogues)
      dbg[2] = t_w;                  // waiting for weight chunks (ring)
    }
  }
  __syncwarp();
}

// ---- host side: weight images + chunk table ------------------------------------
inline uint16_t f2bf(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);  // NaN
  uint32_t lsb = (u >> 16) & 1u;
  u += 0x7fffu + lsb;  // round to nearest even
  return (uint16_t)(u >> 16);
}

struct HostLayer {
  const float* W;  // host fp32 [*, Kw]
  int N, Kw, Npad, Kpad;
  std::vector<int> colmap;  // size Kpad: weight column, -1 (zero), or kBiasHi / kBiasLo
  // bias folded into the MMA: the operand carries 1.0 in the kBiasHi and kBiasLo columns and the image
  // holds bf16(b) and bf16(b - bf16(b)) there (error 2^-17 |b|); `scale` multiplies weights and bias
  // (log2 e for layers whose ELU is evaluated on the exp2 scale, ln 2 for their consumers)
  const float* bias = nullptr;
  float scale = 1.f;
  float bias_scale = -1.f;  // < 0: same as `scale` (differs when the layer CONSUMES a log2-scaled operand
                            // and PRODUCES an exp2-scale accumulator: weights x ln2 x log2e = 1, bias x log2e)
  std::vector<float> colscale;  // optional, size Kpad: extra factor per OPERAND column (operand tiles that mix
                                // exp2-scale activations with true-scale encodings)
};
constexpr int kBiasHi = -2, kBiasLo = -3;
inline float bf2f(uint16_t h) {
  uint32_t u = (uint32_t)h << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}

// rows [n0, n0 + nb) of a layer as a layer of its own (an N-block)
inline HostLayer layer_rows(const HostLayer& L, int n0, int nb) {
  HostLayer B = L;
  B.N = L.N - n0 < nb ? (L.N - n0 > 0 ? L.N - n0 : 0) : nb;
  B.Npad = nb;
  if (B.N > 0) {
    B.W = L.W + (size_t)n0 * L.Kw;
    if (L.bias != nullptr) B.bias = L.bias + n0;
  }
  return B;
}

// One N-block (L.Npad <= kNB outputs), k-steps [k_begin, k_end), cut into chunks of at most one ring stage;
// `first_flags` go on the first chunk, `last_flags` on the last.
inline void append_block(const HostLayer& L, std::vector<uint8_t>& img, std::vector<FusedChunk>& tab,
                         int d_col, int a_kgroup0, int first_flags, int last_flags, int stage_bytes, int k_begin,
                         int k_end) {
  int steps_per_chunk = stage_bytes / (L.Npad * 32);
  if (steps_per_chunk > 8) steps_per_chunk = 8;
  for (int k0 = k_begin; k0 < k_end; k0 += steps_per_chunk) {
    const int ks = (k_end - k0) < steps_per_chunk ? (k_end - k0) : steps_per_chunk;
    FusedChunk ch;
    ch.off = (uint32_t)img.size();
    ch.bytes = (uint32_t)(L.Npad * 32 * ks);
    ch.npad = (uint16_t)L.Npad;
    ch.ksteps = (uint8_t)ks;
    ch.flags = (uint8_t)((k0 == k_begin ? first_flags : 0) | (k0 + ks >= k_end ? last_flags : 0));
    ch.a_kgroup = (uint16_t)(a_kgroup0 + k0 * 2);
    ch.d_col = (uint16_t)d_col;
    img.resize(img.size() + ch.bytes, 0);
    uint16_t* dst = reinterpret_cast<uint16_t*>(img.data() + ch.off);
    for (int n = 0; n < L.Npad; ++n)
      for (int kk = 0; kk < ks * 16; ++kk) {
        const int col = L.colmap[k0 * 16 + kk];
        float val = 0.f;
        if (n < L.N) {
          if (col >= 0) {
            val = L.W[(size_t)n * L.Kw + col] * L.scale * (L.colscale.empty() ? 1.f : L.colscale[k0 * 16 + kk]);
          } else if (L.bias != nullptr && (col == kBiasHi || col == kBiasLo)) {
            const float b = L.bias[n] * (L.bias_scale >= 0.f ? L.bias_scale : L.scale), hi = bf2f(f2bf(b));
            val = col == kBiasHi ? hi : b - hi;
          }
        }
        dst[tile_off((uint32_t)L.Npad, (uint32_t)n, (uint32_t)kk) / 2] = f2bf(val);
      }
    tab.push_back(ch);
  }
}

// A layer as N-blocks of at most kNB output columns, each streamed over all of K before the next one (the
// MMA warpgroup keeps one N-block's accumulators in registers).  The operand wait of `first_flags` (1) goes
// on the layer's first chunk, its 8 ("overwrite D") on the first chunk of every N-block.
inline void append_layer(const HostLayer& L, std::vector<uint8_t>& img, std::vector<FusedChunk>& tab,
                         int d_col = 0, int a_kgroup0 = 0, int first_flags = 9, bool last = true,
                         int stage_bytes = kStageBytes) {
  for (int n0 = 0; n0 < L.Npad; n0 += kNB)
    append_block(layer_rows(L, n0, L.Npad - n0 < kNB ? L.Npad - n0 : kNB), img, tab, d_col + n0, a_kgroup0,
                 32 | (n0 == 0 ? first_flags & 1 : 0) | (first_flags & 8),
                 16 | (last && n0 + kNB >= L.Npad ? 2 : 0), stage_bytes, 0, L.Kpad / 16);
}

inline std::vector<int> identity_map(int K, int Kpad) {
  std::vector<int> m(Kpad, -1);
  for (int i = 0; i < K; ++i) m[i] = i;
  return m;
}

}  // namespace fe
}  // namespace dyn
