// Warpgroup engine of the Hopper fused kernels (view_wg.cu, chains_wg.cu, motion_wg.cu): one persistent CTA per SM with two
// consumer warpgroups and a producer warpgroup.  Each consumer warpgroup owns 64 rows of the CTA's 128-row
// iteration and issues its own wgmmas, one instruction per k-step for the whole layer width; the accumulators
// stay in registers, and a hidden layer's output, packed to bf16 pairs, is the register A operand of the next
// layer (tc::acc_to_afrag).  Both warpgroups consume the same weight chunks from one ring; a slot is refilled
// only when both have retired it, so the weights are fetched once per 128 rows.
//
// Fragment layout (warp w of the warpgroup, lane l, q = l % 4): accumulator i holds row 16 w + l / 4 + 8 h,
// column 8 j + 2 q + e with j = i / 4, h = (i / 2) % 2, e = i % 2.  A row's dot products are quad shuffles
// (xor 1, 2); 8 or 16 aligned rows of one warp's 16-row slab are shuffles over the row lanes (xor 4, 8, 16)
// plus, for 16 rows, the in-thread h pair.
#pragma once
#include <vector>

#include "fused_engine.cuh"

namespace dyn {
namespace wg {

using namespace tc;
using namespace fe;

constexpr int kWgRing = 8;
constexpr int kWgStage = 16384;
// two consumer warpgroups + a producer warpgroup; setmaxnreg moves the producer's registers to the consumers:
// 2 x 128 x 232 + 128 x 40 <= 64 K
constexpr int kWgThreads = 3 * 128;
constexpr int kConsumerRegs = 232, kProducerRegs = 40;
constexpr int kWgMaxChunks = 72;  // the MotionMLP's image has 68 chunks

// k-steps per weight chunk of a layer N wide (one ring stage; at most 8, as fe::append_block cuts them)
__host__ __device__ constexpr int wg_chunk_ksteps(int N) { return kWgStage / (N * 32) < 8 ? kWgStage / (N * 32) : 8; }

// 8 consecutive columns [c0, c0 + 8) of a row of a 64-row operand tile -> one 16-byte store
__device__ __forceinline__ void store8_64(uint8_t* arow, int c0, const float* v) {
  *reinterpret_cast<uint4*>(arow + (c0 >> 3) * 1024) =
      make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
}

// The weight ring as one consumer warpgroup sees it: chunk `cnt` sits in slot cnt % RING.
template <int RING>
struct RingN {
  uint8_t* base;
  uint32_t bar0;  // [0, RING) full, [RING, 2 RING) empty
  uint32_t cnt;
  bool prof;
  long long wait_cycles;  // profiling: cycles spent waiting for weights
  __device__ __forceinline__ uint32_t wait_full(uint32_t c) {
    const uint32_t st = c % RING;
    const long long t0 = prof ? clock64() : 0;
    mbar_wait(bar0 + 8u * st, (c / RING) & 1);
    if (prof) wait_cycles += clock64() - t0;
    return smem_u32(base + st * kWgStage);
  }
  // this warp's wgmmas that read chunk c have retired (the empty barrier counts 4 warps x 2 warpgroups)
  __device__ __forceinline__ void release(uint32_t c) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(bar0 + 8u * (RING + c % RING));
  }
};
using Ring = RingN<kWgRing>;

// A weight image resident in shared memory for the kernel's lifetime, landed once before the first iteration:
// chunk c of an iteration sits in slot c, so there is nothing to wait for and nothing to release.  The consumer
// resets cnt to 0 at the start of every iteration.
struct Resident {
  uint8_t* base;
  uint32_t cnt;
  __device__ __forceinline__ uint32_t wait_full(uint32_t c) const { return smem_u32(base + c * kWgStage); }
  __device__ __forceinline__ void release(uint32_t) const {}
};

// Issues one layer, D[64 x N] = A[64 x 16 KS] W^T, chunk by chunk as the weights arrive; each chunk's slot is
// released as soon as the next chunk's wgmmas are committed and its own have retired.  The last chunk stays in
// flight: layer_finish waits for it.  mma(acc, kstep, b_desc, scale_d) issues one k-step.
template <int N, int KS, class RG, class Mma>
__device__ __forceinline__ void layer_issue(float* acc, RG& rg, Mma mma) {
  constexpr int KC = wg_chunk_ksteps(N), NCH = (KS + KC - 1) / KC;
  fence_regs<N / 2>(acc);
  wgmma_fence();
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    const uint32_t w = rg.wait_full(rg.cnt + c);
#pragma unroll
    for (int s = 0; s < KC; ++s)
      if (c * KC + s < KS) mma(acc, c * KC + s, smem_desc(w + s * N * 32u, N * 16u, 128u), (c | s) ? 1u : 0u);
    wgmma_commit();
    if (c > 0) {
      wgmma_wait<1>();
      rg.release(rg.cnt + c - 1);
    }
  }
  rg.cnt += NCH;
}
template <int N, class RG>
__device__ __forceinline__ void layer_finish(float* acc, RG& rg) {
  wgmma_wait<0>();
  fence_regs<N / 2>(acc);
  rg.release(rg.cnt - 1);
}

// A from a K-major operand tile of ROWS rows (this warpgroup's 64 rows start at a_tile)
template <int N, int KS, int ROWS = 64, class RG>
__device__ __forceinline__ void layer_ss(float* acc, uint32_t a_tile, RG& rg) {
  layer_issue<N, KS>(acc, rg, [&](float* d, int ks, uint64_t bd, uint32_t sc) {
    Wgmma<N, 0, 0>::mma(d, smem_desc(a_tile + ks * (ROWS * 32u), ROWS * 16u, 128u), bd, sc);
  });
}
template <int N, int KS, class RG>
__device__ __forceinline__ void layer_rs(float* acc, const uint32_t (&af)[KS][4], RG& rg) {
  layer_issue<N, KS>(acc, rg, [&](float* d, int ks, uint64_t bd, uint32_t sc) { WgmmaRS<N>::mma(d, af[ks], bd, sc); });
  layer_finish<N>(acc, rg);
}
// One layer whose first KR k-steps take A from register fragments and the rest from a 64-row operand tile.
template <int N, int KS, int KR, class RG>
__device__ __forceinline__ void layer_rs_ss(float* acc, const uint32_t (*af)[4], uint32_t tile64, RG& rg) {
  layer_issue<N, KS>(acc, rg, [&](float* d, int ks, uint64_t bd, uint32_t sc) {
    if (ks < KR) WgmmaRS<N>::mma(d, af[ks < KR ? ks : 0], bd, sc);
    else Wgmma<N, 0, 0>::mma(d, smem_desc(tile64 + (ks - KR) * 2048u, 1024u, 128u), bd, sc);
  });
  layer_finish<N>(acc, rg);
}

// ReLU(acc + bias[column]) in place, N columns of fragment layout (q = lane % 4)
template <int N>
__device__ __forceinline__ void bias_relu(float* acc, const float* bias, int q) {
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    const float2 b = *reinterpret_cast<const float2*>(bias + 8 * j + 2 * q);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      acc[4 * j + 2 * h] = fmaxf(acc[4 * j + 2 * h] + b.x, 0.f);
      acc[4 * j + 2 * h + 1] = fmaxf(acc[4 * j + 2 * h + 1] + b.y, 0.f);
    }
  }
}
// ELU(acc + bias[column]) in place, N columns of fragment layout (q = lane % 4)
template <int N>
__device__ __forceinline__ void bias_elu(float* acc, const float* bias, int q) {
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    const float2 b = *reinterpret_cast<const float2*>(bias + 8 * j + 2 * q);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      acc[4 * j + 2 * h] = elu_fast(acc[4 * j + 2 * h] + b.x);
      acc[4 * j + 2 * h + 1] = elu_fast(acc[4 * j + 2 * h + 1] + b.y);
    }
  }
}
template <int KS>
__device__ __forceinline__ void to_afrag(const float* acc, uint32_t (&af)[KS][4]) {
#pragma unroll
  for (int s = 0; s < KS; ++s) acc_to_afrag(acc, s, af[s]);
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
// sum over the row lanes of a fragment (8 rows of one h)
__device__ __forceinline__ float rows8_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  v += __shfl_xor_sync(0xffffffffu, v, 8);
  return v + __shfl_xor_sync(0xffffffffu, v, 16);
}
// sum over a point's view slots of per-row values v[h] (VP = 8: the point of row half h; VP = 16: both halves)
template <int VP>
__device__ __forceinline__ void views_sum(const float* v, float* s) {
  if (VP == 16) {
    s[0] = s[1] = rows8_sum(v[0] + v[1]);
  } else {
    s[0] = rows8_sum(v[0]);
    s[1] = rows8_sum(v[1]);
  }
}

// ---- host side: weight images as full-width chunks, in the order the warpgroups consume them ----
inline void append_wg_layer(const HostLayer& L, std::vector<uint8_t>& img, std::vector<FusedChunk>& tab) {
  append_block(L, img, tab, 0, 0, 0, 0, kWgStage, 0, L.Kpad / 16);
}

// copies an image and its chunk table to dst_dev (image first, table 256-byte aligned after it)
inline int upload_wg_image(const std::vector<uint8_t>& img, const std::vector<FusedChunk>& tab, void* dst_dev,
                           size_t dst_bytes, const char* what, ChainImage* out, cudaStream_t st) {
  const size_t img_bytes = (img.size() + 255) & ~(size_t)255;
  const size_t need = img_bytes + tab.size() * sizeof(FusedChunk);
  if (need > dst_bytes) return fail(DYN_E_INVALID, "%s images need %zu bytes, have %zu", what, need, dst_bytes);
  if (tab.size() > (size_t)kWgMaxChunks) return fail(DYN_E_INVALID, "%s chunk table too long (%zu)", what, tab.size());
  DYN_CUDA(cudaMemcpyAsync(dst_dev, img.data(), img.size(), cudaMemcpyHostToDevice, st));
  DYN_CUDA(cudaMemcpyAsync(reinterpret_cast<char*>(dst_dev) + img_bytes, tab.data(), tab.size() * sizeof(FusedChunk),
                           cudaMemcpyHostToDevice, st));
  DYN_CUDA(cudaStreamSynchronize(st));
  out->img = dst_dev;
  out->tab = reinterpret_cast<const FusedChunk*>(reinterpret_cast<char*>(dst_dev) + img_bytes);
  out->nchunks = (int)tab.size();
  return DYN_OK;
}

}  // namespace wg
}  // namespace dyn
