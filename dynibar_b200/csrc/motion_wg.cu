// The MotionMLP in one tensor-core kernel, built for Hopper on the warpgroup engine (wg_engine.cuh):
//
//   motion_wg_kernel : PE(xyzt) -> 8 x (256, ReLU) with skip -> 18 coeffs
//                      (mlp_network.py:605-618 + render_ray.py:459-472)
//
// One persistent CTA per SM; each of the two consumer warpgroups owns 64 rows of the CTA's 128-row iteration.
// A warpgroup writes PE(xyzt) of its rows to a 64-row bf16 operand tile once per iteration; pts_linears.0 reads
// A from that tile, every later layer from the previous layer's registers, and the skip layer pts_linears.5 on
// cat([PE, h]) takes the 16 k-steps of h from registers first and then the 9 PE k-steps from the tile.  Each
// layer is one wgmma per k-step at its full width.  The biases stay out of the MMA: the epilogue adds them in
// fp32 on the accumulator registers (bias_relu), as the fp32 path does.
//
// Rounding points: bf16 PE and weights, fp32 accumulation and bias, bf16 hidden activations, fp32 coefficients.
#include "nets.cuh"
#include "wg_engine.cuh"

namespace dyn {

using namespace tc;
using namespace fe;
using namespace wg;

namespace {

// operand columns of PE(xyzt): for k in 0..15: [cos(f_k x)(4) | sin(f_k x)(4)], then [x(4) | 0 x 12]
constexpr int kPeCols = 144, kPeKsteps = kPeCols / 16;
constexpr int kPeTileBytes = 64 * kPeCols * 2;
// constants (floats): the biases of pts_linears.0 .. 7 (256 each), then coeff_linear's (32, zero past ncoef)
constexpr int kMotionConst = 8 * 256 + 32;
// shared memory: weight ring | one PE tile per consumer warpgroup | constants | ring barriers
constexpr int kPeOff = kWgRing * kWgStage;
constexpr int kConstOff = kPeOff + 2 * kPeTileBytes;
constexpr int kBarOff = kConstOff + kMotionConst * 4;
constexpr int kSmemMotion = kBarOff + 2 * kWgRing * 8;
static_assert(kSmemMotion + kWgMaxChunks * 16 <= 227 * 1024, "shared memory of one CTA");

// PE(xyzt) of dims d0, d0 + 1 (values x2) of one row into the 64-row operand tile (row byte offset `arow`); the
// other thread of the row writes the other two dims.  f_k = 1 + k * 16/15 (torch.linspace(1, 17, 16)), by the
// angle-addition recurrence.  Rows past N get zeros.
__device__ __forceinline__ void motion_pe(uint8_t* arow, const float* x2, int d0, bool valid) {
  const float delta = 16.f / 15.f;
  float c[2], s[2], cd[2], sd[2];
#pragma unroll
  for (int d = 0; d < 2; ++d) {
    __sincosf(x2[d], &s[d], &c[d]);
    __sincosf(x2[d] * delta, &sd[d], &cd[d]);
  }
  // column group k: cos of dims 0..3 at bytes 0..7, sin at 8..15; dims d0, d0 + 1 are 2 d0 bytes in
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    uint8_t* g = arow + k * 1024 + 2 * d0;
    *reinterpret_cast<uint32_t*>(g) = valid ? pack_bf16x2(c[0], c[1]) : 0u;
    *reinterpret_cast<uint32_t*>(g + 8) = valid ? pack_bf16x2(s[0], s[1]) : 0u;
#pragma unroll
    for (int d = 0; d < 2; ++d) {
      const float cn = c[d] * cd[d] - s[d] * sd[d];
      const float sn = s[d] * cd[d] + c[d] * sd[d];
      c[d] = cn; s[d] = sn;
    }
  }
  uint8_t* g = arow + 16 * 1024 + 2 * d0;
  *reinterpret_cast<uint32_t*>(g) = valid ? pack_bf16x2(x2[0], x2[1]) : 0u;
  *reinterpret_cast<uint32_t*>(g + 8) = 0u;
  *reinterpret_cast<uint2*>(arow + 17 * 1024 + d0 * 4) = make_uint2(0u, 0u);
}

__global__ void __launch_bounds__(kWgThreads, 1) motion_wg_kernel(const __grid_constant__ MotionFusedArgs a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ __align__(16) FusedChunk s_tab[kWgMaxChunks];
  const int tid = threadIdx.x, lane = tid & 31;
  const uint32_t bar0 = smem_u32(smem + kBarOff);
  float* cst = reinterpret_cast<float*>(smem + kConstOff);
  stage_chunks(s_tab, a.chunks, a.nchunks);
  for (int i = tid; i < 2048; i += blockDim.x) cst[i] = a.params[a.o_bias[i >> 8] + (i & 255)];
  if (tid < 32) cst[2048 + tid] = tid < a.ncoef ? a.params[a.o_bias[8] + tid] : 0.f;
  if (tid == 0) {
    for (int i = 0; i < kWgRing; ++i) {
      mbar_init(bar0 + 8u * i, 1);
      mbar_init(bar0 + 8u * (kWgRing + i), 8);  // 4 warps x 2 warpgroups
    }
    mbar_fence_init();
  }
  __syncthreads();
  const int n_iter = (int)((a.N + 127) / 128);
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);  // warpgroup index, uniform to the compiler
  if (wg == 2) {
    setmaxnreg_dec<kProducerRegs>();
    if ((tid & 127) == 0) producer_loop<kWgRing, kWgStage>(s_tab, a.nchunks, a.wimg, n_iter, smem, bar0);
    return;
  }
  setmaxnreg_inc<kConsumerRegs>();
  const int q = lane & 3, ww = (tid & 127) >> 5;
  const int fr[2] = {16 * ww + (lane >> 2), 16 * ww + (lane >> 2) + 8};
  Ring rg{smem, bar0, 0u, false, 0};
  uint8_t* pe = smem + kPeOff + wg * kPeTileBytes;
  const uint32_t pe_tile = smem_u32(pe);
  // PE rows: thread t of the warpgroup writes dims 2 (t / 64), + 1 of row t % 64
  const int r = tid & 63, d0 = 2 * ((tid & 127) >> 6);
  uint8_t* arow = pe + (r >> 3) * 128 + (r & 7) * 16;
  for (int it = blockIdx.x; it < n_iter; it += gridDim.x) {
    const long long row0 = (long long)it * 128 + 64 * wg;
    {
      named_bar_sync(1 + wg, 128);  // the previous iteration's wgmmas have retired before the tile is rewritten
      const long long row = row0 + r;
      const bool valid = row < a.N;
      float x2[2] = {0.f, d0 == 0 ? 0.f : a.time};  // dims d0, d0 + 1 of (x, y, z, t)
      if (valid) {
        const float* src = a.x + row * a.ldx + d0;
        x2[0] = src[0];
        if (d0 == 0 || a.time_is_column) x2[1] = src[1];
      }
      motion_pe(arow, x2, d0, valid);
      fence_proxy_async_smem();
      named_bar_sync(1 + wg, 128);  // the tile is complete
    }
    float acc[128];
    uint32_t af[16][4];
    layer_ss<256, kPeKsteps>(acc, pe_tile, rg);  // pts_linears.0
    layer_finish<256>(acc, rg);
#pragma unroll 1
    for (int l = 0; l < 7; ++l) {
      bias_relu<256>(acc, cst + 256 * l, q);
      to_afrag<16>(acc, af);
      if (l == 4) layer_rs_ss<256, 16 + kPeKsteps, 16>(acc, af, pe_tile, rg);  // pts_linears.5: h, then PE
      else layer_rs<256, 16>(acc, af, rg);                                     // pts_linears.1 .. 4, 6, 7
    }
    bias_relu<256>(acc, cst + 256 * 7, q);
    to_afrag<16>(acc, af);
    layer_rs<32, 16>(acc, af, rg);  // coeff_linear (ncoef of 32 columns)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long row = row0 + fr[h];
      if (row < a.N) {
        float* dst = a.coeff + row * a.ncoef;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int c = 8 * j + 2 * q;
          if (c < a.ncoef) dst[c] = acc[4 * j + 2 * h] + cst[2048 + c];
          if (c + 1 < a.ncoef) dst[c + 1] = acc[4 * j + 2 * h + 1] + cst[2048 + c + 1];
        }
      }
    }
  }
}

}  // namespace

size_t motion_wg_bytes() { return (size_t)(1280 * 1024); }

int motion_wg_build(dyn_net* n, const float* P, void* dst_dev, size_t dst_bytes, cudaStream_t st) {
  std::vector<uint8_t> img;
  std::vector<FusedChunk> tab;
  auto add = [&](const LinearP& l, int N, int Npad, std::vector<int> map) {
    HostLayer L;
    L.W = P + l.w; L.N = N; L.Kw = l.in; L.Npad = Npad; L.Kpad = (int)map.size();
    L.colmap = std::move(map);
    append_wg_layer(L, img, tab);
  };
  const MotionLayout& L = n->ml;
  // operand order: k-major [cos f_k (4) | sin f_k (4)] x 16, then x(4): weight column of each
  std::vector<int> pe(kPeCols, -1);
  for (int k = 0; k < 16; ++k)
    for (int d = 0; d < 4; ++d) { pe[8 * k + d] = 4 + 4 * k + d; pe[8 * k + 4 + d] = 68 + 4 * k + d; }
  for (int d = 0; d < 4; ++d) pe[128 + d] = d;
  add(L.pts[0], 256, 256, pe);
  for (int i = 1; i < 5; ++i) add(L.pts[i], 256, 256, identity_map(256, 256));
  {  // pts_linears.5 on cat([pe(132), h(256)]): the h columns first, then the PE columns
    std::vector<int> m(256 + kPeCols);
    for (int i = 0; i < 256; ++i) m[i] = 132 + i;
    for (int i = 0; i < kPeCols; ++i) m[256 + i] = pe[i];
    add(L.pts[5], 256, 256, m);
  }
  add(L.pts[6], 256, 256, identity_map(256, 256));
  add(L.pts[7], 256, 256, identity_map(256, 256));
  add(L.coeff, 3 * n->nb, 32, identity_map(256, 256));
  return upload_wg_image(img, tab, dst_dev, dst_bytes, "motion", &n->motion, st);
}

int launch_motion_wg(const dyn_net* n, MotionFusedArgs& a, cudaStream_t st) {
  if (!n->motion.img) return fail(DYN_E_INVALID, "motion net has no fused images");
  a.wimg = n->motion.img; a.chunks = n->motion.tab; a.nchunks = n->motion.nchunks;
  a.params = n->params;
  for (int i = 0; i < 8; ++i) a.o_bias[i] = n->ml.pts[i].b;
  a.o_bias[8] = n->ml.coeff.b;
  a.ncoef = 3 * n->nb;
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    DYN_CUDA(cudaGetDevice(&dev));
    DYN_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    DYN_CUDA(cudaFuncSetAttribute(motion_wg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMotion));
  }
  ProfScope prof(PROF_MOTION, st);
  const long long n_iter = (a.N + 127) / 128;
  const int grid = (int)(n_iter < sms ? n_iter : sms);  // one persistent CTA per SM
  if (grid == 0) return DYN_OK;
  motion_wg_kernel<<<grid, kWgThreads, kSmemMotion, st>>>(a);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

}  // namespace dyn
