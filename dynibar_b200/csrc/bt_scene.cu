// The output frames of a monocular bullet-time sweep (render_monocular_bt.py:346-354, restated).  DESIGN §3.9 gives
// the semantics.
//
//   dyn_bt_frames        per group: rendered rgb [K,H,W,3] fp32 -> cropped uint8 frames, one launch
//
// The view pools and rays of a group come from dyn_scene_pools (csrc/scene.cu) and dyn_nvi_rays (csrc/nvi_scene.cu).
#include "common.cuh"

namespace dyn {
namespace {

constexpr int kThreads = 256;

// One thread per output byte: (255 * clip(x, 0, 1)).astype(np.uint8).  The clip maps -inf / +inf / NaN as
// fmaxf / fminf do (NaN -> 0, which is also what numpy's cast of NaN gives on x86); the float32 product is rounded
// on its own (no contraction) and the cast truncates toward zero.
__global__ void __launch_bounds__(kThreads) frames_kernel(const float* __restrict__ rgb, int K, int H, int W,
                                                          int crop_h, int crop_w, uint8_t* __restrict__ out) {
  const int ho = H - 2 * crop_h, wo = W - 2 * crop_w;
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= (long long)K * ho * wo * 3) return;
  const int c = (int)(i % 3);
  const long long px = i / 3;
  const int x = (int)(px % wo);
  const long long ky = px / wo;
  const int y = (int)(ky % ho), k = (int)(ky / ho);
  const float v = rgb[(((long long)k * H + y + crop_h) * W + x + crop_w) * 3 + c];
  out[i] = (uint8_t)__float2uint_rz(__fmul_rn(255.0f, fminf(fmaxf(v, 0.0f), 1.0f)));
}

}  // namespace
}  // namespace dyn

using namespace dyn;

extern "C" {

int dyn_bt_frames(const float* rgb, int K, int H, int W, int crop_h, int crop_w, uint8_t* out, void* stream) {
  DYN_CHECK_ARG(rgb && out && K >= 1 && H >= 1 && W >= 1 && crop_h >= 0 && crop_w >= 0);
  DYN_CHECK_ARG(2 * crop_h < H && 2 * crop_w < W && (long long)K * H * W * 3 < (1ll << 31));
  const long long n = (long long)K * (H - 2 * crop_h) * (W - 2 * crop_w) * 3;
  frames_kernel<<<(unsigned)cdiv(n, kThreads), kThreads, 0, (cudaStream_t)stream>>>(rgb, K, H, W, crop_h, crop_w, out);
  DYN_LAUNCH_CHECK();
  return DYN_OK;
}

}  // extern "C"
