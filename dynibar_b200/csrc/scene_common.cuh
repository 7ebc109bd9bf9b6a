// Device helpers the scene kernels share (csrc/scene.cu: the monocular scene, csrc/nvi_scene.cu: the Nvidia scene).
#pragma once

#include <math.h>

namespace dyn {

// cv2 resizeNN (INTER_NEAREST): src index of dst index x = min(floor(x * (1 / (dst / src))), src - 1), in double
__device__ __forceinline__ int nn_index(int x, int dst, int src) {
  const double ifx = 1.0 / ((double)dst / (double)src);
  return min((int)floor((double)x * ifx), src - 1);
}

// u8 / 255.0f as numpy rounds it
__device__ __forceinline__ float u8f(uint8_t v) { return __fdiv_rn((float)v, 255.0f); }

// The ray of pixel (u, v) (sample_ray.py:143-163): cam = M [3x3 row-major] | t [3] with M = R_c2w K^-1 formed on the
// host in float32; ray_d = M [u, v, 1]^T summed left to right without contraction, ray_o = t.
__device__ __forceinline__ void pixel_ray(const float* __restrict__ cam, float u, float v, float* __restrict__ ray_o,
                                          float* __restrict__ ray_d) {
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    ray_d[a] = __fadd_rn(__fadd_rn(__fmul_rn(cam[3 * a], u), __fmul_rn(cam[3 * a + 1], v)), cam[3 * a + 2]);
    ray_o[a] = cam[9 + a];
  }
}

}  // namespace dyn
