// Shared geometry helpers (camera packing, projection) used by geometry.cu and
// the fused per-view kernel.
#pragma once
#include "common.cuh"

namespace dyn {

// target cameras of one multi-camera launch (dyn_net_static_fused_mc, dyn_project_gather_mc)
constexpr int kMaxTargets = 16;

struct ViewCams {
  float P[kMaxViews][12];   // rows 0..2 of K * inv(c2w)  (projection.py:46-48)
  float center[kMaxViews][3];  // c2w[:3,3]
  float tgt[3];             // target camera centre
  float h_img, w_img;       // train_cameras[0][:2] (projection.py:136)
  float tgts[kMaxTargets][3];  // multi-camera launches: centre of target camera k (tgts[0] == tgt)
};

__device__ __forceinline__ void project_point(const float* P, float x, float y, float z, float& u,
                                              float& v, bool& front) {
  float px = P[0] * x + P[1] * y + P[2] * z + P[3];
  float py = P[4] * x + P[5] * y + P[6] * z + P[7];
  float pz = P[8] * x + P[9] * y + P[10] * z + P[11];
  float d = fmaxf(pz, 1e-8f);  // clamp(min=1e-8), projection.py:51-53
  u = fminf(fmaxf(px / d, -1e6f), 1e6f);
  v = fminf(fmaxf(py / d, -1e6f), 1e6f);
  front = pz > 0.f;
}


// query_cam: n_query target cameras [n_query,34] (n_query <= kMaxTargets) or null
int build_view_cams(const float* src_cams, int V, const float* query_cam, cudaStream_t st,
                    ViewCams* vc, int n_query = 1);
int launch_to_channels_last(const float* featmaps, float* out, int V, int C, int hw, cudaStream_t st);
int launch_to_channels_last_bf16(const float* featmaps, void* out, int V, int C, int hw, cudaStream_t st);
int launch_rgb_to_rgba(const float* rgbs, float* out, long long npix, cudaStream_t st);

}  // namespace dyn
