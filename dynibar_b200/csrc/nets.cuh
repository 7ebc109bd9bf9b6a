// Internal interfaces between the network implementations and the C ABI.
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"

namespace dyn {

int net_rows_per_chunk(int S, int V);

// fp32 SIMT parity mode (nets_f32.cu)
size_t net_dynamic_f32_workspace(int R, int S, int V);
size_t net_static_f32_workspace(int R, int S, int V);
size_t motion_f32_workspace(long long N);
int net_dynamic_f32(const dyn_net* n, const float* pts, const float* rgb_feat, const float* ray_dir,
                    const float* mask, float time, int R, int S, int V, float* raw, void* ws,
                    size_t ws_bytes, int prec, cudaStream_t st, bool train = false);
int net_static_f32(const dyn_net* n, const float* pts, const float* ref_rays, const float* src_rays,
                   const float* rgb_feat, const float* ray_diff, const float* mask, int R, int S, int V,
                   float* raw, void* ws, size_t ws_bytes, int prec, cudaStream_t st, bool train = false);
int motion_f32(const dyn_net* n, const float* x, int ldx, bool time_is_column, float time, long long N,
               float* coeff, void* ws, size_t ws_bytes, int prec, cudaStream_t st);
// fused DYN_PREC_BF16 path (per-view stage = nets_fused.cu)
size_t net_fused_workspace(int kind, int R, int S, int V);
// query_cams [K,34]; query_idx [R] (device) = target camera of each ray, null for one camera
int net_static_fused(const dyn_net* n, const float* pts, const float* ray_o, const float* ray_d,
                     const float* query_cams, int K, const int* query_idx, const float* src_rgbs,
                     const float* src_cams, const void* feat_cl, int R, int S, int V, int H, int W, int h,
                     int w, float* raw, float* mask_out, void* ws, size_t ws_bytes, cudaStream_t st);
int net_dynamic_fused(const dyn_net* n, const float* pts, const float* pts_seq, const float* ray_dir,
                      const float* query_cam, const float* src_rgbs, const float* src_cams,
                      const void* feat_cl, float time, int R, int S, int V, int H, int W, int h, int w,
                      float* raw, float* mask_out, void* ws, size_t ws_bytes, cudaStream_t st);
int debug_point_chain(const dyn_net* n, const float* G, const float* nvalid, const float* pts,
                      const float* ray_dir, int R, int S, float* g2, float* Q, float* K, float* V,
                      float* O, float* out_a, float* out_b, float* posenc_ws, cudaStream_t st);
int debug_attention(const float* Q, const float* K, const float* V, const float* nvalid, int R, int S, float* O,
                    cudaStream_t st);
int debug_rgb_head(const dyn_net* n, const float* X, const float* vis2, const float* ray_diff, const float* mask_eff,
                   const float* rgb_in, const float* GW, const float* sigma, long long P, int V, float* raw,
                   cudaStream_t st);
void set_view_capture(float* G, float* nvalid, float* X, float* vis2, float* mask_eff, float* ray_diff,
                      float* rgb_in);
// tensor-core ray-transformer attention (attention_tc.cu); S must divide 128
bool attention_tc_supported(int S);
int launch_attention_tc(const __nv_bfloat16* Q, const __nv_bfloat16* K, const __nv_bfloat16* V,
                        const float* nvalid, long long P, int S, __nv_bfloat16* O, cudaStream_t st);
int zero_last_samples(float* coeff, int R, int S, int width, cudaStream_t st);
// training slice of the MotionMLP (motion_train.cu); embedding hooks live in nets_f32.cu
int motion_embed(const float* xyzt, long long N, float* x0, cudaStream_t st);
void motion_freqs(float f[16]);
size_t motion_train_workspace(long long N);
int motion_train_forward(const dyn_net* n, const float* xyzt, long long N, float* coeff, void* ws,
                         size_t ws_bytes, int prec, cudaStream_t st);
int motion_train_backward(const dyn_net* n, const float* xyzt, const float* d_coeff, long long N, void* ws,
                          size_t ws_bytes, float* d_params, float* d_xyzt, int prec, cudaStream_t st);

// training backward of the two aggregation nets (nets_train.cu); the forward is net_*_f32(..., train = true)
size_t net_train_workspace(int kind, int R, int S, int V);
size_t net_backward_scratch(int kind, int R, int S, int V);
int net_dynamic_backward(const dyn_net* n, const float* pts, const float* rgb_feat, const float* ray_dir,
                         const float* mask, int R, int S, int V, const float* d_raw, void* ws, size_t ws_bytes,
                         void* scratch, size_t scratch_bytes, float* d_params, float* d_rgb_feat, float* d_pts,
                         int prec, cudaStream_t st);
int net_static_backward(const dyn_net* n, const float* rgb_feat, const float* ray_diff, int R, int S, int V,
                        const float* d_raw, void* ws, size_t ws_bytes, void* scratch, size_t scratch_bytes,
                        float* d_params, float* d_rgb_feat, int prec, cudaStream_t st);

}  // namespace dyn
