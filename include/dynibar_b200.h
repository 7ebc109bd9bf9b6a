/* dynibar_b200 -- C ABI of the CUDA-native DynIBaR per-ray IBR hot path (H100, sm_90a).
 *
 * The reference (google/dynibar @ 5412b55) has no FFI layer: its boundary for
 * this path is the Python call surface of ibrnet/render_ray.py,
 * ibrnet/projection.py and ibrnet/mlp_network.py.  Each entry point below
 * names the reference function (file:line in the reference checkout) it replaces;
 * the Python modules under dynibar_b200/ bind them with ctypes behind the reference's own
 * function / class names (see INTEGRATION.md).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless its name ends in `_host`;
 *     tensors are dense row-major fp32 unless stated; shapes in comments.
 *     The tiny per-frame arrays (`*_cam`, `*_cams`, `basis`) may be HOST
 *     pointers as well: host copies are read without synchronising the stream.
 *   - the caller owns every buffer (inputs, outputs, workspace, packed
 *     weights); the library keeps no device pointer after return except inside
 *     a `dyn_net_t` handle.  Its one allocation: on the first fused tensor-core
 *     launch on a device it allocates device memory for the accumulators of the
 *     fused kernels (2 x SMs x 256 KB, kept for the life of the process; a
 *     CTA holds one slot of it while it runs, so streams can share it).  The
 *     first fused launches on a device must not be inside a stream capture.
 *   - workspaces and scratch buffers (`workspace`, `scratch`, `feat_cl_ws`,
 *     `posenc_ws`, ...): the base must be 256-byte aligned, because the
 *     library carves them into sub-buffers that assume it.  An entry point
 *     neither depends on what a workspace held before the call (every byte
 *     it reads it wrote first in the same call) nor writes past the size its
 *     `*_workspace_bytes` / `*_scratch_bytes` function declares, whatever
 *     the buffer's real size.  Outputs likewise: an entry point writes only
 *     inside their stated extents and reads none of their prior contents
 *     unless it says it accumulates into them (the `d_params` of the
 *     training backwards).
 *   - `saved` buffers (the train forwards) are not scratch: they carry state
 *     from a train forward to its backward and must be passed unchanged.
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it,
 *     nothing synchronises.
 *   - return 0 on success, a negative DYN_E_* otherwise; `dyn_last_error()`
 *     returns a thread-local message.  No C++ exceptions cross the ABI.
 *   - R rays, S samples per ray, V source views, C feature channels (32),
 *     F = C + 3.
 */
#ifndef DYNIBAR_B200_H_
#define DYNIBAR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DYN_OK 0
#define DYN_E_INVALID -1 /* bad argument / unsupported shape */
#define DYN_E_CUDA -2    /* a CUDA runtime call or launch failed */
#define DYN_E_WORKSPACE -3 /* workspace too small */

#define DYN_NET_DYNAMIC 0 /* DynibarDynamic, mlp_network.py:129 */
#define DYN_NET_STATIC 1  /* DynibarStatic,  mlp_network.py:319 */
#define DYN_NET_MOTION 2  /* MotionMLP,      mlp_network.py:558 */

#define DYN_PREC_FP32 0 /* SIMT fp32 everywhere (parity mode) */
#define DYN_PREC_BF16 1 /* tensor cores (wgmma): bf16 operands, fp32 accumulate/statistics */

typedef struct dyn_net* dyn_net_t;

int dyn_version(void);
const char* dyn_last_error(void);
/* Number of SMs etc. of the current device (for grid sizing diagnostics). */
int dyn_device_sm_count(void);
/* Kernels launched by this library since load (or the last reset). */
unsigned long long dyn_launch_count(int reset);

/* (debug / measurement hooks below -- dyn_profile_*, dyn_debug_*, dyn_launch_count -- keep process-global
 * state and are NOT thread-safe; the entry points of the path itself only touch caller-owned buffers.) */
/* Optional device timing of the big kernels (CUDA events on the launching
 * stream, recorded inside the library around each launch).  Classes: 0 fused
 * static per-view stage, 1 fused dynamic per-view stage, 2 MotionMLP, 3 point
 * stage 1, 4 point stage 2, 5 static blending head, 6 ray-transformer attention,
 * 7 stand-alone projection+gather.  enable(1) clears previous records. */
void dyn_profile_enable(int on);
int dyn_profile_read(int cls, float* total_ms, int* launches);

/* ---- weights ------------------------------------------------------------
 * `params` is the flat fp32 concatenation of the network's state_dict tensors
 * in the canonical order documented in dynibar_b200/weights.py (reference key
 * names, mlp_network.py:159-214 / :349-403 / :591-603).  `n_params` is checked
 * against the expected count.  `packed` is a caller-owned device buffer of
 * dyn_net_packed_bytes(kind) bytes that receives the tensor-core operand
 * images (bf16, wgmma canonical layout); it may be NULL for DYN_PREC_FP32 use.
 * n_samples sizes the sinusoid table of the dynamic net (mlp_network.py:218).
 */
size_t dyn_net_param_count(int kind);
size_t dyn_net_packed_bytes(int kind);
int dyn_net_create(int kind, const float* params, size_t n_params, void* packed,
                   int n_samples, float shift, int anti_alias_pooling,
                   int mask_rgb, void* stream, dyn_net_t* out);
/* pack_level: 0 = fp32 parameters only (packed may be NULL), 1 = per-layer tensor-core images only
 * (dyn_net_layer_images_bytes(kind) bytes: enough for the staged DYN_PREC_BF16 evaluation and the bf16 training
 * step, cheap enough to rebuild after every optimizer step), 2 = everything (== dyn_net_create). */
size_t dyn_net_layer_images_bytes(int kind);
int dyn_net_create_ex(int kind, const float* params, size_t n_params, void* packed, int pack_level,
                      int n_samples, float shift, int anti_alias_pooling, int mask_rgb, void* stream,
                      dyn_net_t* out);
void dyn_net_destroy(dyn_net_t net);

/* ---- a2: sample_along_camera_ray, render_ray.py:67-131 -------------------
 * ray_o, ray_d [R,3]; jitter [R,S] of U[0,1) or NULL (det=True).
 * Outputs pts [R,S,3], z_vals [R,S], s_vals [R,S]. */
int dyn_sample_rays(const float* ray_o, const float* ray_d, float near_depth,
                    float far_depth, int R, int S, int inv_uniform,
                    const float* jitter, float* pts, float* z_vals,
                    float* s_vals, void* stream);

/* pts = z * d + o and s = z_to_s(z) for given depths
 * (render_ray.py:822-831, :399-404).  s_vals may be NULL. */
int dyn_points_from_depths(const float* ray_o, const float* ray_d,
                           const float* z_vals, float near_depth,
                           float far_depth, int R, int S, float* pts,
                           float* s_vals, void* stream);

/* ---- a3: MotionMLP + trajectory displacement ------------------------------
 * mlp_network.py:605-618; render_ray.py:361-369, :462-500.
 * coeff [R,S,3*nb] with the last round(0.1*S) samples zeroed. */
size_t dyn_motion_workspace_bytes(int R, int S);
int dyn_motion_coeffs(dyn_net_t motion, const float* pts, float time, int R,
                      int S, float* coeff, void* workspace,
                      size_t workspace_bytes, int precision, void* stream);
/* generic MotionMLP forward on xyzt rows [N,4] -> [N,3*nb]
 * (MotionMLP.forward, no zeroing). */
int dyn_motion_mlp(dyn_net_t motion, const float* xyzt, int N, float* coeff,
                   void* workspace, size_t workspace_bytes, int precision,
                   void* stream);
/* pts_seq[v] = pts + traj(frame+off_v) - traj(frame) for the n_off temporal
 * offsets, followed by num_vv copies of pts.  basis [T,nb] (model.py:18-30).
 * offsets_host is a HOST array.  pts_seq [n_off+num_vv, R, S, 3]. */
int dyn_traj_displace(const float* pts, const float* coeff, const float* basis,
                      int T, int nb, int frame_idx, const int* offsets_host,
                      int n_off, int num_vv, int R, int S, float* pts_seq,
                      void* stream);

/* ---- a16 helpers: cross-time branch of render_rays_mono, render_ray.py:1099-1270
 * out[v] = traj(frames_a[v]) - traj(frames_b[v]) with traj(f) = sum_k coeff_k basis[f,k]
 * (scene-flow sequence :1101-1105); frames_*_host are HOST arrays, n <= 8. */
int dyn_traj_delta(const float* coeff, const float* basis, int T, int nb,
                   const int* frames_a_host, const int* frames_b_host, int n,
                   int R, int S, float* out, void* stream);
/* occ [R,S] = 1 - |w_ref - w_anchor|, occ_map [R] = 1 - |sum_s (w_ref - w_anchor)| (:1224-1257) */
int dyn_occlusion_weights(const float* w_ref, const float* w_anchor, int R, int S,
                          float* occ, float* occ_map, void* stream);

/* ---- a4-a6: Projector.compute_with_motions, projection.py:103-176 ---------
 * xyz_st [R,S,3]; xyz [V,R,S,3] or NULL (every view uses xyz_st: the static
 * branch, render_ray.py:498-500); query_cam [34]; src_rgbs [V,H,W,3]
 * channels-last in [0,1]; src_cams [V,34]; featmaps [V,C,h,w] (reference
 * layout).  Outputs rgb_feat [R,S,V,3+C], ray_diff [R,S,V,4], mask [R,S,V].
 * feat_cl_ws: workspace of V*h*w*C floats for the channels-last copy of the
 * feature maps. */
int dyn_project_gather(const float* xyz_st, const float* xyz,
                       const float* query_cam, const float* src_rgbs,
                       const float* src_cams, const float* featmaps, int V,
                       int R, int S, int H, int W, int C, int h, int w,
                       float* feat_cl_ws, float* rgb_feat, float* ray_diff,
                       float* mask, void* stream);
/* Multi-camera form of dyn_project_gather: the rays of K target cameras of one time step in one call.
 * query_cams [K,34] (host or device, read like query_cam), 1 <= K <= 16; query_idx [R] (device, int32):
 * ray r belongs to target camera query_idx[r], whose centre enters its ray_diff.  query_idx may be NULL
 * only when K = 1 (it is ignored then: the call is dyn_project_gather).  The kernel trusts the index
 * values: the caller keeps them in [0, K).  K and query_idx are checked before any CUDA call. */
int dyn_project_gather_mc(const float* xyz_st, const float* xyz,
                          const float* query_cams, int K, const int* query_idx,
                          const float* src_rgbs, const float* src_cams,
                          const float* featmaps, int V, int R, int S, int H,
                          int W, int C, int h, int w, float* feat_cl_ws,
                          float* rgb_feat, float* ray_diff, float* mask,
                          void* stream);
/* Pooled multi-camera form: every target camera has its own view slots, drawn from one shared pool of source
 * views.  src_rgbs [pool,H,W,3], src_cams [pool,34] and featmaps [pool,C,h,w] hold the pool (1 <= pool <= 32);
 * view_tbl [K,V] int32 (host or device) names the pool entry of slot v of camera k, camera_index [R] (device,
 * int32; NULL allowed when K = 1) the camera of each ray.  Slot v of ray r projects onto, and gathers from, pool
 * entry view_tbl[camera_index[r], v]; xyz [V,R,S,3] and the outputs stay indexed by slot.  With
 * view_tbl[k] = 0..V-1 for every k the call is dyn_project_gather_mc.  K, camera_index, view_tbl, pool and
 * 1 <= V <= 32 are checked before any CUDA call; the table's values (in [0, pool)) are checked before any launch.
 * The kernel trusts camera_index to lie in [0, K). */
int dyn_project_gather_tbl(const float* xyz_st, const float* xyz,
                           const float* query_cams, int K, const int* camera_index,
                           const int* view_tbl, int pool, const float* src_rgbs,
                           const float* src_cams, const float* featmaps, int V, int R,
                           int S, int H, int W, int C, int h, int w, float* feat_cl_ws,
                           float* rgb_feat, float* ray_diff, float* mask, void* stream);
/* compute_projections only (projection.py:32-59): pix [V,N,2], front [V,N] u8 */
int dyn_compute_projections(const float* xyz, const float* src_cams, int V,
                            int N, float* pix, uint8_t* front, void* stream);

/* compute_angle only (projection.py:61-101): xyz_st [st_views,N,3] with st_views 1 (same reference
 * point for every view) or V; xyz [V,N,3]; ray_diff [V,N,4] = [normalize(a - b), a . b] with
 * a = normalize(c_tgt - xyz_st), b = normalize(c_src_v - xyz_v). */
int dyn_compute_angle(const float* xyz_st, int st_views, const float* xyz,
                      const float* query_cam, const float* src_cams, int V, int N,
                      float* ray_diff, void* stream);

/* ---- a7: Plucker coordinates, render_ray.py:372-396 ---------------------- */
int dyn_plucker_ref(const float* ray_o, const float* ray_d, int R, float* out6,
                    void* stream);
int dyn_plucker_src(const float* pts, const float* src_cams, int V, int R,
                    int S, float* out /* [R,S,V,6] */, void* stream);
/* Pooled form (see dyn_project_gather_tbl): src_cams [pool,34]; slot v of ray r is the centre of pool entry
 * view_tbl[camera_index[r], v].  Same checks as dyn_project_gather_tbl. */
int dyn_plucker_src_tbl(const float* pts, const float* src_cams, int pool, int K,
                        const int* camera_index, const int* view_tbl, int V, int R,
                        int S, float* out /* [R,S,V,6] */, void* stream);

/* ---- a8-a11: the two aggregation networks ---------------------------------
 * DynibarDynamic.forward mlp_network.py:236-316 -> raw [R,S,4].
 * ray_dir [R,3] is the NORMALISED target ray direction (render_ray.py:455). */
size_t dyn_net_workspace_bytes(int kind, int R, int S, int V);
int dyn_net_dynamic(dyn_net_t net, const float* pts, const float* rgb_feat,
                    const float* ray_dir, const float* mask, float time, int R,
                    int S, int V, float* raw, void* workspace,
                    size_t workspace_bytes, int precision, void* stream);
/* DynibarStatic.forward mlp_network.py:423-527 -> raw [R,S,4].
 * ref_rays [R,6], src_rays [R,S,V,6] are the Plucker coordinates. */
int dyn_net_static(dyn_net_t net, const float* pts, const float* ref_rays,
                   const float* src_rays, const float* rgb_feat,
                   const float* ray_diff, const float* mask, int R, int S,
                   int V, float* raw, void* workspace, size_t workspace_bytes,
                   int precision, void* stream);

/* ---- fused a4-a11 (DYN_PREC_BF16): Projector.compute_with_motions fused INTO
 * the network evaluation -- the [R,S,V,35] gather output never reaches HBM.
 * Replaces the call pairs at render_ray.py:503-521 + :538-564 (== :715-774,
 * :998-1059).  The source views arrive in two packed per-frame layouts (pack them ONCE per frame):
 *   feat_cl  = channels-last bf16 copy [V,h,w,C] of the feature maps (dyn_featmaps_channels_last):
 *              one bilinear tap of all C = 32 channels is 64 contiguous bytes;
 *   src_rgba = the source images [V,H,W,3] padded to [V,H,W,4] fp32 (dyn_rgbs_rgba): one tap is
 *              one aligned 16-byte load.
 * mask_out [R,S,V] receives the projector mask (needed by dyn_composite).  V <= 16.
 * static:  needs ray_o, ray_d [R,3] (Plucker coordinates are formed inside).
 * dynamic: pts_seq [V,R,S,3] displaced points, ray_dir [R,3] normalised. */
size_t dyn_net_fused_workspace_bytes(int kind, int R, int S, int V);
int dyn_featmaps_channels_last(const float* featmaps, void* out_bf16, int V, int C,
                               int h, int w, void* stream);
int dyn_rgbs_rgba(const float* src_rgbs, float* out_rgba, int V, int H, int W,
                  void* stream);
int dyn_net_static_fused(dyn_net_t net, const float* pts, const float* ray_o,
                         const float* ray_d, const float* query_cam,
                         const float* src_rgba, const float* src_cams,
                         const void* feat_cl, int R, int S, int V, int H,
                         int W, int C, int h, int w, float* raw,
                         float* mask_out, void* workspace,
                         size_t workspace_bytes, void* stream);
/* Multi-camera form of dyn_net_static_fused: query_cams [K,34] and query_idx [R] as for
 * dyn_project_gather_mc (1 <= K <= 16, query_idx non-NULL when K > 1, values trusted to lie in [0, K);
 * K = 1 is dyn_net_static_fused).  Only the view-direction term of ray_diff reads the target camera.
 * Runs on the warpgroup per-view kernel only: with the twin-warp kernel selected
 * (dyn_debug_set_view_kernel(0)) a call with K > 1 fails with DYN_E_INVALID. */
int dyn_net_static_fused_mc(dyn_net_t net, const float* pts, const float* ray_o,
                            const float* ray_d, const float* query_cams, int K,
                            const int* query_idx, const float* src_rgba,
                            const float* src_cams, const void* feat_cl, int R,
                            int S, int V, int H, int W, int C, int h, int w,
                            float* raw, float* mask_out, void* workspace,
                            size_t workspace_bytes, void* stream);
int dyn_net_dynamic_fused(dyn_net_t net, const float* pts, const float* pts_seq,
                          const float* ray_dir, const float* query_cam,
                          const float* src_rgba, const float* src_cams,
                          const void* feat_cl, float time, int R, int S, int V,
                          int H, int W, int C, int h, int w, float* raw,
                          float* mask_out, void* workspace,
                          size_t workspace_bytes, void* stream);
/* Pooled multi-camera forms of the two fused calls (see dyn_project_gather_tbl): src_rgba [pool,H,W,4],
 * src_cams [pool,34] and feat_cl [pool,h,w,C] hold the pool (pool <= 32), view_tbl [K,V] int32 and
 * camera_index [R] map each ray's slots into it, V <= 16.  Every output, per (point, slot) included, equals the
 * single-camera call on that camera's own views, pool[view_tbl[k]], bit for bit.  The dynamic net reads the
 * table only (its target camera does not enter its outputs): query_cam is one camera [34].  Checks as for
 * dyn_project_gather_tbl; warpgroup per-view kernel only (DYN_E_INVALID with the twin-warp kernel selected). */
int dyn_net_static_fused_tbl(dyn_net_t net, const float* pts, const float* ray_o,
                             const float* ray_d, const float* query_cams, int K,
                             const int* camera_index, const int* view_tbl, int pool,
                             const float* src_rgba, const float* src_cams,
                             const void* feat_cl, int R, int S, int V, int H, int W,
                             int C, int h, int w, float* raw, float* mask_out,
                             void* workspace, size_t workspace_bytes, void* stream);
int dyn_net_dynamic_fused_tbl(dyn_net_t net, const float* pts, const float* pts_seq,
                              const float* ray_dir, const float* query_cam, int K,
                              const int* camera_index, const int* view_tbl, int pool,
                              const float* src_rgba, const float* src_cams,
                              const void* feat_cl, float time, int R, int S, int V,
                              int H, int W, int C, int h, int w, float* raw,
                              float* mask_out, void* workspace,
                              size_t workspace_bytes, void* stream);

/* ---- a12: raw2outputs / raw2outputs_vanilla, render_ray.py:134-330 --------
 * raw_* [R,S,4]; z_vals [R,S]; mask_* [R,S,V*] as produced by
 * dyn_project_gather; a sample is "observed" when more than `min_views_*`
 * views see it (1 for the reference-time pass render_ray.py:524-529, 0 for the
 * anchor pass :1198-1200); ray mask = observed samples > 8.
 * out_rays [R,11]: rgb(3) rgb_static(3) rgb_dy(3) depth(1) mask(1, 0/1);
 * out_samples [5,R,S]: alpha_dy, weights_dy, weights_st, alpha, weights. */
int dyn_composite(const float* raw_dy, const float* raw_st,
                  const float* z_vals, const float* mask_dy, int V_dy,
                  int min_views_dy, const float* mask_st, int V_st,
                  int min_views_st, int R, int S, float* out_rays,
                  float* out_samples, void* stream);
/* out_rays [R,5]: rgb(3) depth(1) mask(1); out_samples [2,R,S]: weights, alpha */
int dyn_composite_vanilla(const float* raw, const float* z_vals,
                          const float* mask, int V, int min_views, int R,
                          int S, float* out_rays, float* out_samples,
                          void* stream);

/* ---- a13: sample_pdf + merge, render_ray.py:19-64, :790-819 ---------------
 * z_vals [R,S], weights [R,S] (coarse `weights`); u [R,Ni] uniforms or NULL
 * (det: linspace(0,1,Ni)).  z_out [R,S+Ni] sorted ascending. */
int dyn_resample(const float* z_vals, const float* weights, const float* u,
                 int R, int S, int Ni, int inv_uniform, float* z_out,
                 void* stream);

/* Training of the 2-D encoder (row f2; autograd of ResNet.forward, feature_network.py:302-311 with BasicBlock.forward
 * :68-84).  The train forward keeps every pre-norm convolution output, activation and InstanceNorm statistic in `saved`
 * (dyn_encoder_train_workspace_bytes); the backward ACCUMULATES d(loss)/d(params) into d_params (n_params floats, the
 * order of dyn_encoder_forward's `params`; the caller zeroes it) from d_coarse / d_fine [N,32,H/4,W/4] (either may be
 * NULL).  The images carry no gradient.  Every convolution is differentiated through its im2col form; `precision`
 * DYN_PREC_BF16 runs the two products per convolution on the tensor cores (bf16 operands, fp32 accumulation). */
size_t dyn_encoder_train_workspace_bytes(int N, int H, int W);
size_t dyn_encoder_backward_scratch_bytes(int N, int H, int W);
int dyn_encoder_train_forward(const float* params, size_t n_params, const float* images, int N, int H, int W,
                              float* coarse, float* fine, void* saved, size_t saved_bytes, void* stream);
int dyn_encoder_backward(const float* params, size_t n_params, const float* images, int N, int H, int W,
                         const float* d_coarse, const float* d_fine, void* saved, size_t saved_bytes,
                         void* scratch, size_t scratch_bytes, float* d_params, int precision, void* stream);

/* ---- a14: flow / expected scene flow, render_ray.py:333-358, :585-595 -----
 * weights [R,S]; pts_seq [V,R,S,3] (first n_flow views used); src_cams
 * [V,34]; uv [R,2]; coeff [R,S,3*nb]; basis [T,nb]; sf_k = 2 (mv) or 1 (mono).
 * flows [n_flow,R,2]; exp_sf [R,3].  With n_flow == 0, pts_seq, src_cams and
 * flows may be NULL. */
int dyn_flow_sceneflow(const float* weights, const float* pts_seq,
                       const float* src_cams, const float* uv,
                       const float* coeff, const float* basis, int T, int nb,
                       int frame_idx, int sf_k, int n_flow, int R, int S,
                       float* flows, float* exp_sf, void* stream);

/* ---- f2 (first slice): backward of the two non-MLP ends of the path -------------------------
 * dyn_composite_backward: raw2outputs (render_ray.py:214-330).  g_rays [R,11] = d/d(rgb, rgb_static,
 * rgb_dy, depth, mask(ignored)), g_samples [5,R,S] = d/d(alpha_dy, weights_dy, weights_st, alpha,
 * weights) or NULL -> g_raw_dy, g_raw_st [R,S,4].  S <= 256.
 * dyn_project_gather_backward: compute_with_motions (projection.py:103-176).  g_rgb_feat [R,S,V,3+C]
 * -> g_featmaps [V,C,h,w] (reference layout; zeroed here, atomically accumulated) and / or g_xyz [V,R,S,3]
 * (either may be NULL).  xyz may be NULL (every view uses xyz_st). */
int dyn_composite_backward(const float* raw_dy, const float* raw_st, const float* z_vals,
                           const float* g_rays, const float* g_samples, int R, int S,
                           float* g_raw_dy, float* g_raw_st, void* stream);
int dyn_project_gather_backward(const float* xyz_st, const float* xyz, const float* src_rgbs,
                                const float* src_cams, const float* featmaps,
                                const float* g_rgb_feat, int V, int R, int S, int H, int W,
                                int C, int h, int w, float* g_featmaps, float* g_xyz,
                                void* stream);

/* MotionMLP training slice (ibrnet/mlp_network.py:605-618; gradients as torch.autograd would produce them
 * for MotionMLP.forward).  The forward keeps the embedding and the eight post-ReLU activations in `saved`
 * (dyn_motion_train_workspace_bytes(N) bytes, also scratch for the backward).  The backward ACCUMULATES
 * d(loss)/d(params) into d_params (flat, the n_params floats of dyn_net_create, same layout as the
 * blob given to dyn_net_create; the caller zeroes it) and writes d(loss)/d(xyzt) [N,4] unless d_xyzt is NULL.
 * fp32; split-K float atomics (not bit-reproducible between runs). */
size_t dyn_motion_train_workspace_bytes(int N);
int dyn_motion_mlp_train_forward(dyn_net_t motion, const float* xyzt, int N, float* coeff, void* saved,
                                 size_t saved_bytes, int precision, void* stream);
int dyn_motion_mlp_backward(dyn_net_t motion, const float* xyzt, const float* d_coeff, int N, void* saved,
                            size_t saved_bytes, float* d_params, float* d_xyzt, int precision, void* stream);

/* ---- f2: training step of the two aggregation networks (DynibarDynamic.forward, ibrnet/mlp_network.py:236-316;
 * DynibarStatic.forward, :423-527; gradients as torch.autograd produces them for those modules).
 * The *_train_forward calls are the fp32 forwards of dyn_net_dynamic / dyn_net_static that keep every activation in
 * `saved` (dyn_net_train_workspace_bytes bytes; R rays must fit one internal chunk: R*S*V <= 4 Mi rows).  The
 * backward reads `saved`, uses `scratch` (dyn_net_backward_scratch_bytes), ACCUMULATES d(loss)/d(params) into
 * d_params (flat, layout of the blob given to dyn_net_create; the caller zeroes it) and writes
 * d_rgb_feat [R,S,V,35] (gradient w.r.t. the gathered colours + features; NULL to skip) and, for the dynamic net,
 * d_pts [R,S,3] (through the positional encoding of ref_pts_fc; NULL to skip).  mask / ray_diff / rays / time carry
 * no gradient (the reference detaches them).  `precision`: DYN_PREC_FP32 = SIMT products; DYN_PREC_BF16 = the
 * products of the large layers on the tensor cores (bf16 operands, fp32 accumulation, fp32 master weights / gradients; the
 * net must have been created with layer images, dyn_net_create_ex pack_level >= 1); everything else stays fp32.
 * Float atomics (not bit-reproducible between runs). */
size_t dyn_net_train_workspace_bytes(int kind, int R, int S, int V);
size_t dyn_net_backward_scratch_bytes(int kind, int R, int S, int V);
int dyn_net_dynamic_train_forward(dyn_net_t net, const float* pts, const float* rgb_feat, const float* ray_dir,
                                  const float* mask, float time, int R, int S, int V, float* raw, void* saved,
                                  size_t saved_bytes, int precision, void* stream);
int dyn_net_dynamic_backward(dyn_net_t net, const float* pts, const float* mask, int R, int S, int V,
                             const float* d_raw, void* saved, size_t saved_bytes, void* scratch,
                             size_t scratch_bytes, float* d_params, float* d_rgb_feat, float* d_pts, int precision,
                             void* stream);
int dyn_net_static_train_forward(dyn_net_t net, const float* pts, const float* ref_rays, const float* src_rays,
                                 const float* rgb_feat, const float* ray_diff, const float* mask, int R, int S,
                                 int V, float* raw, void* saved, size_t saved_bytes, int precision, void* stream);
int dyn_net_static_backward(dyn_net_t net, const float* rgb_feat, const float* ray_diff, int R, int S, int V,
                            const float* d_raw, void* saved, size_t saved_bytes, void* scratch,
                            size_t scratch_bytes, float* d_params, float* d_rgb_feat, int precision, void* stream);

/* Smaller pieces of the training step:
 * dyn_composite_vanilla_backward: raw2outputs_vanilla (render_ray.py:134-211).  g_rays [R,5] = d/d(rgb, depth,
 *   mask(ignored)), g_samples [2,R,S] = d/d(weights, alpha) or NULL -> g_raw [R,S,4].  S <= 256.
 * dyn_traj_combine(_backward): compute_traj_pts and the displacements built from it (render_ray.py:361-369,
 *   :462-500, :1101-1176): out[i,p,:] = (base ? base[p,:] : 0) + sum_k coeff[p, axis*nb + k] * D[i,k]; D [n,nb]
 *   (DEVICE; rows = differences of DCT basis rows), coeff [P,3*nb], base [P,3] or NULL, out [n,P,3].  The backward
 *   writes g_coeff [P,3*nb] and / or g_base [P,3] (either may be NULL).
 * dyn_flow_backward: compute_optical_flow (render_ray.py:333-358) -> g_weights [R,S], g_pts_seq [n_flow,R,S,3]
 *   (either may be NULL).  S <= 256.  n_flow == 0 writes a zero g_weights. */
int dyn_composite_vanilla_backward(const float* raw, const float* z_vals, const float* g_rays,
                                   const float* g_samples, int R, int S, float* g_raw, void* stream);
int dyn_traj_combine(const float* coeff, const float* D, const float* base, int n, int nb, int P, float* out,
                     void* stream);
int dyn_traj_combine_backward(const float* g_out, const float* D, int n, int nb, int P, float* g_coeff,
                              float* g_base, void* stream);
int dyn_flow_backward(const float* weights, const float* pts_seq, const float* src_cams, const float* g_flows,
                      int n_flow, int R, int S, float* g_weights, float* g_pts_seq, void* stream);

/* Trainable trajectory basis (trajectory_basis / trajectory_basis_fine, ibrnet/model.py:94-118, :331-351):
 * dyn_traj_combine_grad_d: the gradient of dyn_traj_combine w.r.t. its rows D, g_D[i,k] = sum_p sum_axis
 *   g_out[i,p,axis] * coeff[p, axis*nb + k] -> g_D [n,nb] (DEVICE).  Autograd routes it to the basis rows each D row
 *   was built from (render_ray.py:361-369, :462-500, :1101-1176).  A two-stage reduction over the P points through
 *   `workspace` (dyn_traj_combine_grad_d_workspace_bytes(n, nb, P) bytes) without float atomics: the same inputs
 *   always give the same bits.  nb <= 8.
 * dyn_expected_scene_flow(_backward): exp_sf (render_ray.py:585-595, the mv fine pass, differentiable there):
 *   sf [2,R,S,3] = (traj(f+k) - traj(f), traj(f-k) - traj(f)), weights [R,S] -> exp_sf [R,3] =
 *   max(sum_s w*sf[0], sum_s w*sf[1]) per axis.  The backward writes g_weights [R,S] and / or g_sf [2,R,S,3] (either
 *   may be NULL); at a tie each side takes half of the gradient, as torch.max(p, m) does. */
size_t dyn_traj_combine_grad_d_workspace_bytes(int n, int nb, int P);
int dyn_traj_combine_grad_d(const float* g_out, const float* coeff, int n, int nb, int P, float* g_D, void* workspace,
                            size_t workspace_bytes, void* stream);
int dyn_expected_scene_flow(const float* weights, const float* sf, int R, int S, float* exp_sf, void* stream);
int dyn_expected_scene_flow_backward(const float* weights, const float* sf, const float* g_exp_sf, int R, int S,
                                     float* g_weights, float* g_sf, void* stream);

/* ---- f2: the monocular training criterion (train.py:187-196 and :300-456, ibrnet/criterion.py, utils.py:32-39) ----
 * Every loss term of a DynibarMono step in one forward and one backward call (csrc/loss.cu).  A term is a bit of
 * `terms` and an entry of `w`; a cleared bit is an absent term (its pointers may be NULL, it contributes 0 and its
 * inputs get no gradient).  Term k, its component c_k = numerator / denominator, and what enters the loss:
 *    0..5  Charbonnier of rgb slot k: sum_r m_r sum_c sqrt((pred - gt)^2 + 1e-6) / (3 sum_r m_r + rgb_eps[k]);
 *          m_r = mask (bytes, 0 / non-0) * w0 (or 1 - w0 with flag 1) * w1 [* (1 - weights_ratio), flag 2],
 *          each factor optional.  rgb_eps: 1e-6 for utils.img2charbonier, 1e-8 for compute_temporal_rgb_loss.
 *          Slots 0-4 add up to rgb_loss (train.py:304-328), slot 5 is the static loss (:426-434, :187-196).
 *    6     disparity :331-342: sum |1 / max(depth, 1e-2) - gt_disp| mask / (sum mask + 1e-8)
 *    7     flow :345-351, criterion.py:83-85: L1 over [n_flow,R,2] under ray mask * flow_masks [n_flow,R]
 *    8     trajectory cycle :359-371 over traj_ref / traj_anchor [K,R,S,3] weighted by occ_weights [R,S]
 *    9-11  scene-flow regularisers :376-397 over sf_seq [n_sf,R,S,3]: mean |x|, mean (x[v] - x[v+1])^2 (give
 *          w = w_reg / 2), mean |x[:, s+1] - x[:, s]|
 *    12    entropy :400-413 of weights_ratio = sum_s weights_dy / max(sum_s weights_dy + sum_s weights_st, 1e-9)
 *    13    distortion :416-423 on dist_w [R, dist_n] (rows dist_ld floats apart) with mid-points and intervals
 *          either given (dist_m, dist_interval [R, dist_n]) or formed from s_vals [R, dist_n + 1]
 *    14    :437-445 sum |sum_s weights_dy * m2| / sum (m2 + 1e-8), m2 = m of slot 5 where weights_ratio < 0.1;
 *          joins slot 5 in static_loss
 * loss = sum_k w[k] c_k.  `out` receives DYN_LOSS_OUT_FLOATS floats: [0..8] loss, flow_loss, disp_loss, rgb_loss,
 * distortion_loss, entropy_loss, static_loss, cycle_loss, reg_loss (the weighted sums train.py:447-464 logs);
 * [9 + k] c_k; [24 + k] w[k] / denominator_k, the table the backward reads.
 * Two launches: one warp per ray writes a block's partial sums into `workspace`
 * (dyn_mono_loss_workspace_bytes(R) bytes), one block then adds them in block order.  No float atomics: the same
 * inputs give the same bits.  S >= 2; with term 9-11 n_sf >= 2; with term 13 dist_n <= 256.
 * The two passes as separate calls, for a batch evaluated in ray slices: dyn_mono_loss_rows runs pass 1 over one
 * slice (`in` holds the slice: in.R is its ray count and the stride of its [n, R, ...] inputs, which are contiguous
 * slices) and writes its cdiv(in.R, 8) rows of 2 * DYN_LOSS_TERMS floats at row `first_block` of `partial`, a
 * batch-wide buffer of dyn_mono_loss_workspace_bytes(R_batch) bytes; a slice starts on a multiple of 8 rays
 * (first_block = first ray / 8) and only the batch's last slice may hold a count that is not a multiple of 8.
 * dyn_mono_loss_finish runs pass 2 once with the batch's R, S, K, n_sf (nblocks = cdiv(R, 8)); the REG, entropy and
 * distortion denominators use that R.  Rows plus finish give the bits dyn_mono_loss gives on the whole batch.  The
 * backward of a slice is dyn_mono_loss_backward on the slice's inputs with the batch's `out`.
 * dyn_mono_loss_backward: `g_loss` is the DEVICE address of d/d loss, `out` the forward's output.  Every non-NULL
 * pointer of `grads` is written exactly once per element in one launch (no zero-fill needed): rgb[k] [R,3],
 * depth [R], flows [n_flow,R,2], weights [R,dist_ld] (columns >= dist_n get 0), weights_dy / weights_st [R,S],
 * traj_ref / traj_anchor [K,R,S,3], sf_seq [n_sf,R,S,3].  The (1 - weights_ratio) factor and m2 carry no gradient
 * (detached in the reference).  Both structs are HOST structs read before the call returns. */
#define DYN_LOSS_RGB_SLOTS 6
#define DYN_LOSS_TERMS 15
#define DYN_LOSS_OUT_FLOATS 40
#define DYN_LOSS_SLOT_COMPLEMENT_W0 1
#define DYN_LOSS_SLOT_TIMES_ONE_MINUS_RATIO 2
typedef struct {
  const float* pred; /* [R,3], rows `ld` floats apart */
  const uint8_t* mask; /* [R] or NULL */
  const float* w0;   /* [R] or NULL */
  const float* w1;   /* [R] or NULL */
  int ld;
  int flags;
} dyn_loss_rgb_slot;
typedef struct {
  dyn_loss_rgb_slot rgb[DYN_LOSS_RGB_SLOTS];
  const float* gt_rgb; /* [R,3] */
  const float* depth;  /* [R], elements depth_ld floats apart */
  const float* gt_disp;
  const uint8_t* ray_mask; /* [R] or NULL: the mask of terms 6 and 7 */
  const float* flows;
  const float* gt_flows;
  const float* flow_masks;
  const float* traj_ref;
  const float* traj_anchor;
  const float* occ_weights;
  const float* sf_seq;
  const float* weights_dy;
  const float* weights_st;
  const float* dist_w;
  const float* s_vals;
  const float* dist_m;
  const float* dist_interval;
  int R, S, depth_ld, n_flow, K, n_sf, dist_ld, dist_n;
} dyn_mono_loss_inputs;
typedef struct {
  unsigned terms;
  float w[DYN_LOSS_TERMS];
  float rgb_eps[DYN_LOSS_RGB_SLOTS];
} dyn_mono_loss_weights;
typedef struct {
  float* rgb[DYN_LOSS_RGB_SLOTS];
  float* depth;
  float* flows;
  float* weights;
  float* weights_dy;
  float* weights_st;
  float* traj_ref;
  float* traj_anchor;
  float* sf_seq;
} dyn_mono_loss_grads;
size_t dyn_mono_loss_workspace_bytes(int R);
int dyn_mono_loss(const dyn_mono_loss_inputs* in_host, const dyn_mono_loss_weights* weights_host, float* out,
                  void* workspace, size_t workspace_bytes, void* stream);
int dyn_mono_loss_backward(const dyn_mono_loss_inputs* in_host, const dyn_mono_loss_weights* weights_host,
                           const float* out, const float* g_loss, const dyn_mono_loss_grads* grads_host,
                           void* stream);
int dyn_mono_loss_rows(const dyn_mono_loss_inputs* in_host, const dyn_mono_loss_weights* weights_host, float* partial,
                       int first_block, void* stream);
int dyn_mono_loss_finish(const float* partial, int nblocks, const dyn_mono_loss_weights* weights_host, int R, int S,
                         int K, int n_sf, float* out, void* stream);

/* Unit-test hooks of the tensor-core training products (csrc/train_tc.cu; bf16 operands, fp32 accumulation):
 * dyn_debug_tc_grad_w: dW[out,width] += dz[rows,out]^T (x[rows,width] * kscale[rows] or 1); out, width <= 256.
 * dyn_debug_tc_grad_in: din[rows,width] = dz[rows,out] W[out, 0:width] (W row-major with ldw columns). */
int dyn_debug_tc_grad_w(const float* dz, int lddz, int out, int rows, const float* x, int ldx, int width,
                        const float* kscale, float* dW, int ldw, void* stream);
int dyn_debug_tc_grad_in(const float* dz, int lddz, int out, int rows, const float* W, int ldw, int width,
                         float* din, int ldd, void* scratch, size_t scratch_bytes, void* stream);
size_t dyn_debug_tc_grad_in_scratch_bytes(void);

/* ---- f1: 2-D feature encoder, ResNet.forward as the reference runs it (feature_network.py:302-311) ----
 * conv 7x7 stride 2 (reflect) -> InstanceNorm -> ReLU -> layer1 (3 BasicBlocks, the first with stride 2)
 * -> 1x1 conv -> coarse (channels 0..31) | fine (channels 32..63).  images [N,3,H,W] fp32;
 * coarse, fine [N,32,H/4,W/4].  `params` = the executed parameters in state_dict order
 * (dynibar_b200/feature_network.py: _EXECUTED), dyn_encoder_param_count() floats. */
size_t dyn_encoder_param_count(void);
size_t dyn_encoder_workspace_bytes(int N, int H, int W);
int dyn_encoder_forward(const float* params, size_t n_params, const float* images,
                        int N, int H, int W, float* coarse, float* fine,
                        void* workspace, size_t workspace_bytes, void* stream);

/* ---- unit-test hook: the fused per-point stage (geometry_fc -> ray transformer
 * -> heads; mlp_network.py:283-315 / :496-506) on caller-provided pooled
 * features G [R*S, 272] (257 used) and nvalid [R*S].  Outputs g2 [R*S,128] (plain
 * fp32 rows); Q, K, V, O [R*S,128]: the bf16 values the kernels exchanged, as fp32 rows
 * (each may be NULL: not written; when S divides 128 and all five are NULL, the product
 * kernel runs instead of its capturing twin); dynamic net: out_a = raw [R*S,4]; static net:
 * out_a = per-point part of rgb_fc.0 [R*S,128], out_b = masked sigma [R*S].
 * posenc_ws: S*128 floats of scratch. */
int dyn_debug_point_chain(dyn_net_t net, const float* G, const float* nvalid,
                          const float* pts, const float* ray_dir, int R, int S,
                          float* g2, float* Q, float* K, float* V, float* O,
                          float* out_a, float* out_b, float* posenc_ws,
                          void* stream);
/* unit-test hook: the fused path's ray-transformer attention (the kernel the product picks for S) on
 * caller-provided Q, K, V [R*S,128] fp32 rows, which are rounded to bf16 as the kernels read them, and
 * nvalid [R*S] -> O [R*S,128] (bf16 values as fp32).  S the kernels cannot run fails with DYN_E_INVALID. */
int dyn_debug_attention(const float* Q, const float* K, const float* V, const float* nvalid,
                        int R, int S, float* O, void* stream);
/* unit-test hook: the static net's per-view blending head and masked softmax over views on rows in the
 * layout dyn_debug_set_view_capture produces: X [P,V,128] (rounded to bf16), vis2, mask_eff [P,V],
 * ray_diff [P,V,4], rgb_in [P,V,3], GW [P,128] (per-point part of rgb_fc.0, bias included), sigma [P]
 * -> raw [P,4] = blended rgb | sigma.  V <= 16. */
int dyn_debug_rgb_head(dyn_net_t net, const float* X, const float* vis2, const float* ray_diff,
                       const float* mask_eff, const float* rgb_in, const float* GW,
                       const float* sigma, long long P, int V, float* raw, void* stream);

/* ---- unit-test hook (HOST only, no GPU needed): pack one nn.Linear [N, Kw] into the bf16
 * wgmma weight image the fused kernels stream (dynibar_b200/csrc/fused_engine.cuh:
 * append_layer).  colmap[Kpad] maps operand column -> weight column, -1 = zero,
 * -2 / -3 = hi / lo bf16 halves of the folded bias; `scale` multiplies weights and
 * bias.  The outputs are packed in N-blocks of nb = min(64, Npad - n0) rows, each cut
 * along K into chunks of at most min(8, stage_bytes / (nb*32)) k-steps of 16;
 * element (n, k) of a chunk that starts at (n0, k0) sits at byte
 * ((k-k0)/8)*(nb*16) + ((n-n0)/8)*128 + ((n-n0)%8)*16 + ((k-k0)%8)*2 of that chunk.
 * Writes the image into out_img (out_bytes capacity), its size into *img_bytes and the
 * number of chunks into *nchunks. */
int dyn_debug_pack_layer(const float* W, const float* bias, int N, int Kw, int Npad,
                         int Kpad, const int* colmap, float scale, int stage_bytes,
                         void* out_img, size_t out_bytes, size_t* img_bytes,
                         int* nchunks);
/* byte offset of (row, 8-column group) in a bf16 tile image with `kgroups` groups per
 * 128-row tile: the layout activations use between the fused kernels. */
size_t dyn_debug_tile_image_off(long long row, int kgroup, int kgroups);

/* comparison hook: which kernel runs the fused per-view stage: 4 = warpgroup kernel (csrc/view_wg.cu:
 * accumulators in registers, two 64-row warpgroups per CTA; the default), 0 = twin-warp kernel
 * (csrc/view_twin.cu: one tile per CTA); -1 = the default.  1 - 3 selected the quad-schedule and the
 * sub-round pipelined twin kernels, which have been removed: with them the fused per-view stage fails
 * with DYN_E_INVALID. */
void dyn_debug_set_view_kernel(int which);

/* profiling hook: when set, block 0 of each fused per-view kernel launch writes clock64() data into
 * dev_buf (zeroed, >= 1232 int64): the static net's launches into [0, 616), the dynamic net's into
 * [616, 1232); a later launch of the same net overwrites an earlier one.  Within a net's part:
 *   warpgroup kernel: per warpgroup w (0, 1: consumers, 2: front end), 32 counters at [32 w, 32 w + 32):
 *     the cycles of every phase accumulated over all of block 0's iterations (index = enum Phase in
 *     csrc/view_wg.cu: front end, named-barrier waits, weight-ring waits, each layer's issue-to-finish and
 *     each epilogue, second pooling and outputs, waits at the front-end handoff), [32 w + 30] its
 *     iterations, [32 w + 31] its lifetime;
 *   twin-warp kernel: timestamps [2 twins][64] and the MMA warpgroup's totals from index 128.
 * tools/view_phases.py prints the warpgroup kernel's counters as shares of the lifetime. */
void dyn_debug_set_view_timestamps(long long* dev_buf);

/* unit-test hook: while any pointer is set, every dyn_net_static_fused / dyn_net_dynamic_fused call copies the
 * outputs of the fused per-view stage (the kernel dyn_debug_set_view_kernel selects) into these DEVICE buffers,
 * chunk by chunk at the chunk's row offset, before the per-point stage runs on them (P = R*S points, V views):
 *   G [P, 272]: pooled mean 0..127 | variance 128..255 | mean pooling weight 256 | 0 | bias columns 264, 265 = 1
 *     (fp32 copy of the bf16 operand of geometry_fc);  nvalid [P]: valid views per point;
 *   static net only: X [P, V, 128] per-view features after the visibility residual (bf16 values as fp32),
 *     vis2 [P, V], mask_eff [P, V] (projector mask after the mask_rgb test), ray_diff [P, V, 4], rgb_in [P, V, 3].
 * Any pointer may be NULL (not captured); all NULL turns the hook off. */
void dyn_debug_set_view_capture(float* G, float* nvalid, float* X, float* vis2, float* mask_eff,
                                float* ray_diff, float* rgb_in);

/* ---- building block: one nn.Linear on the tensor cores -----------------------
 * Y[M,N] = act(X[M,K] W[N,K]^T + b) with bf16 operands / fp32 accumulation
 * (wgmma).  act: 0 none, 1 ELU, 2 ReLU, 3 sigmoid.  N <= 256.  packed_ws must
 * hold dyn_linear_tc_packed_bytes(N, K) bytes (bf16 wgmma image of W).  This is
 * the kernel behind every nn.Linear of mlp_network.py in DYN_PREC_BF16 mode;
 * exported for unit testing. */
size_t dyn_linear_tc_packed_bytes(int N, int K);
int dyn_linear_tc(const float* X, int ldx, const float* W, const float* b, int M,
                  int N, int K, int act, float* Y, int ldy, void* packed_ws,
                  size_t packed_ws_bytes, void* stream);

/* ---- virtual source views of a monocular frame (render_source_vv.py; offline data preparation) --------------
 * Deterministic softmax forward splatting: every source pixel adds value * bilinear weight to the four target pixels
 * around (x + flow_x, y + flow_y) (NW corner floor(.), a corner outside the image is dropped on its own), and the
 * output is sum(value e w) / (sum(e w) + 1e-7) with e = exp(metric).  No float atomics: sources are grouped by cell
 * with a stable sort and summed in a fixed order, so the same inputs give the same bits.  B items, C channels. */
/* workspace of dyn_splat_softmax / dyn_forward_splat for B items of H x W; 0 for an unsupported shape */
size_t dyn_splat_workspace_bytes(int B, int H, int W);
/* splatting_function('softmax', frame, flow, metric) (the external `splatting` extension, render_source_vv.py:58):
 * frame [B,C,H,W], flow [B,2,H,W], metric [B,1,H,W] -> out [B,C,H,W].  C <= 8. */
int dyn_splat_softmax(const float* frame, const float* flow, const float* metric, int B, int C, int H, int W,
                      float* out, void* workspace, size_t workspace_bytes, void* stream);
/* render_forward_splat (render_source_vv.py:15): imgs [B,H,W,C], depths [B,H,W], cams [B,30] = K_src^-1 | R | t |
 * K_dst (row-major, fp32).  Each pixel goes to p = K_dst (R (d K_src^-1 [x,y,1]^T) + t), weighted by
 * exp((imp - min) / (max - min + 1e-6) * 20 - 10), imp = 1 / p_z, min / max per item.
 * out [B,C+1,H,W] = splatted image channels | splatted 1 / p_z.  C <= 7. */
int dyn_forward_splat(const float* imgs, const float* depths, const float* cams, int B, int C, int H, int W, float* out,
                      void* workspace, size_t workspace_bytes, void* stream);
/* sobel_fg_alpha (render_source_vv.py:118): x [N,H,W] -> alpha [N,H,W] = exp(-beta sqrt(gx^2 + gy^2)), unnormalised
 * 3x3 Sobel with the border replicated. */
int dyn_sobel_alpha(const float* x, int N, int H, int W, float beta, float* alpha, void* stream);
/* One frame's V virtual source views (render_source_vv.py:283-330): img [H,W,3] in [0,1], disp [H,W], cams [V,30]
 * (as dyn_forward_splat, K_src = K_dst) -> out [V,H,W,3] uint8.  rgba = [img * 255, sobel alpha of (1/disp)/10 with
 * beta 0.5] is splatted from depth 1/disp; rgb = clip(F_rgb / 255, 0, 1), mask = F_a > 0.5 eroded by the 3x3 cross
 * (edge replicated), out = uint8(255 rgb mask), truncating. */
size_t dyn_virtual_views_workspace_bytes(int V, int H, int W);
int dyn_virtual_views(const float* img, const float* disp, const float* cams, int V, int H, int W, uint8_t* out,
                      void* workspace, size_t workspace_bytes, void* stream);

/* ---- scores of rendered views (eval_nvidia.py:201-247, :380-457; DESIGN §3.6) ---------------------------------------
 * pred, gt (and mask) [K,H,W,3] fp32, channels-last, contiguous; H, W >= 7.  SSIM is skimage 0.19.3
 * structural_similarity(multichannel=True, full=True) on float32: 7x7 uniform window, 'reflect' border, sample
 * covariance, data_range 2.  For each mask row m: den = sum(w_m) + 1e-8 over all H*W*3 elements,
 * PSNR = 10 log10(den / sum((pred - gt)^2 w_m)) in fp64 (0 when that sum is 0), SSIM = sum(S w_m) / den.
 * scores [K,M,2] fp64 = (PSNR, SSIM) per image and row.
 *   DYN_SCORES_PLAIN  M = 1: the given images, w_0 = mask (1 where mask is NULL).
 *   DYN_SCORES_EVAL   eval_nvidia.py's scoring of a camera: valid = ((r + g) + b) > 1e-3f on pred (float32), both
 *                     images multiplied by valid, rows w = valid, mask, 1 - mask (M = 3), or valid alone (M = 1) when
 *                     mask is NULL.
 * ssim_map [K,H,W,3] fp32 receives S when not NULL.  Two launches, no float atomics: the same inputs give the same
 * bits, and an image's scores do not depend on K or the other images. */
#define DYN_SCORES_PLAIN 0
#define DYN_SCORES_EVAL 1
/* workspace of dyn_image_scores for K images of H x W; 0 for an unsupported shape */
size_t dyn_image_scores_workspace_bytes(int K, int H, int W);
int dyn_image_scores(const float* pred, const float* gt, const float* mask, int K, int H, int W, int mode,
                     double* scores, float* ssim_map, void* workspace, size_t workspace_bytes, void* stream);

/* ---- a monocular training scene resident on the device (DESIGN §3.7; csrc/scene.cu) --------------------------------
 * MonocularDataset.__getitem__ (ibrnet/data_loaders/monocular.py:146-426) and RaySamplerSingleImage.random_sample
 * (ibrnet/sample_ray.py:262-331) on a scene uploaded once.  Float values are the reference's float32 expressions,
 * rounded as numpy rounds them: u8 / 255.0f, 1 - x, the masked view's product.  No float atomics, no host
 * synchronisation: the same inputs give the same bits. */
typedef struct {
  const uint8_t* frames;     /* [N,H,W,3] images_WxH */
  const uint8_t* vviews;     /* [N,8,H,W,3] source_virtual_views_WxH */
  const uint8_t* srcmask;    /* [N,H,W,mc] nearest-resized dynamic masks, raw values (load_src_view's mask) */
  const uint8_t* motion;     /* [N,H,W] {0,1} */
  const uint8_t* stat;       /* [N,H,W] {0,1} */
  const float* disp;         /* [N,H,W] disparity / float32(scale) */
  const float* flows;        /* [NF,6,H,W,2]: frame flow_base + i, offsets 1, 2, 3, -1, -2, -3 */
  const uint8_t* flow_masks; /* [NF,6,H,W] {0,1} */
  int N, H, W, mc, flow_base, NF;
} dyn_scene_t;
/* workspace of dyn_scene_masks: the eroded masks at eh x ew */
size_t dyn_scene_masks_workspace_bytes(int N, int eh, int ew);
/* Masks of N frames (monocular.py:131-142, :164-204): dyn [N,mh,mw,mc] uint8 (mc 1 or 3; channel 0 is the motion
 * mask's), st [N,sh,sw] uint8.  cv2 INTER_NEAREST resizes (src index min(floor(x (1 / (dst / src))), src - 1) in
 * double).  motion [N,H,W] = nearest (H, W) of the erosion by disk(radius) (scipy grey_erosion, mode 'reflect') of
 * (1 - dyn / 255 > 1e-3) at its nearest (eh, ew) (eh = 288, ew = round(288 W / H)); stat [N,H,W] = 1 - st / 255 >
 * 1e-3 at its nearest (H, W); srcmask [N,H,W,mc] = dyn at its nearest (H, W).  radius <= 16.  Two launches. */
int dyn_scene_masks(const uint8_t* dyn, int mh, int mw, int mc, const uint8_t* st, int sh, int sw, int N, int H, int W,
                    int eh, int ew, int radius, uint8_t* motion, uint8_t* stat, uint8_t* srcmask, void* workspace,
                    size_t workspace_bytes, void* stream);
/* One step's source-view stacks and target frame, one launch.  table (device, 16-byte aligned) int32 [(V + 1) * 4]:
 * rows 0..V-1 = (frame, virtual view 0..7 or -1 for the frame itself, masked, stack << 8 | slot) with stack 0 src,
 * 1 anchor, 2 static; row V = (target frame, -, -, -).  A masked view is multiplied by its frame's srcmask / 255
 * (a 1-channel mask broadcasts over the 3 channels).  Stacks [n_*,H,W,3] fp32; rgb [H,W,3], disp / motion_mask /
 * static_mask [H,W], flows [6,H,W,2], masks [6,H,W] fp32 of the target frame. */
int dyn_scene_views(const dyn_scene_t* scene, const int* table, int V, float* src_rgbs, int n_src,
                    float* anchor_src_rgbs, int n_anchor, float* static_src_rgbs, int n_static, float* rgb, float* disp,
                    float* motion_mask, float* static_mask, float* flows, float* masks, void* stream);
/* R rays of the target frame *target (device int), one thread per ray: pixel sel[i] (device int32 [R]; NULL: pixel i,
 * R = H W).  cam (device) fp32 [12] = M (3x3 row-major) | t with M = R_c2w K^-1 formed on the host in float32:
 * ray_d = (M0 u + M1 v) + M2 per row, ray_o = t, uv_grid = (u, v).  With rgb != NULL also rgb [R,3], disp /
 * motion_mask / static_mask [R], flows [6,R,2], masks [6,R,1] at the selected pixels. */
int dyn_scene_rays(const dyn_scene_t* scene, const float* cam, const int* target, const int* sel, int R, float* ray_o,
                   float* ray_d, float* uv_grid, float* rgb, float* disp, float* motion_mask, float* static_mask,
                   float* flows, float* masks, void* stream);
/* The source-view pools of a bullet-time group (DESIGN §3.9), one launch: dyn_scene_views's view rows without its
 * target row.  table (device, 16-byte aligned) int32 [V * 4], rows (frame, virtual view 0..7 or -1, masked,
 * stack << 8 | slot) with stack 0 -> src_rgbs [n_src,H,W,3] and stack 2 -> static_src_rgbs [n_static,H,W,3] fp32.
 * Only frames and vviews are read (srcmask for masked rows); a virtual-view row's frame names one [8,H,W,3] set of
 * vviews, which may hold fewer sets than there are frames (the caller's table stays in range). */
int dyn_scene_pools(const dyn_scene_t* scene, const int* table, int V, float* src_rgbs, int n_src,
                    float* static_src_rgbs, int n_static, void* stream);

/* ---- an Nvidia-benchmark scene resident on the device (DESIGN §3.8; csrc/nvi_scene.cu) -----------------------------
 * eval_nvidia.py's DynamicVideoDataset.__getitem__ (:71-198) and its ground-truth / mask reads (:383-428) on a scene
 * uploaded once.  No float atomics, no host synchronisation: the same inputs give the same bits. */
/* cv2.resize(INTER_AREA) of N uint8 images src [N,sh,sw,C] -> dst [N,dh,dw,C], C 1..4, downscaling only (sh >= dh,
 * sw >= dw).  Integer factors in both axes: the integer box sum s of a = fy fx pixels, (s + 2) >> 2 at 2 x 2, else
 * s * (1.f / a) in float32 rounded to nearest even.  Any other factor: OpenCV's area tables in double (alpha as
 * float32, slivers <= 1e-3 dropped), horizontal then vertical weights in table order, float32 products and sums
 * without contraction, rounded to nearest even.  One launch, one 32 x 8 output tile per CTA. */
int dyn_area_resize(const uint8_t* src, int N, int sh, int sw, int C, int dh, int dw, uint8_t* dst, void* stream);
/* cv2.resize(INTER_NEAREST) of N uint8 images [N,sh,sw,C] -> [N,dh,dw,C] (resizeNN's index rule, dyn_scene_masks);
 * threshold != 0 writes (value > 0) as 0 / 1, which equals thresholding at > 1e-3 before the resize. */
int dyn_nearest_resize(const uint8_t* src, int N, int sh, int sw, int C, int dh, int dw, int threshold, uint8_t* dst,
                       void* stream);
typedef struct {
  const uint8_t* frames; /* [N,H,W,3] images_WxH */
  const uint8_t* smask;  /* [N,H,W] coarse static masks at frame size, raw values (255 where none applies) */
  const uint8_t* gt;     /* [T*S,H,W,3] ground truth resized to the render size */
  const uint8_t* dmask;  /* [T*S,H,W,3] dynamic masks at the render size, 0 / 1, BGR channel order */
  int N, H, W, T, S;
} dyn_nvi_scene_t;
/* One time step, one launch.  table (device) int32 [nd + ns + K]: nd dynamic source frames, ns static source frames,
 * K ground-truth rows (t * S + s).  Writes src_rgbs [nd,H,W,3], static_src_rgbs [ns,H,W,3] as u8 / 255.0f,
 * static_src_masks [ns,H,W] = smask / 255.0f, static_masked [ns,H,W,3] = static_src_rgbs * mask (__fmul_rn),
 * gt [K,H,W,3] = u8 / 255.0f and dynamic_mask [K,H,W,3] (0 / 1), all fp32. */
int dyn_nvi_time_step(const dyn_nvi_scene_t* scene, const int* table, int nd, int ns, int K, float* src_rgbs,
                      float* static_src_rgbs, float* static_src_masks, float* static_masked, float* gt,
                      float* dynamic_mask, void* stream);
/* Every pixel's ray of K <= 16 target cameras of H x W, one launch: cams (device) fp32 [K,12] = M | t per camera
 * (dyn_scene_rays); ray k H W + p is camera k's pixel p: ray_o, ray_d [K H W,3], uv_grid [K H W,2],
 * camera_index int32 [K H W] = k. */
int dyn_nvi_rays(const float* cams, int K, int H, int W, float* ray_o, float* ray_d, float* uv_grid, int* camera_index,
                 void* stream);

/* ---- a monocular bullet-time sweep from a device-resident scene (DESIGN §3.9; csrc/bt_scene.cu) -------------------
 * render_monocular_bt.py's loader on a scene uploaded once: dyn_nearest_resize (masks), dyn_scene_pools (pools),
 * dyn_nvi_rays (rays), and the output frames below. */
/* rgb [K,H,W,3] fp32 -> out [K,H-2 crop_h,W-2 crop_w,3] uint8 = (255 * clip(x, 0, 1)).astype(np.uint8) of the
 * cropped window (:346-354): a float32 product without contraction, truncated toward zero.  One launch. */
int dyn_bt_frames(const float* rgb, int K, int H, int W, int crop_h, int crop_w, uint8_t* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DYNIBAR_B200_H_ */
