"""One fine-stage training step of render_rays_mv (DynibarFF) against its float64 reference (tests/train_mv_step_ref.py),
on the device.

The library runs the step as tools/train_mv_bench.py does: render_rays_mv with the fine stage trainable (its coarse
pass and resampling under no_grad, the differentiable fine pass render_ray._render_mv_train), a stand-in loss
(train_mv_step_ref.stand_in_loss, fp32), backward, with fine_featmaps[0] / [2] and trajectory_basis_fine as leaves.
The reference is the oracle's render_rays_mv in float64 at the library's fine depths, with the library's nets swapped in
(mode "kernel" for precision bf16, "exact" for fp32).  Compared, per tensor, as relative L2 error and max |error| /
max |reference|: the loss, every fine output (the masks bit for bit), and the gradient of every parameter of
net_fine_dy, net_fine_st (`s` included) and motion_mlp_fine, of trajectory_basis_fine and of fine_featmaps[0] / [2].
A tensor that is exactly zero in the reference -- the MotionMLP trunk's gradients behind a zero coeff_linear, the basis
gradient when every coefficient is 0, the basis rows the step does not read -- must be exactly zero.  The library's
fine depths are checked separately against geometry_stage_ref's float64 resampling of the library's own coarse weights
and depths, at that file's bars; the coarse outputs are compared with the reference's coarse pass for information
only (the fused forward kernels, which mode "kernel" does not model).

Cases (train_mv_step_ref.CASES):
  nvidia  the Nvidia configs' step: 1024 rays, 288x512 frames, 7 + 11 views, 64 + 64 samples, inv_uniform,
          anti_alias_pooling 1, random u: 1 441 792 static and 917 504 dynamic (point, view) rows per net call, every
          product on the tensor cores in bf16, split-K dW slabs and the 11-view group sums at training size
  linear  1031 rays, linear depths, deterministic u, anti_alias_pooling 0, mask_rgb 1
  fresh   256 rays, coeff_linear zero and the DCT basis, as the reference initialises them: motion exactly 0, exp_sf
          ties on every ray and its half-split gradient is what reaches coeff_linear
  edges   105 rays on 48x64 frames, reference frame 1 (basis rows wrap), rays no static view sees, samples with fewer
          than 2 valid dynamic views; per-ray products in SIMT
  short   3 + 2 samples: fine S = 5, round(0.5) = 0, so the coefficients of every sample are zeroed
  sliced  nvidia rendered by the library in slices of 400, 400 and 224 rays

BARS: per precision and tensor, 2x the worst value measured over this file's cases on an H100 80GB HBM3 (700 W power
limit), rounded up to one digit, at least 1e-5 (fp32) / 1e-4 (bf16); the comment beside each bar records the measured
worst relative L2 error, the worst max-abs ratio and their cases.  The masks are equal bit for bit and every
exactly-zero reference tensor is exactly zero in the library in every case; the fine depths of every case lie within
the resampling bars.  bf16: outputs 2e-5 - 1.5e-3 (weights_st), the nets' trunks and per-view layers 1e-4 - 1.4e-3,
the MotionMLP 1e-5 - 9e-4, the feature maps 1e-3 - 1.4e-3, trajectory_basis_fine 1e-5, the static blending head up to
2.5e-2 (rgb_fc.4.weight, short) and `s` 5e-2 (short: anti-aliasing weights of 5 samples, as ill-conditioned as in
tests/test_train_gpu.py).  fp32: 1e-7 - 5e-5, `s` 2.8e-3 (nvidia).  The coarse outputs (no bar) are 1e-4 - 2e-3 from the
reference's coarse pass in bf16 and 1e-6 - 8e-6 in fp32.

Measured per case (library step, then the reference; wall time incl. host work, peak device memory allocated):
  nvidia / sliced bf16   library 0.3 - 0.7 s / 24.0 - 26.6 GB, reference 1.2 - 2.2 s / 16.7 - 19.5 GB (128-ray chunks)
  nvidia fp32            library 0.5 s / 26.7 GB, reference 1.0 s / 19.3 GB
  linear bf16            library 0.3 - 0.4 s / 26.9 GB, reference 1.2 s / 19.4 GB (8 chunks of 128 - 129 rays)
  fresh bf16 / fp32      library 0.2 - 0.3 s / 15.3 GB, reference 0.4 s / 19.5 GB (2 chunks)
  edges bf16 / fp32      library 0.1 - 0.2 s / 13.0 GB, reference 0.2 - 0.3 s / 17.9 GB (one chunk)
  short bf16             library 0.1 s / 11.4 GB, reference 0.2 s / 11.5 GB
(the library's peaks include the tensors earlier cases of the same process left in torch's allocator.)

PLANTS: each fine-pass wiring error of train_mv_step_ref.PLANTS, planted in the float64 reference on edges, moves some
compared tensor by at least PLANT_MARGIN times its bf16 bar; the test prints every margin.  Measured: exp_sf_rows_1
4188x (exp_sf), exp_sf_min 4531x (exp_sf), fine_rows_coarse_basis 10000x (fine_dy mask), keep_coarse_S 54x
(motion_mlp_fine.pts_linears.5.weight), static_feat_dy_map 3118x (fine_featmaps[0]), flows_from_undisplaced 9012x
(coeff_linear.weight), fine_time_zero 35921x (net_fine_dy.out_geometry_fc.2.bias).

Library mutations, each built once and run against these bars: the basis-row gradient dropping its last partial
1024-point block fails linear (72x, trajectory_basis_fine; nvidia, fresh and sliced have no partial block, and on edges
and short the last block's rays carry no gradient); the expected scene flow's backward giving the full gradient to both
sides of a tie fails fresh (3.0x, coeff_linear.weight; elsewhere no ray ties); the flow backward skipping its last view
fails every case but short (3.3x - 8600x).  At the parent's _keep_mask (no sample zeroed when round(0.1 S) is 0) short
fails at 12000x its bar and with non-zero MotionMLP gradients.
"""

import time

import pytest
import torch

import geometry_stage_ref as G
import train_mv_step_ref as T

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MODE = {"bf16": "kernel", "fp32": "exact"}
RUNS = [("nvidia", "bf16"), ("nvidia", "fp32"), ("linear", "bf16"), ("fresh", "bf16"), ("fresh", "fp32"),
        ("edges", "bf16"), ("edges", "fp32"), ("short", "bf16"), ("sliced", "bf16")]

BARS = {
    "bf16": {
        "grad.fine_featmaps[0]": (3e-03, 2e-03),  # 1.02e-03 7.64e-04 linear
        "grad.fine_featmaps[2]": (3e-03, 3e-03),  # 1.38e-03 1.21e-03 edges / short
        "grad.motion_mlp_fine.coeff_linear.bias": (1e-04, 1e-04),  # 7.28e-06 7.70e-06 edges
        "grad.motion_mlp_fine.coeff_linear.weight": (1e-04, 1e-04),  # 2.65e-05 3.56e-05 edges
        "grad.motion_mlp_fine.pts_linears.0.bias": (9e-04, 8e-04),  # 4.38e-04 3.78e-04 edges
        "grad.motion_mlp_fine.pts_linears.0.weight": (2e-03, 8e-04),  # 5.95e-04 3.60e-04 edges
        "grad.motion_mlp_fine.pts_linears.1.bias": (7e-04, 2e-03),  # 3.41e-04 7.30e-04 edges
        "grad.motion_mlp_fine.pts_linears.1.weight": (9e-04, 2e-03),  # 4.29e-04 8.78e-04 edges
        "grad.motion_mlp_fine.pts_linears.2.bias": (6e-04, 6e-04),  # 2.55e-04 2.61e-04 edges
        "grad.motion_mlp_fine.pts_linears.2.weight": (7e-04, 6e-04),  # 3.04e-04 2.82e-04 edges
        "grad.motion_mlp_fine.pts_linears.3.bias": (5e-04, 8e-04),  # 2.10e-04 3.73e-04 edges
        "grad.motion_mlp_fine.pts_linears.3.weight": (5e-04, 9e-04),  # 2.40e-04 4.19e-04 edges
        "grad.motion_mlp_fine.pts_linears.4.bias": (4e-04, 4e-04),  # 1.61e-04 1.88e-04 edges
        "grad.motion_mlp_fine.pts_linears.4.weight": (4e-04, 5e-04),  # 1.80e-04 2.05e-04 edges
        "grad.motion_mlp_fine.pts_linears.5.bias": (3e-04, 2e-04),  # 1.44e-04 9.43e-05 edges
        "grad.motion_mlp_fine.pts_linears.5.weight": (5e-04, 3e-04),  # 2.21e-04 1.21e-04 edges
        "grad.motion_mlp_fine.pts_linears.6.bias": (3e-04, 2e-04),  # 1.04e-04 8.82e-05 edges
        "grad.motion_mlp_fine.pts_linears.6.weight": (3e-04, 3e-04),  # 1.47e-04 1.47e-04 edges
        "grad.motion_mlp_fine.pts_linears.7.bias": (2e-04, 4e-04),  # 8.18e-05 1.86e-04 edges
        "grad.motion_mlp_fine.pts_linears.7.weight": (3e-04, 5e-04),  # 1.07e-04 2.21e-04 edges
        "grad.net_fine_dy.base_fc.0.bias": (2e-03, 9e-04),  # 5.33e-04 4.10e-04 edges
        "grad.net_fine_dy.base_fc.0.weight": (2e-03, 2e-03),  # 5.92e-04 6.19e-04 edges / short
        "grad.net_fine_dy.base_fc.2.bias": (2e-03, 1e-03),  # 5.19e-04 4.81e-04 edges
        "grad.net_fine_dy.base_fc.2.weight": (2e-03, 1e-03),  # 5.05e-04 4.65e-04 edges
        "grad.net_fine_dy.geometry_fc.0.bias": (8e-04, 2e-03),  # 3.97e-04 5.27e-04 edges
        "grad.net_fine_dy.geometry_fc.0.weight": (1e-03, 2e-03),  # 4.96e-04 5.25e-04 edges
        "grad.net_fine_dy.geometry_fc.2.bias": (8e-04, 7e-04),  # 3.84e-04 3.27e-04 edges
        "grad.net_fine_dy.geometry_fc.2.weight": (1e-03, 9e-04),  # 4.67e-04 4.26e-04 edges
        "grad.net_fine_dy.out_geometry_fc.0.bias": (4e-04, 1e-03),  # 1.79e-04 4.74e-04 short
        "grad.net_fine_dy.out_geometry_fc.0.weight": (3e-03, 3e-03),  # 1.09e-03 1.38e-03 short
        "grad.net_fine_dy.out_geometry_fc.2.bias": (2e-04, 2e-04),  # 7.92e-05 7.92e-05 short
        "grad.net_fine_dy.out_geometry_fc.2.weight": (3e-03, 2e-03),  # 1.42e-03 9.44e-04 short
        "grad.net_fine_dy.ray_attention.fc.weight": (2e-03, 2e-03),  # 5.37e-04 6.59e-04 edges
        "grad.net_fine_dy.ray_attention.layer_norm.bias": (8e-04, 8e-04),  # 3.64e-04 3.82e-04 edges
        "grad.net_fine_dy.ray_attention.layer_norm.weight": (2e-03, 2e-03),  # 5.78e-04 5.58e-04 edges
        "grad.net_fine_dy.ray_attention.w_ks.weight": (3e-03, 2e-03),  # 1.15e-03 8.46e-04 edges / short
        "grad.net_fine_dy.ray_attention.w_qs.weight": (3e-03, 2e-03),  # 1.01e-03 8.90e-04 short
        "grad.net_fine_dy.ray_attention.w_vs.weight": (2e-03, 2e-03),  # 5.97e-04 5.66e-04 edges
        "grad.net_fine_dy.ray_dir_fc.0.bias": (2e-03, 2e-03),  # 5.54e-04 5.35e-04 edges
        "grad.net_fine_dy.ray_dir_fc.0.weight": (2e-03, 2e-03),  # 5.54e-04 5.35e-04 edges
        "grad.net_fine_dy.ray_dir_fc.2.bias": (2e-03, 2e-03),  # 5.86e-04 5.76e-04 edges
        "grad.net_fine_dy.ray_dir_fc.2.weight": (2e-03, 2e-03),  # 5.86e-04 5.76e-04 edges
        "grad.net_fine_dy.ref_pts_fc.0.bias": (5e-04, 4e-04),  # 2.11e-04 1.92e-04 short
        "grad.net_fine_dy.ref_pts_fc.0.weight": (2e-03, 1e-03),  # 5.11e-04 4.79e-04 edges
        "grad.net_fine_dy.ref_pts_fc.2.bias": (4e-04, 4e-04),  # 1.61e-04 1.66e-04 short
        "grad.net_fine_dy.ref_pts_fc.2.weight": (8e-04, 9e-04),  # 3.92e-04 4.45e-04 edges
        "grad.net_fine_dy.rgb_fc.0.bias": (2e-04, 2e-04),  # 8.73e-05 8.43e-05 fresh
        "grad.net_fine_dy.rgb_fc.0.weight": (6e-04, 6e-04),  # 2.94e-04 2.72e-04 fresh
        "grad.net_fine_dy.rgb_fc.2.bias": (1e-04, 2e-04),  # 4.17e-05 5.21e-05 fresh / short
        "grad.net_fine_dy.rgb_fc.2.weight": (7e-04, 6e-04),  # 3.24e-04 2.51e-04 fresh
        "grad.net_fine_dy.rgb_fc.4.bias": (1e-04, 1e-04),  # 4.09e-05 4.62e-05 fresh
        "grad.net_fine_dy.rgb_fc.4.weight": (8e-04, 7e-04),  # 3.90e-04 3.41e-04 fresh
        "grad.net_fine_dy.vis_fc.0.bias": (1e-03, 2e-03),  # 4.74e-04 6.07e-04 edges
        "grad.net_fine_dy.vis_fc.0.weight": (2e-03, 2e-03),  # 6.29e-04 5.35e-04 edges / short
        "grad.net_fine_dy.vis_fc.2.bias": (2e-03, 1e-03),  # 5.15e-04 4.74e-04 edges
        "grad.net_fine_dy.vis_fc.2.weight": (2e-03, 1e-03),  # 5.34e-04 4.99e-04 edges
        "grad.net_fine_dy.vis_fc2.0.bias": (2e-03, 9e-04),  # 5.96e-04 4.09e-04 edges
        "grad.net_fine_dy.vis_fc2.0.weight": (2e-03, 3e-03),  # 7.67e-04 1.49e-03 short
        "grad.net_fine_dy.vis_fc2.2.bias": (1e-04, 2e-04),  # 1.53e-05 5.17e-05 edges
        "grad.net_fine_dy.vis_fc2.2.weight": (4e-03, 4e-03),  # 1.58e-03 1.79e-03 short
        "grad.net_fine_st.base_fc.0.bias": (2e-04, 2e-04),  # 8.92e-05 8.96e-05 edges
        "grad.net_fine_st.base_fc.0.weight": (5e-04, 5e-04),  # 2.37e-04 2.01e-04 edges
        "grad.net_fine_st.base_fc.2.bias": (2e-04, 3e-04),  # 8.56e-05 1.04e-04 edges
        "grad.net_fine_st.base_fc.2.weight": (4e-04, 3e-04),  # 1.72e-04 1.08e-04 edges
        "grad.net_fine_st.geometry_fc.0.bias": (2e-04, 2e-04),  # 7.69e-05 8.04e-05 short
        "grad.net_fine_st.geometry_fc.0.weight": (3e-04, 3e-04),  # 1.06e-04 1.18e-04 edges
        "grad.net_fine_st.geometry_fc.2.bias": (2e-04, 2e-04),  # 7.58e-05 6.47e-05 short
        "grad.net_fine_st.geometry_fc.2.weight": (2e-04, 2e-04),  # 9.75e-05 8.52e-05 short
        "grad.net_fine_st.out_geometry_fc.0.bias": (2e-04, 3e-04),  # 6.88e-05 1.07e-04 short
        "grad.net_fine_st.out_geometry_fc.0.weight": (3e-04, 4e-04),  # 1.39e-04 1.80e-04 short
        "grad.net_fine_st.out_geometry_fc.2.bias": (1e-04, 1e-04),  # 4.03e-05 4.03e-05 short
        "grad.net_fine_st.out_geometry_fc.2.weight": (4e-04, 3e-04),  # 1.61e-04 1.14e-04 short
        "grad.net_fine_st.ray_attention.fc.weight": (3e-04, 5e-04),  # 1.49e-04 2.07e-04 short / edges
        "grad.net_fine_st.ray_attention.layer_norm.bias": (2e-04, 2e-04),  # 7.01e-05 7.78e-05 short
        "grad.net_fine_st.ray_attention.layer_norm.weight": (4e-04, 5e-04),  # 1.54e-04 2.18e-04 short
        "grad.net_fine_st.ray_attention.w_ks.weight": (1e-02, 8e-03),  # 4.74e-03 3.69e-03 short
        "grad.net_fine_st.ray_attention.w_qs.weight": (1e-02, 2e-02),  # 4.83e-03 5.22e-03 short
        "grad.net_fine_st.ray_attention.w_vs.weight": (3e-04, 3e-04),  # 1.21e-04 1.42e-04 short / edges
        "grad.net_fine_st.ray_dir_fc.0.bias": (4e-04, 4e-04),  # 1.57e-04 1.98e-04 short
        "grad.net_fine_st.ray_dir_fc.0.weight": (6e-04, 8e-04),  # 2.86e-04 3.53e-04 short / edges
        "grad.net_fine_st.ray_dir_fc.2.bias": (3e-04, 3e-04),  # 1.17e-04 1.17e-04 short
        "grad.net_fine_st.ray_dir_fc.2.weight": (6e-04, 5e-04),  # 2.56e-04 2.49e-04 short
        "grad.net_fine_st.ref_feature_fc.0.bias": (4e-04, 4e-04),  # 1.83e-04 1.70e-04 edges / short
        "grad.net_fine_st.ref_feature_fc.0.weight": (5e-04, 5e-04),  # 2.10e-04 2.31e-04 edges / short
        "grad.net_fine_st.rgb_fc.0.bias": (2e-03, 6e-03),  # 9.23e-04 2.98e-03 short
        "grad.net_fine_st.rgb_fc.0.weight": (3e-02, 2e-02),  # 1.12e-02 7.67e-03 short
        "grad.net_fine_st.rgb_fc.2.bias": (2e-03, 8e-03),  # 5.09e-04 3.89e-03 short
        "grad.net_fine_st.rgb_fc.2.weight": (4e-02, 6e-02),  # 1.83e-02 2.65e-02 short
        "grad.net_fine_st.rgb_fc.4.bias": (1e-04, 1e-04),  # 3.39e-06 1.20e-05 short
        "grad.net_fine_st.rgb_fc.4.weight": (5e-02, 9e-02),  # 2.39e-02 4.00e-02 short
        "grad.net_fine_st.s": (2e-01, 2e-01),  # 5.03e-02 5.03e-02 short
        "grad.net_fine_st.vis_fc.0.bias": (2e-04, 3e-04),  # 9.96e-05 1.11e-04 short
        "grad.net_fine_st.vis_fc.0.weight": (5e-04, 4e-04),  # 2.20e-04 1.66e-04 edges / short
        "grad.net_fine_st.vis_fc.2.bias": (2e-04, 2e-04),  # 8.25e-05 9.66e-05 edges
        "grad.net_fine_st.vis_fc.2.weight": (3e-04, 3e-04),  # 1.01e-04 1.10e-04 edges / short
        "grad.net_fine_st.vis_fc2.0.bias": (5e-03, 3e-03),  # 2.29e-03 1.13e-03 short
        "grad.net_fine_st.vis_fc2.0.weight": (2e-03, 2e-03),  # 7.04e-04 8.13e-04 edges
        "grad.net_fine_st.vis_fc2.2.bias": (3e-04, 1e-03),  # 1.26e-04 4.83e-04 short
        "grad.net_fine_st.vis_fc2.2.weight": (2e-03, 2e-03),  # 6.74e-04 7.27e-04 edges
        "grad.trajectory_basis_fine": (1e-04, 1e-04),  # 1.07e-05 1.06e-05 edges
        "out.fine/alpha": (2e-04, 1e-04),  # 8.22e-05 4.61e-05 fresh
        "out.fine/alpha_dy": (1e-04, 1e-04),  # 3.74e-05 2.22e-05 nvidia / linear
        "out.fine/depth": (1e-04, 4e-04),  # 4.78e-05 1.58e-04 fresh / nvidia
        "out.fine/exp_sf": (2e-04, 3e-04),  # 5.81e-05 1.31e-04 linear
        "out.fine/mask": (1e-04, 1e-04),  # 0.00e+00 0.00e+00 nvidia
        "out.fine/render_flows": (1e-04, 3e-04),  # 4.78e-05 1.37e-04 fresh / nvidia
        "out.fine/rgb": (1e-04, 2e-04),  # 3.29e-05 9.65e-05 short
        "out.fine/rgb_dy": (2e-04, 4e-04),  # 5.78e-05 1.99e-04 short
        "out.fine/rgb_static": (2e-04, 3e-04),  # 5.23e-05 1.40e-04 nvidia / linear
        "out.fine/weights": (5e-04, 2e-03),  # 2.32e-04 9.78e-04 fresh / nvidia
        "out.fine/weights_dy": (4e-04, 2e-03),  # 1.83e-04 6.64e-04 fresh / linear
        "out.fine/weights_st": (9e-04, 3e-03),  # 4.47e-04 1.46e-03 fresh / linear
        "out.fine_dy/depth": (1e-04, 2e-04),  # 2.58e-05 7.97e-05 nvidia
        "out.fine_dy/mask": (1e-04, 1e-04),  # 0.00e+00 0.00e+00 nvidia
        "out.fine_dy/rgb": (2e-04, 5e-04),  # 5.83e-05 2.06e-04 short
        "out.fine_dy/weights": (3e-04, 4e-04),  # 1.35e-04 1.87e-04 nvidia
        "term.loss": (1e-04, 1e-04),  # 4.07e-06 4.07e-06 nvidia
    },
    "fp32": {
        "grad.fine_featmaps[0]": (2e-05, 2e-05),  # 5.43e-06 9.40e-06 fresh
        "grad.fine_featmaps[2]": (4e-05, 5e-05),  # 1.65e-05 2.28e-05 fresh / nvidia
        "grad.motion_mlp_fine.coeff_linear.bias": (1e-05, 1e-05),  # 2.16e-06 2.34e-06 nvidia
        "grad.motion_mlp_fine.coeff_linear.weight": (1e-05, 1e-05),  # 2.22e-06 2.75e-06 nvidia
        "grad.motion_mlp_fine.pts_linears.0.bias": (4e-05, 4e-05),  # 1.80e-05 1.78e-05 nvidia
        "grad.motion_mlp_fine.pts_linears.0.weight": (5e-05, 4e-05),  # 2.49e-05 1.62e-05 nvidia
        "grad.motion_mlp_fine.pts_linears.1.bias": (4e-05, 3e-05),  # 1.50e-05 1.35e-05 nvidia / edges
        "grad.motion_mlp_fine.pts_linears.1.weight": (4e-05, 6e-05),  # 1.79e-05 2.96e-05 nvidia / edges
        "grad.motion_mlp_fine.pts_linears.2.bias": (3e-05, 5e-05),  # 1.25e-05 2.10e-05 nvidia
        "grad.motion_mlp_fine.pts_linears.2.weight": (3e-05, 6e-05),  # 1.32e-05 2.56e-05 nvidia
        "grad.motion_mlp_fine.pts_linears.3.bias": (2e-05, 3e-05),  # 8.06e-06 1.09e-05 nvidia / edges
        "grad.motion_mlp_fine.pts_linears.3.weight": (2e-05, 3e-05),  # 8.11e-06 1.19e-05 nvidia / edges
        "grad.motion_mlp_fine.pts_linears.4.bias": (2e-05, 2e-05),  # 7.07e-06 6.03e-06 nvidia
        "grad.motion_mlp_fine.pts_linears.4.weight": (2e-05, 2e-05),  # 6.97e-06 5.90e-06 nvidia
        "grad.motion_mlp_fine.pts_linears.5.bias": (2e-05, 2e-05),  # 6.89e-06 6.85e-06 nvidia
        "grad.motion_mlp_fine.pts_linears.5.weight": (2e-05, 2e-05),  # 9.87e-06 6.42e-06 nvidia
        "grad.motion_mlp_fine.pts_linears.6.bias": (1e-05, 1e-05),  # 4.92e-06 2.80e-06 nvidia
        "grad.motion_mlp_fine.pts_linears.6.weight": (2e-05, 1e-05),  # 6.11e-06 3.33e-06 nvidia
        "grad.motion_mlp_fine.pts_linears.7.bias": (1e-05, 3e-05),  # 3.65e-06 1.02e-05 nvidia
        "grad.motion_mlp_fine.pts_linears.7.weight": (1e-05, 3e-05),  # 3.98e-06 1.41e-05 nvidia
        "grad.net_fine_dy.base_fc.0.bias": (1e-05, 1e-05),  # 4.27e-07 7.85e-07 nvidia
        "grad.net_fine_dy.base_fc.0.weight": (1e-05, 1e-05),  # 1.48e-06 1.89e-06 edges
        "grad.net_fine_dy.base_fc.2.bias": (1e-05, 1e-05),  # 3.43e-07 5.25e-07 nvidia / edges
        "grad.net_fine_dy.base_fc.2.weight": (1e-05, 1e-05),  # 1.77e-06 2.56e-06 edges
        "grad.net_fine_dy.geometry_fc.0.bias": (1e-05, 1e-05),  # 3.59e-07 7.45e-07 edges
        "grad.net_fine_dy.geometry_fc.0.weight": (1e-05, 1e-05),  # 1.34e-06 2.31e-06 edges
        "grad.net_fine_dy.geometry_fc.2.bias": (1e-05, 1e-05),  # 3.10e-07 4.05e-07 edges
        "grad.net_fine_dy.geometry_fc.2.weight": (1e-05, 2e-05),  # 3.18e-06 7.20e-06 edges
        "grad.net_fine_dy.out_geometry_fc.0.bias": (1e-05, 1e-05),  # 2.90e-07 5.08e-07 edges
        "grad.net_fine_dy.out_geometry_fc.0.weight": (1e-05, 1e-05),  # 1.31e-06 2.29e-06 edges
        "grad.net_fine_dy.out_geometry_fc.2.bias": (1e-05, 1e-05),  # 3.37e-07 3.37e-07 nvidia
        "grad.net_fine_dy.out_geometry_fc.2.weight": (1e-05, 1e-05),  # 1.12e-06 1.46e-06 edges
        "grad.net_fine_dy.ray_attention.fc.weight": (1e-05, 1e-05),  # 1.25e-06 2.68e-06 edges
        "grad.net_fine_dy.ray_attention.layer_norm.bias": (1e-05, 1e-05),  # 5.53e-07 6.69e-07 nvidia
        "grad.net_fine_dy.ray_attention.layer_norm.weight": (1e-05, 1e-05),  # 4.49e-07 6.98e-07 nvidia
        "grad.net_fine_dy.ray_attention.w_ks.weight": (1e-05, 1e-05),  # 1.42e-06 2.11e-06 edges
        "grad.net_fine_dy.ray_attention.w_qs.weight": (1e-05, 1e-05),  # 1.33e-06 2.49e-06 edges
        "grad.net_fine_dy.ray_attention.w_vs.weight": (1e-05, 2e-05),  # 1.95e-06 6.43e-06 edges
        "grad.net_fine_dy.ray_dir_fc.0.bias": (1e-05, 1e-05),  # 3.68e-07 4.09e-07 edges / nvidia
        "grad.net_fine_dy.ray_dir_fc.0.weight": (1e-05, 1e-05),  # 3.64e-07 4.27e-07 edges / nvidia
        "grad.net_fine_dy.ray_dir_fc.2.bias": (1e-05, 1e-05),  # 3.66e-07 5.96e-07 edges
        "grad.net_fine_dy.ray_dir_fc.2.weight": (1e-05, 1e-05),  # 3.84e-07 6.84e-07 edges
        "grad.net_fine_dy.ref_pts_fc.0.bias": (1e-05, 1e-05),  # 3.40e-07 8.24e-07 edges
        "grad.net_fine_dy.ref_pts_fc.0.weight": (1e-05, 1e-05),  # 1.29e-06 3.74e-06 edges
        "grad.net_fine_dy.ref_pts_fc.2.bias": (1e-05, 1e-05),  # 3.22e-07 5.64e-07 edges
        "grad.net_fine_dy.ref_pts_fc.2.weight": (1e-05, 1e-05),  # 1.26e-06 2.26e-06 edges
        "grad.net_fine_dy.rgb_fc.0.bias": (1e-05, 1e-05),  # 6.33e-07 7.55e-07 fresh
        "grad.net_fine_dy.rgb_fc.0.weight": (1e-05, 1e-05),  # 8.63e-07 9.70e-07 fresh
        "grad.net_fine_dy.rgb_fc.2.bias": (1e-05, 1e-05),  # 5.61e-07 5.14e-07 fresh
        "grad.net_fine_dy.rgb_fc.2.weight": (1e-05, 1e-05),  # 1.11e-06 1.44e-06 fresh
        "grad.net_fine_dy.rgb_fc.4.bias": (1e-05, 1e-05),  # 5.28e-07 5.54e-07 fresh
        "grad.net_fine_dy.rgb_fc.4.weight": (1e-05, 1e-05),  # 1.16e-06 2.44e-06 fresh
        "grad.net_fine_dy.vis_fc.0.bias": (1e-05, 1e-05),  # 3.68e-07 4.78e-07 nvidia / edges
        "grad.net_fine_dy.vis_fc.0.weight": (1e-05, 1e-05),  # 1.78e-06 2.60e-06 edges
        "grad.net_fine_dy.vis_fc.2.bias": (1e-05, 1e-05),  # 4.16e-07 6.96e-07 nvidia
        "grad.net_fine_dy.vis_fc.2.weight": (1e-05, 1e-05),  # 2.03e-06 4.06e-06 edges
        "grad.net_fine_dy.vis_fc2.0.bias": (1e-05, 1e-05),  # 3.64e-06 2.42e-06 edges
        "grad.net_fine_dy.vis_fc2.0.weight": (1e-05, 1e-05),  # 1.99e-06 3.03e-06 edges
        "grad.net_fine_dy.vis_fc2.2.bias": (1e-05, 1e-05),  # 2.90e-07 9.78e-07 edges
        "grad.net_fine_dy.vis_fc2.2.weight": (1e-05, 1e-05),  # 2.36e-06 2.24e-06 edges
        "grad.net_fine_st.base_fc.0.bias": (1e-05, 1e-05),  # 4.50e-07 6.76e-07 nvidia
        "grad.net_fine_st.base_fc.0.weight": (1e-05, 1e-05),  # 7.69e-07 1.20e-06 fresh
        "grad.net_fine_st.base_fc.2.bias": (1e-05, 1e-05),  # 3.96e-07 6.79e-07 nvidia
        "grad.net_fine_st.base_fc.2.weight": (1e-05, 1e-05),  # 6.76e-07 6.79e-07 fresh / nvidia
        "grad.net_fine_st.geometry_fc.0.bias": (1e-05, 1e-05),  # 3.11e-07 3.52e-07 edges / nvidia
        "grad.net_fine_st.geometry_fc.0.weight": (1e-05, 1e-05),  # 5.46e-07 9.51e-07 edges
        "grad.net_fine_st.geometry_fc.2.bias": (1e-05, 1e-05),  # 3.08e-07 3.36e-07 edges
        "grad.net_fine_st.geometry_fc.2.weight": (1e-05, 1e-05),  # 5.66e-07 7.76e-07 edges
        "grad.net_fine_st.out_geometry_fc.0.bias": (1e-05, 1e-05),  # 3.08e-07 3.63e-07 edges
        "grad.net_fine_st.out_geometry_fc.0.weight": (1e-05, 1e-05),  # 5.30e-07 1.22e-06 edges
        "grad.net_fine_st.out_geometry_fc.2.bias": (1e-05, 1e-05),  # 3.22e-07 3.22e-07 edges
        "grad.net_fine_st.out_geometry_fc.2.weight": (1e-05, 1e-05),  # 4.90e-07 6.47e-07 edges
        "grad.net_fine_st.ray_attention.fc.weight": (1e-05, 1e-05),  # 6.57e-07 8.46e-07 fresh / edges
        "grad.net_fine_st.ray_attention.layer_norm.bias": (1e-05, 1e-05),  # 5.46e-07 7.70e-07 nvidia
        "grad.net_fine_st.ray_attention.layer_norm.weight": (1e-05, 1e-05),  # 5.64e-07 7.86e-07 nvidia
        "grad.net_fine_st.ray_attention.w_ks.weight": (5e-05, 5e-05),  # 2.11e-05 2.42e-05 fresh
        "grad.net_fine_st.ray_attention.w_qs.weight": (5e-05, 6e-05),  # 2.16e-05 2.55e-05 fresh
        "grad.net_fine_st.ray_attention.w_vs.weight": (1e-05, 1e-05),  # 7.05e-07 1.08e-06 fresh / edges
        "grad.net_fine_st.ray_dir_fc.0.bias": (1e-05, 1e-05),  # 5.32e-07 9.37e-07 nvidia
        "grad.net_fine_st.ray_dir_fc.0.weight": (1e-05, 1e-05),  # 8.68e-07 1.82e-06 nvidia
        "grad.net_fine_st.ray_dir_fc.2.bias": (1e-05, 1e-05),  # 3.17e-07 4.05e-07 edges
        "grad.net_fine_st.ray_dir_fc.2.weight": (1e-05, 1e-05),  # 8.28e-07 7.19e-07 nvidia
        "grad.net_fine_st.ref_feature_fc.0.bias": (1e-05, 1e-05),  # 6.74e-07 7.51e-07 fresh
        "grad.net_fine_st.ref_feature_fc.0.weight": (1e-05, 1e-05),  # 7.48e-07 1.10e-06 nvidia
        "grad.net_fine_st.rgb_fc.0.bias": (1e-05, 3e-05),  # 3.17e-06 1.34e-05 nvidia / fresh
        "grad.net_fine_st.rgb_fc.0.weight": (1e-04, 8e-05),  # 4.87e-05 3.55e-05 nvidia / fresh
        "grad.net_fine_st.rgb_fc.2.bias": (1e-05, 7e-05),  # 3.76e-06 3.31e-05 fresh
        "grad.net_fine_st.rgb_fc.2.weight": (7e-05, 1e-04),  # 3.06e-05 4.52e-05 nvidia / fresh
        "grad.net_fine_st.rgb_fc.4.bias": (1e-05, 1e-05),  # 1.16e-06 3.52e-06 fresh
        "grad.net_fine_st.rgb_fc.4.weight": (6e-05, 6e-05),  # 2.66e-05 2.85e-05 nvidia / fresh
        "grad.net_fine_st.s": (6e-03, 6e-03),  # 2.83e-03 2.83e-03 nvidia
        "grad.net_fine_st.vis_fc.0.bias": (1e-05, 1e-05),  # 4.79e-07 9.91e-07 nvidia
        "grad.net_fine_st.vis_fc.0.weight": (1e-05, 1e-05),  # 6.31e-07 7.85e-07 fresh
        "grad.net_fine_st.vis_fc.2.bias": (1e-05, 1e-05),  # 4.21e-07 6.81e-07 nvidia
        "grad.net_fine_st.vis_fc.2.weight": (1e-05, 1e-05),  # 3.36e-07 6.53e-07 edges / nvidia
        "grad.net_fine_st.vis_fc2.0.bias": (1e-05, 1e-05),  # 4.43e-06 3.03e-06 edges
        "grad.net_fine_st.vis_fc2.0.weight": (1e-05, 1e-05),  # 6.20e-07 8.28e-07 edges
        "grad.net_fine_st.vis_fc2.2.bias": (1e-05, 1e-05),  # 2.50e-07 9.48e-07 edges
        "grad.net_fine_st.vis_fc2.2.weight": (1e-05, 1e-05),  # 7.40e-07 7.83e-07 edges
        "grad.trajectory_basis_fine": (1e-05, 1e-05),  # 2.67e-06 3.25e-06 nvidia
        "out.fine/alpha": (1e-05, 2e-05),  # 1.46e-06 6.98e-06 fresh
        "out.fine/alpha_dy": (1e-05, 1e-05),  # 3.47e-07 8.74e-08 fresh / nvidia
        "out.fine/depth": (1e-05, 1e-05),  # 7.45e-07 1.90e-06 fresh / nvidia
        "out.fine/exp_sf": (1e-05, 1e-05),  # 1.85e-07 3.64e-07 edges / nvidia
        "out.fine/mask": (1e-05, 1e-05),  # 0.00e+00 0.00e+00 nvidia
        "out.fine/render_flows": (1e-05, 1e-05),  # 1.14e-06 3.00e-06 nvidia
        "out.fine/rgb": (1e-05, 1e-05),  # 4.67e-07 4.39e-06 fresh / nvidia
        "out.fine/rgb_dy": (1e-05, 1e-05),  # 3.10e-07 1.04e-06 fresh / nvidia
        "out.fine/rgb_static": (1e-05, 3e-05),  # 1.16e-06 1.05e-05 nvidia
        "out.fine/weights": (1e-05, 1e-05),  # 1.50e-06 4.79e-06 nvidia
        "out.fine/weights_dy": (1e-05, 2e-05),  # 1.85e-06 6.30e-06 fresh
        "out.fine/weights_st": (1e-05, 2e-05),  # 2.91e-06 6.30e-06 nvidia / fresh
        "out.fine_dy/depth": (1e-05, 1e-05),  # 1.08e-06 1.68e-06 fresh / nvidia
        "out.fine_dy/mask": (1e-05, 1e-05),  # 0.00e+00 0.00e+00 nvidia
        "out.fine_dy/rgb": (1e-05, 1e-05),  # 9.07e-08 3.26e-07 fresh
        "out.fine_dy/weights": (1e-05, 1e-05),  # 1.65e-06 2.62e-06 fresh / nvidia
        "term.loss": (1e-05, 1e-05),  # 1.28e-06 1.28e-06 fresh
    },
}


def bar(prec, name):
  return BARS[prec][name]


def ratios(errs, prec):
  return {k: max(r / bar(prec, k)[0], m / bar(prec, k)[1]) for k, (r, m) in errs.items()}


def resample_check(c, got):
  """Rows of the library's fine depths outside geometry_stage_ref's float64 resampling of its own coarse weights."""
  case = dict(z=got["coarse"]["z_vals"].float(), weights=got["coarse"]["weights"].float(),
              u=None if c["det"] else c["u"].float(), R=c["R"], S=c["Sc"], Ni=c["Si"], inv_uniform=bool(c["inv"]),
              det=c["det"])
  return G.resample_check(case, G.resample(case), got["z_fine"])


def run(case, prec):
  """Library step, then (its tensors freed) the reference -> (errors, zero violations, resampling rows out of bounds,
  coarse errors, stats)."""
  c = T.make_case(case)
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  t0 = time.perf_counter()
  got = T.library(c, DEV, prec)
  torch.cuda.synchronize()
  stats = {"library_s": time.perf_counter() - t0, "library_peak_GB": torch.cuda.max_memory_allocated() / 2 ** 30}
  torch.cuda.empty_cache()
  torch.cuda.reset_peak_memory_stats()
  t0 = time.perf_counter()
  ref = T.reference(c, DEV, MODE[prec], z_fine=got["z_fine"], chunk=c["chunk"])
  torch.cuda.synchronize()
  stats.update(reference_s=time.perf_counter() - t0, reference_peak_GB=torch.cuda.max_memory_allocated() / 2 ** 30)
  errs = T.errors(got, ref, c["V_st"])
  zero = T.zero_violations(got, ref)
  coarse = T.coarse_errors(got, ref)
  del ref
  torch.cuda.empty_cache()
  bad_rows, _ = resample_check(c, got)
  return errs, zero, bad_rows, coarse, stats


@pytest.mark.parametrize("case,prec", RUNS)
def test_fine_training_step_matches_reference(case, prec):
  errs, zero, bad_rows, coarse, stats = run(case, prec)
  r = ratios(errs, prec)
  worst = max(r.items(), key=lambda kv: kv[1])
  print("\nmv step %s %s: worst %s, %.2f of its bar; %s" % (case, prec, worst[0], worst[1],
                                                            ", ".join("%s %.2f" % kv for kv in stats.items())))
  for name, (rel, mx) in sorted(errs.items()):
    print("  ERR %s %s %s %.3e %.3e" % (case, prec, name, rel, mx))
  for name, (rel, mx) in sorted(coarse.items()):
    print("  COARSE (no bar) %s %s %s %.3e %.3e" % (case, prec, name, rel, mx))
  assert not zero, (case, prec, zero)
  assert not bad_rows, (case, prec, "fine depths outside the float64 resampling", bad_rows[:10])
  for k in ("out.fine/mask", "out.fine_dy/mask"):
    assert errs[k] == (0.0, 0.0), (case, prec, k, errs[k])
  bad = {k: (errs[k], bar(prec, k)) for k, v in r.items() if not v <= 1.0}
  assert not bad, (case, prec, bad)


def plant_margins():
  """{plant: (the compared tensor it moves most, relative to its bf16 bar; that ratio)} on T.PLANT_CASE.  Both
  evaluations resample with the oracle, which no plant touches (each acts on the fine pass only)."""
  c = T.make_case(T.PLANT_CASE)
  clean = T.reference(c, DEV, "kernel")
  out = {}
  for plant in T.PLANTS:
    r = ratios(T.errors(T.reference(c, DEV, "kernel", plant=plant), clean, c["V_st"]), "bf16")
    out[plant] = max(r.items(), key=lambda kv: kv[1])
  return out


def test_plants_exceed_bars():
  margins = plant_margins()
  for plant, (name, m) in margins.items():
    print("\nplant %s: %s moves %.1fx its bar" % (plant, name, m))
  low = {p: v for p, v in margins.items() if not v[1] >= T.PLANT_MARGIN}
  assert not low, low
