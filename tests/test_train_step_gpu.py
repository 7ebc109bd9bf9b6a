"""One whole monocular training step against its float64 reference (tests/train_step_ref.py), on the device.

The library runs the step as train.py does: render_rays_mono(is_train=True) over the whole batch with its cross-time
branch, criterion.mono_step_loss, backward, with the feature maps and trajectory_basis as leaves.  The reference is the
oracle's render_rays_mono in float64 with the library's nets swapped in (mode "kernel" for precision bf16, which
rounds exactly the products the library puts on the tensor cores; "exact" for fp32) and loss_ref's criterion.
Compared, per tensor, as relative L2 error and max |error| / max |reference|: the nine loss terms, every output the
criterion reads (render_flows and the masks included), and the gradient of every parameter of net_coarse_dy,
net_coarse_st (`s` where anti-aliasing is on) and motion_mlp, of trajectory_basis and of featmaps[0..2].

Cases (train_step_ref.CASES):
  shipped      the shipped config's step: 1024 rays x 64 samples, 288x512 frames, 7 + 3 dynamic and 14 static views,
               the anchor stack, anti_alias_pooling 0, mask_rgb 1, epoch 0: 917 504 static and 655 360 dynamic
               (point, view) rows per net call, so the split-K dW slabs, the featmap scatter-adds and the 14-view
               group sums run at training size
  late         the same step past 5 init_decay_epoch: static_dy on, dynamic_rgb off
  edges_occ*   105 rays on 48x64 frames, reference frame 1 (basis rows wrap, anchor cycle lists shrink), the anchor one
               frame away, anti-aliasing on, occ_weights_mode 1 / 2, rays no static view sees, rays with fewer than
               2 valid dynamic views

Bars (BARS): per precision and tensor, 2x the worst value measured over this file's cases on an H100 80GB HBM3
(700 W power limit), rounded up to one digit, at least 1e-5 (fp32) / 1e-4 (bf16); the comment beside each bar records
the measured worst relative L2 error, the worst max-abs ratio and their cases.  The four masks are equal bit for bit
in every case; the loss terms agree to within 9e-7 in fp32 and 7e-5 (cycle_loss, edges_occ1) in bf16.
  fp32: outputs and net gradients 1e-7 - 6e-5 (worst net_coarse_st.rgb_fc.0.weight 5.6e-5, shipped).  The MotionMLP's
        pts_linears gradients reach 8.4e-4 (pts_linears.0.weight, edges_occ1): ReLU flips, a unit whose pre-activation
        lies within fp32 rounding of 0 takes the other side.  The same reference evaluated in float32 on the CPU is
        7.9e-4 from its float64 evaluation on that tensor, so this is fp32 arithmetic, not wiring.
  bf16: outputs 2e-6 - 6e-4 (sf_seq, edges_occ2), trunk and per-view gradients 1e-4 - 6e-3, trajectory_basis
        4e-4, the feature maps 1.5e-3 - 3.1e-3, the MotionMLP 4e-4 - 1e-2
        (ReLU flips again), the static blending head up to 2.2e-2 (net_coarse_st.rgb_fc.4.weight, late; rgb_fc.2
        1.5e-2).  None needs test_train_gpu.py's 5e-2 / 1.5e-1.  The reference evaluated in float32 (mode "kernel") is
        as far from its float64 evaluation on the same tensors -- rgb_fc.2.weight 9.6e-3, rgb_fc.4.weight 1.0e-2 on
        shipped; pts_linears.0.weight 6.1e-3 on edges_occ1 -- so the size is bf16 double rounding compounding through
        the blending head (tests/test_train_stage_gpu.py), not a wiring error.

Measured per case (library step, then the reference; wall time incl. host work, peak device memory allocated):
  shipped bf16   library 0.98 s (first call) / 15.7 GB, reference 2.2 s / 11.3 GB (128-ray chunks)
  shipped fp32   library 0.36 s / 17.9 GB, reference 1.5 s / 11.3 GB
  late bf16      library 0.22 s / 17.9 GB, reference 1.4 s / 13.1 GB
  edges bf16     library 0.07 s / 6.0 - 6.2 GB, reference 0.3 - 0.6 s / 10.1 - 10.3 GB (one chunk)
  edges fp32     library 0.1 - 0.3 s / 6.0 GB, reference 0.16 s / 10.1 GB

PLANTS: each glue wiring error of train_step_ref.PLANTS, planted in the float64 reference on edges_occ1, moves some
compared tensor by at least PLANT_MARGIN times its bf16 bar; the test prints every plant's margin.  Measured:
anchor_raw_st_detached 3644x (net_coarse_st.out_geometry_fc.2.bias), anchor_feat_to_f0 244x (featmaps[0]),
sf_seq_shifted 696x (sf_seq), occ_not_detached 117x (net_coarse_dy.vis_fc.2.weight), flow_views_shifted 7178x
(render_flows), anchor_basis_detached 638x (trajectory_basis), vv_rows_displaced 85x (anchor_dy occ_weight_map).
"""

import time

import pytest
import torch

import train_step_ref as T

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MODE = {"bf16": "kernel", "fp32": "exact"}
RUNS = [("shipped", "bf16"), ("shipped", "fp32"), ("late", "bf16"), ("edges_occ1", "bf16"), ("edges_occ1", "fp32"),
        ("edges_occ2", "bf16"), ("edges_occ2", "fp32")]

BARS = {
    "bf16": {
        "grad.featmaps[0]": (6e-03, 7e-03),  # 2.65e-03 3.35e-03 shipped
        "grad.featmaps[1]": (7e-03, 6e-03),  # 3.13e-03 2.80e-03 shipped
        "grad.featmaps[2]": (4e-03, 7e-03),  # 1.54e-03 3.31e-03 shipped
        "grad.motion_mlp.coeff_linear.bias": (8e-04, 7e-04),  # 3.70e-04 3.43e-04 late
        "grad.motion_mlp.coeff_linear.weight": (9e-04, 7e-04),  # 4.25e-04 3.21e-04 edges_occ1
        "grad.motion_mlp.pts_linears.0.bias": (1e-02, 2e-02),  # 4.67e-03 5.09e-03 edges_occ1
        "grad.motion_mlp.pts_linears.0.weight": (2e-02, 6e-02),  # 9.77e-03 2.80e-02 edges_occ1
        "grad.motion_mlp.pts_linears.1.bias": (8e-03, 7e-03),  # 3.65e-03 3.10e-03 edges_occ1 / edges_occ2
        "grad.motion_mlp.pts_linears.1.weight": (2e-02, 2e-02),  # 7.50e-03 5.86e-03 edges_occ1
        "grad.motion_mlp.pts_linears.2.bias": (7e-03, 6e-03),  # 3.20e-03 2.78e-03 edges_occ1
        "grad.motion_mlp.pts_linears.2.weight": (2e-02, 1e-02),  # 5.81e-03 4.65e-03 edges_occ1
        "grad.motion_mlp.pts_linears.3.bias": (6e-03, 8e-03),  # 2.75e-03 3.64e-03 edges_occ1
        "grad.motion_mlp.pts_linears.3.weight": (9e-03, 1e-02),  # 4.18e-03 4.65e-03 edges_occ1
        "grad.motion_mlp.pts_linears.4.bias": (5e-03, 5e-03),  # 2.16e-03 2.47e-03 edges_occ1
        "grad.motion_mlp.pts_linears.4.weight": (6e-03, 7e-03),  # 2.94e-03 3.10e-03 edges_occ1
        "grad.motion_mlp.pts_linears.5.bias": (4e-03, 4e-03),  # 1.72e-03 1.56e-03 edges_occ1
        "grad.motion_mlp.pts_linears.5.weight": (7e-03, 2e-02),  # 3.48e-03 9.40e-03 edges_occ1
        "grad.motion_mlp.pts_linears.6.bias": (3e-03, 3e-03),  # 1.41e-03 1.50e-03 edges_occ1
        "grad.motion_mlp.pts_linears.6.weight": (6e-03, 8e-03),  # 2.72e-03 3.66e-03 edges_occ1
        "grad.motion_mlp.pts_linears.7.bias": (2e-03, 3e-03),  # 9.04e-04 1.11e-03 edges_occ1
        "grad.motion_mlp.pts_linears.7.weight": (4e-03, 5e-03),  # 1.58e-03 2.42e-03 edges_occ1
        "grad.net_coarse_dy.base_fc.0.bias": (2e-03, 2e-03),  # 8.78e-04 8.59e-04 edges_occ1 / edges_occ2
        "grad.net_coarse_dy.base_fc.0.weight": (3e-03, 3e-03),  # 1.07e-03 1.14e-03 edges_occ1
        "grad.net_coarse_dy.base_fc.2.bias": (2e-03, 3e-03),  # 9.11e-04 1.03e-03 edges_occ1
        "grad.net_coarse_dy.base_fc.2.weight": (2e-03, 2e-03),  # 9.63e-04 9.40e-04 edges_occ1
        "grad.net_coarse_dy.geometry_fc.0.bias": (2e-03, 2e-03),  # 8.62e-04 8.38e-04 edges_occ1
        "grad.net_coarse_dy.geometry_fc.0.weight": (2e-03, 3e-03),  # 9.98e-04 1.06e-03 edges_occ1
        "grad.net_coarse_dy.geometry_fc.2.bias": (2e-03, 2e-03),  # 8.18e-04 7.41e-04 edges_occ1
        "grad.net_coarse_dy.geometry_fc.2.weight": (2e-03, 2e-03),  # 9.24e-04 9.44e-04 edges_occ1 / edges_occ2
        "grad.net_coarse_dy.out_geometry_fc.0.bias": (2e-03, 2e-03),  # 5.22e-04 5.18e-04 edges_occ1
        "grad.net_coarse_dy.out_geometry_fc.0.weight": (2e-03, 2e-03),  # 6.67e-04 8.04e-04 edges_occ1 / edges_occ2
        "grad.net_coarse_dy.out_geometry_fc.2.bias": (2e-03, 2e-03),  # 5.20e-04 5.20e-04 edges_occ1
        "grad.net_coarse_dy.out_geometry_fc.2.weight": (2e-03, 2e-03),  # 7.33e-04 6.24e-04 edges_occ1 / edges_occ2
        "grad.net_coarse_dy.ray_attention.fc.weight": (3e-03, 3e-03),  # 1.05e-03 1.05e-03 edges_occ1
        "grad.net_coarse_dy.ray_attention.layer_norm.bias": (2e-03, 3e-03),  # 8.95e-04 1.08e-03 edges_occ1
        "grad.net_coarse_dy.ray_attention.layer_norm.weight": (3e-03, 3e-03),  # 1.24e-03 1.45e-03 edges_occ1
        "grad.net_coarse_dy.ray_attention.w_ks.weight": (5e-03, 4e-03),  # 2.01e-03 1.97e-03 edges_occ1
        "grad.net_coarse_dy.ray_attention.w_qs.weight": (4e-03, 4e-03),  # 1.64e-03 1.51e-03 edges_occ1 / edges_occ2
        "grad.net_coarse_dy.ray_attention.w_vs.weight": (3e-03, 3e-03),  # 1.12e-03 1.12e-03 edges_occ1
        "grad.net_coarse_dy.ray_dir_fc.0.bias": (3e-03, 3e-03),  # 1.15e-03 1.10e-03 edges_occ1
        "grad.net_coarse_dy.ray_dir_fc.0.weight": (3e-03, 3e-03),  # 1.11e-03 1.05e-03 edges_occ1
        "grad.net_coarse_dy.ray_dir_fc.2.bias": (3e-03, 3e-03),  # 1.18e-03 1.11e-03 edges_occ1 / edges_occ2
        "grad.net_coarse_dy.ray_dir_fc.2.weight": (3e-03, 3e-03),  # 1.14e-03 1.02e-03 edges_occ1 / edges_occ2
        "grad.net_coarse_dy.ref_pts_fc.0.bias": (2e-03, 2e-03),  # 8.04e-04 8.25e-04 edges_occ1
        "grad.net_coarse_dy.ref_pts_fc.0.weight": (4e-03, 6e-03),  # 1.96e-03 2.68e-03 edges_occ1
        "grad.net_coarse_dy.ref_pts_fc.2.bias": (2e-03, 1e-03),  # 6.14e-04 4.95e-04 edges_occ1
        "grad.net_coarse_dy.ref_pts_fc.2.weight": (4e-03, 5e-03),  # 1.67e-03 2.41e-03 edges_occ1
        "grad.net_coarse_dy.rgb_fc.0.bias": (7e-04, 6e-04),  # 3.15e-04 3.00e-04 edges_occ1
        "grad.net_coarse_dy.rgb_fc.0.weight": (2e-03, 2e-03),  # 8.00e-04 7.74e-04 edges_occ1 / edges_occ2
        "grad.net_coarse_dy.rgb_fc.2.bias": (5e-04, 4e-04),  # 2.15e-04 1.77e-04 shipped
        "grad.net_coarse_dy.rgb_fc.2.weight": (2e-03, 3e-03),  # 9.85e-04 1.18e-03 edges_occ1
        "grad.net_coarse_dy.rgb_fc.4.bias": (5e-04, 5e-04),  # 2.21e-04 2.32e-04 shipped
        "grad.net_coarse_dy.rgb_fc.4.weight": (3e-03, 3e-03),  # 1.00e-03 1.04e-03 edges_occ1
        "grad.net_coarse_dy.vis_fc.0.bias": (2e-03, 2e-03),  # 8.66e-04 8.78e-04 edges_occ1 / edges_occ2
        "grad.net_coarse_dy.vis_fc.0.weight": (3e-03, 4e-03),  # 1.15e-03 1.70e-03 edges_occ2 / edges_occ1
        "grad.net_coarse_dy.vis_fc.2.bias": (2e-03, 2e-03),  # 9.24e-04 9.63e-04 edges_occ1
        "grad.net_coarse_dy.vis_fc.2.weight": (2e-03, 2e-03),  # 9.06e-04 9.80e-04 edges_occ1
        "grad.net_coarse_dy.vis_fc2.0.bias": (4e-03, 5e-03),  # 1.96e-03 2.44e-03 edges_occ1
        "grad.net_coarse_dy.vis_fc2.0.weight": (4e-03, 5e-03),  # 1.96e-03 2.06e-03 edges_occ1
        "grad.net_coarse_dy.vis_fc2.2.bias": (2e-04, 4e-04),  # 5.69e-05 1.97e-04 edges_occ1
        "grad.net_coarse_dy.vis_fc2.2.weight": (4e-03, 4e-03),  # 1.65e-03 1.55e-03 edges_occ1
        "grad.net_coarse_st.base_fc.0.bias": (7e-04, 7e-04),  # 3.03e-04 3.21e-04 edges_occ2 / edges_occ1
        "grad.net_coarse_st.base_fc.0.weight": (2e-03, 2e-03),  # 7.01e-04 5.82e-04 edges_occ2
        "grad.net_coarse_st.base_fc.2.bias": (7e-04, 6e-04),  # 3.06e-04 2.62e-04 edges_occ2
        "grad.net_coarse_st.base_fc.2.weight": (2e-03, 8e-04),  # 5.35e-04 3.82e-04 edges_occ2 / edges_occ1
        "grad.net_coarse_st.geometry_fc.0.bias": (5e-04, 5e-04),  # 2.09e-04 2.00e-04 edges_occ2
        "grad.net_coarse_st.geometry_fc.0.weight": (9e-04, 9e-04),  # 4.22e-04 4.17e-04 edges_occ2
        "grad.net_coarse_st.geometry_fc.2.bias": (3e-04, 3e-04),  # 1.21e-04 1.45e-04 edges_occ2
        "grad.net_coarse_st.geometry_fc.2.weight": (6e-04, 9e-04),  # 2.81e-04 4.39e-04 edges_occ2
        "grad.net_coarse_st.out_geometry_fc.0.bias": (3e-04, 5e-04),  # 1.22e-04 2.48e-04 edges_occ2
        "grad.net_coarse_st.out_geometry_fc.0.weight": (7e-04, 2e-03),  # 3.39e-04 5.15e-04 edges_occ2
        "grad.net_coarse_st.out_geometry_fc.2.bias": (2e-04, 2e-04),  # 9.95e-05 9.95e-05 edges_occ2
        "grad.net_coarse_st.out_geometry_fc.2.weight": (8e-04, 2e-03),  # 3.93e-04 5.85e-04 edges_occ2
        "grad.net_coarse_st.ray_attention.fc.weight": (2e-03, 2e-03),  # 6.17e-04 9.53e-04 edges_occ2
        "grad.net_coarse_st.ray_attention.layer_norm.bias": (3e-04, 3e-04),  # 1.30e-04 1.31e-04 edges_occ2
        "grad.net_coarse_st.ray_attention.layer_norm.weight": (6e-04, 8e-04),  # 2.72e-04 3.62e-04 edges_occ2
        "grad.net_coarse_st.ray_attention.w_ks.weight": (5e-03, 6e-03),  # 2.31e-03 2.67e-03 edges_occ1
        "grad.net_coarse_st.ray_attention.w_qs.weight": (4e-03, 3e-03),  # 1.65e-03 1.48e-03 edges_occ2 / edges_occ1
        "grad.net_coarse_st.ray_attention.w_vs.weight": (2e-03, 2e-03),  # 6.42e-04 9.82e-04 edges_occ2
        "grad.net_coarse_st.ray_dir_fc.0.bias": (9e-04, 8e-04),  # 4.09e-04 3.83e-04 edges_occ2
        "grad.net_coarse_st.ray_dir_fc.0.weight": (2e-03, 2e-03),  # 6.60e-04 8.79e-04 edges_occ2 / edges_occ1
        "grad.net_coarse_st.ray_dir_fc.2.bias": (1e-03, 9e-04),  # 4.56e-04 4.47e-04 edges_occ2
        "grad.net_coarse_st.ray_dir_fc.2.weight": (2e-03, 2e-03),  # 6.00e-04 5.04e-04 edges_occ2
        "grad.net_coarse_st.ref_feature_fc.0.bias": (2e-03, 2e-03),  # 6.36e-04 5.87e-04 edges_occ2
        "grad.net_coarse_st.ref_feature_fc.0.weight": (2e-03, 2e-03),  # 6.39e-04 5.24e-04 edges_occ2 / edges_occ1
        "grad.net_coarse_st.rgb_fc.0.bias": (2e-03, 4e-03),  # 6.78e-04 1.68e-03 late
        "grad.net_coarse_st.rgb_fc.0.weight": (2e-02, 1e-02),  # 8.43e-03 4.66e-03 late
        "grad.net_coarse_st.rgb_fc.2.bias": (8e-04, 6e-03),  # 3.78e-04 2.75e-03 late / shipped
        "grad.net_coarse_st.rgb_fc.2.weight": (4e-02, 5e-02),  # 1.51e-02 2.19e-02 late
        "grad.net_coarse_st.rgb_fc.4.bias": (1e-04, 1e-04),  # 1.34e-06 5.01e-06 edges_occ1
        "grad.net_coarse_st.rgb_fc.4.weight": (5e-02, 8e-02),  # 2.23e-02 3.52e-02 late
        "grad.net_coarse_st.s": (4e-03, 4e-03),  # 1.56e-03 1.56e-03 edges_occ2
        "grad.net_coarse_st.vis_fc.0.bias": (7e-04, 8e-04),  # 3.34e-04 3.85e-04 edges_occ1
        "grad.net_coarse_st.vis_fc.0.weight": (3e-03, 2e-03),  # 1.03e-03 9.15e-04 edges_occ1 / edges_occ2
        "grad.net_coarse_st.vis_fc.2.bias": (7e-04, 6e-04),  # 3.05e-04 2.51e-04 edges_occ2
        "grad.net_coarse_st.vis_fc.2.weight": (8e-04, 9e-04),  # 3.54e-04 4.29e-04 edges_occ2
        "grad.net_coarse_st.vis_fc2.0.bias": (2e-02, 6e-03),  # 5.70e-03 2.86e-03 edges_occ1
        "grad.net_coarse_st.vis_fc2.0.weight": (4e-03, 6e-03),  # 1.77e-03 2.58e-03 edges_occ1
        "grad.net_coarse_st.vis_fc2.2.bias": (9e-04, 4e-03),  # 4.42e-04 1.58e-03 edges_occ1
        "grad.net_coarse_st.vis_fc2.2.weight": (7e-03, 6e-03),  # 3.11e-03 2.64e-03 edges_occ1
        "grad.trajectory_basis": (9e-04, 1e-03),  # 4.06e-04 4.99e-04 edges_occ1
        "out.anchor/mask": (1e-04, 1e-04),  # 0.00e+00 0.00e+00 edges_occ2
        "out.anchor/occ_weight_map": (1e-04, 1e-04),  # 7.52e-06 2.99e-05 shipped
        "out.anchor/occ_weights": (1e-04, 1e-04),  # 2.20e-06 1.73e-05 shipped
        "out.anchor/pts_traj_anchor": (1e-04, 1e-04),  # 2.92e-06 1.01e-05 edges_occ2 / late
        "out.anchor/pts_traj_ref": (1e-04, 1e-04),  # 1.68e-06 5.75e-06 edges_occ1 / shipped
        "out.anchor/rgb": (1e-04, 2e-04),  # 1.85e-05 6.71e-05 late
        "out.anchor/sf_seq": (2e-03, 6e-03),  # 6.27e-04 2.74e-03 edges_occ2 / late
        "out.anchor_dy/mask": (1e-04, 1e-04),  # 0.00e+00 0.00e+00 edges_occ2
        "out.anchor_dy/occ_weight_map": (1e-04, 1e-04),  # 2.52e-06 2.34e-05 edges_occ1 / edges_occ2
        "out.anchor_dy/rgb": (1e-04, 4e-04),  # 3.44e-05 1.54e-04 late
        "out.ref/depth": (2e-04, 4e-04),  # 6.30e-05 1.82e-04 shipped / late
        "out.ref/mask": (1e-04, 1e-04),  # 0.00e+00 0.00e+00 edges_occ2
        "out.ref/render_flows": (2e-04, 6e-04),  # 6.22e-05 2.54e-04 late / shipped
        "out.ref/rgb": (1e-04, 2e-04),  # 1.86e-05 6.37e-05 late
        "out.ref/rgb_dy": (1e-04, 3e-04),  # 4.94e-05 1.50e-04 late
        "out.ref/rgb_static": (1e-04, 3e-04),  # 3.31e-05 1.22e-04 shipped / late
        "out.ref/s_vals": (1e-04, 1e-04),  # 6.61e-08 1.51e-07 edges_occ1 / shipped
        "out.ref/weights": (4e-04, 5e-04),  # 1.83e-04 2.48e-04 shipped / late
        "out.ref/weights_dy": (3e-04, 5e-04),  # 1.38e-04 2.48e-04 shipped / late
        "out.ref/weights_st": (6e-04, 5e-04),  # 2.50e-04 2.48e-04 shipped / late
        "out.ref_dy/mask": (1e-04, 1e-04),  # 0.00e+00 0.00e+00 edges_occ2
        "out.ref_dy/rgb": (1e-04, 4e-04),  # 3.46e-05 1.65e-04 late
        "term.cycle_loss": (2e-04, 2e-04),  # 7.34e-05 7.34e-05 edges_occ1
        "term.disp_loss": (1e-04, 1e-04),  # 8.29e-06 8.29e-06 edges_occ1
        "term.distortion_loss": (1e-04, 1e-04),  # 1.55e-06 1.55e-06 edges_occ1
        "term.entropy_loss": (1e-04, 1e-04),  # 3.80e-07 3.80e-07 late
        "term.flow_loss": (1e-04, 1e-04),  # 2.41e-06 2.41e-06 edges_occ2
        "term.loss": (1e-04, 1e-04),  # 3.53e-06 3.53e-06 edges_occ1
        "term.reg_loss": (1e-04, 1e-04),  # 3.16e-06 3.16e-06 late
        "term.rgb_loss": (1e-04, 1e-04),  # 4.08e-06 4.08e-06 edges_occ1
        "term.static_loss": (1e-04, 1e-04),  # 2.08e-06 2.08e-06 edges_occ2
    },
    "fp32": {
        "grad.featmaps[0]": (2e-05, 3e-05),  # 7.99e-06 1.14e-05 shipped
        "grad.featmaps[1]": (2e-05, 3e-05),  # 9.95e-06 1.03e-05 shipped
        "grad.featmaps[2]": (2e-05, 3e-05),  # 9.87e-06 1.39e-05 shipped
        "grad.motion_mlp.coeff_linear.bias": (2e-05, 2e-05),  # 9.92e-06 8.04e-06 edges_occ1
        "grad.motion_mlp.coeff_linear.weight": (6e-05, 6e-05),  # 2.98e-05 2.70e-05 edges_occ1 / edges_occ2
        "grad.motion_mlp.pts_linears.0.bias": (2e-03, 2e-03),  # 6.29e-04 6.65e-04 edges_occ1
        "grad.motion_mlp.pts_linears.0.weight": (2e-03, 4e-03),  # 8.41e-04 1.66e-03 edges_occ1
        "grad.motion_mlp.pts_linears.1.bias": (2e-03, 2e-03),  # 5.21e-04 6.45e-04 edges_occ1
        "grad.motion_mlp.pts_linears.1.weight": (2e-03, 3e-03),  # 6.23e-04 1.32e-03 edges_occ1
        "grad.motion_mlp.pts_linears.2.bias": (9e-04, 2e-03),  # 4.09e-04 7.64e-04 edges_occ1
        "grad.motion_mlp.pts_linears.2.weight": (9e-04, 3e-03),  # 4.27e-04 1.00e-03 edges_occ1
        "grad.motion_mlp.pts_linears.3.bias": (7e-04, 9e-04),  # 3.21e-04 4.28e-04 edges_occ1
        "grad.motion_mlp.pts_linears.3.weight": (7e-04, 9e-04),  # 3.33e-04 4.19e-04 edges_occ1
        "grad.motion_mlp.pts_linears.4.bias": (6e-04, 8e-04),  # 2.82e-04 3.55e-04 edges_occ1
        "grad.motion_mlp.pts_linears.4.weight": (6e-04, 8e-04),  # 2.90e-04 3.91e-04 edges_occ1
        "grad.motion_mlp.pts_linears.5.bias": (6e-04, 6e-04),  # 2.57e-04 2.97e-04 edges_occ1 / edges_occ2
        "grad.motion_mlp.pts_linears.5.weight": (7e-04, 9e-04),  # 3.27e-04 4.30e-04 edges_occ1 / edges_occ2
        "grad.motion_mlp.pts_linears.6.bias": (4e-04, 5e-04),  # 1.90e-04 2.31e-04 edges_occ1 / edges_occ2
        "grad.motion_mlp.pts_linears.6.weight": (5e-04, 9e-04),  # 2.40e-04 4.25e-04 edges_occ1 / edges_occ2
        "grad.motion_mlp.pts_linears.7.bias": (3e-04, 1e-03),  # 1.41e-04 4.63e-04 edges_occ1
        "grad.motion_mlp.pts_linears.7.weight": (4e-04, 2e-03),  # 1.69e-04 6.82e-04 edges_occ1
        "grad.net_coarse_dy.base_fc.0.bias": (1e-05, 1e-05),  # 3.84e-06 3.45e-06 edges_occ2
        "grad.net_coarse_dy.base_fc.0.weight": (1e-05, 1e-05),  # 3.78e-06 4.46e-06 edges_occ2
        "grad.net_coarse_dy.base_fc.2.bias": (1e-05, 1e-05),  # 4.05e-06 3.86e-06 edges_occ2
        "grad.net_coarse_dy.base_fc.2.weight": (1e-05, 1e-05),  # 3.95e-06 4.24e-06 edges_occ2
        "grad.net_coarse_dy.geometry_fc.0.bias": (1e-05, 1e-05),  # 4.96e-06 4.00e-06 edges_occ2
        "grad.net_coarse_dy.geometry_fc.0.weight": (1e-05, 1e-05),  # 4.93e-06 4.08e-06 edges_occ2
        "grad.net_coarse_dy.geometry_fc.2.bias": (1e-05, 1e-05),  # 4.88e-06 4.90e-06 edges_occ2
        "grad.net_coarse_dy.geometry_fc.2.weight": (1e-05, 2e-05),  # 4.98e-06 5.50e-06 edges_occ2
        "grad.net_coarse_dy.out_geometry_fc.0.bias": (4e-05, 4e-05),  # 1.83e-05 1.64e-05 edges_occ2
        "grad.net_coarse_dy.out_geometry_fc.0.weight": (3e-05, 3e-05),  # 1.40e-05 1.49e-05 edges_occ2
        "grad.net_coarse_dy.out_geometry_fc.2.bias": (4e-05, 4e-05),  # 1.80e-05 1.80e-05 edges_occ2
        "grad.net_coarse_dy.out_geometry_fc.2.weight": (3e-05, 3e-05),  # 1.41e-05 1.34e-05 edges_occ2
        "grad.net_coarse_dy.ray_attention.fc.weight": (1e-05, 1e-05),  # 4.96e-06 4.80e-06 edges_occ2
        "grad.net_coarse_dy.ray_attention.layer_norm.bias": (1e-05, 1e-05),  # 4.96e-06 4.98e-06 edges_occ2
        "grad.net_coarse_dy.ray_attention.layer_norm.weight": (2e-05, 2e-05),  # 5.57e-06 5.15e-06 edges_occ2
        "grad.net_coarse_dy.ray_attention.w_ks.weight": (2e-05, 2e-05),  # 5.30e-06 6.38e-06 edges_occ2 / edges_occ1
        "grad.net_coarse_dy.ray_attention.w_qs.weight": (2e-05, 2e-05),  # 5.64e-06 8.01e-06 edges_occ2
        "grad.net_coarse_dy.ray_attention.w_vs.weight": (1e-05, 2e-05),  # 4.97e-06 6.43e-06 edges_occ2
        "grad.net_coarse_dy.ray_dir_fc.0.bias": (1e-05, 2e-05),  # 4.76e-06 5.00e-06 edges_occ2
        "grad.net_coarse_dy.ray_dir_fc.0.weight": (1e-05, 1e-05),  # 3.65e-06 3.63e-06 edges_occ2
        "grad.net_coarse_dy.ray_dir_fc.2.bias": (1e-05, 2e-05),  # 4.76e-06 5.78e-06 edges_occ2
        "grad.net_coarse_dy.ray_dir_fc.2.weight": (1e-05, 1e-05),  # 3.69e-06 4.63e-06 edges_occ2
        "grad.net_coarse_dy.ref_pts_fc.0.bias": (1e-05, 2e-05),  # 4.13e-06 7.48e-06 edges_occ2 / edges_occ1
        "grad.net_coarse_dy.ref_pts_fc.0.weight": (3e-05, 5e-05),  # 1.36e-05 2.33e-05 edges_occ1
        "grad.net_coarse_dy.ref_pts_fc.2.bias": (1e-05, 1e-05),  # 3.66e-06 3.22e-06 edges_occ2
        "grad.net_coarse_dy.ref_pts_fc.2.weight": (3e-05, 2e-05),  # 1.22e-05 9.56e-06 edges_occ1 / edges_occ2
        "grad.net_coarse_dy.rgb_fc.0.bias": (1e-05, 1e-05),  # 2.14e-06 2.39e-06 edges_occ2
        "grad.net_coarse_dy.rgb_fc.0.weight": (2e-05, 2e-05),  # 6.61e-06 5.17e-06 edges_occ1 / edges_occ2
        "grad.net_coarse_dy.rgb_fc.2.bias": (1e-05, 1e-05),  # 2.41e-06 2.27e-06 edges_occ2
        "grad.net_coarse_dy.rgb_fc.2.weight": (2e-05, 2e-05),  # 6.44e-06 5.75e-06 edges_occ1
        "grad.net_coarse_dy.rgb_fc.4.bias": (1e-05, 1e-05),  # 1.98e-06 2.37e-06 edges_occ2
        "grad.net_coarse_dy.rgb_fc.4.weight": (2e-05, 2e-05),  # 5.69e-06 5.20e-06 edges_occ1
        "grad.net_coarse_dy.vis_fc.0.bias": (1e-05, 1e-05),  # 3.96e-06 4.73e-06 edges_occ2
        "grad.net_coarse_dy.vis_fc.0.weight": (1e-05, 1e-05),  # 3.26e-06 3.24e-06 edges_occ2
        "grad.net_coarse_dy.vis_fc.2.bias": (1e-05, 1e-05),  # 4.11e-06 4.13e-06 edges_occ2
        "grad.net_coarse_dy.vis_fc.2.weight": (1e-05, 1e-05),  # 4.14e-06 4.33e-06 edges_occ2
        "grad.net_coarse_dy.vis_fc2.0.bias": (2e-05, 2e-05),  # 7.65e-06 6.54e-06 edges_occ2
        "grad.net_coarse_dy.vis_fc2.0.weight": (2e-05, 2e-05),  # 5.14e-06 6.38e-06 edges_occ2
        "grad.net_coarse_dy.vis_fc2.2.bias": (1e-05, 1e-05),  # 1.12e-07 5.48e-07 shipped
        "grad.net_coarse_dy.vis_fc2.2.weight": (2e-05, 2e-05),  # 6.09e-06 5.78e-06 edges_occ2
        "grad.net_coarse_st.base_fc.0.bias": (1e-05, 1e-05),  # 3.85e-06 3.61e-06 edges_occ2
        "grad.net_coarse_st.base_fc.0.weight": (2e-05, 2e-05),  # 5.49e-06 5.33e-06 edges_occ2
        "grad.net_coarse_st.base_fc.2.bias": (1e-05, 1e-05),  # 3.85e-06 3.86e-06 edges_occ2
        "grad.net_coarse_st.base_fc.2.weight": (2e-05, 2e-05),  # 5.27e-06 5.39e-06 edges_occ2
        "grad.net_coarse_st.geometry_fc.0.bias": (1e-05, 1e-05),  # 3.73e-06 3.82e-06 edges_occ2
        "grad.net_coarse_st.geometry_fc.0.weight": (1e-05, 2e-05),  # 4.94e-06 6.78e-06 edges_occ2
        "grad.net_coarse_st.geometry_fc.2.bias": (1e-05, 1e-05),  # 3.74e-06 3.91e-06 edges_occ2
        "grad.net_coarse_st.geometry_fc.2.weight": (1e-05, 2e-05),  # 4.51e-06 5.25e-06 edges_occ2
        "grad.net_coarse_st.out_geometry_fc.0.bias": (1e-05, 1e-05),  # 3.70e-06 3.88e-06 edges_occ2
        "grad.net_coarse_st.out_geometry_fc.0.weight": (1e-05, 1e-05),  # 4.05e-06 4.95e-06 edges_occ2
        "grad.net_coarse_st.out_geometry_fc.2.bias": (1e-05, 1e-05),  # 3.59e-06 3.59e-06 edges_occ2
        "grad.net_coarse_st.out_geometry_fc.2.weight": (1e-05, 1e-05),  # 4.18e-06 4.26e-06 edges_occ2
        "grad.net_coarse_st.ray_attention.fc.weight": (1e-05, 1e-05),  # 3.96e-06 4.82e-06 edges_occ2
        "grad.net_coarse_st.ray_attention.layer_norm.bias": (1e-05, 1e-05),  # 3.67e-06 3.73e-06 edges_occ2
        "grad.net_coarse_st.ray_attention.layer_norm.weight": (1e-05, 1e-05),  # 3.70e-06 4.05e-06 edges_occ2
        "grad.net_coarse_st.ray_attention.w_ks.weight": (2e-05, 2e-05),  # 5.11e-06 5.69e-06 edges_occ2
        "grad.net_coarse_st.ray_attention.w_qs.weight": (1e-05, 2e-05),  # 4.96e-06 5.14e-06 edges_occ2
        "grad.net_coarse_st.ray_attention.w_vs.weight": (1e-05, 1e-05),  # 4.12e-06 4.42e-06 edges_occ2
        "grad.net_coarse_st.ray_dir_fc.0.bias": (2e-05, 2e-05),  # 5.27e-06 5.32e-06 edges_occ2
        "grad.net_coarse_st.ray_dir_fc.0.weight": (2e-05, 2e-05),  # 5.81e-06 7.33e-06 edges_occ2
        "grad.net_coarse_st.ray_dir_fc.2.bias": (2e-05, 2e-05),  # 5.54e-06 6.14e-06 edges_occ2
        "grad.net_coarse_st.ray_dir_fc.2.weight": (2e-05, 2e-05),  # 5.92e-06 5.87e-06 edges_occ2
        "grad.net_coarse_st.ref_feature_fc.0.bias": (1e-05, 2e-05),  # 4.45e-06 5.89e-06 edges_occ2
        "grad.net_coarse_st.ref_feature_fc.0.weight": (2e-05, 2e-05),  # 5.07e-06 5.40e-06 edges_occ2
        "grad.net_coarse_st.rgb_fc.0.bias": (1e-05, 2e-05),  # 1.70e-06 5.59e-06 shipped
        "grad.net_coarse_st.rgb_fc.0.weight": (2e-04, 2e-04),  # 5.61e-05 9.98e-05 shipped
        "grad.net_coarse_st.rgb_fc.2.bias": (1e-05, 4e-05),  # 2.14e-06 1.73e-05 shipped
        "grad.net_coarse_st.rgb_fc.2.weight": (2e-04, 1e-04),  # 5.61e-05 4.67e-05 shipped
        "grad.net_coarse_st.rgb_fc.4.bias": (1e-05, 2e-05),  # 2.57e-06 7.92e-06 shipped
        "grad.net_coarse_st.rgb_fc.4.weight": (2e-04, 9e-05),  # 5.40e-05 4.49e-05 shipped
        "grad.net_coarse_st.s": (2e-04, 2e-04),  # 7.20e-05 7.20e-05 edges_occ1
        "grad.net_coarse_st.vis_fc.0.bias": (1e-05, 1e-05),  # 3.84e-06 3.94e-06 edges_occ2
        "grad.net_coarse_st.vis_fc.0.weight": (1e-05, 2e-05),  # 4.74e-06 5.78e-06 edges_occ2
        "grad.net_coarse_st.vis_fc.2.bias": (1e-05, 1e-05),  # 3.78e-06 4.05e-06 edges_occ2
        "grad.net_coarse_st.vis_fc.2.weight": (1e-05, 1e-05),  # 3.85e-06 4.10e-06 edges_occ2
        "grad.net_coarse_st.vis_fc2.0.bias": (2e-05, 2e-05),  # 9.06e-06 7.92e-06 edges_occ2
        "grad.net_coarse_st.vis_fc2.0.weight": (1e-05, 1e-05),  # 3.26e-06 4.28e-06 edges_occ2
        "grad.net_coarse_st.vis_fc2.2.bias": (1e-05, 1e-05),  # 3.35e-07 1.32e-06 edges_occ2
        "grad.net_coarse_st.vis_fc2.2.weight": (1e-05, 1e-05),  # 3.38e-06 2.82e-06 edges_occ2
        "grad.trajectory_basis": (7e-05, 7e-05),  # 3.36e-05 3.49e-05 edges_occ1
        "out.anchor/mask": (1e-05, 1e-05),  # 0.00e+00 0.00e+00 edges_occ2
        "out.anchor/occ_weight_map": (1e-05, 1e-05),  # 1.28e-07 4.77e-07 edges_occ2
        "out.anchor/occ_weights": (1e-05, 1e-05),  # 2.70e-08 1.76e-07 edges_occ2
        "out.anchor/pts_traj_anchor": (1e-05, 1e-05),  # 6.30e-07 8.60e-07 shipped
        "out.anchor/pts_traj_ref": (1e-05, 1e-05),  # 6.29e-07 8.60e-07 shipped
        "out.anchor/rgb": (1e-05, 1e-05),  # 4.28e-07 2.13e-06 shipped
        "out.anchor/sf_seq": (1e-05, 3e-05),  # 3.94e-06 1.05e-05 edges_occ2 / shipped
        "out.anchor_dy/mask": (1e-05, 1e-05),  # 0.00e+00 0.00e+00 edges_occ2
        "out.anchor_dy/occ_weight_map": (1e-05, 1e-05),  # 1.15e-07 3.58e-07 edges_occ2 / shipped
        "out.anchor_dy/rgb": (1e-05, 1e-05),  # 2.06e-07 5.67e-07 edges_occ2 / shipped
        "out.ref/depth": (1e-05, 1e-05),  # 1.37e-06 1.71e-06 edges_occ1
        "out.ref/mask": (1e-05, 1e-05),  # 0.00e+00 0.00e+00 edges_occ2
        "out.ref/render_flows": (1e-05, 1e-05),  # 1.77e-06 4.46e-06 shipped
        "out.ref/rgb": (1e-05, 1e-05),  # 4.28e-07 2.04e-06 shipped
        "out.ref/rgb_dy": (1e-05, 1e-05),  # 2.77e-07 6.01e-07 edges_occ2 / edges_occ1
        "out.ref/rgb_static": (1e-05, 1e-05),  # 8.41e-07 4.07e-06 shipped
        "out.ref/s_vals": (1e-05, 1e-05),  # 6.61e-08 1.51e-07 edges_occ1 / shipped
        "out.ref/weights": (1e-05, 1e-05),  # 1.26e-06 1.50e-06 edges_occ1
        "out.ref/weights_dy": (1e-05, 1e-05),  # 1.43e-06 1.83e-06 edges_occ1
        "out.ref/weights_st": (1e-05, 1e-05),  # 1.47e-06 1.50e-06 edges_occ1
        "out.ref_dy/mask": (1e-05, 1e-05),  # 0.00e+00 0.00e+00 edges_occ2
        "out.ref_dy/rgb": (1e-05, 1e-05),  # 1.97e-07 5.87e-07 edges_occ2 / shipped
        "term.cycle_loss": (1e-05, 1e-05),  # 8.45e-07 8.45e-07 edges_occ1
        "term.disp_loss": (1e-05, 1e-05),  # 7.27e-07 7.27e-07 edges_occ1
        "term.distortion_loss": (1e-05, 1e-05),  # 2.81e-07 2.81e-07 edges_occ2
        "term.entropy_loss": (1e-05, 1e-05),  # 2.87e-07 2.87e-07 shipped
        "term.flow_loss": (1e-05, 1e-05),  # 7.54e-07 7.54e-07 shipped
        "term.loss": (1e-05, 1e-05),  # 1.98e-07 1.98e-07 shipped
        "term.reg_loss": (1e-05, 1e-05),  # 1.05e-07 1.05e-07 shipped
        "term.rgb_loss": (1e-05, 1e-05),  # 1.27e-07 1.27e-07 edges_occ2
        "term.static_loss": (1e-05, 1e-05),  # 2.40e-07 2.40e-07 shipped
    },
}


def bar(prec, name):
  return BARS[prec][name]


def ratios(errs, prec):
  return {k: max(r / bar(prec, k)[0], m / bar(prec, k)[1]) for k, (r, m) in errs.items()}


def run(case, prec):
  """Library step, then (its tensors freed) the reference -> (errors, stats)."""
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
  ref = T.reference(c, DEV, MODE[prec], chunk=c["chunk"])
  torch.cuda.synchronize()
  stats.update(reference_s=time.perf_counter() - t0, reference_peak_GB=torch.cuda.max_memory_allocated() / 2 ** 30)
  errs = T.errors(got, ref, c["V_st"])
  del ref
  torch.cuda.empty_cache()
  return errs, stats


@pytest.mark.parametrize("case,prec", RUNS)
def test_training_step_matches_reference(case, prec):
  errs, stats = run(case, prec)
  r = ratios(errs, prec)
  worst = max(r.items(), key=lambda kv: kv[1])
  print("\nstep %s %s: worst %s, %.2f of its bar; %s" % (case, prec, worst[0], worst[1],
                                                         ", ".join("%s %.2f" % kv for kv in stats.items())))
  for name, (rel, mx) in sorted(errs.items()):
    print("  ERR %s %s %s %.3e %.3e" % (case, prec, name, rel, mx))
  bad = {k: (errs[k], bar(prec, k)) for k, v in r.items() if not v <= 1.0}
  assert not bad, (case, prec, bad)


def plant_margins():
  """{plant: (the compared tensor it moves most, relative to its bf16 bar; that ratio)} on edges_occ1."""
  c = T.make_case("edges_occ1")
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
