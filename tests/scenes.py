"""Seeded scene/model configurations shared by the golden generator and tests."""

import zlib

import torch

from dynibar_b200 import synthetic

# name -> config.  Small enough that the reference finishes in seconds on CPU.
GOLDEN_CONFIGS = {
    # render_rays_mv: coarse + fine, 7 dynamic + 5 static views, masks stressed
    "mv_small": dict(mono=False, H=48, W=64, V_dy=7, V_st=5, rays=40,
                     N_samples=16, N_importance=16, num_vv=0, inv_uniform=True,
                     anti_alias_pooling=1, mask_rgb=0, seed=11, stress=True),
    # same path, linear-depth sampling, no anti-alias pooling, mask_rgb on
    "mv_linear": dict(mono=False, H=40, W=56, V_dy=7, V_st=4, rays=24,
                      N_samples=20, N_importance=12, num_vv=0, inv_uniform=False,
                      anti_alias_pooling=0, mask_rgb=1, seed=12, stress=False),
    # render_rays_mono (BASELINE config 1 shape scaled): 32 samples,
    # 6 temporal + 2 virtual dynamic views, 4 static views, shift=5
    "mono_small": dict(mono=True, H=36, W=64, V_dy=8, V_st=4, rays=24,
                       N_samples=32, N_importance=0, num_vv=2, inv_uniform=True,
                       anti_alias_pooling=1, mask_rgb=1, seed=13, stress=True),
    # render_rays_mono(is_train=True): reference-time + cross-time (anchor) branch, row a16
    "mono_train": dict(mono=True, H=36, W=64, V_dy=8, V_st=4, rays=20,
                       N_samples=32, N_importance=0, num_vv=2, inv_uniform=True,
                       anti_alias_pooling=1, mask_rgb=1, seed=14, stress=False,
                       anchor_offset=2, occ_weights_mode=0),
    # same branch with the anchor one frame away: occ_weights_mode 0 then takes the "full" disocclusion
    # score (render_ray.py:1233-1242), the other arm of the mode switch
    "mono_train_near": dict(mono=True, H=36, W=64, V_dy=8, V_st=4, rays=16,
                            N_samples=32, N_importance=0, num_vv=2, inv_uniform=True,
                            anti_alias_pooling=1, mask_rgb=1, seed=15, stress=False,
                            anchor_offset=-1, occ_weights_mode=0),
}


def build(cfg, sigma_bias=-4.0):
  batch, feat_c, feat_f, frame, t, offs = synthetic.make_scene(
      H=cfg["H"], W=cfg["W"], V_dy=cfg["V_dy"], V_st=cfg["V_st"],
      num_vv=cfg["num_vv"], seed=cfg["seed"], rays=cfg["rays"],
      stress=cfg.get("stress", False), anchor_offset=cfg.get("anchor_offset"))
  args = synthetic.make_args(cfg["anti_alias_pooling"], cfg["mask_rgb"],
                             cfg.get("occ_weights_mode", 0))
  model, args = synthetic.make_model(cfg["N_samples"], cfg["N_importance"],
                                     args=args, seed=cfg["seed"],
                                     mono=cfg["mono"], sigma_bias=sigma_bias)
  return batch, feat_c, feat_f, frame, t, offs, model, args


# ---- frame-level fixtures (tests/golden/make_golden_frame.py) ----------------------------------
FRAME_CONFIGS = {
    # render_single_image_nvi (render_image.py:9-217): a whole 12x16 frame in chunks of 50 rays
    "frame_nvi": dict(GOLDEN_CONFIGS["mv_small"], H=12, W=16, rays=None, chunk=50),
    # render_single_image_mono (render_image.py:220-439), is_train=True (cross-time branch included)
    "frame_mono": dict(GOLDEN_CONFIGS["mono_train"], H=12, W=16, rays=None, chunk=70),
}
# occlusion-weight modes 1 and 2 of the cross-time branch (render_ray.py:1243-1252)
OCC_MODE_CONFIGS = {
    "occ_mode1": dict(GOLDEN_CONFIGS["mono_train"], rays=12, occ_weights_mode=1),
    "occ_mode2": dict(GOLDEN_CONFIGS["mono_train"], rays=12, occ_weights_mode=2),
}


def sampler_data(batch, H, W, seed, n_flow=6):
  """The per-frame `data` dict a dataset hands to RaySamplerSingleImage (sample_ray.py:50-141):
  cameras and source views from the scene + seeded per-pixel supervision."""
  g = torch.Generator().manual_seed(seed + 500)
  data = {k: batch[k] for k in ("camera", "depth_range", "src_rgbs", "src_cameras", "static_src_rgbs",
                                "static_src_cameras")}
  for k in ("anchor_camera", "anchor_src_rgbs", "anchor_src_cameras"):
    if k in batch:
      data[k] = batch[k]
  data["rgb_path"] = "synthetic"
  data["rgb"] = torch.rand(1, H, W, 3, generator=g)
  data["disp"] = torch.rand(1, H, W, generator=g)
  data["motion_mask"] = (torch.rand(1, H, W, generator=g) > 0.5).float()
  data["static_mask"] = 1.0 - data["motion_mask"]
  data["flows"] = torch.randn(1, n_flow, H, W, 2, generator=g)
  data["masks"] = (torch.rand(1, n_flow, H, W, generator=g) > 0.3).float()
  return data


def encoder_weights(m, seed):
  """Seeded parameters for a 2-D encoder of the reference's ResNet layout (this repository's or the reference's own
  module): each parameter is drawn from a generator of its own (seed, name), so both get the same values."""
  with torch.no_grad():
    for name, p in m.named_parameters():
      g = torch.Generator().manual_seed(seed * 1000003 + zlib.crc32(name.encode()))
      if name.endswith("bn1.weight") or name.endswith("bn2.weight") or name.endswith("downsample.1.weight"):
        p.copy_(torch.rand(p.shape, generator=g) + 0.5)
      elif name.endswith(".bias"):
        p.copy_(torch.rand(p.shape, generator=g) * 0.6 - 0.3)
      else:
        p.copy_(torch.randn(p.shape, generator=g) * (2.0 / p[0].numel()) ** 0.5)
  return m.requires_grad_(False)
