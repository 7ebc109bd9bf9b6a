"""Target-view ray bundles: host-side mirror of `RaySamplerSingleImage`
(ibrnet/sample_ray.py:19-331), kornia-free.

Like the reference, per-pixel rays are built once per frame on the host
(sample_ray.py:143-163) and moved to the device by `get_all` /
`random_sample`; this is frame set-up, not the per-ray hot loop.  The
dictionaries returned have the reference's keys (SURVEY.md 8b `ray_batch`).
"""

import numpy as np
import torch

# Same seeded generator the reference uses for training pixel selection
# (sample_ray.py:8) so `random_sample` draws identical pixels.
rng = np.random.RandomState(234)

_PER_RAY_KEYS_2D = ("rgb", "disp", "motion_mask", "static_mask")


def parse_camera(params):
  """[B,34] -> W, H, K[B,4,4], c2w[B,4,4] (sample_ray.py:11-16)."""
  return (params[:, 1], params[:, 0], params[:, 2:18].reshape(-1, 4, 4),
          params[:, 18:34].reshape(-1, 4, 4))


def pixel_rays(H, W, K, c2w, stride=1):
  """ray_d = R_c2w K^-1 [u,v,1]^T at integer pixel coordinates (no +0.5),
  ray_o = t_c2w; uv in (x, y) order (sample_ray.py:83-87, :143-163)."""
  us = torch.arange(0, W, stride, dtype=torch.float32)
  vs = torch.arange(0, H, stride, dtype=torch.float32)
  v, u = torch.meshgrid(vs, us, indexing="ij")
  u, v = u.reshape(-1), v.reshape(-1)
  pix = torch.stack([u, v, torch.ones_like(u)], 0)
  M = c2w[:3, :3].float() @ torch.inverse(K[:3, :3].float())
  ray_d = (M @ pix).t().contiguous()
  ray_o = c2w[:3, 3].float()[None].repeat(ray_d.shape[0], 1)
  return ray_o, ray_d, torch.stack([u, v], -1)


class RaySamplerSingleImage(object):
  """Drop-in for ibrnet.sample_ray.RaySamplerSingleImage (same constructor,
  `get_all`, `sample_random_pixel`, `random_sample`)."""

  _passthrough = ("src_rgbs", "src_cameras", "anchor_src_rgbs",
                  "anchor_src_cameras", "static_src_rgbs",
                  "static_src_cameras", "static_src_masks")

  def __init__(self, data, device, resize_factor=1, render_stride=1):
    self.render_stride = render_stride
    self.device = device
    g = data.get
    self.rgb, self.disp = g("rgb"), g("disp")
    self.motion_mask, self.static_mask = g("motion_mask"), g("static_mask")
    self.flows = data["flows"].squeeze(0) if "flows" in data else None
    self.masks = data["masks"].squeeze(0) if "masks" in data else None
    self.camera = data["camera"]
    self.render_camera = g("render_camera")
    self.anchor_camera = g("anchor_camera")
    self.rgb_path = g("rgb_path")
    self.depth_range = data["depth_range"]
    W, H, self.intrinsics, self.c2w_mat = parse_camera(self.camera)
    self.batch_size = len(self.camera)
    assert self.batch_size == 1, "only batch_size=1 (projection.py:122-126)"
    self.H, self.W = int(H[0]), int(W[0])
    self.rays_o, self.rays_d, uv = pixel_rays(
        self.H, self.W, self.intrinsics[0], self.c2w_mat[0], render_stride)
    # The reference's uv_grid is the un-strided full-resolution grid
    # (sample_ray.py:83-87,109).
    if render_stride == 1:
      self.uv_grid = uv
    else:
      _, _, self.uv_grid = pixel_rays(self.H, self.W, self.intrinsics[0],
                                      self.c2w_mat[0], 1)
    if self.rgb is not None:
      self.rgb = self.rgb.reshape(-1, 3)
    for k in ("disp", "motion_mask", "static_mask"):
      v = getattr(self, k)
      if v is not None:
        setattr(self, k, v.reshape(-1, 1))
    if self.flows is not None:
      self.flows = self.flows.reshape(self.flows.shape[0], -1, 2)
      self.masks = self.masks.reshape(self.masks.shape[0], -1, 1)
    for k in self._passthrough:
      setattr(self, k, g(k))

  def _dev(self, x):
    return x.to(self.device, non_blocking=True) if x is not None else None

  def get_all(self):
    """All rays of the target view (sample_ray.py:165-235)."""
    sq = lambda x: self._dev(x).squeeze() if x is not None else None
    ret = {
        "ray_o": self._dev(self.rays_o), "ray_d": self._dev(self.rays_d),
        "depth_range": self._dev(self.depth_range),
        "camera": self._dev(self.camera),
        "render_camera": self._dev(self.render_camera),
        "anchor_camera": self._dev(self.anchor_camera),
        "rgb": self._dev(self.rgb),
        "disp": sq(self.disp), "motion_mask": sq(self.motion_mask),
        "static_mask": sq(self.static_mask),
        "uv_grid": self._dev(self.uv_grid),
        "flows": self._dev(self.flows), "masks": self._dev(self.masks),
    }
    for k in self._passthrough:
      ret[k] = self._dev(getattr(self, k))
    return ret

  def sample_random_pixel(self, N_rand, sample_mode, center_ratio=0.8):
    """sample_ray.py:237-260 (same RandomState stream)."""
    if sample_mode == "center":
      bH = int(self.H * (1 - center_ratio) / 2.0)
      bW = int(self.W * (1 - center_ratio) / 2.0)
      u, v = np.meshgrid(np.arange(bH, self.H - bH), np.arange(bW, self.W - bW))
      u, v = u.reshape(-1), v.reshape(-1)
      sel = rng.choice(u.shape[0], size=(N_rand,), replace=False)
      return v[sel] + self.W * u[sel]
    if sample_mode == "uniform":
      return rng.choice(self.H * self.W, size=(N_rand,), replace=False)
    raise NotImplementedError

  def random_sample(self, N_rand, sample_mode, center_ratio=0.8):
    """N_rand training rays + their supervision (sample_ray.py:262-331)."""
    if self.rgb is None:
      raise NotImplementedError
    sel = self.sample_random_pixel(N_rand, sample_mode, center_ratio)
    ret = {
        "ray_o": self._dev(self.rays_o[sel]), "ray_d": self._dev(self.rays_d[sel]),
        "camera": self._dev(self.camera),
        "anchor_camera": self._dev(self.anchor_camera),
        "depth_range": self._dev(self.depth_range),
        "rgb": self._dev(self.rgb[sel]),
        "disp": self._dev(self.disp[sel].squeeze()),
        "motion_mask": self._dev(self.motion_mask[sel].squeeze()),
        "static_mask": self._dev(self.static_mask[sel].squeeze()),
        "uv_grid": self._dev(self.uv_grid[sel]),
        "flows": self._dev(self.flows[:, sel, :]),
        "masks": self._dev(self.masks[:, sel, :]),
        "selected_inds": sel,
    }
    for k in self._passthrough:
      ret[k] = self._dev(getattr(self, k))
    return ret


# what the target cameras of one time step share (eval_nvidia.py:305-378: DynamicVideoDataset builds the
# source views from render_idx only)
_FRAME_KEYS = ("src_cameras", "static_src_cameras", "depth_range", "src_rgbs", "static_src_rgbs")
_RAY_KEYS = ("ray_o", "ray_d", "uv_grid", "rgb", "disp", "motion_mask", "static_mask")
_CAMERA_KEYS = ("camera", "render_camera", "anchor_camera")


def _same(a, b):
  if a is b:
    return True
  if a is None or b is None:
    return False
  return a.shape == b.shape and a.device == b.device and torch.equal(a, b)


def _stack(batches, k, dim):
  vals = [b.get(k) for b in batches]
  if all(v is None for v in vals):
    return None
  if any(v is None for v in vals):
    raise ValueError("stack_ray_batches: '%s' is missing from some of the batches" % k)
  return torch.cat(vals, dim)


def stack_ray_batches(batches):
  """K `get_all()` batches of the target cameras of ONE time step -> (multi-camera batch, per-camera ray
  counts, (H, W) of the target images).

  The multi-camera batch is an ordinary ray batch whose `camera` is [K,34] and whose per-ray tensors are the
  K batches' concatenated in order; `camera_index` (int32 [R], on the rays' device) names each ray's row of
  `camera`.  Per-frame tensors (source views, depth range) are shared: they must be the same in every batch
  (same tensor or equal values), otherwise ValueError.  render_image.render_multi_image_nvi renders it and
  splits the outputs back with the counts."""
  K = len(batches)
  if not 1 <= K <= 16:
    raise ValueError("stack_ray_batches: %d batches, 1..16 target cameras per batch" % K)
  first = batches[0]
  for i, b in enumerate(batches[1:], 1):
    for k in _FRAME_KEYS:
      if not _same(first.get(k), b.get(k)):
        raise ValueError("stack_ray_batches: batch %d does not share '%s' with batch 0 (the target cameras "
                         "of one time step see the same source views and depth range)" % (i, k))
  cams = [b["camera"] for b in batches]
  if any(c.dim() != 2 or c.shape[0] != 1 for c in cams):
    raise ValueError("stack_ray_batches: every batch has one target camera [1,34]")
  hw = {(int(c[0, 0]), int(c[0, 1])) for c in cams}
  if len(hw) != 1:
    raise ValueError("stack_ray_batches: the target cameras have different image sizes %s" % sorted(hw))
  out = dict(first)
  for k in _CAMERA_KEYS + _RAY_KEYS:
    if k in first:
      out[k] = _stack(batches, k, 0)
  for k in ("flows", "masks"):  # [n_views, R, c]
    if k in first:
      out[k] = _stack(batches, k, 1)
  counts = [b["ray_o"].shape[0] for b in batches]
  dev = first["ray_o"].device
  out["camera_index"] = torch.repeat_interleave(torch.arange(K, dtype=torch.int32),
                                                torch.tensor(counts)).to(dev)
  return out, counts, hw.pop()
