"""Full-frame driver: drop-in for ibrnet/render_image.py
(`render_single_image_nvi` :9-217, `render_single_image_mono` :220-439).

Same signatures and the same returned structure (an OrderedDict of per-output
OrderedDicts whose tensors live on the CPU, reshaped to [H, W, ...]; `rgb` is
zeroed where the ray `mask` is 0, render_image.py:161-163).  Unlike the
reference, chunks are merged ON THE DEVICE and copied to the host once per
frame (the reference issues one blocking `.cpu()` per output per chunk,
render_image.py:123-135, which drains the GPU 18 x 11 times per frame).
`render_multi_image_nvi` renders the target cameras of one time step together (one stacked ray batch,
sample_ray.stack_ray_batches) and returns one such result per camera; `render_multi_image_mono` does the same
for a monocular scene, where every camera has its own source views drawn from shared pools
(sample_ray.stack_pooled_ray_batches).
"""

from collections import OrderedDict

import torch

from dynibar_b200.render_ray import _with_host_copies, camera_count, is_pooled, render_rays_mono, render_rays_mv

_SHARED_KEYS = ("camera", "anchor_camera", "depth_range", "src_rgbs", "src_cameras",
                "anchor_src_rgbs", "anchor_src_cameras", "static_src_rgbs", "static_src_cameras",
                "src_views", "static_src_views")


def _chunk(ray_batch, i, chunk_size):
  """Per-chunk view of the ray batch (render_image.py:69-89)."""
  out = OrderedDict()
  for k, v in ray_batch.items():
    if v is None or k in _SHARED_KEYS or not torch.is_tensor(v):
      out[k] = v
    elif v.dim() == 3:  # flows / masks: [n_views, n_rays, c]
      out[k] = v[:, i:i + chunk_size, ...]
    else:
      out[k] = v[i:i + chunk_size]
  return out


def _merge(chunks, H, W):
  """list of per-chunk dicts -> one dict of CPU tensors shaped like the
  reference's (render_image.py:141-163)."""
  merged = OrderedDict()
  if not chunks:
    return merged
  for k in chunks[0]:
    parts = [c[k] for c in chunks]
    if parts[0].dim() == 4:  # left as the list of chunks by the reference
      merged[k] = [p.cpu() for p in parts]
      continue
    if parts[0].dim() == 3:
      t = torch.cat(parts, dim=1).reshape(parts[0].shape[0], H, W, -1)
    else:
      t = torch.cat(parts, dim=0).reshape(H, W, -1)
    merged[k] = t.squeeze()
  if "rgb" in merged and "mask" in merged:
    merged["rgb"] = merged["rgb"].masked_fill((merged["mask"] == 0)[..., None], 0.0)
  return OrderedDict((k, (v if isinstance(v, list) else v.cpu())) for k, v in merged.items())


def _merge_multi(chunks, counts, hws):
  """list of per-chunk dicts over the rays of K target cameras (chunks may straddle cameras) -> K dicts, each
  shaped like `_merge`'s for that camera.  Chunks are concatenated on the device and each output is copied to
  the host once for all cameras."""
  merged = [OrderedDict() for _ in counts]
  if not chunks:
    return merged
  for k in chunks[0]:
    parts = [c[k] for c in chunks]
    assert parts[0].dim() <= 3, k  # render_rays_mv returns [R, ...] and [n, R, c] outputs only
    ax = 1 if parts[0].dim() == 3 else 0
    full = torch.cat(parts, dim=ax).cpu()
    for m, piece, (H, W) in zip(merged, full.split(counts, dim=ax), hws):
      t = piece.reshape(piece.shape[0], H, W, -1) if ax else piece.reshape(H, W, -1)
      m[k] = t.squeeze()
  for m in merged:
    if "rgb" in m and "mask" in m:
      m["rgb"] = m["rgb"].masked_fill((m["mask"] == 0)[..., None], 0.0)
  return merged


def _frame_hw(ray_sampler, render_stride):
  H = len(range(0, ray_sampler.H, render_stride))
  W = len(range(0, ray_sampler.W, render_stride))
  return H, W


def render_single_image_nvi(frame_idx, time_embedding, time_offset, ray_sampler, ray_batch, model,
                            projector, chunk_size, N_samples, args, inv_uniform=False, N_importance=0,
                            det=False, white_bkgd=False, render_stride=1, coarse_featmaps=None,
                            fine_featmaps=None, is_train=True):
  """Render a target view for the Nvidia dataset (render_image.py:9-217)."""
  N_rays = ray_batch["ray_o"].shape[0]
  coarse, fine = [], []
  for i in range(0, N_rays, chunk_size):
    ret = render_rays_mv(frame_idx=frame_idx, time_embedding=time_embedding, time_offset=time_offset,
                         ray_batch=_chunk(ray_batch, i, chunk_size), model=model,
                         coarse_featmaps=coarse_featmaps, fine_featmaps=fine_featmaps,
                         projector=projector, N_samples=N_samples, args=args, inv_uniform=inv_uniform,
                         N_importance=N_importance, raw_noise_std=0.0, det=det, white_bkgd=white_bkgd,
                         is_train=is_train)
    coarse.append(ret["outputs_coarse_ref"])
    fine.append(ret["outputs_fine_ref"])
  H, W = _frame_hw(ray_sampler, render_stride)
  all_ret = OrderedDict([("outputs_fine_anchor", OrderedDict()),
                         ("outputs_fine_ref", _merge(fine, H, W)),
                         ("outputs_coarse_ref", _merge(coarse, H, W))])
  all_ret["outputs_fine"] = None
  return all_ret


def render_multi_image_nvi(frame_idx, time_embedding, time_offset, ray_samplers, ray_batch, model,
                           projector, chunk_size, N_samples, args, inv_uniform=False, N_importance=0,
                           det=False, white_bkgd=False, render_stride=1, coarse_featmaps=None,
                           fine_featmaps=None, is_train=True):
  """Render the K target views of ONE time step of the Nvidia dataset in one pass over their rays.

  Same arguments as `render_single_image_nvi`, except `ray_samplers` (the K RaySamplerSingleImage of the
  time step, in order) and `ray_batch` (their get_all() batches stacked by sample_ray.stack_ray_batches).
  Returns a list of K OrderedDicts, each shaped exactly like render_single_image_nvi's result for that camera.
  The per-frame work (host copies of cameras and depth range, packing the source views) runs once for all K
  cameras, and chunks of `chunk_size` rays run across camera boundaries."""
  K = camera_count(ray_batch)
  if len(ray_samplers) != K:
    raise ValueError("render_multi_image_nvi: %d ray samplers for %d target cameras" % (len(ray_samplers), K))
  hws = [_frame_hw(s, render_stride) for s in ray_samplers]
  counts = [H * W for H, W in hws]
  N_rays = ray_batch["ray_o"].shape[0]
  if sum(counts) != N_rays:
    raise ValueError("render_multi_image_nvi: the samplers' frames hold %d rays, the batch %d" % (sum(counts), N_rays))
  _check_camera_index(ray_batch, K, N_rays, "render_multi_image_nvi")
  rb, _ = _with_host_copies(ray_batch, model, ())
  coarse, fine = [], []
  for i in range(0, N_rays, chunk_size):
    ret = render_rays_mv(frame_idx=frame_idx, time_embedding=time_embedding, time_offset=time_offset,
                         ray_batch=_chunk(rb, i, chunk_size), model=model,
                         coarse_featmaps=coarse_featmaps, fine_featmaps=fine_featmaps,
                         projector=projector, N_samples=N_samples, args=args, inv_uniform=inv_uniform,
                         N_importance=N_importance, raw_noise_std=0.0, det=det, white_bkgd=white_bkgd,
                         is_train=is_train)
    coarse.append(ret["outputs_coarse_ref"])
    fine.append(ret["outputs_fine_ref"])
  out = []
  for f, c in zip(_merge_multi(fine, counts, hws), _merge_multi(coarse, counts, hws)):
    all_ret = OrderedDict([("outputs_fine_anchor", OrderedDict()), ("outputs_fine_ref", f),
                           ("outputs_coarse_ref", c)])
    all_ret["outputs_fine"] = None
    out.append(all_ret)
  return out


def _check_camera_index(ray_batch, K, N_rays, what):
  ci = ray_batch.get("camera_index")
  if ci is not None and N_rays > 0:
    lo, hi = torch.stack(torch.aminmax(ci)).tolist()  # the kernels trust the index: one check per frame
    if lo < 0 or hi >= K:
      raise ValueError("%s: camera_index spans [%d, %d], the batch has %d cameras" % (what, lo, hi, K))


def render_single_image_mono(frame_idx, time_embedding, time_offset, ray_sampler, ray_batch, model,
                             projector, chunk_size, N_samples, args, inv_uniform=False, N_importance=0,
                             det=False, white_bkgd=False, render_stride=1, featmaps=None, is_train=True,
                             num_vv=2):
  """Render a target view for monocular video (render_image.py:220-439)."""
  N_rays = ray_batch["ray_o"].shape[0]
  ref, st, anchor = [], [], []
  for i in range(0, N_rays, chunk_size):
    ret = render_rays_mono(frame_idx=frame_idx, time_embedding=time_embedding, time_offset=time_offset,
                           ray_batch=_chunk(ray_batch, i, chunk_size), model=model, featmaps=featmaps,
                           projector=projector, N_samples=N_samples, args=args, inv_uniform=inv_uniform,
                           N_importance=N_importance, raw_noise_std=0.0, det=det, white_bkgd=white_bkgd,
                           is_train=is_train, num_vv=num_vv)
    ref.append(ret["outputs_coarse_ref"])
    st.append(ret["outputs_coarse_st"])
    if is_train:
      anchor.append(ret["outputs_coarse_anchor"])
  H, W = _frame_hw(ray_sampler, render_stride)
  all_ret = OrderedDict([("outputs_coarse_ref", _merge(ref, H, W)),
                         ("outputs_coarse_st", _merge(st, H, W)),
                         ("outputs_coarse_anchor", _merge(anchor, H, W))])
  all_ret["outputs_fine"] = None
  return all_ret


def render_multi_image_mono(frame_idx, time_embedding, time_offset, ray_samplers, ray_batch, model,
                            projector, chunk_size, N_samples, args, inv_uniform=False, N_importance=0,
                            det=False, white_bkgd=False, render_stride=1, featmaps=None, is_train=False,
                            num_vv=2):
  """Render K target views of ONE time step of a monocular video in one pass over their rays (a bullet-time
  sweep: dynibar_b200/bullet_time.py), each camera with its own source views drawn from shared pools.

  Same arguments as `render_single_image_mono`, except `ray_samplers` (the K RaySamplerSingleImage, in order) and
  `ray_batch` (their get_all() batches pooled by sample_ray.stack_pooled_ray_batches); `featmaps` are the pools'
  feature maps, (dynamic pool, None, static pool).  Rendering only: is_train must be False and no gradient is
  taken.  Returns a list of K OrderedDicts, each shaped exactly like render_single_image_mono's result for that
  camera (an empty outputs_coarse_anchor).  The per-frame work (host copies of cameras, packing the pools) runs
  once for all K cameras, and chunks of `chunk_size` rays run across camera boundaries."""
  if is_train:
    raise NotImplementedError("render_multi_image_mono renders only (is_train=False): the cross-time branch and "
                              "training take one target camera per call")
  if not is_pooled(ray_batch):
    raise ValueError("render_multi_image_mono: the batch has no view tables (sample_ray.stack_pooled_ray_batches)")
  K = camera_count(ray_batch)
  if len(ray_samplers) != K:
    raise ValueError("render_multi_image_mono: %d ray samplers for %d target cameras" % (len(ray_samplers), K))
  hws = [_frame_hw(s, render_stride) for s in ray_samplers]
  counts = [H * W for H, W in hws]
  N_rays = ray_batch["ray_o"].shape[0]
  if sum(counts) != N_rays:
    raise ValueError("render_multi_image_mono: the samplers' frames hold %d rays, the batch %d" % (sum(counts), N_rays))
  _check_camera_index(ray_batch, K, N_rays, "render_multi_image_mono")
  rb, _ = _with_host_copies(ray_batch, model, ())
  for key, pool_key in (("src_views", "src_cameras"), ("static_src_views", "static_src_cameras")):
    tbl = rb[key].detach().to("cpu", torch.int32).contiguous()  # one host copy per call; the kernels read it so
    pool = rb[pool_key].shape[1]
    if tbl.dim() != 2 or tbl.shape[0] != K:
      raise ValueError("render_multi_image_mono: %s is %s, expected [%d, slots]" % (key, tuple(tbl.shape), K))
    if tbl.numel() and (int(tbl.min()) < 0 or int(tbl.max()) >= pool):
      raise ValueError("render_multi_image_mono: %s spans [%d, %d], the pool has %d views"
                       % (key, int(tbl.min()), int(tbl.max()), pool))
    rb[key] = tbl
  ref, st = [], []
  for i in range(0, N_rays, chunk_size):
    ret = render_rays_mono(frame_idx=frame_idx, time_embedding=time_embedding, time_offset=time_offset,
                           ray_batch=_chunk(rb, i, chunk_size), model=model, featmaps=featmaps,
                           projector=projector, N_samples=N_samples, args=args, inv_uniform=inv_uniform,
                           N_importance=N_importance, raw_noise_std=0.0, det=det, white_bkgd=white_bkgd,
                           is_train=False, num_vv=num_vv)
    ref.append(ret["outputs_coarse_ref"])
    st.append(ret["outputs_coarse_st"])
  out = []
  for r, s_ in zip(_merge_multi(ref, counts, hws), _merge_multi(st, counts, hws)):
    all_ret = OrderedDict([("outputs_coarse_ref", r), ("outputs_coarse_st", s_),
                           ("outputs_coarse_anchor", OrderedDict())])
    all_ret["outputs_fine"] = None
    out.append(all_ret)
  return out
