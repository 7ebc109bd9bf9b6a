"""A monocular bullet-time sweep from a scene resident on the device: the front end of the reference's
render_monocular_bt.py (its DynamicVideoDataset under a DataLoader, RaySamplerSingleImage.get_all and the uint8
output frames) without imageio, and without decoding any file after the scene is loaded.

  scene = BulletTimeScene(scene_path, args, device)      # reads <scene_path> (the reference's `dense` folder) once
  for cameras, frames in scene.sweep(model, projector, args):
    ...                                                  # frames: uint8 [k, H', W', 3] on the host, RGB

The 50 target cameras of the wander path around frame args.render_idx are split into groups of at most 16 cameras
whose source views fit two pools of at most 32 views (bullet_time.group_cameras).  Per group the host writes one
small pinned staging buffer (view table, cameras, depth range) and copies it with one asynchronous copy; two kernels
assemble what sample_ray.stack_pooled_ray_batches would return for the group's get_all() batches; the encoder runs
once per pool, render_image.render_multi_image_mono renders the group, and csrc/bt_scene.cu turns the rendered rgb
into the script's cropped uint8 frames, which reach the host in one copy (the renderer itself still hands its
outputs back on the host).  DESIGN §3.9 gives the semantics.
"""

import os
import types

import numpy as np
import torch

from . import _lib
from . import bullet_time as bt
from .mono_scene import N_VIRTUAL, _TORCH, _Layout, _imread, _opencv_camera, load_cameras

OFFSETS = (-3, -2, -1, 0, 1, 2, 3)  # render_monocular_bt.py:113-115: the temporal views, sorted
CROP_RATIO = 0.03  # :295
_RING = 4  # pinned staging buffers in flight


# ---- host planning (render_monocular_bt.py:45-259) ---------------------------------------------------------------

def depth_range(near, top):
  """The sweep's depth range [near 0.9, far 1.5] (:69-74, :245) from the scaled bounds' min and max.  numpy 1.x, the
  reference's environment, evaluates `np.max(bds) + 15.0` and `x * 0.9` on float32 scalars in float64, and
  torch.tensor keeps the float64 pair: float64 [2]."""
  near, top = float(near), float(top)
  far = min(50, top + 15.0) if top < 10 else min(50, max(20, top))
  return np.array([near * 0.9, far * 1.5], np.float64)


def camera_row(H, W, K, c2w):
  """The 34 floats of a camera: (h, w, K 4x4, c2w 4x4) as float32 (:109-111)."""
  return np.concatenate(([H, W], np.asarray(K).reshape(-1), np.asarray(c2w).reshape(-1))).astype(np.float32)


def plan_sweep(cams, render_idx, num_source_views, max_range, num_vv):
  """The sweep of render_idx on a scene's cameras (mono_scene.load_cameras) -> dict:
    cameras   float32 [50, 34]: the target cameras of the wander path (render intrinsics and poses)
    render_K  float64 [50, 4, 4]
    selections  per camera (temporal ids, virtual-view ids, static ids), bullet_time.select_source_views
    groups    bullet_time.group_cameras's (start, stop) ranges."""
  H, W = cams["hw"]
  path = np.array(bt.wander_path(cams["poses"][render_idx])).astype(np.float32)
  parsed = [_opencv_camera(p) for p in path]
  render_K = np.stack([p[0] for p in parsed])
  render_c2w = np.stack([p[1] for p in parsed])
  sel = [bt.select_source_views(c, cams["c2w"], cams["vv_c2w"], render_idx, num_source_views, max_range, num_vv)
         for c in render_c2w]
  return dict(cameras=np.stack([camera_row(H, W, k, c) for k, c in zip(render_K, render_c2w)]), render_K=render_K,
              render_c2w=render_c2w, selections=sel, groups=bt.group_cameras(sel))


def plan_group(cams, plan, render_idx, lo, hi, mask_src_view):
  """The pools of cameras lo..hi-1, as sample_ray.stack_pooled_ray_batches forms them from the cameras' batches:
  each pool holds the union of the cameras' views by identity in the order first met (camera lo's slots first), so
  the dynamic pool starts with the 7 temporal frames.  Returns dict with
    dy_ids, st_ids        per camera, the identities of its slots (frame id, or ("vv", j) for a virtual view)
    dy_pool, st_pool      the pools' identities in pool order
    src_views, static_src_views   int32 [k, 7 + num_vv] / [k, 2 num_source_views + 1]: pool entry of every slot
    src_cameras, static_src_cameras  float32 [P, 34]: a frame's row holds its own intrinsics; a virtual view's row
                          holds the render camera's intrinsics (:195-199), those of the first camera that names it
    table                 int32 [Pd + Ps, 4]: dyn_scene_pools rows (frame, virtual view or -1, masked,
                          stack << 8 | slot); a virtual view's frame is 0, the scene's one set of virtual views."""
  H, W = cams["hw"]
  dy_ids, st_ids = [], []
  for k in range(lo, hi):
    t, vv, st = plan["selections"][k]
    dy_ids.append(list(t) + [("vv", j) for j in vv])
    st_ids.append(list(st))

  def pool(ids_per_cam, row_of):
    index, rows, tbl = {}, [], []
    for k, ids in zip(range(lo, hi), ids_per_cam):
      r = []
      for ident in ids:
        if ident not in index:
          index[ident] = len(rows)
          rows.append(row_of(ident, k))
        r.append(index[ident])
      tbl.append(r)
    return list(index), np.stack(rows), np.array(tbl, np.int32)

  def dy_row(ident, k):
    if isinstance(ident, tuple):
      return camera_row(H, W, plan["render_K"][k], cams["vv_c2w"][render_idx, ident[1]])
    return camera_row(H, W, cams["K"][ident], cams["c2w"][ident])

  st_row = lambda ident, k: camera_row(H, W, cams["K"][ident], cams["c2w"][ident])
  dy_pool, src_cameras, src_views = pool(dy_ids, dy_row)
  st_pool, st_cameras, st_views = pool(st_ids, st_row)
  table = []
  for slot, ident in enumerate(dy_pool):
    table.append((0, ident[1], 0, slot) if isinstance(ident, tuple) else (ident, -1, 0, slot))
  for slot, ident in enumerate(st_pool):
    table.append((ident, -1, int(bool(mask_src_view)), 2 << 8 | slot))
  return dict(dy_ids=dy_ids, st_ids=st_ids, dy_pool=dy_pool, st_pool=st_pool, src_views=src_views,
              static_src_views=st_views, src_cameras=src_cameras, static_src_cameras=st_cameras,
              table=np.array(table, np.int32))


def crop_of(H, W):
  """(crop_h, crop_w) of the output frames (:350-352)."""
  return int(H * CROP_RATIO), int(W * CROP_RATIO)


# ---- the scene ---------------------------------------------------------------------------------------------------

class BulletTimeScene(object):
  """A monocular scene (the reference's `dense` folder) on one device, for the bullet-time sweep of one frame.
  args: training_height, num_source_views, max_range, num_vv, mask_src_view, render_idx (the reference's rendering
  options; sweep also reads N_samples, chunk_size, inv_uniform and, when present, N_importance and white_bkgd)."""

  def __init__(self, scene_path, args, device):
    self.device = torch.device(device)
    if self.device.type != "cuda":
      raise RuntimeError("BulletTimeScene runs on CUDA only (no CPU fallback)")
    self.scene_path = scene_path
    self.render_idx = int(args.render_idx)
    self.num_source_views, self.max_range = int(args.num_source_views), int(args.max_range)
    self.num_vv, self.mask_src_view = int(args.num_vv), bool(args.mask_src_view)
    if not 0 <= self.num_vv <= N_VIRTUAL:
      raise ValueError("BulletTimeScene: num_vv %d, 0..%d" % (self.num_vv, N_VIRTUAL))
    if not 1 <= self.num_source_views <= self.max_range:
      raise ValueError("BulletTimeScene: num_source_views %d and max_range %d; the static views are chosen at an "
                       "interval of max_range // num_source_views >= 1" % (self.num_source_views, self.max_range))
    if 2 * self.num_source_views + 1 > bt.MAX_POOL or 7 + self.num_vv > bt.MAX_POOL:
      raise ValueError("BulletTimeScene: %d static / %d dynamic views per camera, at most %d"
                       % (2 * self.num_source_views + 1, 7 + self.num_vv, bt.MAX_POOL))
    cams = self.cams = load_cameras(scene_path, args.training_height)
    n = self.num_frames = len(cams["rgb_files"])
    if not 3 <= self.render_idx <= n - 4:
      raise ValueError("BulletTimeScene: render_idx %d; the temporal views are render_idx - 3 .. render_idx + 3, so "
                       "render_idx must lie in [3, %d] for %d frames" % (self.render_idx, n - 4, n))
    H, W = self.H, self.W = cams["hw"]
    self.depth_range = depth_range(*cams["bounds"])
    self.plan = plan_sweep(cams, self.render_idx, self.num_source_views, self.max_range, self.num_vv)
    self.groups = self.plan["groups"]
    self._cam_rows = np.stack([camera_row(H, W, cams["K"][i], cams["c2w"][i]) for i in range(n)])
    self._ray_rows = np.stack([self._ray_row(r) for r in self.plan["cameras"]])
    self._load()
    self._ring = [None] * _RING
    self._turn = 0

  @staticmethod
  def _ray_row(row):
    """M = R_c2w K^-1 | t of one camera row, formed in float32 as sample_ray.pixel_rays does."""
    c = torch.from_numpy(row)
    c2w, K = c[18:34].reshape(4, 4), c[2:18].reshape(4, 4)
    return torch.cat([(c2w[:3, :3] @ torch.inverse(K[:3, :3])).reshape(-1), c2w[:3, 3]]).numpy()

  # -- loading --
  def _load(self):
    n, H, W, p = self.num_frames, self.H, self.W, self.scene_path

    def image(path, what):
      a = _imread(path)
      if a.shape != (H, W, 3):
        raise ValueError("BulletTimeScene: %s %s is %s, the frames are %s" % (what, path, a.shape, (H, W, 3)))
      return a

    frames = np.stack([image(f, "frame") for f in self.cams["rgb_files"]])
    vdir = os.path.join(p, "source_virtual_views_%dx%d" % (W, H), "%05d" % self.render_idx)
    if not os.path.isdir(vdir):
      raise ValueError("BulletTimeScene: missing directory %s (the virtual views of render_idx %d)"
                       % (vdir, self.render_idx))
    vviews = np.stack([image(os.path.join(vdir, "%02d.png" % j), "virtual view") for j in range(N_VIRTUAL)])
    masks = None
    if self.mask_src_view:
      mdir = os.path.join(p, "dynamic_masks")
      if not os.path.isdir(mdir):
        raise ValueError("BulletTimeScene: missing directory %s (mask_src_view is set)" % mdir)
      count = len([f for f in os.listdir(mdir) if f.endswith(".png")])
      if count != n:
        raise ValueError("BulletTimeScene: %d dynamic masks in %s for %d frames" % (count, mdir, n))
      ms = [_imread(os.path.join(mdir, "%d.png" % i)) for i in range(n)]
      if len({m.shape for m in ms}) != 1:
        raise ValueError("BulletTimeScene: the dynamic masks differ in size or channels between frames")
      masks = np.stack(ms)
      if masks.ndim == 3:
        masks = masks[..., None]
    mc = 0 if masks is None else masks.shape[-1]
    self.nbytes = frames.nbytes + vviews.nbytes + n * H * W * mc
    need = self.nbytes + (0 if masks is None else masks.nbytes)
    free, total = torch.cuda.mem_get_info(self.device)
    if need > free:
      raise MemoryError("BulletTimeScene: the scene needs %.2f GB on %s while loading, %.2f GB of %.2f GB are free"
                        % (need / 1e9, self.device, free / 1e9, total / 1e9))
    with torch.cuda.device(self.device):
      self._frames = torch.from_numpy(frames).to(self.device)
      self._vviews = torch.from_numpy(vviews).to(self.device)
      self._srcmask = None
      if masks is not None:
        raw = torch.from_numpy(masks).to(self.device)
        self._srcmask = torch.empty(n, H, W, mc, dtype=torch.uint8, device=self.device)
        _lib.check(_lib.lib.dyn_nearest_resize(raw.data_ptr(), n, raw.shape[1], raw.shape[2], mc, H, W, 0,
                                               self._srcmask.data_ptr(), _lib.stream()))
        torch.cuda.current_stream().synchronize()  # the raw masks are freed here
        del raw
    self._scene = _lib.Scene(self._frames.data_ptr(), self._vviews.data_ptr(),
                             None if self._srcmask is None else self._srcmask.data_ptr(), None, None, None, None, None,
                             n, H, W, max(mc, 1), 0, 0)

  # -- per group --
  def __len__(self):
    return len(self.groups)

  def _staging(self, nbytes):
    """A pinned buffer of at least nbytes whose previous copy has finished (round robin over _RING buffers)."""
    k = self._turn = (self._turn + 1) % _RING
    slot = self._ring[k]
    if slot is not None:
      slot[1].synchronize()  # the copy of _RING groups ago: long done unless the host runs far ahead
    if slot is None or slot[0].numel() < nbytes:
      slot = (torch.empty(max(nbytes, 1 << 14), dtype=torch.uint8, pin_memory=True), torch.cuda.Event())
      self._ring[k] = slot
    return slot

  def group_batch(self, g):
    """Group g of the sweep (cameras groups[g][0] .. groups[g][1] - 1), assembled on the device without a host
    synchronisation:

      ray_batch     what sample_ray.stack_pooled_ray_batches returns for the cameras' RaySamplerSingleImage(item)
                    .get_all() batches: camera [k,34], camera_index, depth_range float64 [1,2], the pools src_rgbs /
                    src_cameras and static_src_rgbs / static_src_cameras, src_views / static_src_views (host int32),
                    src_view_ids / static_src_view_ids; rgb is None (the script's ground truth is never used)
      ray_samplers  k objects with H and W (what render_multi_image_mono reads)
      frame_idx, time_embedding, time_offset   as the script's loop builds them (:300-305)
      cameras       the cameras' indices in the sweep."""
    lo, hi = self.groups[g]
    grp = plan_group(self.cams, self.plan, self.render_idx, lo, hi, self.mask_src_view)
    K, H, W = hi - lo, self.H, self.W
    nd, ns = len(grp["dy_pool"]), len(grp["st_pool"])
    L = _Layout()
    L.add("table", np.int32, (nd + ns, 4))
    L.add("rays", np.float32, (K, 12))
    L.add("camera", np.float32, (K, 34))
    L.add("src_cameras", np.float32, (1, nd, 34))
    L.add("static_src_cameras", np.float32, (1, ns, 34))
    L.add("depth_range", np.float64, (1, 2))
    L.add("ref_time", np.float64, (1,))
    pinned, event = self._staging(L.nbytes)
    buf = pinned.numpy()
    view = {name: buf[off:off + nb].view(dt).reshape(shape) for name, dt, shape, off, nb in L.parts}
    view["table"][:] = grp["table"]
    view["rays"][:] = self._ray_rows[lo:hi]
    view["camera"][:] = self.plan["cameras"][lo:hi]
    view["src_cameras"][0] = grp["src_cameras"]
    view["static_src_cameras"][0] = grp["static_src_cameras"]
    view["depth_range"][0] = self.depth_range
    view["ref_time"][0] = float(self.render_idx / float(self.num_frames))
    d = torch.empty(L.nbytes, dtype=torch.uint8, device=self.device)
    d.copy_(pinned[:L.nbytes], non_blocking=True)
    event.record()
    d = {name: d[off:off + nb].view(_TORCH[dt]).reshape(shape) for name, dt, shape, off, nb in L.parts}

    e = dict(dtype=torch.float32, device=self.device)
    R = K * H * W
    rb = dict(ray_o=torch.empty(R, 3, **e), ray_d=torch.empty(R, 3, **e), depth_range=d["depth_range"],
              camera=d["camera"], render_camera=None, anchor_camera=None, rgb=None, disp=None, motion_mask=None,
              static_mask=None, uv_grid=torch.empty(R, 2, **e), flows=None, masks=None,
              src_rgbs=torch.empty(1, nd, H, W, 3, **e), src_cameras=d["src_cameras"],
              static_src_rgbs=torch.empty(1, ns, H, W, 3, **e), static_src_cameras=d["static_src_cameras"],
              src_views=torch.from_numpy(grp["src_views"]), static_src_views=torch.from_numpy(grp["static_src_views"]),
              src_view_ids=grp["dy_pool"], static_src_view_ids=grp["st_pool"],
              camera_index=torch.empty(R, dtype=torch.int32, device=self.device))
    with torch.cuda.device(self.device):
      st_ = _lib.stream()
      p = lambda x: x.data_ptr()
      _lib.check(_lib.lib.dyn_scene_pools(self._scene, p(d["table"]), nd + ns, p(rb["src_rgbs"]), nd,
                                          p(rb["static_src_rgbs"]), ns, st_))
      _lib.check(_lib.lib.dyn_nvi_rays(p(d["rays"]), K, H, W, p(rb["ray_o"]), p(rb["ray_d"]), p(rb["uv_grid"]),
                                       p(rb["camera_index"]), st_))
    return dict(ray_batch=rb, ray_samplers=[types.SimpleNamespace(H=H, W=W) for _ in range(K)],
                frame_idx=(self.render_idx, None), time_embedding=(d["ref_time"], None),
                time_offset=([int(o) for o in OFFSETS], None), cameras=list(range(lo, hi)))

  @staticmethod
  def encode(step, model):
    """The encoder once per pool (:312-320): feature_net's first output over the dynamic pool, feature_net_st's
    first output over the static pool."""
    rb = step["ray_batch"]
    ref_featmaps, _ = model.feature_net(rb["src_rgbs"].squeeze(0).permute(0, 3, 1, 2))
    static_featmaps, _ = model.feature_net_st(rb["static_src_rgbs"].squeeze(0).permute(0, 3, 1, 2))
    return ref_featmaps, None, static_featmaps

  @staticmethod
  def render(step, featmaps, model, projector, args):
    """render_multi_image_mono over the group (det=True, is_train=False) -> rgb [k, H, W, 3] on the scene's device."""
    from .render_image import render_multi_image_mono
    rets = render_multi_image_mono(
        frame_idx=step["frame_idx"], time_embedding=step["time_embedding"], time_offset=step["time_offset"],
        ray_samplers=step["ray_samplers"], ray_batch=step["ray_batch"], model=model, projector=projector,
        chunk_size=args.chunk_size, N_samples=args.N_samples, args=args, inv_uniform=args.inv_uniform,
        N_importance=getattr(args, "N_importance", 0), det=True, white_bkgd=getattr(args, "white_bkgd", False),
        featmaps=featmaps, is_train=False, num_vv=args.num_vv)
    # render_multi_image_mono hands its outputs back on the host, as render_single_image_mono does
    return torch.stack([r["outputs_coarse_ref"]["rgb"] for r in rets]).to(step["ray_batch"]["ray_o"].device)

  def frames_device(self, rgb):
    """rgb [k, H, W, 3] fp32 on the device -> the script's cropped uint8 frames [k, H', W', 3], on the device."""
    if rgb.dim() != 4 or rgb.shape[1:] != (self.H, self.W, 3):
      raise ValueError("BulletTimeScene: rgb is %s, [k, %d, %d, 3] expected" % (tuple(rgb.shape), self.H, self.W))
    return bt_frames(rgb)

  def sweep(self, model, projector, args):
    """The script's loop, one group at a time: yields (camera indices, uint8 frames [k, H', W', 3] on the host).
    Per group: the pools and rays (group_batch), one encoder pass per pool, one render_multi_image_mono, the frame
    kernel and one device-to-host copy of the frames."""
    for g in range(len(self.groups)):
      step = self.group_batch(g)
      with torch.no_grad():
        rgb = self.render(step, self.encode(step, model), model, projector, args)
        out = self.frames_device(rgb)
      yield step["cameras"], out.cpu().numpy()


def bt_frames(rgb):
  """(255 * clip(rgb, 0, 1)).astype(np.uint8) of the cropped window (:346-354), on the device: rgb [k, H, W, 3] fp32
  (CUDA) -> uint8 [k, H - 2 crop_h, W - 2 crop_w, 3]."""
  if rgb.dim() != 4 or rgb.shape[-1] != 3:
    raise ValueError("bt_frames: rgb is %s, [k, H, W, 3] expected" % (tuple(rgb.shape),))
  K, H, W, _ = rgb.shape
  ch, cw = crop_of(H, W)
  x = rgb.contiguous()
  out = torch.empty(K, H - 2 * ch, W - 2 * cw, 3, dtype=torch.uint8, device=rgb.device)
  with torch.cuda.device(rgb.device):
    _lib.check(_lib.lib.dyn_bt_frames(_lib.ptr(x), K, H, W, ch, cw, out.data_ptr(), _lib.stream()))
  return out
