"""An Nvidia-benchmark scene resident on the device: the reference's evaluation front end (eval_nvidia.py
DynamicVideoDataset under its DataLoader, RaySamplerSingleImage.get_all and the cv2 ground-truth / mask reads of its
__main__ block) without imageio or scikit-image, and without decoding any file after the scene is loaded.

  scene = NvidiaScene(scene_path, args, device)    # reads <scene_path> (the reference's `dense` folder) once
  step = scene.time_step(img_i)                     # one time step's batch, ground truth and masks, on the device
  result = scene.evaluate(model, projector, args)   # eval_nvidia.py:305-481: PSNR / SSIM of every camera
  result = scene.evaluate(model, projector, args, lpips=LPIPSWeights(alexnet, lin))   # and LPIPS

Frames, coarse static masks, ground truth and dynamic masks are uploaded once: the ground truth is resized to the
render size on the device (csrc/nvi_scene.cu: cv2's INTER_AREA, byte for byte) and the masks with cv2's
INTER_NEAREST rule.  Per time step the host writes one small pinned staging buffer (view table, cameras, ids) and
copies it with one asynchronous copy; two kernels assemble the batch.  No call of `time_step` synchronises with the
device.  DESIGN §3.8 gives the semantics and what was measured.
"""

import collections
import os
import types

import numpy as np
import torch

from . import _lib
from .mono_scene import _TORCH, _Layout, _image_files, _imread, _npload, _opencv_camera

CYCLE = 12  # eval_nvidia.py:96: the benchmark's cameras, one per frame in a round robin
HEIGHT = 288  # eval_nvidia.py:41
OFFSETS = (-3, -2, -1, 0, 1, 2, 3)  # eval_nvidia.py:92-94, sorted
_RING = 4  # pinned staging buffers in flight


def _cv2():
  import cv2
  return cv2


# ---- poses (llff_data_utils.py:57-123, :126-185, :216-318; eval_nvidia.py:39-66) -----------------------------------

def _normalize(x):
  return x / np.linalg.norm(x)


def _poses_avg(poses):
  """llff poses_avg + viewmatrix: float32 in, [3, 5] out (normalize applied twice to the z axis, as there)."""
  hwf = poses[0, :3, -1:]
  center = poses[:, :3, 3].mean(0)
  z = _normalize(_normalize(poses[:, :3, 2].sum(0)))
  x = _normalize(np.cross(poses[:, :3, 1].sum(0), z))
  y = _normalize(np.cross(z, x))
  return np.concatenate([np.stack([x, y, z, center], 1), hwf], 1)


def _recenter_poses(poses):
  """llff recenter_poses: poses [N, 3, 5] float32 -> float32, in the mean camera's frame."""
  out = poses + 0
  bottom = np.reshape([0, 0, 0, 1.0], [1, 4])
  c2w = np.concatenate([_poses_avg(poses)[:3, :4], bottom], -2)
  last = np.tile(np.reshape(bottom, [1, 1, 4]), [poses.shape[0], 1, 1])
  out[:, :3, :4] = (np.linalg.inv(c2w) @ np.concatenate([poses[:, :3, :4], last], -2))[:, :3, :4]
  return out


def load_cameras(scene_path, height=HEIGHT, bd_factor=0.75):
  """The scene's cameras as DynamicVideoDataset.__init__ builds them (load_llff_data with load_imgs=False).

  Returns a dict: rgb_files, hw (of the frames), K [N,4,4], c2w [N,4,4] (float64), scale (float64) and depth_range
  float64 [2] = (min(bds) 0.9, (max(bds) + 15) 1.5).  numpy 1.x, the reference's environment, evaluates
  `bds.min() * bd_factor` and `np.max(bds) + 15.0` in float64 and applies the float64 scale to the float32 arrays as
  float32(scale); torch.tensor of the two float64 scalars is float64."""
  arr = _npload(os.path.join(scene_path, "poses_bounds_cvd.npy"))
  if arr.ndim != 2 or arr.shape[1] != 17:
    raise ValueError("NvidiaScene: poses_bounds_cvd.npy is %s, [N, 17] expected" % (arr.shape,))
  poses = arr[:, :-2].reshape([-1, 3, 5]).transpose([1, 2, 0])
  bds = arr[:, -2:].transpose([1, 0])
  orig = _image_files(os.path.join(scene_path, "images"))
  if not orig:
    raise ValueError("NvidiaScene: no images in %s" % os.path.join(scene_path, "images"))
  sh = _imread(orig[0]).shape
  factor = sh[0] / float(height)
  width = int(round(sh[1] / factor))
  files = _image_files(os.path.join(scene_path, "images_%dx%d" % (width, height)))
  if poses.shape[-1] != len(files):
    raise ValueError("NvidiaScene: %d images and %d poses" % (len(files), poses.shape[-1]))
  hw = _imread(files[0]).shape[:2]
  poses[:2, 4, :] = np.array(hw).reshape([2, 1])
  poses = np.concatenate([poses[:, 1:2, :], -poses[:, 0:1, :], poses[:, 2:, :]], 1)
  poses = np.moveaxis(poses, -1, 0).astype(np.float32)
  bds = np.moveaxis(bds, -1, 0).astype(np.float32)
  scale = 1.0 / (float(bds.min()) * bd_factor)
  s32 = np.float32(scale)
  poses[:, :3, 3] *= s32
  bds *= s32
  poses = _recenter_poses(poses).astype(np.float32)
  cams = [_opencv_camera(p) for p in poses]
  near, far = float(bds.min()), float(bds.max()) + 15.0
  return dict(rgb_files=files, hw=tuple(int(x) for x in hw), K=np.stack([c[0] for c in cams]),
              c2w=np.stack([c[1] for c in cams]), scale=scale, depth_range=np.array([near * 0.9, far * 1.5]))


# ---- view selection (eval_nvidia.py:92-119) ----------------------------------------------------------------------

def dynamic_ids(img_i):
  return [img_i + o for o in OFFSETS]


def static_ids(img_i, n):
  """For every residue class mod 12 but img_i's, the frame of that class nearest img_i (the first on a tie), sorted."""
  groups = collections.defaultdict(list)
  for j in range(n):
    if j % CYCLE != img_i % CYCLE:
      groups[j % CYCLE].append(j)
  return sorted(int(g[int(np.argmin(np.abs(np.array(g) - img_i)))]) for g in groups.values())


def target_cameras(img_i):
  """The cameras scored at img_i: 0..11 but img_i % 12.  Camera i's pose and intrinsics are frame i's."""
  return [i for i in range(CYCLE) if i != img_i % CYCLE]


# ---- the scene ---------------------------------------------------------------------------------------------------

class NvidiaScene(object):
  """An Nvidia-benchmark scene (the reference's `<folder_path>/<scene>/dense`) on one device.
  args: mask_static (the reference's evaluation option; also read by evaluate: chunk_size, N_samples, N_importance,
  inv_uniform, white_bkgd)."""

  def __init__(self, scene_path, args, device):
    self.device = torch.device(device)
    if self.device.type != "cuda":
      raise RuntimeError("NvidiaScene runs on CUDA only (no CPU fallback)")
    self.scene_path = scene_path
    self.mask_static = bool(args.mask_static)
    cams = self.cams = load_cameras(scene_path)
    n = self.num_frames = len(cams["rgb_files"])
    if n < CYCLE:
      raise ValueError("NvidiaScene: %d frames; the benchmark's round robin of %d cameras needs at least %d"
                       % (n, CYCLE, CYCLE))
    H, W = self.H, self.W = cams["hw"]
    self.steps = list(range(3, n - 3))
    with torch.cuda.device(self.device):
      self._load()
    self._cam_rows = np.concatenate([np.full((n, 2), (H, W), np.float64), cams["K"].reshape(n, 16),
                                     cams["c2w"].reshape(n, 16)], 1).astype(np.float32)
    # ray matrices M = R_c2w K^-1 | t of every frame's camera, formed in float32 as sample_ray.pixel_rays does
    rows = []
    for i in range(n):
      c = torch.from_numpy(self._cam_rows[i])
      c2w, K = c[18:34].reshape(4, 4), c[2:18].reshape(4, 4)
      rows.append(torch.cat([(c2w[:3, :3] @ torch.inverse(K[:3, :3])).reshape(-1), c2w[:3, 3]]).numpy())
    self._ray_rows = np.stack(rows).astype(np.float32)
    self._ring = [None] * _RING
    self._turn = 0

  # -- loading --
  def _load(self):
    cv2 = _cv2()
    n, H, W, dev, p = self.num_frames, self.H, self.W, self.device, self.scene_path
    frames = []
    for f in self.cams["rgb_files"]:
      a = _imread(f)
      if a.shape != (H, W, 3):
        raise ValueError("NvidiaScene: frame %s is %s, the first frame is %s" % (f, a.shape, (H, W, 3)))
      frames.append(a)
    self._frames = torch.from_numpy(np.stack(frames)).to(dev)
    self._smask = torch.full((n, H, W), 255, dtype=torch.uint8, device=dev)
    if self.mask_static:
      for i in range(3, n - 3):
        m = _imread(os.path.join(p, "coarse_masks", "%05d.png" % i))
        if m.ndim != 2:
          raise ValueError("NvidiaScene: coarse mask %d is %s; single-channel masks expected (eval_nvidia.py:353 "
                           "broadcasts [H, W] masks only)" % (i, m.shape))
        self._nearest(torch.from_numpy(np.array(m)).to(dev)[None, ..., None], H, W, False,
                      self._smask[i:i + 1])
    T, S = len(self.steps), CYCLE - 1
    self._gt = torch.empty(T, S, H, W, 3, dtype=torch.uint8, device=dev)
    self._dmask = torch.empty_like(self._gt)
    for t, img_i in enumerate(self.steps):
      gts, masks = [], []
      for s, cam in enumerate(target_cameras(img_i)):
        gp = os.path.join(p, "mv_images", "%05d" % img_i, "cam%02d.jpg" % (cam + 1))
        mp = os.path.join(p, "mv_masks", "%05d" % img_i, "cam%02d.png" % (cam + 1))
        g, m = self._cv2_read(cv2, gp), self._cv2_read(cv2, mp)
        if g.shape[0] < H or g.shape[1] < W:
          raise ValueError("NvidiaScene: ground truth %s is %dx%d, smaller than the %dx%d render; upscaling "
                           "(cv2's bilinear INTER_AREA branch) is not built" % (gp, g.shape[1], g.shape[0], W, H))
        gts.append(np.ascontiguousarray(g[:, :, ::-1]))  # eval_nvidia.py:387
        masks.append(m)  # :423: BGR, never reversed
      self._resize_group(gts, self._gt[t], area=True)
      self._resize_group(masks, self._dmask[t], area=False)
    torch.cuda.current_stream(dev).synchronize()  # the host images above are released once the uploads are done
    self.nbytes = sum(x.numel() for x in (self._frames, self._smask, self._gt, self._dmask))
    self._scene = _lib.NviScene(self._frames.data_ptr(), self._smask.data_ptr(), self._gt.data_ptr(),
                                self._dmask.data_ptr(), n, H, W, T, S)

  @staticmethod
  def _cv2_read(cv2, path):
    if not os.path.isfile(path):
      raise ValueError("NvidiaScene: missing file %s" % path)
    a = cv2.imread(path)
    if a is None:
      raise ValueError("NvidiaScene: cv2 cannot read %s" % path)
    return a

  def _resize_group(self, imgs, out, area):
    """Resize the images of one time step into out [S, H, W, 3], one launch per distinct source size."""
    by_size = collections.defaultdict(list)
    for s, a in enumerate(imgs):
      by_size[a.shape].append(s)
    for shape, idx in by_size.items():
      src = torch.from_numpy(np.stack([imgs[s] for s in idx])).to(self.device)
      dst = out if len(idx) == len(imgs) else torch.empty((len(idx),) + tuple(out.shape[1:]), dtype=torch.uint8,
                                                           device=self.device)
      if area:
        _lib.check(_lib.lib.dyn_area_resize(src.data_ptr(), len(idx), shape[0], shape[1], 3, self.H, self.W,
                                            dst.data_ptr(), _lib.stream()))
      else:
        self._nearest(src, self.H, self.W, True, dst)
      if dst is not out:
        out[torch.tensor(idx, device=self.device)] = dst

  @staticmethod
  def _nearest(src, H, W, threshold, dst):
    N, sh, sw, C = src.shape
    _lib.check(_lib.lib.dyn_nearest_resize(src.data_ptr(), N, sh, sw, C, H, W, int(threshold), dst.data_ptr(),
                                           _lib.stream()))

  # -- per time step --
  def __len__(self):
    return len(self.steps)

  def _staging(self, nbytes):
    """A pinned buffer of at least nbytes whose previous copy has finished (round robin over _RING buffers)."""
    k = self._turn = (self._turn + 1) % _RING
    slot = self._ring[k]
    if slot is not None:
      slot[1].synchronize()  # the copy of _RING steps ago: long done unless the host runs far ahead
    if slot is None or slot[0].numel() < nbytes:
      slot = (torch.empty(max(nbytes, 1 << 14), dtype=torch.uint8, pin_memory=True), torch.cuda.Event())
      self._ring[k] = slot
    return slot

  def time_step(self, img_i):
    """One time step of eval_nvidia.py's loop (img_i in 3 .. num_frames - 4), all on the device:

      ray_batch     sample_ray.stack_ray_batches over the 11 RaySamplerSingleImage(item).get_all() batches: the same
                    keys, shapes and dtypes (camera [11,34], camera_index, depth_range float64 [1,2], the source
                    stacks, static_src_masks [1,11,H,W])
      ray_samplers  11 objects with H and W (what render_multi_image_nvi reads)
      frame_idx, time_embedding, time_offset   as eval_nvidia.py:323-328 builds them, in render_*_nvi's form
      static_src_masked  [11,3,H,W]: static_src_rgbs * static_src_masks, the fine encoder's input (:350-358)
      gt_rgb [11,H,W,3] float32 u8 / 255, dynamic_mask [11,H,W,3] float32 0 / 1 (BGR order), cameras (0..11)."""
    n, H, W = self.num_frames, self.H, self.W
    if img_i not in range(3, n - 3):
      raise ValueError("NvidiaScene.time_step: img_i %d, 3 .. %d" % (img_i, n - 4))
    dyn, st, cams = dynamic_ids(img_i), static_ids(img_i, n), target_cameras(img_i)
    t = img_i - 3
    nd, ns, K = len(dyn), len(st), len(cams)
    L = _Layout()
    L.add("table", np.int32, (nd + ns + K,))
    L.add("rays", np.float32, (K, 12))
    L.add("camera", np.float32, (K, 34))
    L.add("src_cameras", np.float32, (1, nd, 34))
    L.add("static_src_cameras", np.float32, (1, ns, 34))
    L.add("depth_range", np.float64, (1, 2))
    L.add("ref_time", np.float64, (1,))
    pinned, event = self._staging(L.nbytes)
    buf = pinned.numpy()
    view = {name: buf[off:off + nb].view(dt).reshape(shape) for name, dt, shape, off, nb in L.parts}
    view["table"][:] = dyn + st + [t * (CYCLE - 1) + s for s in range(K)]
    view["rays"][:] = self._ray_rows[cams]
    view["camera"][:] = self._cam_rows[cams]
    view["src_cameras"][0] = self._cam_rows[dyn]
    view["static_src_cameras"][0] = self._cam_rows[st]
    view["depth_range"][0] = self.cams["depth_range"]
    view["ref_time"][0] = float(img_i / float(n))
    d = torch.empty(L.nbytes, dtype=torch.uint8, device=self.device)
    d.copy_(pinned[:L.nbytes], non_blocking=True)
    event.record()
    d = {name: d[off:off + nb].view(_TORCH[dt]).reshape(shape) for name, dt, shape, off, nb in L.parts}

    e = dict(dtype=torch.float32, device=self.device)
    R = K * H * W
    rb = dict(ray_o=torch.empty(R, 3, **e), ray_d=torch.empty(R, 3, **e), depth_range=d["depth_range"],
              camera=d["camera"], render_camera=None, anchor_camera=None, rgb=None, disp=None, motion_mask=None,
              static_mask=None, uv_grid=torch.empty(R, 2, **e), flows=None, masks=None,
              src_rgbs=torch.empty(1, nd, H, W, 3, **e), src_cameras=d["src_cameras"], anchor_src_rgbs=None,
              anchor_src_cameras=None, static_src_rgbs=torch.empty(1, ns, H, W, 3, **e),
              static_src_cameras=d["static_src_cameras"], static_src_masks=torch.empty(1, ns, H, W, **e),
              camera_index=torch.empty(R, dtype=torch.int32, device=self.device))
    masked = torch.empty(ns, H, W, 3, **e)
    gt, dmask = torch.empty(K, H, W, 3, **e), torch.empty(K, H, W, 3, **e)
    with torch.cuda.device(self.device):
      st_ = _lib.stream()
      p = lambda x: x.data_ptr()
      _lib.check(_lib.lib.dyn_nvi_time_step(self._scene, p(d["table"]), nd, ns, K, p(rb["src_rgbs"]),
                                            p(rb["static_src_rgbs"]), p(rb["static_src_masks"]), p(masked), p(gt),
                                            p(dmask), st_))
      _lib.check(_lib.lib.dyn_nvi_rays(p(d["rays"]), K, H, W, p(rb["ray_o"]), p(rb["ray_d"]), p(rb["uv_grid"]),
                                       p(rb["camera_index"]), st_))
    return dict(ray_batch=rb, ray_samplers=[types.SimpleNamespace(H=H, W=W) for _ in cams],
                frame_idx=(img_i, None), time_embedding=(d["ref_time"], None),
                time_offset=([int(o) for o in OFFSETS], None), static_src_masked=masked.permute(0, 3, 1, 2),
                gt_rgb=gt, dynamic_mask=dmask, cameras=cams, id=img_i, nearest_pose_ids=dyn, static_pose_ids=st)

  def render(self, step, model, projector, args):
    """The encoder passes (eval_nvidia.py:335-358) and one render_multi_image_nvi over the time step's cameras ->
    predicted rgb [K, H, W, 3] on the device."""
    from .render_image import render_multi_image_nvi
    rb = step["ray_batch"]
    src = rb["src_rgbs"].squeeze(0).permute(0, 3, 1, 2)
    static_src = rb["static_src_rgbs"].squeeze(0).permute(0, 3, 1, 2)
    ref_featmaps, _ = model.feature_net(src)
    _, static_featmaps = model.feature_net(static_src)
    ref_featmaps_fine, _ = model.feature_net_fine(src)
    _, static_featmaps_fine = model.feature_net_fine(step["static_src_masked"] if self.mask_static else static_src)
    rets = render_multi_image_nvi(
        frame_idx=step["frame_idx"], time_embedding=step["time_embedding"], time_offset=step["time_offset"],
        ray_samplers=step["ray_samplers"], ray_batch=rb, model=model, projector=projector,
        chunk_size=args.chunk_size, det=True, N_samples=args.N_samples, args=args, inv_uniform=args.inv_uniform,
        N_importance=args.N_importance, white_bkgd=args.white_bkgd,
        coarse_featmaps=(ref_featmaps, None, static_featmaps),
        fine_featmaps=(ref_featmaps_fine, None, static_featmaps_fine), is_train=False)
    return torch.stack([r["outputs_fine_ref"]["rgb"] for r in rets]).to(self.device)

  def evaluate(self, model, projector, args, on_step=None, lpips=None):
    """eval_nvidia.py:305-481: per time step the encoder passes, one render_multi_image_nvi, one score_views and one
    read-back of the scores.  on_step(img_i, scores so far [t+1, 11, 3, 2]) is called after each time step (the script
    prints its MOVING lines there).

    Returns dict(scores float64 [T, 11, 3, 2] (full / dynamic / static x PSNR / SSIM, cameras in target_cameras
    order), mean float64 [3, 2] (np.mean over every camera of every time step, as the AVG lines), steps).

    lpips: an LPIPSWeights (dynibar_b200.metrics) adds one lpips_views per time step, read back with the scores; the
    result gains lpips float64 [T, 11, 3] and lpips_mean [3] (averaged as `mean`), and on_step receives the LPIPS
    values so far [t+1, 11, 3] as a third argument.  Without it nothing of the above changes."""
    from .metrics import lpips_views, score_views
    out, lp = [], []
    for img_i in self.steps:
      step = self.time_step(img_i)
      with torch.no_grad():
        pred = self.render(step, model, projector, args)
        scores = score_views(pred, step["gt_rgb"], step["dynamic_mask"])
        if lpips is not None:
          lp.append(lpips_views(pred, step["gt_rgb"], step["dynamic_mask"], weights=lpips).cpu().numpy())
      out.append(scores.cpu().numpy())
      if on_step is not None:
        if lpips is None:
          on_step(img_i, np.stack(out))
        else:
          on_step(img_i, np.stack(out), np.stack(lp))
    scores = np.stack(out)
    res = dict(scores=scores, mean=mean_scores(scores), steps=list(self.steps))
    if lpips is not None:
      res.update(lpips=np.stack(lp), lpips_mean=mean_lpips(np.stack(lp)))
    return res


def mean_scores(scores):
  """The AVG / MOVING lines' np.mean over the flat per-camera lists (time-major, cameras in order) -> [3, 2]."""
  flat = scores.reshape(-1, 3, 2)
  return np.array([[np.mean(np.array(flat[:, r, c].tolist())) for c in range(2)] for r in range(3)])


def mean_lpips(lpips):
  """The LPIPS AVG / MOVING lines: lpips [T, 11, 3] -> [3], averaged as mean_scores averages."""
  flat = lpips.reshape(-1, 3)
  return np.array([np.mean(np.array(flat[:, r].tolist())) for r in range(3)])
