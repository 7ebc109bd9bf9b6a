"""A monocular training scene resident on the device: the reference's data loader (ibrnet/data_loaders/monocular.py
MonocularDataset) and `RaySamplerSingleImage.random_sample` (ibrnet/sample_ray.py) without imageio or scikit-image,
and without decoding any file after the scene is loaded.

  scene = MonocularScene(scene_path, args, device)      # reads <scene_path> (the reference's `dense` folder) once
  scene.set_epoch(epoch)
  train_data, ray_batch = scene.sample(rng, args.N_rand, args.sample_mode)
  for train_data, ray_batch in scene.loader(rng, args.N_rand, args.sample_mode): ...   # num_frames steps

`rng` is a np.random.RandomState: the host makes exactly the calls __getitem__ makes on np.random, in its order, so
RandomState(s) draws what the reference draws after np.random.seed(s).  Pixels are drawn from `sample_ray.rng`, as
the library's RaySamplerSingleImage.sample_random_pixel draws them.  `train_data` is __getitem__'s item as the
DataLoader collates it (batch dimension 1) with its tensors on the device; `ray_batch` is what
RaySamplerSingleImage(train_data, device).random_sample(...) returns, and shares the source-view stacks with
`train_data`.

Frames, virtual views, disparity, flows and masks are uploaded once (csrc/scene.cu prepares the masks of every frame
on the device: the motion mask's erosion at height 288, the static mask, the source-view mask).  Per step the host
makes the draws, writes one small pinned staging buffer (view table, cameras, ids, pixel indices) and copies it with
one asynchronous copy; two kernels assemble the batch.  No call of `sample` synchronises with the device.
DESIGN §3.7 gives the semantics and what was measured.
"""

import os
import types

import numpy as np
import torch

from . import _lib
from . import sample_ray

ERODE_H = 288  # monocular.py:186: the motion mask is eroded at height 288 whatever training_height is
N_VIRTUAL = 8
_OFFSETS = (1, 2, 3, -1, -2, -3)  # monocular.py:216: the temporal source views, and the flows' order
_RING = 4  # pinned staging buffers in flight


# ---- files -------------------------------------------------------------------------------------------------------

def _imread(path):
  """PNG / JPEG as uint8 [H, W] or [H, W, 3] (alpha dropped), through PIL as imageio reads PNG."""
  from PIL import Image
  if not os.path.isfile(path):
    raise ValueError("MonocularScene: missing file %s" % path)
  with Image.open(path) as im:
    if im.mode == "P":
      im = im.convert("RGBA" if "transparency" in im.info else "RGB")
    if im.mode not in ("L", "LA", "RGB", "RGBA"):
      raise ValueError("MonocularScene: %s has mode %s; 8-bit grey or RGB(A) images expected (16-bit data is not "
                       "supported)" % (path, im.mode))
    a = np.asarray(im)
  if a.ndim == 3 and a.shape[2] in (2, 4):
    a = a[..., :a.shape[2] - 1]
  if a.ndim == 3 and a.shape[2] == 1:
    a = a[..., 0]
  return np.ascontiguousarray(a)


def _npload(path):
  if not os.path.isfile(path):
    raise ValueError("MonocularScene: missing file %s" % path)
  return np.load(path)


def _image_files(d):
  if not os.path.isdir(d):
    raise ValueError("MonocularScene: missing directory %s" % d)
  return [os.path.join(d, f) for f in sorted(os.listdir(d)) if f.endswith(("JPG", "jpg", "png"))]


# ---- poses (llff_data_utils.py:14-54, :57-123, :126-213, :321-410; monocular.py:61-89) ------------------------------

def _unit(x):
  return x / np.linalg.norm(x)


def _average_c2w(poses):
  """The mean camera of poses [N, 3, >=4]: mean centre, summed z and y axes (llff poses_avg)."""
  z = _unit(poses[:, :3, 2].sum(0))
  x = _unit(np.cross(poses[:, :3, 1].sum(0), z))
  y = _unit(np.cross(z, x))
  m = np.stack([x, y, z, poses[:, :3, 3].mean(0)], 1)
  return np.concatenate([m, np.array([[0, 0, 0, 1.0]])], 0)


def _recenter(poses, vv):
  """recenter_poses_mono: poses [N, 3, 5], vv [N, 8, 3, 4] -> (poses [N, 3, 5], vv [N, 8, 3, 5]) in the mean camera's
  frame; the mean is taken over the frames only."""
  inv = np.linalg.inv(_average_c2w(poses))
  last = np.tile(np.array([[[0, 0, 0, 1.0]]]), [poses.shape[0], 1, 1])
  out = poses + 0
  out[:, :3, :4] = (inv @ np.concatenate([poses[:, :3, :4], last], 1))[:, :3, :4]
  hwf = poses[:, :, 4:5]
  vv_out = np.zeros((vv.shape[1], vv.shape[0], 3, 5))
  for j in range(vv.shape[1]):
    vv_out[j] = np.concatenate([(inv @ np.concatenate([vv[:, j, :3, :4], last], 1))[:, :3, :], hwf], 2)
  return out, np.moveaxis(vv_out, 1, 0)


def _opencv_camera(pose):
  """llff [3, 5] (c2w | h, w, f) -> (K [4, 4], c2w [4, 4]) float64 with the y and z axes flipped."""
  h, w, f = pose[:3, -1]
  c2w = np.eye(4)
  c2w[:3] = pose[:3, :4]
  c2w[:, 1:3] *= -1
  K = np.array([[f, 0, w / 2.0, 0], [0, f, h / 2.0, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
  return K, c2w


def load_cameras(scene_path, height, bd_factor=0.75):
  """The scene's cameras as MonocularDataset.__init__ builds them (load_mono_data with load_imgs=False).

  Returns a dict: rgb_files, hw (of the training images), K [N,4,4], c2w [N,4,4], vv_c2w [N,8,4,4] (float64),
  scale (float64), depth_range float32 [2] (near * 0.9, far * 1.5), poses float32 [N,3,5] (the recentred llff
  poses) and bounds (min, max of the scaled bounds as Python floats).  `scale` is computed in float64 and applied as
  float32(scale) in float32, as numpy 1.x (the reference's environment) evaluates the float32 array operations with
  a float64 scalar; the near / far arithmetic is float64, rounded to float32 at the end, as numpy 1.x does."""
  arr = _npload(os.path.join(scene_path, "poses_bounds_cvd.npy"))
  if arr.ndim != 2 or arr.shape[1] != 17:
    raise ValueError("MonocularScene: poses_bounds_cvd.npy is %s, [N, 17] expected" % (arr.shape,))
  poses = arr[:, :-2].reshape([-1, 3, 5]).transpose([1, 2, 0])
  bds = arr[:, -2:].transpose([1, 0])
  orig = _image_files(os.path.join(scene_path, "images"))
  if not orig:
    raise ValueError("MonocularScene: no images in %s" % os.path.join(scene_path, "images"))
  sh = _imread(orig[0]).shape
  factor = sh[0] / float(height)
  width = int(round(sh[1] / factor))
  files = _image_files(os.path.join(scene_path, "images_%dx%d" % (width, height)))
  if poses.shape[-1] != len(files):
    raise ValueError("MonocularScene: %d images and %d poses" % (len(files), poses.shape[-1]))
  hw = _imread(files[0]).shape[:2]
  poses[:2, 4, :] = np.array(hw).reshape([2, 1])
  vv = _npload(os.path.join(scene_path, "source_vv_poses.npy"))
  if vv.shape != (N_VIRTUAL, 3, 4, len(files)):
    raise ValueError("MonocularScene: source_vv_poses.npy is %s, [8, 3, 4, %d] expected" % (vv.shape, len(files)))
  # [x, y, z] -> [y, -x, z] columns, frame axis first
  poses = np.concatenate([poses[:, 1:2, :], -poses[:, 0:1, :], poses[:, 2:, :]], 1)
  vv = np.concatenate([vv[:, :, 1:2, :], -vv[:, :, 0:1, :], vv[:, :, 2:, :]], 2)
  poses = np.moveaxis(poses, -1, 0).astype(np.float32)
  vv = np.moveaxis(vv, -1, 0).astype(np.float32)
  bds = np.moveaxis(bds, -1, 0).astype(np.float32)
  scale = 1.0 / (float(bds.min()) * bd_factor)
  s32 = np.float32(scale)
  poses[:, :3, 3] *= s32
  vv[..., :3, 3] *= s32
  bds *= s32
  poses, vv = _recenter(poses, vv)
  poses = poses.astype(np.float32)
  near, top = float(bds.min()), float(bds.max())
  far = min(20, top + 15.0) if top < 10 else min(50, max(20, top))
  cams = [_opencv_camera(p) for p in poses]
  vv_c2w = np.stack([np.stack([_opencv_camera(p)[1] for p in frame]) for frame in vv])
  return dict(rgb_files=files, hw=tuple(hw), K=np.stack([c[0] for c in cams]), c2w=np.stack([c[1] for c in cams]),
              vv_c2w=vv_c2w, scale=scale, depth_range=np.array([near * 0.9, far * 1.5]).astype(np.float32),
              poses=poses, bounds=(near, top))


# ---- the draws (monocular.py:148, :215-298, :313-315, :375-377) --------------------------------------------------

def draw_views(rng, n, epoch, init_decay_epoch, num_source_views, max_range, num_vv, c2w):
  """__getitem__'s random draws and view selection, in its order -> dict of ids."""
  idx = int(rng.randint(3, n - 3))
  steps = min(3, epoch // init_decay_epoch + 1)
  pool = [i for i in range(1, steps + 1)] + [-i for i in range(1, steps + 1)]
  anchor = idx + pool[rng.choice(len(pool))]
  anchor_ids = [anchor + o for o in (3, 2, 1, 0, -1, -2, -3) if 0 <= anchor + o < n and anchor + o != idx]
  if rng.choice([0, 1], p=[1.0 - 0.005, 0.005]):  # occasionally the target frame itself
    anchor_ids.append(idx)
  dist = np.linalg.norm(c2w[idx][None, :3, 3].repeat(n, 0) - c2w[:, :3, 3], axis=1)
  dist[idx] = 1e3
  by_dist = np.argsort(dist)
  max_interval = max_range // num_source_views
  interval = rng.randint(max(2, max_interval - 2), max_interval + 1)
  static = []
  for k in range(-num_source_views, num_source_views):
    j = idx + interval * k + rng.randint(1, interval + 1)
    if 0 <= j < n and j != idx:
      static.append(j)
  chosen = set(static)
  for j in by_dist[::5]:  # too few: every fifth frame by camera distance
    if len(static) >= 2 * num_source_views:
      break
    if j not in chosen:
      static.append(j)
  vv = rng.choice(list(range(0, N_VIRTUAL)), size=num_vv, replace=False)
  anchor_vv = rng.choice(list(range(0, N_VIRTUAL)), size=num_vv, replace=False)
  return dict(idx=idx, anchor=int(anchor), nearest=[idx + o for o in _OFFSETS],
              anchor_nearest=[int(j) for j in np.sort(anchor_ids)], static=[int(j) for j in np.sort(static)],
              vv=[int(j) for j in vv], anchor_vv=[int(j) for j in anchor_vv])


def select_pixels(H, W, N_rand, sample_mode, center_ratio=0.8):
  """RaySamplerSingleImage.sample_random_pixel on the library's sample_ray.rng (sample_ray.py:237-260)."""
  return sample_ray.RaySamplerSingleImage.sample_random_pixel(types.SimpleNamespace(H=H, W=W), N_rand, sample_mode,
                                                              center_ratio)


# ---- the scene ---------------------------------------------------------------------------------------------------

class _Layout(object):
  """Byte offsets of named arrays in one staging buffer, each 16-byte aligned."""

  def __init__(self):
    self.parts, self.nbytes = [], 0

  def add(self, name, dtype, shape):
    n = int(np.prod(shape)) * np.dtype(dtype).itemsize
    self.parts.append((name, dtype, tuple(shape), self.nbytes, n))
    self.nbytes += (n + 15) // 16 * 16


_TORCH = {np.int32: torch.int32, np.int64: torch.int64, np.float32: torch.float32, np.float64: torch.float64}


class MonocularScene(object):
  """A monocular scene (the reference's `dense` folder) on one device.  args: training_height, num_source_views,
  max_range, num_vv, mask_src_view, erosion_radius, init_decay_epoch (the reference's training options)."""

  def __init__(self, scene_path, args, device):
    self.device = torch.device(device)
    if self.device.type != "cuda":
      raise RuntimeError("MonocularScene runs on CUDA only (no CPU fallback)")
    self.scene_path = scene_path
    self.args = args
    self.num_vv = int(args.num_vv)
    self.mask_src_view = bool(args.mask_src_view)
    self.radius = int(args.erosion_radius)
    if not 0 <= self.radius <= 16:
      raise ValueError("MonocularScene: erosion_radius %d, 0..16 supported" % self.radius)
    if not 0 <= self.num_vv <= N_VIRTUAL:
      raise ValueError("MonocularScene: num_vv %d, 0..8" % self.num_vv)
    cams = load_cameras(scene_path, args.training_height)
    self.cams = cams
    n = self.num_frames = len(cams["rgb_files"])
    if n < 7:
      raise ValueError("MonocularScene: %d frames; training draws frames 3 .. n - 4, so at least 7" % n)
    H, W = self.H, self.W = cams["hw"]
    self.current_epoch = 0
    host = self._read(cams)
    self.nbytes = sum(a.nbytes for k, a in host.items() if k not in ("dynamic", "static")) + \
        n * H * W * (2 + host["dynamic"].shape[-1])
    eh, ew = ERODE_H, int(round(ERODE_H * W / H))
    need = self.nbytes + host["dynamic"].nbytes + host["static"].nbytes + n * eh * ew
    free, total = torch.cuda.mem_get_info(self.device)
    if need > free:
      raise MemoryError("MonocularScene: the scene needs %.2f GB on %s while loading, %.2f GB of %.2f GB are free"
                        % (need / 1e9, self.device, free / 1e9, total / 1e9))
    dev = {k: torch.from_numpy(a).to(self.device) for k, a in host.items()}
    mc = dev["dynamic"].shape[-1]
    self._motion = torch.empty(n, H, W, dtype=torch.uint8, device=self.device)
    self._static = torch.empty_like(self._motion)
    self._srcmask = torch.empty(n, H, W, mc, dtype=torch.uint8, device=self.device)
    with torch.cuda.device(self.device):
      ws = torch.empty(max(1, _lib.lib.dyn_scene_masks_workspace_bytes(n, eh, ew)), dtype=torch.uint8,
                       device=self.device)
      d, s = dev.pop("dynamic"), dev.pop("static")
      _lib.check(_lib.lib.dyn_scene_masks(d.data_ptr(), d.shape[1], d.shape[2], mc, s.data_ptr(), s.shape[1],
                                          s.shape[2], n, H, W, eh, ew, self.radius, self._motion.data_ptr(),
                                          self._static.data_ptr(), self._srcmask.data_ptr(), ws.data_ptr(),
                                          ws.numel(), _lib.stream()))
      torch.cuda.current_stream().synchronize()  # the raw masks and the workspace are freed here
    del d, s, ws
    self._frames, self._vviews, self._disp = dev["frames"], dev["vviews"], dev["disp"]
    self._flows, self._flow_masks = dev["flows"], dev["flow_masks"]
    self._scene = _lib.Scene(self._frames.data_ptr(), self._vviews.data_ptr(), self._srcmask.data_ptr(),
                             self._motion.data_ptr(), self._static.data_ptr(), self._disp.data_ptr(),
                             self._flows.data_ptr(), self._flow_masks.data_ptr(), n, H, W, mc, 3, n - 6)
    self._cam_rows = np.concatenate([np.full((n, 2), (H, W), np.float64), cams["K"].reshape(n, 16),
                                     cams["c2w"].reshape(n, 16)], 1).astype(np.float32)
    self._ring = [None] * _RING
    self._turn = 0

  # -- loading --
  def _read(self, cams):
    n, (H, W) = len(cams["rgb_files"]), cams["hw"]
    p = self.scene_path

    def image(path, what):
      a = _imread(path)
      if a.shape != (H, W, 3):
        raise ValueError("MonocularScene: %s %s is %s, the frames are %s" % (what, path, a.shape, (H, W, 3)))
      return a

    frames = np.stack([image(f, "frame") for f in cams["rgb_files"]])
    vdir = os.path.join(p, "source_virtual_views_%dx%d" % (W, H))
    vviews = np.stack([np.stack([image(os.path.join(vdir, "%05d" % i, "%02d.png" % j), "virtual view")
                                 for j in range(N_VIRTUAL)]) for i in range(n)])
    s32 = np.float32(cams["scale"])
    disp = []
    for f in cams["rgb_files"]:
      d = _npload(os.path.join(p, "disp", os.path.basename(f)[:-4] + ".npy"))
      if d.shape != (H, W):
        raise ValueError("MonocularScene: disparity of %s is %s, the frames are %s" % (f, d.shape, (H, W)))
      disp.append((d / s32 if d.dtype == np.float32 else d / cams["scale"]).astype(np.float32))
    dyn = [_imread(os.path.join(p, "dynamic_masks", "%d.png" % i)) for i in range(n)]
    st = [_imread(os.path.join(p, "static_masks", "%d.png" % i)) for i in range(n)]
    if len({m.shape for m in dyn}) != 1 or len({m.shape for m in st}) != 1:
      raise ValueError("MonocularScene: the dynamic (or static) masks differ in size or channels between frames")
    if st[0].ndim != 2:
      raise ValueError("MonocularScene: static masks must be single-channel, got %s" % (st[0].shape,))
    dyn = np.stack(dyn)
    if dyn.ndim == 3:
      dyn = dyn[..., None]
    flows = np.zeros((n - 6, 6, H, W, 2), np.float32)
    fmasks = np.zeros((n - 6, 6, H, W), np.uint8)
    for i in range(3, n - 3):
      for k, o in enumerate(_OFFSETS):
        z = _npload(os.path.join(p, "flow_i%d" % abs(o), "%05d_%s.npz" % (i, "fwd" if o > 0 else "bwd")))
        fl, m = z["flow"], z["mask"]
        if fl.shape != (H, W, 2) or m.shape != (H, W):
          raise ValueError("MonocularScene: flow %d of frame %d is %s / mask %s, the frames are %s"
                           % (o, i, fl.shape, m.shape, (H, W)))
        m32 = np.float32(m)
        if not np.all((m32 == 0) | (m32 == 1)):
          raise ValueError("MonocularScene: flow mask %d of frame %d is not 0 / 1" % (o, i))
        flows[i - 3, k] = fl
        fmasks[i - 3, k] = m32
    return dict(frames=frames, vviews=vviews, disp=np.stack(disp), flows=flows, flow_masks=fmasks, dynamic=dyn,
                static=np.stack(st))

  # -- per step --
  def set_epoch(self, epoch):
    self.current_epoch = epoch

  def __len__(self):
    return self.num_frames

  def _camera(self, c2w, K):
    return np.concatenate(([self.H, self.W], K.reshape(-1), c2w.reshape(-1))).astype(np.float32)

  def _staging(self, nbytes):
    """A pinned buffer of at least nbytes whose previous copy has finished (round robin over _RING buffers)."""
    k = self._turn = (self._turn + 1) % _RING
    slot = self._ring[k]
    if slot is not None:
      slot[1].synchronize()  # the copy of _RING steps ago: long done unless the host runs far ahead
    if slot is None or slot[0].numel() < nbytes:
      slot = (torch.empty(max(nbytes, 1 << 16), dtype=torch.uint8, pin_memory=True), torch.cuda.Event())
      self._ring[k] = slot
    return slot

  def sample(self, rng, N_rand, sample_mode, center_ratio=0.8):
    """One training step's (train_data, ray_batch); see the module docstring."""
    a, c = self.args, self.cams
    ids = draw_views(rng, self.num_frames, self.current_epoch, a.init_decay_epoch, a.num_source_views, a.max_range,
                     self.num_vv, c["c2w"])
    sel = np.asarray(select_pixels(self.H, self.W, N_rand, sample_mode, center_ratio))
    i, an = ids["idx"], ids["anchor"]
    rows, cams = [[], [], []], [[], [], []]
    for j in ids["nearest"]:
      rows[0].append((j, -1, 0)), cams[0].append(self._cam_rows[j])
    for v in ids["vv"]:
      rows[0].append((i, v, 0)), cams[0].append(self._camera(c["vv_c2w"][i, v], c["K"][i]))
    for j in ids["anchor_nearest"]:
      rows[1].append((j, -1, 0)), cams[1].append(self._cam_rows[j])
    for v in ids["anchor_vv"]:  # the target frame's intrinsics (monocular.py:385-388)
      rows[1].append((an, v, 0)), cams[1].append(self._camera(c["vv_c2w"][an, v], c["K"][i]))
    for j in ids["static"]:
      rows[2].append((j, -1, int(self.mask_src_view))), cams[2].append(self._cam_rows[j])
    nv = [len(r) for r in rows]
    V = sum(nv)
    cam = torch.from_numpy(self._cam_rows[i])
    c2w, K = cam[18:34].reshape(4, 4), cam[2:18].reshape(4, 4)
    M = (c2w[:3, :3] @ torch.inverse(K[:3, :3])).numpy()

    L = _Layout()
    L.add("table", np.int32, (V + 1, 4))
    L.add("sel", np.int32, (len(sel),))
    L.add("ray_cam", np.float32, (12,))
    L.add("camera", np.float32, (1, 34))
    L.add("anchor_camera", np.float32, (1, 34))
    for k, n in zip(("src_cameras", "anchor_src_cameras", "static_src_cameras"), nv):
      L.add(k, np.float32, (1, n, 34))
    L.add("depth_range", np.float32, (1, 2))
    for k, shape in (("id", (1,)), ("anchor_id", (1,)), ("num_frames", (1,)), ("nearest_pose_ids", (1, 6)),
                     ("anchor_nearest_pose_ids", (1, len(ids["anchor_nearest"])))):
      L.add(k, np.int64, shape)
    L.add("ref_time", np.float64, (1,))
    L.add("anchor_time", np.float64, (1,))
    pinned, event = self._staging(L.nbytes)
    buf = pinned.numpy()
    view = {name: buf[off:off + n].view(dt).reshape(shape) for name, dt, shape, off, n in L.parts}
    t = view["table"]
    t[:] = 0
    for s, r in enumerate(rows):
      for slot, (f, vv, masked) in enumerate(r):
        t[sum(nv[:s]) + slot] = (f, vv, masked, s << 8 | slot)
    t[V, 0] = i
    view["sel"][:] = sel
    view["ray_cam"][:9], view["ray_cam"][9:] = M.reshape(-1), cam[18:34].reshape(4, 4)[:3, 3].numpy()
    view["camera"][0] = self._cam_rows[i]
    view["anchor_camera"][0] = self._cam_rows[an]
    for k, cs in zip(("src_cameras", "anchor_src_cameras", "static_src_cameras"), cams):
      if cs:
        view[k][0] = np.stack(cs)
    view["depth_range"][0] = c["depth_range"]
    view["id"][0], view["anchor_id"][0], view["num_frames"][0] = i, an, self.num_frames
    view["nearest_pose_ids"][0] = ids["nearest"]
    view["anchor_nearest_pose_ids"][0] = ids["anchor_nearest"]
    view["ref_time"][0] = float(i / float(self.num_frames))
    view["anchor_time"][0] = float(an / float(self.num_frames))

    dev = torch.empty(L.nbytes, dtype=torch.uint8, device=self.device)
    dev.copy_(pinned[:L.nbytes], non_blocking=True)
    event.record()
    d = {name: dev[off:off + n].view(_TORCH[dt]).reshape(shape) for name, dt, shape, off, n in L.parts}

    H, W, R, e = self.H, self.W, len(sel), dict(dtype=torch.float32, device=self.device)
    stacks = [torch.empty(1, n, H, W, 3, **e) for n in nv]
    td = dict(id=d["id"], anchor_id=d["anchor_id"], num_frames=d["num_frames"], ref_time=d["ref_time"],
              anchor_time=d["anchor_time"], nearest_pose_ids=d["nearest_pose_ids"],
              anchor_nearest_pose_ids=d["anchor_nearest_pose_ids"], rgb=torch.empty(1, H, W, 3, **e),
              disp=torch.empty(1, H, W, **e), motion_mask=torch.empty(1, H, W, **e),
              static_mask=torch.empty(1, H, W, **e), flows=torch.empty(1, 6, H, W, 2, **e),
              masks=torch.empty(1, 6, H, W, **e), camera=d["camera"], anchor_camera=d["anchor_camera"],
              rgb_path=[c["rgb_files"][i]], src_rgbs=stacks[0], src_cameras=d["src_cameras"],
              static_src_rgbs=stacks[2], static_src_cameras=d["static_src_cameras"], anchor_src_rgbs=stacks[1],
              anchor_src_cameras=d["anchor_src_cameras"], depth_range=d["depth_range"])
    rb = dict(ray_o=torch.empty(R, 3, **e), ray_d=torch.empty(R, 3, **e), camera=td["camera"],
              anchor_camera=td["anchor_camera"], depth_range=td["depth_range"], rgb=torch.empty(R, 3, **e),
              disp=torch.empty(R, **e), motion_mask=torch.empty(R, **e), static_mask=torch.empty(R, **e),
              uv_grid=torch.empty(R, 2, **e), flows=torch.empty(6, R, 2, **e), masks=torch.empty(6, R, 1, **e),
              src_rgbs=td["src_rgbs"], src_cameras=td["src_cameras"], static_src_rgbs=td["static_src_rgbs"],
              static_src_cameras=td["static_src_cameras"], static_src_masks=None,
              anchor_src_rgbs=td["anchor_src_rgbs"], anchor_src_cameras=td["anchor_src_cameras"],
              selected_inds=sel)
    with torch.cuda.device(self.device):
      st = _lib.stream()
      p = lambda x: x.data_ptr()
      _lib.check(_lib.lib.dyn_scene_views(
          self._scene, p(d["table"]), V, p(stacks[0]), nv[0], p(stacks[1]), nv[1], p(stacks[2]), nv[2], p(td["rgb"]),
          p(td["disp"]), p(td["motion_mask"]), p(td["static_mask"]), p(td["flows"]), p(td["masks"]), st))
      _lib.check(_lib.lib.dyn_scene_rays(
          self._scene, p(d["ray_cam"]), p(d["table"][V]), p(d["sel"]), R, p(rb["ray_o"]), p(rb["ray_d"]),
          p(rb["uv_grid"]), p(rb["rgb"]), p(rb["disp"]), p(rb["motion_mask"]), p(rb["static_mask"]), p(rb["flows"]),
          p(rb["masks"]), st))
    return td, rb

  def get_all(self, train_data):
    """RaySamplerSingleImage(train_data, device).get_all() for a train_data of this scene: every pixel's rays from
    the rays kernel, the rest reshaped from train_data.  For logging a training view: it reads the camera back."""
    cam = train_data["camera"][0].cpu()
    c2w, K = cam[18:34].reshape(4, 4), cam[2:18].reshape(4, 4)
    host = torch.cat([(c2w[:3, :3] @ torch.inverse(K[:3, :3])).reshape(-1), c2w[:3, 3]])
    rc = host.to(self.device)
    HW = self.H * self.W
    e = dict(dtype=torch.float32, device=self.device)
    ray_o, ray_d, uv = torch.empty(HW, 3, **e), torch.empty(HW, 3, **e), torch.empty(HW, 2, **e)
    with torch.cuda.device(self.device):
      _lib.check(_lib.lib.dyn_scene_rays(self._scene, rc.data_ptr(), None, None, HW, ray_o.data_ptr(),
                                         ray_d.data_ptr(), uv.data_ptr(), None, None, None, None, None, None,
                                         _lib.stream()))
    out = dict(ray_o=ray_o, ray_d=ray_d, depth_range=train_data["depth_range"], camera=train_data["camera"],
               render_camera=train_data.get("render_camera"), anchor_camera=train_data.get("anchor_camera"),
               rgb=train_data["rgb"].reshape(-1, 3), disp=train_data["disp"].reshape(-1, 1).squeeze(),
               motion_mask=train_data["motion_mask"].reshape(-1, 1).squeeze(),
               static_mask=train_data["static_mask"].reshape(-1, 1).squeeze(), uv_grid=uv,
               flows=train_data["flows"].squeeze(0).reshape(6, -1, 2),
               masks=train_data["masks"].squeeze(0).reshape(6, -1, 1))
    for k in ("src_rgbs", "src_cameras", "anchor_src_rgbs", "anchor_src_cameras", "static_src_rgbs",
              "static_src_cameras", "static_src_masks"):
      out[k] = train_data.get(k)
    return out

  def loader(self, rng, N_rand, sample_mode, center_ratio=0.8):
    """One epoch: num_frames (train_data, ray_batch) pairs, as train_loader yields num_frames items."""
    for _ in range(self.num_frames):
      yield self.sample(rng, N_rand, sample_mode, center_ratio)
