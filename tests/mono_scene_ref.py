"""Restatement of the monocular training loader (ibrnet/data_loaders/monocular.py MonocularDataset.__getitem__ and
ibrnet/sample_ray.py random_sample) with cv2, scipy and PIL, for tests/test_mono_scene_*.py, tests/golden/
make_golden_scene.py and tools/train_scene_bench.py.

skimage and imageio are not installed here, so their parts are restated from their definitions:
  disk(r)            skimage.morphology.disk: X^2 + Y^2 <= r^2 on a (2r+1)^2 grid;
  erosion(m, fp)     skimage 0.19.3 erosion = scipy.ndimage.grey_erosion(m, footprint=fp), mode 'reflect';
  imread             imageio 2.22 reads PNG through PIL.
cv2.resize(INTER_NEAREST) is called as it is.

Also here: a seeded synthetic scene in the reference's layout (`synthetic_scene`, `write_scene`), so the fixture,
the tests and the benchmark write the same files.

`plant` selects a deliberate error (PLANTS) so the tests can show the comparison bars would catch it.
"""

import os

import cv2
import numpy as np
import scipy.ndimage as ndi
import torch

PLANTS = ("square_footprint", "nearest_border", "src_over_dst", "ge_threshold", "static_unthresholded",
          "erode_at_frame_height", "source_mask_thresholded", "swapped_anchor_pool", "anchor_keeps_idx")
ERODE_H = 288  # monocular.py:186: the motion mask is eroded at height 288 whatever training_height is


# ---- synthetic scene --------------------------------------------------------------------------------------------

def _rot(rng, scale):
  a = rng.normal(size=3) * scale
  t = np.linalg.norm(a)
  K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]]) / max(t, 1e-12)
  return np.eye(3) + np.sin(t) * K + (1 - np.cos(t)) * K @ K


def _blobs(rng, n, h, w, levels):
  """uint8 masks [n, h, w]: 255 background with random discs of values drawn from `levels`."""
  ys, xs = np.mgrid[0:h, 0:w]
  out = np.full((n, h, w), 255, np.uint8)
  for i in range(n):
    for _ in range(3):
      cy, cx = rng.uniform(0, h), rng.uniform(0, w)
      r = rng.uniform(0.1, 0.35) * max(h, w)
      ry = r * (h / max(h, w)) if h < w else r
      rx = r * (w / max(h, w)) if w < h else r
      inside = ((ys - cy) / max(ry, 1)) ** 2 + ((xs - cx) / max(rx, 1)) ** 2 <= 1
      out[i][inside] = rng.choice(levels, size=int(inside.sum()))
  return out


def synthetic_scene(seed, n, h, w, mask_hw=None, orig_hw=None, mask_channels=0, far_max=8.0, levels=16):
  """Raw arrays of a seeded scene of n frames of h x w.  Colours take `levels` values so the fixture compresses."""
  rng = np.random.default_rng(seed)
  mh, mw = mask_hw or (h, w)
  oh, ow = orig_hw or (2 * h, 2 * w)
  q = lambda lv, *s: (rng.integers(0, lv, size=s) * (255 // (lv - 1))).astype(np.uint8)
  poses = np.zeros((n, 17))
  c2ws = []
  for i in range(n):
    c2w = np.eye(4)
    c2w[:3, :3] = _rot(rng, 0.05)
    c2w[:3, 3] = np.array([0.05 * i, 0.01 * np.sin(i), 0.02 * np.cos(i)]) + rng.normal(size=3) * 0.01
    c2ws.append(c2w)
    p = np.concatenate([c2w[:3, :4], np.array([[oh], [ow], [0.9 * max(h, w)]])], 1)
    poses[i, :15] = p.reshape(-1)
    poses[i, 15:] = [rng.uniform(1.0, 2.0), rng.uniform(far_max * 0.6, far_max)]
  vv = np.zeros((8, 3, 4, n), np.float32)
  for i in range(n):
    for j in range(8):
      c = c2ws[i].copy()
      c[:3, :3] = c[:3, :3] @ _rot(rng, 0.02)
      c[:3, 3] += rng.normal(size=3) * 0.03
      vv[j, :, :, i] = c[:3, :4]
  dyn = _blobs(rng, n, mh, mw, np.array([0, 0, 0, 40, 128, 200, 254]))
  if mask_channels == 3:
    dyn = np.stack([dyn, np.roll(dyn, 1, 2), 255 - (255 - dyn) // 2], -1)
  return dict(
      poses_bounds=poses, vv_poses=vv,
      frames=q(levels, n, h, w, 3), vviews=q(4, n, 8, h, w, 3), orig=np.zeros((oh, ow, 3), np.uint8),
      disp=(rng.integers(1, 64, size=(n, h, w)) / 32.0).astype(np.float32),
      dynamic=dyn, static=_blobs(rng, n, mh, mw, np.array([0, 100, 254])),
      flows=(rng.integers(-2, 3, size=(n, 6, h, w, 2)) * np.float32(0.75)).astype(np.float32),
      flow_masks=rng.integers(0, 2, size=(n, 6, h, w)).astype(bool))


def write_png(path, arr):
  from PIL import Image
  Image.fromarray(arr).save(path, format="PNG")


def write_scene(root, s):
  """The reference's layout under root (= <folder_path>/<scene>/dense): returns root."""
  n, h, w = s["frames"].shape[:3]
  img = os.path.join(root, "images_%dx%d" % (w, h))
  for d in ("images", img, "disp", "dynamic_masks", "static_masks", "flow_i1", "flow_i2", "flow_i3"):
    os.makedirs(os.path.join(root, d), exist_ok=True)
  write_png(os.path.join(root, "images", "00000.png"), s["orig"])
  np.save(os.path.join(root, "poses_bounds_cvd.npy"), s["poses_bounds"])
  np.save(os.path.join(root, "source_vv_poses.npy"), s["vv_poses"])
  for i in range(n):
    write_png(os.path.join(img, "%05d.png" % i), s["frames"][i])
    vd = os.path.join(root, "source_virtual_views_%dx%d" % (w, h), "%05d" % i)
    os.makedirs(vd, exist_ok=True)
    for j in range(8):
      write_png(os.path.join(vd, "%02d.png" % j), s["vviews"][i, j])
    np.save(os.path.join(root, "disp", "%05d.npy" % i), s["disp"][i])
    write_png(os.path.join(root, "dynamic_masks", "%d.png" % i), s["dynamic"][i])
    write_png(os.path.join(root, "static_masks", "%d.png" % i), s["static"][i])
    if 3 <= i < n - 3:  # the frames __getitem__ can draw read flows at 1, 2, 3 frames in both directions
      for k, (fwd, step) in enumerate([(True, 1), (True, 2), (True, 3), (False, 1), (False, 2), (False, 3)]):
        np.savez(os.path.join(root, "flow_i%d" % step, "%05d_%s.npz" % (i, "fwd" if fwd else "bwd")),
                 flow=s["flows"][i, k], mask=s["flow_masks"][i, k])
  return root


# ---- image operations -------------------------------------------------------------------------------------------

def imread(path):
  from PIL import Image
  return np.asarray(Image.open(path))


def resize_nn(a, w, h, plant=None):
  """cv2.resize(a, (w, h), INTER_NEAREST); plant 'src_over_dst' maps with src / dst instead of cv2's 1 / (dst / src)."""
  if plant != "src_over_dst":
    return cv2.resize(a, (w, h), interpolation=cv2.INTER_NEAREST)
  sh, sw = a.shape[:2]
  ys = np.minimum(np.floor(np.arange(h) * (sh / h)).astype(int), sh - 1)
  xs = np.minimum(np.floor(np.arange(w) * (sw / w)).astype(int), sw - 1)
  return a[ys][:, xs]


def resize_nn_index(src, dst):
  """cv2's resizeNN source index of each destination index, restated: min(floor(x * (1 / (dst / src))), src - 1)."""
  ifx = 1.0 / (float(dst) / src)
  return np.minimum(np.floor(np.arange(dst) * ifx).astype(np.int64), src - 1)


def disk(r):
  L = np.arange(-r, r + 1)
  X, Y = np.meshgrid(L, L)
  return (X ** 2 + Y ** 2 <= r ** 2).astype(np.uint8)


def erosion(mask, r, plant=None):
  fp = np.ones((2 * r + 1, 2 * r + 1), np.uint8) if plant == "square_footprint" else disk(r)
  mode = "nearest" if plant == "nearest_border" else "reflect"
  return ndi.grey_erosion(mask, footprint=fp, mode=mode)


def motion_mask(m, h, w, r, plant=None):
  """monocular.py:164-203: uint8 dynamic mask [mh, mw(, C)] -> float32 {0, 1} [h, w]."""
  x = np.float32(1.0) - m.astype(np.float32) / np.float32(255.0)
  eh = h if plant == "erode_at_frame_height" else ERODE_H
  x = resize_nn(x, int(round(eh * w / h)), eh, plant)
  if x.ndim == 3:
    x = x[..., 0]
  b = (x >= np.float32(1e-3)) if plant == "ge_threshold" else (x > np.float32(1e-3))
  e = erosion(b, r, plant)
  return np.float32(resize_nn(np.float32(e), w, h, plant))


def static_mask(s, h, w, plant=None):
  """monocular.py:170-181, :204."""
  x = np.float32(1.0) - s.astype(np.float32) / np.float32(255.0)
  x = resize_nn(x, w, h, plant)
  if plant == "static_unthresholded":
    return np.float32(x)
  if plant == "ge_threshold":
    return np.float32(x >= np.float32(1e-3))
  return np.float32(x > np.float32(1e-3))


def source_mask(m, h, w, plant=None):
  """load_src_view's mask (monocular.py:131-142): m / 255, not thresholded, nearest to the frame size, [h, w, 1 or 3]."""
  x = resize_nn(m.astype(np.float32) / np.float32(255.0), w, h, plant)
  if plant == "source_mask_thresholded":
    x = np.float32(x > np.float32(1e-3))
  return x[..., None] if x.ndim == 2 else x


MASK_SIZES = [(288, 512, 288, 512), (288, 512, 540, 960), (288, 512, 144, 256), (37, 53, 29, 61), (24, 40, 30, 50),
              (24, 40, 22, 26), (288, 7, 288, 7), (5, 3, 11, 2)]  # (H, W) of the frames, (mh, mw) of the mask files


def mask_inputs(H, W, mh, mw, channels, n=3):
  """Seeded dynamic masks (random, blob, all-ones motion) and a static mask for the mask-kernel tests."""
  rng = np.random.default_rng(H * 1000 + W + mh + channels)
  rand = rng.choice(np.array([0, 17, 128, 254, 255], np.uint8), size=(n, mh, mw), p=[.2, .1, .1, .1, .5])
  blob = _blobs(rng, n, mh, mw, np.array([0, 40, 200, 254]))
  ones = np.zeros((n, mh, mw), np.uint8)  # 1 - 0 / 255: the motion mask is all ones
  out = []
  for kind, dyn in (("random", rand), ("blob", blob), ("ones", ones)):
    if channels == 3:
      dyn = np.stack([dyn, np.roll(dyn, 1, 1), 255 - dyn], -1)
    out.append((kind, dyn, np.roll(blob, 2, 2)))
  return out


# ---- view selection ---------------------------------------------------------------------------------------------

def draw_ids(rng, n, epoch, cfg, c2w, plant=None):
  """__getitem__'s draws in its order (monocular.py:148, :217-244, :269-298, :313-315, :375-377) -> dict of ids."""
  idx = int(rng.randint(3, n - 3))
  max_step = min(3, epoch // cfg["init_decay_epoch"] + 1)
  pool = list(range(1, max_step + 1)) + [-i for i in range(1, max_step + 1)]
  if plant == "swapped_anchor_pool":
    pool = [-i for i in range(1, max_step + 1)] + list(range(1, max_step + 1))
  anchor = idx + pool[rng.choice(len(pool))]
  anchor_ids = [anchor + o for o in [3, 2, 1, 0, -1, -2, -3]
                if 0 <= anchor + o < n and (anchor + o != idx or plant == "anchor_keeps_idx")]
  if rng.choice([0, 1], p=[1.0 - 0.005, 0.005]):
    anchor_ids.append(idx)
  anchor_ids = np.sort(anchor_ids)
  d = np.linalg.norm(c2w[idx][None, :3, 3].repeat(n, 0) - c2w[:, :3, 3], axis=1)
  d[idx] = 1e3
  sp = np.argsort(d)
  ns = cfg["num_source_views"]
  max_interval = cfg["max_range"] // ns
  interval = rng.randint(max(2, max_interval - 2), max_interval + 1)
  static = []
  for ii in range(-ns, ns):
    s = idx + interval * ii + rng.randint(1, interval + 1)
    if 0 <= s < n and s != idx:
      static.append(s)
  seen = set(static)
  for s in sp[::5]:
    if len(static) >= 2 * ns:
      break
    if s not in seen:
      static.append(s)
  vv = rng.choice(list(range(0, 8)), size=cfg["num_vv"], replace=False)
  anchor_vv = rng.choice(list(range(0, 8)), size=cfg["num_vv"], replace=False)
  return dict(idx=idx, anchor=int(anchor), nearest=[idx + o for o in [1, 2, 3, -1, -2, -3]],
              anchor_nearest=[int(a) for a in anchor_ids], static=[int(s) for s in np.sort(static)],
              vv=[int(v) for v in vv], anchor_vv=[int(v) for v in anchor_vv])


def select_pixels(rng, H, W, N_rand, sample_mode, center_ratio=0.8):
  """sample_ray.py:237-260."""
  if sample_mode == "center":
    bH, bW = int(H * (1 - center_ratio) / 2.0), int(W * (1 - center_ratio) / 2.0)
    u, v = np.meshgrid(np.arange(bH, H - bH), np.arange(bW, W - bW))
    u, v = u.reshape(-1), v.reshape(-1)
    sel = rng.choice(u.shape[0], size=(N_rand,), replace=False)
    return v[sel] + W * u[sel]
  if sample_mode == "uniform":
    return rng.choice(H * W, size=(N_rand,), replace=False)
  raise NotImplementedError


# ---- the item ---------------------------------------------------------------------------------------------------

class Item(object):
  """__getitem__ on a scene's raw arrays (synthetic_scene's dict) given its cameras (from the fixture or the library).

  cams: dict c2w [n,4,4], K [n,4,4], vv_c2w [n,8,4,4] (float64, as batch_parse_*_poses give them), scale (float),
  depth_range float32 [2]."""

  def __init__(self, s, cams, cfg, plant=None):
    self.s, self.cams, self.cfg, self.plant = s, cams, cfg, plant
    self.n, self.h, self.w = s["frames"].shape[:3]

  def camera(self, c2w, K):
    return np.concatenate(([self.h, self.w], K.flatten(), c2w.flatten())).astype(np.float32)

  def view(self, img, c2w, K, mask=None):
    rgb = img.astype(np.float32) / np.float32(255.0)
    if mask is not None:
      rgb = rgb * source_mask(mask, self.h, self.w, self.plant)
    return rgb, self.camera(c2w, K)

  def __call__(self, rng, epoch):
    s, c, cfg, p = self.s, self.cams, self.cfg, self.plant
    ids = draw_ids(rng, self.n, epoch, cfg, c["c2w"], p)
    i, a = ids["idx"], ids["anchor"]
    K = c["K"][i]
    out = dict(ids=ids)
    out["rgb"], out["camera"] = self.view(s["frames"][i], c["c2w"][i], K)
    out["anchor_camera"] = self.camera(c["c2w"][a], c["K"][a])
    out["disp"] = s["disp"][i] / np.float32(c["scale"])
    out["motion_mask"] = motion_mask(s["dynamic"][i], self.h, self.w, cfg["erosion_radius"], p)
    out["static_mask"] = static_mask(s["static"][i], self.h, self.w, p)
    out["flows"], out["masks"] = s["flows"][i], s["flow_masks"][i].astype(np.float32)
    views = lambda lst: [np.stack(x) for x in zip(*lst)]
    out["src_rgbs"], out["src_cameras"] = views(
        [self.view(s["frames"][j], c["c2w"][j], c["K"][j]) for j in ids["nearest"]] +
        [self.view(s["vviews"][i, v], c["vv_c2w"][i, v], K) for v in ids["vv"]])
    out["static_src_rgbs"], out["static_src_cameras"] = views(
        [self.view(s["frames"][j], c["c2w"][j], c["K"][j], s["dynamic"][j] if cfg["mask_src_view"] else None)
         for j in ids["static"]])
    out["anchor_src_rgbs"], out["anchor_src_cameras"] = views(
        [self.view(s["frames"][j], c["c2w"][j], c["K"][j]) for j in ids["anchor_nearest"]] +
        [self.view(s["vviews"][a, v], c["vv_c2w"][a, v], K) for v in ids["anchor_vv"]])
    out["depth_range"] = np.asarray(c["depth_range"], np.float32)
    return out


def rays(camera, sel):
  """sample_ray.py:143-163 for the selected pixels: float32 torch on the host, as the reference."""
  cam = torch.as_tensor(camera).float().reshape(1, 34)
  H, W = int(cam[0, 0]), int(cam[0, 1])
  K, c2w = cam[:, 2:18].reshape(1, 4, 4), cam[:, 18:34].reshape(1, 4, 4)
  u, v = np.meshgrid(np.arange(W), np.arange(H))
  pix = torch.from_numpy(np.stack((u.reshape(-1), v.reshape(-1), np.ones(H * W)), 0).astype(np.float32))[None]
  d = c2w[:, :3, :3].bmm(torch.inverse(K[:, :3, :3])).bmm(pix).transpose(1, 2).reshape(-1, 3)
  sel = torch.as_tensor(np.asarray(sel, np.int64))
  return c2w[0, :3, 3][None].repeat(len(sel), 1), d[sel]


def to_numpy(obj):
  """Every tensor in nested dicts / lists / tuples -> numpy array (the fixture's storage form)."""
  if torch.is_tensor(obj):
    return obj.numpy()
  if isinstance(obj, dict):
    return {k: to_numpy(v) for k, v in obj.items()}
  if isinstance(obj, (list, tuple)):
    return type(obj)(to_numpy(v) for v in obj)
  return obj


def _to_torch(obj):
  if isinstance(obj, np.ndarray):
    return torch.from_numpy(obj)
  if isinstance(obj, dict):
    return {k: _to_torch(v) for k, v in obj.items()}
  if isinstance(obj, (list, tuple)):
    return type(obj)(_to_torch(v) for v in obj)
  return obj


def load_golden(path):
  """tests/golden/mono_scene.pt with its numpy arrays back as tensors."""
  return _to_torch(torch.load(path, weights_only=False))


def pack_mask(m):
  """A {0, 1} mask [H, W] (tensor or array) -> (bit-packed uint8 bytes, shape), as the fixture stores masks."""
  a = np.asarray(torch.as_tensor(m).detach().cpu().numpy()) != 0
  return np.packbits(a.reshape(-1)).tobytes(), a.shape


def unpack_mask(packed):
  """pack_mask's inverse -> float32 {0, 1} [H, W]."""
  b, shape = packed
  return np.unpackbits(np.frombuffer(b, np.uint8))[:int(np.prod(shape))].reshape(shape).astype(np.float32)


def hash_f32(t):
  import hashlib
  a = np.ascontiguousarray(torch.as_tensor(t).detach().cpu().float().numpy())
  return hashlib.sha256(a.tobytes()).hexdigest()
