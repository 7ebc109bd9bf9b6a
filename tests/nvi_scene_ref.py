"""Restatement of the Nvidia evaluation front end (eval_nvidia.py DynamicVideoDataset.__getitem__ and the ground-truth /
mask reads of its __main__ block, :92-198, :383-428) with numpy, for tests/test_nvi_scene_*.py,
tests/golden/make_golden_nvi_scene.py and tools/nvidia_eval_bench.py.

cv2.resize(INTER_AREA) is restated from OpenCV's resize (4.x, the version installed beside the tests):
  integer factors in both axes   resizeAreaFast: the integer box sum s over the a = fy fx source pixels; at 2 x 2
                                 rounded half up, (s + 2) >> 2 (its vector path), at every other factor
                                 float32(s) * (1.f / a) rounded to nearest even;
  any other factor               resizeArea: computeResizeAreaTab's tables in double (scale = 1 / (dst / src), alpha
                                 stored as float32, slivers of <= 1e-3 dropped); each output accumulates the
                                 horizontal weights in table order, then the vertical ones, float32 products and sums
                                 without contraction, rounded to nearest even at the end.
A factor of 1 in both axes is a copy.  The tests check both rules against cv2 itself.

`plant` selects a deliberate error (PLANTS) so the tests can show the comparison would catch it.
"""

import collections
import os

import cv2
import numpy as np
import torch

import mono_scene_ref as msr

PLANTS = ("int_half_even", "float_path_at_int", "float64_accumulate", "mask_rgb_order", "keep_held_out",
          "static_wrong_residue", "target_pose_of_img_i")
CYCLE = 12  # eval_nvidia.py:96: cameras of the benchmark's round robin


# ---- INTER_AREA -------------------------------------------------------------------------------------------------

def area_table(ssize, dsize):
  """computeResizeAreaTab -> list over destination index of [(source index, float32 alpha), ...] in table order."""
  scale = 1.0 / (float(dsize) / ssize)
  out = []
  for dx in range(dsize):
    fsx1 = dx * scale
    fsx2 = fsx1 + scale
    cell = min(scale, ssize - fsx1)
    sx1, sx2 = int(np.ceil(fsx1)), int(np.floor(fsx2))
    sx2 = min(sx2, ssize - 1)
    sx1 = min(sx1, sx2)
    row = []
    if sx1 - fsx1 > 1e-3:
      row.append((sx1 - 1, np.float32((sx1 - fsx1) / cell)))
    for sx in range(sx1, sx2):
      row.append((sx, np.float32(1.0 / cell)))
    if fsx2 - sx2 > 1e-3:
      row.append((sx2, np.float32(min(min(fsx2 - sx2, 1.0), cell) / cell)))
    out.append(row)
  return out


def _area_float(src, dh, dw, acc=np.float32):
  sh, sw = src.shape[:2]
  s = src.astype(acc)
  xt, yt = area_table(sw, dw), area_table(sh, dh)
  buf = np.zeros((sh, dw) + src.shape[2:], acc)
  for k in range(max(len(r) for r in xt)):
    dxs = [dx for dx, r in enumerate(xt) if len(r) > k]
    sxs = [xt[dx][k][0] for dx in dxs]
    a = np.array([xt[dx][k][1] for dx in dxs], acc).reshape((1, -1) + (1,) * (src.ndim - 2))
    buf[:, dxs] = buf[:, dxs] + s[:, sxs] * a
  out = np.zeros((dh, dw) + src.shape[2:], acc)
  for dy, r in enumerate(yt):
    for k, (sy, beta) in enumerate(r):
      t = acc(beta) * buf[sy]
      out[dy] = t if k == 0 else out[dy] + t
  return np.clip(np.rint(out), 0, 255).astype(np.uint8)


def area_resize(src, dh, dw, plant=None):
  """cv2.resize(src, (dw, dh), interpolation=cv2.INTER_AREA) for uint8 src [sh, sw(, C)] with sh >= dh, sw >= dw."""
  sh, sw = src.shape[:2]
  if sh < dh or sw < dw:
    raise ValueError("area_resize: upscaling is not restated")
  if (sh, sw) == (dh, dw):
    return src.copy()
  if sh % dh == 0 and sw % dw == 0 and plant != "float_path_at_int":
    fy, fx = sh // dh, sw // dw
    s = src.astype(np.int64).reshape((dh, fy, dw, fx) + src.shape[2:]).sum((1, 3))
    a = fy * fx
    if fy == 2 and fx == 2 and plant != "int_half_even":  # the 2 x 2 vector path: (s + 2) >> 2
      return ((s + 2) >> 2).astype(np.uint8)
    # every other integer factor: saturate_cast<uchar>(sum * (1.f / area)), float32, half to even
    return np.clip(np.rint(s.astype(np.float32) * (np.float32(1) / np.float32(a))), 0, 255).astype(np.uint8)
  return _area_float(src, dh, dw, np.float64 if plant == "float64_accumulate" else np.float32)


# ---- the ground truth and masks of one camera (eval_nvidia.py:387-393, :416-428) ----------------------------------

def gt_image(bgr, H, W, plant=None):
  """cv2.imread(...)[:, :, ::-1], INTER_AREA to (H, W), float32 / 255."""
  return np.float32(area_resize(np.ascontiguousarray(bgr[:, :, ::-1]), H, W, plant)) / np.float32(255)


def dynamic_mask(bgr, H, W, plant=None):
  """np.float32(cv2.imread(path) > 1e-3) (BGR, never reversed), INTER_NEAREST to (H, W)."""
  m = bgr[:, :, ::-1] if plant == "mask_rgb_order" else bgr
  return cv2.resize(np.float32(m > 1e-3), (W, H), interpolation=cv2.INTER_NEAREST)


def coarse_mask(u8, H, W):
  """imageio.v2.imread(...).astype(np.float32) / 255.0, INTER_NEAREST to (H, W)."""
  return cv2.resize(u8.astype(np.float32) / 255.0, (W, H), interpolation=cv2.INTER_NEAREST)


# ---- view selection (eval_nvidia.py:92-119) ---------------------------------------------------------------------

def static_ids(img_i, n, plant=None):
  held = (img_i + 1) % CYCLE if plant == "static_wrong_residue" else img_i % CYCLE
  groups = collections.defaultdict(list)
  for j in range(n):
    if j % CYCLE != held:
      groups[j % CYCLE].append(j)
  return sorted(int(g[int(np.argmin(np.abs(np.array(g) - img_i)))]) for g in groups.values())


def target_cameras(img_i, plant=None):
  return [i for i in range(CYCLE) if plant == "keep_held_out" or i != img_i % CYCLE]


# ---- a synthetic Nvidia scene in the reference's layout ----------------------------------------------------------

def _discs(rng, h, w, values):
  """uint8 [h, w]: 0 background with three discs, each of one value from `values`."""
  ys, xs = np.mgrid[0:h, 0:w]
  out = np.zeros((h, w), np.uint8)
  for v in rng.choice(values, size=3):
    cy, cx, r = rng.uniform(0, h), rng.uniform(0, w), rng.uniform(0.15, 0.4) * max(h, w)
    out[((ys - cy) * w / h) ** 2 + (xs - cx) ** 2 <= (r * w / max(h, w)) ** 2] = v
  return out


def _waves(rng, h, w):
  """uint8 [h, w, 3]: two seeded low-frequency waves per channel."""
  ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
  ch = []
  for _ in range(3):
    f, ph = rng.uniform(0.005, 0.03, 2), rng.uniform(0, 2 * np.pi, 2)
    ch.append(128 + 60 * np.sin(ys * f[0] + ph[0]) + 40 * np.sin((3 * xs + ys) * f[1] + ph[1]))
  return np.clip(np.stack(ch, -1), 0, 255).astype(np.uint8)


def synthetic_scene(seed, n, h, w, gt_hw, mask_hw, coarse_hw, coloured_masks, levels=4):
  """Raw arrays of a seeded scene of n frames of h x w, CYCLE cameras per time step.  gt_hw: one (gh, gw) per camera
  (cycled); ground truth is a seeded sum of waves per channel, smooth so that its JPEGs stay small."""
  base = msr.synthetic_scene(seed, n, h, w, orig_hw=(2 * h, 2 * w), levels=levels)
  rng = np.random.default_rng(seed + 1000)
  gts, masks = [], []
  for t in range(n):
    gts.append([]), masks.append([])
    for c in range(CYCLE):
      gh, gw = gt_hw[c % len(gt_hw)]
      gts[t].append(_waves(rng, gh, gw))
      m = _discs(rng, mask_hw[0], mask_hw[1], (1, 90, 255))
      if coloured_masks:
        m = np.stack([m, np.roll(m, 2, 1), np.where(m > 0, 0, 200).astype(np.uint8)], -1)
      else:
        m = np.repeat(m[..., None], 3, -1)
      masks[t].append(m.astype(np.uint8))
  coarse = msr._blobs(rng, n, coarse_hw[0], coarse_hw[1], np.array([0, 51, 128, 255]))
  return dict(poses_bounds=base["poses_bounds"], frames=base["frames"], orig=base["orig"], gt=gts, masks=masks,
              coarse=coarse)


def write_scene(root, s):
  """The reference's Nvidia layout under root (= <folder_path>/<scene>/dense): returns root."""
  n, h, w = s["frames"].shape[:3]
  img = os.path.join(root, "images_%dx%d" % (w, h))
  for d in ("images", img, "coarse_masks"):
    os.makedirs(os.path.join(root, d), exist_ok=True)
  msr.write_png(os.path.join(root, "images", "00000.png"), s["orig"])
  np.save(os.path.join(root, "poses_bounds_cvd.npy"), s["poses_bounds"])
  for i in range(n):
    msr.write_png(os.path.join(img, "%05d.png" % i), s["frames"][i])
    msr.write_png(os.path.join(root, "coarse_masks", "%05d.png" % i), s["coarse"][i])
    gd = os.path.join(root, "mv_images", "%05d" % i)
    md = os.path.join(root, "mv_masks", "%05d" % i)
    os.makedirs(gd, exist_ok=True)
    os.makedirs(md, exist_ok=True)
    for c in range(CYCLE):
      cv2.imwrite(os.path.join(gd, "cam%02d.jpg" % (c + 1)), s["gt"][i][c], [cv2.IMWRITE_JPEG_QUALITY, 75])
      cv2.imwrite(os.path.join(md, "cam%02d.png" % (c + 1)), s["masks"][i][c])
  return root


# ---- the stand-in renderer's prediction and the script's printed scores ------------------------------------------

def prediction(img_i, cam, H, W):
  """A seeded float32 prediction [H, W, 3] per (time step, camera), about 10 % of its pixels all zero."""
  rng = np.random.default_rng(1000 * img_i + cam)
  p = rng.random((H, W, 3), dtype=np.float32)
  p[rng.random((H, W)) < 0.1] = 0
  return p


def printed_scores(text):
  """eval_nvidia.py's stdout -> (per-camera dict {(img_i, cam): float64 [3, 2]}, {line label: value})."""
  per, avg, cur, rows = {}, {}, None, []
  for line in text.splitlines():
    f = line.split()
    if line.startswith("img_i "):
      cur, rows = (int(f[1]), int(f[2])), []
    elif line.startswith(("MOVING", "AVG")):
      avg.setdefault(" ".join(f[:-1]), []).append(float(f[-1]))
    elif cur is not None and len(f) == 3 and len(rows) < 3:
      try:
        rows.append([float(f[0]), float(f[1])])
      except ValueError:
        continue
      if len(rows) == 3:
        per[cur] = np.array(rows)
  return per, avg


# ---- one collated item (eval_nvidia.py:71-198 under the DataLoader) -----------------------------------------------

def _read_frame(root, j, hw):
  from PIL import Image
  H, W = hw
  return np.asarray(Image.open(os.path.join(root, "images_%dx%d" % (W, H), "%05d.png" % j)))[..., :3]


def item(root, img_i, cam, n, K, c2w, depth_range, mask_static, plant=None):
  """The DataLoader's collated item for target camera `cam` at img_i, restated: torch tensors on the host.
  K, c2w [n,4,4] float64 are the scene's (the fixture's); depth_range [2] as the reference's environment gives it."""
  from PIL import Image
  H, W = _read_frame(root, 0, _hw(root)).shape[:2]
  camera = lambda j: np.concatenate(([H, W], K[j].flatten(), c2w[j].flatten())).astype(np.float32)
  dyn = sorted(img_i + o for o in (1, 2, 3, 0, -1, -2, -3))
  st = static_ids(img_i, n, plant)
  rgb = lambda j: _read_frame(root, j, (H, W)).astype(np.float32) / 255.0
  masks = []
  for j in st:
    if mask_static and 3 <= j < n - 3:
      masks.append(coarse_mask(np.asarray(Image.open(os.path.join(root, "coarse_masks", "%05d.png" % j))), H, W))
    else:
      masks.append(np.ones((H, W), np.float32))
  t = lambda a: torch.from_numpy(np.ascontiguousarray(np.stack(a)))[None].float()
  target = img_i if plant == "target_pose_of_img_i" else cam
  return dict(camera=torch.from_numpy(camera(target))[None], src_rgbs=t([rgb(j) for j in dyn]),
              src_cameras=t([camera(j) for j in dyn]), static_src_rgbs=t([rgb(j) for j in st]),
              static_src_cameras=t([camera(j) for j in st]), static_src_masks=t(masks),
              depth_range=torch.as_tensor(np.asarray(depth_range))[None], ref_time=torch.tensor([img_i / float(n)],
                                                                                                   dtype=torch.float64),
              id=torch.tensor([img_i]), nearest_pose_ids=torch.tensor([dyn]),
              rgb_path=[os.path.join(root, "mv_images", "%05d" % img_i, "cam%02d.jpg" % (cam + 1))])


def _hw(root):
  d = [x for x in os.listdir(root) if x.startswith("images_")][0]
  W, H = d[len("images_"):].split("x")
  return int(H), int(W)


def ground_truth(root, img_i, cams, H, W, plant=None):
  """The ground truth [K, H, W, 3] float32 and dynamic masks [K, H, W, 3] float32 of the cameras, as eval_nvidia.py
  reads them (cv2 on the host)."""
  gt, dm = [], []
  for c in cams:
    gt.append(gt_image(cv2.imread(os.path.join(root, "mv_images", "%05d" % img_i, "cam%02d.jpg" % (c + 1))), H, W,
                       plant))
    dm.append(dynamic_mask(cv2.imread(os.path.join(root, "mv_masks", "%05d" % img_i, "cam%02d.png" % (c + 1))), H, W,
                           plant))
  return np.stack(gt), np.stack(dm)


def write_files(root, files):
  """A fixture's scene (relative path -> bytes) under root; returns root."""
  for rel, data in files.items():
    p = os.path.join(root, rel)
    os.makedirs(os.path.dirname(p), exist_ok=True)
    with open(p, "wb") as f:
      f.write(data)
  return root


# ---- the fixture's storage form ----------------------------------------------------------------------------------

def pack_masks(masks):
  """A list of {0, 1} masks of one shape -> (zlib of their packed bits, stacked shape)."""
  import zlib
  a = np.stack(masks) != 0
  return zlib.compress(np.packbits(a.reshape(-1)).tobytes(), 9), a.shape


def unpack_masks(packed):
  import zlib
  b, shape = packed
  bits = np.unpackbits(np.frombuffer(zlib.decompress(b), np.uint8))[:int(np.prod(shape))]
  return list(bits.reshape(shape).astype(np.float32))


def load_golden(path):
  """tests/golden/nvi_scene.pt with tensors back, per scene `items`: one record per (time step, camera) of the
  recorded time steps (the step's shared fields plus img_i, cam, camera [1, 34] and rgb_path; `rays` on the recorded
  camera), and `dynamic_masks` unpacked to float32 arrays."""
  g = msr.load_golden(path)
  for s in g["scenes"].values():
    items = []
    for img_i, step in sorted(s.pop("steps").items()):
      for cam in range(len(step["rgb_path"])):
        it = {k: v for k, v in step.items() if k not in ("camera", "rgb_path", "rays")}
        it.update(img_i=img_i, cam=cam, camera=step["camera"][cam][None], rgb_path=step["rgb_path"][cam])
        if "rays" in step and int(step["rays"]["cam"]) == cam:
          it["rays"] = step["rays"]
        items.append(it)
    s["items"] = items
    s["dynamic_masks"] = unpack_masks(s["dynamic_masks"])
  return g
