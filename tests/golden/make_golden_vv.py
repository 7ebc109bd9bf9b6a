"""tests/golden/virtual_views.pt: the reference's render_source_vv.py, run unmodified, on a seeded synthetic scene
(run where the reference is, as make_golden.py):

    python tests/golden/make_golden_vv.py

The script's __main__ runs with runpy on the CPU.  Four modules it imports cannot run here and are replaced:
  splatting  splatting_function computes tests/virtual_views_ref.splat64 (the extension's restated forward) and
             records its inputs (input_data, flow, weights);
  kornia     filters.spatial_gradient returns the unnormalised Sobel gradients of a replicate-padded plane (float64,
             returned as the input's dtype) and records the plane;
  skimage    morphology.disk(1) / erosion as skimage 0.19.3 computes them: scipy.ndimage.grey_erosion, cross footprint;
  imageio    imread reads the first image's shape, imsave records the PNG bytes it writes.
torch.Tensor.cuda is the identity, and cv2.resize is wrapped to record the resized inputs.  The fixture therefore pins
all of the script's own glue (cameras, poses, resizing, projection, weights, the rgba layout, masking and
quantisation); the splat, the Sobel filter and the erosion are pinned by their restatements only.

The output height is fixed at 288 (FINAL_H); a 288 x 10 frame keeps the file under 1 MB.
"""

import io
import os
import runpy
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import virtual_views_ref as vr  # noqa: E402

REF = os.environ.get("DYNIBAR_REFERENCE", "/root/reference")
FRAMES, H0, W0, SRC_H, SRC_W, SEED = 2, 288, 10, 144, 5, 7


def _rot(rng, scale):
  a = rng.normal(size=3) * scale
  K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
  return np.eye(3) + np.sin(np.linalg.norm(a)) / max(np.linalg.norm(a), 1e-12) * K + \
      (1 - np.cos(np.linalg.norm(a))) / max(np.linalg.norm(a), 1e-12) ** 2 * K @ K


def write_scene(root, rng):
  """cvd_dir/%05d.npz as dynamic-video-depth writes them; a far slanted background and a near band (~14 % of pixels,
  sets the 5th depth percentile), so the virtual cameras move the background by a few pixels only."""
  dense = os.path.join(root, "data", "dense", "images")
  cvd = os.path.join(root, "cvd")
  os.makedirs(dense)
  os.makedirs(cvd)
  from PIL import Image
  Image.fromarray(np.zeros((H0, W0, 3), np.uint8)).save(os.path.join(dense, "00000.png"))
  K = np.array([[120.0, 0.0, 2.5], [0.0, 120.0, 72.0], [0.0, 0.0, 1.0]], np.float32)
  ys, xs = np.mgrid[0:SRC_H, 0:SRC_W].astype(np.float32)
  for i in range(FRAMES):
    depth = 15.0 + 10.0 * ys / SRC_H + rng.uniform(0, 0.5, (SRC_H, SRC_W))
    depth[50 + 5 * i:70 + 5 * i, :] = 1.0 + rng.uniform(0, 0.1, (20, SRC_W))
    img = 0.5 + 0.4 * np.sin(0.3 * ys + 1.1 * xs + i)[None] * np.array([1.0, 0.7, -0.5])[:, None, None]
    img = img + rng.uniform(0, 0.1, (3, SRC_H, SRC_W))
    c2w = np.eye(4)
    c2w[:3, :3] = _rot(rng, 0.05)
    c2w[:3, 3] = rng.normal(size=3) * 0.1
    np.savez(os.path.join(cvd, "%05d.npz" % i), depth=depth[None, None].astype(np.float32),
             cam_c2w=c2w[None].astype(np.float32), img_1=img[None].astype(np.float32),
             K=K.T[None, None, None].copy())
  return os.path.join(root, "data"), cvd


def install_stubs(rec):
  import cv2
  import scipy.ndimage as ndi

  def splatting_function(kind, frame, flow, metric, eps=vr.EPS):
    assert kind == "softmax"
    rec["splat"].append((frame.clone(), flow.clone(), metric.clone()))
    return torch.from_numpy(vr.splat64(frame, flow, metric)).to(frame.dtype)

  def spatial_gradient(x, mode="sobel", normalized=True):
    assert mode == "sobel" and not normalized
    rec["sobel_in"].append(x.clone())
    p = np.pad(x.double().numpy(), ((0, 0), (0, 0), (1, 1), (1, 1)), mode="edge")
    H, W = x.shape[-2:]
    a = lambda j, i: p[..., j:j + H, i:i + W]
    gx = (a(0, 2) - a(0, 0)) + 2 * (a(1, 2) - a(1, 0)) + (a(2, 2) - a(2, 0))
    gy = (a(2, 0) - a(0, 0)) + 2 * (a(2, 1) - a(0, 1)) + (a(2, 2) - a(0, 2))
    return torch.from_numpy(np.stack([gx, gy], 2)).to(x.dtype)

  def imsave(path, arr):
    buf = io.BytesIO()
    from PIL import Image
    Image.fromarray(arr).save(buf, format="PNG")
    rec["png"][os.path.relpath(path, rec["data"])] = buf.getvalue()

  def imread(path):
    from PIL import Image
    return np.asarray(Image.open(path))

  def resize(src, dsize, interpolation=None):
    out = cv2_resize(src, dsize, interpolation=interpolation)
    rec["resize"].append((int(interpolation), out.copy()))
    return out

  cv2_resize = cv2.resize
  cv2.resize = resize
  mods = {
      "splatting": dict(splatting_function=splatting_function),
      "kornia": dict(filters=types.SimpleNamespace(spatial_gradient=spatial_gradient)),
      "skimage": {}, "skimage.morphology": dict(
          disk=lambda r: np.array([[0, 1, 0], [1, 1, 1], [0, 1, 0]], np.uint8) if r == 1 else None,
          erosion=lambda image, footprint: ndi.grey_erosion(image, footprint=footprint)),
      "imageio": {}, "imageio.v2": dict(imread=imread, imsave=imsave),
  }
  for name, attrs in mods.items():
    m = types.ModuleType(name)
    for k, v in attrs.items():
      setattr(m, k, v)
    sys.modules[name] = m
  sys.modules["skimage"].morphology = sys.modules["skimage.morphology"]
  sys.modules["imageio"].v2 = sys.modules["imageio.v2"]
  torch.Tensor.cuda = lambda self, *a, **k: self


def main():
  rng = np.random.default_rng(SEED)
  np.random.seed(SEED)
  with tempfile.TemporaryDirectory() as root:
    data, cvd = write_scene(root, rng)
    rec = dict(splat=[], sobel_in=[], png={}, resize=[], data=os.path.join(data, "dense"))
    install_stubs(rec)
    argv = sys.argv
    sys.argv = ["render_source_vv.py", "--data_dir", data, "--cvd_dir", cvd]
    try:
      runpy.run_path(os.path.join(REF, "render_source_vv.py"), run_name="__main__")
    finally:
      sys.argv = argv
    poses = np.load(os.path.join(data, "dense", "source_vv_poses.npy"))
    npz = [dict(np.load(os.path.join(cvd, "%05d.npz" % i))) for i in range(FRAMES)]
  V = len(rec["splat"]) // FRAMES
  frames = []
  for i in range(FRAMES):
    calls = rec["splat"][i * V:(i + 1) * V]
    near, area, linear = rec["resize"][3 * i:3 * i + 3]  # depth (nearest), image (area), disparity (linear)
    assert (near[0], area[0], linear[0]) == (0, 3, 1)
    rgba = calls[0][0][0, :4].permute(1, 2, 0).contiguous()
    assert all(torch.equal(c[0][0, :4].permute(1, 2, 0), rgba) and torch.equal(c[0][0, 5], torch.ones_like(c[0][0, 5]))
               for c in calls)
    frames.append(dict(
        img=torch.from_numpy(area[1]), disp=torch.from_numpy(linear[1]), sobel_in=rec["sobel_in"][i][0, 0],
        rgba=rgba, flow=torch.cat([c[1] for c in calls]), weights=torch.cat([c[2] for c in calls]),
        png=[rec["png"][os.path.join("source_virtual_views_%dx%d" % (W0, H0), "%05d" % i, "%02d.png" % k)]
             for k in range(V)]))
  fx = dict(poses=torch.from_numpy(poses), frames=frames, npz=npz, final_hw=(H0, W0))
  path = os.path.join(HERE, "virtual_views.pt")
  torch.save(fx, path)
  print("->", path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
  main()
