"""Helpers of the bullet-time scene tests: the on-disk scenes of tests/golden/bt_scene.pt (make_golden_bt_scene.py)
and the per-camera get_all() batches rebuilt from the fixture's items."""

import hashlib
import os

import numpy as np
import torch

SCENE_H, SCENE_W = 36, 48  # images_48x36
ORIG_H, ORIG_W = 72, 96    # images/: only its size is read (training_height 36 -> factor 2)
N_FRAMES = 16


def write_png(path, a):
  """Lossless PNG of uint8 [H, W] or [H, W, 3] RGB (cv2 writes BGR)."""
  import cv2
  os.makedirs(os.path.dirname(path), exist_ok=True)
  if a.ndim == 3:
    a = a[:, :, ::-1]
  assert cv2.imwrite(path, np.ascontiguousarray(a)), path


def write_scene(root, s):
  """Write scene dict s (the fixture's 'scenes' entry) as the reference's `dense` folder under root; returns root."""
  n = s["frames"].shape[0]
  H, W = s["frames"].shape[1:3]
  os.makedirs(root, exist_ok=True)
  np.save(os.path.join(root, "poses_bounds_cvd.npy"), s["poses_bounds"])
  np.save(os.path.join(root, "source_vv_poses.npy"), s["vv_poses"])
  write_png(os.path.join(root, "images", "00000.png"), np.zeros(tuple(s["orig_hw"]) + (3,), np.uint8))
  for i in range(n):
    write_png(os.path.join(root, "images_%dx%d" % (W, H), "%05d.png" % i), s["frames"][i])
  for ridx, views in s["vviews"].items():
    for j, v in enumerate(views):
      write_png(os.path.join(root, "source_virtual_views_%dx%d" % (W, H), "%05d" % ridx, "%02d.png" % j), v)
  for i, m in enumerate(s["masks"]):
    write_png(os.path.join(root, "dynamic_masks", "%d.png" % i), m)
  return root


def item_batch(case, k, src_rgbs, static_src_rgbs, device):
  """RaySamplerSingleImage(item, device).get_all() of camera k of a fixture case, with the given source images (the
  fixture's own, or the device pools' views); the item's unused ground truth is left out."""
  from dynibar_b200 import sample_ray as sr
  data = dict(camera=case["camera"][k][None], depth_range=case["depth_range"][None],
              src_rgbs=src_rgbs[None], src_cameras=case["src_cameras"][k][None],
              static_src_rgbs=static_src_rgbs[None], static_src_cameras=case["static_src_cameras"][k][None])
  return sr.RaySamplerSingleImage(data, device).get_all()


def ids_of(case, k):
  """(dynamic slot identities, static slot identities) of camera k, as stack_pooled_ray_batches names them."""
  t, vv, st = case["selections"][k]
  return list(t) + [("vv", j) for j in vv], list(st)


def digest(t):
  """SHA-256 of a float32 array's bytes and shape (the fixture pins images this way)."""
  a = np.ascontiguousarray(np.asarray(t.cpu() if torch.is_tensor(t) else t, dtype=np.float32))
  return hashlib.sha256(repr(a.shape).encode() + a.tobytes()).hexdigest()


def unpack_cameras(case):
  """Fill case['src_cameras'] [50,Vd,34] and case['static_src_cameras'] [50,Vs,34] from the fixture's distinct
  camera rows and per-slot indices."""
  rows = case["camera_rows"]
  case["src_cameras"] = rows[case["src_camera_index"].long()]
  case["static_src_cameras"] = rows[case["static_camera_index"].long()]
  return case


def load_golden(path):
  """tests/golden/bt_scene.pt with every case's source cameras unpacked."""
  g = torch.load(path, weights_only=False)
  for case in g["cases"]:
    unpack_cameras(case)
  return g
