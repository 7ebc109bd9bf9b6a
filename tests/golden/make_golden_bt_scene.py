"""tests/golden/bt_scene.pt: what the reference's render_monocular_bt.py loader gives on small on-disk scenes, run
where the reference is:

    python tests/golden/make_golden_bt_scene.py

Two seeded 16-frame scenes at 48x36 are written to a temporary `dense` folder, and the script's DynamicVideoDataset
runs unmodified over them, constructor (load_mono_data, batch_parse_*) and __getitem__ for all 50 cameras of the
wander path.  imageio is stubbed with a cv2 reader (cv2 itself is real, and resizes the masks); the model, renderer
and config modules the script imports are empty stubs.  Two adjustments, both outside the reference's code:
  - numpy 1.x, the reference's environment, computes the depth range in float64 (`np.max(bds) + 15.0` and
    `x * 0.9` on float32 scalars); numpy 2 keeps float32.  The constructor's render_depth_range is recomputed from
    the same bounds as numpy 1.x evaluates it, so __getitem__ returns numpy 1.x's float64 pair.  The bounds' minimum
    is 1.0, so the scene scale is the same under both.
  - __getitem__ indexes render_depth_range, h, w (num_frames equal entries each) and train_rgb_files (read as a
    ground truth nothing uses) by the camera index idx = 0..49, so the script needs at least 50 frames.  The lists
    are padded to 50 entries (the same values; frame 0's path); every source view indexes the real 16 frames.
The focal lengths (48 or 96) make the wander path's 48 / f exact in float32 under either numpy.

Recorded per case and camera: camera, src_cameras, static_src_cameras, depth_range, nearest_pose_ids and the
selection (temporal, virtual-view and static ids, from the files read), and the SHA-256 of every camera's src_rgbs /
static_src_rgbs (float32 bytes and shape), which pins them bit for bit without storing them.  The source cameras are
stored as their distinct rows and per-slot indices, and the arrays with pickle protocol 4, which keeps the file
small.  The scenes' raw arrays are stored too, so the tests rewrite the same files.
"""

import os
import re
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import bt_scene_ref as bsr  # noqa: E402

REF = os.environ.get("DYNIBAR_REFERENCE", "/root/reference")
N_VV = 8
# (scene, mask_src_view, render_idx, num_source_views, max_range, num_vv).  max_range 6 with 3
# views takes every second frame; within 7.5 frames of render_idx 3 or 12 fewer than 7 remain, so the [::5] fallback
# fills in.
CASES = (("A", True, 3, 3, 6, 3), ("A", False, 8, 3, 6, 3), ("B", True, 12, 3, 6, 3), ("B", True, 8, 3, 6, 2))


def _stub(name, **attrs):
  m = types.ModuleType(name)
  m.__dict__.update(attrs)
  sys.modules[name] = m
  return m


def _install_stubs(reads):
  import cv2

  def imread(path, **kw):
    reads.append(path)
    a = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    assert a is not None, path
    if a.ndim == 3:
      a = a[:, :, ::-1].copy()
    return a

  img = _stub("imageio", imread=imread)
  img.v2 = _stub("imageio.v2", imread=imread)
  _stub("config", config_parser=None)
  _stub("ibrnet.sample_ray", RaySamplerSingleImage=None)
  _stub("ibrnet.render_image", render_single_image_mono=None)
  _stub("ibrnet.model", DynibarMono=None)
  _stub("ibrnet.projection", Projector=None)
  # the loaders package's __init__ imports every dataset (and scikit-image): load its modules without it
  _stub("ibrnet.data_loaders").__path__ = [os.path.join(REF, "ibrnet", "data_loaders")]


def _scene(seed, top, mask_shape, ridx):
  """Raw arrays of one scene: LLFF poses drifting along x with small rotations, bounds with minimum 1.0 and maximum
  `top`, 8 virtual views per frame, frames, the virtual views of the frames in ridx, and masks of mask_shape with 0,
  255 and values between."""
  rng = np.random.RandomState(seed)
  n, H, W = bsr.N_FRAMES, bsr.SCENE_H, bsr.SCENE_W

  def llff(c, a, f):
    ca, sa = np.cos(a), np.sin(a)
    R = np.array([[ca, 0.0, sa], [0.0, 1.0, 0.0], [-sa, 0.0, ca]])
    return np.concatenate([R, c[:, None], np.array([[bsr.ORIG_H], [bsr.ORIG_W], [f]])], 1)

  poses = [llff(np.array([0.05 * i + rng.normal(0, 0.01), rng.normal(0, 0.01), rng.normal(0, 0.01)]),
                rng.normal(0, 0.02), 48.0 if i % 2 == 0 else 96.0) for i in range(n)]
  bds = np.stack([rng.uniform(1.0, 2.0, n), rng.uniform(3.0, top, n)], 1)
  bds[rng.randint(n), 0], bds[rng.randint(n), 1] = 1.0, top
  pb = np.concatenate([np.stack(poses).reshape(n, 15), bds], 1)
  vv = np.stack([[llff(p[:, 3] + rng.normal(0, 0.06, 3), rng.normal(0, 0.05), 48.0)[:, :4] for _ in range(N_VV)]
                 for p in poses])  # [n, 8, 3, 4]
  frames = rng.randint(0, 256, (n, H, W, 3)).astype(np.uint8)
  vviews = {r: rng.randint(0, 256, (N_VV, H, W, 3)).astype(np.uint8) for r in ridx}
  masks = rng.choice(np.array([0, 255, 255, 255, 128, 7], np.uint8), (n,) + mask_shape)
  return dict(poses_bounds=pb, vv_poses=np.ascontiguousarray(np.transpose(vv, (1, 2, 3, 0))), frames=frames,
              vviews=vviews, masks=masks, orig_hw=(bsr.ORIG_H, bsr.ORIG_W))


def _pack_cameras(rec, src, static):
  """The source cameras of all 50 cameras as their distinct rows and, per camera and slot, the row's index
  (bt_scene_ref.unpack_cameras inverts it)."""
  rows = torch.unique(torch.cat([src.reshape(-1, 34), static.reshape(-1, 34)]), dim=0)
  index = lambda c: torch.stack([torch.nonzero((rows == r).all(1))[0, 0] for r in c.reshape(-1, 34)]).reshape(
      c.shape[:2]).to(torch.int16)
  rec.update(camera_rows=rows, src_camera_index=index(src), static_camera_index=index(static))
  bsr.unpack_cameras(rec)
  assert torch.equal(rec.pop("src_cameras"), src) and torch.equal(rec.pop("static_src_cameras"), static)


def main():
  sys.path.insert(0, REF)
  reads = []
  _install_stubs(reads)
  from ibrnet.data_loaders import llff_data_utils as llff
  import render_monocular_bt as bt
  ridx = lambda name: sorted({c[2] for c in CASES if c[0] == name})
  scenes = {"A": _scene(3, 6.0, (18, 24), ridx("A")), "B": _scene(4, 30.0, (30, 40, 3), ridx("B"))}
  cases = []
  with tempfile.TemporaryDirectory() as tmp:
    for name, s in scenes.items():
      bsr.write_scene(os.path.join(tmp, name, "dense"), s)
    for name, mask, ridx, nsv, max_range, num_vv in CASES:
      args = types.SimpleNamespace(folder_path=tmp, num_source_views=nsv, mask_src_view=mask, render_idx=ridx,
                                   max_range=max_range, num_vv=num_vv, training_height=bsr.SCENE_H)
      bt.args = args  # __getitem__ reads the script's global args
      ds = bt.DynamicVideoDataset(args, scenes=[name])
      # numpy 1.x's depth range (the module docstring)
      _, _, _, bds, _, _, files, _ = llff.load_mono_data(os.path.join(tmp, name, "dense"), height=bsr.SCENE_H,
                                                         render_idx=ridx, load_imgs=False)
      near, top = np.float64(np.min(bds)), np.float64(np.max(bds))
      far = min(50, top + 15.0) if top < 10 else min(50, max(20, top))
      ds.render_depth_range = [[near, np.float64(far)]] * len(ds.render_poses)
      ds.train_rgb_files = list(files) + [files[0]] * (50 - len(files))
      ds.h, ds.w = ds.h[:1] * len(ds.render_poses), ds.w[:1] * len(ds.render_poses)
      rec = dict(scene=name, mask_src_view=mask, render_idx=ridx, num_source_views=nsv, max_range=max_range,
                 num_vv=num_vv, camera=[], src_cameras=[], static_src_cameras=[], selections=[], images={})
      for idx in range(len(ds)):
        del reads[:]
        item = ds[idx]
        paths = reads[1:]  # reads[0]: the unused ground truth
        frame_of = lambda p: int(re.search(r"(\d+)\.png$", p).group(1))
        temporal = [frame_of(p) for p in paths[:7]]
        vv = [frame_of(p) for p in paths[7:7 + num_vv]]
        assert all("source_virtual_views" in p for p in paths[7:7 + num_vv])
        rest = paths[7 + num_vv:]
        static = [frame_of(p) for p in rest if "images_" in p]
        assert len(rest) == len(static) * (2 if mask else 1), rest
        assert list(item["nearest_pose_ids"]) == temporal
        rec["selections"].append((temporal, vv, static))
        rec["camera"].append(item["camera"])
        rec["src_cameras"].append(item["src_cameras"])
        rec["static_src_cameras"].append(item["static_src_cameras"])
        assert item["depth_range"].dtype == torch.float64
        if idx == 0:
          rec["depth_range"] = item["depth_range"]
        assert torch.equal(item["depth_range"], rec["depth_range"])
        rec["images"][idx] = (bsr.digest(item["src_rgbs"]), bsr.digest(item["static_src_rgbs"]))
      rec["camera"] = torch.stack(rec["camera"])
      _pack_cameras(rec, torch.stack(rec.pop("src_cameras")), torch.stack(rec.pop("static_src_cameras")))
      fallback = any(abs(f - ridx) > max_range + nsv * 0.5 for sel in rec["selections"] for f in sel[2])
      rec["fallback"] = fallback
      cases.append(rec)
  assert cases[0]["fallback"] and cases[2]["fallback"]
  torch.save(dict(scenes=scenes, cases=cases), os.path.join(HERE, "bt_scene.pt"), pickle_protocol=4)


if __name__ == "__main__":
  main()
