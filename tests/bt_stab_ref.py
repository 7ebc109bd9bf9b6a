"""Helpers of the stabilised-video tests (tests/golden/bt_stab.pt, make_golden_bt_stab.py): the fixture's on-disk
scenes, rebuilt from their seeds, and the fixture's items by camera."""

import hashlib

import numpy as np
import torch

import bt_scene_ref as bsr
from golden import make_golden_bt_scene as mgb

FIRST, LAST = 3, bsr.N_FRAMES - 4  # the rendered cameras of a 16-frame video


def scene_digest(s):
  """SHA-256 of a scene's raw arrays (the fixture records it beside each scene's seed)."""
  h = hashlib.sha256()
  for a in (s["poses_bounds"], s["vv_poses"], s["frames"], np.stack([s["vviews"][f] for f in sorted(s["vviews"])]),
            s["masks"]):
    a = np.ascontiguousarray(a)
    h.update(repr((a.dtype.str, a.shape)).encode() + a.tobytes())
  return h.hexdigest()


def make_scene(seed, top, mask_shape):
  """make_golden_bt_scene's seeded 16-frame scene with the virtual views of every frame."""
  return mgb._scene(seed, top, tuple(mask_shape), range(bsr.N_FRAMES))


def load_golden(path):
  """tests/golden/bt_stab.pt with every scene rebuilt (and checked against its digest) and every case's source
  cameras unpacked.  A case's per-camera lists hold cameras FIRST..LAST in order; case['ids'] names them."""
  g = torch.load(path, weights_only=False)
  scenes = {}
  for name, r in g["scenes"].items():
    s = make_scene(r["seed"], r["top"], r["mask_shape"])
    assert scene_digest(s) == r["digest"], "scene %s does not rebuild from its seed" % name
    scenes[name] = s
  g["scenes"] = scenes
  for case in g["cases"]:
    bsr.unpack_cameras(case)
  return g
