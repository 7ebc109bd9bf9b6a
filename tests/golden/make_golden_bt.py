"""tests/golden/bullet_time.pt: the reference's bullet-time camera path and per-camera source-view selection, run
where the reference is, as make_golden.py:

    python tests/golden/make_golden_bt.py

render_monocular_bt.py's DynamicVideoDataset.__getitem__ runs unmodified on seeded synthetic poses; its constructor
(which reads a scene from disk) is bypassed by setting the attributes it would set.  Modules it imports that cannot
run here are stubbed: imageio.imread records the file it is asked for and returns a black image, cv2 is never called
(mask_src_view is off), and the model / renderer / config modules are empty.  The frames it reads give each camera's
temporal, virtual and static source views.  render_wander_path comes from the reference's llff_data_utils as is.
"""

import os
import re
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("DYNIBAR_REFERENCE", "/root/reference")
N_FRAMES, N_VV, SEED, NUM_VV = 60, 8, 11, 3
# (render_idx, num_source_views, max_range): configs/test_kid-running.txt has 7 and 10.  Near the video's ends with
# max_range 7 fewer than 15 frames lie in range, so the [::5] fallback fills in; max_range 8 with 4 views takes
# every second frame.
CASES = ((3, 7, 7), (30, 7, 10), (56, 7, 10), (56, 7, 7), (20, 4, 8))


def _stub(name, **attrs):
  m = types.ModuleType(name)
  m.__dict__.update(attrs)
  sys.modules[name] = m
  return m


def _install_stubs(reads):
  def imread(path):
    reads.append(path)
    return np.zeros((4, 6, 3), np.uint8)

  img = _stub("imageio", imread=imread)
  img.v2 = _stub("imageio.v2", imread=imread)
  _stub("cv2")
  _stub("config", config_parser=None)
  _stub("ibrnet.sample_ray", RaySamplerSingleImage=None)
  _stub("ibrnet.render_image", render_single_image_mono=None)
  _stub("ibrnet.model", DynibarMono=None)
  _stub("ibrnet.projection", Projector=None)
  # the loaders package's __init__ imports every dataset (and scikit-image): load its modules without it
  _stub("ibrnet.data_loaders").__path__ = [os.path.join(REF, "ibrnet", "data_loaders")]


def _poses(rng):
  """LLFF [N,3,5] poses (rotation | centre | hwf) drifting along x with small rotations, and per frame N_VV virtual
  views scattered around it."""
  def llff(c, a):
    ca, sa = np.cos(a), np.sin(a)
    R = np.array([[ca, 0.0, sa], [0.0, 1.0, 0.0], [-sa, 0.0, ca]])
    return np.concatenate([R, c[:, None], np.array([[288.0], [512.0], [400.0]])], 1)

  train = [llff(np.array([0.05 * i + rng.normal(0, 0.01), rng.normal(0, 0.01), rng.normal(0, 0.01)]),
                rng.normal(0, 0.02)) for i in range(N_FRAMES)]
  vv = [[llff(t[:, 3] + rng.normal(0, 0.06, 3), rng.normal(0, 0.05)) for _ in range(N_VV)] for t in train]
  return np.stack(train).astype(np.float32), np.stack(vv).astype(np.float32)


def main():
  sys.path.insert(0, REF)
  reads = []
  _install_stubs(reads)
  from ibrnet.data_loaders import llff_data_utils as llff
  import render_monocular_bt as bt
  rng = np.random.RandomState(SEED)
  train_llff, vv_llff = _poses(rng)
  _, train_c2w = llff.batch_parse_llff_poses(train_llff)
  src_vv_c2w = llff.batch_parse_vv_poses(vv_llff)
  cases = []
  for render_idx, nsv, max_range in CASES:
    path = np.array(llff.render_wander_path(train_llff[render_idx])).astype(np.float32)
    intr, render_c2w = llff.batch_parse_llff_poses(path)
    ds = bt.DynamicVideoDataset.__new__(bt.DynamicVideoDataset)
    ds.render_poses, ds.render_intrinsics = render_c2w, intr
    ds.render_depth_range = np.tile(np.array([[1.0, 10.0]], np.float32), (len(path), 1))
    ds.train_rgb_files = ["/scene/dense/images/%05d.png" % i for i in range(N_FRAMES)]
    ds.train_poses, ds.train_intrinsics = train_c2w, np.tile(intr[:1], (N_FRAMES, 1, 1))
    ds.src_vv_c2w_mats = src_vv_c2w
    ds.num_source_views, ds.max_range, ds.render_idx, ds.num_vv = nsv, max_range, render_idx, NUM_VV
    ds.num_frames, ds.mask_src_view = N_FRAMES, False
    ds.h, ds.w = [288] * len(path), [512] * len(path)
    bt.args = types.SimpleNamespace(max_range=max_range)  # __getitem__ reads the script's global args
    sel = []
    for idx in range(len(path)):
      del reads[:]
      ds[idx]
      frames = [int(re.search(r"(\d+)\.png$", p).group(1)) for p in reads]
      # reads: the target's own frame, 7 temporal frames, NUM_VV virtual views, 2 NUM_SOURCE_VIEWS + 1 static frames
      assert len(frames) == 1 + 7 + NUM_VV + 2 * nsv + 1, frames
      assert all("source_virtual_views" in p for p in reads[8:8 + NUM_VV])
      sel.append((frames[1:8], frames[8:8 + NUM_VV], frames[8 + NUM_VV:]))
    fallback = any(abs(f - render_idx) > max_range + nsv * 0.5 for s_ in sel for f in s_[2])
    cases.append(dict(render_idx=render_idx, num_source_views=nsv, max_range=max_range, fallback=fallback,
                      llff_c2w=torch.from_numpy(train_llff[render_idx]),
                      wander=torch.from_numpy(path), render_c2w=torch.from_numpy(render_c2w), selections=sel))
  assert cases[0]["fallback"] and cases[3]["fallback"] and not cases[1]["fallback"]
  torch.save(dict(train_c2w=torch.from_numpy(train_c2w), src_vv_c2w=torch.from_numpy(src_vv_c2w), num_vv=NUM_VV,
                  cases=cases),
             os.path.join(HERE, "bullet_time.pt"))


if __name__ == "__main__":
  main()
