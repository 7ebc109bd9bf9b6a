"""Host planning of the bullet-time scene (no GPU) against the reference's render_monocular_bt.py loader
(tests/golden/bt_scene.pt, make_golden_bt_scene.py): the target cameras, each camera's source views and their camera
rows through the pools, and the depth range with its dtype.  Planted errors (the training loader's far rule, a frame's
intrinsics on a virtual view, an eroded or thresholded mask) change recorded values."""

import os

import cv2
import numpy as np
import pytest
import scipy.ndimage
import torch

import bt_scene_ref as bsr
from dynibar_b200 import bt_scene
from dynibar_b200.mono_scene import load_cameras

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bt_scene.pt")


@pytest.fixture(scope="module")
def golden():
  return bsr.load_golden(GOLDEN)


@pytest.fixture(scope="module")
def roots(golden, tmp_path_factory):
  base = tmp_path_factory.mktemp("bt")
  return {name: bsr.write_scene(str(base / name / "dense"), s) for name, s in golden["scenes"].items()}


def _plan(case, root):
  cams = load_cameras(root, bsr.SCENE_H)
  return cams, bt_scene.plan_sweep(cams, case["render_idx"], case["num_source_views"], case["max_range"],
                                   case["num_vv"])


def test_cameras_selections_and_pools_match_reference(golden, roots):
  fallbacks = 0
  for case in golden["cases"]:
    cams, plan = _plan(case, roots[case["scene"]])
    np.testing.assert_array_equal(plan["cameras"], case["camera"].numpy())
    assert [tuple(list(x) for x in s) for s in plan["selections"]] == [tuple(s) for s in case["selections"]]
    fallbacks += case["fallback"]
    covered = []
    for lo, hi in plan["groups"]:
      grp = bt_scene.plan_group(cams, plan, case["render_idx"], lo, hi, case["mask_src_view"])
      assert grp["table"].dtype == np.int32 and grp["src_views"].dtype == np.int32
      assert grp["dy_pool"][:7] == case["selections"][lo][0]  # the temporal frames lead the dynamic pool
      assert len(grp["dy_pool"]) <= 32 and len(grp["st_pool"]) <= 32
      for k in range(lo, hi):
        np.testing.assert_array_equal(grp["src_cameras"][grp["src_views"][k - lo]], case["src_cameras"][k].numpy())
        np.testing.assert_array_equal(grp["static_src_cameras"][grp["static_src_views"][k - lo]],
                                      case["static_src_cameras"][k].numpy())
        dy, st = bsr.ids_of(case, k)
        assert [grp["dy_pool"][i] for i in grp["src_views"][k - lo]] == dy
        assert [grp["st_pool"][i] for i in grp["static_src_views"][k - lo]] == st
      # the pool rows: frames by id, virtual views from the scene's one set, static rows masked when asked
      for slot, (f, vv, masked, code) in enumerate(grp["table"]):
        ident = (grp["dy_pool"] + grp["st_pool"])[slot]
        if slot < len(grp["dy_pool"]):
          assert code == slot and masked == 0
          assert (f, vv) == ((0, ident[1]) if isinstance(ident, tuple) else (ident, -1))
        else:
          assert code == (2 << 8 | slot - len(grp["dy_pool"])) and (f, vv) == (ident, -1)
          assert masked == int(case["mask_src_view"])
      covered += list(range(lo, hi))
    assert covered == list(range(50))
  assert fallbacks >= 2


def test_depth_range_matches_reference_with_its_dtype(golden, roots):
  for case in golden["cases"]:
    cams = load_cameras(roots[case["scene"]], bsr.SCENE_H)
    got = bt_scene.depth_range(*cams["bounds"])
    assert got.dtype == np.float64 and case["depth_range"].dtype == torch.float64
    np.testing.assert_array_equal(got, case["depth_range"].numpy())


def test_planted_far_rule_and_intrinsics_differ(golden, roots):
  # scene A's largest bound is below 10: training's min(20, max + 15) is another far bound
  case = next(c for c in golden["cases"] if c["scene"] == "A")
  cams = load_cameras(roots["A"], bsr.SCENE_H)
  near, top = cams["bounds"]
  assert top < 10
  training = np.array([near * 0.9, min(20, top + 15.0) * 1.5])
  assert not np.array_equal(training, case["depth_range"].numpy())
  # numpy 2's float32 arithmetic is another range too
  n32 = np.array([np.float32(near) * np.float32(0.9), (np.float32(top) + np.float32(15)) * np.float32(1.5)])
  assert not np.array_equal(n32.astype(np.float64), case["depth_range"].numpy())
  # a virtual view's row with the intrinsics of frame idx (the script's rgb_file) in place of the render camera's
  H, W = cams["hw"]
  differs = 0
  for k in range(len(cams["rgb_files"])):
    row = bt_scene.camera_row(H, W, cams["K"][k], cams["vv_c2w"][case["render_idx"], case["selections"][k][1][0]])
    differs += not np.array_equal(row, case["src_cameras"][k][7].numpy())
  assert differs > 0


def _masked_static(scene, case, k, mask_fn):
  H, W = bsr.SCENE_H, bsr.SCENE_W
  out = []
  for f in case["selections"][k][2]:
    rgb = scene["frames"][f].astype(np.float32) / 255.0
    m = mask_fn(scene["masks"][f].astype(np.float32) / 255.0)
    m = cv2.resize(m, (W, H), interpolation=cv2.INTER_NEAREST)
    out.append(rgb * (m[..., None] if m.ndim == 2 else m))
  return np.stack(out)


def test_masked_static_views_restated_and_planted(golden):
  """The static views are rgb * nearest-resized raw mask / 255 (1 or 3 channels); eroding or thresholding the mask,
  as training does, gives other images."""
  seen = set()
  for case in golden["cases"]:
    scene = golden["scenes"][case["scene"]]
    assert sorted(case["images"]) == list(range(50))
    for k, (src, want) in case["images"].items():
      # the dynamic views are the temporal frames and the render frame's virtual views, unmasked
      views = [scene["frames"][f] for f in case["selections"][k][0]]
      views += [scene["vviews"][case["render_idx"]][j] for j in case["selections"][k][1]]
      assert bsr.digest(np.stack(views).astype(np.float32) / 255.0) == src
      if not case["mask_src_view"]:
        assert bsr.digest(np.stack([scene["frames"][f] for f in case["selections"][k][2]])
                          .astype(np.float32) / 255.0) == want
        continue
      seen.add(scene["masks"].ndim)
      assert bsr.digest(_masked_static(scene, case, k, lambda m: m)) == want
      if k % 10 == 0:
        thr = _masked_static(scene, case, k, lambda m: (1.0 - m > 1e-3).astype(np.float32))
        ero = _masked_static(scene, case, k, lambda m: scipy.ndimage.grey_erosion(m, size=(3, 3) + m.shape[2:]))
        assert bsr.digest(thr) != want and bsr.digest(ero) != want
  assert seen == {3, 4}  # 1- and 3-channel masks


def test_crop_and_refusals():
  assert bt_scene.crop_of(288, 512) == (8, 15)
  assert bt_scene.crop_of(36, 48) == (1, 1)
  from dynibar_b200 import _lib
  fake = 0x1000  # never dereferenced: the checks return first
  for K, H, W, ch, cw in ((1, 4, 4, 2, 0), (1, 4, 4, 0, 2), (0, 4, 4, 0, 0), (1, 4, 4, -1, 0)):
    assert _lib.lib.dyn_bt_frames(fake, K, H, W, ch, cw, fake, None) == -1
  assert _lib.lib.dyn_scene_pools(None, fake, 3, fake, 2, fake, 1, None) == -1
