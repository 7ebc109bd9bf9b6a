"""Host planning of the stabilised video (render_idx < 0, no GPU) against the reference's render_monocular_bt.py
loader (tests/golden/bt_stab.pt, make_golden_bt_stab.py): the smoothed path bit for bit, and per camera i its
camera, selections, virtual-view rows, pool tables, time and offsets.  Planted errors (the reference's fixed
render_idx, frame 0's virtual views, a frame's intrinsics on a virtual view, training's far rule) change recorded
values."""

import os

import cv2
import numpy as np
import pytest

import bt_scene_ref as bsr
import bt_stab_ref as bst
from dynibar_b200 import bt_scene, bullet_time as bt
from dynibar_b200.mono_scene import load_cameras

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bt_stab.pt")
RENDERED = list(range(bst.FIRST, bst.LAST + 1))


@pytest.fixture(scope="module")
def golden():
  return bst.load_golden(GOLDEN)


@pytest.fixture(scope="module")
def roots(golden, tmp_path_factory):
  base = tmp_path_factory.mktemp("stab")
  return {name: bsr.write_scene(str(base / name / "dense"), s) for name, s in golden["scenes"].items()}


def _plan(case, root, render_idx=-1):
  cams = load_cameras(root, bsr.SCENE_H)
  return cams, bt_scene.plan_sweep(cams, render_idx, case["num_source_views"], case["max_range"], case["num_vv"])


def test_stabilization_path_equals_reference_render_poses(golden, roots):
  for case in golden["cases"]:
    cams = load_cameras(roots[case["scene"]], bsr.SCENE_H)
    path = bt.stabilization_path(cams["poses"])
    want = case["render_poses"].numpy()
    assert path.dtype == np.float32 and path.shape == want.shape == (bsr.N_FRAMES, 3, 5)
    np.testing.assert_array_equal(path, want)
    # smoothing moved the poses, and every pose carries frame 0's hwf
    assert not np.array_equal(path[:, :, :4], cams["poses"][:, :, :4])
    np.testing.assert_array_equal(path[:, :, 4], np.repeat(cams["poses"][:1, :, 4], bsr.N_FRAMES, 0))


def test_cameras_selections_pools_and_time_match_reference(golden, roots):
  for case in golden["cases"]:
    cams, plan = _plan(case, roots[case["scene"]])
    n = bsr.N_FRAMES
    assert case["ids"] == RENDERED
    assert plan["cameras"].shape == (n, 34) and plan["frames"] == list(range(n))
    assert [i for i, s in enumerate(plan["selections"]) if s is not None] == RENDERED
    # one camera per group: each renders at its own time
    assert plan["groups"] == [(i, i + 1) for i in RENDERED]
    for k, i in enumerate(case["ids"]):
      np.testing.assert_array_equal(plan["cameras"][i], case["camera"][k].numpy())
      assert tuple(list(x) for x in plan["selections"][i]) == tuple(case["selections"][k])
      # ref_time = i / n (float64) and the offsets -3 .. 3 follow from the camera's frame
      assert case["ref_time"][k] == float(plan["frames"][i] / float(n))
      assert [f - plan["frames"][i] for f in case["selections"][k][0]] == list(bt_scene.OFFSETS)
      grp = bt_scene.plan_group(cams, plan, -1, i, i + 1, case["mask_src_view"])
      t, vv, st = case["selections"][k]
      assert grp["dy_pool"] == list(t) + [("vv", i, j) for j in vv] and grp["st_pool"] == list(st)
      assert grp["src_views"].tolist() == [list(range(7 + len(vv)))]
      np.testing.assert_array_equal(grp["src_cameras"][grp["src_views"][0]], case["src_cameras"][k].numpy())
      np.testing.assert_array_equal(grp["static_src_cameras"][grp["static_src_views"][0]],
                                    case["static_src_cameras"][k].numpy())
      # pool rows: temporal frames, then frame i's virtual views, then the static frames (masked when asked)
      want = [(f, -1, 0, s) for s, f in enumerate(t)] + [(i, j, 0, 7 + s) for s, j in enumerate(vv)]
      want += [(f, -1, int(case["mask_src_view"]), 2 << 8 | s) for s, f in enumerate(st)]
      assert grp["table"].dtype == np.int32 and grp["table"].tolist() == [list(r) for r in want]
    fb = case["fallback"]
    assert fb[0] and fb[-1] and not all(fb)


def test_depth_range_matches_reference(golden, roots):
  for case in golden["cases"]:
    cams = load_cameras(roots[case["scene"]], bsr.SCENE_H)
    np.testing.assert_array_equal(bt_scene.depth_range(*cams["bounds"]), case["depth_range"].numpy())


def test_source_images_restated(golden):
  """The dynamic views are the temporal frames and frame i's virtual views; the static views are the frames, times
  the nearest-resized raw mask / 255 when mask_src_view is set.  Frame 0's virtual views are other images."""
  for case in golden["cases"]:
    scene = golden["scenes"][case["scene"]]
    for i, (src, want) in case["images"].items():
      t, vv, st = case["selections"][i - bst.FIRST]
      views = lambda f: np.stack([scene["frames"][x] for x in t] + [scene["vviews"][f][j] for j in vv])
      assert bsr.digest(views(i).astype(np.float32) / 255.0) == src
      assert bsr.digest(views(0).astype(np.float32) / 255.0) != src
      static = []
      for f in st:
        rgb = scene["frames"][f].astype(np.float32) / 255.0
        if case["mask_src_view"]:
          m = cv2.resize(scene["masks"][f].astype(np.float32) / 255.0, (bsr.SCENE_W, bsr.SCENE_H),
                         interpolation=cv2.INTER_NEAREST)
          rgb = rgb * (m[..., None] if m.ndim == 2 else m)
        static.append(rgb)
      assert bsr.digest(np.stack(static)) == want


def test_planted_errors_differ(golden, roots):
  for case in golden["cases"]:
    cams, plan = _plan(case, roots[case["scene"]])
    H, W = cams["hw"]
    args = (case["num_source_views"], case["max_range"], case["num_vv"])
    fixed = frame0 = frame_K = 0
    for k, i in enumerate(case["ids"]):
      c2w = plan["render_c2w"][i]
      # the reference's own behaviour: the temporal views and time of the fixed render_idx -1 (its static views
      # cannot be chosen there at all: the script's assert fails)
      fixed += ([-1 + o for o in bt_scene.OFFSETS] != case["selections"][k][0]
                and case["ref_time"][k] != -1 / float(bsr.N_FRAMES))
      # frame 0's virtual views in place of frame i's
      vv0 = bt.select_source_views(c2w, cams["c2w"], cams["vv_c2w"][[0] * bsr.N_FRAMES], i, *args)[1]
      row0 = bt_scene.camera_row(H, W, plan["render_K"][i], cams["vv_c2w"][0, vv0[0]])
      frame0 += not np.array_equal(row0, case["src_cameras"][k][7].numpy())
      # frame i's intrinsics on a virtual view's row in place of the render camera's
      row = bt_scene.camera_row(H, W, cams["K"][i], cams["vv_c2w"][i, case["selections"][k][1][0]])
      frame_K += not np.array_equal(row, case["src_cameras"][k][7].numpy())
    assert fixed == len(case["ids"]) and frame0 == len(case["ids"]) and frame_K > 0
  # training's far rule min(20, max + 15) gives another range where the largest bound is below 10
  case = next(c for c in golden["cases"] if c["scene"] == "D")
  near, top = load_cameras(roots["D"], bsr.SCENE_H)["bounds"]
  assert top < 10
  assert not np.array_equal(np.array([near * 0.9, min(20, top + 15.0) * 1.5]), case["depth_range"].numpy())


def test_groups_hold_one_frame(golden, roots):
  """A bullet-time plan has one frame for all cameras, so naming the frames leaves its groups as they were; cameras
  of two frames never share a group, and cameras without a selection are in none."""
  case = golden["cases"][0]
  cams, plan = _plan(case, roots[case["scene"]], render_idx=8)
  sel = plan["selections"]
  assert plan["frames"] == [8] * 50 and all(s is not None for s in sel)
  assert plan["groups"] == bt.group_cameras(sel)
  assert any(lo < 25 < hi for lo, hi in plan["groups"])
  split = bt.group_cameras(sel, frames=[8] * 25 + [9] * 25)
  assert [c for lo, hi in split for c in range(lo, hi)] == list(range(50))
  assert not any(lo < 25 < hi for lo, hi in split)
  holes = bt.group_cameras([None] * 3 + sel[3:20] + [None] + sel[21:])
  assert [c for lo, hi in holes for c in range(lo, hi)] == [c for c in range(50) if c >= 3 and c != 20]
