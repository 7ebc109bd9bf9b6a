"""The restatement of the Nvidia evaluation front end (tests/nvi_scene_ref.py), and NvidiaScene's host side, against
the reference's own outputs (tests/golden/nvi_scene.pt, made by tests/golden/make_golden_nvi_scene.py) and cv2.

The restatement's INTER_AREA equals cv2.resize byte for byte at the benchmark's sizes, at mixed, odd and unit factors;
each planted error changes recorded values."""

import os

import cv2
import numpy as np
import pytest
import torch

import mono_scene_ref as msr
import nvi_scene_ref as nsr
from dynibar_b200 import nvidia_scene as ns

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nvi_scene.pt")
BENCH_SIZES = [(1080, 1920), (720, 1280), (576, 1024), (864, 1536), (1152, 2048)]
# (sh, sw, dh, dw): integer in one axis only, odd sizes down to 1 pixel, a factor of 1
OTHER_SIZES = [(576, 700, 288, 350), (600, 1024, 288, 512), (13, 26, 13, 13), (26, 13, 13, 13), (77, 133, 30, 41),
               (108, 192, 29, 51), (5, 7, 1, 1), (9, 4, 3, 1), (1, 9, 1, 2), (13, 13, 13, 13), (31, 17, 7, 17),
               (24, 24, 6, 6), (8, 8, 2, 2), (37, 23, 12, 7), (1000, 1000, 300, 300), (1080, 1920, 300, 500)]


@pytest.fixture(scope="module")
def golden():
  return nsr.load_golden(GOLDEN)


@pytest.fixture(scope="module")
def scenes(golden, tmp_path_factory):
  root = tmp_path_factory.mktemp("nvi")
  return {name: nsr.write_files(str(root / name / "dense"), s["files"]) for name, s in golden["scenes"].items()}


def area_input(sh, sw, seed, smooth=True):
  rng = np.random.default_rng(seed)
  a = rng.integers(0, 256, size=(sh, sw, 3), dtype=np.uint8)
  return cv2.GaussianBlur(a, (0, 0), 2) if smooth and min(sh, sw) > 8 else a


@pytest.mark.parametrize("sh,sw", BENCH_SIZES)
def test_area_resize_equals_cv2_at_benchmark_sizes(sh, sw):
  a = area_input(sh, sw, sh + sw)
  assert np.array_equal(nsr.area_resize(a, 288, 512), cv2.resize(a, (512, 288), interpolation=cv2.INTER_AREA))


@pytest.mark.parametrize("sh,sw,dh,dw", OTHER_SIZES)
def test_area_resize_equals_cv2_at_other_factors(sh, sw, dh, dw):
  for smooth in (True, False):
    a = area_input(sh, sw, sh * sw, smooth)
    assert np.array_equal(nsr.area_resize(a, dh, dw), cv2.resize(a, (dw, dh), interpolation=cv2.INTER_AREA))


@pytest.mark.parametrize("plant,sh,sw,dh,dw", [("int_half_even", 576, 1024, 288, 512),
                                               ("float_path_at_int", 576, 1024, 288, 512),
                                               ("float64_accumulate", 1000, 1000, 300, 300),
                                               ("float64_accumulate", 1080, 1920, 300, 500)])
def test_area_plants_change_bytes(plant, sh, sw, dh, dw):
  """float64 accumulation cannot change a byte at 3.75x, 2.5x or 1.5x (the exact sums there stay at least 1/450 away
  from a rounding tie); at 3.33x it does."""
  a = area_input(sh, sw, 7, smooth=False)
  assert not np.array_equal(nsr.area_resize(a, dh, dw, plant), nsr.area_resize(a, dh, dw))


def _items(s):
  return {(int(it["img_i"]), int(it["cam"])): it for it in s["items"]}


def test_host_cameras_equal_fixture(golden, scenes):
  """load_cameras against DynamicVideoDataset: cameras within one float32 ulp (the fixture was recorded under numpy 2,
  whose float32 scale differs from numpy 1.x's), depth range float64 as numpy 1.x gives it."""
  for name, s in golden["scenes"].items():
    c = ns.load_cameras(scenes[name])
    assert c["hw"] == tuple(int(x) for x in s["hw"])
    assert c["depth_range"].dtype == np.float64
    np.testing.assert_allclose(np.float32(c["depth_range"]), s["items"][0]["depth_range"][0].numpy(), rtol=1.2e-7,
                               atol=0)
    for k in ("K", "c2w"):
      np.testing.assert_allclose(np.float32(c[k]), s[k].numpy().astype(np.float32), rtol=0, atol=2.4e-7)


def test_view_selection_equals_fixture(golden):
  for s in golden["scenes"].values():
    n = int(s["n"])
    for (img_i, cam), it in _items(s).items():
      frames = [int(os.path.basename(r)[:-4]) for r in it["reads"] if r.startswith("images_")]
      assert frames == ns.dynamic_ids(img_i) + ns.static_ids(img_i, n)
      assert frames[7:] == nsr.static_ids(img_i, n)
      coarse = [int(os.path.basename(r)[:-4]) for r in it["reads"] if r.startswith("coarse_masks")]
      assert coarse == ([j for j in frames[7:] if 3 <= j < n - 3] if s["mask_static"] else [])
      assert it["nearest_pose_ids"][0].tolist() == ns.dynamic_ids(img_i)
      assert it["rgb_path"] == os.path.join("mv_images", "%05d" % img_i, "cam%02d.jpg" % (cam + 1))
      assert it["ref_time"].dtype == torch.float64 and it["ref_time"].item() == img_i / float(n)
    assert ns.target_cameras(3) == nsr.target_cameras(3) == [i for i in range(12) if i != 3]


def test_restated_items_equal_fixture(golden, scenes):
  for name, s in golden["scenes"].items():
    n = int(s["n"])
    for (img_i, cam), it in _items(s).items():
      got = nsr.item(scenes[name], img_i, cam, n, s["K"].numpy(), s["c2w"].numpy(), s["depth_range"].numpy(),
                     s["mask_static"])
      for k in ("src_rgbs", "static_src_rgbs", "static_src_masks"):
        assert msr.hash_f32(got[k]) == it["hash"][k], (name, img_i, cam, k)
      for k in ("camera", "src_cameras", "static_src_cameras", "id", "nearest_pose_ids"):
        assert torch.equal(got[k], it[k]), (name, img_i, cam, k)


def test_restated_ground_truth_and_masks_equal_fixture(golden, scenes):
  for name, s in golden["scenes"].items():
    n, (H, W) = int(s["n"]), s["hw"]
    gts, masks = [], []
    for img_i in range(3, n - 3):
      gt, dm = nsr.ground_truth(scenes[name], img_i, nsr.target_cameras(img_i), int(H), int(W))
      gts += [msr.hash_f32(g) for g in gt]
      masks += [dm_ for dm_ in dm]
    assert gts == list(s["gt_hash"])
    for got, want in zip(masks, s["dynamic_masks"]):
      assert np.array_equal(got, want)


def test_plants_change_recorded_values(golden, scenes):
  s = golden["scenes"]["A"]  # coloured masks, generic area path, mask_static on
  n, (H, W) = int(s["n"]), (int(s["hw"][0]), int(s["hw"][1]))
  root = scenes["A"]
  _, dm = nsr.ground_truth(root, 3, nsr.target_cameras(3), H, W, plant="mask_rgb_order")
  assert any(not np.array_equal(a, b) for a, b in zip(dm, s["dynamic_masks"][:11]))
  assert len(nsr.target_cameras(3, plant="keep_held_out")) != len([it for it in s["items"] if it["img_i"] == 3]) - 1
  it = _items(s)[(5, 0)]
  for plant, key in (("static_wrong_residue", "static_src_cameras"), ("target_pose_of_img_i", "camera")):
    got = nsr.item(root, 5, 0, n, s["K"].numpy(), s["c2w"].numpy(), s["depth_range"].numpy(), True, plant)
    assert not torch.equal(got[key], it[key]), plant
  b = golden["scenes"]["B"]  # integer factors
  gt, _ = nsr.ground_truth(scenes["B"], 3, nsr.target_cameras(3), int(b["hw"][0]), int(b["hw"][1]),
                           plant="float_path_at_int")
  assert [msr.hash_f32(g) for g in gt] != list(b["gt_hash"][:11])
  gt, _ = nsr.ground_truth(scenes["B"], 3, nsr.target_cameras(3), int(b["hw"][0]), int(b["hw"][1]),
                           plant="int_half_even")
  assert [msr.hash_f32(g) for g in gt] != list(b["gt_hash"][:11])


def test_printed_scores_parse(golden):
  for s in golden["scenes"].values():
    per, avg = nsr.printed_scores(s["printed"])
    n = int(s["n"])
    assert sorted(per) == [(i, c) for i in range(3, n - 3) for c in nsr.target_cameras(i)]
    assert len(avg["AVG PSNR"]) == 1 and len(avg["MOVING PSNR"]) == n - 6
    flat = np.stack([per[k] for k in sorted(per)])
    want = np.array([[avg["AVG PSNR"][0], avg["AVG SSIM"][0]], [avg["AVG DYNAMIC PSNR"][0], avg["AVG DYNAMIC SSIM"][0]],
                     [avg["AVG Static PSNR"][0], avg["AVG Static SSIM"][0]]])
    # the fixture was recorded under numpy 2, where SSIM is float32 (printed to 8 digits); under numpy 1.x float64
    np.testing.assert_allclose(ns.mean_scores(flat)[:, 0], want[:, 0], rtol=1e-12)
    np.testing.assert_allclose(ns.mean_scores(flat)[:, 1], want[:, 1], rtol=3e-7)


def test_scene_errors(golden, tmp_path):
  import types
  s = golden["scenes"]["B"]
  root = nsr.write_files(str(tmp_path / "B" / "dense"), s["files"])
  with pytest.raises(RuntimeError):
    ns.NvidiaScene(root, types.SimpleNamespace(mask_static=False), "cpu")
  os.remove(os.path.join(root, "poses_bounds_cvd.npy"))
  with pytest.raises(ValueError):
    ns.load_cameras(root)
