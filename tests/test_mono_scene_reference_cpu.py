"""tests/mono_scene_ref.py (cv2 + scipy) against the reference's own loader (tests/golden/mono_scene.pt), and the planted
errors the GPU comparisons must catch.  The GPU bars for ids, masks and images are bit-exactness, so a plant fails them
when it changes any recorded value (and fails them at least threefold exactly when it changes one)."""

import io
import os

import numpy as np
import pytest
import torch

import mono_scene_ref as msr


@pytest.fixture(scope="module")
def golden():
  return msr.load_golden(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mono_scene.pt"))


def _cams(sc):
  return dict(c2w=sc["c2w"].numpy(), K=sc["K"].numpy(), vv_c2w=sc["vv_c2w"].numpy(), scale=sc["scale"],
              depth_range=np.float32(sc["depth_range"].numpy() * [0.9, 1.5]))


def _items(golden, plant=None):
  raw = {k: dict(np.load(io.BytesIO(sc["raw"]))) for k, sc in golden["scenes"].items()}
  for c in golden["cases"]:
    cfg = dict(golden["base"], mask_src_view=c["mask_src_view"], erosion_radius=c["erosion_radius"])
    item = msr.Item(raw[c["scene"]], _cams(golden["scenes"][c["scene"]]), cfg, plant)
    yield c, item(np.random.RandomState(c["seed"]), c["epoch"])


def _mismatches(c, it):
  """Which recorded values the item does not reproduce exactly."""
  bad = []
  ids = it["ids"]
  if ids["idx"] != int(c["id"]) or ids["anchor"] != int(c["anchor_id"]):
    bad.append("ids")
  if ids["anchor_nearest"] != c["anchor_nearest_pose_ids"][0].tolist():
    bad.append("anchor_nearest_pose_ids")
  for k in ("motion_mask", "static_mask"):
    if not np.array_equal(it[k], msr.unpack_mask(c[k])):
      bad.append(k)
  for k in ("rgb", "disp", "flows", "masks", "src_rgbs", "static_src_rgbs", "anchor_src_rgbs"):
    if msr.hash_f32(torch.from_numpy(np.ascontiguousarray(it[k]))[None]) != c["hash"][k]:
      bad.append(k)
  for k in ("camera", "anchor_camera"):
    if not np.array_equal(it[k], c[k][0].numpy()):
      bad.append(k)
  for k in ("src_cameras", "static_src_cameras", "anchor_src_cameras"):
    if it[k].shape != tuple(c[k].shape[1:]) or not np.array_equal(it[k], c[k][0].numpy()):
      bad.append(k)
  return bad


def test_restatement_equals_the_reference_loader(golden):
  n = 0
  for c, it in _items(golden):
    assert _mismatches(c, it) == [], (c["scene"], c["seed"])
    sel = c["rays"]["selected_inds"].numpy()
    ray_o, ray_d = msr.rays(it["camera"], sel)
    assert torch.equal(ray_o, c["rays"]["ray_o"]) and torch.equal(ray_d, c["rays"]["ray_d"])
    n += 1
  assert n == len(golden["cases"]) >= 10


def test_pixel_selection_restatement(golden):
  for c in golden["cases"]:
    H, W = (int(v) for v in c["camera"][0, :2])
    got = msr.select_pixels(np.random.RandomState(c["pixel_seed"]), H, W, golden["n_rand"], c["sample_mode"])
    assert np.array_equal(got, c["rays"]["selected_inds"].numpy())


MASK_PLANTS = ("square_footprint", "nearest_border", "src_over_dst", "static_unthresholded", "erode_at_frame_height",
               "source_mask_thresholded")


def _mask_pixels_changed(plant):
  """Pixels the planted restatement changes on the mask-kernel tests' inputs (which the GPU compares bit for bit)."""
  n = 0
  for H, W, mh, mw in msr.MASK_SIZES:
    for channels in (0, 3):
      for _, dyn, st in msr.mask_inputs(H, W, mh, mw, channels, n=1):
        for r in (3,):
          n += int((msr.motion_mask(dyn[0], H, W, r, plant) != msr.motion_mask(dyn[0], H, W, r)).sum())
        n += int((msr.static_mask(st[0], H, W, plant) != msr.static_mask(st[0], H, W)).sum())
        n += int((msr.source_mask(dyn[0], H, W, plant) != msr.source_mask(dyn[0], H, W)).sum())
  return n


@pytest.mark.parametrize("plant", [p for p in msr.PLANTS if p not in ("ge_threshold", "nearest_border")])
def test_planted_error_fails_the_bars(golden, plant):
  """Every plant changes recorded values of the fixture, or (mask plants) at least 3 pixels of the mask tests."""
  hits = sum(bool(_mismatches(c, it)) for c, it in _items(golden, plant))
  if plant in MASK_PLANTS:
    hits += _mask_pixels_changed(plant) >= 3
  assert hits >= 1, plant


def test_ge_threshold_is_indistinguishable_on_8_bit_masks(golden):
  """`>=` for `>` at 1e-3 cannot change a mask read from an 8-bit PNG: 1 - m / 255 is 0 or at least 1 / 255 (3.9e-3),
  never float32(1e-3).  This plant is the one no comparison can catch, and none is needed."""
  v = np.float32(1.0) - np.arange(256, dtype=np.float32) / np.float32(255.0)
  assert np.array_equal(v > np.float32(1e-3), v >= np.float32(1e-3))
  assert all(not _mismatches(c, it) for c, it in _items(golden, "ge_threshold"))


def test_nearest_border_is_indistinguishable_in_disk_erosion():
  """scipy's `nearest` for `reflect` cannot change an erosion by a disk: a point (y - k, x + j) beyond the top edge
  reflects to row k - y - 1 and repeats row 0, and both lie inside the disk around (y, x), since |k - 2y - 1| < k and
  y < k; likewise at every edge and corner.  The minimum is the same, so no comparison can catch this plant; it is
  checked here on every image up to 9 x 9 and on the mask tests' inputs."""
  rng = np.random.default_rng(1)
  for h in range(1, 10):
    for w in range(1, 10):
      for r in range(6):
        b = rng.random((h, w)) > 0.2
        assert np.array_equal(msr.erosion(b, r, "nearest_border"), msr.erosion(b, r))
  assert _mask_pixels_changed("nearest_border") == 0


def test_nearest_resize_index_is_cv2s():
  """cv2's resizeNN index min(floor(x * (1 / (dst / src))), src - 1), which csrc/scene.cu evaluates in double, equals
  cv2.resize over every pair of sizes up to 80 and the sizes of the fixtures and tests; src / dst does not."""
  differs = 0
  for src in list(range(1, 81)) + [288, 512, 540, 960, 30, 50, 480]:
    for dst in list(range(1, 81)) + [288, 512, 480, 24, 40]:
      a = np.arange(src, dtype=np.float32)[None].repeat(2, 0)
      got = msr.resize_nn(a, dst, 2)[0].astype(np.int64)
      assert np.array_equal(got, msr.resize_nn_index(src, dst)), (src, dst)
      differs += not np.array_equal(got, msr.resize_nn(a, dst, 2, "src_over_dst")[0].astype(np.int64))
  assert differs > 0


def test_reflect_rule_is_scipys():
  """scene.cu's reflect index (period 2n, d c b a | a b c d), which also covers a disk wider than the image, gives
  scipy's grey_erosion for every image up to 8 x 8 and every radius up to 5."""
  def refl(i, n):
    i %= 2 * n
    return i if i < n else 2 * n - 1 - i
  rng = np.random.default_rng(0)
  for h in range(1, 9):
    for w in range(1, 9):
      for r in range(6):
        b = rng.random((h, w)) > 0.3
        fp = msr.disk(r)
        got = np.array([[all(b[refl(y + dy, h), refl(x + dx, w)] for dy in range(-r, r + 1) for dx in range(-r, r + 1)
                             if fp[dy + r, dx + r]) for x in range(w)] for y in range(h)])
        assert np.array_equal(got, msr.erosion(b, r)), (h, w, r)
