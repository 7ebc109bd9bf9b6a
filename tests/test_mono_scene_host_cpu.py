"""Host side of the device-resident monocular scene (dynibar_b200.mono_scene) without a GPU, against the reference's own
loader (tests/golden/mono_scene.pt, make_golden_scene.py): the replayed draws, the cameras, near / far, and the
refusal of malformed scenes."""

import io
import os
import shutil

import numpy as np
import pytest
import torch

import mono_scene_ref as msr
from dynibar_b200 import mono_scene as ms

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mono_scene.pt")


@pytest.fixture(scope="module")
def golden():
  return msr.load_golden(GOLDEN)


@pytest.fixture(scope="module")
def scene_dirs(golden, tmp_path_factory):
  root = tmp_path_factory.mktemp("mono_scene")
  return {name: msr.write_scene(str(root / name / "dense"), dict(np.load(io.BytesIO(sc["raw"]))))
          for name, sc in golden["scenes"].items()}


def test_replayed_draws_give_the_reference_ids(golden, scene_dirs):
  b = golden["base"]
  for c in golden["cases"]:
    cams = ms.load_cameras(scene_dirs[c["scene"]], golden["scenes"][c["scene"]]["height"])
    ids = ms.draw_views(np.random.RandomState(c["seed"]), len(cams["rgb_files"]), c["epoch"], b["init_decay_epoch"],
                        b["num_source_views"], b["max_range"], b["num_vv"], cams["c2w"])
    assert ids["idx"] == int(c["id"]) and ids["anchor"] == int(c["anchor_id"])
    assert ids["nearest"] == c["nearest_pose_ids"][0].tolist()
    assert ids["anchor_nearest"] == c["anchor_nearest_pose_ids"][0].tolist()
    loads = c["loads"]
    nv, na = b["num_vv"], len(ids["anchor_nearest"])
    ns = len(loads) - 1 - (6 + nv) - (na + nv)
    files = [p for p, _ in loads]
    assert files[1 + 6 + nv:1 + 6 + nv + ns] == ["images_%dx%d/%05d.png" % (
        cams["hw"][1], cams["hw"][0], j) for j in ids["static"]]
    vv = lambda p: int(os.path.basename(p)[:-4])
    assert [vv(p) for p in files[1 + 6:1 + 6 + nv]] == ids["vv"]
    assert [vv(p) for p in files[-nv:]] == ids["anchor_vv"]
    masks = [m for _, m in loads[1 + 6 + nv:1 + 6 + nv + ns]]
    assert masks == (["dynamic_masks/%d.png" % j for j in ids["static"]] if c["mask_src_view"] else [None] * ns)
  rare = [c for c in golden["cases"] if c["seed"] == golden["rare_seed"]]
  assert rare and int(rare[0]["id"]) in rare[0]["anchor_nearest_pose_ids"][0].tolist()


def _ulps(a, b):
  a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
  return np.max(np.abs(a - b) / (np.finfo(np.float32).eps * np.maximum(np.abs(a), np.abs(b)) + 1e-300))


def test_cameras_and_near_far_match_the_reference(golden, scene_dirs):
  for name, sc in golden["scenes"].items():
    cams = ms.load_cameras(scene_dirs[name], sc["height"])
    np.testing.assert_array_equal(cams["K"], sc["K"].numpy())
    # numpy 2's float32 scale moves the camera centres, the mean camera and through it the recentred rotations by
    # about one float32 ulp: within one ulp of the largest entry of each block
    eps = np.finfo(np.float32).eps
    for got, want in ((cams["c2w"], sc["c2w"].numpy()), (cams["vv_c2w"], sc["vv_c2w"].numpy())):
      for blk in (np.s_[..., :3, :3], np.s_[..., :3, 3]):
        tol = eps * np.abs(want[blk]).max()
        assert np.abs(got[blk] - want[blk]).max() <= tol, (name, np.abs(got[blk] - want[blk]).max() / tol)
    assert _ulps(cams["depth_range"], np.float32([sc["depth_range"][0] * 0.9, sc["depth_range"][1] * 1.5])) <= 1
    assert sc["scale_dtype"] == "float32"  # what numpy 2 gives; the library follows numpy 1 (next test)
    assert _ulps(np.float32(cams["scale"]), np.float32(sc["scale"])) <= 1


def test_scale_follows_numpy1(golden, scene_dirs):
  """numpy 1.x: scale = 1. / (bds.min() * bd_factor) is a float64 scalar; float32 arrays meet it as float32(scale);
  near * 0.9 and far * 1.5 are float64 until torch.tensor(...).float()."""
  for name, sc in golden["scenes"].items():
    cams = ms.load_cameras(scene_dirs[name], sc["height"])
    arr = np.load(os.path.join(scene_dirs[name], "poses_bounds_cvd.npy"))
    bds = arr[:, -2:].astype(np.float32)
    scale = 1.0 / (np.float64(bds.min()) * 0.75)
    assert cams["scale"] == scale
    b = bds * np.float32(scale)
    near, top = np.float64(b.min()), np.float64(b.max())
    far = min(20, top + 15.0) if top < 10 else min(50, max(20, top))
    np.testing.assert_array_equal(cams["depth_range"], np.array([near * 0.9, far * 1.5]).astype(np.float32))
    d = np.load(os.path.join(scene_dirs[name], "disp", "00003.npy"))
    assert (d / np.float32(scale)).dtype == np.float32


def test_pixel_selection_uses_the_library_stream(golden):
  from dynibar_b200 import sample_ray
  for c in golden["cases"][:4]:
    H, W = (int(v) for v in c["camera"][0, :2])
    sample_ray.rng = np.random.RandomState(c["pixel_seed"])
    got = ms.select_pixels(H, W, golden["n_rand"], c["sample_mode"])
    assert np.array_equal(got, c["rays"]["selected_inds"].numpy())


def test_kernel_ray_arithmetic_against_reference_bmm(golden):
  """ray_d as csrc/scene.cu evaluates it ((M0 u + M1 v) + M2 in fp32, rounded at each step) against the reference's
  bmm on the fixture: the number tests/test_mono_scene_gpu.py's RAY_BAR is 2x of."""
  worst = 0.0
  for c in golden["cases"]:
    cam = c["camera"][0]
    c2w, K = cam[18:34].reshape(4, 4), cam[2:18].reshape(4, 4)
    M = (c2w[:3, :3] @ torch.inverse(K[:3, :3])).numpy()
    sel = c["rays"]["selected_inds"].numpy()
    W = int(cam[1])
    u, v = (sel % W).astype(np.float32), (sel // W).astype(np.float32)
    d = np.stack([(M[a, 0] * u + M[a, 1] * v) + M[a, 2] for a in range(3)], -1).astype(np.float32)
    worst = max(worst, float(np.abs(d - c["rays"]["ray_d"].numpy()).max()))
  print("ray_d worst abs err vs the reference's bmm: %.3e" % worst)
  assert worst <= 1.2e-7  # measured 1.192e-7


def _copy(src, tmp_path):
  dst = str(tmp_path / "dense")
  shutil.copytree(src, dst)
  return dst


def _args(height):
  from types import SimpleNamespace
  return SimpleNamespace(training_height=height, num_source_views=3, max_range=9, num_vv=3, mask_src_view=True,
                         erosion_radius=3, init_decay_epoch=2)


@pytest.mark.parametrize("break_it,match", [
    (lambda d: os.remove(os.path.join(d, "disp", "00004.npy")), "missing file"),
    (lambda d: os.remove(os.path.join(d, "flow_i2", "00005_bwd.npz")), "missing file"),
    (lambda d: os.remove(os.path.join(d, "source_virtual_views_40x24", "00002", "07.png")), "missing file"),
    (lambda d: os.remove(os.path.join(d, "static_masks", "3.png")), "missing file"),
    (lambda d: np.save(os.path.join(d, "disp", "00004.npy"), np.ones((24, 41), np.float32)), "disparity"),
    (lambda d: np.savez(os.path.join(d, "flow_i1", "00006_fwd.npz"), flow=np.zeros((24, 40, 3), np.float32),
                        mask=np.ones((24, 40), bool)), "flow"),
    (lambda d: msr.write_png(os.path.join(d, "images_40x24", "00003.png"), np.zeros((24, 39, 3), np.uint8)),
     "frame"),
    (lambda d: _png16(os.path.join(d, "images_40x24", "00002.png")), "16-bit"),
    (lambda d: os.remove(os.path.join(d, "images_40x24", "00015.png")), "images and"),
])
def test_malformed_scene_raises(golden, scene_dirs, tmp_path, break_it, match):
  d = _copy(scene_dirs["B"], tmp_path)
  break_it(d)
  with pytest.raises(ValueError, match=match):
    ms.MonocularScene(d, _args(24), "cuda:0")


def _png16(path):
  from PIL import Image
  Image.fromarray(np.zeros((24, 40), np.uint16) + 300).save(path)
