"""The host restatement of eval_nvidia.py's scoring (tests/metrics_ref.py) against the reference's own
calculate_psnr / calculate_ssim recorded in tests/golden/eval_metrics.pt, its two SSIM maps against each other, and the
errors a port could make against the GPU bars.  Also the argument checks of dynibar_b200.metrics and of the C ABI that
run before any device work."""

import numpy as np
import pytest
import torch

import metrics_ref as mr
from dynibar_b200 import _lib
from dynibar_b200 import metrics


def test_restatement_equals_the_reference_glue(golden):
  fx = golden("eval_metrics")
  assert len(fx["cases"]) >= 9
  for c in fx["cases"]:
    a, b, m = c["img1"].numpy(), c["img2"].numpy(), c["mask"].numpy()
    assert mr.calculate_psnr(a, b, m) == c["psnr"], c["name"]
    assert float(mr.calculate_ssim32(a, b, m)) == c["ssim"], c["name"]
    # the float64 sums the GPU computes differ from the reference's float32 np.sum within the fixture bar
    assert abs(mr.ssim_score64(mr.ssim_map32(a, b), m) - c["ssim"]) <= mr.BARS["fixture"], c["name"]
  by_name = {c["name"]: c for c in fx["cases"]}
  assert by_name["identical"]["psnr"] == 0.0 and by_name["empty_mask"]["psnr"] == 0.0
  assert by_name["empty_mask"]["ssim"] == 0.0


@pytest.mark.parametrize("kind", ["random", "smooth", "constant", "identical", "binary"])
def test_float32_and_float64_maps_agree(kind):
  for H, W in ((7, 7), (8, 9), (7, 40), (33, 47)):
    x, y = mr.pair(kind, H, W)
    err = np.abs(mr.ssim_map32(x, y) - mr.ssim_map64(x, y)).max()
    assert err <= mr.MAP32_VS_64, (kind, H, W, err)


def test_valid_mask_sum_is_float32_left_to_right():
  """eval_nvidia.py:384's np.sum over the channels is ((r + g) + b) in float32, which the kernel computes."""
  rng = np.random.default_rng(3)
  x = (rng.random((4096, 3), dtype=np.float32) * np.float32(1e-3)).astype(np.float32)
  want = (x[:, 0] + x[:, 1]) + x[:, 2]
  assert np.array_equal(np.sum(x, axis=-1), want)


def _map_err(plant):
  x, y = mr.pair("random", 40, 48, seed=5)
  kw = dict(data_range_1=dict(data_range=1.0), population_cov=dict(cov=1.0), border_nearest=dict(mode="nearest"),
            border_mirror=dict(mode="mirror"))[plant]
  return np.abs(mr.ssim_map32(x, y, **kw) - mr.ssim_map32(x, y)).max()


@pytest.mark.parametrize("plant", mr.PLANTS)
def test_planted_errors_exceed_the_bars(plant):
  score_bar = max(mr.BARS["score"], mr.BARS["fixture"])
  err = 0.0
  for mask_kind in ("blobs", "empty"):
    pred, gt, dyn = mr.eval_case(1, 40, 56, seed=9, mask_kind=mask_kind)
    base = mr.eval_scores(pred[0], gt[0], dyn[0])
    got = mr.eval_scores(pred[0], gt[0], dyn[0], plant=plant)
    with np.errstate(invalid="ignore"):
      d = np.abs(got - base)
    err = max(err, np.inf if not np.isfinite(d).all() else d.max())
  assert err >= 3 * score_bar, (plant, err)
  if plant in ("data_range_1", "population_cov", "border_nearest", "border_mirror"):
    e = _map_err(plant)  # the map itself, against the bar of the GPU map vs ssim_map32
    assert e >= 3 * mr.BARS["smap32"], (plant, e)


def test_drop_in_argument_errors_before_any_device_work():
  x = np.zeros((8, 9, 3), np.float32)
  with pytest.raises(TypeError):
    metrics.calculate_ssim(np.zeros((8, 9, 3), np.uint8), x, np.ones_like(x))
  with pytest.raises(TypeError):
    metrics.calculate_psnr(x, torch.zeros(8, 9, 3, dtype=torch.int32), np.ones_like(x))
  with pytest.raises(ValueError, match="win_size exceeds image extent"):
    metrics.calculate_ssim(np.zeros((6, 9, 3), np.float32), np.zeros((6, 9, 3), np.float32), np.ones((6, 9, 3)))
  with pytest.raises(ValueError, match="win_size exceeds image extent"):
    metrics.score_views(np.zeros((2, 9, 6, 3), np.float32), np.zeros((2, 9, 6, 3), np.float32))
  with pytest.raises(ValueError, match="same dimensions"):
    metrics.calculate_ssim(x, np.zeros((8, 10, 3), np.float32), np.ones_like(x))
  with pytest.raises(ValueError):
    metrics.calculate_psnr(x, x, np.ones((8, 9, 2), np.float32))
  with pytest.raises(ValueError):
    metrics.score_views(x[None], x[None], np.ones((1, 8, 9, 2), np.float32))


def test_abi_rejects_bad_arguments_without_a_gpu():
  lib = _lib.lib
  assert lib.dyn_image_scores_workspace_bytes(0, 8, 8) == 0
  assert lib.dyn_image_scores_workspace_bytes(1, 6, 8) == 0 and lib.dyn_image_scores_workspace_bytes(1, 8, 6) == 0
  # one row of 9 fp64 sums per 32 x 16 tile
  assert lib.dyn_image_scores_workspace_bytes(11, 288, 512) == 11 * 16 * 18 * 9 * 8
  p = 256  # never dereferenced: every call below fails its argument check first
  for args in ((p, p, None, 0, 8, 8, 0), (p, p, None, 1, 6, 8, 0), (p, p, None, 1, 8, 6, 0),
               (None, p, None, 1, 8, 8, 0), (p, None, None, 1, 8, 8, 1), (p, p, None, 1, 8, 8, 2)):
    rc = lib.dyn_image_scores(*args, p, None, p, 1 << 20, None)
    assert rc == -1 and b"argument check failed" in lib.dyn_last_error(), args
  rc = lib.dyn_image_scores(p, p, None, 1, 8, 8, 0, None, None, p, 1 << 20, None)
  assert rc == -1
  rc = lib.dyn_image_scores(p, p, None, 1, 8, 8, 0, p, None, p, 8, None)
  assert rc == -3 and b"workspace" in lib.dyn_last_error()
