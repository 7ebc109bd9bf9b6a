"""The restatement of render_source_vv.py's device work (tests/virtual_views_ref.py) on the CPU: it reproduces what
the unmodified reference script computed on the fixture's scene (tests/golden/virtual_views.pt: flow, weights, the
rgba layout, the poses bit for bit, the PNGs), its erosion is scipy's, and every planted error would fail the GPU
comparison (tests/test_virtual_views_gpu.py) by a wide margin, so that test's bars are not vacuous."""

import numpy as np
import pytest
import scipy.ndimage as ndi
import torch

import virtual_views_ref as vr
from dynibar_b200 import virtual_views as vv

MARGIN = 3.0  # a planted error must exceed the GPU test's bar by this factor


@pytest.fixture(scope="module")
def fx(golden):
  return golden("virtual_views")


def test_poses_bit_for_bit(fx):
  npz = fx["npz"]
  H, W = fx["final_hw"]
  Ks = [vv.scaled_intrinsics(z["K"], z["img_1"].shape[2:], (H, W)) for z in npz]
  npy, c2w = vv.virtual_view_poses(np.stack([z["cam_c2w"][0] for z in npz]), [z["depth"][0, 0] for z in npz],
                                   Ks[-1], (H, W))
  assert npy.dtype == np.float32 and npy.shape == (8, 3, 4, len(npz))
  assert np.array_equal(npy, fx["poses"].numpy())
  assert c2w.shape == (len(npz), 8, 3, 4)


@pytest.mark.parametrize("i", [0, 1])
def test_flow_weights_and_layout(fx, i):
  """The fp32 projection in the CUDA kernel's operation order gives the reference's flow to a few fp32 ulps of the
  target coordinate (the reference's matmuls sum in their own order), the weights to a few ulps of their range,
  and the splatted frame is [img * 255, alpha of (1 / disp) / 10] bit for bit up to the Sobel."""
  img, disp, K, ref2w, tgt = vr.fixture_frame_inputs(fx, i)
  f = fx["frames"][i]
  R, t = vr.ref2tgt(ref2w, tgt)
  V = R.shape[0]
  k = torch.from_numpy(np.array(K)).float()[None].expand(V, 3, 3)
  depth = (1.0 / disp.float())[None].expand(V, -1, -1)
  flow, inv_z = vr.project32(depth, R, t, k, k)
  H, W = disp.shape
  scale = max(H, W) * 2.0 ** -23 * 8
  assert vr.max_err(flow, f["flow"]) <= scale, vr.max_err(flow, f["flow"])
  assert vr.max_err(vr.weights32(inv_z), f["weights"]) <= 20 * 2.0 ** -20
  assert torch.equal(f["sobel_in"], (1.0 / disp) / 10.0)
  assert torch.equal(f["rgba"][..., :3], img * 255.0)
  alpha = vr.sobel_alpha64(f["sobel_in"][None], 0.5)[0]
  assert vr.max_err(f["rgba"][..., 3], alpha) <= 1e-6
  assert np.array_equal(vr.rgba_of_frame(img, disp)[..., :3], f["rgba"][..., :3].numpy())


@pytest.mark.parametrize("i", [0, 1])
def test_pngs_from_splat_inputs(fx, i):
  """The splat, threshold, erosion and quantisation restated give the reference's PNGs exactly."""
  f = fx["frames"][i]
  got = vr.views_from_splat_inputs(f["rgba"], f["flow"], f["weights"])
  want = vr.decode_pngs(f["png"])
  assert got.dtype == np.uint8 and np.array_equal(got, want)
  assert 0.3 < (want > 0).any(-1).mean() < 0.95  # the views are neither empty nor unmasked


def test_erosion_is_scipy_grey_erosion_with_the_cross():
  g = np.random.default_rng(0)
  cross = np.array([[0, 1, 0], [1, 1, 1], [0, 1, 0]], bool)
  for shape in [(7, 9), (1, 5), (4, 1), (30, 31)]:
    m = g.random(shape) > 0.2
    assert np.array_equal(vr.erode_cross(m), ndi.grey_erosion(m, footprint=cross))
    assert np.array_equal(vr.erode_cross(m, "square_erosion"), ndi.grey_erosion(m, footprint=np.ones((3, 3), bool)))


def test_splat_conserves_weight_and_places_corners():
  """One source at (1.25, 2.5) of a 4 x 5 image: weights 0.375 / 0.125 / 0.375 / 0.125 at (1,2) (2,2) (1,3) (2,3);
  a source at x in (-1, 0) reaches column 0 through its NE / SE corners only."""
  frame = torch.zeros(1, 1, 4, 5)
  flow = torch.full((1, 2, 4, 5), -100.0)
  metric = torch.zeros(1, 1, 4, 5)
  frame[0, 0, 0, 0] = 2.0
  flow[0, :, 0, 0] = torch.tensor([1.25, 2.5])
  frame[0, 0, 3, 4] = 4.0
  flow[0, :, 3, 4] = torch.tensor([-4.75, -3.0])  # -> (-0.75, 0.0)
  out = vr.splat64(frame, flow, metric)[0, 0]
  e = 1.0
  np.testing.assert_allclose(out[2, 1], 2.0 * 0.375 * e / (0.375 * e + vr.EPS))
  np.testing.assert_allclose(out[3, 2], 2.0 * 0.125 / (0.125 + vr.EPS))
  np.testing.assert_allclose(out[0, 0], 4.0 * 0.25 / (0.25 + vr.EPS))
  assert (out[:, 1:][out[:, 1:] != 0].size) == 4


def _plant_error(plant):
  """How far the planted restatement moves the compared quantity, in units of the GPU bar."""
  if plant in ("trunc_for_floor", "no_eps"):
    c = vr.splat_case("edges")
    return vr.ratio(vr.max_err(vr.splat64(*c, plant=plant), vr.splat64(*c)), vr.BARS["splat"])
  if plant == "swap_ne_sw":
    c = vr.splat_case("odd")
    return vr.ratio(vr.max_err(vr.splat64(*c, plant=plant), vr.splat64(*c)), vr.BARS["splat"])
  if plant == "batch_minmax":
    imgs, d, r, t, k = vr.forward_case("batch")
    got = vr.render_forward_splat64(imgs, d, r, t, k, k, plant=plant)[0]
    return vr.ratio(vr.max_err(got, vr.render_forward_splat64(imgs, d, r, t, k, k)[0]), vr.BARS["forward_image"])
  if plant == "zero_pad":
    x = vr.sobel_case()
    return vr.ratio(vr.max_err(vr.sobel_alpha64(x, 10.0, plant), vr.sobel_alpha64(x, 10.0)), vr.BARS["sobel"])
  if plant == "square_erosion":
    c = vr.frame_case()
    return vr.ratio(vr.png_mismatch(vr.views64(*c, plant=plant), vr.views64(*c)), vr.PNG_FRAC_BAR)
  raise KeyError(plant)


@pytest.mark.parametrize("plant", vr.PLANTS)
def test_planted_error_exceeds_gpu_bar(plant):
  m = _plant_error(plant)
  assert m >= MARGIN, (plant, m)


def test_argument_checks_without_gpu():
  """Bad arguments fail before any CUDA call; CPU tensors and modes without a kernel are refused."""
  from dynibar_b200 import _lib
  rc = _lib.lib.dyn_splat_softmax(None, None, None, 1, 3, 8, 8, None, None, 0, None)
  assert rc == -1 and b"argument check failed" in _lib.lib.dyn_last_error()
  assert _lib.lib.dyn_forward_splat(None, None, None, 0, 3, 8, 8, None, None, 0, None) == -1
  assert _lib.lib.dyn_sobel_alpha(None, 1, 8, 8, 1.0, None, None) == -1
  assert _lib.lib.dyn_virtual_views(None, None, None, 8, 8, 8, None, None, 0, None) == -1
  x = torch.zeros(1, 3, 8, 8)
  with pytest.raises(RuntimeError, match="no CPU fallback"):
    vv.splatting_function("softmax", x, torch.zeros(1, 2, 8, 8), torch.zeros(1, 1, 8, 8))
  with pytest.raises(RuntimeError, match="no CPU fallback"):
    vv.render_forward_splat(torch.zeros(1, 8, 8, 3), torch.ones(1, 8, 8), torch.eye(3)[None], torch.zeros(1, 3),
                            torch.eye(3)[None], torch.eye(3)[None])
  with pytest.raises(RuntimeError, match="no CPU fallback"):
    vv.sobel_fg_alpha(torch.zeros(1, 1, 8, 8))
  with pytest.raises(NotImplementedError):
    vv.splatting_function("summation", x, x[:, :2], x[:, :1])
  with pytest.raises(NotImplementedError):
    vv.sobel_fg_alpha(x, mode="scharr")
