"""NvidiaScene (csrc/nvi_scene.cu) against the reference's Nvidia evaluation front end (tests/golden/nvi_scene.pt) and
cv2: time steps bit for bit, the area kernel byte for byte, the reference's printed scores, and a whole evaluation
against the INTEGRATION loop fed by the restated items."""

import os
import types

import cv2
import numpy as np
import pytest
import torch

import metrics_ref as mr
import mono_scene_ref as msr
import nvi_scene_ref as nsr
from dynibar_b200 import _lib, metrics, nvidia_scene as ns, sample_ray as sr, synthetic
from dynibar_b200.projection import Projector
from dynibar_b200.render_image import render_multi_image_nvi

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nvi_scene.pt")
RAY_BAR = 2.4e-7  # ray_d against RaySamplerSingleImage.get_all (DESIGN §3.7)
# scene.evaluate against the INTEGRATION loop fed by the restated items, max abs over PSNR / SSIM: 2x the measured
# worst difference on an H100 (DESIGN §3.8); ray_d's last bit is the only expected source
EVAL_BAR = 8.6e-2


@pytest.fixture(scope="module")
def golden():
  return nsr.load_golden(GOLDEN)


@pytest.fixture(scope="module")
def scenes(golden, tmp_path_factory):
  root = tmp_path_factory.mktemp("nvi")
  out = {}
  for name, s in golden["scenes"].items():
    path = nsr.write_files(str(root / name / "dense"), s["files"])
    out[name] = (path, ns.NvidiaScene(path, types.SimpleNamespace(mask_static=bool(s["mask_static"])), DEV))
  return out


def _ulp_close(got, want):
  g, w = got.detach().cpu().to(torch.float32), want.to(torch.float32)
  assert torch.all((g - w).abs() <= torch.maximum(w.abs(), torch.ones_like(w)) * 1.2e-7), (g - w).abs().max()


def test_time_step_equals_fixture(golden, scenes):
  for name, s in golden["scenes"].items():
    root, scene = scenes[name]
    items = {(int(it["img_i"]), int(it["cam"])): it for it in s["items"]}
    for img_i in sorted({k[0] for k in items}):
      step = scene.time_step(img_i)
      rb = step["ray_batch"]
      cams = ns.target_cameras(img_i)
      assert step["cameras"] == cams
      first = items[(img_i, cams[0])]
      want_keys = dict(first["ray_keys"], camera_index=("torch.int32", None))
      assert sorted(rb) == sorted(want_keys)
      for k, v in rb.items():
        if v is None or want_keys[k] is None:
          assert v is None and want_keys[k] is None, k
      for k in ("src_rgbs", "static_src_rgbs", "static_src_masks"):
        assert msr.hash_f32(rb[k]) == first["hash"][k], (name, img_i, k)
        assert (str(rb[k].dtype), tuple(rb[k].shape)) == want_keys[k]
      for k in ("src_cameras", "static_src_cameras"):
        _ulp_close(rb[k], first[k])
      _ulp_close(rb["camera"], torch.cat([items[(img_i, c)]["camera"] for c in cams]))
      assert rb["depth_range"].dtype == torch.float64 and tuple(rb["depth_range"].shape) == (1, 2)
      _ulp_close(rb["depth_range"], first["depth_range"])
      assert step["frame_idx"] == (int(first["id"]), None)
      assert step["time_offset"][0] == [int(j) - img_i for j in first["nearest_pose_ids"][0]]
      t = step["time_embedding"][0]
      assert t.dtype == torch.float64 and t.is_cuda and torch.equal(t.cpu(), first["ref_time"])
      masked = (rb["static_src_rgbs"][0] * rb["static_src_masks"][0][..., None]).permute(0, 3, 1, 2)
      assert torch.equal(step["static_src_masked"], masked)
      # rays: the restated RaySamplerSingleImage of every camera, and the reference's own for the recorded one
      H, W = scene.H, scene.W
      assert rb["ray_o"].shape == (len(cams) * H * W, 3)
      assert torch.equal(rb["camera_index"].cpu(), torch.arange(len(cams), dtype=torch.int32).repeat_interleave(H * W))
      for k, c in enumerate(cams):
        o, d = msr.rays(rb["camera"][k].cpu(), np.arange(H * W))
        sl = slice(k * H * W, (k + 1) * H * W)
        assert torch.equal(rb["ray_o"][sl].cpu(), o)
        assert (rb["ray_d"][sl].cpu() - d).abs().max().item() <= RAY_BAR
        if "rays" in items[(img_i, c)]:  # the reference's own rays, from the fixture's (numpy 2) camera
          ref = items[(img_i, c)]["rays"]
          at = lambda x: x[sl].cpu()[ref["sel"]]
          _ulp_close(at(rb["ray_o"]), ref["ray_o"])
          assert (at(rb["ray_d"]) - ref["ray_d"]).abs().max().item() <= RAY_BAR
          assert torch.equal(at(rb["uv_grid"]), ref["uv_grid"])
    # ground truth and dynamic masks of every time step, in the script's order
    gts, masks = [], []
    for img_i in scene.steps:
      step = scene.time_step(img_i)
      gts += [msr.hash_f32(g) for g in step["gt_rgb"]]
      masks += list(step["dynamic_mask"].cpu().numpy())
    assert gts == list(s["gt_hash"])
    for got, want in zip(masks, s["dynamic_masks"]):
      assert np.array_equal(got, want)


AREA_CASES = [((sh, sw), (288, 512)) for sh, sw in [(1080, 1920), (720, 1280), (576, 1024), (864, 1536), (1152, 2048)]]
AREA_CASES += [((sh, sw), (dh, dw)) for sh, sw, dh, dw in [(576, 700, 288, 350), (600, 1024, 288, 512), (13, 26, 13, 13),
                                                           (26, 13, 13, 13), (77, 133, 30, 41), (108, 192, 29, 51),
                                                           (5, 7, 1, 1), (9, 4, 3, 1), (1, 9, 1, 2), (13, 13, 13, 13),
                                                           (31, 17, 7, 17), (24, 24, 6, 6), (8, 8, 2, 2),
                                                           (1000, 1000, 300, 300), (1080, 1920, 300, 500)]]


@pytest.mark.parametrize("src_hw,dst_hw", AREA_CASES)
def test_area_kernel_equals_cv2(src_hw, dst_hw):
  (sh, sw), (dh, dw) = src_hw, dst_hw
  rng = np.random.default_rng(sh * 7 + sw)
  imgs = rng.integers(0, 256, size=(3, sh, sw, 3), dtype=np.uint8)
  if min(sh, sw) > 8:
    imgs[1] = cv2.GaussianBlur(imgs[1], (0, 0), 2)
  imgs[2] = imgs[2] // 64 * 64  # few levels: many exact ties
  src = torch.from_numpy(imgs).to(DEV)
  out = torch.empty(3, dh, dw, 3, dtype=torch.uint8, device=DEV)
  _lib.check(_lib.lib.dyn_area_resize(src.data_ptr(), 3, sh, sw, 3, dh, dw, out.data_ptr(), _lib.stream()))
  for i in range(3):
    assert np.array_equal(out[i].cpu().numpy(), cv2.resize(imgs[i], (dw, dh), interpolation=cv2.INTER_AREA)), i


def test_scores_of_recorded_predictions_equal_printed(golden, scenes):
  for name, s in golden["scenes"].items():
    _, scene = scenes[name]
    per, avg = nsr.printed_scores(s["printed"])
    got = []
    for img_i in scene.steps:
      step = scene.time_step(img_i)
      pred = np.stack([nsr.prediction(img_i, c, scene.H, scene.W) for c in step["cameras"]])
      sc = metrics.score_views(torch.from_numpy(pred).to(DEV), step["gt_rgb"], step["dynamic_mask"]).cpu().numpy()
      for k, c in enumerate(step["cameras"]):
        want = per[(img_i, c)]
        assert np.abs(sc[k, :, 0] - want[:, 0]).max() <= mr.BARS["fixture"], (name, img_i, c)
        # SSIM was printed in float32 (numpy 2): 8 significant digits
        assert np.abs(sc[k, :, 1] - want[:, 1]).max() <= mr.BARS["fixture"] + 6e-8, (name, img_i, c)
      got.append(sc)
    mean = ns.mean_scores(np.stack(got))
    assert abs(mean[0, 0] - avg["AVG PSNR"][0]) <= mr.BARS["fixture"]
    assert abs(mean[2, 0] - avg["AVG Static PSNR"][0]) <= mr.BARS["fixture"]


def _model(n):
  from dynibar_b200.feature_network import ResNet
  model, args = synthetic.make_model(N_samples=16, N_importance=16, num_frames=n, seed=3)
  model = synthetic.model_to(model, DEV)
  torch.manual_seed(4)
  model.feature_net = ResNet().to(DEV).requires_grad_(False)
  model.feature_net_fine = ResNet().to(DEV).requires_grad_(False)
  args.chunk_size, args.N_samples, args.N_importance = 8192, 16, 16
  args.inv_uniform, args.white_bkgd = True, False
  return model, args


def _integration_step(root, s, img_i, model, args, mask_static):
  """The INTEGRATION loop on the restated items: RaySamplerSingleImage -> stack_ray_batches -> the four encoder passes
  -> render_multi_image_nvi -> host cv2 ground truth and masks -> score_views."""
  n = int(s["n"])
  cams = nsr.target_cameras(img_i)
  c = ns.load_cameras(root)  # the fixture's cameras within one float32 ulp (test_time_step_equals_fixture)
  data = [nsr.item(root, img_i, k, n, c["K"], c["c2w"], c["depth_range"], mask_static) for k in cams]
  samplers = [sr.RaySamplerSingleImage(d, device=DEV) for d in data]
  rb, _, _ = sr.stack_ray_batches([x.get_all() for x in samplers])
  src = rb["src_rgbs"].squeeze(0).permute(0, 3, 1, 2)
  static_src = rb["static_src_rgbs"].squeeze(0).permute(0, 3, 1, 2)
  ref_fm, _ = model.feature_net(src)
  _, st_fm = model.feature_net(static_src)
  ref_fm_f, _ = model.feature_net_fine(src)
  st_ = static_src * rb["static_src_masks"].squeeze(0)[:, None, ...] if mask_static else static_src
  _, st_fm_f = model.feature_net_fine(st_)
  offs = [int(j - img_i) for j in data[0]["nearest_pose_ids"].squeeze().tolist()]
  rets = render_multi_image_nvi(frame_idx=(img_i, None), time_embedding=(data[0]["ref_time"].to(DEV), None),
                                time_offset=(offs, None), ray_samplers=samplers, ray_batch=rb, model=model,
                                projector=Projector(DEV), chunk_size=args.chunk_size, det=True,
                                N_samples=args.N_samples, args=args, inv_uniform=args.inv_uniform,
                                N_importance=args.N_importance, white_bkgd=args.white_bkgd,
                                coarse_featmaps=(ref_fm, None, st_fm), fine_featmaps=(ref_fm_f, None, st_fm_f),
                                is_train=False)
  pred = torch.stack([r["outputs_fine_ref"]["rgb"] for r in rets])
  H, W = pred.shape[1:3]
  gt, dm = nsr.ground_truth(root, img_i, cams, H, W)
  return metrics.score_views(pred, gt, dm).cpu().numpy()


def test_evaluate_equals_integration_loop(golden, scenes):
  s = golden["scenes"]["B"]
  root, scene = scenes["B"]
  model, args = _model(scene.num_frames)
  args.mask_static = bool(s["mask_static"])
  with torch.no_grad():
    res = scene.evaluate(model, Projector(DEV), args)
    want = np.stack([_integration_step(root, s, i, model, args, args.mask_static) for i in scene.steps])
  assert res["scores"].shape == (len(scene.steps), 11, 3, 2) and res["scores"].dtype == np.float64
  diff = np.abs(res["scores"] - want).max()
  print("evaluate vs INTEGRATION loop: max abs score difference %.3e" % diff)
  assert diff <= EVAL_BAR
  np.testing.assert_allclose(res["mean"], ns.mean_scores(want), rtol=0, atol=EVAL_BAR)


def test_repeats_bit_identical_and_no_sync(scenes):
  _, scene = scenes["A"]
  img_i = scene.steps[1]
  a = scene.time_step(img_i)
  torch.cuda.synchronize()
  torch.cuda.set_sync_debug_mode("error")
  try:
    b = scene.time_step(img_i)
  finally:
    torch.cuda.set_sync_debug_mode(0)
  for k in ("ray_o", "ray_d", "uv_grid", "camera_index", "src_rgbs", "static_src_rgbs", "static_src_masks", "camera"):
    assert torch.equal(a["ray_batch"][k], b["ray_batch"][k]), k
  for k in ("gt_rgb", "dynamic_mask", "static_src_masked"):
    assert torch.equal(a[k], b[k]), k


def test_errors(golden, tmp_path):
  s = golden["scenes"]["A"]
  args = types.SimpleNamespace(mask_static=True)
  root = nsr.write_files(str(tmp_path / "small" / "dense"), s["files"])
  gt = os.path.join(root, "mv_images", "00005", "cam01.jpg")
  cv2.imwrite(gt, np.zeros((100, 4, 3), np.uint8))  # narrower than the 8-pixel render
  with pytest.raises(ValueError, match="smaller"):
    ns.NvidiaScene(root, args, DEV)
  os.remove(gt)
  with pytest.raises(ValueError, match="missing"):
    ns.NvidiaScene(root, args, DEV)
  root = nsr.write_files(str(tmp_path / "rgbmask" / "dense"), s["files"])
  msr.write_png(os.path.join(root, "coarse_masks", "00004.png"), np.zeros((300, 10, 3), np.uint8))
  with pytest.raises(ValueError, match="single-channel"):
    ns.NvidiaScene(root, args, DEV)
  root = nsr.write_files(str(tmp_path / "few" / "dense"), s["files"])
  arr = np.load(os.path.join(root, "poses_bounds_cvd.npy"))
  np.save(os.path.join(root, "poses_bounds_cvd.npy"), arr[:11])
  os.remove(os.path.join(root, "images_8x288", "00011.png"))
  with pytest.raises(ValueError, match="at least 12"):
    ns.NvidiaScene(root, args, DEV)
