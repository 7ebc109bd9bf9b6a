"""The view-scoring kernels (csrc/metrics.cu, dynibar_b200.metrics) on the GPU: the SSIM map against the float32
restatement through scipy and the float64 one (tests/metrics_ref.py), the scores against eval_nvidia.py's glue
restated on the same inputs and against the reference's own calculate_psnr / calculate_ssim
(tests/golden/eval_metrics.pt), bit-reproducibility across batch sizes and repeats, the drop-ins' input kinds,
argument errors, and one rendered time step.  Bars: tests/metrics_ref.py BARS, stated in DESIGN §3.6."""

import numpy as np
import pytest
import torch

import metrics_ref as mr
from dynibar_b200 import _lib
from dynibar_b200 import metrics

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _report(name, value):
  print("\n[metrics] %s = %.3e" % (name, value), end="")


def _smap(x, y):
  """S [H, W, 3] of the kernel (plain mode, the test hook)."""
  a, b = torch.from_numpy(x)[None].to(DEV), torch.from_numpy(y)[None].to(DEV)
  S = torch.empty_like(a)
  metrics._scores(a, b, None, _lib.SCORES_PLAIN, ssim_map=S)
  return S[0].cpu().numpy()


@pytest.mark.parametrize("kind,H,W", [("random", 64, 80), ("smooth", 64, 80), ("constant", 40, 48),
                                      ("identical", 40, 48), ("binary", 64, 80), ("random", 7, 7),
                                      ("random", 7, 513), ("random", 8, 9), ("random", 289, 513),
                                      ("smooth", 288, 512), ("random", 540, 960)])
def test_ssim_map_matches_restatements(kind, H, W):
  x, y = mr.pair(kind, H, W, seed=H + W)
  got = _smap(x, y)
  want32 = mr.ssim_map32(x, y)
  e32 = float(np.abs(got - want32).max())
  e64 = float(np.abs(got - mr.ssim_map64(x, y)).max())
  n_diff = int((got != want32).sum())
  _report("S map[%s %dx%d] vs ssim_map32 max abs err (%d of %d elements differ)" % (kind, H, W, n_diff, got.size), e32)
  _report("S map[%s %dx%d] vs ssim_map64 max abs err" % (kind, H, W), e64)
  assert np.isfinite(got).all()
  assert e32 <= mr.BARS["smap32"] and e64 <= mr.BARS["smap64"], (e32, e64)
  if kind == "identical":
    assert (got == 1).all()


def _check_views(pred, gt, dyn, tag):
  got = metrics.score_views(torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV),
                            None if dyn is None else torch.from_numpy(dyn).to(DEV))
  assert got.is_cuda and got.dtype == torch.float64
  assert tuple(got.shape) == (pred.shape[0], 1 if dyn is None else 3, 2)
  got = got.cpu().numpy()
  err = 0.0
  for k in range(pred.shape[0]):
    want = mr.eval_scores(pred[k], gt[k], None if dyn is None else dyn[k])
    err = max(err, float(np.abs(got[k] - want).max()))
  _report("scores[%s] vs restatement max abs err" % tag, err)
  assert err <= mr.BARS["score"], err
  return got


@pytest.mark.parametrize("K", [1, 3, 11, 16, 17])
def test_scores_match_restatement(K):
  pred, gt, dyn = mr.eval_case(K, 40, 56, seed=K)
  _check_views(pred, gt, dyn, "K=%d blobs" % K)


@pytest.mark.parametrize("mask_kind", ["blobs", "empty", "full", "per_channel", None])
def test_scores_match_restatement_per_mask(mask_kind):
  pred, gt, dyn = mr.eval_case(3, 45, 71, seed=7, mask_kind=mask_kind or "blobs")
  got = _check_views(pred, gt, None if mask_kind is None else dyn, "mask %s" % mask_kind)
  if mask_kind == "empty":  # no dynamic pixels: mse 0 -> PSNR 0, SSIM 0
    assert (got[:, 1] == 0).all()


def test_scores_match_restatement_at_eval_size():
  pred, gt, dyn = mr.eval_case(11, 288, 512, seed=1)
  _check_views(pred, gt, dyn, "K=11 288x512")


def test_valid_threshold_is_strict_and_float32():
  """Pixels whose float32 channel sum is exactly float32(1e-3) are invalid; its float32 neighbour above is valid."""
  H, W = 16, 20
  eps = np.float32(1e-3)
  pred = np.full((1, H, W, 3), 0.5, np.float32)
  gt = np.full((1, H, W, 3), 0.25, np.float32)
  pred[0, :, :W // 2] = 0
  pred[0, :4, :W // 2, 1] = eps
  pred[0, 4:8, :W // 2, 2] = np.nextafter(eps, np.float32(1))
  pred[0, 8:12, :W // 2, 0] = np.nextafter(eps, np.float32(0))
  got = _check_views(pred, gt, None, "threshold")
  # the case tells a >= threshold apart from the > one
  assert np.abs(mr.eval_scores(pred[0], gt[0], plant="valid_ge") - got[0]).max() > 3 * mr.BARS["score"]


def test_drop_ins_match_the_reference_fixture(golden):
  fx = golden("eval_metrics")
  err = 0.0
  for c in fx["cases"]:
    a, b, m = c["img1"].numpy(), c["img2"].numpy(), c["mask"].numpy()
    psnr, ssim = metrics.calculate_psnr(a, b, m), metrics.calculate_ssim(a, b, m)
    assert isinstance(psnr, float) and isinstance(ssim, float)
    err = max(err, abs(psnr - c["psnr"]), abs(ssim - c["ssim"]))
    if c["psnr"] == 0.0:
      assert psnr == 0.0, c["name"]
  _report("drop-ins vs eval_metrics.pt max abs err", err)
  assert err <= mr.BARS["fixture"], err


def test_drop_ins_accept_numpy_cpu_and_cuda_inputs():
  x, y = mr.pair("random", 23, 37, seed=4)
  m = mr.blobs(23, 37, np.random.default_rng(4))
  want = (metrics.calculate_psnr(x, y, m), metrics.calculate_ssim(x, y, m))
  variants = [
      (torch.from_numpy(x), torch.from_numpy(y), torch.from_numpy(m)),
      (torch.from_numpy(x).to(DEV), torch.from_numpy(y).to(DEV), torch.from_numpy(m).to(DEV)),
      (x, y, m[..., 0]), (x, y, m[..., :1]), (x, y, m[..., 0] > 0.5),
      (x.astype(np.float64), y, m.astype(np.float64)),
      (np.asfortranarray(x), y[:, :, ::-1][:, :, ::-1], m),
  ]
  for a, b, w in variants:
    assert (metrics.calculate_psnr(a, b, w), metrics.calculate_ssim(a, b, w)) == want
  err = max(abs(want[0] - mr.calculate_psnr(x, y, m)), abs(want[1] - mr.ssim_score64(mr.ssim_map32(x, y), m)))
  _report("drop-ins vs restatement max abs err", err)
  assert err <= mr.BARS["score"], err


def test_batched_equals_single_camera_and_repeats_are_bit_identical():
  pred, gt, dyn = mr.eval_case(17, 45, 71, seed=2, mask_kind="per_channel")
  p, g, d = (torch.from_numpy(a).to(DEV) for a in (pred, gt, dyn))
  batched = metrics.score_views(p, g, d)
  assert torch.equal(batched, metrics.score_views(p, g, d))
  for k in range(17):
    assert torch.equal(batched[k:k + 1], metrics.score_views(p[k:k + 1], g[k:k + 1], d[k:k + 1])), k
  # host inputs, a [K, H, W] bool mask and a CPU tensor give the same bits
  assert torch.equal(batched, metrics.score_views(pred, gt, torch.from_numpy(dyn)))
  blob = mr.eval_case(4, 45, 71, seed=2)[2]
  a = metrics.score_views(pred[:4], gt[:4], blob[..., 0] > 0.5)
  assert torch.equal(a, metrics.score_views(p[:4], g[:4], torch.from_numpy(blob).to(DEV)))
  x, y = mr.pair("random", 289, 513, seed=1)
  assert np.array_equal(_smap(x, y), _smap(x, y))


def test_argument_errors():
  x = torch.zeros(1, 8, 9, 3, device=DEV)
  S = torch.empty(1, 8, 9, 3, device=DEV)
  sc = torch.empty(1, 1, 2, dtype=torch.float64, device=DEV)
  ws = torch.empty(16, dtype=torch.uint8, device=DEV)
  rc = _lib.lib.dyn_image_scores(x.data_ptr(), x.data_ptr(), None, 1, 8, 9, 0, sc.data_ptr(), S.data_ptr(),
                                 ws.data_ptr(), ws.numel(), _lib.stream())
  assert rc == -3 and b"workspace" in _lib.lib.dyn_last_error()
  rc = _lib.lib.dyn_image_scores(x.data_ptr(), x.data_ptr(), None, 1, 8, 9, 7, sc.data_ptr(), S.data_ptr(),
                                 ws.data_ptr(), 1 << 20, _lib.stream())
  assert rc == -1
  with pytest.raises(TypeError):
    metrics.score_views(x.to(torch.uint8), x)
  with pytest.raises(ValueError, match="win_size"):
    metrics.calculate_psnr(x[0, :6], x[0, :6], x[0, :6])
  with pytest.raises(ValueError):
    metrics.score_views(x, x[:, :, :8])


def test_scores_a_rendered_time_step():
  """Two target cameras rendered in one render_multi_image_nvi call, scored by score_views, against the restatement
  on the host copies."""
  import scenes
  from dynibar_b200 import sample_ray as sr
  from dynibar_b200 import synthetic
  from dynibar_b200.projection import Projector
  from dynibar_b200.render_image import render_multi_image_nvi
  H, W = 24, 40
  cfg = dict(scenes.GOLDEN_CONFIGS["mv_small"], H=H, W=W, V_st=5, rays=None, seed=21, stress=False)
  batch, feat_c, feat_f, frame, t, offs, model, args = scenes.build(cfg)
  data = scenes.sampler_data(batch, H, W, cfg["seed"])
  K_mat = sr.parse_camera(batch["camera"])[2][0]
  samplers = []
  for off in ((0.0, 0.0, 0.0), (0.045, 0.012, -0.02)):
    c2w = torch.eye(4)
    c2w[:3, 3] = torch.tensor(off)
    samplers.append(sr.RaySamplerSingleImage(dict(data, camera=synthetic.camera_vector(H, W, K_mat, c2w)[None]), DEV))
  rays, _, _ = sr.stack_ray_batches([smp.get_all() for smp in samplers])
  dev = lambda v: synthetic.to_device(v, DEV)
  with torch.no_grad():
    out = render_multi_image_nvi(frame, t, offs, samplers, rays, synthetic.model_to(model, DEV), Projector(DEV), 1000,
                                 cfg["N_samples"], args, inv_uniform=cfg["inv_uniform"],
                                 N_importance=cfg["N_importance"], det=True, coarse_featmaps=dev(feat_c),
                                 fine_featmaps=dev(feat_f), is_train=False)
  pred = torch.stack([o["outputs_fine_ref"]["rgb"] for o in out])
  assert tuple(pred.shape) == (2, H, W, 3)
  rng = np.random.default_rng(0)
  gt = np.clip(pred.numpy() + np.float32(0.05) * rng.standard_normal(pred.shape, dtype=np.float32), 0, 1)
  dyn = np.stack([mr.blobs(H, W, rng) for _ in range(2)])
  got = metrics.score_views(pred, gt, dyn).cpu().numpy()
  err = max(float(np.abs(got[k] - mr.eval_scores(pred[k].numpy(), gt[k], dyn[k])).max()) for k in range(2))
  _report("rendered time step scores vs restatement max abs err", err)
  assert err <= mr.BARS["score"], err
