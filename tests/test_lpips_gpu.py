"""LPIPS on the GPU (csrc/lpips.cu, dynibar_b200.metrics.lpips_views / PerceptualLoss) against the float64 restatement
(tests/lpips_ref.py), its invariants, its memory contract, and eval_nvidia.py's printed LPIPS values on the golden
scene (tests/golden/lpips_glue.pt)."""

import os
import types

import numpy as np
import pytest
import torch

import lpips_ref as lr
import memory_contract as mc
from dynibar_b200 import metrics

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lpips_glue.pt")

# (H, W, K, images, mask)
CASES = [
    (31, 31, 1, "random", "blob"),
    (31, 31, 11, "smooth", "empty"),
    (31, 47, 11, "random", "percam"),
    (47, 31, 1, "identical", "full"),
    (33, 64, 16, "smooth", "blob"),
    (33, 64, 11, "invalid", "percam"),
    (288, 512, 11, "random", "percam"),
    (288, 512, 1, "smooth", "full"),
    (288, 512, 11, "identical", "blob"),
    (540, 960, 16, "random", "blob"),
    (540, 960, 1, "smooth", "empty"),
]


@pytest.fixture(scope="module")
def weights():
  alex, lin = lr.random_weights(5)
  return alex, lin, metrics.LPIPSWeights(alex, lin, device=DEV)


def _dev(*a):
  return [torch.from_numpy(x).to(DEV) for x in a]


@pytest.mark.parametrize("H,W,K,images,mask", CASES)
def test_against_float64_reference(weights, H, W, K, images, mask):
  alex, lin, w = weights
  seed = H * 7 + W + K
  pred, gt = lr.case(images, K, H, W, seed)
  dyn = lr.mask_of(mask, K, H, W, seed)
  p, g, m = _dev(pred, gt, dyn)
  for mk in (m, None):
    got = metrics.lpips_views(p, g, mk, weights=w)
    assert got.dtype == torch.float64 and got.shape == (K, 3 if mk is not None else 1) and got.device == DEV
    want = lr.lpips(p, g, mk, alex, lin, device=DEV)
    err = (got - want).abs().max().item()
    print("\nlpips %dx%d K=%d %s/%s: max |err| %.3e (scores up to %.3f)"
          % (H, W, K, images, mask if mk is not None else "none", err, want.abs().max().item()))
    if images in ("identical", "invalid"):  # d_l == 0 everywhere
      assert torch.equal(got, torch.zeros_like(got))
    elif mask == "empty" and mk is not None:  # a row whose pooled mask sums to 0 in every tap
      assert torch.equal(got[:, 1], torch.zeros(K, dtype=torch.float64, device=DEV))
    assert err <= lr.BAR, err


def test_smallest_image(weights):
  _, _, w = weights
  for H, W in ((31, 31), (31, 200), (200, 31)):
    pred, gt = lr.case("random", 1, H, W, 1)
    metrics.lpips_views(*_dev(pred, gt), weights=w)
  for H, W in ((30, 31), (31, 30), (30, 64)):
    pred, gt = lr.case("random", 1, H, W, 1)
    with pytest.raises(ValueError, match="at least 31"):
      metrics.lpips_views(*_dev(pred, gt), weights=w)
  from dynibar_b200 import _lib
  assert _lib.lib.dyn_lpips_workspace_bytes(1, 30, 31) == 0 and _lib.lib.dyn_lpips_workspace_bytes(1, 31, 31) > 0


def test_invariants(weights):
  alex, lin, w = weights
  K, H, W = 5, 64, 96
  pred, gt = lr.case("random", K, H, W, 3)
  p, g, m = _dev(pred, gt, lr.mask_of("percam", K, H, W, 3))
  a = metrics.lpips_views(p, g, m, weights=w)
  # bit-identical repeats
  assert torch.equal(a, metrics.lpips_views(p, g, m, weights=w))
  # a camera's scores equal a call with that camera alone
  for k in range(K):
    assert torch.equal(a[k], metrics.lpips_views(p[k:k + 1], g[k:k + 1], m[k:k + 1], weights=w)[0]), k
  # symmetry in pred / gt: every pixel valid in both, so the valid mask does not change
  sp, sg = _dev(*lr.case("smooth", K, H, W, 4))
  assert torch.equal(metrics.lpips_views(sp, sg, m, weights=w), metrics.lpips_views(sg, sp, m, weights=w))
  loss = metrics.PerceptualLoss(model="net-lin", net="alex", use_gpu=True, version=0.1, alexnet=alex, lin=lin)
  x0, x1 = (sp * 2 - 1).permute(0, 3, 1, 2), (sg * 2 - 1).permute(0, 3, 1, 2)
  assert torch.equal(loss.forward(x0, x1), loss.forward(x1, x0))
  # PLAIN without a mask equals PLAIN with a ones mask
  assert torch.equal(loss.forward(x0, x1), loss.forward(x0, x1, torch.ones_like(x0)))
  # PerceptualLoss.forward on eval_nvidia.py's tensors equals lpips_views' rows, camera by camera
  valid = ((p[..., 0] + p[..., 1]) + p[..., 2] > 1e-3).float()[..., None].expand(K, H, W, 3)
  for k in range(K):
    gt0 = (g[k] * valid[k] * 2 - 1).permute(2, 0, 1)[None]
    pr0 = (p[k] * valid[k] * 2 - 1).permute(2, 0, 1)[None]
    rows = (valid[k], m[k], 1 - m[k])
    for r, mask in enumerate(rows):
      v = loss.forward(gt0, pr0, mask.permute(2, 0, 1)[None])
      assert v.shape == (1,)
      assert v.item() == a[k, r].item(), (k, r, v.item(), a[k, r].item())


@pytest.mark.parametrize("H,W,K", [(31, 45, 3), (100, 77, 2)])
def test_memory_contract(weights, H, W, K):
  alex, lin, _ = weights
  pred, gt = lr.case("random", K, H, W, H)
  dyn = lr.mask_of("percam", K, H, W, H)
  w = metrics.LPIPSWeights(alex, lin, device=DEV)  # its blob comes from torch.cat, not a poisoned allocation
  runs = {}
  for pat in mc.PATTERNS:
    with mc.poisoned(pat):
      p, g, m = _dev(pred, gt, dyn)
      out = [metrics.lpips_views(p, g, m, weights=w), metrics.lpips_views(p, g, weights=w),
             metrics.PerceptualLoss(alexnet=alex, lin=lin).forward(p.permute(0, 3, 1, 2), g.permute(0, 3, 1, 2))]
      runs["0x%02X" % pat] = mc.flatten(out)
  mc.assert_bit_identical(runs, "lpips %dx%d K=%d" % (H, W, K))


def test_golden_glue(weights, tmp_path):
  """eval_nvidia.py's printed LPIPS values on the fixture scene, from NvidiaScene's ground truth and masks plus
  lpips_views on the fixture's predictions; evaluate(..., lpips=w) keeps evaluate()'s scores bit for bit."""
  import nvi_scene_ref as nsr
  from dynibar_b200 import nvidia_scene as ns
  g = torch.load(GOLDEN, weights_only=False)
  alex, lin = lr.random_weights(int(g["weights_seed"]))
  w = metrics.LPIPSWeights(alex, lin, device=DEV)
  root = nsr.write_files(str(tmp_path / "C" / "dense"), g["files"])
  scene = ns.NvidiaScene(root, types.SimpleNamespace(mask_static=bool(g["mask_static"])), DEV)
  per, avg = g["per_camera"], g["avg"]
  got = []
  worst = 0.0
  for img_i in scene.steps:
    step = scene.time_step(img_i)
    pred = np.stack([nsr.prediction(img_i, c, scene.H, scene.W) for c in step["cameras"]])
    v = metrics.lpips_views(torch.from_numpy(pred).to(DEV), step["gt_rgb"], step["dynamic_mask"], weights=w)
    v = v.cpu().numpy()
    for k, c in enumerate(step["cameras"]):
      worst = max(worst, np.abs(v[k] - np.asarray(per[(img_i, c)])).max())
    got.append(v)
  mean = ns.mean_lpips(np.stack(got))
  print("\nlpips glue: max |err| per camera %.3e, AVG %s vs %s" % (worst, mean, avg))
  assert worst <= lr.BAR
  np.testing.assert_allclose(mean, np.asarray(avg), rtol=0, atol=lr.BAR)

  # evaluate(..., lpips=w): scores bit-identical to evaluate(...), and the LPIPS of the rendered views
  from test_nvi_scene_gpu import _model
  from dynibar_b200.projection import Projector
  model, args = _model(scene.num_frames)
  args.mask_static = bool(g["mask_static"])
  steps = scene.steps
  scene.steps = steps[:2]
  calls = []
  with torch.no_grad():
    a = scene.evaluate(model, Projector(DEV), args)
    b = scene.evaluate(model, Projector(DEV), args, on_step=lambda *x: calls.append(x), lpips=w)
  assert sorted(a) == ["mean", "scores", "steps"]
  assert np.array_equal(a["scores"], b["scores"]) and np.array_equal(a["mean"], b["mean"])
  assert b["lpips"].shape == (2, 11, 3) and b["lpips"].dtype == np.float64 and b["lpips_mean"].shape == (3,)
  assert len(calls) == 2 and calls[-1][2].shape == (2, 11, 3)
  np.testing.assert_array_equal(b["lpips_mean"], ns.mean_lpips(b["lpips"]))
