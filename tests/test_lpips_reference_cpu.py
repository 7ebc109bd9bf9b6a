"""The float64 LPIPS restatement (tests/lpips_ref.py) on the CPU: its taps against torchvision's AlexNet, the
unmasked case against the published spatial mean, planted errors that the GPU bar would catch, and LPIPSWeights'
argument checks."""

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import lpips_ref as lr


@pytest.fixture(scope="module")
def weights():
  return lr.random_weights(5)


def test_taps_equal_torchvision_alexnet(weights):
  tv = pytest.importorskip("torchvision")
  alex, _ = weights
  net = tv.models.alexnet(weights=None).double()
  net.load_state_dict({k: v.double() for k, v in alex.items() if k.startswith("features.")}, strict=False)
  x = torch.randn(2, 3, 67, 93, dtype=torch.float64, generator=torch.Generator().manual_seed(1))
  got = lr.taps(x, alex)
  # LPIPS v0.1's alexnet slices: features[0:2], [2:5], [5:8], [8:10], [10:12]
  want, h = [], x
  for a, b in ((0, 2), (2, 5), (5, 8), (8, 10), (10, 12)):
    h = net.features[a:b](h)
    want.append(h)
  for g, w in zip(got, want):
    assert g.shape == w.shape
    torch.testing.assert_close(g, w, rtol=0, atol=1e-12)


def test_tap_sizes_and_smallest_image(weights):
  alex, lin = weights
  f = lr.taps(torch.zeros(1, 3, 288, 512, dtype=torch.float64), alex)
  assert [tuple(t.shape[2:]) for t in f] == [(71, 127), (35, 63), (17, 31), (17, 31), (17, 31)]
  # 31 is the smallest side: conv1 -> 7, pool -> 3, conv2 -> 3, pool -> 1; at 30 the second pool has no output
  f = lr.taps(torch.zeros(1, 3, 31, 31, dtype=torch.float64), alex)
  assert [tuple(t.shape[2:]) for t in f] == [(7, 7), (3, 3), (1, 1), (1, 1), (1, 1)]
  with pytest.raises(RuntimeError):
    lr.taps(torch.zeros(1, 3, 30, 40, dtype=torch.float64), alex)
  with pytest.raises(RuntimeError):
    lr.taps(torch.zeros(1, 3, 40, 30, dtype=torch.float64), alex)


def test_ones_mask_is_the_spatial_mean(weights):
  alex, lin = weights
  pred, gt = lr.case("smooth", 2, 40, 52, seed=3)

  def published(a, b):  # LPIPS v0.1: spatial average per tap, summed
    f0 = lr.taps(lr.scale_images(a, False, None), alex)
    f1 = lr.taps(lr.scale_images(b, False, None), alex)
    return sum(dl.mean((1, 2)) for dl in lr.tap_distances(f0, f1, lin))

  p1, g1 = pred * 2 - 1, gt * 2 - 1  # float32, as PerceptualLoss receives them
  want = published(torch.from_numpy(p1).double(), torch.from_numpy(g1).double())
  torch.testing.assert_close(lr.lpips(p1, g1, None, alex, lin, mode="plain")[:, 0], want, rtol=1e-14, atol=0)
  ones = lr.lpips(p1, g1, np.ones_like(pred), alex, lin, mode="plain")[:, 0]
  torch.testing.assert_close(ones, want, rtol=1e-14, atol=0)
  # EVAL with every pixel valid: the full row is the published value on 2x - 1
  want = published(torch.from_numpy(pred).double() * 2 - 1, torch.from_numpy(gt).double() * 2 - 1)
  torch.testing.assert_close(lr.lpips(pred, gt, None, alex, lin)[:, 0], want, rtol=1e-14, atol=0)


@pytest.mark.parametrize("plant", lr.PLANTS)
def test_planted_errors_miss_the_bar(plant):
  # pad 0 needs a larger image for conv5 to keep an output; the eps plant needs taps small against 1e-10
  H, W = (200, 232) if plant == "pad0" else (64, 80)
  alex, lin = lr.random_weights(5, scale=1e-6 if plant == "eps_in_sqrt" else 1.0)
  pred, gt = lr.case("random", 2, H, W, seed=11)
  mask = lr.mask_of("blob", 2, H, W, seed=11)
  want = lr.lpips(pred, gt, mask, alex, lin)
  got = lr.lpips(pred, gt, mask, alex, lin, plant=plant)
  miss = (got - want).abs().max().item()
  print("%s: max |score difference| %.3e = %.0f bars" % (plant, miss, miss / lr.BAR))
  assert miss >= lr.PLANT_MARGIN * lr.BAR, (plant, miss)


def test_weights_rejects_bad_dicts(weights):
  from dynibar_b200 import metrics
  alex, lin = weights
  bad = []
  a = dict(alex)
  del a["features.6.bias"]
  bad.append((a, lin, "no features.6.bias"))
  a = dict(alex, **{"features.3.weight": torch.zeros(192, 64, 3, 3)})
  bad.append((a, lin, "features.3.weight"))
  l = dict(lin)
  del l["lin4.model.1.weight"]
  bad.append((alex, l, "no lin4"))
  l = dict(lin, **{"lin2.model.1.weight": torch.zeros(384)})
  bad.append((alex, l, "lin2.model.1.weight"))
  l = dict(lin, **{"lin1.model.1.weight": -lin["lin1.model.1.weight"]})
  bad.append((alex, l, "negative"))
  bad.append(([1, 2], lin, "path or a state dict"))
  for a, l, msg in bad:
    with pytest.raises(ValueError, match=msg):
      metrics.LPIPSWeights(a, l, device="cpu")
