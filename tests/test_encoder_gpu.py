"""2-D feature encoder (row f1) against the reference's own ResNet (ibrnet/feature_network.py:179-311):
committed fixtures of the unmodified reference: tests/golden/encoder.pt (full maps of a small batch) and
tests/golden/live_reference.pt (make_golden_live.py: a seeded sample of positions at three image sizes)."""

import os

import pytest
import torch

import scenes
from dynibar_b200 import feature_network as fn

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = os.path.join(os.path.dirname(__file__), "golden", "encoder.pt")


def _model(seed):
  torch.manual_seed(seed)
  m = fn.ResNet()
  with torch.no_grad():  # non-trivial affine parameters / biases (defaults are 1 / 0)
    for name, p in m.named_parameters():
      if name.endswith("bn1.weight") or name.endswith("bn2.weight") or name.endswith("downsample.1.weight"):
        p.uniform_(0.5, 1.5)
      elif name.endswith(".bias"):
        p.uniform_(-0.3, 0.3)
  return m.requires_grad_(False)


def test_encoder_matches_reference_fixture():
  fx = torch.load(GOLD, weights_only=False)
  m = _model(fx["seed"])
  g = torch.Generator().manual_seed(fx["seed"] + 1)
  x = torch.rand(*fx["shape"], generator=g)
  assert abs(float(x.double().sum()) - fx["input_sum"]) < 1e-6 * fx["input_sum"]
  c, f = m.to(DEV)(x.to(DEV))
  torch.cuda.synchronize()
  assert c.shape == fx["coarse"].shape and f.shape == fx["fine"].shape
  torch.testing.assert_close(c.cpu(), fx["coarse"], rtol=2e-4, atol=2e-4)
  torch.testing.assert_close(f.cpu(), fx["fine"], rtol=2e-4, atol=2e-4)


@pytest.mark.parametrize("N,H,W", [(2, 288, 512), (3, 37, 53), (1, 135 * 4 // 4, 240)])
def test_encoder_matches_live_reference(N, H, W):
  from golden import make_golden_live as ml
  fx = torch.load(os.path.join(os.path.dirname(GOLD), "live_reference.pt"), weights_only=False)["encoder"][(N, H, W)]
  m = scenes.encoder_weights(fn.ResNet(), N * 1000 + H)
  x = ml.encoder_input(N, H, W)
  assert abs(float(x.double().sum()) - fx["input_sum"]) < 1e-6 * fx["input_sum"]
  c, f = m.to(DEV)(x.to(DEV))
  torch.cuda.synchronize()
  assert tuple(c.shape) == fx["shape"] and tuple(f.shape) == fx["shape"]
  idx = ml.encoder_sample(c.numel(), N, H)
  torch.testing.assert_close(c.cpu().flatten()[idx], fx["coarse"], rtol=2e-4, atol=2e-4)
  torch.testing.assert_close(f.cpu().flatten()[idx], fx["fine"], rtol=2e-4, atol=2e-4)


def test_encoder_feeds_the_renderer_layout():
  """[V,3,H,W] images -> [V,32,H/4,W/4] maps, the `featmaps` layout render_rays_* take."""
  m = _model(1).to(DEV)
  c, f = m(torch.rand(8, 3, 288, 512, device=DEV))
  assert c.shape == (8, 32, 72, 128) and f.shape == (8, 32, 72, 128) and torch.isfinite(c).all()


@pytest.mark.parametrize("N,H,W,prec", [(2, 60, 84, "fp32"), (3, 37, 53, "fp32"), (2, 192, 256, "bf16")])
def test_encoder_backward_matches_oracle_autograd(N, H, W, prec):
  """Row f2: gradients of every executed encoder parameter.  fp32: against torch autograd through the oracle's
  restatement of ResNet.forward (pinned to the reference by tests/test_oracle_golden.py), 2e-3 relative L2 per tensor
  (InstanceNorm + ReLU network; the ReLU kinks make a few units flip with the summation order).  bf16 (every product
  on the tensor cores at this shape): against tests/encoder_ref.py in mode "kernel", which rounds the operands of
  exactly those products to bf16, with its per-tensor bf16 bars (tests/test_encoder_train_gpu.py says how they were
  measured)."""
  import encoder_ref as er
  from dynibar_b200 import render_ray as rr
  from oracle import dynibar_oracle as orc
  m = _model(N * 100 + H).requires_grad_(True)
  g = torch.Generator().manual_seed(N + H)
  x = torch.rand(N, 3, H, W, generator=g)
  w = {k: v.detach().clone().requires_grad_(True) for k, v in m.state_dict().items() if k in fn._EXECUTED}
  wc, wf = orc.encoder_forward(w, x)
  gc, gf = torch.randn(wc.shape, generator=g), torch.randn(wf.shape, generator=g)
  ((wc * gc).sum() + (wf * gf).sum()).backward()
  ref = None
  if prec == "bf16":
    ref = er.reference(dict(mod=m, x=x, gc=gc, gf=gf), DEV, "kernel")
  md = m.to(DEV)
  with rr.precision_scope(prec):
    c, f = md(x.to(DEV))
    assert c.requires_grad and f.requires_grad
    ((c * gc.to(DEV)).sum() + (f * gf.to(DEV)).sum()).backward()
  torch.testing.assert_close(c.detach().cpu(), wc.detach(), rtol=2e-4, atol=2e-4)
  sd = md.state_dict(keep_vars=True)
  for k in fn._EXECUTED:
    assert sd[k].grad is not None, k
  if prec == "bf16":
    got = {k: sd[k].grad for k in fn._EXECUTED}
    ref = {k: ref[k] for k in fn._EXECUTED}
    r = er.ratios("bf16", got, ref)
    print("\nbf16 encoder backward %dx%dx%d: worst %s, %.2f of its bar" % (N, H, W, *max(r.items(), key=lambda kv: kv[1])))
    bad = {k: er.errors(got, ref)[k] for k, v in r.items() if not v <= 1.0}
    assert not bad, bad
  else:
    for k in fn._EXECUTED:
      d = (sd[k].grad.cpu().double() - w[k].grad.double()).norm().item()
      assert d <= 2e-3 * w[k].grad.double().norm().item() + 1e-6, (k, d, w[k].grad.norm().item())
  for k, p in md.named_parameters():  # parameters the reference builds but never runs get no gradient
    if k not in fn._EXECUTED:
      assert p.grad is None, k
