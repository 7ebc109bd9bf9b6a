"""Backward kernels of the first f2 slice against torch autograd through the oracle's restatement of the same
reference functions (compute_with_motions projection.py:103-176; the MotionMLP).  Compositing forward and
backward are checked element by element against a float64 reference in test_geometry_stage_gpu.py."""

import pytest
import torch

import scenes
from dynibar_b200 import synthetic
from oracle import dynibar_oracle as orc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("name", ["mv_linear", "mono_train"])
def test_project_gather_backward_matches_oracle_autograd(golden, name):
  from dynibar_b200 import autograd as ag
  fx = golden(name)
  cfg, st = fx["cfg"], fx["stages"]
  batch, feat_c, feat_f, frame, t, offs, model, args = scenes.build(cfg)
  pts, seq = st["pts"], st["seq"]
  fm = feat_c[0]
  # oracle (CPU, torch autograd through grid_sample)
  fo, so = fm.clone().requires_grad_(True), seq.clone().requires_grad_(True)
  want_f, _, want_m = orc.project_gather(pts, so, batch["camera"], batch["src_rgbs"], batch["src_cameras"], fo)
  g = torch.randn_like(want_f)
  (want_f * g).sum().backward()
  fd, sd = fm.to(DEV).requires_grad_(True), seq.to(DEV).requires_grad_(True)
  d = lambda x: synthetic.to_device(x, DEV)
  got_f, got_rd, got_m = ag.project_gather(d(pts), sd, d(batch["camera"]), d(batch["src_rgbs"]),
                                            d(batch["src_cameras"]), fd)
  assert not got_rd.requires_grad and not got_m.requires_grad
  (got_f * g.to(DEV)).sum().backward()
  torch.testing.assert_close(fd.grad.cpu(), fo.grad, rtol=2e-4, atol=2e-4)
  # d/d xyz: compare where the sample is inside the image (the in-bounds edge is a kink of the zero-padded bilinear)
  inb = (want_m[..., 0] > 0).permute(2, 0, 1)  # [V,R,S]
  gx, wx = sd.grad.cpu()[inb], so.grad[inb]
  bad = ((gx - wx).abs() > 1e-3 + 1e-3 * wx.abs()).float().mean().item()
  assert bad < 2e-3, bad


@pytest.mark.parametrize("N,nb,tol", [(300, 6, 1e-3), (5000, 4, 1e-2)])
def test_motion_mlp_backward_matches_oracle_autograd(N, nb, tol):
  """MotionMLP (mlp_network.py:605-618): coefficients, d/d(every parameter) and d/d(xyzt) against autograd through
  the oracle's restatement (in float64); 5000 rows exercise the split-K accumulation of the weight gradients.
  Bar: 1e-3 relative in the L2 norm per tensor (max-abs: 5x that of the largest entry) on 300 rows.  A
  pre-activation within rounding distance of 0 can take the other side of the ReLU kink on the GPU (different
  summation order); with random upstream gradients one row is ~1/sqrt(N) of a gradient's norm, so each such flip
  moves a tensor by ~1e-3 relative.  The 5000-row case (about ten expected flips in 10 M activations) therefore
  uses 1e-2: a wrong or missing split-K partial sum would be an O(1) error."""
  from dynibar_b200 import autograd as ag, mlp_network as nets
  torch.manual_seed(N)
  mod = nets.MotionMLP(num_basis=nb)
  with torch.no_grad():  # the shipped init zeroes coeff_linear (mlp_network.py:602-603)
    mod.coeff_linear.weight.normal_(0, 0.05)
    mod.coeff_linear.bias.normal_(0, 0.05)
  xyzt = torch.cat([torch.randn(N, 3) * 2, torch.rand(N, 1)], -1)
  gen = torch.randn(N, 3 * nb)
  # ---- oracle + torch autograd (CPU, fp32) ----
  w = {k: v.detach().clone().double().requires_grad_(True) for k, v in mod.state_dict().items()}
  xo = xyzt.clone().double().requires_grad_(True)
  want = orc.motion_mlp(w, xo)
  (want * gen.double()).sum().backward()
  want = want.float()
  # ---- library ----
  mod = mod.to(DEV)
  xd = xyzt.to(DEV).requires_grad_(True)
  got = ag.motion_mlp(mod, xd, precision="fp32")
  torch.testing.assert_close(got.detach().cpu(), want.detach(), rtol=1e-4, atol=1e-5)
  (got * gen.to(DEV)).sum().backward()
  def close(name, got_t, ref):
    d = got_t.detach().cpu().double() - ref
    assert d.norm().item() <= tol * ref.norm().item() + 1e-12, (name, d.norm().item(), ref.norm().item())
    assert d.abs().max().item() <= 5 * tol * ref.abs().max().item() + 1e-12, (name, d.abs().max().item())
  for k, p in mod.named_parameters():
    close(k, p.grad, w[k].grad)
  close("xyzt", xd.grad, xo.grad)
